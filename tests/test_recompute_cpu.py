"""The host side of training with recomputed activations (DESIGN.md §3.12): the constructor flag, the CLIs' --recompute,
and the training set's byte count in each mode against DESIGN.md's table."""
import os
import re
import sys

import pytest

from progen_b200 import ProGen
from progen_b200.engine import training_set

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
TINY = dict(num_tokens=256, dim=128, seq_len=128, depth=2, window_size=64, heads=2, dim_head=64, global_mlp_depth=1)


def test_constructor_flag_is_not_part_of_the_config():
    m = ProGen(**TINY, recompute=True)
    assert m.recompute is True and 'recompute' not in m.config
    assert ProGen(**TINY).recompute is False
    m.recompute = False                                  # before the engine exists: only the flag changes
    assert m.recompute is False and m._engine is None


class _Stop(Exception):
    pass


def _stand_in(seen):
    """a ProGen stand-in that records its keywords and stops the CLI before any device work"""
    def make(**kw):
        seen.append(kw)
        raise _Stop
    return make


def _base_checkpoint(path):
    from progen_b200.checkpoint import get_checkpoint_fns
    get_checkpoint_fns(path)[2]({'next_seq_index': 0, 'params': ProGen(**TINY).init(0), 'optim_state': None,
                                 'model_config': dict(TINY), 'run_id': None})


@pytest.mark.parametrize('flag', [False, True])
def test_clis_pass_recompute_to_the_constructor(tmp_path, monkeypatch, flag):
    import toml
    from click.testing import CliRunner
    import dpo
    import fitness
    import train
    seen = []
    extra = ['--recompute'] if flag else []
    (tmp_path / 'tiny.toml').write_text(toml.dumps(TINY))
    base = tmp_path / 'base'
    _base_checkpoint(base)
    (tmp_path / 'pairs.tsv').write_text('MKV\tMKL\n')
    (tmp_path / 'train.tsv').write_text('MKVLA\t0.5\nMKLLA\t0.25\n')
    calls = [
        (train, train.main, ['--config_path', str(tmp_path), '--model_name', 'tiny', '--synthetic',
                             '--checkpoint_path', str(tmp_path / 'ck')]),
        (dpo, dpo.main, ['--init_checkpoint', str(base), '--pairs', str(tmp_path / 'pairs.tsv'),
                         '--checkpoint_path', str(tmp_path / 'dpo')]),
        (fitness, fitness.train, ['--init_checkpoint', str(base), '--train', str(tmp_path / 'train.tsv'), '--task',
                                  'regression', '--lora_rank', '8', '--checkpoint_path', str(tmp_path / 'fit')]),
    ]
    for mod, cmd, args in calls:
        monkeypatch.setattr(mod, 'ProGen', _stand_in(seen))
        res = CliRunner().invoke(cmd, args + extra)
        assert isinstance(res.exception, _Stop), (mod.__name__, res.output, res.exception)
        kw = seen.pop()
        assert kw['recompute'] is flag, mod.__name__
        assert {k: v for k, v in kw.items() if k not in ('recompute', 'mixed_precision')} == TINY, mod.__name__


def _design_table():
    """DESIGN.md §3.12's byte table: {(config, B): (resident bytes, recompute bytes)}"""
    text = open(os.path.join(ROOT, 'DESIGN.md')).read()
    sec = text[text.index('### 3.12'):]
    sec = sec[:sec.index('\n### ', 1)] if '\n### ' in sec[1:] else sec
    out = {}
    for m in re.finditer(r'^\| (cfg\d) \| (\d+) \| ([\d ]+) \| ([\d ]+) \|', sec, re.M):
        out[(m.group(1), int(m.group(2)))] = (int(m.group(3).replace(' ', '')), int(m.group(4).replace(' ', '')))
    return out


def test_training_set_bytes_match_the_design_table():
    from bench import CONFIGS
    table = _design_table()
    assert {('cfg2', 64), ('cfg3', 8), ('cfg4', 4), ('cfg4', 8), ('cfg4', 16)} <= set(table), table
    for (name, B), (resident, recomputed) in table.items():
        cfg = ProGen(**CONFIGS[name]['kwargs']).config
        assert training_set(cfg, B, True, False)[1] == resident, (name, B)
        assert training_set(cfg, B, True, True)[1] == recomputed, (name, B)


@pytest.mark.parametrize('kw', [TINY, dict(TINY, ff_glu=False), dict(TINY, global_mlp_depth=0), dict(TINY, depth=4)])
def test_recompute_set_aliases(kw):
    """one checkpoint per layer input, one shared attention output, one scratch per layer kind over one storage; the
    resident set has distinct buffers everywhere"""
    cfg = ProGen(**kw).config
    nl = cfg['depth']
    r, _ = training_set(cfg, 2, True, False)
    c, _ = training_set(cfg, 2, True, True)
    assert len({id(x) for x in r['X']}) == 2 * nl + 1 and len({id(s) for s in r['lay']}) == nl
    assert len({id(x) for x in c['X'][0::2]}) == nl + 1 and len({id(x) for x in c['X'][1::2]}) == 1
    kinds = [s.get('gn') is not None for s in c['lay']]
    for i in range(nl):
        j = kinds.index(kinds[i])
        assert c['lay'][i] is c['lay'][j]
        assert {k: tuple(v.shape) for k, v in c['lay'][i].items()} == {k: tuple(v.shape) for k, v in r['lay'][i].items()}
    assert set(c) == set(r)
    for k in c:
        if k not in ('X', 'lay'):
            assert tuple(c[k].shape) == tuple(r[k].shape) and c[k].dtype == r[k].dtype, k
