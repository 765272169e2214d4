"""Low-rank adapters without a GPU: the adapter tree's shapes per layer kind, argument and tree validation, the float64
merge, the GLU column interleave of the engine layout, checkpoint package resolution, and train.py refusing flags that
would change a resumed run."""
import os
import sys

import numpy as np
import pytest

from progen_b200 import ProGen
from progen_b200 import lib as L
from progen_b200.engine import P
from progen_b200.lora import adapter_modules, build_adapter_specs, merge_adapters

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CFG = dict(num_tokens=64, dim=64, seq_len=64, depth=3, window_size=32, global_mlp_depth=1, heads=2, dim_head=32)


def test_tree_shapes_per_layer_kind():
    for ff_glu, kinds in ((True, ('glu', 'glu', 'sgu')), (False, ('gelu', 'gelu', 'sgu'))):
        m = ProGen(**CFG, ff_glu=ff_glu)
        ad = m.init_adapters(0, 16)
        assert len(ad) == 4 * CFG['depth']
        d, inner, hid = 64, 64, 256
        for i, kind in enumerate(kinds):
            a, f = P + f'attn{i}/~/', P + f'ff{i}/~/'
            h_in = 2 * hid if kind == 'glu' else hid
            h_out = hid // 2 if kind == 'sgu' else hid
            for mod, fin, fout in ((a + 'linear', d, 3 * inner), (a + 'linear_1', inner, d), (f + 'linear', d, h_in),
                                   (f + 'linear_1', h_out, d)):
                assert ad[mod]['lora_a'].shape == (fin, 16) and ad[mod]['lora_b'].shape == (16, fout)
                assert not ad[mod]['lora_b'].any()
                assert ad[mod]['lora_a'].dtype == np.float32
                assert np.abs(ad[mod]['lora_a']).max() <= 2.0 * fin ** -0.5 + 1e-7
                # the adapted weight has the base weight's shape
                assert m.param_shapes()[mod]['w'] == (fin, fout)
    a1, a2 = ProGen(**CFG).init_adapters(3, 8), ProGen(**CFG).init_adapters(3, 8)
    assert all(np.array_equal(a1[k]['lora_a'], a2[k]['lora_a']) for k in a1)


@pytest.mark.parametrize('rank', [0, 4, 12, 72, 16.0, True, '16'])
def test_bad_rank_raises(rank):
    with pytest.raises(L.ProgenError, match='rank'):
        ProGen(**CFG).init_adapters(0, rank)


@pytest.mark.parametrize('alpha', [0, -1.0, float('nan'), float('inf'), 'x'])
def test_bad_alpha_raises(alpha):
    with pytest.raises(L.ProgenError, match='lora_alpha'):
        ProGen(**CFG).init_adapters(0, 8, alpha=alpha)


def test_tree_validation_names_the_leaf():
    m = ProGen(**CFG)
    params = m.init(0)
    good = m.init_adapters(0, 8)
    mod = P + 'ff1/~/linear'

    def broken(fn):
        ad = {k: dict(v) for k, v in good.items()}
        fn(ad)
        return ad

    cases = [
        (lambda ad: ad.pop(mod), 'missing module ' + mod),
        (lambda ad: ad.__setitem__(P + 'linear', {'lora_a': np.zeros((64, 8)), 'lora_b': np.zeros((8, 64))}), 'unexpected module'),
        (lambda ad: ad[mod].pop('lora_b'), mod),
        (lambda ad: ad[mod].__setitem__('lora_c', 0), mod),
        (lambda ad: ad[mod].__setitem__('lora_b', np.zeros((8, 7), np.float32)), mod + '/lora_b'),
        (lambda ad: ad[mod].__setitem__('lora_a', np.zeros((64,), np.float32)), mod + '/lora_a'),
        (lambda ad: ad[mod].__setitem__('lora_a', np.zeros((64, 16), np.float32)), mod + '/lora_a'),
        (lambda ad: ad[mod].__setitem__('lora_b', np.full((8, 512), np.nan, np.float32)), mod + '/lora_b'),
    ]
    for fn, msg in cases:
        with pytest.raises(L.ProgenError, match=msg.replace('/', '.').replace('~', '.')):
            m.merge_adapters(params, broken(fn))
    mixed = {k: {'lora_a': np.zeros((v['lora_a'].shape[0], 16), np.float32), 'lora_b': np.zeros((16, v['lora_b'].shape[1]), np.float32)}
             for k, v in good.items()}
    mixed[mod] = good[mod]
    with pytest.raises(L.ProgenError, match='rank'):
        m.merge_adapters(params, mixed)
    with pytest.raises(L.ProgenError, match='lora_alpha'):
        m.merge_adapters(params, good, lora_alpha=0.0)


def test_merge_matches_float64():
    m = ProGen(**CFG)
    params = m.init(1)
    rng = np.random.default_rng(2)
    ad = m.init_adapters(1, 16)
    for v in ad.values():
        v['lora_b'] = rng.standard_normal(v['lora_b'].shape).astype(np.float32)
    merged = m.merge_adapters(params, ad, lora_alpha=4.0)
    for mod, leaves in merged.items():
        for name, a in leaves.items():
            if mod in ad and name == 'w':
                want = (params[mod]['w'].astype(np.float64) + 0.25 * ad[mod]['lora_a'].astype(np.float64)
                        @ ad[mod]['lora_b'].astype(np.float64)).astype(np.float32)
                assert a.dtype == np.float32 and np.array_equal(a, want), mod
            else:
                assert a is params[mod][name]
    # B = 0: the merge is the base
    base = m.merge_adapters(params, m.init_adapters(5, 8))
    assert all(np.array_equal(base[k]['w'], params[k]['w']) for k in ad)


def test_glu_interleave_round_trip():
    """Engine layout of the adapter buffer: every A, then every B, on 64-element boundaries; a GLU feed-forward input's
    B is interleaved (value_j, gate_j) like the base weight, and the export gives the haiku order back."""
    from progen_b200.engine import _deinterleave, _interleave
    cfg = ProGen(**CFG).config
    specs, n, n_a = build_adapter_specs(cfg, 8)
    assert [s.name for s in specs] == ['lora_a'] * (len(specs) // 2) + ['lora_b'] * (len(specs) // 2)
    assert all(s.offset % 64 == 0 for s in specs) and n % 64 == 0 and n_a == specs[len(specs) // 2].offset
    assert all(s.decay for s in specs)
    glu = {m for m, _, _, g in adapter_modules(cfg) if g}
    assert glu == {P + 'ff0/~/linear', P + 'ff1/~/linear'}
    assert {s.module for s in specs if s.interleave} == glu and all(s.name == 'lora_b' for s in specs if s.interleave)
    b = np.arange(8 * 512, dtype=np.float32).reshape(8, 512)
    il = _interleave(b)
    assert np.array_equal(il[:, 0::2], b[:, :256]) and np.array_equal(il[:, 1::2], b[:, 256:])
    assert np.array_equal(_deinterleave(il), b)


def test_checkpoint_package_resolution(tmp_path):
    from progen_b200.checkpoint import (count_params, get_checkpoint_fns, last_checkpoint_file, load_checkpoint_file,
                                        package_params)
    m = ProGen(**CFG)
    params = m.init(0)
    base_dir, lora_dir = tmp_path / 'base', tmp_path / 'lora'
    _, get_last, save = get_checkpoint_fns(base_dir)
    save({'next_seq_index': 8, 'params': params, 'optim_state': None, 'model_config': CFG, 'run_id': None})
    assert package_params(get_last()) is not None
    base_file = last_checkpoint_file(base_dir)
    assert base_file.endswith('.pkl') and base_file.startswith('/')
    ad = m.init_adapters(1, 8)
    rng = np.random.default_rng(3)
    for v in ad.values():
        v['lora_b'] = rng.standard_normal(v['lora_b'].shape).astype(np.float32)
    pkg = {'next_seq_index': 16, 'adapters': ad, 'lora': {'rank': 8, 'alpha': 16.0}, 'optim_state': None,
           'model_config': CFG, 'run_id': None, 'base_checkpoint': base_file, 'num_params': count_params(params)}
    _, get_last_lora, save_lora = get_checkpoint_fns(lora_dir)
    save_lora(pkg)
    got = package_params(get_last_lora())
    want = merge_adapters(params, ad, 2.0)
    assert all(np.array_equal(got[k][n], want[k][n]) for k in want for n in want[k])
    assert 'params' not in load_checkpoint_file(last_checkpoint_file(lora_dir))
    with pytest.raises(L.ProgenError, match='parameters'):
        package_params({**pkg, 'num_params': pkg['num_params'] + 1})
    (base_dir / base_file.rsplit('/', 1)[1]).unlink()
    with pytest.raises(L.ProgenError, match='missing'):
        package_params(get_last_lora())


def test_train_cli_refuses_conflicting_lora_flags(tmp_path):
    """flags that would change a resumed run's mode or adapter settings are refused before any device work"""
    from click.testing import CliRunner
    from progen_b200.checkpoint import count_params, get_checkpoint_fns, last_checkpoint_file
    sys.path.insert(0, ROOT)
    import train
    m = ProGen(**CFG)
    params = m.init(0)
    dirs = {k: tmp_path / k for k in ('base', 'other', 'full', 'lora', 'empty')}
    for k in ('base', 'other', 'full'):
        get_checkpoint_fns(dirs[k])[2]({'next_seq_index': 8, 'params': params, 'optim_state': None, 'model_config': CFG,
                                        'run_id': None})
    get_checkpoint_fns(dirs['lora'])[2]({'next_seq_index': 16, 'adapters': m.init_adapters(1, 8),
                                         'lora': {'rank': 8, 'alpha': 8.0}, 'optim_state': None, 'model_config': CFG,
                                         'run_id': None, 'base_checkpoint': last_checkpoint_file(dirs['base']),
                                         'num_params': count_params(params)})
    cases = [
        (['--checkpoint_path', dirs['full'], '--lora_rank', '16'], 'full-parameter checkpoint'),
        (['--checkpoint_path', dirs['full'], '--init_checkpoint', dirs['base'], '--lora_rank', '16'], 'full-parameter checkpoint'),
        (['--checkpoint_path', dirs['lora'], '--lora_rank', '16'], 'rank 8'),
        (['--checkpoint_path', dirs['lora'], '--lora_alpha', '4'], 'alpha 8.0'),
        (['--checkpoint_path', dirs['lora'], '--init_checkpoint', dirs['other']], 'the base'),
        (['--checkpoint_path', dirs['empty'], '--lora_alpha', '4'], '--lora_alpha needs --lora_rank'),
        (['--checkpoint_path', dirs['empty'], '--lora_rank', '16'], '--lora_rank needs --init_checkpoint'),
    ]
    for args, msg in cases:
        res = CliRunner().invoke(train.main, [str(a) for a in args])
        assert res.exit_code == 2, (args, res.exit_code, res.output, res.exception)
        assert msg in ' '.join(res.output.split()), (args, res.output)
