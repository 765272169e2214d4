"""Argument checks of the generation constraints (logit bias, minimum length, repetition penalty): every invalid value
raises ProgenError before anything needs a device, in ProGen.generate and in generate.py."""
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KW = dict(num_tokens=256, dim=64, seq_len=64, depth=2, window_size=16, global_mlp_depth=1, heads=2, dim_head=32)


def _bias(**set_):
    b = np.zeros(256, np.float32)
    for k, v in set_.items():
        b[int(k[1:])] = v
    return b


_all_banned = np.full(256, -np.inf, np.float32)
_all_banned[0] = 0.0                                    # only EOS left


@pytest.mark.parametrize('kwargs', [
    dict(logit_bias=np.zeros(255, np.float32)),         # wrong shape
    dict(logit_bias=np.zeros((1, 256), np.float32)),
    dict(logit_bias=[[0.0]]),
    dict(logit_bias='abc'),
    dict(logit_bias=_bias(c7=np.nan)),
    dict(logit_bias=_bias(c7=np.inf)),
    dict(logit_bias=np.full(256, 1e300)),               # +inf once it is the kernel's float32
    dict(logit_bias=_all_banned),                       # nothing in [1, V) left to draw
    dict(logit_bias=np.full(256, -np.inf, np.float32)),
    dict(min_new_tokens=-1),
    dict(min_new_tokens=63),                            # > max_length - 2 = 62
    dict(min_new_tokens=9, max_length=10),
    dict(min_new_tokens=2.0),
    dict(min_new_tokens=True),
    dict(repetition_penalty=0.0),
    dict(repetition_penalty=-1.2),
    dict(repetition_penalty=float('inf')),
    dict(repetition_penalty=float('nan')),
    dict(repetition_penalty='high'),
    dict(repetition_window=-1),
    dict(repetition_window=65),                         # > seq_len
    dict(repetition_window=1.5),
])
def test_constraints_reject_invalid_arguments_without_a_device(kwargs):
    from progen_b200 import ProGen
    from progen_b200.lib import ProgenError
    model = ProGen(**KW)
    with pytest.raises(ProgenError):
        model.generate({}, 'MK', **kwargs)
    assert model._engine is None and model._gen_decoder is None


def test_alphabet_bias():
    from generate import alphabet_bias
    from progen_b200.lib import ProgenError
    b = alphabet_bias('ACDEFGHIKLMNPQRSTVWY', 256)
    allowed = {0} | {ord(ch) + 1 for ch in 'ACDEFGHIKLMNPQRSTVWY'}
    assert b.dtype == np.float32 and b.shape == (256,)
    assert all((b[i] == 0.0) == (i in allowed) for i in range(256))
    assert (b[[i for i in range(256) if i not in allowed]] == -np.inf).all()
    for bad in ('', 'ACÿ', 'AĀ'):             # ord 255 and 256 encode to ids >= V
        with pytest.raises(ProgenError):
            alphabet_bias(bad, 256)


def test_cli_rejects_an_unknown_alphabet_character(tmp_path):
    from progen_b200.checkpoint import file_save_checkpoint
    from progen_b200 import ProGen
    (tmp_path / 'ckpts').mkdir()
    file_save_checkpoint(tmp_path / 'ckpts', dict(next_seq_index=0, params=ProGen(**KW).init(1), optim_state=None,
                                                  model_config=KW, run_id=None))
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'generate.py'), '--checkpoint_path', str(tmp_path / 'ckpts'),
                        '--alphabet', 'ACDĀ', '--output', str(tmp_path / 'x.fasta')],
                       cwd=str(tmp_path), env=dict(os.environ, PYTHONPATH=ROOT), capture_output=True, text=True, timeout=600)
    assert r.returncode != 0
    assert 'ProgenError' in r.stderr and '--alphabet' in r.stderr, r.stderr[-2000:]
    assert not (tmp_path / 'x.fasta').exists()
