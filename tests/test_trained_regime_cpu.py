"""CPU tests of the trained-regime fixture (tests/trained_regime.py): sharpened parameters reach every regime threshold in
the float64 oracle, plain randomize_params reaches none of the attention, logit and GELU thresholds (so the fixture
cannot drift back to the easy regime unnoticed), and the oracle's probe changes no output."""
import json

import numpy as np
import pytest
import torch

from oracle import progen_ref as O
from oracle import progen_torch as T
import trained_regime as R

STACKS = {
    'd256': dict(num_tokens=256, dim=256, seq_len=256, depth=2, global_mlp_depth=1, window_size=64, heads=4, dim_head=64),
    'd512': dict(num_tokens=256, dim=512, seq_len=1024, depth=2, global_mlp_depth=1, window_size=256, heads=8, dim_head=64),
}
EASY_ONLY = ['attn_max_prob_median', 'top1_prob_median', 'logit_absmax', 'gelu_saturated_share']


def _case(name):
    cfg = O.make_config(**STACKS[name])
    params = O.randomize_params(O.init_params(cfg, 11), 12)
    ids = np.random.default_rng(0).integers(1, cfg['num_tokens'], (2, cfg['seq_len']))
    return cfg, params, ids


@pytest.mark.parametrize('name', sorted(STACKS))
def test_sharpened_parameters_reach_the_trained_regime(name):
    cfg, params, ids = _case(name)
    sharp = R.sharpen(params, cfg, 0)
    m = R.regime_metrics(sharp, ids, cfg)
    print(json.dumps(dict(case=f'sharpened_{name}', **{k: round(v, 4) for k, v in m.items()})))
    assert not R.unmet(m), (R.unmet(m), m)
    assert all(v.dtype == np.float32 for d in sharp.values() for v in d.values())
    again = R.sharpen(params, cfg, 0)
    assert all(np.array_equal(again[k][kk], vv) for k, d in sharp.items() for kk, vv in d.items())
    # sharpen copies: the randomized parameters are untouched
    assert np.array_equal(params[O.P + 'linear']['w'], O.randomize_params(O.init_params(cfg, 11), 12)[O.P + 'linear']['w'])


@pytest.mark.parametrize('name', sorted(STACKS))
def test_randomized_parameters_stay_in_the_easy_regime(name):
    cfg, params, ids = _case(name)
    m = R.regime_metrics(params, ids, cfg)
    print(json.dumps(dict(case=f'randomized_{name}', **{k: round(v, 4) for k, v in m.items()})))
    assert set(EASY_ONLY) <= set(R.unmet(m)), m


def test_probe_changes_no_output():
    cfg, params, ids = _case('d256')
    sharp = R.sharpen(params, cfg, 0)
    prm = T.to_torch(sharp)
    ids = torch.as_tensor(ids)
    probe = {}
    ref, hid = T.forward(prm, ids, cfg, return_hidden=True)
    got, hid2 = T.forward(prm, ids, cfg, return_hidden=True, probe=probe)
    assert torch.equal(ref, got) and torch.equal(hid, hid2)
    assert len(probe['attn']) == len(probe['gelu_in']) == cfg['depth'] and len(probe['resid']) == cfg['depth'] + 1
    # the probe's attention rows are distributions over the 2w keys of a window
    a = probe['attn'][0]
    assert a.shape == (2, cfg['heads'], cfg['seq_len'] // cfg['window_size'], cfg['window_size'], 2 * cfg['window_size'])
    assert torch.allclose(a.sum(-1), torch.ones((), dtype=a.dtype))
    np.testing.assert_allclose(ref[0].numpy(), O.forward(sharp, ids[0].numpy(), cfg), rtol=0, atol=1e-9)
