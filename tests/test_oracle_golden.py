"""CPU tests: the oracle (oracle/progen_ref.py, oracle/progen_torch.py) against golden vectors produced by running
the reference's own source under the numpy shim (tests/golden/make_golden.py)."""
import numpy as np
import pytest
import torch

from oracle import progen_ref as O
from oracle import progen_torch as T
from golden_util import load_case, CASES

TINY = [n for n in CASES if n != 'cfg1']


@pytest.mark.parametrize('name', TINY)
def test_forward_matches_reference_source(name):
    cfg, params, data, g = load_case(name)
    for b in range(data.shape[0]):
        logits = O.forward(params, data[b, :-1], cfg, np.float64)
        np.testing.assert_allclose(logits, g['logits'][b], rtol=0, atol=1e-11)
        ce = O.cross_entropy(logits, data[b, 1:])
        assert abs(ce - g['ce_per_row'][b]) < 1e-11
    assert abs(O.batch_loss(params, data, cfg) - float(g['loss'])) < 1e-11


def test_forward_cfg1_matches_reference_source():
    cfg, params, data, g = load_case('cfg1')
    rows = g['logits_rows']
    logits = O.forward(params, data[0, :-1], cfg, np.float64)
    np.testing.assert_allclose(logits[rows], g['logits'][0], rtol=0, atol=2e-6)   # stored as float32
    assert abs(O.cross_entropy(logits, data[0, 1:]) - g['ce_per_row'][0]) < 1e-10
    # fp32 oracle stays within the north_star fp32 tolerance of the fp64 truth
    l32 = O.forward(params, data[0, :-1], cfg, np.float32)
    assert np.abs(l32 - logits).max() < 1e-4


@pytest.mark.parametrize('name', TINY)
@pytest.mark.parametrize('add_bos', [False, True])
def test_greedy_sampler_matches_reference_source(name, add_bos):
    cfg, params, data, g = load_case(name)
    s = O.sample_greedy(params, g['prime'], cfg['seq_len'], cfg, top_k=25, add_bos=add_bos)
    np.testing.assert_array_equal(s, g[f'sample_bos{int(add_bos)}'])


@pytest.mark.parametrize('name', TINY)
def test_torch_twin_matches_numpy_oracle_and_grad_fingerprints(name):
    cfg, params, data, g = load_case(name)
    prm = T.to_torch(params)
    ids = torch.as_tensor(data[:, :-1].astype(np.int64))
    logits = T.forward(prm, ids, cfg).numpy()
    np.testing.assert_allclose(logits, g['logits'], rtol=0, atol=1e-11)
    loss, grads = T.loss_and_grads(params, data, cfg)
    assert abs(loss - float(g['loss'])) < 1e-11
    for key, norm, head in zip(g['grad_keys'], g['grad_norms'], g['grad_head']):
        m, k = str(key).split('|')
        gr = grads[m][k]
        assert abs(np.linalg.norm(gr) - norm) <= 1e-9 * max(1.0, norm)
        np.testing.assert_allclose(np.resize(gr.ravel()[:8], 8), head, rtol=0, atol=1e-12)


def test_torch_twin_hidden_state():
    """return_hidden leaves the logits bit-identical and returns the head's input: the final LayerNorm output, which is
    the [I | 0]-head read of the numpy oracle's hidden state"""
    cfg, params, data, g = load_case('tiny_glu_sgu')
    prm = T.to_torch(params)
    ids = torch.as_tensor(data[:, :-1].astype(np.int64))
    logits, hidden = T.forward(prm, ids, cfg, return_hidden=True)
    assert torch.equal(logits, T.forward(prm, ids, cfg))
    head = prm[O.P + 'linear']
    assert torch.equal(hidden @ head['w'] + head['b'], logits)
    d, V = cfg['dim'], cfg['num_tokens']
    p = dict(params)
    p[O.P + 'linear'] = {'w': np.eye(d, V, dtype=np.float32), 'b': np.zeros(V, np.float32)}
    ref = np.stack([O.forward(p, r, cfg)[:, :d] for r in data[:, :-1]])
    np.testing.assert_allclose(hidden.numpy(), ref, rtol=0, atol=1e-11)


def test_torch_twin_gradients_match_finite_differences():
    cfg, params, data, g = load_case('tiny_glu_sgu')
    _, grads = T.loss_and_grads(params, data, cfg)
    rng = np.random.default_rng(0)
    p64 = {m: {k: v.astype(np.float64) for k, v in d.items()} for m, d in params.items()}
    eps = 1e-6
    for m in list(params)[::3]:
        for k, a in params[m].items():
            idx = tuple(rng.integers(0, s) for s in a.shape)
            if k == 'spatial_weights':
                idx = (max(idx), min(idx))                      # lower triangle (upper has zero gradient)
            orig = p64[m][k][idx]
            p64[m][k][idx] = orig + eps
            lp = O.batch_loss(p64, data, cfg)
            p64[m][k][idx] = orig - eps
            lm = O.batch_loss(p64, data, cfg)
            p64[m][k][idx] = orig
            fd = (lp - lm) / (2 * eps)
            assert abs(fd - grads[m][k][idx]) < 1e-6 + 1e-4 * abs(fd), (m, k, idx, fd, grads[m][k][idx])


def test_sgu_upper_triangle_receives_no_gradient():
    cfg, params, data, g = load_case('tiny_glu_sgu')
    _, grads = T.loss_and_grads(params, data, cfg)
    gw = grads[O.P + 'ff2/~/sgu']['spatial_weights']
    assert np.abs(np.triu(gw, 1)).max() == 0.0 and np.abs(np.tril(gw)).max() > 0


def test_quirks():
    # Q1: window-0 queries attend w zero keys: row i of any window sees w + i + 1 keys
    cfg = O.make_config(num_tokens=256, dim=64, seq_len=32, depth=1, window_size=8, global_mlp_depth=0, heads=2, dim_head=32)
    # Q6: top-k keeps k-1 entries, the rest become 0.0
    logits = -np.arange(1, 11, dtype=np.float64)
    mask, out = O.select_top_k(logits, 3)
    assert mask.sum() == 2 and (out[2:] == 0).all()
    assert int(np.argmax(out)) == 2                 # all kept logits negative -> first filtered index wins
    # Q8: loss mask = non-zero labels + first zero
    t = np.array([5, 0, 7, 0, 0])
    np.testing.assert_array_equal(O.loss_mask(t), [True, True, True, False, False])
    # Q9 tokenizer
    assert O.encode_tokens('A#') == [66, 36] and O.decode_tokens(np.array([66, 36])) == 'A#'
    # layer schedule (progen.py:211-212)
    assert O.layer_kinds(dict(depth=12, global_mlp_depth=2, ff_glu=True)) == ['glu'] * 10 + ['sgu'] * 2


def test_optimizer_chain_semantics():
    """apply_every(4): parameters move only on every 4th call; Adam moments advance every call; weight decay only on
    ndim > 1 leaves (train.py:115-121)."""
    params = {'m': {'w': np.ones((3, 2), np.float32), 'b': np.ones(2, np.float32)}}
    st = O.optim_init(params, every=4)
    rng = np.random.default_rng(0)
    p = params
    for step in range(8):
        grads = {'m': {'w': rng.standard_normal((3, 2)), 'b': rng.standard_normal(2)}}
        p2, gn = O.optim_step(p, grads, st)
        moved = not np.array_equal(p2['m']['w'], p['m']['w'])
        assert moved == (step % 4 == 3)
        p = p2
    assert st['count'] == 8
    # zero gradient: only weight decay acts, and only on the matrix
    st = O.optim_init(params, every=1)
    z = {'m': {'w': np.zeros((3, 2)), 'b': np.zeros(2)}}
    p2, _ = O.optim_step(params, z, st, lr=1.0, wd=0.5)
    np.testing.assert_allclose(p2['m']['w'], 0.5)
    np.testing.assert_allclose(p2['m']['b'], 1.0)
