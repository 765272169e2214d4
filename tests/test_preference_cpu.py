"""Preference (DPO) fine-tuning without a GPU: every input check of `ProGen.preference_loss_and_grad`,
`Trainer.preference_step` (`preference.check_pairs`) and the dpo.py pairs file, and the float64 reference loss the GPU tests
compare against (its log-likelihood, its gradient against finite differences, and its value and gradient at policy =
reference)."""
import math

import numpy as np
import pytest
import torch

from oracle import progen_ref as O
from oracle import progen_torch as T
from preference_oracle import preference_loss, preference_loss_and_grads, seq_log_likelihood

KW = dict(num_tokens=256, dim=128, seq_len=128, depth=2, window_size=64, global_mlp_depth=1, heads=2, dim_head=64)


def _rows(P, n=128, seed=0):
    return np.random.default_rng(seed).integers(1, 256, (P, n + 1)).astype(np.uint16)


def _model():
    from progen_b200 import ProGen
    return ProGen(**KW)


@pytest.mark.parametrize('change, match', [
    (dict(chosen=np.zeros((2, 128), np.int64)), r'chosen must be \(P, seq_len \+ 1 = 129\)'),
    (dict(chosen=np.zeros(129, np.int64)), r'chosen must be \(P, seq_len \+ 1 = 129\)'),
    (dict(rejected=np.zeros((2, 129), np.float32)), 'rejected must hold integer token ids'),
    (dict(rejected=_rows(3)), 'chosen and rejected must have the same shape'),
    (dict(chosen=_rows(0), rejected=_rows(0), ref_chosen=[], ref_rejected=[]), r'needs at least one pair \(P >= 1\)'),
    (dict(ref_chosen=[1.0]), r'ref_chosen must have shape \(2,\)'),
    (dict(ref_rejected=np.zeros((2, 1))), r'ref_rejected must have shape \(2,\)'),
    (dict(ref_chosen=['a', 'b']), 'ref_chosen must be 2 floats'),
    (dict(ref_chosen=[0.0, float('nan')]), r'ref_chosen must be finite \(in float32\)'),
    (dict(ref_rejected=[-1e300, 0.0]), r'ref_rejected must be finite \(in float32\)'),
    (dict(beta=0.0), 'beta must be a finite number > 0'),
    (dict(beta=-0.1), 'beta must be a finite number > 0'),
    (dict(beta=float('inf')), 'beta must be a finite number > 0'),
    (dict(beta=float('nan')), 'beta must be a finite number > 0'),
    (dict(beta=1e-50), 'beta must be a finite number > 0'),
    (dict(beta=1e300), 'beta must be a finite number > 0'),
    (dict(beta=True), 'beta must be a finite number > 0'),
    (dict(beta='0.1'), 'beta must be a finite number > 0'),
])
def test_preference_loss_and_grad_checks_inputs_before_device_work(change, match):
    from progen_b200.lib import ProgenError
    args = dict(chosen=_rows(2), rejected=_rows(2, seed=1), ref_chosen=[-300.0, -310.0], ref_rejected=[-305.0, -290.0],
                beta=0.1)
    args.update(change)
    model = _model()
    with pytest.raises(ProgenError, match='preference_loss_and_grad: ' + match):
        model.preference_loss_and_grad(None, args['chosen'], args['rejected'], args['ref_chosen'], args['ref_rejected'],
                                       beta=args['beta'])
    assert model._engine is None


@pytest.mark.parametrize('P, global_pairs, match', [
    (2, 1, r'global_pairs must be an integer >= the pairs given \(2\)'),
    (2, 2.0, 'global_pairs must be an integer'),
    (2, True, 'global_pairs must be an integer'),
    (0, 0, r'global_pairs must be an integer >= the pairs given \(1\)'),
    (0, None, 'a rank without pairs needs global_pairs'),
])
def test_preference_step_checks(P, global_pairs, match):
    """Trainer.preference_step runs these checks (what='preference_step'), which also admit a rank without pairs"""
    from progen_b200.lib import ProgenError
    from progen_b200.preference import check_pairs
    with pytest.raises(ProgenError, match='preference_step: ' + match):
        check_pairs(_rows(P), _rows(P, seed=1), np.zeros(P), np.zeros(P), 0.1, global_pairs, 128, what='preference_step',
                    allow_empty=True)


def test_check_pairs_layout():
    from progen_b200.preference import check_pairs
    c, r = _rows(3), _rows(3, seed=1)
    rows, ref, beta, gp = check_pairs(c, r, [1, 2, 3], [4, 5, 6], 0.5, None, 128)
    assert rows.dtype == np.int32 and rows.shape == (6, 129)
    np.testing.assert_array_equal(rows[:3], c)
    np.testing.assert_array_equal(rows[3:], r)
    np.testing.assert_array_equal(ref, np.float32([1, 2, 3, 4, 5, 6]))
    assert (beta, gp) == (0.5, 3)
    rows, ref, _, gp = check_pairs(_rows(0), _rows(0), [], [], 0.1, 5, 128, allow_empty=True)
    assert rows.shape == (0, 129) and ref.shape == (0,) and gp == 5


def test_read_pairs():
    from progen_b200.lib import ProgenError
    from progen_b200.preference import read_pairs
    c, r = read_pairs(['MKV\tMKL\n', '\n', '   \n', 'AAA\tCCC\r\n'])
    assert (c, r) == (['MKV', 'AAA'], ['MKL', 'CCC'])
    with pytest.raises(ProgenError, match=r'pairs line 3: expected `chosen<TAB>rejected` \(exactly one tab\), found 0'):
        read_pairs(['A\tB', '', 'AB'])
    with pytest.raises(ProgenError, match='pairs line 2: .* found 2 tabs'):
        read_pairs(['A\tB', 'A\tB\tC'])
    with pytest.raises(ProgenError, match='pairs line 1: the chosen and the rejected sequence must both be non-empty'):
        read_pairs([' \tB'])


def test_dpo_cli_names_the_bad_line(tmp_path):
    """the pairs file is read before any checkpoint or device work"""
    from click.testing import CliRunner
    import dpo
    p = tmp_path / 'pairs.tsv'
    p.write_text('MKV\tMKL\n\nMKVL MKLV\n')
    res = CliRunner().invoke(dpo.main, ['--init_checkpoint', str(tmp_path / 'none'), '--pairs', str(p),
                                        '--checkpoint_path', str(tmp_path / 'out')])
    assert res.exit_code != 0
    assert 'pairs line 3: expected `chosen<TAB>rejected`' in res.output, res.output
    p.write_text('\n')
    res = CliRunner().invoke(dpo.main, ['--init_checkpoint', str(tmp_path / 'none'), '--pairs', str(p)])
    assert res.exit_code != 0 and 'no pairs' in res.output


def test_epoch_order_is_a_seeded_permutation():
    import dpo
    a, b = dpo.epoch_order(10, 0, 3), dpo.epoch_order(10, 1, 3)
    assert sorted(a) == list(range(10)) and sorted(b) == list(range(10))
    assert not np.array_equal(a, b)
    np.testing.assert_array_equal(a, dpo.epoch_order(10, 0, 3))


# ---- the float64 reference
TINY = dict(num_tokens=16, dim=16, seq_len=8, depth=2, window_size=4, global_mlp_depth=1, heads=2, dim_head=8)


def _tiny(seed=3):
    cfg = O.make_config(**TINY)
    params = O.randomize_params(O.init_params(cfg, seed), seed + 1)
    rng = np.random.default_rng(seed + 2)
    c = rng.integers(1, 16, (2, 9)).astype(np.int64)
    r = rng.integers(1, 16, (2, 9)).astype(np.int64)
    c[1, 5:] = 0                                        # a row that ends early
    r[0, 3:] = 0
    return cfg, params, c, r


def test_seq_log_likelihood_is_minus_cross_entropy_times_count():
    cfg, params, c, r = _tiny()
    data = torch.as_tensor(np.concatenate([c, r]))
    prm = T.to_torch(params)
    s = seq_log_likelihood(prm, data, cfg).numpy()
    ce = T.cross_entropy(T.forward(prm, data[:, :-1], cfg), data[:, 1:]).numpy()
    count = O.loss_mask(data[:, 1:].numpy()).sum(-1)
    np.testing.assert_allclose(s, -ce * count, rtol=1e-13, atol=1e-12)


def test_dpo_gradient_matches_finite_differences():
    cfg, params, c, r = _tiny()
    ref_c, ref_r = np.array([-20.0, -12.0]), np.array([-11.0, -19.5])
    beta = 0.7
    _, grads, _ = preference_loss_and_grads(params, c, r, ref_c, ref_r, cfg, beta)
    ct, rt = torch.as_tensor(c), torch.as_tensor(r)

    def f(p):
        return float(preference_loss(T.to_torch(p), ct, rt, ref_c, ref_r, cfg, beta)[0])

    rng = np.random.default_rng(0)
    checked = 0
    for m, d in params.items():
        for k, v in d.items():
            for _ in range(2):
                idx = tuple(int(rng.integers(0, s)) for s in v.shape)
                h = 1e-6
                hi = {mm: {kk: vv.astype(np.float64).copy() for kk, vv in dd.items()} for mm, dd in params.items()}
                lo = {mm: {kk: vv.astype(np.float64).copy() for kk, vv in dd.items()} for mm, dd in params.items()}
                hi[m][k][idx] += h
                lo[m][k][idx] -= h
                fd = (f(hi) - f(lo)) / (2 * h)
                assert abs(fd - grads[m][k][idx]) < 1e-6 + 1e-5 * abs(fd), (m, k, idx, fd, grads[m][k][idx])
                checked += 1
    assert checked >= 20


def test_policy_equal_to_reference_gives_ln2_and_half_the_likelihood_gradient():
    cfg, params, c, r = _tiny()
    beta = 0.3
    prm = T.to_torch(params)
    s = seq_log_likelihood(prm, torch.as_tensor(np.concatenate([c, r])), cfg).numpy()
    loss, grads, stats = preference_loss_and_grads(params, c, r, s[:2], s[2:], cfg, beta)
    assert abs(loss - math.log(2)) < 1e-12
    np.testing.assert_array_equal(stats['margin'], 0.0)
    # d softplus(-z)/dz = -1/2 at z = 0:  grad = -beta/2 * mean_i (grad s(c_i) - grad s(r_i))
    prm = T.to_torch(params, requires_grad=True)
    ss = seq_log_likelihood(prm, torch.as_tensor(np.concatenate([c, r])), cfg)
    (ss[:2] - ss[2:]).mean().backward()
    for m, d in prm.items():
        for k, v in d.items():
            np.testing.assert_allclose(grads[m][k], -beta / 2 * v.grad.numpy(), rtol=1e-10, atol=1e-14)
