"""The host side of policy-gradient fine-tuning (DESIGN.md §3.14): the float64 head reference (tests/policy_oracle.py)
against finite differences, the LM loss at beta = 0 and A = 1, a zero KL and gradient against itself; group advantages
against a float64 replay; samples to rows; every refusal of the batch check; the C declarations against lib.py."""
import os
import re
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
from policy_oracle import policy_head, span_mask             # noqa: E402
from progen_b200.lib import ProgenError                      # noqa: E402
from progen_b200.policy import check_policy_batch, group_advantages, samples_to_rows   # noqa: E402


def _case(seed, B=3, n=9, V=12):
    rng = np.random.default_rng(seed)
    s, z = rng.standard_normal((B, n, V)) * 2, rng.standard_normal((B, n, V)) * 3
    labels = rng.integers(1, V, (B, n))
    labels[2, 3] = V + 7                                    # clamped to V - 1
    span = np.array([[0, 9], [2, 5], [8, 9]])
    adv = rng.standard_normal(B)
    return s, z, labels, span, adv


@pytest.mark.parametrize('beta', [0.0, 0.04, 1.0])
def test_oracle_gradient_matches_finite_differences(beta):
    s, z, labels, span, adv = _case(1)
    loss, grad, _ = policy_head(s, z, labels, span, adv, beta, inv_rows=0.2)
    rng = np.random.default_rng(2)
    eps = 1e-6
    for _ in range(40):
        idx = tuple(rng.integers(0, k) for k in s.shape)
        sp, sm = s.copy(), s.copy()
        sp[idx] += eps
        sm[idx] -= eps
        fd = (policy_head(sp, z, labels, span, adv, beta, 0.2)[0] - policy_head(sm, z, labels, span, adv, beta, 0.2)[0]) / (2 * eps)
        assert abs(fd - grad[idx]) < 1e-7 + 1e-6 * abs(fd), (idx, fd, grad[idx])
    m = span_mask(span, *s.shape[:2])
    assert np.all(grad[m == 0] == 0.0)


def test_beta_zero_unit_advantage_over_the_counted_positions_is_the_lm_loss():
    from oracle import progen_torch as T
    s, _, labels, _, _ = _case(3)
    labels[0, 5:] = 0                                       # counted: 0..5 (the first pad is the EOS, Q8)
    span = np.array([[0, 6], [0, 9], [0, 9]])
    loss, _, stats = policy_head(s, None, labels, span, np.ones(3), 0.0)
    ref = T.cross_entropy(torch.tensor(s), torch.tensor(np.clip(labels, 0, s.shape[-1] - 1)))
    assert np.allclose(-stats[:, 0], ref.numpy(), rtol=1e-12, atol=1e-12)
    assert abs(loss - float(ref.mean())) < 1e-12


def test_reference_equal_to_policy_gives_zero_kl_and_zero_gradient_at_zero_advantage():
    s, _, labels, span, _ = _case(4)
    loss, grad, stats = policy_head(s, s.copy(), labels, span, np.zeros(3), 0.5)
    assert np.abs(stats[:, 1]).max() < 1e-15 and abs(loss) < 1e-15 and np.abs(grad).max() < 1e-15


def test_group_advantages_match_a_float64_replay():
    rng = np.random.default_rng(5)
    r = rng.standard_normal(12) * 3
    r[4:8] = 0.1                                            # a group of equal rewards
    for scale in ('std', 'none'):
        got = group_advantages(r, 4, scale)
        want = []
        for g in r.reshape(3, 4):
            a = g - g.mean()
            if scale == 'std':
                a = a / (g.std() + 1e-6)
            want.append(a)
        want = np.concatenate(want)
        want[4:8] = 0.0
        assert got.dtype == np.float64 and np.array_equal(got, want)
        assert np.all(got[4:8] == 0.0)
    assert np.array_equal(group_advantages(r, 1), np.zeros(12))
    for bad in (dict(group_size=5), dict(group_size=0), dict(group_size=True), dict(scale='rank')):
        with pytest.raises(ProgenError):
            group_advantages(r, **{'group_size': 4, **bad})
    with pytest.raises(ProgenError, match='reward 3'):
        group_advantages(np.where(np.arange(12) == 3, np.nan, r), 4)


def test_samples_to_rows():
    n = 8
    tokens = np.zeros((4, n), np.int64)
    tokens[0, :6] = [0, 5, 6, 7, 8, 0]       # prompt (5,), generated 6 7 8 then EOS: start 2, length 4
    tokens[1, :8] = [0, 5, 6, 7, 8, 9, 10, 11]   # unfinished at max_length 8: start 2, length 6
    tokens[2, :3] = [0, 4, 0]                # empty prompt: start 1, generated 4 then EOS
    tokens[3, :4] = [0, 3, 4, 9]             # length-1 row at max_length 4: start 3, generated 9
    samples = dict(tokens=tokens, start=np.array([2, 2, 1, 3]), length=np.array([4, 6, 2, 1]),
                   finished=np.array([True, False, True, False]))
    rows, span = samples_to_rows(samples)
    assert rows.dtype == np.int32 and rows.shape == (4, n + 1)
    assert np.array_equal(rows[:, :n], tokens) and np.all(rows[:, n] == 0)
    assert span.dtype == np.int32 and span.tolist() == [[1, 5], [1, 7], [0, 2], [2, 3]]
    labels = rows[:, 1:]
    for i, (lo, hi) in enumerate(span):
        gen = tokens[i, samples['start'][i]:samples['start'][i] + samples['length'][i]]
        assert np.array_equal(labels[i, lo:hi], gen)            # the labels of the span are the generated tokens
    # an unfinished row's trailing pad is not counted; every span passes the batch check
    check_policy_batch(rows, span, np.zeros(4), 0.1, None, n)


def test_every_refusal_names_the_row():
    n = 8
    rows = np.zeros((3, n + 1), np.int32)
    rows[:, 1:6] = 5                                         # labels 5 at 0..4, the EOS at 5, pads after it
    span = np.array([[0, 6], [1, 3], [2, 5]])
    adv = np.zeros(3)
    got = check_policy_batch(rows, span, adv, 0.0, None, n)
    assert got[0].dtype == np.int32 and got[1].dtype == np.int32 and got[2].dtype == np.float32 and got[4] == 3
    for bad_span, row in (([[0, 6], [3, 3], [2, 5]], 1), ([[0, 6], [1, 3], [4, 2]], 2), ([[-1, 6], [1, 3], [2, 5]], 0),
                          ([[0, 6], [1, 9], [2, 5]], 1), ([[0, 7], [1, 3], [2, 5]], 0)):
        with pytest.raises(ProgenError, match=f'row {row}:'):
            check_policy_batch(rows, np.array(bad_span), adv, 0.0, None, n)
    gap = rows.copy()
    gap[2, 2:4] = 0                                          # labels 1 and 2 pads, then labels again: 2 is not counted
    check_policy_batch(gap, np.array([[0, 6], [1, 3], [3, 5]]), adv, 0.0, None, n)
    with pytest.raises(ProgenError, match='row 2:'):
        check_policy_batch(gap, np.array([[0, 6], [1, 3], [1, 4]]), adv, 0.0, None, n)
    for a, row in (([0.0, np.inf, 0.0], 1), ([0.0, 0.0, 1e39], 2), ([np.nan, 0.0, 0.0], 0)):
        with pytest.raises(ProgenError, match=f'row {row}:'):
            check_policy_batch(rows, span, np.array(a), 0.0, None, n)
    for beta in (-0.1, np.nan, np.inf, 1e39, True, '0.1'):
        with pytest.raises(ProgenError, match='beta'):
            check_policy_batch(rows, span, adv, beta, None, n)
    for gr in (2, 0, 3.0, True):
        with pytest.raises(ProgenError, match='global_rows'):
            check_policy_batch(rows, span, adv, 0.0, gr, n)
    for bad in (dict(rows=rows[:, :-1]), dict(rows=rows.astype(np.float32)), dict(span=span[:2]), dict(advantages=adv[:2])):
        kw = {**dict(rows=rows, span=span, advantages=adv, beta=0.0, global_rows=None, seq_len=n), **bad}
        with pytest.raises(ProgenError):
            check_policy_batch(**kw)
    with pytest.raises(ProgenError):
        check_policy_batch(rows[:0], span[:0], adv[:0], 0.0, None, n)
    assert check_policy_batch(rows[:0], span[:0], adv[:0], 0.0, 4, n, allow_empty=True)[4] == 4


def _declared_args(name):
    src = open(os.path.join(ROOT, 'include', 'progen_b200.h')).read()
    src = re.sub(r'/\*.*?\*/', '', src, flags=re.S)
    m = re.search(r'\b' + name + r'\s*\(([^)]*)\)', src)
    return [a.strip() for a in m.group(1).split(',')]


@pytest.mark.parametrize('name', ['progen_policy_head', 'progen_decode_load_weight'])
def test_header_and_argtypes_agree(name):
    import ctypes as C
    from progen_b200 import lib as L
    args = _declared_args(name)
    want = L.PROTOTYPES[name]
    assert len(args) == len(want), (args, want)
    for decl, t in zip(args, want):
        kind = C.c_void_p if '*' in decl else C.c_longlong if decl.startswith('long long') else \
            C.c_float if decl.startswith('float') else C.c_int
        assert t is kind, (decl, t)
