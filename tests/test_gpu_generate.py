"""Generation with the standard sampler (sampler 1 of csrc/decode_persist.cu; BatchDecoder.generate, ProGen.generate,
generate.py): greedy ids and logits against the oracle, an exact host replay of the filter and the Philox Gumbel draw,
the sampled distribution, token log-probabilities against `score`, the EOS early exit, seeding and batching, and that
the reference sampler (sampler 0) is untouched."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from golden_util import load_case, CASES

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TINY = [n for n in CASES if n != 'cfg1']
HEAD_B = 'pro_gen_base/~/linear'                      # the logits head (its bias raises or removes EOS)
_M32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(c, key):
    """Philox4x32-10 on numpy arrays: c = 4 counter words, key = 2 words -> 4 output words (uint64 holding uint32)"""
    c = [np.asarray(x, np.uint64) & _M32 for x in c]
    k0, k1 = np.uint64(key[0]) & _M32, np.uint64(key[1]) & _M32
    for i in range(10):
        if i:
            k0, k1 = (k0 + np.uint64(0x9E3779B9)) & _M32, (k1 + np.uint64(0xBB67AE85)) & _M32
        p0, p1 = np.uint64(0xD2511F53) * c[0], np.uint64(0xCD9E8D57) * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & _M32, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & _M32]
    return c


def gumbel(seed, sid, p, V):
    """the kernel's noise for tokens 0..V-1 drawn at position p of stream sid (float64)"""
    c = np.arange(V, dtype=np.uint64)
    w = philox4x32_10([c >> np.uint64(2), np.full(V, p, np.uint64), np.full(V, sid & 0xFFFFFFFF, np.uint64),
                       np.full(V, sid >> 32, np.uint64)], (seed & 0xFFFFFFFF, seed >> 32))
    x = np.choose((c & np.uint64(3)).astype(np.int64), w)
    u = (2.0 * (x >> np.uint64(9)).astype(np.float64) + 1.0) * 2.0 ** -24
    return -np.log(-np.log(u))


def host_filter(l, T, top_k, top_p, tol=1e-5):
    """-> (kept mask, ambiguous): top-k (ties kept), then the q-descending prefix whose mass reaches top_p"""
    l = np.asarray(l, np.float64)
    V = len(l)
    keep = np.ones(V, bool)
    amb = False
    if top_k:
        s = np.sort(l)[::-1]
        keep = l >= s[top_k - 1]
        amb |= top_k < V and s[top_k - 1] - s[top_k] < tol
    if top_p is not None and top_p < 1:
        z = np.where(keep, l / T, -np.inf)
        q = np.exp(z - z.max())
        q /= q.sum()
        order = np.lexsort((np.arange(V), -l))            # logit (= q) descending, ties by lower id
        before = np.concatenate([[0.0], np.cumsum(q[order])[:-1]])
        amb |= bool(np.any(np.abs(before - top_p)[keep[order]] < tol))
        kk = np.zeros(V, bool)
        kk[order] = before < top_p
        keep &= kk
    return keep, amb


def host_draw(l, T, top_k, top_p, g, margin=1e-4):
    """-> (id, kept mask, ambiguous) of the kernel's draw from logits l with noise g"""
    l = np.asarray(l, np.float64)
    if T == 0:
        s = np.sort(l)[::-1]
        return int(np.argmax(l)), np.ones(len(l), bool), bool(s[0] - s[1] <= margin)
    keep, amb = host_filter(l, T, top_k, top_p)
    sc = np.where(keep, l / T + g, -np.inf)
    s = np.sort(sc)[::-1]
    return int(np.argmax(sc)), keep, bool(amb or (np.isfinite(s[1]) and s[0] - s[1] <= margin))


def test_philox_known_answers():
    """Random123's known-answer vectors for Philox4x32-10 (the host replay below depends on this implementation)"""
    h = lambda c, k: [int(x) for x in philox4x32_10(c, k)]
    assert h([0, 0, 0, 0], (0, 0)) == [0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8]
    assert h([0xffffffff] * 4, (0xffffffff, 0xffffffff)) == [0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd]
    assert h([0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344], (0xa4093822, 0x299f31d0)) == \
        [0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1]


def _prompts(rng, lengths):
    return [rng.integers(1, 256, L).astype(np.int64) for L in lengths]


def _drawn(res, b, max_length):
    """positions row b drew"""
    return range(int(res['start'][b]), min(int(res['end'][b]) + 1, max_length))


@pytest.mark.parametrize('name', TINY)
def test_greedy_generate_matches_oracle(name):
    from progen_b200.decode import BatchDecoder
    from oracle import progen_ref as O
    cfg, params, data, g = load_case(name)
    n = cfg['seq_len']
    prompts = _prompts(np.random.default_rng(1), [0, 1, 7])
    dec = BatchDecoder(cfg, params, batch=3, keep_logits=True)
    res = dec.generate(prompts, temperature=0.0, seed=5)
    got = dec.logits_all.cpu().numpy()
    for b in range(3):
        assert res['start'][b] == 1 + len(prompts[b])
        assert res['ids'][b, 0] == 0 and (res['ids'][b, 1:1 + len(prompts[b])] == prompts[b]).all()
        ref = O.forward(params, res['ids'][b], cfg)
        assert np.abs(got[b, :n - 1] - ref[:n - 1]).max() < 2e-5 * max(1.0, np.abs(ref).max()), b
        checked = 0
        for t in _drawn(res, b, n):
            top2 = np.sort(ref[t - 1].astype(np.float64))[-2:]
            if top2[1] - top2[0] > 1e-3:
                assert res['ids'][b, t] == np.argmax(ref[t - 1]), (b, t)
                checked += 1
        assert checked > 0


def test_sampler_matches_host_replay():
    """T x top_k x top_p grid at B = 24: the kernel's id == the float64 host replay (Philox noise, filter, Gumbel-max on the
    kernel's own logits) wherever the draw is unambiguous; >= 99 % of positions are; every id lies in the kept set"""
    from progen_b200.decode import BatchDecoder
    cfg, params, data, g = load_case('tiny_all_glu')
    n, V, B = cfg['seq_len'], cfg['num_tokens'], 24
    rng = np.random.default_rng(7)
    prompts = _prompts(rng, rng.integers(0, 9, B))
    dec = BatchDecoder(cfg, params, batch=B, keep_logits=True)
    total = unamb = 0
    seed = 0x1234_5678_9ABC
    for T in (0.7, 1.0, 1.5):
        for top_k in (None, 5, 40):
            for top_p in (None, 0.5, 0.9):
                sids = np.arange(B, dtype=np.int64) * 1000 + (1 << 33)       # upper words in use too
                res = dec.generate(prompts, temperature=T, top_k=top_k, top_p=top_p, seed=seed, sample_ids=sids)
                lg = dec.logits_all.cpu().numpy()
                for b in range(B):
                    for t in _drawn(res, b, n):
                        want, keep, amb = host_draw(lg[b, t - 1], T, top_k, top_p, gumbel(seed, int(sids[b]), t, V))
                        got = int(res['ids'][b, t])
                        assert keep[got], (T, top_k, top_p, b, t, got)
                        total += 1
                        if not amb:
                            unamb += 1
                            assert got == want, (T, top_k, top_p, b, t, got, want)
    assert total > 1000 and unamb >= 0.99 * total, (unamb, total)


@pytest.mark.parametrize('T,top_k,top_p', [(0.8, None, 0.9), (1.2, 10, None)])
def test_first_draw_distribution_chi_square(T, top_k, top_p):
    """first drawn position over many sample ids against the exact filtered softmax of the oracle's float64 logits"""
    from scipy import stats
    from progen_b200.decode import BatchDecoder
    from oracle import progen_ref as O
    cfg, params, data, g = load_case('tiny_all_glu')
    n, V, B, runs = cfg['seq_len'], cfg['num_tokens'], 64, 40
    prompt = np.asarray(g['prime']).astype(np.int64)
    row = np.zeros(n, np.int64)
    row[1:1 + len(prompt)] = prompt
    l = O.forward(params, row, cfg)[len(prompt)].astype(np.float64)
    keep, amb = host_filter(l, T, top_k, top_p, tol=1e-4)
    assert not amb, 'the chosen top_p / top_k sits on a boundary: pick another'
    z = np.where(keep, l / T, -np.inf)
    probs = np.exp(z - z.max())
    probs /= probs.sum()
    dec = BatchDecoder(cfg, params, batch=B)
    counts = np.zeros(V, np.int64)
    for r in range(runs):
        res = dec.generate([prompt] * B, temperature=T, top_k=top_k, top_p=top_p, seed=11,
                           sample_ids=np.arange(r * B, (r + 1) * B), max_length=len(prompt) + 2)
        counts += np.bincount(res['ids'][:, 1 + len(prompt)], minlength=V)
    assert counts.sum() == B * runs
    assert counts[~keep].sum() == 0
    exp_counts = probs * counts.sum()
    big = exp_counts >= 5
    obs = np.append(counts[big], counts[~big].sum())
    exp_ = np.append(exp_counts[big], exp_counts[~big].sum())
    if exp_[-1] == 0:
        obs, exp_ = obs[:-1], exp_[:-1]
    chi2 = ((obs - exp_) ** 2 / exp_).sum()
    pval = 1.0 - stats.chi2.cdf(chi2, len(obs) - 1)
    assert pval > 1e-3, (chi2, len(obs), pval)


def test_token_logp_equals_score():
    from progen_b200 import ProGen
    cfg, params, data, g = load_case('tiny_glu_sgu')
    model = ProGen(**CASES['tiny_glu_sgu'])
    n = cfg['seq_len']
    prompts = _prompts(np.random.default_rng(3), [0, 2, 5, 9])
    res = model.generate(params, prompts, num_samples=3, temperature=1.0, seed=9, top_p=0.95)
    rows = np.concatenate([res['tokens'], np.zeros((len(res['tokens']), 1), np.int64)], axis=1)
    sc = model.score(params, rows, return_tokens=True)['token_logp']
    for i in range(len(rows)):
        s, ln = int(res['start'][i]), int(res['length'][i])
        want = sc[i, s - 1:s - 1 + ln].astype(np.float64)
        got = res['token_logp'][i, s:s + ln].astype(np.float64)
        assert np.abs(got - want).max() < 1e-4, i
        assert (res['token_logp'][i, :s] == 0).all() and (res['token_logp'][i, s + ln:] == 0).all()
        assert abs(res['log_likelihood'][i] - got.sum()) <= 1e-5 * abs(got.sum()), i


def _eos_params(params, cfg, prompt, p_eos):
    """parameters whose head bias on token 0 makes EOS about p_eos likely right after the prompt"""
    from oracle import progen_ref as O
    row = np.zeros(cfg['seq_len'], np.int64)
    row[1:1 + len(prompt)] = prompt
    l = O.forward(params, row, cfg)[len(prompt)].astype(np.float64)
    rest = np.log(np.exp(l[1:] - l.max()).sum()) + l.max()
    out = {k: {kk: np.array(vv, copy=True) for kk, vv in v.items()} for k, v in params.items()}
    out[HEAD_B]['b'][0] += np.float32(np.log(p_eos / (1 - p_eos)) + rest - l[0])
    return out


def test_eos_ends_sequences_and_the_launch():
    from progen_b200.decode import BatchDecoder
    cfg, params, data, g = load_case('tiny_all_glu')
    n, B = cfg['seq_len'], 24
    prompts = _prompts(np.random.default_rng(4), np.random.default_rng(5).integers(0, 6, B))
    eos = _eos_params(params, cfg, prompts[0], 0.15)
    dec = BatchDecoder(cfg, eos, batch=B)
    res = dec.generate(prompts, temperature=1.0, seed=2)
    end, start = res['end'], res['start']
    assert (end < n).all(), 'every row should have sampled EOS'
    for b in range(B):
        assert res['ids'][b, end[b]] == 0 and (res['ids'][b, start[b]:end[b]] != 0).all()
        assert (res['ids'][b, end[b] + 1:] == 0).all() and (res['token_logp'][b, end[b] + 1:] == 0).all()
        assert res['token_logp'][b, end[b]] < 0
    first = int(start.min()) - 1
    assert res['steps_run'] == int(end.max()) - first
    assert res['steps_run'] < n - 1 - first
    # EOS unreachable: every row runs to max_length
    never = {k: {kk: np.array(vv, copy=True) for kk, vv in v.items()} for k, v in params.items()}
    never[HEAD_B]['b'][0] = -np.inf
    from progen_b200 import ProGen
    model = ProGen(**CASES['tiny_all_glu'])
    out = model.generate(never, prompts, temperature=1.0, seed=2, max_length=100)
    assert not out['finished'].any()
    np.testing.assert_array_equal(out['length'], 100 - out['start'])
    assert (out['tokens'][:, 1:100][np.arange(99)[None, :] + 1 >= out['start'][:, None]] != 0).all()
    assert (out['tokens'][:, 100:] == 0).all()
    out = model.generate(eos, prompts, temperature=1.0, seed=2)
    np.testing.assert_array_equal(out['finished'], True)
    np.testing.assert_array_equal(out['length'], end[:len(prompts)] + 1 - start)


@pytest.mark.parametrize('T', [0.0, 1.0])
def test_nan_logits_end_the_row(T):
    """a row whose logits are all NaN (a diverged checkpoint) has no candidate to draw: it ends with EOS at its first
    position, like a sampled EOS, and reports the NaN log-probability"""
    from progen_b200.decode import BatchDecoder
    cfg, params, data, g = load_case('tiny_all_glu')
    bad = {k: {kk: np.array(vv, copy=True) for kk, vv in v.items()} for k, v in params.items()}
    bad[HEAD_B]['b'][:] = np.nan
    res = BatchDecoder(cfg, bad, batch=12).generate(_prompts(np.random.default_rng(8), [2] * 12), temperature=T,
                                                    top_k=None if T == 0 else 20, top_p=None if T == 0 else 0.9)
    np.testing.assert_array_equal(res['end'], res['start'])
    assert (res['ids'][np.arange(12), res['start']] == 0).all() and np.isnan(res['token_logp'][np.arange(12), res['start']]).all()
    assert res['steps_run'] == 1


def test_seeding_and_batching():
    from progen_b200 import ProGen
    from progen_b200.decode import BatchDecoder
    cfg, params, data, g = load_case('tiny_all_glu')
    n, V = cfg['seq_len'], cfg['num_tokens']
    model = ProGen(**CASES['tiny_all_glu'])
    prompts = ['', 'MKV', np.array([20, 30, 40, 50, 60])]
    kw = dict(num_samples=30, temperature=1.0, top_k=50, top_p=0.9, seed=17)
    a = model.generate(params, prompts, batch_size=64, **kw)
    assert len(a['tokens']) == 90
    np.testing.assert_array_equal(a['prompt_index'], np.repeat(np.arange(3), 30))
    for bs in (64, 12, 30):
        b = model.generate(params, prompts, batch_size=bs, **kw)
        for k in ('tokens', 'token_logp', 'length', 'finished', 'start', 'log_likelihood'):
            np.testing.assert_array_equal(a[k], b[k], err_msg=f'{k} batch_size={bs}')
    c = model.generate(params, prompts, batch_size=64, **{**kw, 'seed': 18})
    assert not np.array_equal(a['tokens'], c['tokens'])
    # 1..8 sequences per launch run another GEMV formulation: logits within round-off, ids equal where the draw is clear
    rows = [np.zeros(0, np.int64), np.array([ord(ch) + 1 for ch in 'MKV']), np.array([20, 30, 40, 50, 60])]
    sids = np.array([0, 31, 62, 89, 45])
    chunk = [rows[int(s) // 30] for s in sids]
    wide = BatchDecoder(cfg, params, batch=12, keep_logits=True)
    ra = wide.generate(chunk + chunk[:4], temperature=1.0, top_k=50, top_p=0.9, seed=17, sample_ids=np.concatenate([sids, sids[:4]]))
    la = wide.logits_all.cpu().numpy()
    narrow = BatchDecoder(cfg, params, batch=5, keep_logits=True)
    rb = narrow.generate(chunk, temperature=1.0, top_k=50, top_p=0.9, seed=17, sample_ids=sids)
    lb = narrow.logits_all.cpu().numpy()
    for i in range(5):
        np.testing.assert_array_equal(ra['ids'][i], a['tokens'][sids[i]])
        diff = np.nonzero(ra['ids'][i] != rb['ids'][i])[0]
        upto = int(diff[0]) if len(diff) else n
        assert np.abs(la[i, :upto - 1] - lb[i, :upto - 1]).max() < 2e-5 * max(1.0, np.abs(la[i, :upto - 1]).max())
        if len(diff):
            t = upto
            _, _, amb = host_draw(la[i, t - 1], 1.0, 50, 0.9, gumbel(17, int(sids[i]), t, V))
            assert amb, (i, t)


H8 = dict(num_tokens=256, dim=256, seq_len=64, depth=2, window_size=16, global_mlp_depth=1, heads=8, dim_head=32)


def _launch_size_plan(cfg, rows, sms, wpb=8):
    """what the kernel would choose for `rows` sequences if it planned for the launch's own row count (as sampler 0 does):
    attention warps per (sequence, head) and SGU splits of the history range"""
    wp = 8
    while wp > 1 and rows * cfg['heads'] * wp > sms * wpb:
        wp //= 2
    cblocks = cfg['dim'] * cfg['ff_mult'] // 2 // 128
    return wp, min(8, max(1, sms // (rows * cblocks)))


@pytest.mark.parametrize('shape,samples,sizes', [('tiny_glu_sgu', 30, (64, 12, 30)), ('h8', 30, (64, 12, 30)),
                                                 ('h8', 3, (8, 5, 3))])
def test_rows_do_not_depend_on_launch_size(shape, samples, sizes):
    """Within one class of rows per launch (9-64, or 2-8) a row is bitwise the same whatever batch_size and chunking put
    it with, on shapes where the attention's warps per (sequence, head) and the SGU's history splits would change with the
    launch's row count (gMLP layers; 8 heads)"""
    from progen_b200 import ProGen
    from oracle import progen_ref as O
    if shape == 'h8':
        kw, cfg = H8, O.make_config(**H8)
        params = O.randomize_params(O.init_params(cfg, 31), 32)
    else:
        kw = CASES[shape]
        cfg, params, _, _ = load_case(shape)
    prompts = ['', 'MKV', np.array([20, 30, 40, 50, 60])]
    N = 3 * samples
    counts = set()                                        # rows of every launch of these calls (ragged chunks padded)
    for bs in sizes:
        per = min(bs, N)
        lo = 9 if per > 8 else (2 if per > 1 else 1)
        counts |= {max(lo, min(per, N - r0)) for r0 in range(0, N, per)}
    sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    assert len({_launch_size_plan(cfg, r, sms) for r in counts}) > 1, 'the shape must exercise launch-size splits'
    model = ProGen(**kw)
    runs = [model.generate(params, prompts, num_samples=samples, temperature=1.0, top_p=0.9, seed=23, batch_size=bs)
            for bs in sizes]
    for bs, b in zip(sizes[1:], runs[1:]):
        for k in ('tokens', 'token_logp', 'length', 'finished', 'log_likelihood'):
            np.testing.assert_array_equal(runs[0][k], b[k], err_msg=f'{k} batch_size={bs} vs {sizes[0]}')


def test_reference_sampler_unaffected_by_generate():
    from progen_b200.decode import BatchDecoder
    cfg, params, data, g = load_case('tiny_glu_sgu')
    one = BatchDecoder(cfg, params, batch=1)
    one.generate([np.array([3, 4])], temperature=0.7, top_k=9, seed=1)
    ids, _, _ = one.sample(g['prime'], top_k=25, add_bos=True, greedy=True)
    np.testing.assert_array_equal(ids, g['sample_bos1'])
    primes = [np.asarray(g['prime']).astype(np.int64)] * 4
    dec = BatchDecoder(cfg, params, batch=4)
    dec.generate(primes[:2], temperature=1.0, top_p=0.5, seed=3)
    a, _, _ = dec.sample(primes, top_k=25, add_bos=True, greedy=False, seed=5)
    b, _, _ = BatchDecoder(cfg, params, batch=4).sample(primes, top_k=25, add_bos=True, greedy=False, seed=5)
    np.testing.assert_array_equal(a, b)


def test_generate_leaves_the_launch_struct_unchanged():
    """generate / generate_queue launch a copy of dec.m, so the struct sample() launches keeps every byte through a static,
    a queue, a forward-prefilled and a refused call, with every constraint field set"""
    from progen_b200 import ProGen
    from progen_b200.decode import BatchDecoder
    from progen_b200.lib import ProgenError
    cfg, params, data, g = load_case('tiny_glu_sgu')
    V = cfg['num_tokens']
    model = ProGen(**CASES['tiny_glu_sgu'])
    model._ensure_loaded(params)
    dec = BatchDecoder(cfg, params, batch=4)
    prompts = _prompts(np.random.default_rng(12), [3, 3, 5, 1])
    bias = np.where(np.arange(V) % 5 == 2, -np.inf, 0.1).astype(np.float32)
    kw = dict(temperature=0.8, top_k=20, top_p=0.9, seed=7, logit_bias=bias, min_new_tokens=2, repetition_penalty=1.2,
              repetition_window=8)
    table = lambda rows: (np.zeros((1, 4, V), np.float32), np.zeros(rows, np.int64))
    before = bytes(dec.m)
    dec.generate(prompts, position_bias=table(4), **kw)
    assert bytes(dec.m) == before, 'static generate'
    dec.generate_queue(prompts * 2, slots=3, position_bias=table(8), **kw)
    assert bytes(dec.m) == before, 'generate_queue'
    P = dec.prefill(model.engine, prompts[:2])
    res = dec.generate(prompts[:2], prefilled=P, position_bias=table(2), **kw)
    assert P == 3 and res['prefill_s'] == 0.0
    assert bytes(dec.m) == before, 'forward-prefilled generate'
    for bad in (dict(top_k=0), dict(position_bias=table(3)), dict(prefilled=4)):
        with pytest.raises(ProgenError):
            dec.generate(prompts, **{**kw, **bad})
    assert bytes(dec.m) == before, 'refused generate'


def test_bf16_weights_generate_and_mostly_agree():
    from progen_b200 import ProGen
    cfg, params, data, g = load_case('tiny_all_glu')
    prompt = np.asarray(g['prime']).astype(np.int64)
    a = ProGen(**CASES['tiny_all_glu']).generate(params, [prompt], temperature=0.0)
    b = ProGen(**CASES['tiny_all_glu'], mixed_precision=True).generate(params, [prompt], temperature=0.0)
    s = int(a['start'][0])
    assert b['length'][0] >= 1 and (a['tokens'][0, :s + 2] == b['tokens'][0, :s + 2]).all()
    assert np.isfinite(b['log_likelihood']).all()


def test_generate_cli(tmp_path):
    from progen_b200.checkpoint import file_save_checkpoint
    from oracle import progen_ref as O
    kwargs = dict(num_tokens=256, dim=128, seq_len=128, depth=2, window_size=64, global_mlp_depth=1, heads=2, dim_head=64)
    params = O.randomize_params(O.init_params(O.make_config(**kwargs), 91), 92)
    (tmp_path / 'ckpts').mkdir()
    file_save_checkpoint(tmp_path / 'ckpts', dict(next_seq_index=0, params=params, optim_state=None, model_config=kwargs,
                                                  run_id=None))
    env = dict(os.environ, PYTHONPATH=ROOT)

    def run(out):
        r = subprocess.run([sys.executable, os.path.join(ROOT, 'generate.py'), '--checkpoint_path', str(tmp_path / 'ckpts'),
                            '--prompt', '[Tax=Mammalia] #', '--prompt', 'MK', '--num_samples', '5', '--seed', '4',
                            '--top_p', '0.95', '--max_length', '100', '--output', str(out)],
                           cwd=str(tmp_path), env=env, capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
        assert 'sequences/s' in r.stdout and 'generated tokens/s' in r.stdout
        return out.read_text()

    text = run(tmp_path / 'a.fasta')
    lines = text.splitlines()
    heads = lines[0::2]
    assert len(heads) == 10 and len(lines) == 20
    pat = re.compile(r'^>(\d+) prompt=(\d+) sample=(\d+) log_likelihood=(-?[\d.]+) length=(\d+) eos=([01])$')
    for row, (h, body) in enumerate(zip(heads, lines[1::2])):
        m = pat.match(h)
        assert m, h
        assert int(m[1]) == row and int(m[2]) == row // 5 and int(m[3]) == row % 5
        assert float(m[4]) <= 0 and len(body) == int(m[5]) - int(m[6])
    assert run(tmp_path / 'b.fasta') == text
