"""Position-specific generation constraints (the position tables of sampler 1 in csrc/decode_persist.cu;
`BatchDecoder.generate(position_bias=)`, `ProGen.generate(position_bias=, fixed=)`): a zero table changes no bit, an exact
host replay of the adjusted logits, fixed residues hold in every batch-tile class, greedy generation against the float64
oracle, the drawn distribution at one offset, queue and chunking equal the static schedule, forward prefill, and the
refusals."""
import ctypes as C

import numpy as np
import pytest
import torch

from golden_util import load_case, CASES
from test_gpu_generate import gumbel, host_draw, _drawn, _eos_params, _prompts
from test_gpu_generate_constraints import adjust, _random_bias

pytestmark = pytest.mark.gpu
AA = 'ACDEFGHIKLMNPQRSTVWY'
OUT_KEYS = ('tokens', 'token_logp', 'start', 'length', 'finished', 'log_likelihood')
GRID = ((0.0, None, None), (1.0, None, None), (0.7, 5, None), (1.5, None, 0.9), (1.0, 40, 0.5))


def _table(rng, L, V, allowed, banned=0.2):
    """[L, V] finite values of both signs with about `banned` of the ids at -inf; EOS banned at half the offsets, and at
    every offset one id of `allowed` kept, so no offset is left without a candidate"""
    t = (rng.standard_normal((L, V)) * 1.5).astype(np.float32)
    t[rng.random((L, V)) < banned] = -np.inf
    t[:, 0] = np.where(rng.random(L) < 0.5, 0.0, -np.inf).astype(np.float32)
    t[np.arange(L), rng.choice(allowed, L)] = 0.25
    return t


def _assert_equal(a, b, what, keys=OUT_KEYS):
    for k in keys:
        np.testing.assert_array_equal(a[k], b[k], err_msg=f'{k} {what}')


@pytest.mark.parametrize('B', [1, 8, 24])
def test_zero_table_changes_no_bit(B):
    """an all-zero table (which runs the constrained code) equals no table bit for bit, static and (B > 1) queue, over the
    temperature / top-k / top-p grid of test_neutral_constraints_change_no_bit"""
    from progen_b200.decode import BatchDecoder
    cfg, params, data, g = load_case('tiny_all_glu')
    V, n = cfg['num_tokens'], cfg['seq_len']
    rng = np.random.default_rng(B)
    dec = BatchDecoder(cfg, params, batch=B)
    prompts = _prompts(rng, rng.integers(0, 7, B))
    qprompts = _prompts(rng, rng.integers(0, 7, 3 * B))
    for T, top_k, top_p in GRID:
        kw = dict(temperature=T, top_k=top_k, top_p=top_p, seed=21)
        zero = (np.zeros((2, n, V), np.float32), np.arange(B) % 2)
        a = dec.generate(prompts, **kw)
        b = dec.generate(prompts, position_bias=zero, **kw)
        _assert_equal(a, b, f'static T={T} top_k={top_k} top_p={top_p}', ('ids', 'token_logp', 'end', 'steps_run'))
        if B > 1:
            zq = (np.zeros((1, 7, V), np.float32), np.zeros(3 * B, np.int64))
            a = dec.generate_queue(qprompts, max_length=48, **kw)
            b = dec.generate_queue(qprompts, max_length=48, position_bias=zq, **kw)
            _assert_equal(a, b, f'queue T={T} top_k={top_k} top_p={top_p}', ('ids', 'token_logp', 'end', 'steps_run'))


def _replay(dec, res, lg, tables, tmap, seed, sids, T, top_k, top_p, ck, max_length):
    """(draws, unambiguous) of a launch; asserts every id is a kept candidate and equals the host replay where unambiguous"""
    V = lg.shape[-1]
    total = unamb = 0
    for b in range(len(res['ids'])):
        ids, st = res['ids'][b], int(res['start'][b])
        for t in _drawn(res, b, max_length):
            a = adjust(lg[b, t - 1], ids, t - 1, st, **ck)
            j = t - st
            if tmap[b] >= 0 and j < tables.shape[1]:
                a = a + tables[tmap[b], j]                   # float32, its own rounding (EOS ban: -inf either way)
            want, keep, amb = host_draw(a, T, top_k, top_p, gumbel(seed, int(sids[b]), t, V))
            got = int(ids[t])
            where = (T, top_k, top_p, b, t, got, want)
            assert a[got] > -np.inf and keep[got], where
            total += 1
            if not amb:
                unamb += 1
                assert got == want, where
    return total, unamb


def test_position_tables_match_host_replay():
    """per-prompt tables of different lengths (zero-padded to one launch table), prompts of different lengths, random
    finite values with -inf, with the logit bias, the penalty and min_new_tokens, over T x top_k x top_p at B = 16: every
    id is a candidate of the adjusted logits and equals the float32 host replay wherever the draw is unambiguous; >= 99 %
    of draws are"""
    from progen_b200.decode import BatchDecoder
    from progen_b200.progen import launch_tables
    cfg, params, data, g = load_case('tiny_all_glu')
    V, B, ml = cfg['num_tokens'], 16, 64
    rng = np.random.default_rng(41)
    prompts = _prompts(rng, rng.integers(0, 9, B))
    bias = _random_bias(np.random.default_rng(70), V)
    allowed = np.flatnonzero(np.isfinite(bias[1:])) + 1
    tabs = [_table(rng, L, V, allowed) for L in (3, 20, 40)]
    tables, tmap = launch_tables(tabs, rng.integers(-1, 3, B), np.arange(B))
    assert tables.shape == (3, 40, V) and (tmap >= 0).sum() >= 8
    dec = BatchDecoder(cfg, params, batch=B, keep_logits=True)
    seed = 0xFEED_0123_4567
    sids = np.arange(B, dtype=np.int64) * 7 + (1 << 34)
    total = unamb = 0
    for cs in (dict(), dict(logit_bias=bias, repetition_penalty=1.3, repetition_window=8, min_new_tokens=5)):
        ck = dict(bias=cs.get('logit_bias'), theta=cs.get('repetition_penalty', 1.0),
                  window=cs.get('repetition_window', 0), min_new=cs.get('min_new_tokens', 0))
        for T in (0.0, 0.7, 1.5):
            for top_k in (None, 5):
                for top_p in (None, 0.9):
                    res = dec.generate(prompts, temperature=T, top_k=top_k, top_p=top_p, seed=seed, sample_ids=sids,
                                       max_length=ml, position_bias=(tables, tmap), **cs)
                    lg = dec.logits_all.cpu().numpy()
                    t_, u_ = _replay(dec, res, lg, tables, tmap, seed, sids, T, top_k, top_p, ck, ml)
                    total += t_
                    unamb += u_
    assert total > 3000 and unamb >= 0.99 * total, (unamb, total)


def _fixed_sets(rng, reach):
    """three per-prompt fixed dicts: a few residues, one dense run, and EOS-forcing room (offsets within reach)"""
    a = {int(k): AA[rng.integers(20)] for k in rng.choice(np.arange(1, reach + 1), 4, replace=False)}
    b = {k: 'C' if k % 2 else 'H' for k in range(2, min(reach, 9))}
    return [a, b, None]


def _check_fixed(out, fixed_per_row, max_length, V):
    """fixed residues at start + k - 1; no row ends before its last fixed offset unless max_length cut it"""
    for i in range(len(out['tokens'])):
        f = fixed_per_row[i]
        if not f:
            continue
        s, ln, fin = int(out['start'][i]), int(out['length'][i]), bool(out['finished'][i])
        for k, res in f.items():
            c = ord(res) + 1 if isinstance(res, str) else int(res)
            if s + k - 1 < max_length:
                assert out['tokens'][i, s + k - 1] == c, (i, k, res, out['tokens'][i, s:s + ln])
        if fin:
            assert ln >= max(f) + 1, (i, ln, max(f))               # EOS only after the last fixed residue


def _check_logp_vs_score(model, params, out, fixed_per_row):
    """token_logp at the fixed positions equals what `score` reports for the returned rows (the bound of
    test_gpu_generate.py::test_token_logp_equals_score)"""
    rows = np.concatenate([out['tokens'], np.zeros((len(out['tokens']), 1), np.int64)], axis=1)
    sc = model.score(params, rows, return_tokens=True)['token_logp']
    checked = 0
    for i in range(len(rows)):
        s, ln = int(out['start'][i]), int(out['length'][i])
        want = sc[i, s - 1:s - 1 + ln].astype(np.float64)
        got = out['token_logp'][i, s:s + ln].astype(np.float64)
        assert np.abs(got - want).max() < 1e-4, i
        for k in (fixed_per_row[i] or {}):
            if k <= ln:
                assert abs(float(out['token_logp'][i, s + k - 1]) - float(sc[i, s + k - 2])) < 1e-4, (i, k)
                checked += 1
    assert checked > 0


@pytest.mark.parametrize('bs', [1, 5, 20])
@pytest.mark.parametrize('mp', [False, True])
def test_fixed_residues_hold(bs, mp):
    """batch-tile classes 1, 2-8 and 9-64 (queue), fp32 and bf16 weights, EOS made likely: every row carries its fixed
    residues and does not end before its last one; fp32: token_logp equals `score` at the fixed positions"""
    from progen_b200 import ProGen
    cfg, params, data, g = load_case('tiny_glu_sgu')
    V, n = cfg['num_tokens'], cfg['seq_len']
    rng = np.random.default_rng(bs + 100 * mp)
    prompts = _prompts(rng, [0, 3, 7])
    eos = _eos_params(params, cfg, prompts[1], 0.2)
    fixed = _fixed_sets(rng, n - 1 - 7 - 1)
    model = ProGen(**CASES['tiny_glu_sgu'], mixed_precision=mp)
    samples = 2 if bs == 1 else 12
    out = model.generate(eos, prompts, num_samples=samples, batch_size=bs, seed=5, top_p=0.95, fixed=fixed)
    per_row = [fixed[i // samples] for i in range(len(out['tokens']))]
    _check_fixed(out, per_row, n, V)
    assert out['finished'].any()
    if not mp:
        _check_logp_vs_score(model, eos, out, per_row)


def test_fixed_residues_hold_config3_width():
    """the depth-3 config-3 stack (d1024 h16 w512 n2048), 9-64-row class, fixed residues up to offset 150"""
    from progen_b200 import ProGen
    from test_gpu_large_config_inference import _model as large
    kw, cfg, params = large('cfg3')
    rng = np.random.default_rng(3)
    prompts = [rng.integers(1, 256, L).astype(np.int64) for L in (0, 3, 40)]
    eos = _eos_params(params, cfg, prompts[1], 0.02)
    fixed = {1: 'M', 17: 'W', 60: 'K', 150: 'D'}
    out = ProGen(**kw).generate(eos, prompts, num_samples=4, batch_size=12, seed=13, max_length=256, fixed=fixed)
    _check_fixed(out, [fixed] * len(out['tokens']), 256, cfg['num_tokens'])
    assert (out['length'] >= 150).all()


@pytest.mark.parametrize('name', [n for n in CASES if n != 'cfg1'])
def test_greedy_with_fixed_residues_matches_oracle(name):
    """greedy generation with fixed residues and a profile: at every drawn position the id is the float64 oracle's argmax
    of the re-forward of the returned row plus the table row (the fixed id where one is fixed); where the oracle's top
    two are within 1e-3 the id is one of them"""
    from progen_b200 import ProGen
    from progen_b200.progen import position_tables
    from oracle import progen_ref as O
    cfg, params, data, g = load_case(name)
    V, n = cfg['num_tokens'], cfg['seq_len']
    rng = np.random.default_rng(9)
    prompts = _prompts(rng, [0, 1, 7])
    prof = (rng.standard_normal((12, V)) * 0.5).astype(np.float32)
    fixed = {2: 'W', 5: 'C', 6: 'H', 11: 'Y'}
    out = ProGen(**CASES[name]).generate(params, prompts, temperature=0.0, position_bias=prof, fixed=fixed)
    tables, pt = position_tables([1 + len(p) for p in prompts], V, n, n, prof, fixed)
    checked = 0
    for i in range(len(prompts)):
        tab = tables[pt[i]]
        s, ln = int(out['start'][i]), int(out['length'][i])
        ref = O.forward(params, out['tokens'][i], cfg)
        for t in range(s, s + ln):
            a = ref[t - 1].astype(np.float64) + (tab[t - s] if t - s < len(tab) else 0.0)
            got = int(out['tokens'][i, t])
            if t - s + 1 in fixed:
                assert got == ord(fixed[t - s + 1]) + 1, (i, t)
                continue
            top = np.sort(a[np.isfinite(a)])[::-1]
            if top[0] - top[1] > 1e-3:
                assert got == int(np.argmax(a)), (i, t, got)
                checked += 1
            else:
                assert a[got] >= top[1] - 1e-3, (i, t, got)
    assert checked > 10


def test_profile_row_distribution_chi_square():
    """offset 1 of an empty prompt with a profile row over the amino acids: 4096 draws against softmax(l + b) over the
    candidates, l the oracle's float64 BOS logits"""
    from scipy import stats
    from progen_b200.decode import BatchDecoder
    from oracle import progen_ref as O
    cfg, params, data, g = load_case('tiny_all_glu')
    n, V, B, runs = cfg['seq_len'], cfg['num_tokens'], 64, 64
    rng = np.random.default_rng(12)
    b = np.full(V, -np.inf, np.float32)
    aa = [ord(ch) + 1 for ch in AA]
    b[aa] = rng.uniform(-1.0, 3.0, len(aa)).astype(np.float32)
    l = O.forward(params, np.zeros(n, np.int64), cfg)[0].astype(np.float64)
    a = l + b
    keep = np.isfinite(a)
    probs = np.exp(np.where(keep, a - a[keep].max(), -np.inf))
    probs /= probs.sum()
    dec = BatchDecoder(cfg, params, batch=B)
    counts = np.zeros(V, np.int64)
    for r in range(runs):
        res = dec.generate([np.zeros(0, np.int64)] * B, temperature=1.0, seed=17, sample_ids=np.arange(r * B, (r + 1) * B),
                           max_length=2, position_bias=(b[None, None, :], np.zeros(B, np.int64)))
        counts += np.bincount(res['ids'][:, 1], minlength=V)
    assert counts.sum() == B * runs == 4096
    assert counts[~keep].sum() == 0
    exp_counts = probs * counts.sum()
    big = exp_counts >= 5
    obs = np.append(counts[big], counts[~big].sum())
    exp_ = np.append(exp_counts[big], exp_counts[~big].sum())
    if exp_[-1] == 0:
        obs, exp_ = obs[:-1], exp_[:-1]
    chi2 = ((obs - exp_) ** 2 / exp_).sum()
    pval = 1.0 - stats.chi2.cdf(chi2, len(obs) - 1)
    assert len(obs) >= 5 and pval > 1e-3, (chi2, len(obs), pval)


def _per_prompt_inputs(rng, k, V, n):
    """k prompts, each with its own profile (some None) and fixed residues (some None)"""
    prompts = [rng.integers(1, 256, L).astype(np.int64) for L in rng.integers(0, 6, k)]
    allowed = np.arange(1, V)
    pb = [None if i % 3 == 2 else _table(rng, int(rng.integers(4, 30)), V, allowed, banned=0.05) for i in range(k)]
    fx = [None if i % 4 == 3 else {int(rng.integers(1, 20)): AA[i % 20]} for i in range(k)]
    for b, f in zip(pb, fx):                              # the profile keeps each fixed residue allowed
        for j, ch in (f or {}).items():
            if b is not None and j <= len(b):
                b[j - 1, ord(ch) + 1] = 0.0
    return prompts, pb, fx


@pytest.mark.parametrize('bs', [6, 20])
def test_queue_equals_static_and_chunking(bs, monkeypatch):
    """`ProGen.generate` (queue, per-prompt tables) equals plan_launches + BatchDecoder.generate with the same tables bit
    for bit; a table budget lowered so that every launch holds at most 3 tables (more chunks) changes no bit"""
    import progen_b200.progen as P
    from progen_b200 import ProGen
    from progen_b200.decode import BatchDecoder
    cfg, params, data, g = load_case('tiny_glu_sgu')
    V, n = cfg['num_tokens'], cfg['seq_len']
    rng = np.random.default_rng(bs)
    prompts, pb, fx = _per_prompt_inputs(rng, 9, V, n)
    eos = _eos_params(params, cfg, prompts[0], 0.1)
    samples = 12
    kw = dict(temperature=1.0, top_p=0.95, seed=8)
    model = ProGen(**CASES['tiny_glu_sgu'])
    got = model.generate(eos, prompts, num_samples=samples, batch_size=bs, position_bias=pb, fixed=fx, **kw)
    # static schedule with the same tables
    tables, pt = P.position_tables([1 + len(p) for p in prompts], V, n, n, pb, fx)
    N = len(prompts) * samples
    row_table = pt[np.arange(N) // samples]
    rows = [prompts[r // samples] for r in range(N)]
    dec = BatchDecoder(cfg, eos, batch=min(bs, N))
    want = dict(tokens=np.zeros((N, n), np.int64), token_logp=np.zeros((N, n), np.float32), start=np.zeros(N, np.int64),
                end=np.zeros(N, np.int64))
    for sids, real in P.plan_launches([len(a) for a in rows], bs):
        res = dec.generate([rows[r] for r in sids], sample_ids=sids, position_bias=P.launch_tables(tables, row_table, sids),
                           **kw)
        r = sids[:real]
        want['tokens'][r], want['token_logp'][r] = res['ids'][:real], res['token_logp'][:real]
        want['start'][r], want['end'][r] = res['start'][:real], res['end'][:real]
    end = want.pop('end')
    want['finished'] = end < n
    want['length'] = np.where(want['finished'], end + 1, n) - want['start']
    want['log_likelihood'] = want['token_logp'].astype(np.float64).sum(axis=-1)
    _assert_equal(got, want, f'queue vs static bs={bs}')
    per_row = [fx[i // samples] for i in range(N)]
    _check_fixed(got, per_row, n, V)
    # a lower table budget: more, smaller chunks, the same bits
    table_bytes = max(t.nbytes for t in tables)
    monkeypatch.setattr(P, 'QUEUE_TABLE_BYTES', 3 * table_bytes)
    slots, chunks = P.plan_queue(N, bs, row_table, table_bytes)
    assert len(chunks) > 1
    low = model.generate(eos, prompts, num_samples=samples, batch_size=bs, position_bias=pb, fixed=fx, **kw)
    _assert_equal(got, low, f'lowered budget bs={bs}')


@pytest.mark.parametrize('name,mp', [('tiny_glu_sgu', False), ('tiny_all_glu', True)])
def test_forward_prefill_with_tables(name, mp):
    """prefill='forward': fixed residues hold, and the drawn ids replay exactly on the launch's own logits"""
    from progen_b200 import ProGen
    from progen_b200.decode import BatchDecoder
    from progen_b200.progen import position_tables, launch_tables
    cfg, params, data, g = load_case(name)
    V, n = cfg['num_tokens'], cfg['seq_len']
    rng = np.random.default_rng(77)
    prompts = _prompts(rng, [6, 6, 2])
    fixed = [{1: 'A', 4: 'W'}, {3: 'C', 9: 'H'}, None]
    prof = [None, None, _table(rng, 10, V, np.arange(1, V), banned=0.1)]
    model = ProGen(**CASES[name], mixed_precision=mp)
    out = model.generate(params, prompts, num_samples=4, batch_size=12, seed=4, prefill='forward', fixed=fixed,
                         position_bias=prof)
    _check_fixed(out, [fixed[i // 4] for i in range(12)], n, V)
    # the replay: one launch of the length-6 prompts, prefilled by the forward, with keep_logits
    tables, pt = position_tables([7, 7], V, n, n, None, fixed[:2])
    tabs, tmap = launch_tables(tables, pt, np.arange(2))
    dec = BatchDecoder(cfg, params, batch=2, weights_dtype=torch.bfloat16 if mp else torch.float32, keep_logits=True)
    P = dec.prefill(model.engine, prompts[:2])
    assert P == 6
    sids = np.array([3, 5])
    for T, top_k, top_p in GRID:
        res = dec.generate(prompts[:2], temperature=T, top_k=top_k, top_p=top_p, seed=99, sample_ids=sids, prefilled=P,
                           position_bias=(tabs, tmap))
        lg = dec.logits_all.cpu().numpy()
        total, unamb = _replay(dec, res, lg, tabs, tmap, 99, sids, T, top_k, top_p, dict(), n)
        assert unamb >= 0.95 * total and total > 10, (T, top_k, top_p, unamb, total)
        for b in range(2):
            s = int(res['start'][b])
            for k, ch in fixed[b].items():
                assert res['ids'][b, s + k - 1] == ord(ch) + 1
        P = dec.prefill(model.engine, prompts[:2])


def test_refusals():
    """ProGen.generate refuses bad tables before any launch; progen_decode_run refuses a table with sampler 0, a table
    without a row map (and a map without a table) and a length outside [1, n]"""
    from progen_b200 import ProGen, lib as L
    from progen_b200.decode import BatchDecoder
    cfg, params, data, g = load_case('tiny_glu_sgu')
    V, n = cfg['num_tokens'], cfg['seq_len']
    model = ProGen(**CASES['tiny_glu_sgu'])
    model.generate(params, 'MK', max_length=8)            # the decoder exists: count launches from here
    lb = np.zeros(V, np.float32)
    lb[ord('W') + 1] = -np.inf
    before = L.load().progen_launch_count()
    bad = [dict(fixed={0: 'A'}), dict(fixed={n - 2: 'A'}), dict(fixed={5: 'A'}, max_length=6), dict(fixed={1: 300}),
           dict(fixed={1: 'Ā'}), dict(fixed=[{1: 'A'}]), dict(position_bias=[None, None, None]),
           dict(position_bias=np.zeros((n + 1, V))), dict(position_bias=np.full((3, V), np.nan)),
           dict(fixed={2: 'W'}, logit_bias=lb), dict(fixed={3: 'W'}, position_bias=np.where(np.arange(V) == ord('W') + 1,
                                                                                       -np.inf, 0)[None].repeat(4, 0))]
    for kw in bad:
        with pytest.raises(L.ProgenError):
            model.generate(params, ['MK', 'A'], **kw)
    torch.cuda.synchronize()
    assert L.load().progen_launch_count() == before
    # BatchDecoder's own checks
    dec = BatchDecoder(cfg, params, batch=4)
    for pbias in ((np.zeros((2, 3, V - 2), np.float32), np.zeros(2)), (np.zeros((2, 3, V), np.float32), np.array([0, 2])),
                  (np.zeros((2, 3, V), np.float32), np.array([-2, 0])), (np.zeros((2, 3, V), np.float32), np.zeros(3)),
                  (np.full((1, 3, V), np.inf, np.float32), np.zeros(2))):
        with pytest.raises(L.ProgenError):
            dec.generate(_prompts(np.random.default_rng(0), [1, 2]), position_bias=pbias)
    # the C entry point
    m = dec.m
    tab = torch.zeros(2, n, V, device=dec.dev)
    tmap = torch.zeros(4, dtype=torch.int32, device=dec.dev)
    cnt = torch.zeros(4, dtype=torch.int32, device=dec.dev)
    sid = torch.zeros(4, dtype=torch.int64, device=dec.dev)
    end = torch.full((4,), n, dtype=torch.int32, device=dec.dev)

    def run(**f):
        base = dict(B=4, sampler=1, temperature=1.0, top_p=1.0, sample_id=sid.data_ptr(), end=end.data_ptr(),
                    n_ended=cnt.data_ptr(), steps_run=cnt.data_ptr() + 4, pos0=0, nsteps=2,
                    position_bias=tab.data_ptr(), position_bias_table=tmap.data_ptr(), position_bias_len=n)
        base.update(f)
        saved = {k: getattr(m, k) for k in base}
        for k, v in base.items():
            setattr(m, k, v)
        try:
            dec.grid_bar.zero_()
            cnt.zero_()
            return dec.lib.progen_decode_run(C.byref(m), L.stream())
        finally:
            for k, v in saved.items():
                setattr(m, k, v)

    torch.cuda.synchronize()
    before = dec.lib.progen_launch_count()
    refused = {'sampler 0 with a table': dict(sampler=0, temperature=0.0, top_p=0.0),
               'table without a map': dict(position_bias_table=0),
               'map without a table': dict(position_bias=0),
               'length 0': dict(position_bias_len=0),
               'length n + 1': dict(position_bias_len=n + 1)}
    for what, f in refused.items():
        assert run(**f) == -2, what                       # PROGEN_ERR_ARG
    assert dec.lib.progen_launch_count() == before
    assert run() == 0                                     # well formed: it launches
    assert dec.lib.progen_launch_count() == before + 1
    torch.cuda.synchronize()
