"""Motif constraints in the standard sampler (progen_motif_t, csrc/decode_persist.cu; `ProGen.generate(require=,
avoid=)`): neutral patterns change no bit, an exact host replay of the bans, every row satisfies the patterns (static
and queued launches, tight max_length, forward prefill), queue equals static launches, a contradiction ends rows with
EOS, the first draw's distribution, token log-probabilities against `score`, the C entry point's refusals, and
generate.py --require / --avoid."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from golden_util import load_case, CASES
from test_gpu_generate import gumbel, host_draw, _drawn, _eos_params, _prompts
from test_gpu_generate_constraints import AA, _aa_bias, adjust
from test_motif_cpu import to_regex, ZINC_FINGER

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT_KEYS = ('tokens', 'token_logp', 'start', 'length', 'finished', 'log_likelihood', 'motif_match')
# Avoided: a glycosylation-like site and a pair of residues that a 20-letter alphabet draws about every 8 positions.
# Their last elements exclude every residue the zinc finger's mandatory positions need (C, H, LIVMFYWC), so they can
# never ban the only residue that keeps the requirement reachable: rows never reach a dead end, and all must match.
AVOID = ['N-{P}-[ST]-[AGS]', '[ACDEFG]-[ADEG]']
SHORTEST = 21                                             # residues of the zinc finger's shortest match


def _decode(cfg, params, B, **kw):
    from progen_b200.decode import BatchDecoder
    return BatchDecoder(cfg, params, batch=B, **kw)


def _motif(require, avoid, V=256, bias=None):
    from progen_b200.motif import Motif
    return Motif(require, avoid, V, bias)


def _rows(out):
    """each row's generated residues (before EOS) as text"""
    gen = out['length'] - out['finished']
    return [''.join(chr(c - 1) for c in out['tokens'][i, s:s + g]) for i, (s, g) in enumerate(zip(out['start'], gen))]


def _satisfied(out, require, avoid):
    """per row: the independent `re` translation agrees that the require pattern occurs and no avoided one does"""
    rx = None if require is None else to_regex(require)
    ax = [to_regex(a) for a in avoid or []]
    return np.array([(rx is None or rx.search(s) is not None) and not any(a.search(s) for a in ax) for s in _rows(out)])


def _as_out(res, max_length):
    """BatchDecoder.generate's dict in ProGen.generate's keys"""
    fin = res['end'] < max_length
    return dict(tokens=res['ids'], start=res['start'], finished=fin,
                length=np.where(fin, res['end'] + 1, max_length) - res['start'])


@pytest.mark.parametrize('B', [1, 8, 24])
def test_neutral_patterns_change_no_bit(B):
    """'<x' with min_new_tokens=1 equals min_new_tokens=1 alone; an avoided pattern with a letter the alphabet bans
    equals the alphabet alone"""
    cfg, params, data, g = load_case('tiny_all_glu')
    V = cfg['num_tokens']
    rng = np.random.default_rng(B)
    prompts = _prompts(rng, rng.integers(0, 7, B))
    dec = _decode(cfg, params, B)
    for T, top_k, top_p in ((0.0, None, None), (1.0, None, None), (0.7, 5, 0.9)):
        kw = dict(temperature=T, top_k=top_k, top_p=top_p, seed=21, max_length=90)
        a = dec.generate(prompts, min_new_tokens=1, **kw)
        b = dec.generate(prompts, min_new_tokens=1, motif=_motif('<x', None, V), **kw)
        c = dec.generate(prompts, logit_bias=_aa_bias(), **kw)
        d = dec.generate(prompts, logit_bias=_aa_bias(), motif=_motif(None, ['A-B-x', 'W-O'], V, _aa_bias()), **kw)
        for k in ('ids', 'token_logp', 'end', 'steps_run'):
            np.testing.assert_array_equal(a[k], b[k], err_msg=f'require <x: {k} T={T}')
            np.testing.assert_array_equal(c[k], d[k], err_msg=f'avoid banned letters: {k} T={T}')


def test_motif_bans_match_host_replay():
    """B = 16, with the constraint sets of the unconstrained replay plus a required and two avoided patterns: every drawn
    id is a candidate of the adjusted, motif-banned logits and equals the host replay wherever the draw is unambiguous"""
    cfg, params, data, g = load_case('tiny_all_glu')
    V, B, ml = cfg['num_tokens'], 16, 64
    rng = np.random.default_rng(17)
    prompts = _prompts(rng, rng.integers(0, 9, B))
    dec = _decode(cfg, params, B, keep_logits=True)
    seed = 0xFEED_0123_4567
    sids = np.arange(B, dtype=np.int64) * 7 + (1 << 34)
    total = unamb = 0
    sets = [dict(logit_bias=_aa_bias()), dict(logit_bias=_aa_bias(), repetition_penalty=1.3, repetition_window=8),
            dict(min_new_tokens=5)]
    for cs in sets:
        motif = _motif('C-x(2,4)-C-x(3)-[LIVMFYWC]', ['[ACDEFG]-[ACDEFG]', 'K-K>'], V, cs.get('logit_bias'))
        ck = dict(bias=cs.get('logit_bias'), theta=cs.get('repetition_penalty', 1.0), window=cs.get('repetition_window', 0),
                  min_new=cs.get('min_new_tokens', 0))
        for T in (0.0, 0.7, 1.5):
            for top_k, top_p in ((None, None), (5, 0.9)):
                res = dec.generate(prompts, temperature=T, top_k=top_k, top_p=top_p, seed=seed, sample_ids=sids,
                                   max_length=ml, motif=motif, **cs)
                lg = dec.logits_all.cpu().numpy()
                for b in range(B):
                    ids, st = res['ids'][b], int(res['start'][b])
                    state = motif.initial_state()
                    for t in _drawn(res, b, ml):
                        a = adjust(lg[b, t - 1], ids, t - 1, st, **ck)
                        a[motif.banned(state, t == st, ml - t - 1)] = -np.inf
                        got = int(ids[t])
                        where = (cs, T, top_k, top_p, b, t, got)
                        if not np.isfinite(a).any():
                            assert got == 0, where                 # no candidate: EOS
                            continue
                        want, keep, amb = host_draw(a, T, top_k, top_p, gumbel(seed, int(sids[b]), t, V))
                        assert a[got] > -np.inf and keep[got], where
                        total += 1
                        if not amb:
                            unamb += 1
                            assert got == want, where + (want,)
                        if got:
                            state = motif.advance(state, got, t == st)
    assert total > 3000 and unamb >= 0.99 * total, (unamb, total)


def _check_all(out, require, avoid, max_length):
    ok = _satisfied(out, require, avoid)
    assert ok.all(), np.flatnonzero(~ok)[:10]
    assert out['motif_match'].all()
    unfinished = ~out['finished']
    assert (out['start'][unfinished] + out['length'][unfinished] == max_length).all()


@pytest.mark.parametrize('bs', [1, 8, 24])
@pytest.mark.parametrize('tight', [False, True])
def test_every_row_satisfies_the_patterns(bs, tight):
    """ProGen.generate (a queue for bs > 1) and static launches of BatchDecoder.generate: every row contains the zinc
    finger and no avoided pattern (rows seldom meet the pattern by chance, so most are forced into it by the lookahead
    near max_length), and with a tight max_length (start + shortest match + 3) rows run to max_length unfinished"""
    from progen_b200 import ProGen
    cfg, params, data, g = load_case('tiny_all_glu')
    V, n = cfg['num_tokens'], cfg['seq_len']
    prompts = [np.array([ord(ch) + 1 for ch in p], np.int64) for p in ('MK', 'MSTV')]
    ml = 1 + 4 + SHORTEST + 3 if tight else n
    eos = _eos_params(params, cfg, prompts[0], 0.2)
    kw = dict(temperature=1.0, top_p=0.95, seed=5, max_length=ml, logit_bias=_aa_bias(), require=ZINC_FINGER, avoid=AVOID)
    samples = 12 if bs == 1 else 48
    out = ProGen(**CASES['tiny_all_glu']).generate(eos, prompts, num_samples=samples, batch_size=bs, **kw)
    _check_all(out, ZINC_FINGER, AVOID, ml)
    if tight:
        assert (~out['finished']).any()
    if bs > 1:                                            # static launches on the same rows
        dec = _decode(cfg, eos, bs)
        rows = [prompts[i % 2] for i in range(bs)]
        res = dec.generate(rows, temperature=1.0, top_p=0.95, seed=5, max_length=ml, logit_bias=_aa_bias(),
                           motif=_motif(ZINC_FINGER, AVOID, V, _aa_bias()))
        st = _as_out(res, ml)
        ok = _satisfied(st, ZINC_FINGER, AVOID)
        assert ok.all(), np.flatnonzero(~ok)


@pytest.mark.parametrize('bs', [6, 20])
def test_queue_equals_static_launches(bs):
    """ProGen.generate's queue launches equal plan_launches + BatchDecoder.generate with the same patterns bit for bit"""
    import progen_b200.progen as P
    from progen_b200 import ProGen
    cfg, params, data, g = load_case('tiny_glu_sgu')
    V, n = cfg['num_tokens'], cfg['seq_len']
    prompts = [np.array([ord(ch) + 1 for ch in p], np.int64) for p in ('', 'M', 'MKV')]
    eos = _eos_params(params, cfg, prompts[1], 0.15)
    require, avoid = 'C-x(0,2)-[DE]', ['[AFG]-[AFG]', 'K>']        # (no avoided pattern ends in C, D or E: no dead end)
    kw = dict(temperature=1.0, top_p=0.95, seed=8, logit_bias=_aa_bias())
    samples = 14
    got = ProGen(**CASES['tiny_glu_sgu']).generate(eos, prompts, num_samples=samples, batch_size=bs, require=require,
                                                   avoid=avoid, **kw)
    motif = _motif(require, avoid, V, _aa_bias())
    N = len(prompts) * samples
    rows = [prompts[r // samples] for r in range(N)]
    dec = _decode(cfg, eos, min(bs, N))
    want = dict(tokens=np.zeros((N, n), np.int64), token_logp=np.zeros((N, n), np.float32), start=np.zeros(N, np.int64),
                end=np.zeros(N, np.int64))
    for sids, real in P.plan_launches([len(a) for a in rows], bs):
        res = dec.generate([rows[r] for r in sids], sample_ids=sids, motif=motif, **kw)
        r = sids[:real]
        want['tokens'][r], want['token_logp'][r] = res['ids'][:real], res['token_logp'][:real]
        want['start'][r], want['end'][r] = res['start'][:real], res['end'][:real]
    end = want.pop('end')
    want['finished'] = end < n
    want['length'] = np.where(want['finished'], end + 1, n) - want['start']
    want['log_likelihood'] = want['token_logp'].astype(np.float64).sum(axis=-1)
    want['motif_match'] = _satisfied(want, require, avoid)
    for k in OUT_KEYS:
        np.testing.assert_array_equal(got[k], want[k], err_msg=f'{k} bs={bs}')
    assert got['motif_match'].all() and got['finished'].any()


@pytest.mark.parametrize('name,mp', [('tiny_glu_sgu', False), ('tiny_all_glu', True)])
def test_forward_prefill_rows_satisfy_the_patterns(name, mp):
    from progen_b200 import ProGen
    cfg, params, data, g = load_case(name)
    prompts = _prompts(np.random.default_rng(77), [6, 6, 2])
    require = '<[AC]-x(1,3)-W' if name == 'tiny_glu_sgu' else ZINC_FINGER
    out = ProGen(**CASES[name], mixed_precision=mp).generate(params, prompts, num_samples=8, batch_size=12, seed=4,
                                                             prefill='forward', logit_bias=_aa_bias(), require=require,
                                                             avoid=AVOID)
    _check_all(out, require, AVOID, cfg['seq_len'])


def test_contradiction_ends_rows_with_eos():
    """a fixed first residue that the '<'-anchored requirement cannot start with: no candidate, EOS, motif_match False,
    and the other prompt's rows are unaffected"""
    from progen_b200 import ProGen
    cfg, params, data, g = load_case('tiny_all_glu')
    model = ProGen(**CASES['tiny_all_glu'])
    out = model.generate(params, ['MK', 'MK'], num_samples=10, batch_size=20, seed=3, logit_bias=_aa_bias(),
                         fixed=[{1: 'A'}, None], require='<M-x(0,3)-[KR]')
    bad = out['prompt_index'] == 0
    assert (out['finished'][bad] & (out['length'][bad] == 1)).all()
    assert not out['motif_match'][bad].any()
    assert out['motif_match'][~bad].all() and (out['tokens'][~bad, 3] == ord('M') + 1).all()


def test_first_draw_distribution_chi_square():
    """the first drawn residue under a '<'-anchored class and an avoided pair against the masked, renormalised
    softmax of the oracle's float64 logits"""
    from scipy import stats
    from oracle import progen_ref as O
    cfg, params, data, g = load_case('tiny_all_glu')
    n, V, B, runs = cfg['seq_len'], cfg['num_tokens'], 64, 40
    prompt = np.asarray(g['prime']).astype(np.int64)
    row = np.zeros(n, np.int64)
    row[1:1 + len(prompt)] = prompt
    l = O.forward(params, row, cfg)[len(prompt)].astype(np.float64)
    bias = np.zeros(V, np.float32)
    allowed = np.array([ord(ch) + 1 for ch in 'ACDEGHKLMW'])
    bias[allowed] = 5.0                                   # real mass on the class
    motif = _motif('<[ACDEGHKLMW]-x(2)', ['W'], V, bias)   # 'W' completes an avoided pattern on its own
    keep = np.zeros(V, bool)
    keep[allowed] = True
    keep[ord('W') + 1] = False
    a = np.where(keep, l + bias, -np.inf)
    probs = np.exp(a - a.max())
    probs /= probs.sum()
    dec = _decode(cfg, params, B)
    counts = np.zeros(V, np.int64)
    for r in range(runs):
        res = dec.generate([prompt] * B, temperature=1.0, seed=11, sample_ids=np.arange(r * B, (r + 1) * B),
                           max_length=len(prompt) + 5, logit_bias=bias, motif=motif)
        counts += np.bincount(res['ids'][:, 1 + len(prompt)], minlength=V)
    assert counts.sum() == B * runs and counts[~keep].sum() == 0
    exp_counts = probs * counts.sum()
    big = exp_counts >= 5
    obs = np.append(counts[big], counts[~big].sum())
    exp_ = np.append(exp_counts[big], exp_counts[~big].sum())
    if exp_[-1] == 0:
        obs, exp_ = obs[:-1], exp_[:-1]
    chi2 = ((obs - exp_) ** 2 / exp_).sum()
    pval = 1.0 - stats.chi2.cdf(chi2, len(obs) - 1)
    assert len(obs) >= 4 and pval > 1e-3, (chi2, len(obs), pval)


def test_token_logp_equals_score_under_patterns():
    from progen_b200 import ProGen
    cfg, params, data, g = load_case('tiny_all_glu')
    model = ProGen(**CASES['tiny_all_glu'])
    res = model.generate(params, ['', 'MK'], num_samples=6, temperature=1.0, seed=9, top_p=0.95, logit_bias=_aa_bias(),
                         require=ZINC_FINGER, avoid=AVOID)
    assert res['motif_match'].all()
    rows = np.concatenate([res['tokens'], np.zeros((len(res['tokens']), 1), np.int64)], axis=1)
    sc = model.score(params, rows, return_tokens=True)['token_logp']
    for i in range(len(rows)):
        s, ln = int(res['start'][i]), int(res['length'][i])
        want = sc[i, s - 1:s - 1 + ln].astype(np.float64)
        got = res['token_logp'][i, s:s + ln].astype(np.float64)
        assert np.abs(got - want).max() < 1e-4, i


def test_refusals_of_the_entry_point():
    """progen_decode_run refuses a descriptor with sampler 0, without max_length, with more than 9 patterns or with a
    null state buffer, and launches nothing"""
    from progen_b200 import lib as L
    from progen_b200.decode import MotifDesc
    cfg, params, data, g = load_case('tiny_glu_sgu')
    n = cfg['seq_len']
    dec = _decode(cfg, params, 4)
    desc = dec._motif_descriptor(_motif('A-C', None), 4)
    m = dec.m
    cnt = torch.zeros(4, dtype=torch.int32, device=dec.dev)
    sid = torch.zeros(4, dtype=torch.int64, device=dec.dev)
    end = torch.full((4,), n, dtype=torch.int32, device=dec.dev)

    def run(desc_patch=None, **f):
        d = desc.clone()
        if desc_patch:
            h = MotifDesc.from_buffer_copy(bytes(d[:C.sizeof(MotifDesc)].cpu().numpy()))
            for k, v in desc_patch.items():
                setattr(h, k, v)
            d[:C.sizeof(MotifDesc)].copy_(torch.from_numpy(np.frombuffer(bytes(h), np.uint8).copy()))
        base = dict(B=4, sampler=1, temperature=1.0, top_p=1.0, sample_id=sid.data_ptr(), end=end.data_ptr(),
                    n_ended=cnt.data_ptr(), steps_run=cnt.data_ptr() + 4, pos0=0, nsteps=2, max_length=n,
                    motif=d.data_ptr())
        base.update(f)
        saved = {k: getattr(m, k) for k in base}
        for k, v in base.items():
            setattr(m, k, v)
        try:
            dec.grid_bar.zero_()
            cnt.zero_()
            rc = dec.lib.progen_decode_run(C.byref(m), L.stream())
            torch.cuda.synchronize()
            return rc
        finally:
            for k, v in saved.items():
                setattr(m, k, v)

    torch.cuda.synchronize()
    before = dec.lib.progen_launch_count()
    refused = {'sampler 0': dict(sampler=0, temperature=0.0, top_p=0.0),
               'no max_length': dict(max_length=0),
               '10 patterns': dict(desc_patch=dict(num_patterns=10)),
               '0 patterns': dict(desc_patch=dict(num_patterns=0)),
               'null state': dict(desc_patch=dict(state=0))}
    for what, f in refused.items():
        assert run(**f) == -2, what                       # PROGEN_ERR_ARG
    assert dec.lib.progen_launch_count() == before
    assert run() == 0
    assert dec.lib.progen_launch_count() == before + 1


def test_generate_cli_motifs(tmp_path):
    from progen_b200.checkpoint import file_save_checkpoint
    from oracle import progen_ref as O
    kwargs = dict(num_tokens=256, dim=128, seq_len=128, depth=2, window_size=64, global_mlp_depth=1, heads=2, dim_head=64)
    params = O.randomize_params(O.init_params(O.make_config(**kwargs), 91), 92)
    (tmp_path / 'ckpts').mkdir()
    file_save_checkpoint(tmp_path / 'ckpts', dict(next_seq_index=0, params=params, optim_state=None, model_config=kwargs,
                                                  run_id=None))
    out = tmp_path / 'm.fasta'
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'generate.py'), '--checkpoint_path', str(tmp_path / 'ckpts'),
                        '--prompt', 'MK', '--num_samples', '16', '--seed', '4', '--max_length', '60', '--alphabet', AA,
                        '--require', ZINC_FINGER, '--avoid', AVOID[0], '--avoid', AVOID[1], '--output', str(out)],
                       cwd=str(tmp_path), env=dict(os.environ, PYTHONPATH=ROOT), capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    lines = out.read_text().splitlines()
    assert len(lines) == 32
    pat = re.compile(r'^>(\d+) prompt=0 sample=(\d+) log_likelihood=(-?[\d.]+) length=(\d+) eos=([01]) motif=1$')
    zf, avoid = to_regex(ZINC_FINGER), [to_regex(a) for a in AVOID]
    for row, (h, body) in enumerate(zip(lines[0::2], lines[1::2])):
        assert pat.match(h), h
        assert zf.search(body) and not any(a.search(body) for a in avoid), body
