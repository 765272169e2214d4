"""Controlled generation (sampler 1 of csrc/decode_persist.cu with a logit bias, a minimum length and a repetition
penalty): neutral arguments change no bit, an exact host replay of the adjusted logits, the filter and the Philox draw,
bans and the minimum length hold, the first draw's distribution, token log-probabilities against `score`, batch
independence, the reference sampler afterwards, and generate.py's --alphabet."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from golden_util import load_case, CASES
from test_gpu_generate import gumbel, host_draw, _drawn, _eos_params, _prompts

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
AA = 'ACDEFGHIKLMNPQRSTVWY'


def _aa_bias(V=256):
    b = np.full(V, -np.inf, np.float32)
    b[0] = 0.0
    b[[ord(ch) + 1 for ch in AA]] = 0.0
    return b


def _random_bias(rng, V=256, banned=0.3):
    """finite values of both signs, about `banned` of the ids at -inf (EOS and some id in [1, V) always allowed)"""
    b = (rng.standard_normal(V) * 1.5).astype(np.float32)
    b[rng.random(V) < banned] = -np.inf
    b[0] = 0.0
    b[1 + rng.integers(V - 1)] = 0.5
    return b


def adjust(l, ids, p, start, bias=None, theta=1.0, window=0, min_new=0):
    """the kernel's adjusted logits a for the draw at p + 1 of a row, in float32: penalty on the ids present at
    max(1, p + 1 - window) .. p, plus the bias, EOS banned while p + 1 < start + min_new"""
    a = np.asarray(l, np.float32).copy()
    if theta != 1.0:
        lo = max(1, p + 1 - window) if window > 0 else 1
        c = np.unique(np.asarray(ids[lo:p + 1]))
        c = c[(c >= 0) & (c < len(a))]
        th = np.float32(theta)
        a[c] = np.where(a[c] > 0, a[c] / th, a[c] * th)
    if bias is not None:
        a = a + np.asarray(bias, np.float32)
    if p + 1 < start + min_new:
        a[0] = -np.inf
    return a


@pytest.mark.parametrize('B', [1, 8, 24])
def test_neutral_constraints_change_no_bit(B):
    """explicit neutral arguments (a zero bias runs the constrained code) equal omitted ones bit for bit"""
    from progen_b200.decode import BatchDecoder
    cfg, params, data, g = load_case('tiny_all_glu')
    rng = np.random.default_rng(B)
    prompts = _prompts(rng, rng.integers(0, 7, B))
    dec = BatchDecoder(cfg, params, batch=B)
    neutral = dict(logit_bias=np.zeros(cfg['num_tokens'], np.float32), repetition_penalty=1.0, repetition_window=0,
                   min_new_tokens=0)
    for T, top_k, top_p in ((0.0, None, None), (1.0, None, None), (0.7, 5, None), (1.5, None, 0.9), (1.0, 40, 0.5)):
        kw = dict(temperature=T, top_k=top_k, top_p=top_p, seed=21)
        a = dec.generate(prompts, **kw)
        b = dec.generate(prompts, **kw, **neutral)
        for k in ('ids', 'token_logp', 'end', 'steps_run'):
            np.testing.assert_array_equal(a[k], b[k], err_msg=f'{k} T={T} top_k={top_k} top_p={top_p}')


def _constraint_sets(V):
    bias = _random_bias(np.random.default_rng(70), V)
    sets = [dict(logit_bias=bias)]
    sets += [dict(repetition_penalty=th, repetition_window=w) for th in (1.3, 0.8) for w in (0, 8)]
    sets += [dict(min_new_tokens=m) for m in (0, 5)]
    sets += [dict(logit_bias=bias, repetition_penalty=1.3, repetition_window=8, min_new_tokens=5)]
    return sets


def test_constrained_sampler_matches_host_replay():
    """T x top_k x top_p x constraint sets at B = 16: every id is a kept candidate of the adjusted logits, and equals the
    host replay (float32 adjustments, float64 filter and Gumbel-max on the kernel's own logits) wherever the draw is
    unambiguous; >= 99 % of positions are"""
    from progen_b200.decode import BatchDecoder
    cfg, params, data, g = load_case('tiny_all_glu')
    V, B = cfg['num_tokens'], 16
    rng = np.random.default_rng(17)
    prompts = _prompts(rng, rng.integers(0, 9, B))
    dec = BatchDecoder(cfg, params, batch=B, keep_logits=True)
    total = unamb = 0
    seed = 0xFEED_0123_4567
    sids = np.arange(B, dtype=np.int64) * 7 + (1 << 34)
    for cs in _constraint_sets(V):
        ck = dict(bias=cs.get('logit_bias'), theta=cs.get('repetition_penalty', 1.0),
                  window=cs.get('repetition_window', 0), min_new=cs.get('min_new_tokens', 0))
        for T in (0.0, 0.7, 1.5):
            for top_k in (None, 5):
                for top_p in (None, 0.9):
                    res = dec.generate(prompts, temperature=T, top_k=top_k, top_p=top_p, seed=seed, sample_ids=sids,
                                       max_length=64, **cs)
                    lg = dec.logits_all.cpu().numpy()
                    for b in range(B):
                        ids, st = res['ids'][b], int(res['start'][b])
                        for t in _drawn(res, b, 64):
                            a = adjust(lg[b, t - 1], ids, t - 1, st, **ck)
                            want, keep, amb = host_draw(a, T, top_k, top_p, gumbel(seed, int(sids[b]), t, V))
                            got = int(ids[t])
                            where = (cs, T, top_k, top_p, b, t, got, want)
                            assert a[got] > -np.inf and keep[got], where
                            total += 1
                            if not amb:
                                unamb += 1
                                assert got == want, where
    assert total > 3000 and unamb >= 0.99 * total, (unamb, total)


def _check_rows(out, max_length, min_new, allowed):
    """finished, length and log_likelihood agree with the tokens; drawn ids are allowed; no EOS before start + min_new"""
    n = out['tokens'].shape[1]
    for i in range(len(out['tokens'])):
        tok, s, ln, fin = out['tokens'][i], int(out['start'][i]), int(out['length'][i]), bool(out['finished'][i])
        gen = tok[s:s + ln]
        assert np.isin(gen, allowed).all(), (i, gen)
        eos = np.nonzero(gen == 0)[0]
        assert fin == (len(eos) > 0)
        if fin:
            assert list(eos) == [ln - 1] and ln >= min_new + 1, (i, ln)
        else:
            assert s + ln == max_length
        assert (tok[s + ln:] == 0).all() and (out['token_logp'][i, s + ln:] == 0).all()
        assert (out['token_logp'][i, s:s + ln] < 0).all()
        ll = out['token_logp'][i, s:s + ln].astype(np.float64).sum()
        assert abs(out['log_likelihood'][i] - ll) <= 1e-6 * max(1.0, abs(ll)), i
    assert out['tokens'].shape == (len(out['start']), n)


def test_bans_and_minimum_length_hold():
    """512 samples with EOS about 30 % likely right after the prompt, a 20-letter alphabet and min_new_tokens 30"""
    from progen_b200 import ProGen
    cfg, params, data, g = load_case('tiny_all_glu')
    prompt = np.array([ord(ch) + 1 for ch in 'MKT'])
    eos = _eos_params(params, cfg, prompt, 0.3)
    allowed = np.array([0] + [ord(ch) + 1 for ch in AA])
    model = ProGen(**CASES['tiny_all_glu'])
    plain = model.generate(eos, [prompt], num_samples=64, temperature=1.0, seed=3)
    assert (plain['length'] == 1).sum() >= 5, 'EOS must be likely enough right after the prompt for the minimum to bind'
    out = model.generate(eos, [prompt], num_samples=512, temperature=1.0, top_p=0.95, seed=3, logit_bias=_aa_bias(),
                         min_new_tokens=30, repetition_penalty=1.2, repetition_window=16)
    _check_rows(out, cfg['seq_len'], 30, allowed)
    assert (out['length'][out['finished']] == 31).any()


def test_min_length_binds_at_24_rows():
    """the launch's early exit waits for the minimum: every row ends, none before start + 30, and steps_run covers it"""
    from progen_b200.decode import BatchDecoder
    cfg, params, data, g = load_case('tiny_all_glu')
    n, B = cfg['seq_len'], 24
    prompts = _prompts(np.random.default_rng(4), np.random.default_rng(5).integers(0, 6, B))
    eos = _eos_params(params, cfg, prompts[0], 0.5)
    dec = BatchDecoder(cfg, eos, batch=B)
    res = dec.generate(prompts, temperature=1.0, seed=2, logit_bias=_aa_bias(), min_new_tokens=30,
                       repetition_penalty=1.3, repetition_window=8)
    end, start = res['end'], res['start']
    assert (end < n).all(), 'every row should have sampled EOS'
    assert (end >= start + 30).all()
    first = int(start.min()) - 1
    assert res['steps_run'] == int(end.max()) - first and res['steps_run'] >= 30
    for b in range(B):
        drawn = res['ids'][b, start[b]:end[b]]
        assert np.isin(drawn, [ord(ch) + 1 for ch in AA]).all() and res['ids'][b, end[b]] == 0


@pytest.mark.parametrize('case', ['bias', 'penalty'])
def test_first_draw_distribution_chi_square(case):
    """first drawn position over many sample ids against softmax(a / T) over the candidates, a from the oracle's float64
    logits: a bias with bans, or a penalty on the prompt's ids (raised by a bias so that the penalty moves real mass)"""
    from scipy import stats
    from progen_b200.decode import BatchDecoder
    from oracle import progen_ref as O
    cfg, params, data, g = load_case('tiny_all_glu')
    n, V, B, runs = cfg['seq_len'], cfg['num_tokens'], 64, 40
    prompt = np.asarray(g['prime']).astype(np.int64)
    row = np.zeros(n, np.int64)
    row[1:1 + len(prompt)] = prompt
    l = O.forward(params, row, cfg)[len(prompt)].astype(np.float64)
    if case == 'bias':
        T, kw = 0.8, dict(logit_bias=_random_bias(np.random.default_rng(5), V))
        a = l + kw['logit_bias']
    else:
        bias = np.zeros(V, np.float32)
        bias[np.unique(prompt)] = 4.0
        T, kw = 1.0, dict(logit_bias=bias, repetition_penalty=2.0)
        a = l.copy()
        c = np.unique(prompt)
        a[c] = np.where(a[c] > 0, a[c] / 2.0, a[c] * 2.0)
        a = a + bias
    keep = np.isfinite(a)
    z = np.where(keep, a / T, -np.inf)
    probs = np.exp(z - z.max())
    probs /= probs.sum()
    dec = BatchDecoder(cfg, params, batch=B)
    counts = np.zeros(V, np.int64)
    for r in range(runs):
        res = dec.generate([prompt] * B, temperature=T, seed=11, sample_ids=np.arange(r * B, (r + 1) * B),
                           max_length=len(prompt) + 2, **kw)
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


ALL = dict(min_new_tokens=4, repetition_penalty=1.3, repetition_window=8)


def test_token_logp_equals_score_under_constraints():
    from progen_b200 import ProGen
    cfg, params, data, g = load_case('tiny_glu_sgu')
    model = ProGen(**CASES['tiny_glu_sgu'])
    prompts = _prompts(np.random.default_rng(3), [0, 2, 5, 9])
    res = model.generate(params, prompts, num_samples=3, temperature=1.0, seed=9, top_p=0.95,
                         logit_bias=_random_bias(np.random.default_rng(6)), **ALL)
    rows = np.concatenate([res['tokens'], np.zeros((len(res['tokens']), 1), np.int64)], axis=1)
    sc = model.score(params, rows, return_tokens=True)['token_logp']
    for i in range(len(rows)):
        s, ln = int(res['start'][i]), int(res['length'][i])
        want = sc[i, s - 1:s - 1 + ln].astype(np.float64)
        got = res['token_logp'][i, s:s + ln].astype(np.float64)
        assert np.abs(got - want).max() < 1e-4, i
        assert (res['token_logp'][i, :s] == 0).all() and (res['token_logp'][i, s + ln:] == 0).all()
        assert abs(res['log_likelihood'][i] - got.sum()) <= 1e-5 * abs(got.sum()), i


def test_rows_do_not_depend_on_launch_size_under_constraints():
    from progen_b200 import ProGen
    cfg, params, _, _ = load_case('tiny_glu_sgu')
    model = ProGen(**CASES['tiny_glu_sgu'])
    prompts = ['', 'MKV', np.array([20, 30, 40, 50, 60])]
    kw = dict(num_samples=30, temperature=1.0, top_p=0.9, seed=23, logit_bias=_aa_bias(), **ALL)
    runs = [model.generate(params, prompts, batch_size=bs, **kw) for bs in (64, 12, 30)]
    for bs, b in zip((12, 30), runs[1:]):
        for k in ('tokens', 'token_logp', 'length', 'finished', 'log_likelihood'):
            np.testing.assert_array_equal(runs[0][k], b[k], err_msg=f'{k} batch_size={bs} vs 64')


@pytest.mark.parametrize('B', [1, 2])
def test_reference_sampler_after_constrained_generate(B):
    """a constrained generate leaves nothing behind: the reference sampler gives a fresh decoder's ids"""
    from progen_b200.decode import BatchDecoder
    cfg, params, data, g = load_case('tiny_glu_sgu')
    primes = [np.asarray(g['prime']).astype(np.int64)] * B
    dec = BatchDecoder(cfg, params, batch=B)
    dec.generate([np.array([3, 4])] * B, temperature=0.7, top_k=9, seed=1, logit_bias=_random_bias(np.random.default_rng(1)),
                 **ALL)
    m = dec.m
    assert (m.sampler, m.logit_bias, m.repetition_penalty, m.repetition_window, m.min_new_tokens) == (0, None, 1.0, 0, 0)
    for greedy in (True, False):
        a, _, _ = dec.sample(primes if B > 1 else primes[0], top_k=25, add_bos=True, greedy=greedy, seed=5)
        b, _, _ = BatchDecoder(cfg, params, batch=B).sample(primes if B > 1 else primes[0], top_k=25, add_bos=True,
                                                            greedy=greedy, seed=5)
        np.testing.assert_array_equal(a, b)
        if greedy and B == 1:
            np.testing.assert_array_equal(a, g['sample_bos1'])


def test_generate_cli_constraints(tmp_path):
    from progen_b200.checkpoint import file_save_checkpoint
    from oracle import progen_ref as O
    kwargs = dict(num_tokens=256, dim=128, seq_len=128, depth=2, window_size=64, global_mlp_depth=1, heads=2, dim_head=64)
    params = O.randomize_params(O.init_params(O.make_config(**kwargs), 91), 92)
    (tmp_path / 'ckpts').mkdir()
    file_save_checkpoint(tmp_path / 'ckpts', dict(next_seq_index=0, params=params, optim_state=None, model_config=kwargs,
                                                  run_id=None))
    out = tmp_path / 'c.fasta'
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'generate.py'), '--checkpoint_path', str(tmp_path / 'ckpts'),
                        '--prompt', 'MK', '--num_samples', '16', '--seed', '4', '--max_length', '100',
                        '--alphabet', AA, '--min_new_tokens', '20', '--repetition_penalty', '1.2',
                        '--repetition_window', '16', '--output', str(out)],
                       cwd=str(tmp_path), env=dict(os.environ, PYTHONPATH=ROOT), capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    lines = out.read_text().splitlines()
    assert len(lines) == 32
    pat = re.compile(r'^>(\d+) prompt=0 sample=(\d+) log_likelihood=(-?[\d.]+) length=(\d+) eos=([01])$')
    for row, (h, body) in enumerate(zip(lines[0::2], lines[1::2])):
        m = pat.match(h)
        assert m and int(m[1]) == row, h
        assert set(body) <= set(AA), body
        assert len(body) == int(m[4]) - int(m[5])
        if m[5] == '1':
            assert len(body) >= 20, h
        else:
            assert int(m[4]) == 100 - 3                       # BOS + 'MK' + 97 generated
