"""Refilled generation (the row queue of csrc/decode_persist.cu; `BatchDecoder.generate_queue`, `ProGen.generate`): a slot
whose row ends takes the next row of the queue.  Every output must be bitwise what the static schedule gives, one launch
of up to batch_size rows after another (`plan_launches` + `BatchDecoder.generate`, the loop `ProGen.generate` ran before
the queue), and the queue launch must run fewer positions than those launches together."""
import numpy as np
import pytest
import torch

from golden_util import load_case, CASES
from test_gpu_generate import _eos_params, HEAD_B, H8

pytestmark = pytest.mark.gpu
OUT_KEYS = ('tokens', 'token_logp', 'start', 'length', 'finished', 'log_likelihood')
GELU_NOSHIFT = dict(CASES['tiny_gelu_sgu'], shift_tokens=False)


def _model(name):
    """(ProGen kwargs, cfg, params) of a test model"""
    from oracle import progen_ref as O
    if name in CASES:
        cfg, params, _, _ = load_case(name)
        return CASES[name], cfg, params
    kw = {'h8': H8, 'noshift': GELU_NOSHIFT}[name]
    cfg = O.make_config(**kw)
    return kw, cfg, O.randomize_params(O.init_params(cfg, 31), 32)


def _prompts(max_length, k=6, seed=1):
    """k prompts of mixed lengths: empty, short, and one leaving 3 positions before max_length"""
    rng = np.random.default_rng(seed)
    lengths = [0, 1, max_length - 4, 5, 2, 9, 3, 7][:k]
    return [rng.integers(1, 256, L).astype(np.int64) for L in lengths]


def _static(cfg, params, prompts, num_samples, batch_size, wdt, max_length=None, **kw):
    """the pre-queue ProGen.generate loop: launches of plan_launches through BatchDecoder.generate.  -> (generate's dict,
    positions the launches ran together)"""
    from progen_b200.decode import BatchDecoder
    from progen_b200.progen import plan_launches
    n = cfg['seq_len']
    max_length = n if max_length is None else max_length
    rows = [np.asarray(prompts[r // num_samples], np.int64) for r in range(len(prompts) * num_samples)]
    N = len(rows)
    dec = BatchDecoder(cfg, params, batch=min(batch_size, N), weights_dtype=wdt)
    out = dict(tokens=np.zeros((N, n), np.int64), token_logp=np.zeros((N, n), np.float32), start=np.zeros(N, np.int64),
               end=np.zeros(N, np.int64))
    positions = 0
    for sids, real in plan_launches([len(a) for a in rows], batch_size):
        res = dec.generate([rows[r] for r in sids], sample_ids=sids, max_length=max_length, **kw)
        r = sids[:real]
        out['tokens'][r] = res['ids'][:real]
        out['token_logp'][r] = res['token_logp'][:real]
        out['start'][r] = res['start'][:real]
        out['end'][r] = res['end'][:real]
        positions += int(res['start'].min()) - 1 + res['steps_run']
    end = out.pop('end')
    out['finished'] = end < max_length
    out['length'] = np.where(out['finished'], end + 1, max_length) - out['start']
    out['log_likelihood'] = out['token_logp'].astype(np.float64).sum(axis=-1)
    return out, positions


def _assert_equal(a, b, what):
    for k in OUT_KEYS:
        np.testing.assert_array_equal(a[k], b[k], err_msg=f'{k} {what}')


SETTINGS = [dict(temperature=1.0, top_p=0.9),
            dict(temperature=0.0),
            dict(temperature=1.0, top_k=20, min_new_tokens=2, repetition_penalty=1.3, repetition_window=6, bias=True),
            dict(temperature=0.8, top_k=40, top_p=0.95, max_length=-7)]


def _setting(i, n, V):
    kw = dict(SETTINGS[i % len(SETTINGS)])
    if kw.pop('bias', False):
        kw['logit_bias'] = np.where(np.arange(V) % 7 == 3, -np.inf, 0.25 * np.sin(np.arange(V))).astype(np.float32)
    if kw.get('max_length', 0) < 0:
        kw['max_length'] = n + kw['max_length']
    return kw


CASES_EQ = [(m, w, bs) for m in ('tiny_glu_sgu', 'h8', 'tiny_gelu_sgu', 'noshift') for w in ('f32', 'bf16')
            for bs in (5, 8, 12, 40, 64)]


@pytest.mark.parametrize('name,wdt,bs', CASES_EQ)
def test_generate_bitwise_equals_static_schedule(name, wdt, bs):
    """ProGen.generate (one queue launch of N = 6 x 17 rows on min(bs, N) slots) against the static launches, with EOS
    raised so that rows end at scattered positions; the sampler settings rotate over the cases"""
    from progen_b200 import ProGen
    kw, cfg, params = _model(name)
    n, V = cfg['seq_len'], cfg['num_tokens']
    s = _setting(CASES_EQ.index((name, wdt, bs)), n, V)
    ml = s.get('max_length', n)
    prompts = _prompts(ml)
    eos = _eos_params(params, cfg, prompts[3], 0.12)
    model = ProGen(**kw, mixed_precision=wdt == 'bf16')
    got = model.generate(eos, prompts, num_samples=17, batch_size=bs, seed=41, **s)
    want, _ = _static(cfg, eos, prompts, 17, bs, torch.bfloat16 if wdt == 'bf16' else torch.float32, seed=41, **s)
    _assert_equal(got, want, f'{name} {wdt} batch_size={bs} {s}')
    assert got['finished'].any()
    assert s['temperature'] == 0 or (got['length'] > 1).any()        # (greedy rows may all draw EOS first)


@pytest.mark.parametrize('setting', range(len(SETTINGS)))
@pytest.mark.parametrize('bs', [12, 64])
def test_every_setting_bitwise_equals_static(setting, bs):
    from progen_b200 import ProGen
    kw, cfg, params = _model('tiny_all_glu')
    n, V = cfg['seq_len'], cfg['num_tokens']
    s = _setting(setting, n, V)
    prompts = _prompts(s.get('max_length', n), seed=setting)
    eos = _eos_params(params, cfg, prompts[3], 0.05)
    got = ProGen(**kw).generate(eos, prompts, num_samples=15, batch_size=bs, seed=7, **s)
    want, _ = _static(cfg, eos, prompts, 15, bs, torch.float32, seed=7, **s)
    _assert_equal(got, want, f'batch_size={bs} {s}')


@pytest.mark.parametrize('slots', [6, 12, 40])
def test_refill_runs_fewer_positions(slots):
    """one queue launch of Q > slots rows: some slot decoded more than one row (Q > slots), the rows are the static
    schedule's, and the launch ran fewer positions than the static launches together"""
    from progen_b200.decode import BatchDecoder
    kw, cfg, params = _model('tiny_all_glu')
    prompts = _prompts(cfg['seq_len'], k=5)
    eos = _eos_params(params, cfg, prompts[3], 0.05)
    rows = [prompts[r // 20] for r in range(100)]
    dec = BatchDecoder(cfg, eos, batch=slots)
    res = dec.generate_queue(rows, temperature=1.0, top_p=0.9, seed=3, sample_ids=np.arange(100))
    want, positions = _static(cfg, eos, prompts, 20, slots, torch.float32, temperature=1.0, top_p=0.9, seed=3)
    np.testing.assert_array_equal(res['ids'], want['tokens'])
    np.testing.assert_array_equal(res['token_logp'], want['token_logp'])
    assert len(rows) > slots
    print(dict(slots=slots, queue_positions=res['steps_run'], static_positions=positions))
    assert res['steps_run'] < positions
    again = dec.generate_queue(rows, temperature=1.0, top_p=0.9, seed=3, sample_ids=np.arange(100))
    for k in ('ids', 'token_logp', 'end', 'steps_run'):
        np.testing.assert_array_equal(again[k], res[k], err_msg=k)


def test_every_row_ends_at_its_first_draw():
    """NaN head: every row draws EOS at its first position, and every refill happens on the next step"""
    from progen_b200 import ProGen
    kw, cfg, params = _model('tiny_all_glu')
    bad = {k: {kk: np.array(vv, copy=True) for kk, vv in v.items()} for k, v in params.items()}
    bad[HEAD_B]['b'][:] = np.nan
    prompts = _prompts(cfg['seq_len'], k=4)
    got = ProGen(**kw).generate(bad, prompts, num_samples=10, batch_size=12, seed=1)
    np.testing.assert_array_equal(got['length'], 1)
    assert got['finished'].all() and np.isnan(got['log_likelihood']).all()
    want, _ = _static(cfg, bad, prompts, 10, 12, torch.float32, seed=1)
    np.testing.assert_array_equal(got['tokens'], want['tokens'])
    np.testing.assert_array_equal(got['start'], want['start'])


@pytest.mark.parametrize('wdt', ['f32', 'bf16'])
def test_queue_of_one_row_per_slot(wdt):
    """Q = B (every slot decodes one row and goes idle) and N < batch_size (the call's slots are its N rows)"""
    from progen_b200 import ProGen
    from progen_b200.decode import BatchDecoder
    kw, cfg, params = _model('tiny_glu_sgu')
    dt = torch.bfloat16 if wdt == 'bf16' else torch.float32
    prompts = _prompts(cfg['seq_len'], k=5)
    eos = _eos_params(params, cfg, prompts[3], 0.1)
    res = BatchDecoder(cfg, eos, batch=10, weights_dtype=dt).generate_queue(prompts + prompts, seed=5)
    ref = BatchDecoder(cfg, eos, batch=10, weights_dtype=dt).generate(prompts + prompts, seed=5)
    for k in ('ids', 'token_logp', 'end'):
        np.testing.assert_array_equal(res[k], ref[k], err_msg=k)
    assert res['steps_run'] <= int(ref['start'].min()) - 1 + ref['steps_run']
    got = ProGen(**kw, mixed_precision=wdt == 'bf16').generate(eos, prompts, num_samples=2, batch_size=64, seed=5)
    want, _ = _static(cfg, eos, prompts, 2, 64, dt, seed=5)
    _assert_equal(got, want, 'N < batch_size')


def test_eos_banned_runs_as_many_positions():
    """every row runs to max_length: the queue runs exactly the static schedule's positions"""
    from progen_b200.decode import BatchDecoder
    kw, cfg, params = _model('tiny_glu_sgu')
    never = {k: {kk: np.array(vv, copy=True) for kk, vv in v.items()} for k, v in params.items()}
    never[HEAD_B]['b'][0] = -np.inf
    prompts = _prompts(cfg['seq_len'], k=3)
    rows = [prompts[r // 10] for r in range(30)]
    res = BatchDecoder(cfg, never, batch=8).generate_queue(rows, seed=2, sample_ids=np.arange(30))
    want, positions = _static(cfg, never, prompts, 10, 8, torch.float32, seed=2)
    np.testing.assert_array_equal(res['ids'], want['tokens'])
    assert not want['finished'].any()
    assert res['steps_run'] == positions == 4 * (cfg['seq_len'] - 1)


def test_token_logp_of_refilled_rows_equals_score():
    """test_gpu_generate.py::test_token_logp_equals_score on rows that ran in refilled slots"""
    from progen_b200 import ProGen
    kw, cfg, params = _model('tiny_glu_sgu')
    prompts = _prompts(cfg['seq_len'], k=4, seed=3)
    eos = _eos_params(params, cfg, prompts[3], 0.1)
    model = ProGen(**kw)
    res = model.generate(eos, prompts, num_samples=8, batch_size=6, temperature=1.0, seed=9, top_p=0.95)
    rows = np.concatenate([res['tokens'], np.zeros((len(res['tokens']), 1), np.int64)], axis=1)
    sc = model.score(eos, rows, return_tokens=True)['token_logp']
    for i in range(len(rows)):
        s, ln = int(res['start'][i]), int(res['length'][i])
        want = sc[i, s - 1:s - 1 + ln].astype(np.float64)
        got = res['token_logp'][i, s:s + ln].astype(np.float64)
        assert np.abs(got - want).max() < 1e-4, i


@pytest.mark.parametrize('bs', [20, 64])
def test_config3_width_bitwise_equals_static(bs):
    """the depth-3 config-3 stack (d1024 h16 w512 n2048) with bf16 weights, rows ending within a few hundred positions"""
    from progen_b200 import ProGen
    from test_gpu_large_config_inference import _model as large
    kw, cfg, params = large('cfg3')
    rng = np.random.default_rng(bs)
    prompts = [rng.integers(1, 256, L).astype(np.int64) for L in (0, 3, 40)]
    eos = _eos_params(params, cfg, prompts[1], 0.01)
    N = bs + bs // 2 + 1
    samples = -(-N // 3)
    got = ProGen(**kw, mixed_precision=True).generate(eos, prompts, num_samples=samples, batch_size=bs, seed=13, top_p=0.95)
    want, positions = _static(cfg, eos, prompts, samples, bs, torch.bfloat16, seed=13, top_p=0.95)
    _assert_equal(got, want, f'cfg3 batch_size={bs}')
    print(dict(batch_size=bs, rows=3 * samples, longest=int(got['length'].max()), static_positions=positions))
    assert got['finished'].mean() > 0.9


def test_rejected_queue_arguments():
    """progen_decode_run refuses a malformed queue with an argument error and launches nothing"""
    import ctypes as C
    from progen_b200 import lib as L
    from progen_b200.decode import BatchDecoder
    kw, cfg, params = _model('tiny_all_glu')
    dec = BatchDecoder(cfg, params, batch=4, keep_logits=True)
    n = cfg['seq_len']
    buf = torch.zeros(64, dtype=torch.int32, device=dec.dev)   # [n_ended, steps_run, next_row, done, slot_row[4] .. slot_pos[4]]
    buf[2] = 4
    buf[4:8] = torch.arange(4, dtype=torch.int32)
    big = torch.zeros(16, n, dtype=torch.int32, device=dec.dev)
    gen = dict(sample_id=torch.zeros(16, dtype=torch.int64, device=dec.dev), end=torch.full((16,), n, dtype=torch.int32, device=dec.dev))
    p = buf.data_ptr()
    m = dec.m

    def queue(**over):
        q = dict(B=4, sampler=1, temperature=1.0, top_p=1.0, sample_id=gen['sample_id'].data_ptr(), end=gen['end'].data_ptr(),
                 n_ended=p, steps_run=p + 4, slot_row=p + 16, slot_pos=p + 48, next_row=p + 8, done=p + 12, num_rows=8,
                 max_length=n, logits_all=0, seq=big.data_ptr(), start=big.data_ptr(), pos0=0, nsteps=4)
        q.update(over)
        return q

    def rc(**f):
        saved = {k: getattr(m, k) for k in f}
        for k, v in f.items():
            setattr(m, k, v)
        try:
            dec.grid_bar.zero_()
            return dec.lib.progen_decode_run(C.byref(m), L.stream())
        finally:
            for k, v in saved.items():
                setattr(m, k, v)

    torch.cuda.synchronize()
    before = dec.lib.progen_launch_count()
    bad = {'queue with sampler 0': queue(sampler=0, temperature=0.0),
           'Q > B with B = 1': queue(B=1),
           'Q < B': queue(num_rows=3),
           'logits_all with Q > B': queue(logits_all=dec.logits_all.data_ptr()),
           'max_length < 2': queue(max_length=1),
           'max_length > n': queue(max_length=n + 1),
           'no done counter': queue(done=0),
           'no next_row counter': queue(next_row=0),
           'no slot rows': queue(slot_row=0)}
    for what, f in bad.items():
        assert rc(**f) == -2, what                        # PROGEN_ERR_ARG
    assert dec.lib.progen_launch_count() == before
    assert rc(**queue()) == 0                             # the same fields, well formed, launch
    assert dec.lib.progen_launch_count() == before + 1
    torch.cuda.synchronize()
