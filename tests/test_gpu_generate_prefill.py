"""Forward prefill of generation (`ProGen.generate(prefill='forward')`, `BatchDecoder.prefill`, `Engine.prefill`,
progen_gather_rows_f32): the caches it writes against the decode kernel's own prefill, the first-draw logits against the
oracle, token log-probabilities against `score`, and that a row's result does not depend on which rows share its launch
or its forward."""
import numpy as np
import pytest
import torch

from golden_util import load_case, CASES

pytestmark = pytest.mark.gpu
TINY = [n for n in CASES if n != 'cfg1']
EXTRA = {
    'h8': dict(num_tokens=256, dim=256, seq_len=64, depth=2, window_size=16, global_mlp_depth=1, heads=8, dim_head=32),
    # shapes the tensor-core (mixed precision) forward accepts: gMLP, 8 heads
    'bf_sgu': dict(num_tokens=256, dim=128, seq_len=128, depth=2, window_size=64, global_mlp_depth=1, heads=2, dim_head=64),
    'bf_h8': dict(num_tokens=256, dim=512, seq_len=128, depth=2, window_size=64, global_mlp_depth=1, heads=8, dim_head=64),
}
ALPHABET = 'ACDEFGHIKLMNPQRSTVWY'


def _case(name):
    from oracle import progen_ref as O
    if name in CASES:
        cfg, params, _, _ = load_case(name)
        return CASES[name], cfg, params
    cfg = O.make_config(**EXTRA[name])
    return EXTRA[name], cfg, O.randomize_params(O.init_params(cfg, 31), 32)


def _prompts(rng, lengths):
    return [rng.integers(1, 256, L).astype(np.int64) for L in lengths]


def _lengths(n):
    return (1, n // 2 - 3, n - 2)


def _both(kw, cfg, params, prompts, mp):
    """the same prompts prefilled by the decode kernel (a) and by the forward (b), each then drawing one position"""
    from progen_b200 import ProGen
    from progen_b200.decode import BatchDecoder
    P = len(prompts[0])
    wdt = torch.bfloat16 if mp else torch.float32
    model = ProGen(**kw, mixed_precision=mp)
    model._ensure_loaded(params)
    a = BatchDecoder(cfg, params, batch=len(prompts), weights_dtype=wdt, keep_logits=True)
    ra = a.generate(prompts, temperature=0.0, max_length=P + 2)
    b = BatchDecoder(cfg, params, batch=len(prompts), weights_dtype=wdt, keep_logits=True)
    assert b.prefill(model.engine, prompts) == P
    rb = b.generate(prompts, temperature=0.0, max_length=P + 2, prefilled=P)
    np.testing.assert_array_equal(ra['start'], rb['start'])
    return model, a, b


@pytest.mark.parametrize('L', [0, 1, 2])
@pytest.mark.parametrize('name', TINY + ['h8'])
def test_fp32_caches_match_the_decode_prefill(name, L):
    """fp32 model: K/V rows, the token-shift slot the kernel reads at P and the SGU gate history at positions < P agree
    with the decode kernel's own prefill to fp32 round-off (rows 0 and 2 share one forward row)"""
    kw, cfg, params = _case(name)
    n, h, dh = cfg['seq_len'], cfg['heads'], cfg['dim_head']
    P = _lengths(n)[L]
    p = _prompts(np.random.default_rng(P), [P, P])
    prompts = [p[0], p[1], p[0]]
    _, a, b = _both(kw, cfg, params, prompts, mp=False)
    R = len(prompts)
    checked = 0
    for i, (ca, cb) in enumerate(zip(a.caches, b.caches)):
        for key in ca:
            x, y = ca[key], cb[key]
            if key in ('kcache', 'vcache'):
                x, y = x.view(R, h, n, dh)[:, :, :P], y.view(R, h, n, dh)[:, :, :P]
            elif key == 'gn_hist':
                x, y = x[:, :P], y[:, :P]
            else:
                x, y = x[:, P & 1], y[:, P & 1]
            scale = float(x.abs().max())
            assert scale > 0, (i, key)
            err = float((x - y).abs().max())
            assert err <= 1e-5 * scale, (i, key, err, scale)
            checked += 1
    assert checked >= 4 * cfg['depth']
    la, lb = a.logits_all.cpu().numpy()[:, P], b.logits_all.cpu().numpy()[:, P]
    assert np.abs(la - lb).max() <= 1e-5 * max(1.0, np.abs(la).max())


@pytest.mark.parametrize('R', [1, 24])
@pytest.mark.parametrize('name,mp', [('tiny_glu_sgu', False), ('bf_sgu', True)])
def test_scatter_at_1_and_24_rows(name, mp, R):
    """the scatter from fp32 and bf16 forwards into 1 and 24 decoder rows (8 distinct prompts for 24 rows): every row's
    caches agree with the decode kernel's prefill (fp32 round-off; bf16 activations in the mixed-precision forward)"""
    kw, cfg, params = _case(name)
    n, h, dh = cfg['seq_len'], cfg['heads'], cfg['dim_head']
    P = n // 2 - 3
    distinct = _prompts(np.random.default_rng(R), [P] * min(R, 8))
    prompts = [distinct[r % len(distinct)] for r in range(R)]
    _, a, b = _both(kw, cfg, params, prompts, mp)
    tol = 5e-2 if mp else 1e-5
    for ca, cb in zip(a.caches, b.caches):
        for key in ('kcache', 'vcache', 'gn_hist'):
            if key not in ca:
                continue
            x = ca[key].view(R, -1, n, ca[key].shape[-1] if key == 'gn_hist' else dh)[:, :, :P]
            y = cb[key].view(R, -1, n, ca[key].shape[-1] if key == 'gn_hist' else dh)[:, :, :P]
            for r in range(R):
                assert float((x[r] - y[r]).abs().max()) <= tol * float(x[r].abs().max()), (key, r)


@pytest.mark.parametrize('L', [0, 1, 2])
@pytest.mark.parametrize('name', ['tiny_all_glu', 'bf_sgu', 'bf_h8'])
def test_bf16_first_draw_logits_within_the_forward_error(name, L):
    """bf16 model: the decoder's logits at the first drawn position, after a forward prefill, are as close to the float64
    oracle as the engine's own `.apply` logits at that position (within 2x)"""
    from oracle import progen_ref as O
    kw, cfg, params = _case(name)
    n = cfg['seq_len']
    P = _lengths(n)[L]
    prompts = _prompts(np.random.default_rng(100 + P), [P, P])
    model, a, b = _both(kw, cfg, params, prompts, mp=True)
    rows = np.zeros((2, n), np.int64)
    for r, pr in enumerate(prompts):
        rows[r, 1:1 + P] = pr
    applied = model.apply(params, None, rows).cpu().numpy().astype(np.float64)
    got = b.logits_all.cpu().numpy().astype(np.float64)
    for r in range(2):
        ref = O.forward(params, rows[r], cfg)[P]
        e_apply = np.abs(applied[r, P] - ref).max()
        e_prefill = np.abs(got[r, P] - ref).max()
        assert e_prefill <= 2 * e_apply, (r, e_prefill, e_apply)


@pytest.mark.parametrize('name', TINY)
def test_greedy_long_prompt_matches_oracle(name):
    from progen_b200 import ProGen
    from progen_b200.decode import BatchDecoder
    from oracle import progen_ref as O
    kw, cfg, params = _case(name)
    n = cfg['seq_len']
    prompts = _prompts(np.random.default_rng(2), [n // 2 + 3] * 2)
    model = ProGen(**kw)
    model._ensure_loaded(params)
    dec = BatchDecoder(cfg, params, batch=2, keep_logits=True)
    P = dec.prefill(model.engine, prompts)
    res = dec.generate(prompts, temperature=0.0, seed=5, prefilled=P)
    got = dec.logits_all.cpu().numpy()
    for b in range(2):
        assert res['start'][b] == P + 1 and (res['ids'][b, 1:P + 1] == prompts[b]).all()
        ref = O.forward(params, res['ids'][b], cfg)
        assert np.abs(got[b, P:n - 1] - ref[P:n - 1]).max() < 2e-5 * max(1.0, np.abs(ref).max()), b
        checked = 0
        for t in range(P + 1, min(int(res['end'][b]) + 1, n)):
            top2 = np.sort(ref[t - 1].astype(np.float64))[-2:]
            if top2[1] - top2[0] > 1e-3:
                assert res['ids'][b, t] == np.argmax(ref[t - 1]), (b, t)
                checked += 1
        assert checked > 0


def test_token_logp_equals_score():
    from progen_b200 import ProGen
    kw, cfg, params = _case('tiny_glu_sgu')
    model = ProGen(**kw)
    prompts = _prompts(np.random.default_rng(3), [0, 2, 9, 20, 9])
    res = model.generate(params, prompts, num_samples=3, temperature=1.0, seed=9, top_p=0.95, prefill='forward')
    rows = np.concatenate([res['tokens'], np.zeros((len(res['tokens']), 1), np.int64)], axis=1)
    sc = model.score(params, rows, return_tokens=True)['token_logp']
    for i in range(len(rows)):
        s, ln = int(res['start'][i]), int(res['length'][i])
        want = sc[i, s - 1:s - 1 + ln].astype(np.float64)
        got = res['token_logp'][i, s:s + ln].astype(np.float64)
        assert np.abs(got - want).max() < 1e-4, i
        assert (res['token_logp'][i, :s] == 0).all() and (res['token_logp'][i, s + ln:] == 0).all()


KEYS = ('tokens', 'token_logp', 'length', 'finished', 'start', 'log_likelihood')


def _same(a, b, rows_a, rows_b, what):
    for k in KEYS:
        np.testing.assert_array_equal(a[k][rows_a], b[k][rows_b], err_msg=f'{k}: {what}')


@pytest.mark.parametrize('name,mp', [('tiny_glu_sgu', False), ('h8', False), ('bf_sgu', True)])
def test_rows_do_not_depend_on_their_company(name, mp):
    """prefill='forward': a row is bitwise the same whether its prompt shares the launch (and the forward) with 0, 1 or 63
    other prompts of equal or different length, whether it is deduplicated, and for every batch_size of one class"""
    from progen_b200 import ProGen
    kw, cfg, params = _case(name)
    model = ProGen(**kw, mixed_precision=mp)
    rng = np.random.default_rng(11)
    A, B, C = _prompts(rng, [12, 12, 20])
    others = _prompts(rng, [12] * 63)
    kw_ = dict(temperature=1.0, top_p=0.9, seed=23, prefill='forward')
    alone = model.generate(params, [A], num_samples=9, **kw_)                      # 9 rows: the 9-64 class
    _same(alone, model.generate(params, [A, B], num_samples=9, **kw_), slice(0, 9), slice(0, 9), 'with B (same length)')
    _same(alone, model.generate(params, [A, C], num_samples=9, **kw_), slice(0, 9), slice(0, 9), 'with C (other length)')
    crowd = model.generate(params, [A] + others, num_samples=1, **kw_)            # 64 distinct prompts in one forward
    _same(alone, crowd, slice(0, 1), slice(0, 1), '63 other prompts')
    dedup = model.generate(params, [A] * 64, num_samples=1, **kw_)                 # 64 copies: one forward row
    _same(alone, dedup, slice(0, 9), slice(0, 9), '64 copies')
    many = model.generate(params, [A, C, B], num_samples=30, batch_size=64, **kw_)
    for bs in (12, 30, 9):
        _same(many, model.generate(params, [A, C, B], num_samples=30, batch_size=bs, **kw_), slice(None), slice(None),
              f'batch_size {bs}')
    # the empty prompt has nothing to prefill: both modes are one computation
    e = dict(kw_, prefill='decode')
    _same(model.generate(params, ['', A], num_samples=9, **kw_), model.generate(params, ['', A], num_samples=9, **e),
          slice(0, 9), slice(0, 9), 'empty prompt')


@pytest.mark.parametrize('constrained', [False, True])
def test_mixed_lengths_come_back_in_prompt_order(constrained):
    """prompts of different lengths (one empty) in one call: prompt-major rows with the right start, length, finished and
    prompt_index, each bitwise equal to its prompt generated on its own with the same sample ids and launch class"""
    from progen_b200 import ProGen
    from progen_b200.decode import BatchDecoder
    from generate import alphabet_bias
    kw, cfg, params = _case('tiny_gelu_sgu')
    n = cfg['seq_len']
    model = ProGen(**kw)
    prompts = _prompts(np.random.default_rng(6), [5, 0, 30, 5])
    S = 4
    con = dict(logit_bias=alphabet_bias(ALPHABET, 256), min_new_tokens=3, repetition_penalty=1.3,
               repetition_window=8) if constrained else {}
    kw_ = dict(temperature=1.0, top_k=40, seed=4, **con)
    res = model.generate(params, prompts, num_samples=S, prefill='forward', **kw_)
    N = len(prompts) * S
    np.testing.assert_array_equal(res['prompt_index'], np.repeat(np.arange(len(prompts)), S))
    end = np.where(res['finished'], res['start'] + res['length'] - 1, n)
    model._ensure_loaded(params)
    dec = BatchDecoder(cfg, params, batch=N)                # per_launch = N = 16: the 9-64 class
    for i, pr in enumerate(prompts):
        rows = np.arange(i * S, (i + 1) * S)
        sids = np.concatenate([rows, np.full(9 - S, rows[-1])])
        chunk = [pr] * len(sids)
        P = dec.prefill(model.engine, chunk)
        one = dec.generate(chunk, sample_ids=sids, prefilled=P, **kw_)
        np.testing.assert_array_equal(res['start'][rows], 1 + len(pr))
        np.testing.assert_array_equal(res['tokens'][rows], one['ids'][:S])
        np.testing.assert_array_equal(res['token_logp'][rows], one['token_logp'][:S])
        np.testing.assert_array_equal(end[rows], one['end'][:S])
        assert (res['tokens'][rows, 1:1 + len(pr)] == pr).all()
        if constrained:
            gen = np.concatenate([res['tokens'][r, res['start'][r]:res['start'][r] + res['length'][r] - int(res['finished'][r])]
                                  for r in rows])
            assert set((gen - 1).tolist()) <= {ord(c) for c in ALPHABET}
            assert (res['length'][rows][res['finished'][rows]] > 3).all()


def test_decode_mode_is_the_default():
    from progen_b200 import ProGen
    kw, cfg, params = _case('tiny_glu_sgu')
    model = ProGen(**kw)
    prompts = _prompts(np.random.default_rng(8), [0, 3, 7])
    kw_ = dict(num_samples=5, temperature=0.8, top_k=30, seed=3)
    a = model.generate(params, prompts, **kw_)
    b = model.generate(params, prompts, prefill='decode', **kw_)
    _same(a, b, slice(None), slice(None), "prefill='decode' vs omitted")


def test_prefill_argument_checks():
    from progen_b200 import ProGen
    from progen_b200.decode import BatchDecoder
    from progen_b200.lib import ProgenError
    kw, cfg, params = _case('tiny_glu_sgu')
    model = ProGen(**kw)
    model._ensure_loaded(params)
    dec = BatchDecoder(cfg, params, batch=4)
    with pytest.raises(ProgenError):
        dec.prefill(model.engine, [np.array([3, 4]), np.array([5])])              # lengths differ
    with pytest.raises(ProgenError):
        dec.prefill(model.engine, [np.array([3, 4])] * 5)                          # more rows than the decoder holds
    other = ProGen(**{**kw, 'depth': 2})
    with pytest.raises(ProgenError):
        dec.prefill(other.engine, [np.array([3, 4])])
    P = dec.prefill(model.engine, [np.array([3, 4])])
    with pytest.raises(ProgenError):
        dec.generate([np.array([3])], prefilled=P)                                 # prompt shorter than the prefill
