"""The model options every other test holds fixed (num_tokens 256, ff_mult 4, shift_tokens on, dim_head 32 / 64) at other
values, through every path that reads them, against the float64 oracle (oracle/progen_torch.py on the GPU).

Each configuration differs from the tested defaults in one or two options and is small enough for the oracle to take
seconds (depth 2: one GLU or GELU layer and one gMLP layer, seq_len 64 or 128):

  name       options                                  what it reaches
  v24        num_tokens 24                            V not a multiple of 32: partial lane groups of the row loops,
                                                      a head GEMV with fewer row pairs than CTAs
  v328       num_tokens 328                           V > 256, not a multiple of 64: two ids per sampler thread
  v384       num_tokens 384                           the engine's largest V (embed_bwd's bins fill 48 KB)
  v64_d64    num_tokens 64, dim 64, heads 1           one partial wgmma tile for the head, every N or K = 64 GEMM
  v320       num_tokens 320                           a 64-column tail in the wgmma head GEMM
  ff2        ff_mult 2                                hid = 256, the narrowest feed-forward the decoder takes
  ff3        ff_mult 3                                hid = 384: trains and scores, no persistent decoder
  no_shift   shift_tokens False                       no token shift in any LayerNorm, GLU and gMLP layers
  dh128      dim_head 128, dim 256                    attn_simt's DH = 128 kernels; no persistent decoder
  dh16_gelu  dim_head 16, ff_glu False, dim 64        the NL = 4 decode attention and the GELU layer in the 9-64 tile

Paths (T: tested here; R: a tested refusal; a, b, c: not run, for the reason given below the table):

  path                                        v24  v328  v384  v64_d64  v320  ff2  ff3  no_shift  dh128  dh16_gelu
  training, apply and score, fp32              T    T     T     T        T     T    T    T         T      T
  training, apply and score, mixed precision   a    a     T     T        T     T    T    T         R      a
  persistent decoder, fp32 and bf16 weights    T    T     T     T        T     T    R    T         R      T
  standard sampler: host replay                T    T     T     b        b     b    R    b         R      b
  reference sampler (BatchDecoder 1)           c    T     c     c        c     c    R    T         R      c
  forward prefill, fp32                        T    T     T     T        T     T    R    T         R      T
  forward prefill, mixed precision             a    a     T     T        T     T    R    T         R      a

  a: mixed precision needs dim, heads * dim_head, seq_len and num_tokens multiples of 64 and dim_head 64; the engine
     refuses the rest (test_gpu_model.py::test_mixed_precision_refuses_shapes_without_a_tensor_core_kernel);
  b: the sampler reads only V and the logits: V = 24 (fewer ids than threads), 328 (a partial second id per thread) and
     384 cover its classes, 64 and 320 fall inside them, 256 is test_gpu_generate.py's;
  c: the reference sampler is the persistent decoder's sampler 0 at one row, whose kernel the row above runs at every
     option; it runs once per option the full re-forward reads differently: V > 256 (two ids per sampler thread) and no
     token shift;
  R: ProGen.generate and BatchDecoder raise ProgenError naming the limit (hid % 256, dim_head <= 64) before allocating;
     the mixed-precision engine refuses dim_head 128.

Kernels at the new values, beside the model-level checks: progen_local_attn_{fwd,bwd}_simt at dim_head 128,
progen_ce_fwd_bwd / progen_token_logprob at V = 24, 328, 384, progen_embed_bwd at V = 384 with d % 32 != 0, the wgmma
GEMM with N = 64 (every epilogue, both B majors) and K = 64.

Bounds are those of the existing tests, quoted where they are used.  Each case prints its measured errors and bounds as
JSON lines."""
import functools

import numpy as np
import pytest
import torch

from test_gpu_elementwise import attn_ref
from test_gpu_gemm_tc import COMBOS, _tol
from test_gpu_generate import _drawn, gumbel, host_draw, host_filter
from test_gpu_generate_prefill import _both
from test_gpu_large_config_inference import _cache_views, _maxabs, _oracle, _report
from test_gpu_score import _pool, _token_logprob

pytestmark = pytest.mark.gpu

_STACK = dict(depth=2, global_mlp_depth=1)
CONFIGS = {
    'v24': dict(num_tokens=24, dim=64, seq_len=64, window_size=32, heads=2, dim_head=32),
    'v328': dict(num_tokens=328, dim=128, seq_len=64, window_size=32, heads=2, dim_head=64),
    'v384': dict(num_tokens=384, dim=128, seq_len=128, window_size=64, heads=2, dim_head=64),
    'v64_d64': dict(num_tokens=64, dim=64, seq_len=128, window_size=64, heads=1, dim_head=64),
    'v320': dict(num_tokens=320, dim=128, seq_len=128, window_size=64, heads=2, dim_head=64),
    'ff2': dict(num_tokens=256, dim=128, seq_len=128, window_size=64, heads=2, dim_head=64, ff_mult=2),
    'ff3': dict(num_tokens=256, dim=128, seq_len=128, window_size=64, heads=2, dim_head=64, ff_mult=3),
    'no_shift': dict(num_tokens=256, dim=128, seq_len=128, window_size=64, heads=2, dim_head=64, shift_tokens=False),
    'dh128': dict(num_tokens=256, dim=256, seq_len=64, window_size=32, heads=2, dim_head=128),
    'dh16_gelu': dict(num_tokens=256, dim=64, seq_len=64, window_size=16, heads=4, dim_head=16, ff_glu=False),
}
NAMES = list(CONFIGS)
MIXED = ['v384', 'v64_d64', 'v320', 'ff2', 'ff3', 'no_shift']     # shapes the tensor-core engine takes
NO_DECODER = ['ff3', 'dh128']                                      # hid % 256 != 0, dim_head > 64
DECODABLE = [n for n in NAMES if n not in NO_DECODER]
TRAIN = [(name, mp) for name in NAMES for mp in (False, True) if not mp or name in MIXED]


@functools.lru_cache(maxsize=None)
def _model(name, rounded=False):
    """(kwargs, cfg, params) of configuration `name`, randomized parameters; `rounded`: the weight matrices ('w' leaves)
    rounded to bf16, the weights a bf16-weight decoder multiplies with"""
    from oracle import progen_ref as O
    kw = {**_STACK, **CONFIGS[name]}
    cfg = O.make_config(**kw)
    s = 10 * (NAMES.index(name) + 1)
    params = O.randomize_params(O.init_params(cfg, s), s + 1)
    if rounded:
        rnd = lambda a: torch.tensor(np.asarray(a, np.float32)).bfloat16().float().numpy()
        params = {k: {kk: (rnd(vv) if kk == 'w' else vv) for kk, vv in v.items()} for k, v in params.items()}
    return kw, cfg, params


def _prompts(rng, lengths, V):
    return [rng.integers(1, V, L).astype(np.int64) for L in lengths]


def _rows(rng, R, n, V):
    """R rows of n + 1 ids in [1, V), row 1 ending early (EOS + padding)"""
    data = rng.integers(1, V, (R, n + 1)).astype(np.uint16)
    data[1, 1 + int(rng.integers(n // 4, 3 * n // 4)):] = 0
    return data


# ------------------------------------------------------------------------------------------------ training and apply
@pytest.mark.parametrize('name,mp', TRAIN)
def test_loss_grad_and_apply(name, mp):
    """loss_and_grad against the float64 loss and gradients with one row ending early: loss within 2e-5 (fp32) / 3e-2
    (mixed precision), every leaf within 3e-4 / 0.12 of its max (test_gpu_model.py::test_edge_configs_loss_and_grad).
    `.apply` logits: fp32 within 1e-5 * max|logit| (::test_fp32_apply_matches_reference_golden); mixed precision max
    error < 5e-2 and mean < 1e-2 (::test_bf16_apply)."""
    from progen_b200 import ProGen
    from oracle import progen_torch as T
    kw, cfg, params = _model(name)
    n, V = cfg['seq_len'], cfg['num_tokens']
    data = _rows(np.random.default_rng(n + V), 2, n, V)
    ref_loss, ref = T.loss_and_grads(params, data, cfg, device='cuda')
    model = ProGen(**kw, mixed_precision=mp)
    loss, grads = model.loss_and_grad(params, data)
    worst, leaf = 0.0, None
    for m, d in ref.items():
        for k, r in d.items():
            rel = float(np.abs(grads[m][k] - r).max()) / max(1e-8, float(np.abs(r).max()))
            if rel >= worst:
                worst, leaf = rel, f'{m}/{k}'
    lg = model.apply(params, None, data[:, :-1]).double()
    ref_lg = _oracle(params, data[:, :-1], cfg)
    err = (lg - ref_lg).abs()
    case = f'train_{name}_mp{int(mp)}'
    if mp:
        _report(case=case, loss_err=abs(loss - ref_loss), loss_bound=3e-2, grad_rel=worst, grad_bound=0.12, leaf=leaf,
                logits_max=float(err.max()), logits_mean=float(err.mean()), logits_bound_max=5e-2, logits_bound_mean=1e-2)
        assert abs(loss - ref_loss) < 3e-2, (loss, ref_loss)
        assert worst < 0.12, (leaf, worst)
        assert float(err.max()) < 5e-2 and float(err.mean()) < 1e-2
    else:
        scale = max(1.0, _maxabs(ref_lg))
        _report(case=case, loss_err=abs(loss - ref_loss), loss_bound=2e-5, grad_rel=worst, grad_bound=3e-4, leaf=leaf,
                logits_err=float(err.max()), logits_bound=1e-5 * scale)
        assert abs(loss - ref_loss) < 2e-5, (loss, ref_loss)
        assert worst < 3e-4, (leaf, worst)
        assert float(err.max()) < 1e-5 * scale


# ------------------------------------------------------------------------------------------------ score and embed
@pytest.mark.parametrize('name,mp', TRAIN)
def test_score_and_embed(name, mp):
    """`score`'s token log-probabilities, log-likelihoods and counts are bitwise progen_token_logprob of `.apply`'s logits
    (test_gpu_score.py::test_score_is_the_apply_forward).  Pooled embedding, with the bounds of
    test_gpu_large_config_inference.py::test_score_and_embed: fp32 within 1e-5 * max of the pooled float64 final-LayerNorm
    output, and -ll / count within 1e-5 of the float64 cross entropy; mixed precision max < 5e-2 and mean < 1e-2 against
    float64 and against the bf16-operand emulation."""
    from progen_b200 import ProGen
    from oracle import progen_torch as T
    kw, cfg, params = _model(name)
    n, V = cfg['seq_len'], cfg['num_tokens']
    data = _rows(np.random.default_rng(n + V + 1), 3, n, V)
    model = ProGen(**kw, mixed_precision=mp)
    logits = model.apply(params, None, data[:, :-1])
    lp, ll, cnt = _token_logprob(logits, data[:, 1:])
    sc = model.score(params, data, return_tokens=True, return_embeddings=True)
    np.testing.assert_array_equal(sc['token_logp'], lp)
    np.testing.assert_array_equal(sc['log_likelihood'], ll)
    np.testing.assert_array_equal(sc['num_tokens'], cnt.astype(np.int64))
    assert sc['num_tokens'][1] < n and (sc['num_tokens'][[0, 2]] == n).all()
    emb = sc['embedding'].astype(np.float64)
    ids = data[:, :-1].astype(np.int64)
    ref, hid = _oracle(params, ids, cfg, hidden=True)
    ref_emb = _pool(hid.cpu().numpy(), data)
    case = f'score_{name}_mp{int(mp)}'
    if not mp:
        labels = torch.as_tensor(data[:, 1:].astype(np.int64), device='cuda')
        ce = -sc['log_likelihood'].astype(np.float64) / sc['num_tokens']
        e_ce = float(np.abs(ce - T.cross_entropy(ref, labels).cpu().numpy()).max())
        e_emb, emb_scale = float(np.abs(emb - ref_emb).max()), max(1.0, float(np.abs(ref_emb).max()))
        _report(case=case, ce_err=e_ce, ce_bound=1e-5, emb_err=e_emb, emb_bound=1e-5 * emb_scale)
        assert e_ce < 1e-5
        assert e_emb < 1e-5 * emb_scale
        return
    _, hid = _oracle(params, ids, cfg, torch.float32, T.bf16_round, hidden=True)
    emu_emb = _pool(hid.double().cpu().numpy(), data)
    err, e2 = np.abs(emb - ref_emb), np.abs(emb - emu_emb)
    _report(case=case, emb_err_max=float(err.max()), emb_err_mean=float(err.mean()), emu_err_max=float(e2.max()),
            emu_err_mean=float(e2.mean()), bound_max=5e-2, bound_mean=1e-2)
    assert err.max() < 5e-2 and err.mean() < 1e-2
    assert e2.max() < 5e-2 and e2.mean() < 1e-2


# ------------------------------------------------------------------------------------------------ persistent decoder
DECODE = [(name, B, wdt) for name in DECODABLE for B in (1, 5, 20, 40) for wdt in ('f32', 'bf16')]


@pytest.mark.parametrize('name,B,wdt', DECODE)
def test_decoder_logits_at_every_position(name, B, wdt):
    """Greedy generation to the full length (min_new_tokens = n bans EOS) from prompts of 1-8 ids at B = 1 / 5 / 20 / 40
    (the single-stream path, the 2-8 tile, the 32-sequence tile, two passes of it): logits_all of rows 0, B // 2 and
    B - 1 at every position against the float64 oracle of the ids the row ended with (bf16 weights: the oracle on the
    bf16-rounded weights), within 1e-4 * max|logit|; greedy ids equal the oracle's argmax wherever its top-2 gap exceeds
    1e-3 (test_gpu_large_config_inference.py::test_decoder_logits_at_every_position)."""
    from progen_b200.decode import BatchDecoder
    kw, cfg, params = _model(name)
    n, V = cfg['seq_len'], cfg['num_tokens']
    rng = np.random.default_rng(B + V)
    prompts = _prompts(rng, rng.integers(1, 9, B), V)
    dec = BatchDecoder(cfg, params, batch=B, weights_dtype=torch.bfloat16 if wdt == 'bf16' else torch.float32,
                       keep_logits=True)
    res = dec.generate(prompts, temperature=0.0, min_new_tokens=n)
    rows = sorted({0, B // 2, B - 1})
    got = dec.logits_all[rows, :n - 1].double()
    del dec
    assert (res['end'] == n).all()
    ids = res['ids'][rows]
    ref = _oracle(_model(name, rounded=wdt == 'bf16')[2], ids, cfg)[:, :n - 1]
    err, scale = _maxabs(got - ref), max(1.0, _maxabs(ref))
    ref = ref.cpu().numpy()[:, :, 1:]                      # the ids a draw may take (EOS banned by min_new_tokens)
    checked = 0
    for j, b in enumerate(rows):
        s = int(res['start'][b])
        assert res['ids'][b, 0] == 0 and (res['ids'][b, 1:s] == prompts[b]).all()
        lg = ref[j, s - 1:]
        top2 = np.sort(lg, axis=-1)[:, -2:]
        clear = top2[:, 1] - top2[:, 0] > 1e-3
        np.testing.assert_array_equal(ids[j, s:][clear], 1 + np.argmax(lg, axis=-1)[clear], err_msg=f'row {b}')
        checked += int(clear.sum())
    _report(case=f'decode_{name}_B{B}_{wdt}', err=err, bound=1e-4 * scale, ids_checked=checked,
            max_id=int(res['ids'].max()))
    assert err < 1e-4 * scale, (err, scale)
    assert checked > len(rows) * (n // 4)


# ------------------------------------------------------------------------------------------------ standard sampler
@pytest.mark.parametrize('name', ['v24', 'v328', 'v384'])
def test_sampler_matches_host_replay(name):
    """T x top_k x top_p grid (top_k <= V) at B = 24 (test_gpu_generate.py::test_sampler_matches_host_replay): the kernel's
    id == the float64 host replay (Philox noise, filter, Gumbel-max on the kernel's own logits) wherever the draw is
    unambiguous, >= 99 % of draws are, every id lies in the kept set; at V > 256 ids >= 256 are drawn."""
    from progen_b200.decode import BatchDecoder
    kw, cfg, params = _model(name)
    V, B, max_length = cfg['num_tokens'], 24, 64
    rng = np.random.default_rng(7)
    prompts = _prompts(rng, rng.integers(0, 9, B), V)
    dec = BatchDecoder(cfg, params, batch=B, keep_logits=True)
    total = unamb = high = 0
    seed = 0x1234_5678_9ABC
    for T in (0.7, 1.0, 1.5):
        for top_k in (None, 5, min(40, V)):
            for top_p in (None, 0.5, 0.9):
                sids = np.arange(B, dtype=np.int64) * 1000 + (1 << 33)
                res = dec.generate(prompts, temperature=T, top_k=top_k, top_p=top_p, seed=seed, sample_ids=sids,
                                   max_length=max_length)
                lg = dec.logits_all.cpu().numpy()
                for b in range(B):
                    for t in _drawn(res, b, max_length):
                        want, keep, amb = host_draw(lg[b, t - 1], T, top_k, top_p, gumbel(seed, int(sids[b]), t, V))
                        got = int(res['ids'][b, t])
                        assert keep[got], (T, top_k, top_p, b, t, got)
                        total += 1
                        high += got >= 256
                        if not amb:
                            unamb += 1
                            assert got == want, (T, top_k, top_p, b, t, got, want)
    _report(case=f'sampler_{name}', draws=total, unambiguous=unamb, ids_at_least_256=high)
    assert total > 1000 and unamb >= 0.99 * total, (unamb, total)
    assert high > 0 if V > 256 else high == 0


def test_first_draw_distribution_chi_square_v384():
    """first drawn position over many sample ids at V = 384 against the exact filtered softmax of the float64 logits,
    chi-square at the 0.1 % level (test_gpu_generate.py::test_first_draw_distribution_chi_square)"""
    from scipy import stats
    from progen_b200.decode import BatchDecoder
    kw, cfg, params = _model('v384')
    n, V, B, runs, T = cfg['seq_len'], cfg['num_tokens'], 64, 40, 1.3
    prompt = np.array([300, 5, 270, 77, 383], np.int64)
    row = np.zeros(n, np.int64)
    row[1:1 + len(prompt)] = prompt
    l = _oracle(params, row[None], cfg)[0, len(prompt)].cpu().numpy()
    # a nucleus whose cumulative mass is not within 1e-4 of a boundary (the draw must not hinge on round-off)
    top_p = next(p for p in (0.95, 0.93, 0.9, 0.85) if not host_filter(l, T, None, p, tol=1e-4)[1])
    keep, _ = host_filter(l, T, None, top_p)
    z = np.where(keep, l / T, -np.inf)
    probs = np.exp(z - z.max())
    probs /= probs.sum()
    dec = BatchDecoder(cfg, params, batch=B)
    counts = np.zeros(V, np.int64)
    for r in range(runs):
        res = dec.generate([prompt] * B, temperature=T, top_p=top_p, seed=11, sample_ids=np.arange(r * B, (r + 1) * B),
                           max_length=len(prompt) + 2)
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
    _report(case='chi_square_v384', top_p=top_p, kept=int(keep.sum()), mass_at_least_256=float(probs[256:].sum()),
            drawn_at_least_256=int(counts[256:].sum()), chi2=float(chi2), pval=float(pval))
    assert counts[256:].sum() > 0
    assert pval > 1e-3, (chi2, len(obs), pval)


@pytest.mark.parametrize('name', ['v328', 'v384'])
def test_logit_bias_banning_every_id_below_256(name):
    """a logit_bias of -inf on ids 0..255 leaves only ids >= 256: every draw is one, and equals the host replay restricted
    to them wherever that is unambiguous (ProGen.generate too)"""
    from progen_b200 import ProGen
    from progen_b200.decode import BatchDecoder
    kw, cfg, params = _model(name)
    V, B, max_length, seed = cfg['num_tokens'], 24, 48, 5
    bias = np.zeros(V, np.float32)
    bias[:256] = -np.inf
    prompts = _prompts(np.random.default_rng(9), [3] * B, V)
    dec = BatchDecoder(cfg, params, batch=B, keep_logits=True)
    total = unamb = 0
    for T, top_k, top_p in ((0.0, None, None), (1.0, None, None), (0.7, 5, None), (1.5, None, 0.9)):
        res = dec.generate(prompts, temperature=T, top_k=top_k, top_p=top_p, seed=seed, logit_bias=bias,
                           max_length=max_length)
        assert (res['end'] == cfg['seq_len']).all()
        lg = dec.logits_all.cpu().numpy()
        for b in range(B):
            for t in _drawn(res, b, max_length):
                got = int(res['ids'][b, t])
                assert got >= 256, (T, top_k, top_p, b, t, got)
                want, keep, amb = host_draw(lg[b, t - 1, 256:], T, top_k, top_p, gumbel(seed, b, t, V)[256:])
                assert keep[got - 256]
                total += 1
                if not amb:
                    unamb += 1
                    assert got == 256 + want, (T, top_k, top_p, b, t, got, want)
    _report(case=f'logit_bias_{name}', draws=total, unambiguous=unamb)
    assert unamb >= 0.99 * total
    out = ProGen(**kw).generate(params, prompts[:4], num_samples=2, temperature=1.0, seed=1, logit_bias=bias,
                                max_length=max_length)
    assert not out['finished'].any()
    for i in range(len(out['tokens'])):
        s = int(out['start'][i])
        assert (out['tokens'][i, s:max_length] >= 256).all()


# ------------------------------------------------------------------------------------------------ reference sampler
@pytest.mark.parametrize('name', ['v328', 'no_shift'])
def test_persistent_reference_sampler_equals_full_reforward(name):
    """`BatchDecoder(batch=1)` greedy ids == the full re-forward `utils.sample` over `ProGen.apply`
    (test_gpu_decode.py::test_persistent_decode_equals_full_reforward_sampler_cfg1_size), and its logits at every position
    within 2e-5 * max|logit| of the float64 oracle (::test_persistent_logits_match_oracle_forward)."""
    from progen_b200 import ProGen
    from progen_b200.decode import BatchDecoder
    from progen_b200.utils import sample
    kw, cfg, params = _model(name)
    n, V = cfg['seq_len'], cfg['num_tokens']
    prime = _prompts(np.random.default_rng(V + n), [6], V)[0]
    dec = BatchDecoder(cfg, params, batch=1, keep_logits=True)
    ids, _, _ = dec.sample(prime, top_k=25, add_bos=True, greedy=True)
    seq = dec.seq[0].cpu().numpy().astype(np.int64)               # before the post-hoc truncation
    got = dec.logits_all[0, :n - 1].double()
    ref = _oracle(params, np.clip(seq, 0, V - 1)[None], cfg)[0, :n - 1]
    err, scale = _maxabs(got - ref), max(1.0, _maxabs(ref))
    want = sample(0, ProGen(**kw).apply, params, prime, n, top_k=25, add_bos=True, greedy=True)
    _report(case=f'reference_sampler_{name}', err=err, bound=2e-5 * scale, max_id=int(seq.max()))
    assert err < 2e-5 * scale
    np.testing.assert_array_equal(ids, want)


# ------------------------------------------------------------------------------------------------ forward prefill
PREFILL = [(name, mp) for name in DECODABLE for mp in (False, True) if not mp or name in MIXED]


@pytest.mark.parametrize('name,mp', PREFILL)
def test_forward_prefill(name, mp):
    """Prompts of n/2 - 3 ids, three rows, rows 0 and 2 sharing one forward row.  Every layer's K / V rows, token-shift slot
    and SGU gate history at positions < P against the decoder's own prefill, per row: 1e-5 of the row's max (fp32) or 5e-2
    (mixed precision) (test_gpu_generate_prefill.py::test_fp32_caches_match_the_decode_prefill,
    ::test_scatter_at_1_and_24_rows).  shift_tokens off: both decoders' shift slots stay exactly zero.  First drawn
    logits: fp32 within 1e-5 * max|logit| of the decoder's; mixed precision within 2x of `.apply`'s error against float64
    (::test_bf16_first_draw_logits_within_the_forward_error)."""
    kw, cfg, params = _model(name)
    n, V, h, dh = cfg['seq_len'], cfg['num_tokens'], cfg['heads'], cfg['dim_head']
    P = n // 2 - 3
    p = _prompts(np.random.default_rng(P + V), [P, P], V)
    prompts = [p[0], p[1], p[0]]
    model, a, b = _both(kw, cfg, params, prompts, mp)
    tol = 5e-2 if mp else 1e-5
    worst = {}
    for i, (ca, cb) in enumerate(zip(a.caches, b.caches)):
        for key in ca:
            if key.startswith('shift') and not cfg['shift_tokens']:
                assert not ca[key].any() and not cb[key].any(), (i, key)
                worst[key] = 0.0
                continue
            x, y = _cache_views(ca, cb, key, 3, n, h, dh, P)
            for r in range(3):
                scale = _maxabs(x[r])
                assert scale > 0, (i, key, r)
                rel = _maxabs(x[r] - y[r]) / scale
                worst[key] = max(worst.get(key, 0.0), rel)
                assert rel <= tol, (i, key, r, rel, tol)
    assert set(worst) == {'kcache', 'vcache', 'shift1', 'shift2', 'gn_hist'}
    case = f'prefill_{name}_mp{int(mp)}'
    _report(case=case, bound=tol, **{f'{k}_rel': v for k, v in worst.items()})
    la, lb = a.logits_all[:, P].double(), b.logits_all[:, P].double()
    if not mp:
        err, scale = _maxabs(la - lb), max(1.0, _maxabs(la))
        _report(case=case + '_first_draw', err=err, bound=1e-5 * scale)
        assert err <= 1e-5 * scale
        return
    rows = np.zeros((2, n), np.int64)
    for r in range(2):
        rows[r, 1:1 + P] = p[r]
    applied = model.apply(params, None, rows)[:, P].double()
    ref = _oracle(params, rows, cfg)[:, P]
    for r in range(2):
        e_apply, e_prefill = _maxabs(applied[r] - ref[r]), _maxabs(lb[r] - ref[r])
        _report(case=case + f'_first_draw_row{r}', err=e_prefill, bound=2 * e_apply)
        assert e_prefill <= 2 * e_apply, (r, e_prefill, e_apply)


# ------------------------------------------------------------------------------------------------ refusals
@pytest.mark.parametrize('name,extra,limit', [('dh128', {}, 'dim_head'), ('ff3', {}, 'ff_mult'),
                                              ('ff3', {'ff_mult': 1}, 'ff_mult')])
def test_decoders_refuse_what_they_cannot_run(name, extra, limit):
    """configurations the engine trains (test_loss_grad_and_apply) but the persistent decoder cannot run: BatchDecoder
    raises ProgenError naming the limit before it allocates a device buffer, and so does ProGen.generate"""
    from progen_b200 import ProGen
    from progen_b200.decode import BatchDecoder
    from progen_b200.lib import ProgenError
    from oracle import progen_ref as O
    kw, cfg, params = _model(name)
    if extra:
        kw = {**kw, **extra}
        cfg = O.make_config(**kw)
        params = O.init_params(cfg, 3)
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    with pytest.raises(ProgenError, match=limit):
        BatchDecoder(cfg, params, batch=4)
    assert torch.cuda.memory_allocated() == before
    with pytest.raises(ProgenError, match=limit):
        ProGen(**kw).generate(params, [np.array([3, 4])], num_samples=2, temperature=0.0, max_length=16)
    with pytest.raises(ProgenError, match=limit):
        ProGen(**kw).generate(params, [np.array([3, 4])], prefill='forward', max_length=16)


# ------------------------------------------------------------------------------------------------ kernels
def _L():
    from progen_b200 import lib as L
    L.require_device()
    return L


@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
@pytest.mark.parametrize('shape', [(2, 64, 32, 2, 128), (1, 96, 48, 3, 128)])
def test_local_attn_simt_dim_head_128(dtype, shape):
    """the DH = 128 instantiations of attn_simt.cu against attn_ref (float64), with the bounds of
    test_gpu_elementwise.py::test_local_attn_simt_fwd_bwd: forward 1e-5 (fp32) / 2e-2 (bf16), backward 2e-5 / 5e-2 of
    max|dqkv|"""
    L = _L()
    B, n, w, h, dh = shape
    g = torch.Generator(device='cuda').manual_seed(n + h)
    T, I = B * n, h * dh
    qkv = torch.randn(T, 3 * I, generator=g, device='cuda').to(dtype)
    out = torch.empty(T, I, device='cuda', dtype=dtype)
    lse = torch.empty(T, h, device='cuda')
    L.check(L.load().progen_local_attn_fwd_simt(qkv.data_ptr(), out.data_ptr(), lse.data_ptr(), L.dt(qkv), B, n, w, h, dh,
                                                L.stream()), 'attn_fwd_simt')
    qd = qkv.double().requires_grad_(True)
    ref = attn_ref(qd, B, n, w, h, dh)
    f32 = dtype == torch.float32
    e_fwd = _maxabs(out.double() - ref)
    dout = torch.randn(T, I, generator=g, device='cuda').to(dtype)
    ref.backward(dout.double())
    dqkv = torch.empty_like(qkv)
    delta = torch.empty(T, h, device='cuda')
    L.check(L.load().progen_local_attn_bwd_simt(qkv.data_ptr(), out.data_ptr(), dout.data_ptr(), lse.data_ptr(),
                                                dqkv.data_ptr(), delta.data_ptr(), L.dt(qkv), B, n, w, h, dh, L.stream()),
            'attn_bwd_simt')
    e_bwd, gscale = _maxabs(dqkv.double() - qd.grad), max(1.0, _maxabs(qd.grad))
    _report(case=f'attn_dh128_{shape}_{str(dtype)[6:]}', fwd_err=e_fwd, fwd_bound=1e-5 if f32 else 2e-2,
            bwd_err=e_bwd, bwd_bound=(2e-5 if f32 else 5e-2) * gscale)
    assert e_fwd < (1e-5 if f32 else 2e-2)
    assert e_bwd < (2e-5 if f32 else 5e-2) * gscale


@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
@pytest.mark.parametrize('V', [24, 328, 384])
def test_cross_entropy_and_token_logprob(V, dtype):
    """progen_ce_fwd_bwd (and, on fp32 logits, progen_token_logprob) at vocabularies that leave a partial group of 128
    columns, with the method and bounds of test_gpu_elementwise.py::test_cross_entropy_fwd_bwd: loss within 1e-4,
    dlogits within 1e-6 (fp32) / 2e-3 * max + 1e-5 (bf16) of float64; token log-probabilities within 1e-5 * max|logit|
    (test_gpu_score.py::test_score_is_the_apply_forward), the counts exact"""
    L = _L()
    from oracle import progen_ref as O
    g = torch.Generator(device='cuda').manual_seed(V)
    B, n = 4, 96
    logits = (torch.randn(B * n, V, generator=g, device='cuda') * 3).to(dtype)
    labels = torch.randint(0, V, (B, n), generator=g, device='cuda', dtype=torch.int32)
    labels[0, :8] = V - 1                   # the last column, in the last (partial) group
    labels[1, 40:] = 0                      # EOS then padding
    labels[2, 0] = 0
    labels[3] = 0
    w = torch.empty(B * n, device='cuda')
    loss = torch.zeros(1, device='cuda')
    dlogits = torch.empty_like(logits)
    L.check(L.load().progen_ce_fwd_bwd(logits.data_ptr(), L.dt(logits), labels.data_ptr(), w.data_ptr(), loss.data_ptr(),
                                       dlogits.data_ptr(), L.dt(dlogits), B, n, V, 1.0 / B, L.stream()), 'ce_fwd_bwd')
    lg = logits.double().view(B, n, V).requires_grad_(True)
    lab = labels.cpu().numpy()
    ref = sum(float(O.cross_entropy(lg[b].detach().cpu().numpy(), lab[b])) for b in range(B)) / B
    logp = torch.log_softmax(lg, -1)
    nll = -logp.gather(-1, labels.long()[..., None])[..., 0]
    mask = torch.as_tensor(np.stack([O.loss_mask(lab[b]) for b in range(B)]), device='cuda').double()
    ((nll * mask).sum(-1) / mask.sum(-1)).mean().backward()
    tol = 1e-6 if dtype == torch.float32 else 2e-3 * _maxabs(lg.grad) + 1e-5
    e_loss, e_grad = abs(loss.item() - ref), _maxabs(dlogits.double().view(B, n, V) - lg.grad)
    rec = dict(case=f'ce_V{V}_{str(dtype)[6:]}', loss_err=e_loss, loss_bound=1e-4 * max(1.0, abs(ref)), grad_err=e_grad,
               grad_bound=tol)
    assert e_loss < 1e-4 * max(1.0, abs(ref))
    assert e_grad < tol
    if dtype == torch.float32:
        lp, ll, cnt = _token_logprob(logits.view(B, n, V), lab)
        ref_lp = (-nll * mask).detach().cpu().numpy()
        scale = max(1.0, _maxabs(lg.detach()))
        rec.update(logprob_err=float(np.abs(lp - ref_lp).max()), logprob_bound=1e-5 * scale)
        np.testing.assert_array_equal(cnt, mask.sum(-1).cpu().numpy())
        assert np.abs(lp - ref_lp).max() < 1e-5 * scale
        assert np.abs(ll - lp.astype(np.float64).sum(-1)).max() <= 1e-5 * max(1.0, float(np.abs(ll).max()))
    _report(**rec)


@pytest.mark.parametrize('V,d', [(384, 100), (24, 36)])
def test_embed_bwd_vocabularies(V, d):
    """progen_embed_bwd at the largest V (V x 32 fp32 bins: all 48 KB of shared memory) and at V = 24, with d % 32 != 0
    (a partial last column block), against a float64 index_add within 1e-4 (test_gpu_elementwise.py::
    test_embed_fwd_bwd_and_colsum)"""
    L = _L()
    g = torch.Generator(device='cuda').manual_seed(V + d)
    T = 5000
    tok = torch.randint(0, V, (T,), generator=g, device='cuda', dtype=torch.int32)
    tok[:16] = V - 1
    table = torch.randn(V, d, generator=g, device='cuda')
    x = torch.empty(T, d, device='cuda')
    L.check(L.load().progen_embed_fwd(tok.data_ptr(), table.data_ptr(), x.data_ptr(), T, d, V, L.stream()), 'embed_fwd')
    assert torch.equal(x, table[tok.long()])
    dx = torch.randn(T, d, generator=g, device='cuda')
    dtab = torch.zeros(V, d, device='cuda')
    L.check(L.load().progen_embed_bwd(tok.data_ptr(), dx.data_ptr(), dtab.data_ptr(), T, d, V, L.stream()), 'embed_bwd')
    ref = torch.zeros(V, d, device='cuda', dtype=torch.float64).index_add_(0, tok.long(), dx.double())
    err = _maxabs(dtab.double() - ref)
    _report(case=f'embed_bwd_V{V}_d{d}', err=err, bound=1e-4)
    assert err < 1e-4


@pytest.mark.parametrize('a_mn,b_mn,epi', COMBOS)
@pytest.mark.parametrize('shape', [(64, 64, 64), (200, 64, 128), (384, 128, 64)])
def test_tc_gemm_n64_and_k64(a_mn, b_mn, epi, shape):
    """wgmma GEMM with N = 64 (one partial column tile: the dim-64 model's QKV / out / head GEMMs, the V = 64 head) and
    K = 64, every instantiated (A major, B major, epilogue), against float64 with test_gpu_gemm_tc.py's tolerances"""
    from progen_b200 import lib as L
    from gemm_cases import run_case
    M, N, K = shape
    if a_mn and M % 8:
        M = 256
    err, scale = run_case(L.BACKEND_TC, torch.bfloat16, M, N, K, a_mn, b_mn, epi, seed=40 + epi,
                          seq_len=64 if epi == L.EPI_ROTARY else None, dim_head=64)
    assert err <= _tol(epi) * max(1.0, scale), (err, scale)
