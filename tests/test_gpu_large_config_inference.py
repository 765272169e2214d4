"""Generation, prompt prefill and scoring of config 3 (d1024 h16x64 w512 n2048) and config 4 (d1536 h8x64 w256 n4096,
inner 512 != d) at their own widths and sequence lengths, against the float64 oracle (oracle/progen_torch.py on the GPU).

The stacks are those of test_gpu_large_configs.py (depth 3: one GLU and two gMLP layers; depth only repeats them), with
randomized biases, LayerNorm scales and spatial weights.  Config 4 reaches decoder geometry no smaller model has: K cut
into 6, 12 and 24 segments of 256 (waves of 5, 2 and 1 row pairs with idle slots), a half-full last activation chunk of
the 2-8-row tile (K = 3072), inner != d, and positions up to 4095 (rotary tables, caches, the SGU history sum).

  * the persistent decoder's logits at every position of a generation to the full length, for each batch-tile class
    (1, 2-8, 9-32, 33-64 rows) with fp32 and bf16 weights, and the greedy ids;
  * the forward prefill (`BatchDecoder.prefill`): caches against the decoder's own prefill and the first drawn logits;
  * `score`: token log-probabilities bitwise equal to the training forward's, logits / cross entropy / pooled embedding
    against float64.

Bounds are those of the existing tests at small shapes, quoted where they are used.  Each case prints its errors, their
bounds, the error of the same oracle evaluated in float32 (the round-off an ideal fp32 engine would have) and its peak
device memory."""
import functools
import gc
import json
import time

import numpy as np
import pytest
import torch

from test_gpu_generate_prefill import _both
from test_gpu_large_configs import CONFIGS, _no_tf32
from test_gpu_score import _pool, _token_logprob

pytestmark = pytest.mark.gpu
NAMES = sorted(CONFIGS)


@pytest.fixture(autouse=True)
def _peak_memory(request):
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    yield
    torch.cuda.synchronize()
    print(json.dumps(dict(case=request.node.callspec.id, peak_device_memory_gib=round(torch.cuda.max_memory_allocated() / 2 ** 30, 2),
                          wall_s=round(time.perf_counter() - t0, 1))))
    gc.collect()
    torch.cuda.empty_cache()


@functools.lru_cache(maxsize=None)
def _model(name, rounded=False):
    """(kwargs, cfg, params) of config `name`; `rounded`: the weight matrices ('w' leaves) rounded to bf16, the weights a
    bf16-weight decoder multiplies with (the other leaves stay fp32 in the decoder too)"""
    from oracle import progen_ref as O
    kw = CONFIGS[name]['kwargs']
    cfg = O.make_config(**kw)
    s = 3 * kw['dim']
    params = O.randomize_params(O.init_params(cfg, s), s + 1)
    if rounded:
        rnd = lambda a: torch.tensor(np.asarray(a, np.float32)).bfloat16().float().numpy()
        params = {k: {kk: (rnd(vv) if kk == 'w' else vv) for kk, vv in v.items()} for k, v in params.items()}
    return kw, cfg, params


def _oracle(params, ids, cfg, dtype=torch.float64, operand_round=None, hidden=False):
    """oracle forward of ids [R, n] on the GPU -> logits [R, n, V] (and the final LayerNorm output) as device tensors"""
    from oracle import progen_torch as T
    if dtype != torch.float64:
        _no_tf32()
    with torch.no_grad():
        prm = T.to_torch(params, dtype, device='cuda')
        return T.forward(prm, torch.as_tensor(np.asarray(ids, np.int64)), cfg, operand_round, device='cuda',
                         return_hidden=hidden)


def _maxabs(t):
    return float(t.abs().max())


def _report(**kw):
    print(json.dumps({k: (float(f'{v:.3e}') if isinstance(v, float) else v) for k, v in kw.items()}))


def _prompts(rng, lengths):
    return [rng.integers(1, 256, L).astype(np.int64) for L in lengths]


# ------------------------------------------------------------------------------------------------ persistent decoder
DECODE = [(name, B, wdt) for name in NAMES for B in (1, 5, 20, 64) for wdt in ('f32', 'bf16')]


@pytest.mark.parametrize('name,B,wdt', DECODE)
def test_decoder_logits_at_every_position(name, B, wdt):
    """Greedy generation to the full length (min_new_tokens = n bans EOS, so no row ends early) from prompts of 1-8 ids,
    B = 1 / 5 / 20 / 64 (single stream, the 2-8 tile, the 32-sequence tile, two passes of it): logits_all of rows 0,
    B // 2 and B - 1 at every position the launch computes (0 .. n - 2) against the float64 oracle of the ids the row
    ended with (bf16 weights: the oracle on the bf16-rounded weights, so the bound stays at fp32 round-off).  Bound:
    1e-4 * max|logit|, the widest existing decoder bound (test_gpu_decode.py::test_decode_deep_models_and_wide_windows).
    Greedy ids equal the oracle's argmax over the ids the draw may take (EOS is banned) wherever its top-2 gap exceeds
    1e-3 (test_gpu_generate.py::test_greedy_generate_matches_oracle)."""
    from progen_b200.decode import BatchDecoder
    kw, cfg, params = _model(name)
    n = cfg['seq_len']
    rng = np.random.default_rng(B)
    prompts = _prompts(rng, rng.integers(1, 9, B))
    dec = BatchDecoder(cfg, params, batch=B, weights_dtype=torch.bfloat16 if wdt == 'bf16' else torch.float32,
                       keep_logits=True)
    res = dec.generate(prompts, temperature=0.0, min_new_tokens=n)
    rows = sorted({0, B // 2, B - 1})
    got = dec.logits_all[rows, :n - 1].double()          # positions 0 .. n-2: the last one draws seq[n - 1]
    del dec
    assert (res['end'] == n).all()
    ids = res['ids'][rows]
    ref_params = _model(name, rounded=wdt == 'bf16')[2]
    ref = _oracle(ref_params, ids, cfg)[:, :n - 1]
    err, scale = _maxabs(got - ref), max(1.0, _maxabs(ref))
    e32 = _maxabs(_oracle(ref_params, ids, cfg, torch.float32)[:, :n - 1].double() - ref)
    worst_pos = int((got - ref).abs().amax(dim=(0, 2)).argmax())
    _report(case=f'decode_{name}_B{B}_{wdt}', err=err, bound=1e-4 * scale, rel=err / scale, fp32_oracle_err=e32,
            worst_position=worst_pos)
    assert err < 1e-4 * scale, (err, scale, e32)
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
    _report(case=f'decode_{name}_B{B}_{wdt}_greedy', ids_checked=checked, of=sum(n - int(res['start'][b]) for b in rows))
    assert checked > len(rows) * (n // 4)


# ------------------------------------------------------------------------------------------------ forward prefill
def _cache_views(ca, cb, key, R, n, h, dh, P):
    """the prompt part of cache `key` of both decoders as [R, ...] views"""
    x, y = ca[key], cb[key]
    if key in ('kcache', 'vcache'):
        return x.view(R, h, n, dh)[:, :, :P], y.view(R, h, n, dh)[:, :, :P]
    if key == 'gn_hist':
        return x[:, :P], y[:, :P]
    return x[:, P & 1], y[:, P & 1]                      # the token-shift slot the kernel reads at position P


def _check_caches(a, b, cfg, R, P, tol, case):
    n, h, dh = cfg['seq_len'], cfg['heads'], cfg['dim_head']
    worst = {}
    for i, (ca, cb) in enumerate(zip(a.caches, b.caches)):
        for key in ca:
            x, y = _cache_views(ca, cb, key, R, n, h, dh, P)
            for r in range(R):
                scale = _maxabs(x[r])
                assert scale > 0, (i, key, r)
                rel = _maxabs(x[r] - y[r]) / scale
                worst[key] = max(worst.get(key, 0.0), rel)
                assert rel <= tol, (i, key, r, rel, tol)
    _report(case=case, bound=tol, **{f'{k}_rel': v for k, v in worst.items()})
    assert set(worst) == {'kcache', 'vcache', 'shift1', 'shift2', 'gn_hist'}


PREFILL = [(name, mp, at) for name in NAMES for mp in (False, True) for at in ('half', 'end')]


@pytest.mark.parametrize('name,mp,at', PREFILL)
def test_forward_prefill(name, mp, at):
    """Prompts of P = n/2 - 3 and n - 66 ids; three rows, rows 0 and 2 share one forward row.  Every layer's K / V rows,
    token-shift slot and SGU gate history at positions < P against the decoder's own prefill of the same prompts, per row:
    1e-5 of the row's max (fp32 model) or 5e-2 (mixed precision: bf16 activations in the forward)
    (test_gpu_generate_prefill.py::test_fp32_caches_match_the_decode_prefill, ::test_scatter_at_1_and_24_rows).  First
    drawn logits: fp32, within 1e-5 * max|logit| of the decoder's after its own prefill (test_fp32_caches_match_the_decode_
    prefill); mixed precision, within 2x of `.apply`'s error against float64
    (::test_bf16_first_draw_logits_within_the_forward_error)."""
    kw, cfg, params = _model(name)
    n = cfg['seq_len']
    P = n // 2 - 3 if at == 'half' else n - 66
    p = _prompts(np.random.default_rng(P), [P, P])
    prompts = [p[0], p[1], p[0]]
    model, a, b = _both(kw, cfg, params, prompts, mp)
    case = f'prefill_{name}_mp{int(mp)}_P{P}'
    _check_caches(a, b, cfg, 3, P, 5e-2 if mp else 1e-5, case)
    la, lb = a.logits_all[:, P].double(), b.logits_all[:, P].double()
    if not mp:
        err, scale = _maxabs(la - lb), max(1.0, _maxabs(la))
        _report(case=case + '_first_draw', err=err, bound=1e-5 * scale)
        assert err <= 1e-5 * scale
        return
    del a
    rows = np.zeros((2, n), np.int64)
    for r in range(2):
        rows[r, 1:1 + P] = p[r]
    applied = model.apply(params, None, rows)[:, P].double()
    ref = _oracle(params, rows, cfg)[:, P]
    for r in range(2):
        e_apply, e_prefill = _maxabs(applied[r] - ref[r]), _maxabs(lb[r] - ref[r])
        _report(case=case + f'_first_draw_row{r}', err=e_prefill, bound=2 * e_apply)
        assert e_prefill <= 2 * e_apply, (r, e_prefill, e_apply)


@pytest.mark.parametrize('mp', [False, True])
def test_forward_prefill_scatter_24_rows(mp):
    """Config 4: 8 distinct prompts of n/2 - 3 ids scattered into 24 decoder rows (the 32-sequence tile); every row's caches
    against the decoder's own prefill with the bounds of test_gpu_generate_prefill.py::test_scatter_at_1_and_24_rows"""
    kw, cfg, params = _model('cfg4')
    P = cfg['seq_len'] // 2 - 3
    distinct = _prompts(np.random.default_rng(24), [P] * 8)
    prompts = [distinct[r % 8] for r in range(24)]
    _, a, b = _both(kw, cfg, params, prompts, mp)
    _check_caches(a, b, cfg, 24, P, 5e-2 if mp else 1e-5, f'prefill_scatter24_cfg4_mp{int(mp)}')


# ------------------------------------------------------------------------------------------------ score and embed
@pytest.mark.parametrize('name', NAMES)
@pytest.mark.parametrize('mp', [False, True])
def test_score_and_embed(name, mp):
    """Three rows of the config's length, row 1 ending early (EOS + padding).
      * `score`'s token log-probabilities and log-likelihoods are bitwise progen_token_logprob of `.apply`'s logits
        (test_gpu_score.py::test_score_is_the_apply_forward): the inference set's shared scratch and in-place residual at
        these layer sizes compute what the training forward does;
      * fp32: `.apply`'s logits within 1e-5 * max|logit| of float64 (test_gpu_model.py::test_fp32_apply_matches_reference_
        golden), -ll / count within 1e-5 of the float64 cross entropy (test_gpu_score.py::test_score_ragged_rows), the
        pooled embedding within 1e-5 * max of the pooled float64 final-LayerNorm output
        (::test_fp32_embedding_matches_oracle);
      * mixed precision: the embedding against float64 and against the bf16-operand emulation (the fp32 oracle with every
        GEMM / attention operand rounded to bf16), max < 5e-2 and mean < 1e-2 (::test_bf16_embedding)."""
    from progen_b200 import ProGen
    from oracle import progen_torch as T
    kw, cfg, params = _model(name)
    n = cfg['seq_len']
    rng = np.random.default_rng(n + int(mp))
    data = rng.integers(1, 256, (3, n + 1)).astype(np.uint16)
    data[1, 1 + int(rng.integers(n // 4, 3 * n // 4)):] = 0
    model = ProGen(**kw, mixed_precision=mp)
    logits = model.apply(params, None, data[:, :-1])
    lp, ll, cnt = _token_logprob(logits, data[:, 1:])
    sc = model.score(params, data, return_tokens=True, return_embeddings=True)
    np.testing.assert_array_equal(sc['token_logp'], lp)
    np.testing.assert_array_equal(sc['log_likelihood'], ll)
    np.testing.assert_array_equal(sc['num_tokens'], cnt.astype(np.int64))
    assert sc['num_tokens'][1] < n and (sc['num_tokens'][[0, 2]] == n).all()
    emb = sc['embedding'].astype(np.float64)
    case = f'score_{name}_mp{int(mp)}'
    ids = data[:, :-1].astype(np.int64)
    labels = torch.as_tensor(data[:, 1:].astype(np.int64), device='cuda')
    ref, hid = _oracle(params, ids, cfg, hidden=True)
    ref_emb = _pool(hid.cpu().numpy(), data)
    del hid
    if not mp:
        lg = logits.double()
        del logits
        scale = max(1.0, _maxabs(ref))
        e_logits = _maxabs(lg - ref)
        ce = -sc['log_likelihood'].astype(np.float64) / sc['num_tokens']
        ce_ref = T.cross_entropy(ref, labels).cpu().numpy()
        e_ce = float(np.abs(ce - ce_ref).max())
        e_emb, emb_scale = float(np.abs(emb - ref_emb).max()), max(1.0, float(np.abs(ref_emb).max()))
        r32, h32 = _oracle(params, ids, cfg, torch.float32, hidden=True)
        _report(case=case, logits_err=e_logits, logits_bound=1e-5 * scale, ce_err=e_ce, ce_bound=1e-5, ce=ce.tolist(),
                emb_err=e_emb, emb_bound=1e-5 * emb_scale, fp32_oracle_logits_err=_maxabs(r32.double() - ref),
                fp32_oracle_ce_err=float(np.abs(T.cross_entropy(r32, labels).double().cpu().numpy() - ce_ref).max()),
                fp32_oracle_emb_err=float(np.abs(_pool(h32.double().cpu().numpy(), data) - ref_emb).max()))
        assert e_logits < 1e-5 * scale, e_logits
        assert e_ce < 1e-5, (ce, ce_ref)
        assert e_emb < 1e-5 * emb_scale, e_emb
        return
    del logits, ref
    _, hid = _oracle(params, ids, cfg, torch.float32, T.bf16_round, hidden=True)
    emu_emb = _pool(hid.double().cpu().numpy(), data)
    err, e2 = np.abs(emb - ref_emb), np.abs(emb - emu_emb)
    _report(case=case, emb_err_max=float(err.max()), emb_err_mean=float(err.mean()), emu_err_max=float(e2.max()),
            emu_err_mean=float(e2.mean()), bound_max=5e-2, bound_mean=1e-2)
    assert err.max() < 5e-2 and err.mean() < 1e-2, (err.max(), err.mean())
    assert e2.max() < 5e-2 and e2.mean() < 1e-2, (e2.max(), e2.mean())
