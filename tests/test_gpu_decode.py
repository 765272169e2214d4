"""KV-cached decode (csrc/decode_persist.cu, progen_b200/decode.py::BatchDecoder) against the reference sampler: greedy
token ids must match the golden samples produced by the reference's own `utils.sample` (tests/golden/make_golden.py)
exactly, the per-position logits must match the oracle's full forward, the cached path must agree with the engine's full
re-forward sampler, and B sequences decoded in lock step must agree with each decoded alone."""
import numpy as np
import pytest
import torch

from golden_util import load_case, CASES

pytestmark = pytest.mark.gpu
TINY = [n for n in CASES if n != 'cfg1']


def test_persistent_stochastic_sampler_is_seeded_and_differs_from_greedy():
    from progen_b200.decode import BatchDecoder
    cfg, params, data, g = load_case('tiny_all_glu')
    dec = BatchDecoder(cfg, params, batch=1)
    a, _, _ = dec.sample(g['prime'], top_k=25, add_bos=True, greedy=False, seed=1)
    b, _, _ = dec.sample(g['prime'], top_k=25, add_bos=True, greedy=False, seed=1)
    c, _, _ = dec.sample(g['prime'], top_k=25, add_bos=True, greedy=True)
    np.testing.assert_array_equal(a, b)
    assert not np.array_equal(a, c)


def test_persistent_decode_equals_full_reforward_sampler_cfg1_size():
    """BASELINE config-5 shape (seq_len 1024, prime '[Tax=Mammalia] #', top_k=25, add_bos) on the config-1 model: the
    KV-cached path must reproduce the bug-compatible full re-forward sampler (utils.sample over ProGen.apply)."""
    from progen_b200 import ProGen
    from progen_b200.decode import BatchDecoder
    from progen_b200.data import encode_tokens
    from progen_b200.utils import sample
    cfg, params, data, g = load_case('cfg1')
    prime = np.array(encode_tokens('[Tax=Mammalia] #'), dtype=np.uint16)
    dec = BatchDecoder(cfg, params, batch=1)
    ids, gen, secs = dec.sample(prime, top_k=25, add_bos=True, greedy=True)
    model = ProGen(**CASES['cfg1'])
    ref = sample(0, model.apply, params, prime, cfg['seq_len'], top_k=25, add_bos=True, greedy=True)
    np.testing.assert_array_equal(ids, ref)
    assert gen >= cfg['seq_len'] - len(prime) - 1
    print(f'persistent decode: {gen} tokens in {secs * 1e3:.1f} ms = {gen / secs:.0f} tokens/s')


def test_persistent_bf16_weight_decode_runs_and_mostly_agrees():
    from progen_b200.decode import BatchDecoder
    cfg, params, data, g = load_case('tiny_all_glu')
    a, _, _ = BatchDecoder(cfg, params, batch=1).sample(g['prime'], top_k=25, add_bos=True, greedy=True)
    b, _, _ = BatchDecoder(cfg, params, batch=1, weights_dtype=torch.bfloat16).sample(g['prime'], top_k=25, add_bos=True,
                                                                                      greedy=True)
    assert a.shape == b.shape and (a[:len(g['prime']) + 2] == b[:len(g['prime']) + 2]).all()


@pytest.mark.parametrize('name', TINY)
@pytest.mark.parametrize('add_bos', [False, True])
def test_persistent_greedy_ids_match_reference_sampler(name, add_bos):
    from progen_b200.decode import BatchDecoder
    cfg, params, data, g = load_case(name)
    dec = BatchDecoder(cfg, params, batch=1, keep_logits=True)
    ids, gen, secs = dec.sample(g['prime'], top_k=25, add_bos=add_bos, greedy=True)
    np.testing.assert_array_equal(ids, g[f'sample_bos{int(add_bos)}'])
    assert gen > 0 and secs > 0


def test_persistent_logits_match_oracle_forward():
    from progen_b200.decode import BatchDecoder
    from oracle import progen_ref as O
    cfg, params, data, g = load_case('tiny_glu_sgu')
    dec = BatchDecoder(cfg, params, batch=1, keep_logits=True)
    dec.sample(g['prime'], top_k=25, add_bos=True, greedy=True)
    seq = dec.seq.cpu().numpy().astype(np.int64)[0]               # final ids BEFORE the post-hoc truncation
    ref = O.forward(params, np.clip(seq, 0, 255), cfg)            # out-of-range ids clamp like a jax gather
    got = dec.logits_all.cpu().numpy()[0]
    n = cfg['seq_len']
    assert np.abs(got[:n - 1] - ref[:n - 1]).max() < 2e-5 * max(1.0, np.abs(ref).max())


@pytest.mark.parametrize('B,wdt', [(33, 'bf16'), (20, 'bf16'), (40, 'f32')])
def test_batched_logits_match_oracle_forward(B, wdt):
    """B > 8 paths (bf16 weights: mma.sync with the activations split into three bf16 terms; fp32 weights: lane = sequence
    FMAs): every sequence's logits against the oracle's full forward of the sequence it ended with.  With bf16 weights the
    oracle runs on the bf16-rounded weights, so the bound stays at fp32 round-off."""
    import torch
    from progen_b200.decode import BatchDecoder
    from oracle import progen_ref as O
    cfg, params, data, g = load_case('tiny_glu_sgu')
    rng = np.random.default_rng(100 + B)
    primes = [rng.integers(1, 256, int(rng.integers(1, 9))).astype(np.int64) for _ in range(B)]
    dt = torch.bfloat16 if wdt == 'bf16' else torch.float32
    dec = BatchDecoder(cfg, params, batch=B, weights_dtype=dt, keep_logits=True)
    dec.sample(primes, top_k=25, add_bos=True, greedy=True)
    seqs = dec.seq.cpu().numpy().astype(np.int64)
    got = dec.logits_all.cpu().numpy()
    ref_params = params
    if wdt == 'bf16':
        rnd = lambda a: torch.tensor(np.asarray(a, np.float32)).bfloat16().float().numpy()
        ref_params = {k: {kk: (rnd(vv) if kk == 'w' else vv) for kk, vv in v.items()} for k, v in params.items()}
    n = cfg['seq_len']
    for b in (0, B // 2, B - 1):
        ref = O.forward(ref_params, np.clip(seqs[b], 0, 255), cfg)
        assert np.abs(got[b, :n - 1] - ref[:n - 1]).max() < 3e-5 * max(1.0, np.abs(ref).max()), b


@pytest.mark.parametrize('B,wdt', [(1, 'f32'), (1, 'bf16'), (5, 'f32'), (12, 'bf16'), (40, 'bf16'), (20, 'f32')])
def test_decode_wide_model_multiwave(B, wdt):
    """d = 1024 (config-3 width): a CTA's share of a GEMV phase no longer fits one wave of weight units (QKV 2 waves, FF-in 4),
    K = 1024 / 4096 inputs are staged in several chunks for B > 8, LayerNorm takes the two-pass path there.  Logits of every
    position against the oracle's forward (bf16 weights: oracle on the rounded weights)."""
    import torch
    from progen_b200.decode import BatchDecoder
    from oracle import progen_ref as O
    cfg = O.make_config(num_tokens=256, dim=1024, seq_len=48, depth=2, window_size=16, global_mlp_depth=1, heads=16, dim_head=64)
    params = O.randomize_params(O.init_params(cfg, 11), 12)
    rng = np.random.default_rng(B)
    primes = [rng.integers(1, 256, int(rng.integers(1, 6))).astype(np.int64) for _ in range(B)]
    dt = torch.bfloat16 if wdt == 'bf16' else torch.float32
    dec = BatchDecoder(cfg, params, batch=B, weights_dtype=dt, keep_logits=True)
    dec.sample(primes if B > 1 else primes[0], top_k=25, add_bos=True, greedy=True)
    seqs = dec.seq.cpu().numpy().astype(np.int64)
    got = dec.logits_all.cpu().numpy()
    ref_params = params
    if wdt == 'bf16':
        rnd = lambda a: torch.tensor(np.asarray(a, np.float32)).bfloat16().float().numpy()
        ref_params = {k: {kk: (rnd(vv) if kk == 'w' else vv) for kk, vv in v.items()} for k, v in params.items()}
    n = cfg['seq_len']
    for b in sorted({0, B // 2, B - 1}):
        ref = O.forward(ref_params, np.clip(seqs[b], 0, 255), cfg)
        assert np.abs(got[b, :n - 1] - ref[:n - 1]).max() < 5e-5 * max(1.0, np.abs(ref).max()), b


@pytest.mark.parametrize('B,wdt,depth,window', [(1, 'f32', 26, 16), (1, 'bf16', 4, 512), (12, 'bf16', 4, 512), (3, 'f32', 26, 16)])
def test_decode_deep_models_and_wide_windows(B, wdt, depth, window):
    """depth 26: the single-stream unit tables no longer fit shared memory (the kernel computes the offsets instead);
    window 512 at seq_len 1024: up to 32 key slices of 32 (single stream) / 64 of 16 (batched) per (sequence, head)"""
    import torch
    from progen_b200.decode import BatchDecoder
    from oracle import progen_ref as O
    n = 1024 if window == 512 else 48
    cfg = O.make_config(num_tokens=256, dim=64, seq_len=n, depth=depth, window_size=window, global_mlp_depth=2, heads=2, dim_head=32)
    params = O.randomize_params(O.init_params(cfg, 21), 22)
    rng = np.random.default_rng(B + depth)
    primes = [rng.integers(1, 256, int(rng.integers(1, 6))).astype(np.int64) for _ in range(B)]
    dt = torch.bfloat16 if wdt == 'bf16' else torch.float32
    dec = BatchDecoder(cfg, params, batch=B, weights_dtype=dt, keep_logits=True)
    dec.sample(primes if B > 1 else primes[0], top_k=25, add_bos=True, greedy=True)
    seqs = dec.seq.cpu().numpy().astype(np.int64)
    got = dec.logits_all.cpu().numpy()
    ref_params = params
    if wdt == 'bf16':
        rnd = lambda a: torch.tensor(np.asarray(a, np.float32)).bfloat16().float().numpy()
        ref_params = {k: {kk: (rnd(vv) if kk == 'w' else vv) for kk, vv in v.items()} for k, v in params.items()}
    for b in sorted({0, B - 1}):
        ref = O.forward(ref_params, np.clip(seqs[b], 0, 255), cfg)
        assert np.abs(got[b, :n - 1] - ref[:n - 1]).max() < 1e-4 * max(1.0, np.abs(ref).max()), b


@pytest.mark.parametrize('B', [12, 40])
def test_batched_tensor_pipe_path_at_model_width_512(B):
    """config-1 width (d = 512, K = 512 / 2048 phases: bulk-copied LayerNorm rows, multi-chunk FF-out, 1-4 n-tiles per CTA) with
    bf16 weights: B sequences on the tensor-pipe path == the same primes decoded alone (single-stream fp32 FMA path, same bf16
    weights) — greedy ids equal, logits within fp32 round-off"""
    import torch
    from progen_b200.decode import BatchDecoder
    cfg, params, data, g = load_case('cfg1')
    rng = np.random.default_rng(B)
    primes = [rng.integers(1, 256, int(rng.integers(2, 12))).astype(np.int64) for _ in range(B)]
    many = BatchDecoder(cfg, params, batch=B, weights_dtype=torch.bfloat16, keep_logits=True)
    ids, gen, secs = many.sample(primes, top_k=25, add_bos=True, greedy=True)
    got = many.logits_all.cpu().numpy()
    one = BatchDecoder(cfg, params, batch=1, weights_dtype=torch.bfloat16, keep_logits=True)
    n = cfg['seq_len']
    for b in (0, B // 3, B - 1):
        ref_ids, _, _ = one.sample(primes[b], top_k=25, add_bos=True, greedy=True)
        ref = one.logits_all.cpu().numpy()[0]
        np.testing.assert_array_equal(ids[b], ref_ids)
        assert np.abs(got[b, :n - 1] - ref[:n - 1]).max() < 5e-5 * max(1.0, np.abs(ref).max()), b


@pytest.mark.parametrize('B', [3, 8, 33])
def test_batched_decode_equals_single_stream(B):
    """B primes of different lengths decoded in lock step == each prime decoded alone (greedy, bit-equal ids)"""
    from progen_b200.decode import BatchDecoder
    cfg, params, data, g = load_case('tiny_glu_sgu')
    rng = np.random.default_rng(B)
    primes = [rng.integers(1, 256, int(rng.integers(1, 9))).astype(np.int64) for _ in range(B)]
    primes[0] = np.asarray(g['prime']).astype(np.int64)
    batch, gen, secs = BatchDecoder(cfg, params, batch=B).sample(primes, top_k=25, add_bos=True, greedy=True)
    single = BatchDecoder(cfg, params, batch=1)
    for b in range(B):
        one, _, _ = single.sample(primes[b], top_k=25, add_bos=True, greedy=True)
        np.testing.assert_array_equal(batch[b], one)
    np.testing.assert_array_equal(batch[0], g['sample_bos1'])


def test_gumbel_topk_sampler_distribution_chi_square():
    """Distribution-level parity of the stochastic sampler (SURVEY 8(f)3): the device sampler draws
    argmax(filtered logits + gumbel) with the reference's quirky top-k filter (utils.py:97-100,121-125: keeps the k-1
    logits above the k-th, sets the rest to 0.0 and removes their noise).  For the FIRST sampled position of many
    independently seeded runs the empirical distribution must match the probabilities that filter implies:
    softmax over {kept logits} U {one atom of value 0.0 standing for all filtered entries (they tie at 0, argmax takes
    the first)}.  Chi-square goodness of fit at the 0.1 % level."""
    from scipy import stats
    from progen_b200.decode import BatchDecoder
    from oracle import progen_ref as O
    cfg, params, data, g = load_case('tiny_all_glu')
    prime = np.asarray(g['prime']).astype(np.int64)
    B, K, runs = 64, 25, 12
    dec = BatchDecoder(cfg, params, batch=B)
    P_ = len(prime)
    counts = np.zeros(cfg['num_tokens'], np.int64)
    for r_ in range(runs):
        ids, _, _ = dec.sample([prime] * B, top_k=K, add_bos=False, greedy=False, seed=1000 + r_)
        # without add_bos position P_ starts at 0, so seq[P_] IS the sampled id of the first draw
        first = dec.seq.cpu().numpy()[:, P_]
        counts += np.bincount(first, minlength=cfg['num_tokens'])
    seq = np.pad(prime, (0, cfg['seq_len'] - P_))
    logits = O.forward(params, seq, cfg)[P_ - 1].astype(np.float64)
    kth = np.sort(logits)[-K]
    keep = logits > kth
    z = np.where(keep, logits, 0.0)
    first_filtered = int(np.argmin(keep))                 # all filtered entries tie at 0.0 (no noise): argmax returns the first
    atoms = np.zeros_like(z)
    atoms[keep] = np.exp(z[keep])
    atoms[first_filtered] = 1.0                            # exp(0): Gumbel-max against a noiseless 0 is NOT a softmax atom ...
    # ... a noiseless entry wins iff every kept (logit + gumbel) < 0: P = prod_i exp(-exp(l_i)) = exp(-sum_i exp(l_i))
    S = np.exp(logits[keep]).sum()
    p0 = np.exp(-S)
    probs = np.zeros_like(z)
    probs[keep] = (1.0 - p0) * np.exp(logits[keep]) / S    # given some kept entry is > 0 ... (exactly: max-stability of Gumbel)
    probs[first_filtered] = p0
    # exact law: M = max_i(l_i + G_i) ~ Gumbel(log S); argmax independent of M; P(M < 0) = exp(-S)
    n_draws = counts.sum()
    assert n_draws == B * runs
    assert counts[~keep & (np.arange(len(keep)) != first_filtered)].sum() == 0
    exp_counts = probs * n_draws
    big = exp_counts >= 5
    obs = np.append(counts[big], counts[~big].sum())
    exp_ = np.append(exp_counts[big], exp_counts[~big].sum())
    if exp_[-1] == 0:
        obs, exp_ = obs[:-1], exp_[:-1]
    chi2 = ((obs - exp_) ** 2 / exp_).sum()
    pval = 1.0 - stats.chi2.cdf(chi2, len(obs) - 1)
    assert pval > 1e-3, (chi2, len(obs), pval)
