"""Low-rank adapters on the GPU: the GEMM's tail operand pair against the physically concatenated operands (bitwise, both
backends), its refused combinations; the adapted model at initialisation is the base model bitwise; loss and adapter
gradients against float64 (the oracle's gradient wrt the merged weight W' = W + s A B, as dA = s dW' B^T and
dB = s A^T dW'); the Trainer against the oracle optimizer over the adapter tree with a bitwise frozen base, graph
replay and a preference step; merged parameters against the adapted forward; the train.py / generate.py / score.py
round trip."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import progen_ref as O
from oracle import progen_torch as T

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

BASE = dict(num_tokens=256, dim=128, seq_len=128, depth=2, window_size=64, heads=2, dim_head=64)
CONFIGS = {
    'glu': dict(BASE, global_mlp_depth=0),
    'gelu': dict(BASE, global_mlp_depth=0, ff_glu=False, shift_tokens=False),
    'sgu': dict(BASE, global_mlp_depth=1),
    'sgu_noshift': dict(BASE, global_mlp_depth=2, shift_tokens=False),
}


# ------------------------------------------------------------------------------------------------ GEMM tail
def _tail_case(L, backend, epi, M, N, K, K2, dtype, rng):
    """(kwargs of one GEMM, its epilogue operands) with A [M, K] K-major; B K-major for the backward kinds, MN-major else"""
    dev = 'cuda'
    mk = lambda *s: torch.tensor(rng.standard_normal(s).astype(np.float32), device=dev).to(dtype)
    b_mn = epi not in (L.EPI_GLU_BWD, L.EPI_GELU_BWD, L.EPI_STORE)
    A, A2 = mk(M, K), mk(M, K2)
    B, B2 = (mk(K, N), mk(K2, N)) if b_mn else (mk(N, K), mk(N, K2))
    kw = dict(epi=epi)
    out_dtype = L.F32 if epi == L.EPI_RESIDUAL else (L.BF16 if dtype == torch.bfloat16 else L.F32)
    act = lambda *s: torch.tensor(rng.standard_normal(s).astype(np.float32), device=dev).to(dtype)
    if epi == L.EPI_ROTARY:
        n, dh = 64, 64
        ang = np.arange(n)[:, None] * (1.0 / 10000 ** (np.arange(0, dh, 2) / dh))[None]
        kw.update(rot_sin=torch.tensor(np.sin(ang), dtype=torch.float32, device=dev),
                  rot_cos=torch.tensor(np.cos(ang), dtype=torch.float32, device=dev), seq_len=n, dim_head=dh)
    if epi in (L.EPI_RESIDUAL, L.EPI_GLU, L.EPI_GELU, L.EPI_STORE):
        kw['bias'] = torch.tensor(rng.standard_normal(N).astype(np.float32), device=dev)
    if epi == L.EPI_RESIDUAL:
        kw.update(aux=torch.tensor(rng.standard_normal((M, N)).astype(np.float32), device=dev), ldaux=N)
    if epi in (L.EPI_GLU_BWD, L.EPI_GELU_BWD):
        w = 2 * N if epi == L.EPI_GLU_BWD else N
        kw.update(aux=act(M, w), ldaux=w, colsum=torch.zeros(w, device=dev))
    out_cols = N // 2 if epi == L.EPI_GLU else 2 * N if epi == L.EPI_GLU_BWD else N
    if epi in (L.EPI_GLU, L.EPI_GELU):
        kw.update(out2=torch.empty(M, N, device=dev, dtype=dtype), ldo2=N)
    return A, A2, B, B2, b_mn, kw, out_cols, out_dtype


def _run_gemm(L, backend, M, N, K, A, lda, B, ldb, b_mn, kw, out_cols, out_dtype, dtype, **tail):
    out = torch.zeros(M, out_cols, device='cuda', dtype=torch.float32 if out_dtype == L.F32 else torch.bfloat16)
    kw = dict(kw)
    for k in ('colsum', 'out2'):
        if k in kw:
            kw[k] = torch.zeros_like(kw[k])
    L.gemm(M=M, N=N, K=K, A=A, lda=lda, B=B, ldb=ldb, b_mn=b_mn, out=out, ldo=out_cols, backend=backend,
           in_dtype=L.BF16 if dtype == torch.bfloat16 else L.F32, out_dtype=out_dtype, **kw, **tail)
    torch.cuda.synchronize()
    return [out] + [kw[k] for k in ('colsum', 'out2') if k in kw]


KINDS = ['STORE', 'ROTARY', 'RESIDUAL', 'GLU', 'GELU', 'GLU_BWD', 'GELU_BWD']


@pytest.mark.parametrize('kind', KINDS)
@pytest.mark.parametrize('backend', ['tc', 'simt'])
@pytest.mark.parametrize('K2', [16, 64])
def test_gemm_tail_equals_concatenated_operands(kind, backend, K2):
    """A B + A2 B2 with the tail is bitwise the GEMM on [A | A2 | 0] and [B ; B2 ; 0] (zero-padded to whole 64-column
    k-blocks, which is what the tail's TMA zero fill reads): the tail's k-blocks run last, in the same order"""
    from progen_b200 import lib as L
    L.require_device()
    epi = getattr(L, 'EPI_' + kind)
    dtype = torch.bfloat16 if backend == 'tc' else torch.float32
    be = L.BACKEND_TC if backend == 'tc' else L.BACKEND_SIMT
    M, N, K = 320, 384, 192
    rng = np.random.default_rng(1000 * KINDS.index(kind) + 10 * K2 + (backend == 'tc'))
    A, A2, B, B2, b_mn, kw, oc, od = _tail_case(L, be, epi, M, N, K, K2, dtype, rng)
    got = _run_gemm(L, be, M, N, K, A, K, B, N if b_mn else K, b_mn, kw, oc, od, dtype,
                    A2=A2, lda2=K2, B2=B2, ldb2=N if b_mn else K2, K2=K2)
    Kp = K + -(-K2 // 64) * 64
    Ac = torch.zeros(M, Kp, device='cuda', dtype=dtype)
    Ac[:, :K], Ac[:, K:K + K2] = A, A2
    if b_mn:
        Bc = torch.zeros(Kp, N, device='cuda', dtype=dtype)
        Bc[:K], Bc[K:K + K2] = B, B2
    else:
        Bc = torch.zeros(N, Kp, device='cuda', dtype=dtype)
        Bc[:, :K], Bc[:, K:K + K2] = B, B2
    want = _run_gemm(L, be, M, N, Kp, Ac, Kp, Bc, N if b_mn else Kp, b_mn, kw, oc, od, dtype)
    base = _run_gemm(L, be, M, N, K, A, K, B, N if b_mn else K, b_mn, kw, oc, od, dtype)
    for g, w in zip(got, want):
        if kind.endswith('_BWD') and g.dim() == 1:
            torch.testing.assert_close(g, w, rtol=1e-5, atol=1e-3)          # column sums: float atomics across tiles
        else:
            assert torch.equal(g, w), (kind, backend, (g.float() - w.float()).abs().max().item())
    assert not torch.equal(got[0], base[0])


@pytest.mark.parametrize('backend', ['tc', 'simt'])
def test_gemm_tail_refusals(backend):
    from progen_b200 import lib as L
    L.require_device()
    dtype = torch.bfloat16 if backend == 'tc' else torch.float32
    be = L.BACKEND_TC if backend == 'tc' else L.BACKEND_SIMT
    dt = L.BF16 if backend == 'tc' else L.F32
    M = N = K = 128
    x = torch.zeros(2 * M, K, device='cuda', dtype=dtype)
    t = torch.zeros(M, 16, device='cuda', dtype=dtype)
    out = torch.zeros(2 * M, N, device='cuda')
    tail = dict(A2=t, lda2=16, B2=t, ldb2=16, K2=16)
    for extra in (dict(split_k=2, epi=L.EPI_ACCUM, atomic=True), dict(causal=1), dict(batch=2, d_batch_rows=M),
                  dict(batch=2, batch_reduce=True, epi=L.EPI_ACCUM, atomic=True), dict(epi=L.EPI_ACCUM)):
        kw = dict(M=M, N=N, K=K, A=x, lda=K, B=x, ldb=K, out=out, ldo=N, backend=be, in_dtype=dt, out_dtype=L.F32)
        kw.update(extra)
        if not (backend == 'simt' and 'split_k' in extra):     # the CUDA-core GEMM has no split-K at all
            L.gemm(**kw)                                       # valid without the tail
        with pytest.raises(L.ProgenError):
            L.gemm(**kw, **tail)


# ------------------------------------------------------------------------------------------------ model
def _setup(name, mp, rank=16, alpha=32.0, seed=0, B=2):
    from progen_b200 import ProGen
    kw = CONFIGS[name]
    cfg = O.make_config(**kw)
    params = O.randomize_params(O.init_params(cfg, 3 + seed), 4 + seed)
    model = ProGen(**kw, mixed_precision=mp)
    ad = model.init_adapters(seed, rank, alpha=alpha)
    rng = np.random.default_rng(50 + seed)
    for v in ad.values():
        v['lora_b'] = (rng.standard_normal(v['lora_b'].shape) * 0.3 * v['lora_b'].shape[0] ** -0.5).astype(np.float32)
    data = rng.integers(0, 256, (B, kw['seq_len'] + 1)).astype(np.uint16)
    data[0, kw['seq_len'] // 2:] = 0
    return model, cfg, params, ad, data


def _oracle_adapter_grads(params, ad, data, cfg, s):
    merged = {m: dict(v) for m, v in params.items()}
    for m, v in ad.items():
        merged[m]['w'] = params[m]['w'].astype(np.float64) + s * (v['lora_a'].astype(np.float64) @ v['lora_b'].astype(np.float64))
    loss, grads = T.loss_and_grads(merged, data, cfg)
    out = {m: {'lora_a': s * grads[m]['w'] @ v['lora_b'].astype(np.float64).T,
               'lora_b': s * v['lora_a'].astype(np.float64).T @ grads[m]['w']} for m, v in ad.items()}
    return loss, out


@pytest.mark.parametrize('mp', [False, True])
@pytest.mark.parametrize('name', ['glu', 'sgu'])
def test_initial_adapters_are_the_base_model_bitwise(name, mp):
    """B = 0: the logits are the base model's bitwise.  The loss is a sum of float atomics over rows (progen_ce_fwd_bwd),
    whose order varies from launch to launch, so it agrees to fp32 round-off only."""
    from progen_b200 import ProGen
    model, cfg, params, _, data = _setup(name, mp)
    ad = model.init_adapters(1, 16)
    base = ProGen(**CONFIGS[name], mixed_precision=mp)
    b_loss, _ = base.loss_and_grad(params, data)
    b_logits = base.engine.logits.clone()
    loss, grads = model.loss_and_grad(params, data, adapters=ad)
    assert torch.equal(model.engine.logits, b_logits)
    assert abs(loss - b_loss) <= 2e-6 * abs(b_loss), (loss, b_loss)
    assert set(grads) == set(ad) and all(np.isfinite(g).all() for v in grads.values() for g in v.values())


@pytest.mark.parametrize('name', sorted(CONFIGS))
def test_fp32_loss_and_adapter_grads_match_float64(name):
    model, cfg, params, ad, data = _setup(name, False, seed=1)
    o_loss, o_grads = _oracle_adapter_grads(params, ad, data, cfg, 2.0)
    loss, grads = model.loss_and_grad(params, data, adapters=ad, lora_alpha=32.0)
    assert abs(loss - o_loss) < 1e-5, (loss, o_loss)
    for m, d in o_grads.items():
        for k, g in d.items():
            scale = max(1e-8, np.abs(g).max())
            assert np.abs(grads[m][k] - g).max() < 2e-4 * scale + 1e-7, (m, k, np.abs(grads[m][k] - g).max(), scale)


@pytest.mark.parametrize('name', ['glu', 'gelu', 'sgu'])
def test_bf16_loss_and_adapter_grads_vs_float64(name):
    model, cfg, params, ad, data = _setup(name, True, seed=2)
    o_loss, o_grads = _oracle_adapter_grads(params, ad, data, cfg, 2.0)
    loss, grads = model.loss_and_grad(params, data, adapters=ad, lora_alpha=32.0)
    assert abs(loss - o_loss) < 3e-2, (loss, o_loss)
    for m, d in o_grads.items():
        for k, g in d.items():
            rel = np.linalg.norm(grads[m][k] - g) / max(1e-8, np.linalg.norm(g))
            assert rel < 0.12, (m, k, rel)


def test_bf16_adapter_grads_at_the_config2_stack():
    from progen_b200 import ProGen
    torch.set_num_threads(max(1, min(32, len(os.sched_getaffinity(0)))))
    kw = dict(num_tokens=256, dim=512, seq_len=1024, depth=12, heads=8, dim_head=64, window_size=256, global_mlp_depth=2)
    cfg = O.make_config(**kw)
    params = O.init_params(cfg, 21)
    model = ProGen(**kw, mixed_precision=True)
    ad = model.init_adapters(3, 16)
    rng = np.random.default_rng(4)
    for v in ad.values():
        v['lora_b'] = (rng.standard_normal(v['lora_b'].shape) * 0.05).astype(np.float32)
    data = rng.integers(1, 256, (1, 1025)).astype(np.uint16)
    o_loss, o_grads = _oracle_adapter_grads(params, ad, data, cfg, 1.0)
    loss, grads = model.loss_and_grad(params, data, adapters=ad)
    assert abs(loss - o_loss) < 3e-2, (loss, o_loss)
    worst = max(np.linalg.norm(grads[m][k] - g) / max(1e-8, np.linalg.norm(g)) for m, d in o_grads.items() for k, g in d.items())
    assert worst < 0.12, worst


@pytest.mark.parametrize('mp', [False, True])
def test_merged_apply_matches_the_adapted_forward(mp):
    model, cfg, params, ad, data = _setup('sgu', mp, seed=3)
    model.loss_and_grad(params, data, adapters=ad, lora_alpha=32.0)
    adapted = model.engine.logits.view(data.shape[0], -1, cfg['num_tokens']).clone()
    merged = model.merge_adapters(params, ad, lora_alpha=32.0)
    logits = model.apply(merged, None, data[:, :-1])
    tol = 5e-2 if mp else 1e-4
    assert float((logits - adapted).abs().max()) < tol * max(1.0, float(adapted.abs().max()))


def _train(mp, params, ad, batches, cuda_graph=False, every=4):
    from progen_b200 import ProGen
    model = ProGen(**CONFIGS['sgu'], mixed_precision=mp)
    tr = model.trainer(params, adapters=ad, lora_alpha=32.0, grad_accum_every=every, learning_rate=1e-2, cuda_graph=cuda_graph)
    base = tr.eng.params.clone()
    losses = [float(tr.step(b).item()) for b in batches]
    assert torch.equal(tr.eng.params, base), 'the base parameters changed'
    return tr, losses


@pytest.mark.parametrize('mp', [False, True])
def test_trainer_steps_match_oracle_optimizer_and_keep_the_base(mp):
    model, cfg, params, ad, _ = _setup('sgu', mp, seed=4)
    rng = np.random.default_rng(9)
    batches = [rng.integers(0, 256, (2, 129)).astype(np.uint16) for _ in range(8)]
    tr, losses = _train(mp, params, ad, batches)
    st = O.optim_init(ad, every=4)
    cur = ad
    for step, b in enumerate(batches):
        ref_loss, grads = _oracle_adapter_grads(params, cur, b, cfg, 2.0)
        cur, _ = O.optim_step(cur, {m: {k: v.astype(np.float32) for k, v in d.items()} for m, d in grads.items()}, st, lr=1e-2)
        assert abs(losses[step] - ref_loss) < (3e-2 if mp else 2e-5), (step, losses[step], ref_loss)
    got = tr.adapters()
    worst = max(float(np.abs(got[m][k] - v).max()) for m, d in cur.items() for k, v in d.items())
    assert worst < (5e-2 if mp else 2e-3), worst
    assert tr.params().keys() == params.keys()
    # the optimizer state covers the adapters and round-trips
    st2 = tr.optim_state()
    assert set(st2['mu']) == set(ad)
    tr.load_optim_state(st2)
    assert tr.optim_state()['count'] == 8


@pytest.mark.parametrize('mp', [False, True])
def test_graph_replay_matches_eager(mp):
    """until the first apply_every emit the replayed and eager steps see the same adapters, so their losses agree to the
    round-off of the loss's float atomics; the adapters then agree within the bounds of
    test_gpu_model.test_trainer_cuda_graph_replay_matches_eager (split-K gradients use float atomics as well)"""
    _, _, params, ad, _ = _setup('sgu', mp, seed=5)
    rng = np.random.default_rng(10)
    batches = [rng.integers(0, 256, (2, 129)).astype(np.uint16) for _ in range(7)]
    te, el = _train(mp, params, ad, batches)
    tg, gl = _train(mp, params, ad, batches, cuda_graph=True)
    assert tg._graph is not None
    np.testing.assert_allclose(gl[:4], el[:4], rtol=2e-6, atol=0)
    np.testing.assert_allclose(gl, el, rtol=0, atol=2e-2 if mp else 2e-5)
    a, b = te.adapters(), tg.adapters()
    worst = max(float(np.abs(a[m][k] - b[m][k]).max()) for m in a for k in a[m])
    assert worst < (5e-2 if mp else 2e-3), worst


def test_preference_step_with_adapters_matches_float64():
    """DPO on adapters: the policy is the adapted model, the frozen reference the base (its log-likelihoods from score).
    The loss, the adapter gradient (from the oracle's gradient wrt W' = W + s A B) and the adapters after one step of
    the oracle optimizer, with the bounds of test_gpu_preference's fp32 tests; the base stays bitwise."""
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from preference_oracle import preference_loss_and_grads
    model, cfg, params, ad, _ = _setup('glu', False, seed=6)
    rng = np.random.default_rng(11)
    c = rng.integers(1, 256, (2, 129)).astype(np.uint16)
    r = rng.integers(1, 256, (2, 129)).astype(np.uint16)
    sc = model.score(params, np.concatenate([c, r]))['log_likelihood']
    tr = model.trainer(params, adapters=ad, lora_alpha=32.0, grad_accum_every=1, learning_rate=1e-3)
    base = tr.eng.params.clone()
    loss = float(tr.preference_step(c, r, sc[:2], sc[2:], beta=0.1).item())
    grads = tr.lora.layout.unpack(tr.lora.grads)             # the optimizer reads the gradient and leaves it in place
    s = 2.0
    merged = {m: dict(v) for m, v in params.items()}
    for m, v in ad.items():
        merged[m]['w'] = params[m]['w'].astype(np.float64) + s * (v['lora_a'].astype(np.float64) @ v['lora_b'].astype(np.float64))
    o_loss, o_w, o_st = preference_loss_and_grads(merged, c, r, sc[:2], sc[2:], cfg, 0.1)
    assert np.ptp(o_st['margin']) > 1e-3, o_st['margin']
    assert abs(loss - o_loss) < 1e-5, (loss, o_loss)
    o_grads = {m: {'lora_a': s * o_w[m]['w'] @ v['lora_b'].astype(np.float64).T,
                   'lora_b': s * v['lora_a'].astype(np.float64).T @ o_w[m]['w']} for m, v in ad.items()}
    for m, d in o_grads.items():
        for k, g in d.items():
            scale = max(1e-8, np.abs(g).max())
            assert np.abs(grads[m][k] - g).max() < 2e-4 * scale + 1e-7, (m, k, np.abs(grads[m][k] - g).max(), scale)
    want, _ = O.optim_step(ad, {m: {k: v.astype(np.float32) for k, v in d.items()} for m, d in o_grads.items()},
                           O.optim_init(ad, every=1), lr=1e-3)
    got = tr.adapters()
    worst = max(float(np.abs(got[m][k] - v).max()) for m, d in want.items() for k, v in d.items())
    assert worst < 2e-3, worst
    assert torch.equal(tr.eng.params, base)


def test_lora_trainer_releases_the_base_gradient():
    """a LoRA trainer keeps no full-size base gradient; the full-gradient path allocates it again"""
    model, _, params, ad, data = _setup('glu', True, seed=7)
    tr = model.trainer(params, adapters=ad)
    assert model.engine.grads is None
    tr.step(data)
    assert model.engine.grads is None
    loss, grads = model.loss_and_grad(params, data)
    assert model.engine.grads is not None and np.isfinite(loss) and set(grads) == set(params)


def test_adapter_gradients_do_not_accumulate():
    """the backward pass scales the whole B gradient by s, so accumulating into an earlier one is refused"""
    from progen_b200 import lib as L
    model, _, params, ad, data = _setup('glu', False)
    model.loss_and_grad(params, data, adapters=ad)
    with pytest.raises(L.ProgenError, match='zero_grads'):
        model.engine.loss_and_grad(data, zero_grads=False)


@pytest.mark.parametrize('mp', [False, True])
def test_two_rank_lora_trainer_equals_single_process(mp):
    """2 ranks (tests/ddp_lora_worker.py) against one process on the same global batches, with the bounds of
    test_gpu_ddp for the loss and gradient; needs two GPUs"""
    import json
    if torch.cuda.device_count() < 2:
        pytest.skip('needs two GPUs')
    port = 29700 + os.getpid() % 1000
    env = dict(os.environ, DDP_TEST_MP='1' if mp else '0', NCCL_DEBUG='WARN')
    r = subprocess.run([sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node', '2', '--master-addr',
                        '127.0.0.1', '--master-port', str(port), os.path.join(ROOT, 'tests', 'ddp_lora_worker.py')],
                       capture_output=True, text=True, env=env, timeout=240)
    line = next((l for l in r.stdout.splitlines() if l.startswith('DDP_RESULT ')), None)
    assert line is not None, r.stdout[-2000:] + r.stderr[-4000:]
    res = json.loads(line[len('DDP_RESULT '):])
    for case, v in res.items():
        np.testing.assert_allclose(v['loss_ddp'], v['loss_single'], rtol=0, atol=2e-3 if mp else 1e-5, err_msg=case)
        assert v['grad_rel_l2'] < (1e-3 if mp else 1e-5), (case, v)
        assert v['adapter_rel_l2'] < (1e-2 if mp else 1e-4), (case, v)
    assert res['even_4_rows_graph']['graph'], 'the data-parallel LoRA step was not captured into a CUDA graph'


def test_cli_lora_train_resume_generate_score(tmp_path):
    """train a base for one step, then adapters on it for 3 steps and 2 more after a resume; generate.py and score.py
    load the adapter package"""
    import pickle
    cfg_dir = tmp_path / 'cfg'
    cfg_dir.mkdir()
    (cfg_dir / 'tiny.toml').write_text('num_tokens = 256\ndim = 128\ndepth = 2\ndim_head = 64\nheads = 2\n'
                                       'window_size = 64\nseq_len = 128\nglobal_mlp_depth = 1\n')
    seqs = tmp_path / 'seqs.txt'
    seqs.write_text('\n'.join('MKTAYIAKQRQISFVKSHFSRQ' * (1 + i % 3) for i in range(40)) + '\n')
    env = dict(os.environ, PYTHONPATH=ROOT)
    run = lambda *a: subprocess.run([sys.executable, *a], cwd=ROOT, env=env, check=True, capture_output=True, text=True)
    common = ['--text_file', str(seqs), '--batch_size', '2', '--grad_accum_every', '1', '--sample_every', '1000',
              '--validate_every', '1000', '--checkpoint_every', '1']
    base, ft = tmp_path / 'base', tmp_path / 'ft'
    run('train.py', '--config_path', str(cfg_dir), '--model_name', 'tiny', '--checkpoint_path', str(base), '--num_steps', '1', *common)
    out = run('train.py', '--checkpoint_path', str(ft), '--init_checkpoint', str(base), '--lora_rank', '16', '--num_steps', '3', *common)
    assert 'adapters: rank 16' in out.stdout, out.stdout
    pkgs = sorted(ft.glob('ckpt_*'))
    assert len(pkgs) >= 1
    pkg = pickle.load(open(pkgs[-1], 'rb'))
    assert 'params' not in pkg and pkg['lora'] == {'rank': 16, 'alpha': 16.0}
    assert os.path.isabs(pkg['base_checkpoint']) and pkg['num_params'] > 0
    out = run('train.py', '--checkpoint_path', str(ft), '--num_steps', '2', *common)
    assert f"starting from sequence {pkg['next_seq_index']}" in out.stdout, out.stdout
    run('generate.py', '--checkpoint_path', str(ft), '--prompt', 'MK', '--num_samples', '2', '--max_length', '32',
        '--output', str(tmp_path / 'gen.fasta'))
    run('score.py', '--checkpoint_path', str(ft), '--input', str(seqs), '--output', str(tmp_path / 'scores.tsv'))
    assert (tmp_path / 'scores.tsv').read_text().count('\n') >= 40
