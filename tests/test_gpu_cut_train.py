"""The training step cut to its rows' counted length (DESIGN.md §3.10) against the full-length step.

What must hold: positions < L of the forward and the gradients into activations are bitwise the full step's; the
token-dimension reductions (weight gradients, column sums, LayerNorm scales, embedding and SGU gradients) only sum in
another order.  Bound for those: re-ordering a float32 sum of T terms moves it by about sqrt(T) * 2^-24 times the
terms' magnitude (at most T * 2^-24 * sum|terms|); with T <= 1536 token rows that is ~1e-6 of a leaf's largest entry,
so 1e-4 of it (fp32) and 1e-3 (bf16 operands, the same fp32 accumulation; the graph tests' run-to-run split-K
differences are of this size) leave a wide margin while still catching a wrong row.  Gradient entries of positions
>= L are exactly zero in both steps."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from test_gpu_elementwise import attn_ref

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BASE = dict(num_tokens=256, dim=128, seq_len=512, depth=2, window_size=256, heads=2, dim_head=64)
CONFIGS = {
    'sgu': dict(BASE, global_mlp_depth=1),
    'gelu': dict(BASE, global_mlp_depth=0, ff_glu=False),
    'noshift': dict(BASE, global_mlp_depth=1, shift_tokens=False),
    'wide_window': dict(BASE, global_mlp_depth=1, window_size=512),       # L = 128 or 384 < w
}
GRAD_TOL = {False: 1e-4, True: 1e-3}


def _rows(B, n, lens, seed):
    """(B, n+1) rows whose labels end after lens[i] residues (counted length lens[i] + 1)"""
    r = np.random.default_rng(seed).integers(1, 256, (B, n + 1)).astype(np.uint16)
    for i, k in enumerate(lens):
        r[i, 1 + k:] = 0
    return r


# ---------------------------------------------------------------------------------------------------- 1. kernels
ATTN_CASES = [(2, 512, 512, 2, 384), (2, 512, 256, 2, 384), (2, 512, 256, 2, 320), (1, 1024, 512, 3, 128),
              (2, 512, 256, 2, 512)]


def _attn_bwd(L, tc, qkv, out, dout, lse, B, n, w, h, cut, rot):
    dqkv = torch.full_like(qkv, float('nan'))
    delta = torch.full((B * n, h), float('nan'), device='cuda')
    lib = L.load()
    if tc:
        fn = lib.progen_local_attn_bwd_cut_tc if cut else lib.progen_local_attn_bwd_tc
        sin, cos = rot if rot else (None, None)
        L.check(fn(qkv.data_ptr(), out.data_ptr(), dout.data_ptr(), lse.data_ptr(), dqkv.data_ptr(), delta.data_ptr(),
                   L.ptr(sin), L.ptr(cos), B, n, w, h, 64, L.stream()))
    else:
        fn = lib.progen_local_attn_bwd_cut_simt if cut else lib.progen_local_attn_bwd_simt
        L.check(fn(qkv.data_ptr(), out.data_ptr(), dout.data_ptr(), lse.data_ptr(), dqkv.data_ptr(), delta.data_ptr(),
                   L.dt(qkv), B, n, w, h, 64, L.stream()))
    torch.cuda.synchronize()
    return dqkv


@pytest.mark.parametrize('kernel', ['tc', 'simt_bf16', 'simt_f32'])
@pytest.mark.parametrize('case', ATTN_CASES)
def test_cut_attention_backward(kernel, case):
    """the cut entry point's rows are bitwise the whole-window entry point's at full length with dout zero from L on,
    equal to it at L = n, and within the attention tests' bound of float64 autograd"""
    from progen_b200 import lib as L
    from gemm_cases import rotary_tables
    B, n, w, h, Lc = case
    tc = kernel == 'tc'
    dt = torch.float32 if kernel == 'simt_f32' else torch.bfloat16
    I, T = h * 64, B * n
    g = torch.Generator(device='cuda').manual_seed(n + w + Lc)
    qkv = (torch.randn(T, 3 * I, generator=g, device='cuda') * 1.5).to(dt)
    out = torch.empty(T, I, device='cuda', dtype=dt)
    lse = torch.empty(T, h, device='cuda')
    if tc:
        L.check(L.load().progen_local_attn_fwd_tc(qkv.data_ptr(), out.data_ptr(), lse.data_ptr(), B, n, w, h, 64, L.stream()))
    else:
        L.check(L.load().progen_local_attn_fwd_simt(qkv.data_ptr(), out.data_ptr(), lse.data_ptr(), L.dt(qkv), B, n, w, h, 64,
                                                    L.stream()))
    dout = torch.randn(T, I, generator=g, device='cuda').to(dt)
    dout.view(B, n, I)[:, Lc:] = 0
    cut = lambda t: t.view(B, n, -1)[:, :Lc].reshape(B * Lc, -1).contiguous()
    for rot in ([False, True] if tc else [False]):
        tabs = rotary_tables(n, 64, 'cuda') if rot else None
        full = _attn_bwd(L, tc, qkv, out, dout, lse, B, n, w, h, False, tabs)
        got = _attn_bwd(L, tc, cut(qkv), cut(out), cut(dout), cut(lse), B, Lc, w, h, True, tabs)
        assert torch.equal(got.view(B, Lc, -1), full.view(B, n, -1)[:, :Lc]), (kernel, case, rot)
        if Lc == n:
            assert torch.equal(got, full)
    qd = qkv.double().requires_grad_(True)
    attn_ref(qd, B, n, w, h, 64).backward(dout.double())
    ref = qd.grad.view(B, n, -1)[:, :Lc].reshape(B * Lc, -1)
    got = _attn_bwd(L, tc, cut(qkv), cut(out), cut(dout), cut(lse), B, Lc, w, h, True, None).double()
    tol = 4e-2 if dt == torch.bfloat16 else 1e-4
    assert (got - ref).abs().max().item() < tol * max(1.0, ref.abs().max().item())


# ---------------------------------------------------------------------------------------------------- 2. LM step
def _zero_beyond(tree, Lc, n):
    """the entries of positions >= Lc: spatial_weights rows and columns, spatial_biases rows"""
    out = []
    for m, d in tree.items():
        for k, v in d.items():
            if k == 'spatial_weights':
                out += [v[Lc:, :], v[:, Lc:]]
            elif k == 'spatial_biases':
                out.append(v[Lc:])
    return out


def _close_trees(a, b, tol):
    for m, d in b.items():
        for k, r in d.items():
            scale = max(1e-8, float(np.abs(r).max()))
            err = float(np.abs(a[m][k] - r).max())
            assert err <= tol * scale + 1e-7, (m, k, err, scale)


def _trainer(name, mp, params, every=2, **kw):
    from progen_b200 import ProGen
    return ProGen(**CONFIGS[name], mixed_precision=mp).trainer(params, learning_rate=1e-2, grad_accum_every=every, **kw)


@pytest.mark.parametrize('mp', [False, True])
@pytest.mark.parametrize('name', list(CONFIGS))
def test_lm_step_at_the_cut(name, mp):
    from oracle import progen_ref as O
    from oracle import progen_torch as T
    from progen_b200 import ProGen
    cfg = O.make_config(**CONFIGS[name])
    n = cfg['seq_len']
    params = O.randomize_params(O.init_params(cfg, 3), 4)
    lens = [100, 20, 60] if name == 'wide_window' else [300, 120, 350]
    rows = _rows(3, n, lens, 5)
    Lc = 128 if name == 'wide_window' else 384
    grads = {}
    for length in (None, n):
        tr = _trainer(name, mp, params)
        loss = float(tr.step(rows, length=length).item())
        grads[length] = (loss, tr.layout.unpack(tr.G))
    (lc, gc), (lf, gf) = grads[None], grads[n]
    assert abs(lc - lf) <= 1e-6 * max(1.0, abs(lf)), (lc, lf)
    _close_trees(gc, gf, GRAD_TOL[mp])
    for z in _zero_beyond(gc, Lc, n) + _zero_beyond(gf, Lc, n):
        assert not z.any()
    # loss_and_grad runs at the cut as well: the float64 oracle, with test_gpu_model's bounds
    loss, g = ProGen(**CONFIGS[name], mixed_precision=mp).loss_and_grad(params, rows)
    ref_loss, ref = T.loss_and_grads(params, rows, cfg)
    assert abs(loss - ref_loss) < (3e-2 if mp else 1e-5), (loss, ref_loss)
    for m, d in ref.items():
        for k, r in d.items():
            scale = max(1e-8, np.abs(r).max())
            err = np.abs(g[m][k] - r).max()
            assert err < (0.12 * scale if mp else 2e-4 * scale + 1e-7), (m, k, err, scale)


# ---------------------------------------------------------------------------------------------------- 3. preference
@pytest.mark.parametrize('mp', [False, True])
def test_preference_step_at_the_cut(mp):
    from oracle import progen_ref as O
    cfg = O.make_config(**CONFIGS['sgu'])
    n = cfg['seq_len']
    params = O.randomize_params(O.init_params(cfg, 6), 7)
    c, r = _rows(2, n, [200, 40], 8), _rows(2, n, [90, 260], 9)
    rc, rr = np.array([-500.0, -100.0], np.float32), np.array([-200.0, -600.0], np.float32)
    out = {}
    for length in (None, n):
        tr = _trainer('sgu', mp, params)
        loss = float(tr.preference_step(c, r, rc, rr, beta=0.1, length=length).item())
        out[length] = (loss, tr.preference_stats(), tr.layout.unpack(tr.G))
    (lc, sc, gc), (lf, sf, gf) = out[None], out[n]
    assert lc == lf, (lc, lf)
    for k in sf:
        np.testing.assert_array_equal(sc[k], sf[k], err_msg=k)
    _close_trees(gc, gf, GRAD_TOL[mp])
    for z in _zero_beyond(gc, 384, n):
        assert not z.any()


# ---------------------------------------------------------------------------------------------------- 4./5. adapters
@pytest.mark.parametrize('mp', [False, True])
@pytest.mark.parametrize('task', ['regression', 'classification'])
def test_property_step_at_the_cut(task, mp):
    from oracle import progen_ref as O
    from progen_b200 import ProGen
    from progen_b200.lora import HEAD
    cfg = O.make_config(**CONFIGS['sgu'])
    n = cfg['seq_len']
    params = O.randomize_params(O.init_params(cfg, 10), 11)
    model = ProGen(**CONFIGS['sgu'], mixed_precision=mp)
    ad = model.init_adapters(1, 16)
    for v in ad.values():
        v['lora_b'] = (0.05 * np.random.default_rng(2).standard_normal(v['lora_b'].shape)).astype(np.float32)
    C = 3
    head = model.init_head(2, C)
    rows = _rows(3, n, [250, 30, 100], 12)
    rng = np.random.default_rng(13)
    y = rng.standard_normal((3, C)).astype(np.float32) if task == 'regression' else rng.integers(0, C, 3)
    out = {}
    for length in (None, n):
        tr = _trainer('sgu', mp, params, adapters=ad, head=head, task=task, lora_alpha=32.0)
        loss = float(tr.property_step(rows, y, length=length).item())
        ad_g, head_g = tr.lora.split(tr.layout.unpack(tr.G))
        out[length] = (loss, tr.property_stats(), ad_g, head_g)
    (lc, sc, ac, hc), (lf, sf, af, hf) = out[None], out[n]
    assert lc == lf, (lc, lf)
    for k in sf:
        np.testing.assert_array_equal(sc[k], sf[k], err_msg=k)
    for k in ('w', 'b'):
        np.testing.assert_array_equal(hc[HEAD][k], hf[HEAD][k], err_msg=k)
    _close_trees(ac, af, GRAD_TOL[mp])


@pytest.mark.parametrize('mp', [False, True])
def test_lora_lm_step_at_the_cut(mp):
    from oracle import progen_ref as O
    from progen_b200 import ProGen
    cfg = O.make_config(**CONFIGS['sgu'])
    n = cfg['seq_len']
    params = O.randomize_params(O.init_params(cfg, 14), 15)
    ad = ProGen(**CONFIGS['sgu']).init_adapters(1, 16)
    for v in ad.values():
        v['lora_b'] = (0.05 * np.random.default_rng(3).standard_normal(v['lora_b'].shape)).astype(np.float32)
    rows = _rows(3, n, [300, 120, 350], 16)
    out = {}
    for length in (None, n):
        tr = _trainer('sgu', mp, params, adapters=ad, lora_alpha=32.0)
        loss = float(tr.step(rows, length=length).item())
        out[length] = (loss, tr.layout.unpack(tr.G))
    assert abs(out[None][0] - out[n][0]) <= 1e-6 * max(1.0, abs(out[n][0]))
    _close_trees(out[None][1], out[n][1], GRAD_TOL[mp])
    # steps of different lengths share one allocation of the adapter activations
    tr = _trainer('sgu', mp, params, adapters=ad, lora_alpha=32.0)
    tr.step(rows)
    epoch = tr.eng.alloc_epoch
    for lens in ([20, 30, 10], [300, 120, 350], [500, 1, 1], [200, 1, 1]):
        tr.step(_rows(3, n, lens, 17))
    assert tr.eng.alloc_epoch == epoch


# ---------------------------------------------------------------------------------------------------- 6. graphs
@pytest.mark.parametrize('mp', [False, True])
def test_graphs_per_length_replay_like_the_eager_loop(mp):
    from oracle import progen_ref as O
    cfg = O.make_config(**CONFIGS['sgu'])
    n = cfg['seq_len']
    params = O.randomize_params(O.init_params(cfg, 18), 19)
    lens = [[100, 20], [300, 200], [511, 5]] * 4                          # lengths 128, 384, n, cycling
    batches = [_rows(2, n, l, 20 + i) for i, l in enumerate(lens[:11])]
    runs = {}
    for graph in (False, True):
        tr = _trainer('sgu', mp, params, every=8, cuda_graph=graph)
        losses, mem = [], []
        for b in batches:
            losses.append(float(tr.step(b).item()))
            torch.cuda.synchronize()
            mem.append(torch.cuda.memory_allocated())
        runs[graph] = (tr, losses, mem)
    (te, el, _), (tg, gl, gmem) = runs[False], runs[True]
    # grad_accum_every=8: both loops see the same parameters for 8 steps, of which steps 7 and 8 replay; the loss sums
    # with float atomics, so it agrees to their round-off
    np.testing.assert_allclose(gl[:8], el[:8], rtol=1e-6, atol=0)
    np.testing.assert_allclose(gl, el, rtol=0, atol=2e-2 if mp else 2e-5)
    assert sorted(length for _, length in tg._graphs) == [128, 384, n]
    assert tg._graph_key == (2, 2) and tg._graph_length in (128, 384, n)
    assert tg.count == len(batches)
    # captures at steps 4, 5, 6 (the second eager step of each length); no capture grows the allocation
    assert gmem[3] == gmem[4] == gmem[5] == gmem[-1], gmem
    pe, pg = te.params(), tg.params()
    worst = max(float(np.abs(pg[m][k] - v).max()) for m, d in pe.items() for k, v in d.items())
    assert worst < (5e-2 if mp else 2e-3), worst


# ---------------------------------------------------------------------------------------------------- 7./8. evaluate, validation
@pytest.mark.parametrize('mp', [False, True])
def test_evaluate_and_length_validation(mp):
    from oracle import progen_ref as O
    from progen_b200 import lib as L
    cfg = O.make_config(**CONFIGS['gelu'])
    n = cfg['seq_len']
    params = O.randomize_params(O.init_params(cfg, 21), 22)
    rows = _rows(3, n, [300, 120, 350], 23)
    tr = _trainer('gelu', mp, params)
    a = float(tr.evaluate(rows).item())
    b = float(tr.evaluate(rows, length=n).item())
    assert abs(a - b) <= 1e-6 * max(1.0, abs(b)), (a, b)
    tr.step(rows)
    state = [t.clone() for t in (tr.P, tr.m, tr.v, tr.acc, tr.eng.loss)]
    count = tr.count
    for bad in (100, 256, n + 128, 2 * n):
        for call in (lambda: tr.step(rows, length=bad), lambda: tr.evaluate(rows, length=bad),
                     lambda: tr.preference_step(rows[:1], rows[1:2], [0.0], [0.0], length=bad)):
            with pytest.raises(L.ProgenError, match='384|length must be'):
                call()
    assert tr.count == count
    assert all(torch.equal(x, y) for x, y in zip(state, (tr.P, tr.m, tr.v, tr.acc, tr.eng.loss)))


# ---------------------------------------------------------------------------------------------------- 9. two ranks
def test_two_rank_cut_step_equals_single_process(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip('needs 2 GPUs')
    import json
    out = tmp_path / 'ddp_cut.json'
    cmd = [sys.executable, '-m', 'torch.distributed.run', '--nproc_per_node', '2', '--master_port', '29531',
           os.path.join(ROOT, 'tests', 'ddp_cut_worker.py'), str(out)]
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    res = json.loads(out.read_text())
    for mp, v in res.items():
        assert v['length'] == 384 and v['shard_lengths'][0] != v['shard_lengths'][1], v
        assert abs(v['loss_ddp'] - v['loss_single']) < (2e-3 if mp == 'True' else 1e-5), v
        assert v['grad_rel_l2'] < (1e-3 if mp == 'True' else 1e-5), v


# ---------------------------------------------------------------------------------------------------- 10. CLI
def _train(tmp_path, ckpt, *extra):
    cmd = [sys.executable, os.path.join(ROOT, 'train.py'), '--text_file', str(tmp_path / 'seqs.txt'), '--checkpoint_path',
           str(ckpt), '--config_path', str(tmp_path), '--model_name', 'tiny', '--wandb_off', '--batch_size', '2',
           '--grad_accum_every', '3', '--checkpoint_every', '1', '--validate_every', '1', '--sample_every', '1000'] + list(extra)
    r = subprocess.run(cmd, cwd=str(tmp_path), capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    return r.stdout


def test_cli_group_by_length(tmp_path):
    import toml
    rng = np.random.default_rng(24)
    lines = [''.join(chr(65 + c) for c in rng.integers(0, 20, int(k))) for k in np.clip(rng.lognormal(4.5, 0.8, 40), 10, 500)]
    (tmp_path / 'seqs.txt').write_text('\n'.join(lines) + '\n')
    (tmp_path / 'tiny.toml').write_text(toml.dumps(CONFIGS['sgu']))
    index = {}
    for tag, extra in (('plain', []), ('grouped', ['--group_by_length']), ('graph', ['--group_by_length', '--cuda_graph'])):
        ckpt = tmp_path / tag
        out = _train(tmp_path, ckpt, '--num_steps', '3', *extra)
        assert 'counted tokens/sec' in out and 'tokens/sec (host clock' in out, out
        losses = [float(l.split()[1]) for l in out.splitlines() if l.startswith('loss:')]
        assert len(losses) == 3 and np.isfinite(losses).all(), out
        out = _train(tmp_path, ckpt, '--num_steps', '1', *extra)               # resume
        index[tag] = [l for l in out.splitlines() if l.startswith('starting from sequence')]
    assert index['plain'] == index['grouped'] == index['graph'] == ['starting from sequence 18'], index
