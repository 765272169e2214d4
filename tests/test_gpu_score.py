"""Scoring: ProGen.score / score.py on the inference forward, and its kernels (progen_token_logprob,
progen_masked_mean_pool, the GLU / GELU epilogues without the pre-activation store)."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from golden_util import load_case, CASES

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TINY = [n for n in CASES if n != 'cfg1']
BF16_OK = ['tiny_all_glu']
# one GLU and one gMLP layer (or GELU + gMLP), two windows of 128: wgmma attention on the bf16 engine
SMALL = dict(num_tokens=256, dim=128, seq_len=256, depth=2, window_size=128, global_mlp_depth=1, heads=2, dim_head=64)


def _case(kwargs, seed, rows):
    from oracle import progen_ref as O
    cfg = O.make_config(**kwargs)
    params = O.randomize_params(O.init_params(cfg, seed), seed + 1)
    rng = np.random.default_rng(seed + 2)
    data = rng.integers(1, 256, (rows, cfg['seq_len'] + 1)).astype(np.uint16)
    for r in range(1, rows, 2):                                   # every other row ends early: EOS + padding
        data[r, 1 + int(rng.integers(1, cfg['seq_len'])):] = 0
    return cfg, params, data


def _hidden_oracle(params, rows, cfg):
    """final-LayerNorm output of the float64 oracle, through oracle.forward itself: with the head weight [I | 0] and no
    bias, the first `dim` logits of each position are the hidden state (x @ I is exact)"""
    from oracle import progen_ref as O
    d, V = cfg['dim'], cfg['num_tokens']
    assert V >= d
    p = dict(params)
    p[O.P + 'linear'] = {'w': np.eye(d, V, dtype=np.float32), 'b': np.zeros(V, np.float32)}
    return np.stack([O.forward(p, r[:-1], cfg)[:, :d] for r in np.asarray(rows)])


def _pool(hidden, rows):
    from oracle import progen_ref as O
    m = O.loss_mask(np.asarray(rows)[:, 1:]).astype(np.float64)
    return (hidden * m[..., None]).sum(1) / m.sum(1)[:, None]


def _token_logprob(logits, labels):
    """progen_token_logprob on device logits (B, n, V) fp32 and labels (B, n) -> (logp, seq_ll, seq_count) numpy"""
    from progen_b200 import lib as L
    B, n, V = logits.shape
    lab = torch.as_tensor(np.asarray(labels).astype(np.int32)).cuda()
    lp, ll, cnt = torch.empty(B * n, device='cuda'), torch.empty(B, device='cuda'), torch.empty(B, device='cuda')
    L.check(L.load().progen_token_logprob(logits.data_ptr(), L.F32, lab.data_ptr(), lp.data_ptr(), ll.data_ptr(), cnt.data_ptr(),
                                          B, n, V, L.stream()), 'token_logprob')
    return lp.cpu().numpy().reshape(B, n), ll.cpu().numpy(), cnt.cpu().numpy()


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', sorted(CASES))
def test_fp32_score_matches_reference_golden(name):
    """-log_likelihood / num_tokens is the per-row cross entropy the reference source computed (ce_per_row)"""
    from progen_b200 import ProGen
    from oracle import progen_ref as O
    cfg, params, data, g = load_case(name)
    sc = ProGen(**CASES[name]).score(params, data)
    ce = -sc['log_likelihood'].astype(np.float64) / sc['num_tokens']
    assert np.abs(ce - g['ce_per_row']).max() < 1e-5, (ce, g['ce_per_row'])
    np.testing.assert_array_equal(sc['num_tokens'], O.loss_mask(data[:, 1:]).sum(-1))


@pytest.mark.parametrize('ff_glu', [True, False])
@pytest.mark.parametrize('mp', [False, True])
def test_score_is_the_apply_forward(mp, ff_glu):
    """The inference forward (in-place residual, no pre-activation store, one shared layer scratch) computes the same
    logits as the training forward behind .apply: the token log-probabilities are bitwise equal."""
    from progen_b200 import ProGen
    from oracle import progen_ref as O
    cfg, params, data = _case({**SMALL, 'ff_glu': ff_glu}, 31, 3)
    model = ProGen(**cfg, mixed_precision=mp)
    logits = model.apply(params, None, data[:, :-1])
    lp, ll, cnt = _token_logprob(logits, data[:, 1:])
    sc = model.score(params, data, return_tokens=True)
    np.testing.assert_array_equal(sc['token_logp'], lp)
    np.testing.assert_array_equal(sc['log_likelihood'], ll)
    np.testing.assert_array_equal(sc['num_tokens'], cnt.astype(np.int64))
    mask = O.loss_mask(data[:, 1:])
    np.testing.assert_array_equal(sc['token_mask'], mask)
    lg = logits.double().cpu().numpy()
    ls = lg - lg.max(-1, keepdims=True)
    ls = ls - np.log(np.exp(ls).sum(-1, keepdims=True))
    ref = np.take_along_axis(ls, data[:, 1:].astype(np.int64)[..., None], -1)[..., 0] * mask
    assert np.abs(sc['token_logp'] - ref).max() < 1e-5 * max(1.0, np.abs(lg).max())


@pytest.mark.parametrize('mp', [False, True])
def test_score_does_not_depend_on_batch_size(mp):
    """fixed-order per-sequence reductions: batch_size 64, 7 (ragged last chunk) and 1 give the same bits"""
    from progen_b200 import ProGen
    cfg, params, data = _case(SMALL, 41, 20)
    model = ProGen(**cfg, mixed_precision=mp)
    runs = [model.score(params, data, batch_size=bs, return_tokens=True, return_embeddings=True) for bs in (64, 7, 1)]
    for r in runs[1:]:
        for k in runs[0]:
            np.testing.assert_array_equal(r[k], runs[0][k], err_msg=k)


@pytest.mark.parametrize('mp', [False, True])
def test_score_agrees_with_training_loss(mp):
    """mean over rows of -ll/count is the loss_and_grad loss (which sums with fp32 atomics, in no fixed order)"""
    from progen_b200 import ProGen
    cfg, params, data = _case(SMALL, 51, 6)
    model = ProGen(**cfg, mixed_precision=mp)
    loss, _ = model.loss_and_grad(params, data)
    sc = model.score(params, data)
    mean = float(np.mean(-sc['log_likelihood'].astype(np.float64) / sc['num_tokens']))
    assert abs(mean - loss) <= 1e-5 * abs(loss), (mean, loss)


def test_score_ragged_rows():
    """a short sequence, an all-pad row (count 1: the first pad), a row without pad (count n), and the label 256 (byte
    0xFF + 1), clamped to V - 1 like the training loss and the embedding gather"""
    from progen_b200 import ProGen
    from oracle import progen_ref as O
    cfg, params, data = _case(SMALL, 61, 4)
    n = cfg['seq_len']
    data[0, 41:] = 0                        # 40 residues -> labels 0..39 plus the EOS at 40
    data[1, :] = 0
    data[2] = np.random.default_rng(0).integers(1, 256, n + 1)
    data[3] = np.random.default_rng(1).integers(1, 256, n + 1)
    data[3, 7] = 256                        # label at position 6, id at position 7
    sc = ProGen(**cfg).score(params, data, return_tokens=True)
    np.testing.assert_array_equal(sc['num_tokens'], [41, 1, n, n])
    clipped = np.clip(data.astype(np.int64), 0, cfg['num_tokens'] - 1)
    ref = np.array([O.cross_entropy(O.forward(params, r[:-1], cfg), r[1:]) for r in clipped])
    ce = -sc['log_likelihood'].astype(np.float64) / sc['num_tokens']
    assert np.abs(ce - ref).max() < 1e-5, (ce, ref)
    assert not sc['token_mask'][0, 41:].any() and sc['token_mask'][0, :41].all()
    assert (sc['token_logp'][~sc['token_mask']] == 0).all()


@pytest.mark.parametrize('name', TINY)
def test_fp32_embedding_matches_oracle(name):
    from progen_b200 import ProGen
    cfg, params, data, _ = load_case(name)
    ref = _pool(_hidden_oracle(params, data, cfg), data)
    emb = ProGen(**CASES[name]).score(params, data, return_embeddings=True)['embedding']
    assert emb.shape == (data.shape[0], cfg['dim'])
    assert np.abs(emb - ref).max() < 1e-5 * max(1.0, np.abs(ref).max()), np.abs(emb - ref).max()


@pytest.mark.parametrize('name', BF16_OK)
def test_bf16_embedding(name):
    """bf16 engine (its final LN output is stored in bf16): bounded against the fp64 oracle and against the CPU emulation
    of a bf16-operand engine (oracle/progen_torch.py), whose hidden state is read through the same [I | 0] head"""
    from progen_b200 import ProGen
    from oracle import progen_ref as O
    from oracle import progen_torch as T
    cfg, params, data, _ = load_case(name)
    emb = ProGen(**CASES[name], mixed_precision=True).score(params, data, return_embeddings=True)['embedding'].astype(np.float64)
    ref = _pool(_hidden_oracle(params, data, cfg), data)
    err = np.abs(emb - ref)
    assert err.max() < 5e-2 and err.mean() < 1e-2, (err.max(), err.mean())
    d, V = cfg['dim'], cfg['num_tokens']
    p = dict(params)
    p[O.P + 'linear'] = {'w': np.eye(d, V, dtype=np.float32), 'b': np.zeros(V, np.float32)}
    ids = torch.as_tensor(data[:, :-1].astype(np.int64))
    hid = T.forward(T.to_torch(p, torch.float32), ids, cfg, T.bf16_round).double().numpy()[..., :d]
    e2 = np.abs(emb - _pool(hid, data))
    assert e2.max() < 5e-2 and e2.mean() < 1e-2, (e2.max(), e2.mean())


@pytest.mark.parametrize('epi', ['glu', 'gelu'])
@pytest.mark.parametrize('backend', ['tc', 'simt'])
def test_preactivation_store_is_optional(backend, epi):
    """EPI_GLU / EPI_GELU with out2 = NULL write the same `out`, bitwise, as with the pre-activation store"""
    from progen_b200 import lib as L
    be, dt, ldt = (L.BACKEND_TC, torch.bfloat16, L.BF16) if backend == 'tc' else (L.BACKEND_SIMT, torch.float32, L.F32)
    g = torch.Generator(device='cuda').manual_seed(3)
    M, K, N = 512, 128, 384
    x = torch.randn(M, K, generator=g, device='cuda').to(dt)
    w = (torch.randn(K, N, generator=g, device='cuda') * K ** -0.5).to(dt)
    bias = torch.randn(N, generator=g, device='cuda')
    kind, N_out = (L.EPI_GLU, N // 2) if epi == 'glu' else (L.EPI_GELU, N)
    outs = []
    for store in (True, False):
        out = torch.full((M, N_out), float('nan'), device='cuda', dtype=dt)
        u = torch.empty(M, N, device='cuda', dtype=dt) if store else None
        L.gemm(M=M, N=N, K=K, A=x, lda=K, B=w, ldb=N, b_mn=True, out=out, ldo=N_out, epi=kind, backend=be, in_dtype=ldt,
               out_dtype=ldt, out2=u, ldo2=N, bias=bias)
        outs.append(out)
    torch.cuda.synchronize()
    assert not outs[1].isnan().any()
    assert torch.equal(outs[0], outs[1])


@pytest.mark.parametrize('mp', [False, True])
def test_score_leaves_captured_training_untouched(mp):
    """score between steps of a Trainer whose step is a captured CUDA graph: the graph stays installed (alloc_epoch is
    unchanged), every buffer the step reads and updates (parameters, bf16 mirror, masked SGU copies, Adam moments,
    accumulator) is bitwise what it was before the call, and the run ends where a run without score calls ends.  (The two
    runs are compared within the bounds of test_trainer_cuda_graph_replay_matches_eager: the backward's split-K and
    bias-gradient atomics add in a different order from run to run.)"""
    from progen_b200 import ProGen
    cfg, params, data = _case(SMALL, 71, 4)
    rng = np.random.default_rng(72)
    batches = [rng.integers(0, 256, (2, cfg['seq_len'] + 1)).astype(np.uint16) for _ in range(6)]
    finals, losses = {}, {}
    for mode in ('plain', 'score'):
        model = ProGen(**cfg, mixed_precision=mp)
        tr = model.trainer(params, grad_accum_every=2, learning_rate=1e-2)
        eng = tr.eng
        out = [float(tr.step(batches[0]).item())]
        tr.capture_graph(2)
        graph, epoch = tr._graph, eng.alloc_epoch
        for b in batches[1:]:
            out.append(float(tr.step(b).item()))
            if mode == 'score':
                state = [t.clone() for t in (eng.params, eng.grads, tr.m, tr.v, tr.acc)]
                state += [eng.params_lp.clone()] if mp else []
                state += [w.clone() for w in eng.wm.values()]
                eng.score(data, batch_size=3, tokens=True, embeddings=True)
                after = [eng.params, eng.grads, tr.m, tr.v, tr.acc] + ([eng.params_lp] if mp else []) + list(eng.wm.values())
                assert all(torch.equal(a, b) for a, b in zip(state, after))
                assert eng.alloc_epoch == epoch and tr._graph is graph and eng.B == 2
        assert tr._graph is graph
        finals[mode], losses[mode] = tr.params(), out
    np.testing.assert_allclose(losses['score'], losses['plain'], rtol=0, atol=2e-2 if mp else 2e-5)
    worst = max(float(np.abs(finals['score'][m][k] - r).max()) for m, d in finals['plain'].items() for k, r in d.items())
    assert worst < (5e-2 if mp else 2e-3), worst


def test_score_memory_config2():
    """config-2 shape, batch_size 64: the inference set is ~18 KB per token (~1.2 GB), far below the ~280 KB per token
    (~18 GB) of the training activations; the peak that score adds stays under 2 GB"""
    from progen_b200 import ProGen
    kwargs = dict(num_tokens=256, dim=512, seq_len=1024, depth=12, heads=8, dim_head=64, window_size=256, global_mlp_depth=2,
                  ff_glu=True)
    model = ProGen(**kwargs, mixed_precision=True)
    params = model.init(0)
    data = np.random.default_rng(42).integers(0, 256, (64, kwargs['seq_len'] + 1)).astype(np.uint16)
    model.engine                                      # the engine's parameter buffers are allocated before the baseline
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    sc = model.score(params, data, batch_size=64)
    torch.cuda.synchronize()
    added = torch.cuda.max_memory_allocated() - base
    print(f'score adds {added / 2**30:.3f} GiB ({added / (64 * kwargs["seq_len"]) / 1024:.1f} KiB per token)')
    assert added < 2 * 10**9, added
    assert np.isfinite(sc['log_likelihood']).all()


def test_score_cli(tmp_path):
    """score.py on a checkpoint: the TSV is model.score of the same rows, the .npy the embeddings"""
    from progen_b200 import ProGen
    from progen_b200.checkpoint import file_save_checkpoint
    from progen_b200.data import collate
    kwargs = dict(num_tokens=256, dim=128, seq_len=128, depth=2, window_size=64, global_mlp_depth=1, heads=2, dim_head=64)
    from oracle import progen_ref as O
    params = O.randomize_params(O.init_params(O.make_config(**kwargs), 81), 82)
    (tmp_path / 'ckpts').mkdir()
    file_save_checkpoint(tmp_path / 'ckpts', dict(next_seq_index=0, params=params, optim_state=None, model_config=kwargs,
                                                  run_id=None))
    seqs = ['[tax=Mammalia] # MKTAYIAKQRQISFVKSHFSRQ', 'ACDEFGHIKLMNPQRSTVWY' * 10, 'MSTNPKPQRKTKRNTNRRPQDVKFPGG']
    (tmp_path / 'in.txt').write_text('\n'.join(seqs) + '\n\n')
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'score.py'), '--checkpoint_path', str(tmp_path / 'ckpts'),
                        '--input', str(tmp_path / 'in.txt'), '--output', str(tmp_path / 'out.tsv'), '--embeddings',
                        str(tmp_path / 'emb.npy'), '--batch_size', '2'], cwd=str(tmp_path), env=env, capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert '3 sequences, 1 truncated to 128 residues' in r.stdout
    lines = (tmp_path / 'out.tsv').read_text().splitlines()
    assert lines[0].split('\t') == ['index', 'residues', 'log_likelihood', 'num_tokens', 'mean_nll', 'perplexity']
    rows = [l.split('\t') for l in lines[1:]]
    assert len(rows) == 3
    ref = ProGen(**kwargs).score(params, collate(seqs, kwargs['seq_len']), return_embeddings=True)
    for i, row in enumerate(rows):
        assert int(row[0]) == i and int(row[1]) == min(len(seqs[i]), 128)
        assert np.float32(float(row[2])) == ref['log_likelihood'][i] and int(row[3]) == ref['num_tokens'][i]
        nll = -float(ref['log_likelihood'][i]) / ref['num_tokens'][i]
        assert abs(float(row[4]) - nll) <= 1e-6 * abs(nll) and abs(float(row[5]) - np.exp(nll)) <= 1e-6 * np.exp(nll)
    emb = np.load(tmp_path / 'emb.npy')
    assert emb.shape == (3, kwargs['dim'])
    np.testing.assert_array_equal(emb, ref['embedding'])
