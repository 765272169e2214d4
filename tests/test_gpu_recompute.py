"""Training with recomputed activations (DESIGN.md §3.12) against the resident training step.

What must hold: a layer re-run from its checkpoint writes the resident forward's activations bitwise (the same launches
on the same inputs), so the logits, the head outputs and the gradient into the residual stream at layer 0 are bitwise
the resident step's.  Weight, adapter and head gradients and the loss only sum in another order from run to run (split-K
and column-sum atomics), within test_gpu_cut_train.py's bounds: 1e-4 (fp32) / 1e-3 (bf16) of a leaf's largest entry.
Inference (`apply`, `score`, `predict`) does not depend on the mode."""
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BASE = dict(num_tokens=256, dim=128, seq_len=512, depth=3, window_size=256, heads=2, dim_head=64)
CONFIGS = {
    'sgu': dict(BASE, global_mlp_depth=1),
    'gelu': dict(BASE, global_mlp_depth=1, ff_glu=False),
    'noshift': dict(BASE, global_mlp_depth=1, shift_tokens=False),
    'wide_window': dict(BASE, global_mlp_depth=1, window_size=512),
}
CFG4 = dict(num_tokens=256, dim=1536, seq_len=4096, depth=3, heads=8, dim_head=64, window_size=256, global_mlp_depth=2)
GRAD_TOL = {False: 1e-4, True: 1e-3}


def _rows(B, n, lens, seed):
    """(B, n+1) rows whose labels end after lens[i] residues (counted length lens[i] + 1)"""
    r = np.random.default_rng(seed).integers(1, 256, (B, n + 1)).astype(np.uint16)
    for i, k in enumerate(lens):
        r[i, 1 + k:] = 0
    return r


def _params(cfg, seed):
    from oracle import progen_ref as O
    return O.randomize_params(O.init_params(O.make_config(**cfg), seed), seed + 1)


def _adapters(model, seed):
    ad = model.init_adapters(seed, 16)
    for v in ad.values():
        v['lora_b'] = (0.05 * np.random.default_rng(seed).standard_normal(v['lora_b'].shape)).astype(np.float32)
    return ad


def _close_trees(a, b, tol):
    for m, d in b.items():
        for k, r in d.items():
            scale = max(1e-8, float(np.abs(r).max()))
            err = float(np.abs(a[m][k] - r).max())
            assert err <= tol * scale + 1e-7, (m, k, err, scale)


# ---------------------------------------------------------------------------------------------------- 1. activations
@pytest.mark.parametrize('lora', [False, True])
@pytest.mark.parametrize('mp', [False, True])
@pytest.mark.parametrize('name', list(CONFIGS))
def test_recomputed_layers_are_the_resident_activations(name, mp, lora):
    """every layer's buffers after recompute_layer (into a NaN-filled shared scratch) are bitwise the resident
    forward's, on the cut (B, L) view of the step"""
    from progen_b200 import ProGen
    cfg = CONFIGS[name]
    params = _params(cfg, 3)
    n = cfg['seq_len']
    rows = _rows(3, n, [300, 120, 350], 5)
    Lc = 384
    T = 3 * Lc
    runs = {}
    for rc in (False, True):
        model = ProGen(**cfg, mixed_precision=mp, recompute=rc)
        model._ensure_loaded(params)
        eng = model.engine
        if lora:
            model._attach_adapters(_adapters(model, 7), 32.0)
        eng.load_batch(rows, Lc)
        eng.train_step((), 3, backward=False, length=Lc)
        runs[rc] = (model, eng, eng.acts.view(3, Lc))
    _, er, vr = runs[False]
    _, ec, vc = runs[True]
    nl = len(ec.kinds)
    assert all(ec.lay[i] is ec.lay[0] or ec.kinds[i] != ec.kinds[0] for i in range(nl))        # one shared scratch
    assert all(ec.X[2 * i + 1] is ec.X[1] for i in range(nl))
    for i in range(nl):
        for t in list(vc.lay[i].values()) + [vc.X[2 * i + 1]]:
            t.fill_(float('nan'))
        mods = []
        if lora:
            a, f = 'pro_gen_base/~/' + f'attn{i}/~/', 'pro_gen_base/~/' + f'ff{i}/~/'
            mods = [a + 'linear', a + 'linear_1', f + 'linear']
            for m in mods:
                ec.lora.u[m].fill_(float('nan'))
        ec.recompute_layer(i, vc)
        torch.cuda.synchronize()
        for k, want in vr.lay[i].items():
            assert torch.equal(vc.lay[i][k], want), (i, k)
        assert torch.equal(vc.X[2 * i + 1], vr.X[2 * i + 1]), i
        for m in mods:
            assert torch.equal(ec.lora.u[m][:T], er.lora.u[m][:T]), (i, m)
    for k in range(0, 2 * nl + 1, 2):                                     # the checkpoints are the resident inputs
        assert torch.equal(vc.X[k], vr.X[k]), k


# ---------------------------------------------------------------------------------------------------- 2. steps
def _run_objective(model, params, objective, rows, seed):
    """(loss, gradient trees, head output, step length) of one step of `objective` through the public surface"""
    from progen_b200.engine import cut_length
    eng = model.engine
    n = model.config['seq_len']
    Lc = cut_length(rows[:, 1:])
    if objective in ('lm', 'lora'):
        ad = _adapters(model, seed) if objective == 'lora' else None
        loss, g = model.loss_and_grad(params, rows, adapters=ad, lora_alpha=32.0 if ad else None)
        B = rows.shape[0]
        head = eng.logits[:B * Lc].clone()
        return loss, [g], head, Lc
    if objective == 'preference':
        P = rows.shape[0] // 2
        ref = np.linspace(-600.0, -100.0, 2 * P).astype(np.float32)
        loss, g, st = model.preference_loss_and_grad(params, rows[:P], rows[P:], ref[:P], ref[P:], beta=0.1)
        return loss, [g], np.stack([st[k] for k in sorted(st)]), Lc
    ad, C = _adapters(model, seed), 3
    head = model.init_head(seed, C)
    rng = np.random.default_rng(seed)
    B = rows.shape[0]
    if objective.startswith('property'):
        task = objective.split('_')[1]
        y = rng.standard_normal((B, C)).astype(np.float32) if task == 'regression' else rng.integers(0, C, B)
        loss, g, hg, pred = model.property_loss_and_grad(params, rows, y, adapters=ad, head=head, task=task,
                                                         lora_alpha=32.0)
        return loss, [g, hg], pred, Lc
    t = np.full((B, n), -1, np.int64)
    for b in range(B):
        k = int((rows[b, 1:] != 0).sum())
        t[b, 1:1 + min(k, n - 1)] = rng.integers(0, C, min(k, n - 1))
    loss, g, hg, pred = model.residue_loss_and_grad(params, rows, t, adapters=ad, head=head, task='classification',
                                                    lora_alpha=32.0)
    return loss, [g, hg], pred, eng.res_view[1]


OBJECTIVES = ['lm', 'lora', 'preference', 'property_regression', 'property_classification', 'residue']


def _check_step(cfg, mp, objective, rows, seed=11):
    from progen_b200 import ProGen
    params = _params(cfg, seed)
    out = {}
    for rc in (False, True):
        model = ProGen(**cfg, mixed_precision=mp, recompute=rc)
        loss, trees, head, Lc = _run_objective(model, params, objective, rows, seed)
        torch.cuda.synchronize()
        out[rc] = (loss, trees, head, Lc, model.engine.dres[:rows.shape[0] * Lc].clone())
    (lr, tr, hr, Lr, dr), (lc, tc, hc, Lcc, dc) = out[False], out[True]
    assert Lr == Lcc
    if isinstance(hr, torch.Tensor):
        assert torch.equal(hr, hc)
    else:
        np.testing.assert_array_equal(hr, hc)
    assert torch.equal(dr, dc)                                            # d loss / d residual stream at layer 0
    assert abs(lr - lc) <= 1e-6 * max(1.0, abs(lr)), (lr, lc)
    for a, b in zip(tc, tr):
        if b is not None:
            _close_trees(a, b, GRAD_TOL[mp])
    return Lr


@pytest.mark.parametrize('objective', OBJECTIVES)
@pytest.mark.parametrize('mp', [False, True])
@pytest.mark.parametrize('name', list(CONFIGS))
@pytest.mark.parametrize('cut', [False, True])
def test_steps_agree_with_the_resident_step(cut, name, mp, objective):
    cfg = CONFIGS[name]
    n = cfg['seq_len']
    lens = ([300, 120, 350, 40] if name != 'wide_window' else [100, 20, 60, 90]) if cut else [511, 120, 350, 40]
    L = _check_step(cfg, mp, objective, _rows(4, n, lens, 17))
    assert (L < n) == cut, L


# ---------------------------------------------------------------------------------------------------- 3. float64
def test_fp32_recompute_loss_and_grad_match_oracle():
    from golden_util import CASES, load_case
    from oracle import progen_torch as T
    from progen_b200 import ProGen
    for name in [k for k in CASES if k != 'cfg1']:
        cfg, params, data, g = load_case(name)
        loss, grads = ProGen(**CASES[name], recompute=True).loss_and_grad(params, data)
        ref_loss, ref = T.loss_and_grads(params, data, cfg)
        assert abs(loss - float(g['loss'])) < 1e-5 and abs(loss - ref_loss) < 1e-5, name
        for m, d in ref.items():
            for k, r in d.items():
                scale = max(1e-8, np.abs(r).max())
                assert np.abs(grads[m][k] - r).max() < 2e-4 * scale + 1e-7, (name, m, k)


# ---------------------------------------------------------------------------------------------------- 4. trainer
@pytest.mark.parametrize('lora', [False, True])
@pytest.mark.parametrize('mp', [False, True])
def test_trainer_graphs_and_five_steps(mp, lora):
    """a recompute trainer with cuda_graph=True captures and replays like its eager loop (steps 6 to 8
    replay); eight steps (two updates) in each mode leave the trained parameters within the bounds"""
    from progen_b200 import ProGen
    cfg = CONFIGS['sgu']
    n = cfg['seq_len']
    params = _params(cfg, 19)
    batches = [_rows(2, n, l, 20 + i) for i, l in enumerate([[100, 20], [300, 200], [511, 5]] * 2)][:5]
    runs = {}
    for rc, graph in ((False, False), (True, False), (True, True)):
        model = ProGen(**cfg, mixed_precision=mp, recompute=rc)
        kw = dict(adapters=_adapters(model, 21), lora_alpha=32.0) if lora else {}
        tr = model.trainer(params, learning_rate=1e-2, grad_accum_every=4, cuda_graph=graph, **kw)
        losses = []
        for b in batches + batches[:1] * 3:                      # the last three steps repeat one (key, length)
            losses.append(float(tr.step(b).item()))
        runs[(rc, graph)] = (tr, losses)
    te, el = runs[(True, False)]
    tg, gl = runs[(True, True)]
    assert sorted(length for _, length in tg._graphs) == [128, 384], 'the steps of lengths 128 and 384 are captured'
    np.testing.assert_allclose(gl, el, rtol=0, atol=2e-2 if mp else 2e-5)
    tres, rl = runs[(False, False)]
    np.testing.assert_allclose(el, rl, rtol=0, atol=2e-2 if mp else 2e-5)
    get = (lambda t: t.adapters()) if lora else (lambda t: t.params())
    worst = lambda a, b: max(float(np.abs(a[m][k] - v).max()) for m, d in b.items() for k, v in d.items())
    assert worst(get(tg), get(te)) < (5e-2 if mp else 2e-3)
    assert worst(get(te), get(tres)) < (5e-2 if mp else 2e-3)


def test_switching_the_mode_reallocates_and_drops_graphs():
    from progen_b200 import ProGen
    cfg = CONFIGS['gelu']
    n = cfg['seq_len']
    params = _params(cfg, 23)
    model = ProGen(**cfg, mixed_precision=True)
    tr = model.trainer(params, cuda_graph=True)
    rows = _rows(2, n, [511, 300], 24)
    for _ in range(3):
        tr.step(rows)
    assert tr._graph is not None
    epoch = model.engine.alloc_epoch
    model.recompute = True
    assert model.engine.recompute and model.engine.alloc_epoch == epoch + 1
    tr.step(rows)                                            # the captured step is dropped, not replayed
    assert tr._graph is None
    assert all(model.engine.X[2 * i + 1] is model.engine.X[1] for i in range(cfg['depth']))


# ---------------------------------------------------------------------------------------------------- 5. memory
def _storage_bytes(eng):
    seen = {}

    def walk(v):
        if isinstance(v, torch.Tensor):
            s = v.untyped_storage()
            seen[s.data_ptr()] = s.nbytes()
        elif isinstance(v, (list, tuple)):
            for x in v:
                walk(x)
        elif isinstance(v, dict):
            for x in v.values():
                walk(x)
    for k in eng._train_keys:
        walk(getattr(eng, k))
    return sum(seen.values()), len(seen)


def test_training_set_bytes_at_config2_widths():
    from bench import CONFIGS as BENCH
    from progen_b200.engine import Engine, training_set
    kw = dict(BENCH['cfg2']['kwargs'], ff_mult=4, shift_tokens=True)
    got = {}
    for rc in (False, True):
        torch.cuda.synchronize()
        eng = Engine(kw, True, recompute=rc)
        before = torch.cuda.memory_allocated()
        eng.ensure_batch(2)
        torch.cuda.synchronize()
        delta = torch.cuda.memory_allocated() - before
        count = training_set(kw, 2, True, rc)[1]
        held, allocations = _storage_bytes(eng)
        assert eng.train_bytes == count == held, (rc, eng.train_bytes, count, held)
        # the caching allocator rounds each block up (to 512 bytes, a large one by less than 1 MiB)
        assert count <= delta <= count + allocations * (1 << 20), (rc, delta, count)
        got[rc] = count
        del eng
        torch.cuda.empty_cache()
    assert got[False] >= 3.5 * got[True], got


def test_lm_steps_at_config4_widths():
    """depth 3 at config 4's widths and sequence length, B = 4: item 2's LM checks (bf16)"""
    n = CFG4['seq_len']
    rows = _rows(4, n, [4095, 3000, 1000, 200], 31)
    _check_step(CFG4, True, 'lm', rows, seed=31)
    rows = _rows(4, n, [2000, 3000, 1000, 200], 32)
    assert _check_step(CFG4, True, 'lm', rows, seed=32) == 3072


# ---------------------------------------------------------------------------------------------------- 6. inference
@pytest.mark.parametrize('mp', [False, True])
def test_inference_does_not_depend_on_the_mode(mp):
    from progen_b200 import ProGen
    cfg = CONFIGS['sgu']
    n = cfg['seq_len']
    params = _params(cfg, 33)
    rows = _rows(3, n, [300, 120, 511], 34)
    out = {}
    for rc in (False, True):
        model = ProGen(**cfg, mixed_precision=mp, recompute=rc)
        head = model.init_head(0, 3)
        logits = model.apply(params, None, rows[:, :-1]).cpu()
        sc = model.score(params, rows, return_tokens=True, return_embeddings=True)
        pr = model.predict(params, head, rows)
        out[rc] = (logits, sc, pr)
    assert torch.equal(out[False][0], out[True][0])
    for k in out[False][1]:
        np.testing.assert_array_equal(out[False][1][k], out[True][1][k], err_msg=k)
    for k in out[False][2]:
        np.testing.assert_array_equal(out[False][2][k], out[True][2][k], err_msg=k)


# ---------------------------------------------------------------------------------------------------- 7. CLIs
def test_cli_recompute(tmp_path):
    cfg_dir = tmp_path / 'cfg'
    cfg_dir.mkdir()
    (cfg_dir / 'tiny.toml').write_text('num_tokens = 256\ndim = 128\ndepth = 2\ndim_head = 64\nheads = 2\n'
                                       'window_size = 64\nseq_len = 128\nglobal_mlp_depth = 1\n')
    env = dict(os.environ, PYTHONPATH=ROOT)
    run = lambda *a: subprocess.run([sys.executable, *a], cwd=ROOT, env=env, check=True, capture_output=True, text=True)
    base, fit = tmp_path / 'base', tmp_path / 'fit'
    out = run('train.py', '--synthetic', '--mixed_precision', '--recompute', '--num_steps', '2', '--config_path', str(cfg_dir),
              '--model_name', 'tiny', '--checkpoint_path', str(base), '--batch_size', '2', '--sample_every', '1000',
              '--validate_every', '1')
    losses = [float(l.split()[1]) for l in out.stdout.splitlines() if l.startswith('loss:')]
    assert len(losses) == 2 and np.isfinite(losses).all(), out.stdout
    pkg = pickle.load(open(sorted(base.glob('ckpt_*'))[-1], 'rb'))
    assert 'recompute' not in pkg['model_config']
    rng = np.random.default_rng(0)
    aa = 'ACDEFGHIKLMNPQRSTVWY'
    seqs = [''.join(rng.choice(list(aa), rng.integers(30, 90))) for _ in range(24)]
    (tmp_path / 'train.tsv').write_text(''.join(f'{s}\t{len(s) / 100:.3f}\n' for s in seqs))
    out = run('fitness.py', 'train', '--init_checkpoint', str(base), '--task', 'regression', '--lora_rank', '8',
              '--train', str(tmp_path / 'train.tsv'), '--checkpoint_path', str(fit), '--batch_size', '8', '--recompute',
              '--mixed_precision', '--cuda_graph')
    assert 'epoch 0: train loss' in out.stdout, out.stdout
    pkg = pickle.load(open(sorted(fit.glob('ckpt_*'))[-1], 'rb'))
    assert 'recompute' not in pkg['model_config']
