"""Distillation on the GPU (DESIGN.md §3.13): `progen_distill_head` against the float64 reference of its own inputs
(random and trained-regime logits, tau in {0.5, 1, 2, 4}, alpha in {0, 0.3, 1}, fp32 and bf16 dlogits, a teacher stride
above n), bitwise repeatable, masked rows exactly +0.0; the model-level loss, gradients and per-row stats against the
float64 twin with a deeper, wider teacher of a longer, non-128-aligned seq_len (full and LoRA, fp32 and bf16); alpha = 1
against `loss_and_grad`; self-distillation at alpha = 0; the cut step against the full-length one; captured against eager
steps and the graph drop after the teacher's inference set is re-allocated; recompute against resident; the teacher's
memory; a two-rank step; train.py end to end, then the student loaded by generate.py and score.py."""
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
from distill_oracle import distill_head, distill_loss_and_grads, loss_mask   # noqa: E402
from oracle import progen_ref as O                                           # noqa: E402
from trained_regime import HEAD_GAIN                                         # noqa: E402

pytestmark = pytest.mark.gpu

# the student runs at 192 positions; the teacher is deeper and wider, with seq_len 320 (not a multiple of 128), so a
# full-length student step reads the teacher at stride teacher_length(192, 320) = 256
STUDENT = dict(num_tokens=256, dim=128, seq_len=192, depth=2, window_size=64, heads=2, dim_head=64, global_mlp_depth=1)
TEACHER = dict(num_tokens=256, dim=192, seq_len=320, depth=3, window_size=64, heads=3, dim_head=64, global_mlp_depth=1)


def _rows(n, B=4, seed=0, lengths=(150, 60, 191, 20)):
    rng = np.random.default_rng(seed)
    rows = rng.integers(1, 256, (B, n + 1)).astype(np.int32)
    for i, k in enumerate(lengths[:B]):
        rows[i, 1 + k:] = 0
    return rows


def _params(kw, seed):
    return O.randomize_params(O.init_params(O.make_config(**kw), seed), seed + 1)


# ------------------------------------------------------------------------------------------------ kernel
def _launch(s, z, stride, labels, B, n, tau, alpha, dl_dtype):
    from progen_b200 import lib as L
    V = s.shape[-1]
    T_ = B * n
    nan = lambda *shape: torch.full(shape, float('nan'), device='cuda')
    w, scratch, stats, loss = nan(T_), nan(2 * T_), nan(B, 2), nan(1)
    dl = torch.full((T_, V), float('nan'), device='cuda', dtype=dl_dtype)
    L.check(L.load().progen_distill_head(s.data_ptr(), L.dt(s), z.data_ptr(), stride, labels.data_ptr(), w.data_ptr(),
                                         scratch.data_ptr(), stats.data_ptr(), loss.data_ptr(), dl.data_ptr(), L.dt(dl), B,
                                         n, V, tau, alpha, 1.0 / B, L.stream()), 'distill_head')
    torch.cuda.synchronize()
    return float(loss.item()), dl.float().cpu().numpy().reshape(B, n, V), stats.cpu().numpy()


@pytest.mark.parametrize('regime', ['random', 'sharp'])
@pytest.mark.parametrize('dl_dtype', [torch.float32, torch.bfloat16])
def test_kernel_against_float64(regime, dl_dtype):
    B, n, V, stride = 3, 70, 256, 96
    rng = np.random.default_rng(1)
    gain = HEAD_GAIN if regime == 'sharp' else 1.0
    s = (rng.standard_normal((B, n, V)) * 2 * gain).astype(np.float32)
    z = (rng.standard_normal((B, stride, V)) * 3 * gain).astype(np.float32)
    if regime == 'sharp':
        s[..., 7] += 4 * gain                              # confident rows: one dominant logit, as in a trained head
        z[..., 7] += 5 * gain
    labels = rng.integers(1, V, (B, n)).astype(np.int32)
    labels[0, 40:] = 0
    labels[1, :] = 0
    labels[2, 3] = 300                                     # clamped to V - 1
    m = loss_mask(labels)
    sd, zd = torch.tensor(s, device='cuda'), torch.tensor(z, device='cuda')
    ld = torch.tensor(labels, device='cuda')
    for tau in (0.5, 1.0, 2.0, 4.0):
        for alpha in (0.0, 0.3, 1.0):
            loss, dl, stats = _launch(sd, zd, stride, ld, B, n, tau, alpha, dl_dtype)
            rl, rg, rs = distill_head(s, z[:, :n], labels, tau, alpha)
            assert abs(loss - rl) <= 1e-4 * abs(rl) + 1e-5, (tau, alpha, loss, rl)
            assert np.abs(stats - rs).max() <= 1e-4 * np.abs(rs).max() + 1e-5, (tau, alpha)
            tol = (1e-4 if dl_dtype == torch.float32 else 1e-2) * np.abs(rg).max() + 1e-8
            assert np.abs(dl - rg).max() <= tol, (tau, alpha, np.abs(dl - rg).max(), tol)
            assert np.all(dl[m == 0] == 0.0) and not np.signbit(dl[m == 0]).any()
            again = _launch(sd, zd, stride, ld, B, n, tau, alpha, dl_dtype)
            assert again[0] == loss and np.array_equal(again[1], dl) and np.array_equal(again[2], stats)
    # bf16 student logits (the progen_ce_fwd_bwd combinations)
    sb = sd.bfloat16()
    loss, dl, _ = _launch(sb, zd, stride, ld, B, n, 2.0, 0.3, torch.bfloat16)
    rl, rg, _ = distill_head(sb.float().cpu().numpy(), z[:, :n], labels, 2.0, 0.3)
    assert abs(loss - rl) <= 1e-4 * abs(rl) + 1e-5 and np.abs(dl - rg).max() <= 1e-2 * np.abs(rg).max()


def test_kernel_refusals():
    from progen_b200 import lib as L
    lib = L.load()
    t = torch.zeros(4 * 8 * 16, device='cuda')
    lab = torch.ones(4 * 8, device='cuda', dtype=torch.int32)
    p = t.data_ptr()

    def call(**kw):
        a = dict(s=p, dt=L.F32, z=p, stride=8, lab=lab.data_ptr(), dl_dt=L.F32, B=4, n=8, V=16, tau=2.0, alpha=0.5, ib=0.25)
        a.update(kw)
        return lib.progen_distill_head(a['s'], a['dt'], a['z'], a['stride'], a['lab'], p, p, p, p, p, a['dl_dt'], a['B'],
                                       a['n'], a['V'], a['tau'], a['alpha'], a['ib'], L.stream())
    assert call() == 0
    for bad in (dict(z=0), dict(lab=0), dict(V=18), dict(stride=7), dict(tau=0.0), dict(tau=float('nan')),
                dict(tau=float('inf')), dict(alpha=-0.5), dict(alpha=1.5), dict(dt=L.BF16, dl_dt=L.F32), dict(dt=7)):
        assert call(**bad) != 0, bad
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ model level
def _rel(a, b):
    return float(np.abs(np.asarray(a) - np.asarray(b)).max()) / max(1e-6, float(np.abs(np.asarray(b)).max()))


@pytest.mark.parametrize('mp', [False, True])
@pytest.mark.parametrize('lora', [False, True])
def test_model_against_float64(mp, lora):
    from progen_b200 import ProGen
    student, teacher = ProGen(**STUDENT, mixed_precision=mp), ProGen(**TEACHER, mixed_precision=mp)
    params, tparams = _params(STUDENT, 3), _params(TEACHER, 5)
    rows = _rows(STUDENT['seq_len'])
    adapters, scale = None, 1.0
    if lora:
        adapters = student.init_adapters(4, 8)
        rng = np.random.default_rng(6)
        adapters = {m: dict(v, lora_b=(rng.standard_normal(v['lora_b'].shape) * 0.05).astype(np.float32))
                    for m, v in adapters.items()}
        scale = 2.0
    for tau, alpha in ((2.0, 0.5), (1.0, 0.0), (4.0, 0.3)):
        loss, grads, stats = student.distill_loss_and_grad(params, rows, teacher=teacher, teacher_params=tparams,
                                                           temperature=tau, alpha=alpha, adapters=adapters,
                                                           lora_alpha=None if adapters is None else 16.0)
        rl, rg, rs = distill_loss_and_grads(params, O.make_config(**STUDENT), tparams, O.make_config(**TEACHER), rows, tau,
                                            alpha, adapters, scale)
        tol_l, tol_g = (5e-2, 0.15) if mp else (1e-4, 2e-3)
        assert abs(loss - rl) <= tol_l * max(1.0, abs(rl)), (tau, alpha, loss, rl)
        assert _rel(np.stack([stats['kl'], stats['ce']], -1), rs) <= tol_l, (tau, alpha)
        worst = max(_rel(grads[m][k], g) for m, d in rg.items() for k, g in d.items())
        assert worst <= tol_g, (tau, alpha, worst)


@pytest.mark.parametrize('mp', [False, True])
def test_alpha_one_is_the_lm_loss_and_self_distillation_is_zero(mp):
    from progen_b200 import ProGen
    student, teacher = ProGen(**STUDENT, mixed_precision=mp), ProGen(**TEACHER, mixed_precision=mp)
    params, tparams = _params(STUDENT, 3), _params(TEACHER, 5)
    rows = _rows(STUDENT['seq_len'])
    lm_loss, lm_grads = student.loss_and_grad(params, rows)
    loss, grads, stats = student.distill_loss_and_grad(params, rows, teacher=teacher, teacher_params=tparams, alpha=1.0)
    assert abs(loss - lm_loss) <= 1e-5 * abs(lm_loss), (loss, lm_loss)
    assert _rel(stats['ce'].mean(), lm_loss) <= 1e-5
    for m, d in lm_grads.items():
        for k, g in d.items():
            assert np.allclose(grads[m][k], g, rtol=1e-4, atol=1e-5 * max(1e-6, np.abs(g).max())), (m, k)
    twin = ProGen(**STUDENT, mixed_precision=mp)
    loss, grads, stats = student.distill_loss_and_grad(params, rows, teacher=twin, teacher_params=params, alpha=0.0)
    assert abs(loss) < 1e-6 and np.abs(stats['kl']).max() < 1e-6, (loss, stats)


@pytest.mark.parametrize('mp', [False, True])
def test_cut_step_equals_full_length(mp):
    """loss, stats and dlogits bitwise; weight gradients to summation order"""
    from progen_b200 import ProGen
    from progen_b200.distill import teacher_length
    student, teacher = ProGen(**STUDENT, mixed_precision=mp), ProGen(**TEACHER, mixed_precision=mp)
    params, tparams = _params(STUDENT, 3), _params(TEACHER, 5)
    rows = _rows(STUDENT['seq_len'], lengths=(100, 60, 20, 7))
    student._ensure_loaded(params)
    teacher._ensure_loaded(tparams)
    eng = student.engine
    eng.attach_teacher(teacher.engine)
    out = {}
    n = STUDENT['seq_len']
    for L_ in (128, n):
        B = eng.load_distill(rows, L_)
        eng.train_step(('distill', 2.0, 0.3), B, length=L_)
        torch.cuda.synchronize()
        dl = eng.dlogits[:B * L_].float().view(B, L_, -1)[:, :128].cpu().numpy()
        assert np.all(eng.dlogits[:B * L_].float().view(B, L_, -1)[:, 128:].cpu().numpy() == 0.0)
        out[L_] = (float(eng.loss.item()), eng.distill_stats(B), dl, eng.export_grads())
        assert teacher_length(L_, TEACHER['seq_len']) == (128 if L_ == 128 else 256)
    (l1, s1, d1, g1), (l2, s2, d2, g2) = out[128], out[n]
    assert l1 == l2 and np.array_equal(s1['kl'], s2['kl']) and np.array_equal(s1['ce'], s2['ce'])
    assert np.array_equal(d1, d2)
    for m, d in g2.items():
        for k, g in d.items():
            assert np.allclose(g1[m][k], g, rtol=1e-3, atol=1e-4 * max(1e-6, np.abs(g).max())), (m, k)


@pytest.mark.parametrize('lora', [False, True])
def test_captured_steps_and_the_teacher_set_drop(lora):
    from progen_b200 import ProGen
    student, teacher = ProGen(**STUDENT, mixed_precision=True), ProGen(**TEACHER, mixed_precision=True)
    params, tparams = _params(STUDENT, 3), _params(TEACHER, 5)
    rows = _rows(STUDENT['seq_len'])
    kw = dict(learning_rate=0.0, weight_decay=0.0, data_parallel=False, teacher=teacher, teacher_params=tparams)
    if lora:
        kw.update(adapters=student.init_adapters(4, 8))
    eager = student.trainer(params, **kw)
    want = [float(eager.distill_step(rows, 2.0, 0.5).item()) for _ in range(3)]
    want_g = eager.G.clone()
    assert eager._graph is None
    tr = student.trainer(params, cuda_graph=True, **kw)
    got = [float(tr.distill_step(rows, 2.0, 0.5).item()) for _ in range(3)]
    assert tr._graph is not None and tr._graph_key[2:] == ('distill', 2.0, 0.5)
    assert got == want
    assert torch.allclose(tr.G, want_g, rtol=1e-3, atol=1e-6 * float(want_g.abs().max()))
    assert np.array_equal(tr.distill_stats()['kl'], eager.distill_stats()['kl'])
    # a larger score call on the teacher re-allocates its inference set: the captured steps are dropped before replay
    teacher.score(tparams, _rows(TEACHER['seq_len'], B=8, lengths=(10,) * 8))
    assert float(tr.distill_step(rows, 2.0, 0.5).item()) == want[0]
    assert tr._graph is None


def test_recompute_equals_resident():
    from progen_b200 import ProGen
    params, tparams = _params(STUDENT, 3), _params(TEACHER, 5)
    rows = _rows(STUDENT['seq_len'])
    out = []
    for rc in (False, True):
        student = ProGen(**STUDENT, mixed_precision=True, recompute=rc)
        out.append(student.distill_loss_and_grad(params, rows, teacher=ProGen(**TEACHER, mixed_precision=True),
                                                 teacher_params=tparams))
    assert out[0][0] == out[1][0]
    assert np.array_equal(out[0][2]['kl'], out[1][2]['kl'])
    for m, d in out[0][1].items():
        for k, g in d.items():
            assert np.allclose(out[1][1][m][k], g, rtol=1e-3, atol=1e-4 * max(1e-6, np.abs(g).max())), (m, k)


def test_teacher_allocates_no_training_state():
    from progen_b200 import ProGen
    student, teacher = ProGen(**STUDENT, mixed_precision=True), ProGen(**TEACHER, mixed_precision=True)
    params, tparams = _params(STUDENT, 3), _params(TEACHER, 5)
    teacher.loss_and_grad(tparams, _rows(TEACHER['seq_len'], B=2))      # the teacher model has trained once
    tr = student.trainer(params, data_parallel=False, teacher=teacher, teacher_params=tparams)
    te = teacher.engine
    assert te.grads is None and te.B == 0 and te.acts is None and te.train_bytes == 0
    assert all(getattr(te, k, None) is None for k in ('X', 'lay', 'logits', 'dlogits', 'dres'))
    tr.distill_step(_rows(STUDENT['seq_len']), 2.0, 0.5)
    torch.cuda.synchronize()
    assert te.grads is None and te.B == 0 and te.infer is not None and te.infer.B == 4
    m = tr.m                                               # the student's optimizer state exists; the teacher has none
    assert m.numel() == student.engine.n_params_padded


def test_two_rank_step():
    if torch.cuda.device_count() < 2:
        pytest.skip('needs two GPUs')
    out = os.path.join(os.environ.get('TMPDIR', '/tmp'), f'distill_ddp_{os.getpid()}.json')
    subprocess.run([sys.executable, '-m', 'torch.distributed.run', '--nproc_per_node', '2',
                    os.path.join(HERE, 'ddp_distill_worker.py'), out], check=True, cwd=ROOT)
    import json
    res = json.load(open(out))
    for mp, r in res.items():
        assert abs(r['loss_ddp'] - r['loss_single']) <= 1e-5 * abs(r['loss_single']), (mp, r)
        assert r['grad_rel_l2'] < (1e-2 if mp == 'True' else 1e-5), (mp, r)


# ------------------------------------------------------------------------------------------------ CLI
def test_train_py_end_to_end(tmp_path):
    cfg_dir = tmp_path / 'cfg'
    cfg_dir.mkdir()
    tom = lambda kw: ''.join(f'{k} = {v}\n' for k, v in kw.items())
    (cfg_dir / 'student.toml').write_text(tom(STUDENT))
    (cfg_dir / 'teacher.toml').write_text(tom(TEACHER))
    env = dict(os.environ, PYTHONPATH=ROOT)
    run = lambda *a: subprocess.run([sys.executable, *a], cwd=ROOT, env=env, check=True, capture_output=True, text=True)
    rng = np.random.default_rng(0)
    aa = 'ACDEFGHIKLMNPQRSTVWY'
    (tmp_path / 'seqs.txt').write_text(''.join(''.join(rng.choice(list(aa), rng.integers(30, 150))) + '\n'
                                               for _ in range(64)))
    common = ['--mixed_precision', '--config_path', str(cfg_dir), '--batch_size', '4', '--grad_accum_every', '2',
              '--sample_every', '1000', '--validate_every', '1', '--checkpoint_every', '1', '--text_file',
              str(tmp_path / 'seqs.txt')]
    teacher_dir, student_dir = tmp_path / 'teacher', tmp_path / 'student'
    run('train.py', *common, '--model_name', 'teacher', '--num_steps', '1', '--checkpoint_path', str(teacher_dir))
    out = run('train.py', *common, '--model_name', 'student', '--num_steps', '2', '--checkpoint_path', str(student_dir),
              '--teacher_checkpoint', str(teacher_dir), '--distill_temperature', '2.0', '--distill_alpha', '0.3',
              '--cuda_graph', '--group_by_length')
    lines = out.stdout.splitlines()
    losses = [float(l.split()[1]) for l in lines if l.startswith('loss:')]
    kls = [float(l.split()[1]) for l in lines if l.startswith('valid_kl:')]
    assert len(losses) == 2 and np.isfinite(losses).all() and len(kls) == 2 and min(kls) >= 0, out.stdout
    pkg = pickle.load(open(sorted(student_dir.glob('ckpt_*'))[-1], 'rb'))
    assert pkg['distill']['temperature'] == 2.0 and pkg['distill']['alpha'] == 0.3 and 'params' in pkg
    assert pkg['model_config']['dim'] == STUDENT['dim']
    out = run('train.py', *common, '--model_name', 'student', '--num_steps', '3', '--checkpoint_path', str(student_dir))
    assert 'distilling' in out.stdout and 'valid_kl:' in out.stdout, out.stdout
    bad = subprocess.run([sys.executable, 'train.py', *common, '--model_name', 'student', '--checkpoint_path',
                          str(student_dir), '--distill_alpha', '0.9'], cwd=ROOT, env=env, capture_output=True, text=True)
    assert bad.returncode == 2 and 'distils with alpha 0.3' in bad.stderr + bad.stdout
    out = run('generate.py', '--checkpoint_path', str(student_dir), '--prompt', 'MK', '--num_samples', '2',
              '--max_length', '40', '--mixed_precision')
    assert out.returncode == 0
    (tmp_path / 'score.txt').write_text('MKVLAAG\nMKKLLE\n')
    run('score.py', '--checkpoint_path', str(student_dir), '--input', str(tmp_path / 'score.txt'), '--output',
        str(tmp_path / 'scores.tsv'), '--mixed_precision')
    assert len((tmp_path / 'scores.tsv').read_text().strip().splitlines()) >= 2
