"""The host side of distillation (DESIGN.md §3.13): the float64 head reference (tests/distill_oracle.py) against finite
differences, the cross entropy at alpha = 1 and the tau^2 convention; every refusal; the teacher length rule; train.py's
flag checks, resume refusals and package round trip; and the launches of the existing objectives, recorded with a
stand-in kernel library, against the ones they made before distillation existed."""
import json
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
from distill_oracle import distill_head, loss_mask          # noqa: E402
from progen_b200 import ProGen                              # noqa: E402
from progen_b200.distill import check_objective, check_teacher, teacher_length   # noqa: E402
from progen_b200.lib import ProgenError                     # noqa: E402

TINY = dict(num_tokens=256, dim=128, seq_len=128, depth=2, window_size=64, heads=2, dim_head=64, global_mlp_depth=1)


def _case(seed, B=3, n=7, V=12):
    rng = np.random.default_rng(seed)
    s, z = rng.standard_normal((B, n, V)) * 2, rng.standard_normal((B, n, V)) * 3
    labels = rng.integers(1, V, (B, n))
    labels[0, 4:] = 0                                       # counted: 0..4
    labels[1, 0:] = 0                                       # counted: position 0 only
    labels[2, 5] = V + 7                                    # clamped to V - 1
    return s, z, labels


@pytest.mark.parametrize('tau,alpha', [(0.5, 0.0), (1.0, 0.3), (2.0, 0.5), (4.0, 1.0), (3.0, 0.9)])
def test_oracle_gradient_matches_finite_differences(tau, alpha):
    s, z, labels = _case(1)
    loss, grad, _ = distill_head(s, z, labels, tau, alpha)
    rng = np.random.default_rng(2)
    eps = 1e-6
    for _ in range(40):
        idx = tuple(rng.integers(0, k) for k in s.shape)
        sp, sm = s.copy(), s.copy()
        sp[idx] += eps
        sm[idx] -= eps
        fd = (distill_head(sp, z, labels, tau, alpha)[0] - distill_head(sm, z, labels, tau, alpha)[0]) / (2 * eps)
        assert abs(fd - grad[idx]) < 1e-7 + 1e-6 * abs(fd), (idx, fd, grad[idx])
    m = loss_mask(labels)
    assert np.all(grad[m == 0] == 0.0)


def test_alpha_one_is_the_reference_cross_entropy_mean():
    from oracle import progen_torch as T
    s, z, labels = _case(3)
    loss, grad, stats = distill_head(s, z, labels, 2.0, 1.0)
    ref = T.cross_entropy(torch.tensor(s), torch.tensor(np.clip(labels, 0, s.shape[-1] - 1)))
    assert np.allclose(stats[:, 1], ref.numpy(), rtol=1e-12, atol=1e-12)
    assert abs(loss - float(ref.mean())) < 1e-12


def test_tau_squared_convention():
    s, z, labels = _case(4)
    m = loss_mask(labels)
    for tau in (0.5, 1.0, 4.0):
        loss, grad, stats = distill_head(s, z, labels, tau, 0.0)
        assert abs(loss - tau ** 2 * stats[:, 0].mean()) < 1e-12
    # at a large temperature, tau (softmax(s / tau) - softmax(z / tau)) tends to ((s - z) - mean(s - z)) / V: the
    # tau^2 factor keeps the gradient's scale independent of tau (Hinton et al. 2015)
    tau, V = 1e4, s.shape[-1]
    _, grad, _ = distill_head(s, z, labels, tau, 0.0)
    c = m.sum(-1)
    w = (m / c[:, None] / s.shape[0])[..., None]
    dz = s - z
    limit = w * (dz - dz.mean(-1, keepdims=True)) / V
    assert np.abs(grad - limit).max() < 1e-3 * np.abs(limit).max()      # the next term is O(|s - z| / tau)


def test_refusals():
    for tau in (0.0, -1.0, float('nan'), float('inf'), 1e-40, 'x', True):
        with pytest.raises(ProgenError, match='temperature'):
            check_objective(tau, 0.5)
    for alpha in (-0.1, 1.5, float('nan'), True):
        with pytest.raises(ProgenError, match='alpha'):
            check_objective(2.0, alpha)
    assert check_objective(2, 1) == (2.0, 1.0)
    student = ProGen(**TINY)
    with pytest.raises(ProgenError, match='the student model itself'):
        check_teacher(student, student)
    with pytest.raises(ProgenError, match='vocabulary'):
        check_teacher(student, ProGen(**dict(TINY, num_tokens=128)))
    with pytest.raises(ProgenError, match="seq_len \\(64\\) is below"):
        check_teacher(student, ProGen(**dict(TINY, seq_len=64)))
    check_teacher(student, ProGen(**dict(TINY, seq_len=192, dim=256, depth=3)))
    # the API refuses before any device work: no engine exists afterwards
    data = np.ones((2, TINY['seq_len'] + 1), np.int64)
    with pytest.raises(ProgenError, match='the student model itself'):
        student.distill_loss_and_grad(None, data, teacher=student, teacher_params=None)
    with pytest.raises(ProgenError, match='alpha'):
        student.distill_loss_and_grad(None, data, teacher=ProGen(**TINY), teacher_params=None, alpha=2.0)
    with pytest.raises(ProgenError, match='vocabulary'):
        student.trainer(None, teacher=ProGen(**dict(TINY, num_tokens=128)), teacher_params={})
    with pytest.raises(ProgenError, match='teacher_params'):
        student.trainer(None, teacher=ProGen(**TINY))
    assert student._engine is None


def test_teacher_length_rule():
    assert teacher_length(128, 1024) == 128
    assert teacher_length(384, 512) == 384
    assert teacher_length(512, 512) == 512
    assert teacher_length(256, 256) == 256
    # the student's full length is not a valid teacher length: the smallest valid one above it
    assert teacher_length(96, 200) == 128
    assert teacher_length(96, 100) == 100
    assert teacher_length(200, 300) == 256
    assert teacher_length(200, 230) == 230
    for L in range(1, 400):
        for tn in (L, L + 1, L + 37, 512, 1024):
            if tn < L:
                continue
            t = teacher_length(L, tn)
            assert L <= t <= tn and (t == tn or t % 128 == 0)
            assert all(not (c == tn or c % 128 == 0) for c in range(L, t)), (L, tn, t)


# ------------------------------------------------------------------------------------------------ train.py
def _package(path, cfg, params=None, **extra):
    from progen_b200.checkpoint import get_checkpoint_fns
    pkg = {'next_seq_index': 0, 'params': ProGen(**cfg).init(0) if params is None else params, 'optim_state': None,
           'model_config': dict(cfg), 'run_id': None}
    pkg.update(extra)
    get_checkpoint_fns(path)[2](pkg)


class _Stop(Exception):
    pass


def _run(monkeypatch, args, seen=None):
    """train.py with args; the Trainer stand-in records its keywords and stops before any device work"""
    from click.testing import CliRunner
    import train

    def trainer(self, params, **kw):
        if seen is not None:
            seen.append(kw)
        raise _Stop
    monkeypatch.setattr(ProGen, 'trainer', trainer)
    return CliRunner().invoke(train.main, args)


def test_train_flags_and_resume_refusals(tmp_path, monkeypatch):
    import toml
    (tmp_path / 'tiny.toml').write_text(toml.dumps(TINY))
    _package(tmp_path / 'teacher', dict(TINY, dim=256, seq_len=192))
    base = ['--config_path', str(tmp_path), '--model_name', 'tiny', '--synthetic']
    res = _run(monkeypatch, base + ['--checkpoint_path', str(tmp_path / 'a'), '--distill_alpha', '0.2'])
    assert res.exit_code == 2 and 'need --teacher_checkpoint' in res.output
    res = _run(monkeypatch, base + ['--checkpoint_path', str(tmp_path / 'a'), '--teacher_checkpoint', str(tmp_path / 'teacher'),
                                    '--distill_temperature', '0'])
    assert res.exit_code == 2 and 'temperature must be finite' in res.output
    res = _run(monkeypatch, base + ['--checkpoint_path', str(tmp_path / 'a'), '--teacher_checkpoint', str(tmp_path / 'none')])
    assert res.exit_code == 2 and 'no checkpoint found' in res.output
    _package(tmp_path / 'small_vocab', dict(TINY, num_tokens=128))
    res = _run(monkeypatch, base + ['--checkpoint_path', str(tmp_path / 'a'), '--teacher_checkpoint',
                                    str(tmp_path / 'small_vocab')])
    assert isinstance(res.exception, ProgenError) and 'vocabulary' in str(res.exception)
    seen = []
    res = _run(monkeypatch, base + ['--checkpoint_path', str(tmp_path / 'a'), '--teacher_checkpoint', str(tmp_path / 'teacher'),
                                    '--distill_temperature', '3', '--mixed_precision'], seen)
    assert isinstance(res.exception, _Stop), res.output
    kw = seen.pop()
    assert kw['teacher'].config['dim'] == 256 and kw['teacher'].mixed_precision
    assert kw['teacher_params'][next(iter(kw['teacher_params']))]['embeddings'].shape == (256, 256)
    # resumed distillation runs: flags that disagree with the package are refused
    from progen_b200.checkpoint import last_checkpoint_file
    tfile = last_checkpoint_file(tmp_path / 'teacher')
    _package(tmp_path / 'run', TINY, distill=dict(teacher_checkpoint=tfile, temperature=3.0, alpha=0.5))
    resume = ['--checkpoint_path', str(tmp_path / 'run')]
    for flags, msg in ((['--distill_temperature', '2'], 'distils at temperature 3.0'),
                       (['--distill_alpha', '0.1'], 'distils with alpha 0.5'),
                       (['--teacher_checkpoint', str(tmp_path / 'small_vocab')], 'the teacher of the run')):
        res = _run(monkeypatch, resume + flags)
        assert res.exit_code == 2 and msg in res.output, (flags, res.output)
    seen = []
    res = _run(monkeypatch, resume + ['--distill_temperature', '3.0', '--teacher_checkpoint', str(tmp_path / 'teacher')], seen)
    assert isinstance(res.exception, _Stop), res.output
    assert seen.pop()['teacher'].config['dim'] == 256
    # a run without a teacher is not switched to distillation
    _package(tmp_path / 'plain', TINY)
    res = _run(monkeypatch, ['--checkpoint_path', str(tmp_path / 'plain'), '--teacher_checkpoint', str(tmp_path / 'teacher')])
    assert res.exit_code == 2 and 'without a teacher' in res.output
    seen = []
    res = _run(monkeypatch, ['--checkpoint_path', str(tmp_path / 'plain')], seen)
    assert isinstance(res.exception, _Stop) and seen.pop()['teacher'] is None


def test_package_round_trip(tmp_path):
    """a student package carries `distill` beside plain params; package_params and the loaders read it unchanged"""
    from progen_b200.checkpoint import get_checkpoint_fns, package_params
    params = ProGen(**TINY).init(3)
    d = dict(teacher_checkpoint='/x/ckpt_1.pkl', temperature=2.0, alpha=0.5)
    _package(tmp_path / 'st', TINY, params=params, distill=d)
    pkg = get_checkpoint_fns(tmp_path / 'st')[1]()
    assert pkg['distill'] == d and pkg['model_config'] == TINY
    got = package_params(pkg)
    for m, leaves in params.items():
        for k, v in leaves.items():
            assert np.array_equal(got[m][k], v)


# ------------------------------------------------------------------------------------------------ unchanged launches
def test_existing_objectives_make_the_parent_launches(monkeypatch):
    """every LM, preference, property and residue step (full / LoRA, fp32 / bf16, full / cut length, resident /
    recompute) makes the launches it made before distillation existed, argument for argument"""
    from launch_recorder import digest, record_steps
    want = json.load(open(os.path.join(HERE, 'golden', 'train_launches.json')))
    got = {k: digest(v) for k, v in record_steps(monkeypatch).items()}
    assert set(got) == set(want)
    assert [k for k in want if got[k] != want[k]] == []
