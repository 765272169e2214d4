"""Preference (DPO) fine-tuning on the GPU: the head's sums are `score`'s, step 0 is exactly ln 2, loss and gradient
against the float64 reference (tests/preference_oracle.py), the Trainer against the oracle optimizer chain, graph
replay against the eager loop, data parallel against one process, and the dpo.py CLI."""
import json
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import progen_ref as O
from oracle import progen_torch as T
from preference_oracle import preference_loss_and_grads

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

BASE = dict(num_tokens=256, dim=128, seq_len=128, depth=2, window_size=64, heads=2, dim_head=64)
CONFIGS = {
    'glu': dict(BASE, global_mlp_depth=0),
    'gelu': dict(BASE, global_mlp_depth=0, ff_glu=False),
    'gmlp': dict(BASE, global_mlp_depth=2),
}


def _pairs(P, n, seed):
    rng = np.random.default_rng(seed)
    c = rng.integers(1, 256, (P, n + 1)).astype(np.uint16)
    r = rng.integers(1, 256, (P, n + 1)).astype(np.uint16)
    c[0, n // 3:] = 0                                   # rows that end early; the others have no padding
    r[min(1, P - 1), n // 2:] = 0
    if P > 2:
        r[2, 7:] = 0
    return c, r


def _setup(name, mp, P=3, seed=0):
    from progen_b200 import ProGen
    kw = CONFIGS[name]
    cfg = O.make_config(**kw)
    params = O.randomize_params(O.init_params(cfg, 3 + seed), 4 + seed)
    c, r = _pairs(P, kw['seq_len'], 5 + seed)
    return ProGen(**kw, mixed_precision=mp), cfg, params, c, r


def _perturbed(params, scale, seed):
    rng = np.random.default_rng(seed)
    return {m: {k: (v + scale * np.abs(v).mean() * rng.standard_normal(v.shape)).astype(np.float32) for k, v in d.items()}
            for m, d in params.items()}


@pytest.mark.parametrize('name', sorted(CONFIGS))
@pytest.mark.parametrize('mp', [False, True])
def test_stats_are_score_and_step_zero_is_ln2(name, mp):
    """policy log-likelihoods are bitwise `score`'s; with references scored at the same parameters every margin is 0.0"""
    model, cfg, params, c, r = _setup(name, mp)
    ref_c = model.score(params, c)['log_likelihood']
    ref_r = model.score(params, r)['log_likelihood']
    loss, grads, st = model.preference_loss_and_grad(params, c, r, ref_c, ref_r, beta=0.1)
    np.testing.assert_array_equal(st['policy_chosen'], ref_c)
    np.testing.assert_array_equal(st['policy_rejected'], ref_r)
    np.testing.assert_array_equal(st['margin'], np.zeros(3, np.float32))
    np.testing.assert_array_equal(st['loss'], np.full(3, np.float32(math.log(2))))
    assert abs(loss - math.log(2)) < 1e-6, loss
    assert all(np.isfinite(g).all() for d in grads.values() for g in d.values())


@pytest.mark.parametrize('name', sorted(CONFIGS))
def test_fp32_loss_and_grad_match_float64(name):
    model, cfg, params, c, r = _setup(name, False, seed=1)
    ref_params = _perturbed(params, 0.02, 9)
    _, _, ref_st = preference_loss_and_grads(ref_params, c, r, np.zeros(3), np.zeros(3), cfg, 0.1)
    ref_c, ref_r = ref_st['policy_chosen'].astype(np.float32), ref_st['policy_rejected'].astype(np.float32)
    o_loss, o_grads, o_st = preference_loss_and_grads(params, c, r, ref_c, ref_r, cfg, 0.1)
    loss, grads, st = model.preference_loss_and_grad(params, c, r, ref_c, ref_r, beta=0.1)
    assert np.ptp(o_st['margin']) > 1e-2, o_st['margin']           # the margins spread
    assert abs(loss - o_loss) < 1e-5, (loss, o_loss)
    np.testing.assert_allclose(st['margin'], o_st['margin'], atol=1e-4)
    for m, d in o_grads.items():
        for k, g in d.items():
            scale = max(1e-8, np.abs(g).max())
            assert np.abs(grads[m][k] - g).max() < 2e-4 * scale + 1e-7, (m, k, np.abs(grads[m][k] - g).max(), scale)


@pytest.mark.parametrize('name', ['glu', 'gelu'])
def test_bf16_loss_and_grad_vs_float64(name):
    model, cfg, params, c, r = _setup(name, True, seed=2)
    ref_params = _perturbed(params, 0.02, 10)
    _, _, ref_st = preference_loss_and_grads(ref_params, c, r, np.zeros(3), np.zeros(3), cfg, 0.1)
    ref_c, ref_r = ref_st['policy_chosen'].astype(np.float32), ref_st['policy_rejected'].astype(np.float32)
    o_loss, o_grads, _ = preference_loss_and_grads(params, c, r, ref_c, ref_r, cfg, 0.1)
    loss, grads, _ = model.preference_loss_and_grad(params, c, r, ref_c, ref_r, beta=0.1)
    assert abs(loss - o_loss) < 3e-2, (loss, o_loss)
    for m, d in o_grads.items():
        for k, g in d.items():
            rel = np.abs(grads[m][k] - g).max() / max(1e-8, np.abs(g).max())
            assert rel < 0.12, (m, k, rel)


def test_bf16_one_pair_at_the_config2_stack():
    """ref (float64) / emu (fp32, bf16-rounded operands) / cuda at config 2's layer stack, with the 2x bounds of
    test_gpu_model.test_bf16_parity_at_benchmarked_shapes"""
    from progen_b200 import ProGen
    torch.set_num_threads(max(1, min(32, len(os.sched_getaffinity(0)))))
    kw = dict(num_tokens=256, dim=512, seq_len=1024, depth=12, heads=8, dim_head=64, window_size=256, global_mlp_depth=2)
    cfg = O.make_config(**kw)
    params = O.init_params(cfg, 21)
    c, r = _pairs(1, 1024, 22)
    model = ProGen(**kw, mixed_precision=True)
    sc = model.score(params, np.concatenate([c, r]))['log_likelihood']
    ref_c, ref_r = sc[:1] + np.float32(2.0), sc[1:] - np.float32(3.0)           # z = -0.5
    ref = preference_loss_and_grads(params, c, r, ref_c, ref_r, cfg, 0.1)
    emu = preference_loss_and_grads(params, c, r, ref_c, ref_r, cfg, 0.1, dtype=torch.float32, operand_round=T.bf16_round)
    loss, grads, _ = model.preference_loss_and_grad(params, c, r, ref_c, ref_r, beta=0.1)
    print(dict(ref=ref[0], emu=emu[0], cuda=loss))
    assert abs(loss - emu[0]) <= 2 * abs(emu[0] - ref[0]) + 2e-3, (loss, emu[0], ref[0])
    bad = []
    for m, d in ref[1].items():
        for k, g in d.items():
            den = max(1e-30, float(np.linalg.norm(g)))
            e_l2 = float(np.linalg.norm(emu[1][m][k] - g)) / den
            ce_l2 = float(np.linalg.norm(grads[m][k] - emu[1][m][k])) / den
            if ce_l2 > 2.0 * e_l2 + 1e-3:
                bad.append((m, k, e_l2, ce_l2))
    assert not bad, bad[:5]


def _ref_lls(model, params, c, r, seed):
    """reference log-likelihoods near the policy's, so that the margins spread without saturating"""
    sc = model.score(params, np.concatenate([c, r]))['log_likelihood']
    noise = np.random.default_rng(seed).normal(0, 3, sc.shape).astype(np.float32)
    P = len(c)
    return sc[:P] + noise[:P], sc[P:] + noise[P:]


@pytest.mark.parametrize('mp', [False, True])
def test_trainer_preference_steps_match_oracle_optimizer(mp):
    """8 micro-steps (clip -> adamw(mask) -> apply_every(4)) against the oracle chain, with the bounds of
    test_gpu_model.test_trainer_steps_match_oracle_optimizer"""
    from progen_b200 import ProGen
    kw = dict(BASE, global_mlp_depth=1)
    cfg = O.make_config(**kw)
    params = O.randomize_params(O.init_params(cfg, 7), 8)
    model = ProGen(**kw, mixed_precision=mp)
    batches = []
    for s in range(8):
        c, r = _pairs(2, 128, 40 + s)
        batches.append((c, r) + _ref_lls(model, params, c, r, 60 + s))
    tr = model.trainer(params, grad_accum_every=4, learning_rate=1e-2)
    st = O.optim_init(params, every=4)
    cur = params
    for step, (c, r, rc, rr) in enumerate(batches):
        loss = float(tr.preference_step(c, r, rc, rr, beta=0.1).item())
        ref_loss, grads, _ = preference_loss_and_grads(cur, c, r, rc, rr, cfg, 0.1)
        cur, _ = O.optim_step(cur, {m: {k: v.astype(np.float32) for k, v in d.items()} for m, d in grads.items()}, st, lr=1e-2)
        assert abs(loss - ref_loss) < (3e-2 if mp else 2e-5), (step, loss, ref_loss)
    got = tr.params()
    worst = max(float(np.abs(got[m][k] - v).max()) for m, d in cur.items() for k, v in d.items())
    assert worst < (5e-2 if mp else 2e-3), worst


def _run(model_kw, mp, params, plan, cuda_graph):
    """plan: list of ('pref', c, r, rc, rr) / ('step', rows) -> (losses, stats of the preference steps, final params)"""
    from progen_b200 import ProGen
    tr = ProGen(**model_kw, mixed_precision=mp).trainer(params, grad_accum_every=4, learning_rate=1e-2, cuda_graph=cuda_graph)
    losses, stats, keys = [], [], []
    for item in plan:
        if item[0] == 'pref':
            losses.append(float(tr.preference_step(*item[1:], beta=0.1).item()))
            stats.append(tr.preference_stats())
        else:
            losses.append(float(tr.step(item[1]).item()))
        keys.append(None if tr._graph is None else tr._graph_key)
    return losses, stats, tr.params(), keys


@pytest.mark.parametrize('mp', [False, True])
def test_graph_replay_matches_eager(mp):
    """Two eager steps, then replays.  Until the first apply_every emit (4 steps) both loops see the same parameters, so
    their losses and stats are bitwise equal; the final parameters agree within the bounds of
    test_gpu_model.test_trainer_cuda_graph_replay_matches_eager (the LayerNorm-scale and split-K weight gradients are summed
    with float atomics, in an order that varies from run to run)."""
    kw = dict(BASE, global_mlp_depth=1)
    cfg = O.make_config(**kw)
    params = O.randomize_params(O.init_params(cfg, 11), 12)
    from progen_b200 import ProGen
    probe = ProGen(**kw, mixed_precision=mp)
    plan = []
    for s in range(7):
        c, r = _pairs(2, 128, 80 + s)
        plan.append(('pref', c, r) + _ref_lls(probe, params, c, r, 90 + s))
    el, es, ep, _ = _run(kw, mp, params, plan, False)
    gl, gs, gp, keys = _run(kw, mp, params, plan, True)
    assert keys[1] is not None and keys[1][2:] == ('preference', 0.1), keys     # captured after two eager steps
    assert el[:4] == gl[:4], (el, gl)
    for a, b in zip(es[:4], gs[:4]):
        for k in a:
            np.testing.assert_array_equal(a[k], b[k], err_msg=k)
    np.testing.assert_allclose(gl, el, rtol=0, atol=2e-2 if mp else 2e-5)
    worst = max(float(np.abs(gp[m][k] - v).max()) for m, d in ep.items() for k, v in d.items())
    assert worst < (5e-2 if mp else 2e-3), worst


@pytest.mark.parametrize('mp', [False, True])
def test_step_and_preference_step_interleaved(mp):
    """one trainer runs plain and preference steps; with cuda_graph each kind is captured in turn and the results are
    those of the eager loop"""
    kw = dict(BASE, global_mlp_depth=1)
    cfg = O.make_config(**kw)
    params = O.randomize_params(O.init_params(cfg, 13), 14)
    from progen_b200 import ProGen
    probe = ProGen(**kw, mixed_precision=mp)
    rng = np.random.default_rng(15)
    plan = []
    for kind in ['pref'] * 3 + ['step'] * 3 + ['pref', 'step', 'pref', 'pref', 'pref']:
        if kind == 'pref':
            c, r = _pairs(2, 128, int(rng.integers(1 << 30)))
            plan.append(('pref', c, r) + _ref_lls(probe, params, c, r, int(rng.integers(1 << 30))))
        else:
            plan.append(('step', rng.integers(0, 256, (4, 129)).astype(np.uint16)))   # 4 rows: the preference shape
    el, _, ep, _ = _run(kw, mp, params, plan, False)
    gl, _, gp, keys = _run(kw, mp, params, plan, True)
    assert keys[2] is not None and keys[2][2] == 'preference' and keys[5] == (4, 4), keys
    np.testing.assert_allclose(gl, el, rtol=0, atol=2e-2 if mp else 2e-5)
    worst = max(float(np.abs(gp[m][k] - v).max()) for m, d in ep.items() for k, v in d.items())
    assert worst < (5e-2 if mp else 2e-3), worst


@pytest.mark.parametrize('mp', [False, True])
def test_two_rank_preference_equals_single_process(mp, tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip('needs two GPUs')
    port = 29700 + os.getpid() % 1000
    env = dict(os.environ, DDP_TEST_MP='1' if mp else '0', NCCL_DEBUG='WARN')
    r = subprocess.run([sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node', '2', '--master-addr',
                        '127.0.0.1', '--master-port', str(port), os.path.join(ROOT, 'tests', 'ddp_preference_worker.py')],
                       capture_output=True, text=True, env=env, timeout=240)
    line = next((l for l in r.stdout.splitlines() if l.startswith('DDP_RESULT ')), None)
    assert line is not None, r.stdout[-2000:] + r.stderr[-4000:]
    res = json.loads(line[len('DDP_RESULT '):])
    for case, v in res.items():                         # the bounds of test_gpu_ddp.py
        assert abs(v['loss_ddp'] - v['loss_single']) < (2e-3 if mp else 1e-5), (case, v)
        assert v['grad_rel_l2'] < (1e-3 if mp else 1e-5), (case, v)
    assert res['one_pair_idle_rank']['shard_pairs'] == 1


def test_dpo_cli_runs_and_resumes(tmp_path):
    from progen_b200 import ProGen
    from progen_b200.checkpoint import get_checkpoint_fns
    kw = dict(num_tokens=256, dim=128, seq_len=128, depth=2, window_size=64, global_mlp_depth=1, heads=2, dim_head=64,
              ff_mult=4, ff_glu=True, attn_dim=None, clamp_gate=True, shift_tokens=True)
    init = tmp_path / 'init'
    get_checkpoint_fns(init)[2]({'next_seq_index': 0, 'params': ProGen(**kw).init(0), 'optim_state': None,
                                 'model_config': kw, 'run_id': None})
    rng = np.random.default_rng(0)
    aa = 'ACDEFGHIKLMNPQRSTVWY'
    seq = lambda: ''.join(rng.choice(list(aa), int(rng.integers(20, 60))))
    pairs = tmp_path / 'pairs.tsv'
    pairs.write_text(''.join(f'{seq()}\t{seq()}\n' + ('\n' if i == 2 else '') for i in range(6)))
    out = tmp_path / 'dpo'
    cmd = [sys.executable, os.path.join(ROOT, 'dpo.py'), '--init_checkpoint', str(init), '--pairs', str(pairs),
           '--checkpoint_path', str(out), '--batch_pairs', '2', '--learning_rate', '1e-4']
    r = subprocess.run(cmd, capture_output=True, text=True, cwd=tmp_path, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    steps = [l for l in r.stdout.splitlines() if l.startswith('step ')]
    assert len(steps) == 3, r.stdout
    assert 'loss 0.693147 ' in steps[0] and 'margin 0.000000 ' in steps[0], steps[0]
    ck = get_checkpoint_fns(out)[1]()
    assert ck['next_pair_index'] == 6 and ck['optim_state']['count'] == 3
    r2 = subprocess.run(cmd + ['--epochs', '2'], capture_output=True, text=True, cwd=tmp_path, timeout=600)
    assert r2.returncode == 0, r2.stdout[-2000:] + r2.stderr[-4000:]
    assert 'starting from pair 6' in r2.stdout, r2.stdout
    steps2 = [l for l in r2.stdout.splitlines() if l.startswith('step ')]
    assert len(steps2) == 3 and steps2[0].startswith('step 0 epoch 1 pairs 6-7:'), steps2
    assert get_checkpoint_fns(out)[1]()['next_pair_index'] == 12
