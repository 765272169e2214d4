"""Per-residue fine-tuning on the GPU: `progen_residue_head` and `progen_residue_head_wgrad` against float64 of their own
inputs (fp32 and bf16 h, C in {1, 3, 8, 64}, d in {64, 512, 1536}, both tasks), bitwise repeatable, a position's
prediction bitwise the same alone and in a batch, dy exactly +0.0 on unlabelled rows; the residue step's loss, adapter and
head gradients against the float64 reference (tests/residue_oracle.py) in fp32 and by the three-way bf16 rule; the cut
step against the full-length one; the trainer's captured steps against eager ones with a bitwise frozen base and separate
graphs per objective; `predict_residues` across batch sizes and against the step; fitness.py --level residue end to end."""
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from oracle import progen_ref as O                      # noqa: E402
from oracle import progen_torch as T                    # noqa: E402
from property_oracle import HEAD                        # noqa: E402
from residue_oracle import residue_loss_and_grads      # noqa: E402

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

BASE = dict(num_tokens=256, dim=128, seq_len=256, depth=2, window_size=64, heads=2, dim_head=64)
CONFIGS = {
    'glu': dict(BASE, global_mlp_depth=0),
    'gelu': dict(BASE, global_mlp_depth=0, ff_glu=False, shift_tokens=False),
    'sgu': dict(BASE, global_mlp_depth=1),
}


# ------------------------------------------------------------------------------------------------ kernels
def _launch(L, h, w, b, B, Ln, task, y, cls, train=True):
    """progen_residue_head (+ wgrad when training) on h [B*Ln, d] -> dict of device outputs"""
    d, C = w.shape
    T_ = B * Ln
    F = lambda *s: torch.full(s, float('nan'), device='cuda')
    out = dict(pred=F(T_, C), pos_loss=F(T_), loss=F(1), dpred=F(T_, C), dw=F(d, C), db=F(C),
               count=torch.full((1,), -7, device='cuda', dtype=torch.int32),
               dy=torch.full((T_, d), float('nan'), device='cuda', dtype=h.dtype))
    p = lambda k: out[k].data_ptr() if train else 0
    yp = y.data_ptr() if (train and y is not None) else 0
    cp = cls.data_ptr() if (train and cls is not None) else 0
    lib = L.load()
    L.check(lib.progen_residue_head(h.data_ptr(), d, L.dt(h), w.data_ptr(), b.data_ptr(), B, Ln, d, C, task, yp, cp,
                                    out['pred'].data_ptr(), p('pos_loss'), p('count'), p('loss'), p('dpred'), p('dy'), d,
                                    L.stream()), 'residue_head')
    if train:
        ws = torch.full((B * (d + 1) * C,), float('nan'), device='cuda')
        L.check(lib.progen_residue_head_wgrad(h.data_ptr(), d, L.dt(h), out['dpred'].data_ptr(), yp, cp, B, Ln, d, C,
                                              ws.data_ptr(), out['dw'].data_ptr(), out['db'].data_ptr(), L.stream()), 'wgrad')
    torch.cuda.synchronize()
    return out


def _kernel_case(task, C, d, dtype, B, Ln, seed):
    rng = np.random.default_rng(seed)
    h = torch.tensor(rng.standard_normal((B * Ln, d)), dtype=torch.float32, device='cuda').to(dtype)
    w = torch.tensor(rng.standard_normal((d, C)) * d ** -0.5, dtype=torch.float32, device='cuda')
    b = torch.tensor(rng.standard_normal(C) * 0.1, dtype=torch.float32, device='cuda')
    lab = rng.random((B, Ln)) < 0.6
    lab[:, 0] = False
    lab[1 % B] = False                              # a row without labels
    lab[0, Ln - 1] = True                           # a labelled last position
    lab = lab.reshape(-1)
    if task == 'regression':
        y = np.where(lab[:, None], rng.standard_normal((B * Ln, C)), np.nan)
        return h, w, b, lab, torch.tensor(y, dtype=torch.float32, device='cuda'), None, y
    cls = np.where(lab, rng.integers(0, C, B * Ln), -1)
    return h, w, b, lab, None, torch.tensor(cls, dtype=torch.int32, device='cuda'), cls


@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
@pytest.mark.parametrize('d', [64, 512, 1536])
@pytest.mark.parametrize('task, C', [('regression', 1), ('regression', 3), ('regression', 8), ('regression', 64),
                                     ('classification', 3), ('classification', 8), ('classification', 64)])
def test_residue_kernels_match_float64(task, C, d, dtype):
    from progen_b200 import lib as L
    L.require_device()
    B, Ln = (16, 1024) if (d, C) == (512, 3) else (4, 96)       # one case at 16 384 rows
    h, w, b, lab, y, cls, targ = _kernel_case(task, C, d, dtype, B, Ln, C * 131 + d)
    code = L.TASK_REGRESSION if task == 'regression' else L.TASK_CLASSIFICATION
    out = _launch(L, h, w, b, B, Ln, code, y, cls)
    h64 = h.float().cpu().double().numpy()
    w64, b64 = w.cpu().double().numpy(), b.cpu().double().numpy()
    p = h64 @ w64 + b64
    N = int(lab.sum())
    if task == 'regression':
        yl = np.nan_to_num(np.asarray(targ, np.float32).astype(np.float64))
        row = np.where(lab, ((p - yl) ** 2).mean(-1), 0.0)
        dp = np.where(lab[:, None], 2 * (p - yl) / C / N, 0.0)
    else:
        m = p.max(-1, keepdims=True)
        lse = (m + np.log(np.exp(p - m).sum(-1, keepdims=True)))[:, 0]
        t = np.clip(targ, 0, C - 1)
        row = np.where(lab, lse - p[np.arange(len(p)), t], 0.0)
        dp = np.where(lab[:, None], (np.exp(p - lse[:, None]) - np.eye(C)[t]) / N, 0.0)
    want = dict(pred=p, pos_loss=row, loss=[row.sum() / N], dpred=dp, dw=h64[lab].T @ dp[lab], db=dp[lab].sum(0),
                dy=dp @ w64.T)
    assert int(out['count'].item()) == N
    for k, v in want.items():
        v = np.asarray(v, np.float64)
        got = out[k].float().cpu().numpy().astype(np.float64).reshape(v.shape)
        # fp32 sums of up to 16 384 terms; dy is rounded once to its dtype
        rel = 1e-2 if (k == 'dy' and dtype == torch.bfloat16) else 2e-5
        tol = rel * max(1e-30, np.abs(v).max()) + (1e-6 * np.sqrt(N) * np.abs(v).max() if k in ('dw', 'db') else 0)
        assert np.abs(got - v).max() <= tol, (k, np.abs(got - v).max(), np.abs(v).max())
    dy = out['dy'].float().cpu()
    assert torch.equal(dy[torch.tensor(~lab)], torch.zeros_like(dy[torch.tensor(~lab)]))
    assert not torch.signbit(dy[torch.tensor(~lab)]).any(), 'unlabelled rows of dy must be +0.0'
    again = _launch(L, h, w, b, B, Ln, code, y, cls)
    assert all(torch.equal(out[k], again[k]) for k in ('pred', 'pos_loss', 'loss', 'dpred', 'dw', 'db', 'count')) and \
        torch.equal(out['dy'].view(torch.int16 if dtype == torch.bfloat16 else torch.int32),
                    again['dy'].view(torch.int16 if dtype == torch.bfloat16 else torch.int32)), 'repeat not bitwise'
    infer = _launch(L, h, w, b, B, Ln, code, y, cls, train=False)
    assert torch.equal(infer['pred'], out['pred'])
    for pos in (0, Ln - 1, B * Ln - 1):                  # one position alone: the same bits as inside the batch
        alone = _launch(L, h[pos:pos + 1].contiguous(), w, b, 1, 1, code, None, None, train=False)
        assert torch.equal(alone['pred'][0], out['pred'][pos])


# ------------------------------------------------------------------------------------------------ model
def _setup(name, mp, task='regression', C=3, rank=16, alpha=32.0, seed=0, B=3, kw=None):
    from progen_b200 import ProGen
    from progen_b200.property import residue_positions
    kw = kw or CONFIGS[name]
    n = kw['seq_len']
    cfg = O.make_config(**kw)
    params = O.randomize_params(O.init_params(cfg, 3 + seed), 4 + seed)
    model = ProGen(**kw, mixed_precision=mp)
    ad = model.init_adapters(seed, rank, alpha=alpha)
    rng = np.random.default_rng(60 + seed)
    for v in ad.values():
        v['lora_b'] = (rng.standard_normal(v['lora_b'].shape) * 0.3 * v['lora_b'].shape[0] ** -0.5).astype(np.float32)
    head = model.init_head(seed, C)
    head[HEAD]['b'] = (rng.standard_normal(C) * 0.1).astype(np.float32)
    rows = rng.integers(1, 256, (B, n + 1)).astype(np.uint16)
    rows[:, 0] = 0
    rows[0, 100:] = 0
    rows[1, 20:] = 0
    rows[2, 200:] = 0
    pos = residue_positions(rows) & (rng.random((B, n)) < 0.7)
    pos[2, 199] = True                                   # the last residue of a row
    if task == 'regression':
        y = np.where(pos[..., None], rng.standard_normal((B, n, C)), np.nan).astype(np.float32)
    else:
        y = np.where(pos, rng.integers(0, C, (B, n)), -1)
    return model, cfg, params, ad, head, rows, y


def _close(got, want, rel=2e-4):
    scale = max(1e-8, float(np.abs(want).max()))
    return float(np.abs(np.asarray(got, np.float64) - want).max()) <= rel * scale + 1e-7


@pytest.mark.parametrize('task', ['regression', 'classification'])
@pytest.mark.parametrize('name', sorted(CONFIGS))
def test_fp32_residue_loss_and_grads_match_float64(name, task):
    model, cfg, params, ad, head, rows, y = _setup(name, False, task, seed=1)
    o_loss, o_grads, o_head, o_pred, _ = residue_loss_and_grads(params, head, rows, y, cfg, task, ad, 2.0)
    loss, grads, hgrads, pred = model.residue_loss_and_grad(params, rows, y, adapters=ad, head=head, task=task,
                                                            lora_alpha=32.0)
    assert abs(loss - o_loss) < 1e-5 * max(1.0, abs(o_loss)), (loss, o_loss)
    assert pred.shape == o_pred.shape
    assert _close(pred[:, :256], o_pred[:, :256], 1e-5)
    for m, d in o_grads.items():
        for k, g in d.items():
            assert _close(grads[m][k], g), (m, k, np.abs(grads[m][k] - g).max(), np.abs(g).max())
    for k in ('w', 'b'):
        assert _close(hgrads[HEAD][k], o_head[HEAD][k]), k


def test_bf16_residue_grads_three_way_at_the_config2_stack():
    """ref (float64) / emu (fp32 with bf16 operands) / cuda at the config-2 layer stack, B = 2: loss, predictions at the
    residues, every adapter gradient and the head gradients, the engine within 2x of emu's distance to ref.  The targets
    are centred at 1, away from the predictions: with zero-mean targets db = sum_t dp_t cancels to a few percent of its
    terms over ~1500 positions, and its relative error then measures that cancellation rather than the engine."""
    from progen_b200 import ProGen
    from progen_b200.property import residue_positions
    assert torch.backends.cuda.matmul.allow_tf32 is False
    kw = dict(num_tokens=256, dim=512, seq_len=1024, depth=12, heads=8, dim_head=64, window_size=256, global_mlp_depth=2)
    cfg = O.make_config(**kw)
    params = O.init_params(cfg, 21)
    model = ProGen(**kw, mixed_precision=True)
    ad = model.init_adapters(3, 16)
    rng = np.random.default_rng(4)
    for v in ad.values():
        v['lora_b'] = (rng.standard_normal(v['lora_b'].shape) * 0.05).astype(np.float32)
    head = model.init_head(5, 3)
    rows = rng.integers(1, 256, (2, 1025)).astype(np.uint16)
    rows[:, 0] = 0
    rows[1, 512:] = 0
    pos = residue_positions(rows)
    y = np.where(pos[..., None], 1.0 + rng.standard_normal((2, 1024, 3)), np.nan).astype(np.float32)
    ref = residue_loss_and_grads(params, head, rows, y, cfg, 'regression', ad, 1.0, device='cuda')
    emu = residue_loss_and_grads(params, head, rows, y, cfg, 'regression', ad, 1.0, dtype=torch.float32,
                                 operand_round=T.bf16_round, device='cuda')
    loss, grads, hgrads, pred = model.residue_loss_and_grad(params, rows, y, adapters=ad, head=head, task='regression')
    rel = lambda a, b: float(np.linalg.norm(np.asarray(a, np.float64) - b) / max(1e-12, np.linalg.norm(b)))
    print('loss', dict(ref=ref[0], emu=emu[0], cuda=loss))
    assert abs(loss - emu[0]) <= 2 * abs(emu[0] - ref[0]) + 2e-3
    pairs = [('pred', pred[pos], emu[3][pos], ref[3][pos])]
    pairs += [(f'{m}/{k}', grads[m][k], emu[1][m][k], ref[1][m][k]) for m in ref[1] for k in ref[1][m]]
    pairs += [(f'head/{k}', hgrads[HEAD][k], emu[2][HEAD][k], ref[2][HEAD][k]) for k in ('w', 'b')]
    rec = {name: (rel(c, np.asarray(e, np.float64)), rel(e, np.asarray(r, np.float64))) for name, c, e, r in pairs}
    print('worst cuda-vs-emu / emu-vs-ref:', max((ce / max(er, 1e-4), name, ce, er) for name, (ce, er) in rec.items()))
    bad = {name: v for name, v in rec.items() if v[0] > 2 * v[1] + 1e-3}
    assert not bad, bad


def _engine_step(model, params, ad, head, rows, y, task, length):
    """one residue step through the engine at an explicit row length -> (loss, adapter grads, head grads, predictions)"""
    from progen_b200 import lib as L
    from progen_b200.property import check_residue_targets, check_rows
    code = L.TASK_REGRESSION if task == 'regression' else L.TASK_CLASSIFICATION
    r = check_rows(rows, model.config['seq_len'], 'test')
    t, _ = check_residue_targets(r, y, task, head[HEAD]['w'].shape[1], 'test')
    model._ensure_loaded(params)
    lo = model._attach_adapters(ad, 32.0, head)
    eng = model.engine
    B = eng.load_residue(r, code, t, length)
    eng.train_step(('residue', code), B, length=length)
    g, hg = lo.split(lo.layout.unpack(lo.grads))
    return float(eng.loss.item()), g, hg, eng.residue_stats(B)['prediction']


@pytest.mark.parametrize('mp', [False, True])
@pytest.mark.parametrize('task', ['regression', 'classification'])
def test_cut_step_matches_full_length(task, mp):
    """rows of at most 200 residues: the step at the cut length 256 of a 512-position model and at 512 give bitwise the
    same loss, predictions and head gradients (the forward at positions < 256 is bitwise, the head reads only labelled
    positions, and its reductions skip the rest in an order that does not depend on L); adapter gradients to round-off"""
    from progen_b200 import ProGen
    kw = dict(CONFIGS['sgu'], seq_len=512)
    _, _, params, ad, head, rows, y = _setup('sgu', mp, task, seed=2, kw=kw)
    model = ProGen(**kw, mixed_precision=mp)
    cut = _engine_step(model, params, ad, head, rows, y, task, 256)
    full = _engine_step(model, params, ad, head, rows, y, task, 512)
    assert cut[0] == full[0]
    assert np.array_equal(cut[3][:, :256], full[3][:, :256]) and not cut[3][:, 256:].any()
    for k in ('w', 'b'):
        assert np.array_equal(cut[2][HEAD][k], full[2][HEAD][k]), k
    tol = 2e-2 if mp else 1e-4
    for m, d in full[1].items():
        for k, g in d.items():
            assert _close(cut[1][m][k], g, tol), (m, k, np.abs(cut[1][m][k] - g).max(), np.abs(g).max())
    via_api = model.residue_loss_and_grad(params, rows, y, adapters=ad, head=head, task=task, lora_alpha=32.0)
    assert via_api[0] == cut[0] and np.array_equal(via_api[3], cut[3])


def _batches(task, C=3, steps=6, seed=9, n=256):
    from progen_b200.property import residue_positions
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(steps):
        r = rng.integers(1, 256, (3, n + 1)).astype(np.uint16)
        r[:, 0] = 0
        r[0, 64:] = 0
        r[1, 120:] = 0
        pos = residue_positions(r) & (rng.random((3, n)) < 0.5)
        y = (np.where(pos[..., None], rng.standard_normal((3, n, C)), np.nan).astype(np.float32) if task == 'regression'
             else np.where(pos, rng.integers(0, C, (3, n)), -1))
        out.append((r, y))
    return out


def _trainer(mp, params, ad, head, task='regression', cuda_graph=False, every=2, lr=1e-2, name='sgu'):
    from progen_b200 import ProGen
    model = ProGen(**CONFIGS[name], mixed_precision=mp)
    return model, model.trainer(params, adapters=ad, head=head, task=task, lora_alpha=32.0, grad_accum_every=every,
                                learning_rate=lr, cuda_graph=cuda_graph)


@pytest.mark.parametrize('task', ['regression', 'classification'])
def test_captured_steps_are_the_eager_ones_and_keep_the_base(task):
    _, _, params, ad, head, _, _ = _setup('sgu', False, task, seed=5)
    batches = _batches(task, seed=10)
    runs = []
    for graph in (False, True):
        _, tr = _trainer(False, params, ad, head, task, cuda_graph=graph)
        base = tr.eng.params.clone()
        losses = [float(tr.residue_step(r, y).item()) for r, y in batches]
        assert torch.equal(tr.eng.params, base), 'the base parameters changed'
        stats = tr.residue_stats()
        assert stats['prediction'].shape == (3, 256, 3) and stats['loss'].shape == (3, 256)
        runs.append((tr, losses))
    (te, el), (tg, gl) = runs
    assert tg._graph is not None and tg._graph_key == (3, 3, 'residue', tg.task)
    assert gl == el, (gl, el)
    for k in ('w', 'b'):
        assert np.array_equal(te.head()[HEAD][k], tg.head()[HEAD][k]), k
    ea, ga = te.adapters(), tg.adapters()
    assert all(np.array_equal(ea[m][k], ga[m][k]) for m in ea for k in ea[m])


def test_residue_property_and_lm_steps_capture_separate_graphs():
    from progen_b200 import lib as L
    _, _, params, ad, head, _, _ = _setup('sgu', False, 'classification', seed=6)
    _, tr = _trainer(False, params, ad, head, 'classification', cuda_graph=True)
    (r, y), = _batches('classification', seed=12, steps=1)
    for _ in range(3):
        tr.residue_step(r, y)
        tr.property_step(r, np.array([0, 1, 2]))
        tr.step(r)
    keys = {k for k, _ in tr._graphs}
    code = L.TASK_CLASSIFICATION
    assert {(3, 3, 'residue', code), (3, 3, 'property', code), (3, 3)} <= keys, keys
    with pytest.raises(L.ProgenError, match='data-parallel residue fine-tuning is not supported'):
        tr.world = 2
        tr.residue_step(r, y)


@pytest.mark.parametrize('mp', [False, True])
def test_predict_residues_batch_independent_and_the_fresh_step(mp):
    """predict_residues is bitwise the same for every batch_size, and with fresh adapters (B = 0) bitwise the residue
    step's predictions at the residues"""
    from progen_b200 import ProGen
    model, cfg, params, _, head, rows, y = _setup('sgu', mp, seed=7, B=5)
    ad = model.init_adapters(1, 16)
    _, _, _, pred = model.residue_loss_and_grad(params, rows, y, adapters=ad, head=head, task='regression')
    fresh = ProGen(**CONFIGS['sgu'], mixed_precision=mp)
    outs = [fresh.predict_residues(params, head, rows, batch_size=bs) for bs in (1, 2, 5, 64)]
    mask = outs[0]['mask']
    assert mask.tolist() == [[t >= 1 and rows[b, t] != 0 for t in range(256)] for b in range(5)]
    for o in outs[1:]:
        assert np.array_equal(o['prediction'], outs[0]['prediction']) and np.array_equal(o['mask'], mask)
    assert np.array_equal(outs[0]['prediction'][mask], pred[mask])
    assert not outs[0]['prediction'][~mask].any()
    part = fresh.predict_residues(params, head, rows[3:4])['prediction']
    assert np.array_equal(part[0], outs[0]['prediction'][3])


def test_refusals():
    from progen_b200 import lib as L
    model, _, params, ad, head, rows, y = _setup('glu', False, seed=8)
    plain = model.trainer(params, adapters=ad)
    with pytest.raises(L.ProgenError, match='no property head'):
        plain.residue_step(rows, y)
    bad = y.copy()
    bad[0, 0] = 1.0
    with pytest.raises(L.ProgenError, match=r'\(0, 0\)'):
        model.residue_loss_and_grad(params, rows, bad, adapters=ad, head=head, task='regression')
    with pytest.raises(L.ProgenError, match='no labelled position'):
        model.residue_loss_and_grad(params, rows, np.full_like(y, np.nan), adapters=ad, head=head, task='regression')


def test_cli_residue_train_resume_predict(tmp_path):
    """a base trained for one step, then fitness.py train --level residue on a task learnable from the residue itself
    (is the residue hydrophobic?): held-out accuracy over 0.95, a resumed run continues at next_index, predict writes one
    line per residue with the class of model.predict_residues"""
    from progen_b200 import ProGen
    from progen_b200.checkpoint import package_params
    from progen_b200.data import collate
    cfg_dir = tmp_path / 'cfg'
    cfg_dir.mkdir()
    (cfg_dir / 'tiny.toml').write_text('num_tokens = 256\ndim = 128\ndepth = 2\ndim_head = 64\nheads = 2\n'
                                       'window_size = 64\nseq_len = 128\nglobal_mlp_depth = 1\n')
    rng = np.random.default_rng(0)
    aa, hyd = 'ACDEFGHIKLMNPQRSTVWY', set('AVILMFWC')
    seqs = [''.join(rng.choice(list(aa), rng.integers(30, 90))) for _ in range(96)]
    label = lambda s: ''.join('h' if c in hyd else ('p' if i % 7 else '.') for i, c in enumerate(s))
    (tmp_path / 'seqs.txt').write_text('\n'.join(seqs) + '\n')
    (tmp_path / 'train.tsv').write_text(''.join(f'{s}\t{label(s)}\n' for s in seqs[:80]))
    (tmp_path / 'valid.tsv').write_text(''.join(f'{s}\t{label(s)}\n' for s in seqs[80:]))
    (tmp_path / 'held.txt').write_text('\n'.join(seqs[80:]) + '\n')
    env = dict(os.environ, PYTHONPATH=ROOT)
    run = lambda *a: subprocess.run([sys.executable, *a], cwd=ROOT, env=env, check=True, capture_output=True, text=True)
    base, fit = tmp_path / 'base', tmp_path / 'fit'
    run('train.py', '--config_path', str(cfg_dir), '--model_name', 'tiny', '--checkpoint_path', str(base), '--num_steps', '1',
        '--text_file', str(tmp_path / 'seqs.txt'), '--batch_size', '2', '--sample_every', '1000', '--validate_every', '1000')
    common = ['--train', str(tmp_path / 'train.tsv'), '--valid', str(tmp_path / 'valid.tsv'), '--checkpoint_path', str(fit),
              '--batch_size', '8', '--learning_rate', '5e-3', '--cuda_graph']
    out = run('fitness.py', 'train', '--init_checkpoint', str(base), '--task', 'classification', '--level', 'residue',
              '--lora_rank', '8', '--epochs', '2', *common)
    assert 'residue level' in out.stdout and 'epoch 1: train loss' in out.stdout, out.stdout
    out = run('fitness.py', 'train', '--epochs', '4', *common)
    assert 'starting from row 160' in out.stdout and 'epoch 3: train loss' in out.stdout, out.stdout
    acc = float(out.stdout.strip().splitlines()[-2].split('valid accuracy ')[1])
    assert acc > 0.95, out.stdout
    pkg = pickle.load(open(sorted(fit.glob('ckpt_*'))[-1], 'rb'))
    assert pkg['next_index'] == 320 and pkg['head']['level'] == 'residue' and pkg['head']['classes'] == ['h', 'p']
    run('fitness.py', 'predict', '--checkpoint_path', str(fit), '--input', str(tmp_path / 'held.txt'),
        '--output', str(tmp_path / 'preds.tsv'))
    lines = (tmp_path / 'preds.tsv').read_text().splitlines()
    assert lines[0] == 'index\tresidue_number\tresidue\tclass\tp_h\tp_p'
    assert len(lines) == 1 + sum(min(len(s), 127) for s in seqs[80:])
    got = [l.split('\t') for l in lines[1:]]
    right = [(f[3] == 'h') == (f[2] in hyd) for f in got]
    assert np.mean(right) > 0.95
    res = ProGen(**pkg['model_config']).predict_residues(package_params(pkg), pkg['head']['params'],
                                                         collate(seqs[80:], 128))
    want = [pkg['head']['classes'][int(res['prediction'][i, t].argmax())] for i in range(16)
            for t in np.flatnonzero(res['mask'][i])]
    assert [f[3] for f in got] == want
