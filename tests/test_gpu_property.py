"""Property fine-tuning on the GPU: `progen_property_head` and `progen_masked_mean_pool_bwd` against float64, bitwise
repeatable; the property step's loss, adapter and head gradients against the float64 reference
(tests/property_oracle.py) in fp32 on every layer kind and by the three-way bf16 rule at the config-2 stack; fresh
adapters give `predict`'s predictions bitwise; after training `predict` on merged parameters has `score`'s embedding
bitwise; the trainer against the oracle optimizer over adapters and head, with a bitwise frozen base and graph replay;
the refusals; the fitness.py train / resume / predict round trip and score.py / generate.py on its package."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from oracle import progen_ref as O                      # noqa: E402
from oracle import progen_torch as T                    # noqa: E402
from property_oracle import HEAD, property_loss_and_grads  # noqa: E402

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

BASE = dict(num_tokens=256, dim=128, seq_len=128, depth=2, window_size=64, heads=2, dim_head=64)
CONFIGS = {
    'glu': dict(BASE, global_mlp_depth=0),
    'gelu': dict(BASE, global_mlp_depth=0, ff_glu=False, shift_tokens=False),
    'sgu': dict(BASE, global_mlp_depth=1),
}


# ------------------------------------------------------------------------------------------------ kernels
def _head_launch(L, emb, w, b, task, y, cls, inv_batch, train=True):
    B, d = emb.shape
    C = w.shape[1]
    F = lambda *s: torch.full(s, float('nan'), device='cuda')
    out = dict(pred=F(B, C), row_loss=F(B), loss=F(1), dpred=F(B, C), dw=F(d, C), db=F(C), demb=F(B, d))
    p = lambda k: out[k].data_ptr() if train else 0
    L.check(L.load().progen_property_head(emb.data_ptr(), w.data_ptr(), b.data_ptr(), B, d, C, task,
                                          y.data_ptr() if (train and y is not None) else 0,
                                          cls.data_ptr() if (train and cls is not None) else 0, inv_batch,
                                          out['pred'].data_ptr(), p('row_loss'), p('loss'), p('dpred'), p('dw'), p('db'),
                                          p('demb'), L.stream()), 'property_head')
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize('d', [128, 520, 1536])
@pytest.mark.parametrize('task, C', [('regression', 1), ('regression', 3), ('regression', 64), ('classification', 2),
                                     ('classification', 3), ('classification', 64)])
def test_property_head_kernel_matches_float64(task, C, d):
    from progen_b200 import lib as L
    L.require_device()
    rng = np.random.default_rng(C * 7 + d)
    B, gb = 5, 8
    emb, w, b = rng.standard_normal((B, d)), rng.standard_normal((d, C)) * d ** -0.5, rng.standard_normal(C) * 0.1
    dev = lambda a, dt=torch.float32: torch.tensor(np.asarray(a), dtype=dt, device='cuda')
    f32 = lambda a: np.asarray(a, np.float32).astype(np.float64)
    e64, w64, b64 = f32(emb), f32(w), f32(b)
    p = e64 @ w64 + b64
    if task == 'regression':
        y = rng.standard_normal((B, C))
        y64 = f32(y)
        row = ((p - y64) ** 2).mean(-1)
        dp = 2 * (p - y64) / C / gb
        args = (dev(y), None)
    else:
        cls = rng.integers(0, C, B)
        m = p.max(-1, keepdims=True)
        lse = (m + np.log(np.exp(p - m).sum(-1, keepdims=True)))[:, 0]
        row = lse - p[np.arange(B), cls]
        dp = (np.exp(p - lse[:, None]) - np.eye(C)[cls]) / gb
        args = (None, dev(cls, torch.int32))
    code = L.TASK_REGRESSION if task == 'regression' else L.TASK_CLASSIFICATION
    out = _head_launch(L, dev(emb), dev(w), dev(b), code, *args, 1.0 / gb)
    want = dict(pred=p, row_loss=row, loss=[row.sum() / gb], dpred=dp, dw=e64.T @ dp, db=dp.sum(0), demb=dp @ w64.T)
    for k, v in want.items():
        v = np.asarray(v, np.float64)
        got = out[k].cpu().numpy().astype(np.float64).reshape(v.shape)
        assert np.abs(got - v).max() <= 1e-5 * max(1.0, np.abs(v).max()), (k, np.abs(got - v).max())
    again = _head_launch(L, dev(emb), dev(w), dev(b), code, *args, 1.0 / gb)
    assert all(torch.equal(out[k], again[k]) for k in out), 'a repeated launch is not bitwise equal'
    infer = _head_launch(L, dev(emb), dev(w), dev(b), code, *args, 1.0 / gb, train=False)
    assert torch.equal(infer['pred'], out['pred']) and torch.isnan(infer['dw']).all()


def test_property_head_kernel_refusals():
    from progen_b200 import lib as L
    L.require_device()
    z = lambda *s: torch.zeros(s, device='cuda')
    lib = L.load()
    for C, task, msg in ((65, L.TASK_REGRESSION, 'the head supports 1..64'), (0, L.TASK_REGRESSION, 'the head supports'),
                         (1, L.TASK_CLASSIFICATION, 'at least 2 classes')):
        w, b, e, p = z(8, max(C, 1)), z(max(C, 1)), z(2, 8), z(2 * max(C, 1))
        rc = lib.progen_property_head(e.data_ptr(), w.data_ptr(), b.data_ptr(), 2, 8, C, task, 0, 0, 1.0, p.data_ptr(),
                                      0, 0, 0, 0, 0, 0, L.stream())
        assert rc != 0 and msg in lib.progen_last_error().decode()


@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
def test_masked_mean_pool_bwd_matches_float64(dtype):
    from progen_b200 import lib as L
    L.require_device()
    B, n, d = 4, 200, 136
    rng = np.random.default_rng(5)
    labels = rng.integers(1, 256, (B, n)).astype(np.int32)
    labels[1, 50:] = 0                      # a row that ends early: positions 0..50 count
    labels[2, :] = 0                        # a row padded from its first label: position 0 alone counts
    labels[3, 30] = 0                       # a pad inside a row: every non-pad label and the first pad count
    mask = labels != 0
    mask |= (np.cumsum(~mask, 1) == 1) & ~mask
    count = mask.sum(1)
    demb = rng.standard_normal((B, d)).astype(np.float32)
    want = np.where(mask[..., None], demb[:, None, :] / count[:, None, None].astype(np.float32), 0).astype(np.float32)
    lab = torch.tensor(labels, device='cuda')
    g = torch.tensor(demb, device='cuda')
    outs = []
    for _ in range(2):
        dy = torch.full((B * n, d), float('nan'), device='cuda', dtype=dtype)
        L.check(L.load().progen_masked_mean_pool_bwd(g.data_ptr(), lab.data_ptr(), dy.data_ptr(), d, L.dt(dy), B, n, d,
                                                     L.stream()), 'pool_bwd')
        torch.cuda.synchronize()
        outs.append(dy)
    assert torch.equal(outs[0], outs[1])
    assert torch.equal(outs[0].float().cpu(), torch.tensor(want).reshape(B * n, d).to(dtype).float())
    assert count.tolist()[1:3] == [51, 1]


# ------------------------------------------------------------------------------------------------ model
def _setup(name, mp, task='regression', C=3, rank=16, alpha=32.0, seed=0, B=3):
    from progen_b200 import ProGen
    kw = CONFIGS[name]
    cfg = O.make_config(**kw)
    params = O.randomize_params(O.init_params(cfg, 3 + seed), 4 + seed)
    model = ProGen(**kw, mixed_precision=mp)
    ad = model.init_adapters(seed, rank, alpha=alpha)
    rng = np.random.default_rng(60 + seed)
    for v in ad.values():
        v['lora_b'] = (rng.standard_normal(v['lora_b'].shape) * 0.3 * v['lora_b'].shape[0] ** -0.5).astype(np.float32)
    head = model.init_head(seed, C)
    head[HEAD]['b'] = (rng.standard_normal(C) * 0.1).astype(np.float32)
    rows = rng.integers(1, 256, (B, kw['seq_len'] + 1)).astype(np.uint16)
    rows[0, kw['seq_len'] // 2:] = 0
    rows[1, 20:] = 0
    y = (rng.standard_normal((B, C)) if task == 'regression' else rng.integers(0, C, B)).astype(
        np.float32 if task == 'regression' else np.int64)
    return model, cfg, params, ad, head, rows, y


def _close(got, want, rel=2e-4):
    scale = max(1e-8, float(np.abs(want).max()))
    return float(np.abs(np.asarray(got, np.float64) - want).max()) <= rel * scale + 1e-7


@pytest.mark.parametrize('task', ['regression', 'classification'])
@pytest.mark.parametrize('name', sorted(CONFIGS))
def test_fp32_property_loss_and_grads_match_float64(name, task):
    model, cfg, params, ad, head, rows, y = _setup(name, False, task, seed=1)
    o_loss, o_grads, o_head, o_pred, _, _ = property_loss_and_grads(params, head, rows, y, cfg, task, ad, 2.0)
    loss, grads, hgrads, pred = model.property_loss_and_grad(params, rows, y, adapters=ad, head=head, task=task,
                                                             lora_alpha=32.0)
    assert abs(loss - o_loss) < 1e-5 * max(1.0, abs(o_loss)), (loss, o_loss)
    assert _close(pred, o_pred, 1e-5)
    for m, d in o_grads.items():
        for k, g in d.items():
            assert _close(grads[m][k], g), (m, k, np.abs(grads[m][k] - g).max(), np.abs(g).max())
    for k in ('w', 'b'):
        assert _close(hgrads[HEAD][k], o_head[HEAD][k]), k
    assert set(grads) == set(ad) and set(hgrads) == {HEAD}


def test_bf16_property_grads_three_way_at_the_config2_stack():
    """ref (float64) / emu (fp32 with bf16 operands) / cuda at the config-2 layer stack, B = 2 (one row padded after n/2):
    loss, predictions, every adapter gradient and the head gradients, the engine within 2x of emu's distance to ref"""
    from progen_b200 import ProGen
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
    rows[1, 512:] = 0
    y = rng.standard_normal((2, 3)).astype(np.float32)
    ref = property_loss_and_grads(params, head, rows, y, cfg, 'regression', ad, 1.0, device='cuda')
    emu = property_loss_and_grads(params, head, rows, y, cfg, 'regression', ad, 1.0, dtype=torch.float32,
                                  operand_round=T.bf16_round, device='cuda')
    loss, grads, hgrads, pred = model.property_loss_and_grad(params, rows, y, adapters=ad, head=head, task='regression')
    rel = lambda a, b: float(np.linalg.norm(np.asarray(a, np.float64) - b) / max(1e-12, np.linalg.norm(b)))
    # the bounds of test_gpu_model.test_bf16_parity_at_benchmarked_shapes: the loss within 2x of |emu - ref| plus 2e-3,
    # predictions and every gradient leaf within 2x of emu's relative L2 distance to ref plus 1e-3
    print('loss', dict(ref=ref[0], emu=emu[0], cuda=loss))
    assert abs(loss - emu[0]) <= 2 * abs(emu[0] - ref[0]) + 2e-3
    pairs = [('pred', pred, emu[3], ref[3])]
    pairs += [(f'{m}/{k}', grads[m][k], emu[1][m][k], ref[1][m][k]) for m in ref[1] for k in ref[1][m]]
    pairs += [(f'head/{k}', hgrads[HEAD][k], emu[2][HEAD][k], ref[2][HEAD][k]) for k in ('w', 'b')]
    rec = {name: (rel(c, np.asarray(e, np.float64)), rel(e, np.asarray(r, np.float64))) for name, c, e, r in pairs}
    print('worst cuda-vs-emu / emu-vs-ref:', max((ce / max(er, 1e-4), name, ce, er) for name, (ce, er) in rec.items()))
    bad = {name: v for name, v in rec.items() if v[0] > 2 * v[1] + 1e-3}
    assert not bad, bad


@pytest.mark.parametrize('mp', [False, True])
def test_fresh_adapters_predict_bitwise(mp):
    """B = 0 adapters: the property step's predictions are bitwise `predict` on the base parameters (the training forward
    at full length against the inference forward cut to the rows' counted length)"""
    from progen_b200 import ProGen
    model, cfg, params, _, head, rows, y = _setup('sgu', mp)
    ad = model.init_adapters(1, 16)
    _, _, _, pred = model.property_loss_and_grad(params, rows, y, adapters=ad, head=head, task='regression')
    got = ProGen(**CONFIGS['sgu'], mixed_precision=mp).predict(params, head, rows, batch_size=2)
    assert np.array_equal(got['prediction'], pred)
    assert np.array_equal(model.predict(params, head, rows)['prediction'], pred)


def _trainer(mp, params, ad, head, task='regression', cuda_graph=False, every=2, lr=1e-2, name='sgu'):
    from progen_b200 import ProGen
    model = ProGen(**CONFIGS[name], mixed_precision=mp)
    return model, model.trainer(params, adapters=ad, head=head, task=task, lora_alpha=32.0, grad_accum_every=every,
                                learning_rate=lr, cuda_graph=cuda_graph)


def _batches(task, C=3, steps=6, seed=9):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(steps):
        r = rng.integers(1, 256, (3, 129)).astype(np.uint16)
        r[0, 64:] = 0
        out.append((r, rng.standard_normal((3, C)).astype(np.float32) if task == 'regression' else rng.integers(0, C, 3)))
    return out


@pytest.mark.parametrize('task', ['regression', 'classification'])
def test_trainer_matches_oracle_optimizer_and_keeps_the_base(task):
    _, cfg, params, ad, head, _, _ = _setup('sgu', False, task, seed=4)
    model, tr = _trainer(False, params, ad, head, task)
    base = tr.eng.params.clone()
    batches = _batches(task)
    tree = {**ad, **head}
    st = O.optim_init(tree, every=2)
    for i, (r, y) in enumerate(batches):
        loss = float(tr.property_step(r, y).item())
        a, h = {m: tree[m] for m in ad}, {HEAD: tree[HEAD]}
        o_loss, o_g, o_h, o_pred, o_row, _ = property_loss_and_grads(params, h, r, y, cfg, task, a, 2.0)
        assert abs(loss - o_loss) < 2e-5 * max(1.0, abs(o_loss)), (i, loss, o_loss)
        stats = tr.property_stats()
        assert _close(stats['prediction'], o_pred, 1e-4) and _close(stats['loss'], o_row, 1e-4)
        g = {**o_g, **o_h}
        # every trained parameter decays (adapters and head, the head bias included), like the trainer's single mask
        tree, _ = _optim_step_all_decay(tree, {m: {k: v.astype(np.float32) for k, v in d.items()} for m, d in g.items()},
                                        st, lr=1e-2)
    got = {**tr.adapters(), **tr.head()}
    worst = max(float(np.abs(got[m][k] - v).max()) for m, d in tree.items() for k, v in d.items())
    assert worst < 2e-3, worst
    assert torch.equal(tr.eng.params, base), 'the base parameters changed'
    assert set(tr.optim_state()['mu']) == set(ad) | {HEAD}


def _optim_step_all_decay(params, grads, st, **kw):
    """O.optim_step with weight decay on every leaf: 1-D leaves are given a second axis for the mask and restored"""
    lift = lambda t: {m: {k: (v[:, None] if np.ndim(v) == 1 else v) for k, v in d.items()} for m, d in t.items()}
    flat = lambda t, ref: {m: {k: (v[:, 0] if np.ndim(ref[m][k]) == 1 else v) for k, v in d.items()} for m, d in t.items()}
    for key in ('mu', 'nu', 'acc'):
        st[key] = lift(st[key])
    new, aux = O.optim_step(lift(params), lift(grads), st, **kw)
    for key in ('mu', 'nu', 'acc'):
        st[key] = flat(st[key], params)
    return flat(new, params), aux


@pytest.mark.parametrize('mp', [False, True])
def test_graph_replay_matches_eager(mp):
    """the replayed step runs the eager step's kernels on the same inputs: the losses and the trained state are bitwise
    equal (every reduction of the property step is in a fixed order; the bf16 split-K weight gradients of the adapters
    sum with float atomics, so the mixed-precision run is compared to round-off)"""
    _, _, params, ad, head, _, _ = _setup('sgu', mp, seed=5)
    batches = _batches('regression', seed=10)
    runs = []
    for graph in (False, True):
        _, tr = _trainer(mp, params, ad, head, cuda_graph=graph)
        losses = [float(tr.property_step(r, y).item()) for r, y in batches]
        runs.append((tr, losses))
    (te, el), (tg, gl) = runs
    assert tg._graph is not None
    if mp:
        np.testing.assert_allclose(gl[:2], el[:2], rtol=0, atol=0)       # the same adapters until the first update
        np.testing.assert_allclose(gl, el, rtol=0, atol=2e-2)
    else:
        assert gl == el, (gl, el)
        assert all(np.array_equal(te.head()[HEAD][k], tg.head()[HEAD][k]) for k in ('w', 'b'))


def test_predict_after_training_matches_score_and_the_step():
    """predict on the merged parameters: its embedding is bitwise score's, its predictions agree with the adapted step's
    own (merged weights are W + s A B rounded once to fp32)"""
    _, cfg, params, ad, head, rows, y = _setup('glu', False, seed=6)
    model, tr = _trainer(False, params, ad, head, every=1, lr=3e-3, name='glu')
    for r, t in _batches('regression', seed=11)[:3]:
        tr.property_step(r, t)
    trained_ad, trained_head = tr.adapters(), tr.head()
    merged = model.merge_adapters(params, trained_ad, lora_alpha=32.0)
    got = model.predict(merged, trained_head, rows)
    emb = model.score(merged, rows, return_embeddings=True)['embedding']
    assert np.array_equal(got['embedding'], emb)
    _, _, _, pred = model.property_loss_and_grad(params, rows, y, adapters=trained_ad, head=trained_head, task='regression',
                                                 lora_alpha=32.0)
    assert np.abs(got['prediction'] - pred).max() < 1e-4 * max(1.0, np.abs(pred).max()), np.abs(got['prediction'] - pred).max()


def test_refusals():
    from progen_b200 import lib as L
    model, _, params, ad, head, rows, y = _setup('glu', False, seed=7)
    _, tr = _trainer(False, params, ad, head, name='glu')
    tr.world = 2
    with pytest.raises(L.ProgenError, match='data-parallel property fine-tuning is not supported'):
        tr.property_step(rows, y)
    model.property_loss_and_grad(params, rows, y, adapters=ad, head=head, task='regression')
    with pytest.raises(L.ProgenError, match='zero_grads'):
        model.engine.train_step(('property', L.TASK_REGRESSION), 3, zero_grads=False)
    big = {HEAD: {'w': np.zeros((128, 65), np.float32), 'b': np.zeros(65, np.float32)}}
    with pytest.raises(L.ProgenError, match='1 to 64'):
        model.trainer(params, adapters=ad, head=big, task='regression')
    with pytest.raises(L.ProgenError, match='at least 2 classes'):
        model.property_loss_and_grad(params, rows, np.zeros(3, np.int64), adapters=ad, head=model.init_head(0, 1),
                                     task='classification')
    plain = model.trainer(params, adapters=ad)
    with pytest.raises(L.ProgenError, match='no property head'):
        plain.property_step(rows, y)


def test_cli_fitness_train_resume_predict_score_generate(tmp_path):
    """a base trained for one step, then fitness.py train (regression, 2 outputs, with validation) for one epoch and a
    resumed second one; predict writes model.predict on package_params, de-standardized; classification trains too;
    score.py and generate.py run on the fitness package"""
    import pickle
    from progen_b200 import ProGen
    from progen_b200.checkpoint import package_params
    from progen_b200.data import collate
    from progen_b200.property import destandardize
    cfg_dir = tmp_path / 'cfg'
    cfg_dir.mkdir()
    (cfg_dir / 'tiny.toml').write_text('num_tokens = 256\ndim = 128\ndepth = 2\ndim_head = 64\nheads = 2\n'
                                       'window_size = 64\nseq_len = 128\nglobal_mlp_depth = 1\n')
    seqs = ['MKTAYIAKQRQISFVKSHFSRQ' * (1 + i % 3) + 'ACDEFGHIK'[:i % 9] for i in range(24)]
    (tmp_path / 'seqs.txt').write_text('\n'.join(seqs) + '\n')
    rng = np.random.default_rng(0)
    vals = rng.standard_normal((24, 2)) * [2.0, 0.5] + [10.0, -1.0]
    (tmp_path / 'train.tsv').write_text(''.join(f'{s}\t{a}\t{b}\n' for s, (a, b) in zip(seqs[:16], vals[:16])))
    (tmp_path / 'valid.tsv').write_text(''.join(f'{s}\t{a}\t{b}\n' for s, (a, b) in zip(seqs[16:], vals[16:])))
    (tmp_path / 'cls.tsv').write_text(''.join(f'{s}\t{"ab"[i % 2]}\n' for i, s in enumerate(seqs)))
    env = dict(os.environ, PYTHONPATH=ROOT)
    run = lambda *a: subprocess.run([sys.executable, *a], cwd=ROOT, env=env, check=True, capture_output=True, text=True)
    base, fit = tmp_path / 'base', tmp_path / 'fit'
    run('train.py', '--config_path', str(cfg_dir), '--model_name', 'tiny', '--checkpoint_path', str(base), '--num_steps', '1',
        '--text_file', str(tmp_path / 'seqs.txt'), '--batch_size', '2', '--sample_every', '1000', '--validate_every', '1000')
    common = ['--train', str(tmp_path / 'train.tsv'), '--valid', str(tmp_path / 'valid.tsv'), '--checkpoint_path', str(fit),
              '--batch_size', '4', '--cuda_graph']
    out = run('fitness.py', 'train', '--init_checkpoint', str(base), '--task', 'regression', '--lora_rank', '8',
              '--epochs', '1', *common)
    assert 'epoch 0: train loss' in out.stdout and 'valid spearman' in out.stdout, out.stdout
    out = run('fitness.py', 'train', '--epochs', '2', *common)
    assert 'starting from row 16' in out.stdout and 'epoch 1: train loss' in out.stdout, out.stdout
    pkg = pickle.load(open(sorted(fit.glob('ckpt_*'))[-1], 'rb'))
    assert pkg['next_index'] == 32 and pkg['head']['task'] == 'regression' and pkg['head']['num_outputs'] == 2
    np.testing.assert_allclose(pkg['head']['target_mean'], vals[:16].mean(0))
    assert 'params' not in pkg and pkg['lora'] == {'rank': 8, 'alpha': 8.0}
    with pytest.raises(subprocess.CalledProcessError):
        run('fitness.py', 'train', '--task', 'classification', '--epochs', '3', *common)
    run('fitness.py', 'predict', '--checkpoint_path', str(fit), '--input', str(tmp_path / 'seqs.txt'),
        '--output', str(tmp_path / 'preds.tsv'))
    lines = (tmp_path / 'preds.tsv').read_text().splitlines()
    assert lines[0] == 'index\tresidues\tvalue_0\tvalue_1' and len(lines) == 25
    got = np.array([[float(v) for v in l.split('\t')[2:]] for l in lines[1:]])
    model = ProGen(**pkg['model_config'])
    pred = model.predict(package_params(pkg), pkg['head']['params'], collate(seqs, 128))['prediction']
    want = destandardize(pred, pkg['head']['target_mean'], pkg['head']['target_std'])
    np.testing.assert_allclose(got, want, rtol=1e-8, atol=1e-6)
    run('score.py', '--checkpoint_path', str(fit), '--input', str(tmp_path / 'seqs.txt'), '--output', str(tmp_path / 's.tsv'))
    assert (tmp_path / 's.tsv').read_text().count('\n') == 25
    run('generate.py', '--checkpoint_path', str(fit), '--prompt', 'MK', '--num_samples', '2', '--max_length', '32',
        '--output', str(tmp_path / 'gen.fasta'))
    cls = tmp_path / 'fit_cls'
    out = run('fitness.py', 'train', '--init_checkpoint', str(base), '--task', 'classification', '--lora_rank', '8',
              '--train', str(tmp_path / 'cls.tsv'), '--valid', str(tmp_path / 'cls.tsv'), '--checkpoint_path', str(cls),
              '--batch_size', '8')
    assert 'valid accuracy' in out.stdout, out.stdout
    run('fitness.py', 'predict', '--checkpoint_path', str(cls), '--input', str(tmp_path / 'seqs.txt'),
        '--output', str(tmp_path / 'cls.tsv.out'))
    rows = (tmp_path / 'cls.tsv.out').read_text().splitlines()
    assert rows[0] == 'index\tresidues\tclass\tp_a\tp_b' and all(r.split('\t')[2] in 'ab' for r in rows[1:])
    probs = np.array([[float(v) for v in r.split('\t')[3:]] for r in rows[1:]])
    np.testing.assert_allclose(probs.sum(1), 1.0, atol=1e-5)
