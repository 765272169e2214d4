"""Property fine-tuning without a GPU: the float64 reference loss the GPU tests compare against (its gradient against
finite differences, for both tasks), every input check of `ProGen.property_loss_and_grad`, `predict`, `init_head` and
`model.trainer(head=, task=)` (all before any device work), the fitness.py labelled-sequence file, target
standardization and the numpy Spearman correlation."""
import numpy as np
import pytest
import torch

from oracle import progen_ref as O
from oracle import progen_torch as T
from property_oracle import HEAD, head_loss, pooled, property_loss_and_grads

KW = dict(num_tokens=256, dim=128, seq_len=128, depth=2, window_size=64, global_mlp_depth=1, heads=2, dim_head=64)


def _rows(B, n=128, seed=0):
    r = np.random.default_rng(seed).integers(1, 256, (B, n + 1)).astype(np.uint16)
    r[0, 40:] = 0
    return r


def _model():
    from progen_b200 import ProGen
    return ProGen(**KW)


# ------------------------------------------------------------------------------------------------ oracle
def _tiny():
    kw = dict(num_tokens=32, dim=16, seq_len=16, depth=2, window_size=8, global_mlp_depth=1, heads=2, dim_head=8)
    cfg = O.make_config(**kw)
    return cfg, O.randomize_params(O.init_params(cfg, 1), 2)


@pytest.mark.parametrize('task', ['regression', 'classification'])
def test_oracle_gradient_matches_finite_differences(task):
    cfg, params = _tiny()
    rng = np.random.default_rng(3)
    rows = rng.integers(1, 32, (3, 17)).astype(np.int64)
    rows[1, 9:] = 0
    C = 3
    head = {HEAD: {'w': rng.standard_normal((16, C)) * 0.5, 'b': rng.standard_normal(C) * 0.1}}
    y = rng.standard_normal((3, C)) if task == 'regression' else np.array([0, 2, 1])
    loss, grads, hgrads, p, row, emb = property_loss_and_grads(params, head, rows, y, cfg, task)
    assert np.isclose(loss, row.mean()) and p.shape == (3, C) and emb.shape == (3, 16)

    def f(prm_np, head_np):
        prm = T.to_torch(prm_np)
        e = pooled(prm, torch.as_tensor(rows), cfg)
        w = torch.tensor(head_np[HEAD]['w'], dtype=torch.float64)
        b = torch.tensor(head_np[HEAD]['b'], dtype=torch.float64)
        return float(head_loss(e, w, b, y, task)[0])

    eps = 1e-6
    probes = [(HEAD, 'w', (4, 1)), (HEAD, 'b', (2,)), (O.P + 'layer_norm', 'scale', (5,)),
              (O.P + 'attn1/~/linear', 'w', (3, 7)), (O.P + 'ff0/~/linear', 'w', (2, 9))]
    for m, k, idx in probes:
        src = head if m == HEAD else params
        plus = {mm: {kk: np.array(vv, np.float64) for kk, vv in d.items()} for mm, d in src.items()}
        minus = {mm: {kk: np.array(vv, np.float64) for kk, vv in d.items()} for mm, d in src.items()}
        plus[m][k][idx] += eps
        minus[m][k][idx] -= eps
        if m == HEAD:
            fd = (f(params, plus) - f(params, minus)) / (2 * eps)
            g = hgrads[m][k][idx]
        else:
            fd = (f(plus, head) - f(minus, head)) / (2 * eps)
            g = grads[m][k][idx]
        assert abs(fd - g) <= 1e-6 + 1e-5 * abs(fd), (m, k, idx, fd, g)


def test_oracle_pool_is_the_masked_mean():
    cfg, params = _tiny()
    rows = np.random.default_rng(4).integers(1, 32, (2, 17)).astype(np.int64)
    rows[0, 6:] = 0
    _, h = T.forward(T.to_torch(params), torch.as_tensor(rows[:, :-1]), cfg, return_hidden=True)
    e = pooled(T.to_torch(params), torch.as_tensor(rows), cfg).numpy()
    np.testing.assert_allclose(e[0], h[0, :6].numpy().mean(0), rtol=1e-12)       # labels 1..4 and the first pad
    np.testing.assert_allclose(e[1], h[1].numpy().mean(0), rtol=1e-12)


# ------------------------------------------------------------------------------------------------ input checks
def _inputs(task='regression', C=2, B=2):
    model = _model()
    params = {}
    ad = model.init_adapters(0, 8)
    head = model.init_head(0, C)
    y = np.zeros((B, C), np.float32) if task == 'regression' else np.zeros(B, np.int64)
    return model, params, ad, head, _rows(B), y


@pytest.mark.parametrize('change, match', [
    (dict(task='ranking'), "task must be 'regression' or 'classification'"),
    (dict(targets=np.zeros((2, 3), np.float32)), r'targets must have shape \(2, 2\)'),
    (dict(targets=np.array([[0, np.nan], [0, 0]])), 'targets must be finite'),
    (dict(targets=np.array([[0, 1e39], [0, 0]])), r'targets must be finite \(in float32\)'),
    (dict(task='classification', targets=np.array([0, 2])), r'class indices must be in \[0, 2\)'),
    (dict(task='classification', targets=np.array([0.0, 1.0])), 'integer class indices'),
    (dict(task='classification', targets=np.array([[0], [1]])), r'targets must have shape \(2,\)'),
    (dict(rows=np.zeros((2, 128), np.int64)), r'rows must be \(B, seq_len \+ 1 = 129\)'),
    (dict(rows=np.zeros((2, 129), np.float32)), 'rows must hold integer token ids'),
    (dict(head={HEAD: {'w': np.zeros((64, 2), np.float32), 'b': np.zeros(2, np.float32)}}), r'w must have shape \[dim = 128'),
    (dict(head={HEAD: {'w': np.zeros((128, 2), np.float32), 'b': np.zeros(3, np.float32)}}), r'b must have shape \(2,\)'),
    (dict(head={HEAD: {'w': np.zeros((128, 65), np.float32), 'b': np.zeros(65, np.float32)}}), '65 outputs; a property head has 1 to 64'),
    (dict(head={'w': np.zeros((128, 2), np.float32)}), 'head must be'),
    (dict(head={HEAD: {'w': np.full((128, 2), np.inf, np.float32), 'b': np.zeros(2, np.float32)}}), 'w has a non-finite value'),
    (dict(adapters={'x': {}}), 'adapters: missing module'),
])
def test_property_loss_and_grad_checks_inputs_before_device_work(change, match):
    from progen_b200 import lib as L
    model, params, ad, head, rows, y = _inputs()
    kw = dict(rows=rows, targets=y, adapters=ad, head=head, task='regression')
    kw.update(change)
    with pytest.raises(L.ProgenError, match=match):
        model.property_loss_and_grad(params, kw.pop('rows'), kw.pop('targets'), **kw)
    assert model._engine is None


def test_classification_needs_two_classes():
    from progen_b200 import lib as L
    model, params, ad, _, rows, _ = _inputs()
    head = model.init_head(0, 1)
    with pytest.raises(L.ProgenError, match='classification needs at least 2 classes'):
        model.property_loss_and_grad(params, rows, np.zeros(2, np.int64), adapters=ad, head=head, task='classification')
    with pytest.raises(L.ProgenError, match='classification needs at least 2 classes'):
        model.trainer(params, adapters=ad, head=head, task='classification')
    assert model._engine is None


def test_single_output_regression_takes_a_vector():
    from progen_b200.property import check_targets
    y = check_targets([1.0, 2.0], 'regression', 1, 2, 'x')
    assert y.shape == (2, 1) and y.dtype == np.float32


def test_trainer_and_predict_check_inputs_before_device_work():
    from progen_b200 import lib as L
    model, params, ad, head, rows, _ = _inputs()
    with pytest.raises(L.ProgenError, match='pass adapters='):
        model.trainer(params, head=head, task='regression')
    with pytest.raises(L.ProgenError, match='both head= and task='):
        model.trainer(params, adapters=ad, head=head)
    with pytest.raises(L.ProgenError, match="task must be 'regression' or 'classification'"):
        model.trainer(params, adapters=ad, head=head, task='rank')
    with pytest.raises(L.ProgenError, match=r'w must have shape \[dim = 128'):
        model.predict(params, {HEAD: {'w': np.zeros((8, 1)), 'b': np.zeros(1)}}, rows)
    with pytest.raises(L.ProgenError, match='batch_size must be an integer >= 1'):
        model.predict(params, head, rows, batch_size=0)
    with pytest.raises(L.ProgenError, match=r'rows must be \(B, seq_len \+ 1 = 129\)'):
        model.predict(params, head, rows[:, :-1])
    assert model._engine is None


def test_init_head():
    from progen_b200 import lib as L
    model = _model()
    h = model.init_head(7, 3)
    assert set(h) == {HEAD} and h[HEAD]['w'].shape == (128, 3) and h[HEAD]['w'].dtype == np.float32
    assert np.all(h[HEAD]['b'] == 0) and np.abs(h[HEAD]['w']).max() <= 2 * 128 ** -0.5
    assert np.array_equal(h[HEAD]['w'], model.init_head(7, 3)[HEAD]['w'])
    for bad in (0, 65, 2.0, True):
        with pytest.raises(L.ProgenError, match=r'num_outputs must be an integer in \[1, 64\]'):
            model.init_head(0, bad)


def test_head_segments_follow_the_adapters():
    """the head is the last segment of the adapter buffer: the compute copy and the B-gradient scale stop before it"""
    from progen_b200.lora import build_adapter_specs
    cfg = _model().config
    lay, lay0 = build_adapter_specs(cfg, 8, 3), build_adapter_specs(cfg, 8)
    specs, n, n_a = lay.specs, lay.size, lay.span([s for s in lay.specs if s.name == 'lora_a'])[1]
    plain, n0, n_a0 = lay0.specs, lay0.size, lay0.span([s for s in lay0.specs if s.name == 'lora_a'])[1]
    assert n_a == n_a0 and [(s.module, s.name, s.offset) for s in specs[:len(plain)]] == \
        [(s.module, s.name, s.offset) for s in plain]
    hw, hb = specs[-2:]
    assert (hw.module, hw.name, hw.shape, hw.offset) == (HEAD, 'w', (128, 3), n0)
    assert (hb.module, hb.name, hb.shape) == (HEAD, 'b', (3,)) and hb.offset % 64 == 0 and n % 64 == 0


# ------------------------------------------------------------------------------------------------ fitness.py data
def test_read_labelled_regression_and_classification():
    from progen_b200.property import read_labelled
    seqs, y = read_labelled(['MKT\t1.5\t2\n', '\n', 'ACD\t-3\t0.25\r\n'], 'regression')
    assert seqs == ['MKT', 'ACD'] and y.shape == (2, 2) and y.dtype == np.float64 and y[1, 0] == -3
    seqs, y = read_labelled(['MKT\tactive\n', 'ACD\tinactive\n'], 'classification')
    assert seqs == ['MKT', 'ACD'] and y == ['active', 'inactive']


@pytest.mark.parametrize('task, lines, match', [
    ('regression', ['MKT\t1\n', 'ACD\n'], 'line 2: expected `sequence<TAB>value`'),
    ('regression', ['MKT\t1\n', '\n', 'ACD\tx\n'], 'line 3: values must be numbers'),
    ('regression', ['MKT\t1\t2\n', 'ACD\t1\n'], 'line 2: 1 values, earlier lines have 2'),
    ('regression', ['MKT\tnan\n'], 'line 1: values must be finite'),
    ('regression', ['\t1\n'], 'line 1: empty sequence'),
    ('classification', ['MKT\ta\n', 'ACD\ta\tb\n'], 'line 2: expected `sequence<TAB>class_name`'),
    ('classification', ['MKT\t \n'], 'line 1: expected `sequence<TAB>class_name`'),
])
def test_read_labelled_names_the_bad_line(task, lines, match):
    from progen_b200 import lib as L
    from progen_b200.property import read_labelled
    with pytest.raises(L.ProgenError, match=match):
        read_labelled(lines, task)


def test_standardization_round_trips():
    from progen_b200.property import destandardize, standardize
    y = np.random.default_rng(0).standard_normal((50, 3)) * [1.0, 40.0, 1e-3] + [5.0, -200.0, 0.0]
    y[:, 2] = 7.0                                     # a constant output keeps std 1
    z, mean, std = standardize(y)
    assert z.dtype == np.float32 and std[2] == 1.0
    np.testing.assert_allclose(z[:, :2].mean(0), 0, atol=1e-6)
    np.testing.assert_allclose(z[:, :2].std(0), 1, atol=1e-6)
    np.testing.assert_allclose(destandardize(z, mean, std), y, rtol=1e-6, atol=1e-4)
    z2, m2, s2 = standardize(y[:5], mean, std)        # other rows with the training statistics
    np.testing.assert_array_equal(z2, z[:5])


def _spearman_definition(x, y):
    """rank correlation from its definition: Pearson correlation of average ranks, ranks counted pairwise"""
    def ranks(v):
        v = np.asarray(v, np.float64)
        return np.array([(v < a).sum() + ((v == a).sum() + 1) / 2.0 for a in v])
    return float(np.corrcoef(ranks(x), ranks(y))[0, 1])


def test_spearman_matches_the_rank_correlation_with_ties():
    from progen_b200.property import rankdata, spearman
    rng = np.random.default_rng(1)
    x = rng.integers(0, 5, 40).astype(np.float64)          # many ties
    y = x + rng.integers(0, 3, 40)
    np.testing.assert_array_equal(rankdata([3, 1, 3, 2]), [3.5, 1, 3.5, 2])
    assert abs(spearman(x, y) - _spearman_definition(x, y)) < 1e-12
    z = rng.standard_normal(30)
    assert abs(spearman(z, -z) + 1.0) < 1e-12
    assert np.isnan(spearman(np.ones(5), np.arange(5)))
