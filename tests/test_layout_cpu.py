"""The flat-buffer engine layout without a GPU: pack / unpack round trips for every layer kind and for the adapter buffer
with and without a property head, the shape check on every leaf (parameters, adapters, optimizer state), and the segment
order, alignment and per-layer ranges the optimizer and the overlapped all-reduce rely on."""
import numpy as np
import pytest
import torch

from progen_b200 import ProGen
from progen_b200 import lib as L
from progen_b200.engine import ALIGN, P, build_param_specs, layer_kinds
from progen_b200.lora import HEAD, build_adapter_specs

CFG = dict(num_tokens=64, dim=64, seq_len=64, depth=3, window_size=32, global_mlp_depth=1, heads=2, dim_head=32)
MODELS = {'glu': dict(CFG), 'gelu': dict(CFG, ff_glu=False), 'sgu': dict(CFG, global_mlp_depth=3)}


def _random_tree(shapes, seed):
    rng = np.random.default_rng(seed)
    return {m: {k: rng.standard_normal(s).astype(np.float32) for k, s in v.items()} for m, v in shapes.items()}


def _layouts():
    for name, kw in MODELS.items():
        cfg = ProGen(**kw).config
        yield name, build_param_specs(cfg)
        for C in (0, 3):
            yield f'{name} adapters head={C}', build_adapter_specs(cfg, 8, C)


@pytest.mark.parametrize('name, lay', list(_layouts()), ids=[n for n, _ in _layouts()])
def test_pack_unpack_round_trip(name, lay):
    tree = _random_tree(lay.shapes(), 0)
    host = lay.pack(tree)
    assert host.dtype == np.float32 and host.shape == (lay.size,)
    back = lay.unpack(torch.from_numpy(host))
    assert list(back) == list(tree) and all(list(back[m]) == list(tree[m]) for m in tree)
    assert all(np.array_equal(back[m][k], tree[m][k]) for m in tree for k in tree[m])
    # torch leaves pack to the same bits
    assert np.array_equal(lay.pack({m: {k: torch.from_numpy(a) for k, a in v.items()} for m, v in tree.items()}), host)
    # padding stays zero, and every leaf sits in its own segment
    used = np.zeros(lay.size, bool)
    for s in lay.specs:
        assert not used[s.offset:s.stop].any()
        used[s.offset:s.offset + s.size] = True
    assert not host[~used].any()


def test_glu_segments_are_interleaved():
    lay = build_param_specs(ProGen(**CFG).config)
    tree = _random_tree(lay.shapes(), 1)
    host = lay.pack(tree)
    m = P + 'ff0/~/linear'
    w, b = tree[m]['w'], tree[m]['b']
    H = w.shape[1] // 2
    sw = lay.seg(host, m, 'w').reshape(w.shape)
    assert np.array_equal(sw[:, 0::2], w[:, :H]) and np.array_equal(sw[:, 1::2], w[:, H:])
    sb = lay.seg(host, m, 'b')
    assert np.array_equal(sb[0::2], b[:H]) and np.array_equal(sb[1::2], b[H:])


@pytest.mark.parametrize('which', ['params', 'adapters'])
def test_wrong_shape_names_the_leaf(which):
    cfg = ProGen(**CFG).config
    lay = build_param_specs(cfg) if which == 'params' else build_adapter_specs(cfg, 8, 3)
    tree = _random_tree(lay.shapes(), 2)
    m, k = (P + 'attn1/~/linear', 'w') if which == 'params' else (P + 'ff0/~/linear', 'lora_b')
    tree[m][k] = tree[m][k].T.copy()                      # the same size, transposed
    with pytest.raises(L.ProgenError, match=f'{m}/{k}: expected shape'.replace('~', '.')):
        lay.pack(tree)


def test_optim_state_rejects_a_wrong_shape():
    from progen_b200.trainer import Trainer
    lay = build_adapter_specs(ProGen(**CFG).config, 8, 3)
    tr = Trainer.__new__(Trainer)
    tr.layout, tr.count = lay, 5
    tr.m, tr.v, tr.acc = (torch.zeros(lay.size) for _ in range(3))
    tr._adam_state = torch.zeros(4, dtype=torch.int64)
    st = {k: _random_tree(lay.shapes(), i) for i, k in enumerate(('mu', 'nu', 'acc'))}
    tr.load_optim_state(dict(count=7, every=4, **st))
    assert tr.count == 7 and torch.equal(tr.v, torch.from_numpy(lay.pack(st['nu'])))
    assert int(tr._adam_state[0]) == 7                   # the optimizer kernel's count follows the loaded one
    st['acc'][HEAD]['w'] = st['acc'][HEAD]['w'].T.copy()
    with pytest.raises(L.ProgenError, match=f'{HEAD}/w: expected shape'):
        tr.load_optim_state(dict(count=9, every=4, **st))
    assert tr.count == 7 and int(tr._adam_state[0]) == 7


@pytest.mark.parametrize('name', list(MODELS))
def test_engine_segments(name):
    """64-aligned, ndim > 1 leaves first, each group in tree order, and each layer's ndim > 1 leaves one contiguous range"""
    kw = MODELS[name]
    cfg = ProGen(**kw).config
    lay = build_param_specs(cfg)
    order = sorted(lay.specs, key=lambda s: s.offset)
    assert order == [s for s in lay.specs if s.decay] + [s for s in lay.specs if not s.decay]
    assert all(s.offset % ALIGN == 0 and s.stop - s.offset == -(-s.size // ALIGN) * ALIGN for s in lay.specs)
    assert all(a.stop == b.offset for a, b in zip(order, order[1:])) and order[0].offset == 0 and order[-1].stop == lay.size
    n_decay = lay.span([s for s in lay.specs if s.decay])[1]
    assert all((s.offset < n_decay) == s.decay for s in lay.specs)
    for i in range(len(layer_kinds(cfg['depth'], cfg['global_mlp_depth'], cfg['ff_glu']))):
        mine = [s for s in lay.specs if s.decay and s.module.startswith((P + f'attn{i}/~/', P + f'ff{i}/~/'))]
        a, b = lay.span(mine)
        assert b - a == sum(s.stop - s.offset for s in mine)


def test_adapter_segments():
    """every A, then every B, then the head, in tree order; A and B are ndim > 1"""
    lay = build_adapter_specs(ProGen(**CFG).config, 8, 3)
    order = sorted(lay.specs, key=lambda s: s.offset)
    assert order == lay.specs and all(s.offset % ALIGN == 0 for s in order)
    assert [s.name for s in order] == ['lora_a'] * 12 + ['lora_b'] * 12 + ['w', 'b']
