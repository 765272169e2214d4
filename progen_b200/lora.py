"""Low-rank adapters (LoRA, Hu et al. 2021) on the four projections of every layer.

An adapted projection with weight W [in, out] computes with W + s A B, A [in, r], B [r, out], s = alpha / r.  The
adapter tree is haiku-shaped, {module: {'lora_a': A, 'lora_b': B}}, over the modules of `adapter_modules`; the columns
of a GLU feed-forward input's B are in haiku order (value | gate) there and interleaved in the engine, like the base
weight.  Everything else of the model stays frozen.

On the device the adapters live in one flat fp32 buffer in engine layout (`engine.Layout`: every A segment, then every
B segment, each on an ALIGN boundary) with a compute copy in the act dtype that holds A and s B: the forward folds u B
into the projection's GEMM as a tail operand pair (progen_gemm's A2 / B2), the backward folds s g A^T into the
input-gradient GEMM the same way (DESIGN.md §3.8)."""
import numpy as np
import torch

from . import lib as L
from .engine import P, Layout, ParamSpec, layer_kinds

RANKS = tuple(range(8, 65, 8))      # multiples of 8: 16-byte TMA row strides, and one tail k-block of 64


def adapter_modules(cfg):
    """[(module, in, out, glu)] of the adapted projections, layer by layer: QKV, attention output, feed-forward in and
    out (gMLP layers included); glu marks a GLU feed-forward input, whose output columns are (value | gate)"""
    d, inner, hid = cfg['dim'], cfg['heads'] * cfg['dim_head'], cfg['dim'] * cfg['ff_mult']
    out = []
    for i, kind in enumerate(layer_kinds(cfg['depth'], cfg['global_mlp_depth'], cfg['ff_glu'])):
        a, f = P + f'attn{i}/~/', P + f'ff{i}/~/'
        h_in = 2 * hid if kind == 'glu' else hid
        h_out = hid // 2 if kind == 'sgu' else hid
        out += [(a + 'linear', d, 3 * inner, False), (a + 'linear_1', inner, d, False),
                (f + 'linear', d, h_in, kind == 'glu'), (f + 'linear_1', h_out, d, False)]
    return out


def adapter_shapes(cfg, rank):
    return {m: {'lora_a': (i, rank), 'lora_b': (rank, o)} for m, i, o, _ in adapter_modules(cfg)}


HEAD = 'property_head'              # module of a property head's {'w': [d, C], 'b': [C]} (DESIGN.md §3.9)


def build_adapter_specs(cfg, rank, head_outputs=0):
    """the Layout of the adapter buffer: every A segment, then every B segment.  A property head of head_outputs > 0
    outputs takes the last segments: the trained flat state is then adapters plus head, and the compute copy (A | s B)
    stops before it."""
    mods = adapter_modules(cfg)
    specs = ([ParamSpec(m, 'lora_a', (i, rank)) for m, i, o, _ in mods] +
             [ParamSpec(m, 'lora_b', (rank, o), interleave=glu) for m, i, o, glu in mods])
    if head_outputs:
        specs += [ParamSpec(HEAD, 'w', (cfg['dim'], head_outputs)), ParamSpec(HEAD, 'b', (head_outputs,))]
    return Layout(specs)


def check_rank_alpha(rank, alpha):
    """-> (rank, alpha as float); alpha None means rank"""
    if isinstance(rank, (bool, np.bool_)) or not isinstance(rank, (int, np.integer)) or int(rank) not in RANKS:
        raise L.ProgenError(f'adapter rank must be an integer multiple of 8 in [8, 64], got {rank!r}')
    rank = int(rank)
    if alpha is None:
        return rank, float(rank)
    try:
        a = float(alpha)
    except (TypeError, ValueError):
        raise L.ProgenError(f'lora_alpha must be a finite number > 0, got {alpha!r}') from None
    if isinstance(alpha, (bool, np.bool_)) or not np.isfinite(a) or a <= 0:
        raise L.ProgenError(f'lora_alpha must be a finite number > 0, got {alpha!r}')
    return rank, a


def check_adapters(cfg, adapters):
    """Validate an adapter tree against the model config -> its rank.  ProgenError names the offending leaf: a missing
    or extra module or leaf, a shape that is not [in, r] / [r, out], ranks that differ between leaves, a non-finite
    value."""
    if not isinstance(adapters, dict):
        raise L.ProgenError('adapters must be a dict {module: {"lora_a": A, "lora_b": B}}')
    mods = {m: (i, o) for m, i, o, _ in adapter_modules(cfg)}
    missing, extra = sorted(set(mods) - set(adapters)), sorted(set(adapters) - set(mods))
    if missing:
        raise L.ProgenError(f'adapters: missing module {missing[0]}')
    if extra:
        raise L.ProgenError(f'adapters: unexpected module {extra[0]}')
    rank = None
    for m, (fin, fout) in mods.items():
        leaves = adapters[m]
        if not isinstance(leaves, dict) or set(leaves) != {'lora_a', 'lora_b'}:
            got = sorted(leaves) if isinstance(leaves, dict) else type(leaves).__name__
            raise L.ProgenError(f'adapters: {m} must hold exactly lora_a and lora_b, got {got}')
        for name in ('lora_a', 'lora_b'):
            a = leaves[name]
            a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
            if a.ndim != 2:
                raise L.ProgenError(f'adapters: {m}/{name} must be 2-D, got shape {a.shape}')
            r = a.shape[1] if name == 'lora_a' else a.shape[0]
            want = (fin, r) if name == 'lora_a' else (r, fout)
            if a.shape != want:
                raise L.ProgenError(f'adapters: {m}/{name} must have shape {want}, got {a.shape}')
            if rank is None:
                rank = r
            elif r != rank:
                raise L.ProgenError(f'adapters: {m}/{name} has rank {r}, other leaves have rank {rank}')
            if not np.issubdtype(a.dtype, np.number) or not np.isfinite(a.astype(np.float64)).all():
                raise L.ProgenError(f'adapters: {m}/{name} has a non-finite value')
    check_rank_alpha(rank, None)
    return rank


def init_adapters(cfg, seed, rank):
    """A ~ TruncatedNormal(1 / sqrt(in)) (the base Linear's initialiser), B = 0: the adapted model is the base model"""
    from .progen import _trunc_normal
    g = np.random.default_rng(seed)
    return {m: {'lora_a': _trunc_normal(g, (i, rank), i ** -0.5), 'lora_b': np.zeros((rank, o), np.float32)}
            for m, i, o, _ in adapter_modules(cfg)}


def merge_adapters(params, adapters, scale):
    """params with every adapted W replaced by float32(W + scale A B), computed in float64 on the host"""
    out = {m: dict(v) for m, v in params.items()}
    for m, leaves in adapters.items():
        host = lambda t: (t.detach().cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)).astype(np.float64)
        w = host(params[m]['w'])
        out[m]['w'] = (w + scale * (host(leaves['lora_a']) @ host(leaves['lora_b']))).astype(np.float32)
    return out


class Adapters:
    """The device state of one adapter tree for an Engine: flat fp32 parameters and gradients in engine layout, the
    act-dtype compute copy (A | s B), and per-projection u = x A activations of the training set."""

    def __init__(self, eng, rank, alpha, head_outputs=0):
        self.eng = eng
        self.r, self.alpha = rank, float(alpha)
        self.scale = self.alpha / rank
        self.head_outputs = int(head_outputs)
        self.layout = lay = build_adapter_specs(eng.cfg, rank, self.head_outputs)
        self.n_a = lay.span([s for s in lay.specs if s.name == 'lora_a'])[1]
        self.n_head = lay.span([s for s in lay.specs if s.module != HEAD])[1]          # end of the A | B segments
        self.num_params = lay.num_params
        f32 = dict(device=eng.dev, dtype=torch.float32)
        self.params = torch.zeros(lay.size, **f32)
        self.grads = torch.zeros(lay.size, **f32)
        self.lp = torch.zeros(lay.size, device=eng.dev, dtype=eng.act)
        self.u, self.g, self.T = None, None, 0

    def head(self, buf, name):
        """the property head's fp32 segment `name` ('w' [d, C] or 'b' [C]) of buffer `buf`"""
        return self.layout.seg(buf, HEAD, name)

    def load(self, tree, head=None):
        """adapter tree (and, with head_outputs, the head tree {'property_head': {'w', 'b'}}) -> the device buffer"""
        self.params.copy_(torch.from_numpy(self.layout.pack(tree if head is None else {**tree, **head})))
        self.refresh()

    def split(self, tree):
        """a tree exported from this buffer -> (adapter tree, head tree or None)"""
        head = tree.pop(HEAD, None)
        return tree, None if head is None else {HEAD: head}

    def refresh(self):
        """compute copy: A as is, B times s, in the act dtype; call after every parameter change.  A property head
        (fp32, read by progen_property_head from the parameters) has no compute copy."""
        lib, st, n_a = self.eng.lib, L.stream(), self.n_a
        L.check(lib.progen_scale_cast_f32(self.params.data_ptr(), self.lp.data_ptr(), self.eng.act_dt, 1.0, n_a, st),
                'adapter copy A')
        L.check(lib.progen_scale_cast_f32(self.params[n_a:].data_ptr(), self.lp[n_a:].data_ptr(), self.eng.act_dt,
                                          self.scale, self.n_head - n_a, st), 'adapter copy s B')

    def scale_b_grads(self):
        """dB = s u^T dy: the wgrad GEMMs accumulate u^T dy, the scale follows in one pass over the B gradients (not
        the property head's)"""
        if self.scale != 1.0:
            g = self.grads[self.n_a:self.n_head]
            L.check(self.eng.lib.progen_scale_cast_f32(g.data_ptr(), g.data_ptr(), L.F32, self.scale, g.numel(), L.stream()),
                    'adapter grad s')

    def activations(self, T):
        """u [T, r] per adapted projection (kept for the backward pass) and one g [T, r] scratch, T the training set's
        B * seq_len rows; a cut step uses their first B * length rows (Engine.lora_fwd / lora_bwd).  A new row count
        re-allocates them, which invalidates captured graphs like Engine.ensure_batch does"""
        if self.T != T:
            A = lambda: torch.empty(T, self.r, device=self.eng.dev, dtype=self.eng.act)
            self.u = {m: A() for m, _, _, _ in adapter_modules(self.eng.cfg)}
            self.g = A()
            self.T = T
            self.eng.alloc_epoch += 1
        return self.u
