"""Host-side orchestration of the ProGen forward / backward pass over the C-ABI kernels.

Mirrors `ProGenBase.__call__` (reference progen.py:224-233) and its gradient (`jax.value_and_grad`, utils.py:72),
batched over sequences (the reference's `vmap`, utils.py:67).  PyTorch provides device buffers and streams only.

Data layout in HBM (tokens are rows, T = B * seq_len):
  * residual stream: fp32 [T, d], one buffer per LayerNorm input (the residual epilogue of each GEMM writes the next
    one, so nothing is copied and every LN backward still has its input); the inference set (`Engine.score`) keeps one
    buffer and updates it in place; a training set in recompute mode keeps one per layer input and one shared
    attention-block output (`training_set`);
  * activations: act dtype (bf16 with mixed_precision, fp32 without), row-major [T, features];
  * q|k|v: one [T, 3*heads*dim_head] buffer, rotated in the QKV GEMM epilogue;
  * parameters, gradients, Adam moments: FLAT fp32 buffers in "engine layout" (ndim > 1 leaves first, then the
    rest; GLU proj_in columns interleaved (value_j, gate_j) so both land in one GEMM tile); a bf16 mirror of the
    parameters feeds the tensor-core GEMMs; SGU spatial weights additionally keep a tril-masked compute copy.
"""
import math
import numpy as np
import torch

from . import lib as L

P = 'pro_gen_base/~/'      # haiku module-path prefix of the reference parameter tree (SURVEY §8(b))
ALIGN = 64                 # every parameter segment starts on a 64-element boundary (TMA needs 16-byte bases)


CUT_ALIGN = 128            # a cut forward's row length: whole 128-row GEMM tiles, and every SGU row tile keeps its k-blocks


def counted_length(labels):
    """labels [N, n] -> [N]: 1 + the last position the loss mask counts (non-pad labels plus the first pad, quirk Q8).
    Positions at or beyond it add nothing to a row's log-likelihood."""
    labels = np.asarray(labels)
    n = labels.shape[1]
    pad = labels == 0
    first = np.where(pad.any(1), pad.argmax(1), n)
    last = np.where((~pad).any(1), n - 1 - (~pad)[:, ::-1].argmax(1), -1)
    return np.minimum(n, np.maximum(first, last) + 1)


def cut_length(labels):
    """the row length of a forward that covers every counted position of labels [N, n]: their largest counted length
    rounded up to CUT_ALIGN, at most n"""
    n = np.asarray(labels).shape[1]
    need = int(counted_length(labels).max()) if len(labels) else 1
    return min(n, -(-need // CUT_ALIGN) * CUT_ALIGN)


def check_length(labels, length, what):
    """the row length of a forward or training step over the rows with labels [N, n] (host): `length` None means their
    cut_length; otherwise it must be n or a multiple of CUT_ALIGN below n that covers every counted position of the
    rows.  ProgenError otherwise, before any device work."""
    labels = np.asarray(labels)
    n = labels.shape[1]
    if length is None:
        return cut_length(labels)
    if isinstance(length, (bool, np.bool_)) or not isinstance(length, (int, np.integer)) or \
            not (length == n or (0 < length < n and length % CUT_ALIGN == 0)):
        raise L.ProgenError(f'{what}: length must be seq_len ({n}) or a multiple of {CUT_ALIGN} below it, got {length!r}')
    if len(labels) and int(counted_length(labels).max()) > length:
        raise L.ProgenError(f'{what}: length {length} cuts off counted positions (cut_length of these rows: '
                            f'{cut_length(labels)})')
    return int(length)


def layer_kinds(depth, global_mlp_depth, ff_glu):
    """reference progen.py:210-212"""
    out = []
    for i in range(depth):
        use_gmlp = (depth - i) <= global_mlp_depth
        out.append('sgu' if use_gmlp else ('glu' if ff_glu else 'gelu'))
    return out


def training_set(cfg, B, mixed_precision, recompute=False, device='meta'):
    """The training activation set of B rows of seq_len positions (Engine.ensure_batch), as {attribute: buffer}, and
    the bytes it allocates.  On the default 'meta' device nothing is allocated: the count is the shapes'.

    Resident (recompute=False): every LayerNorm input X[k] and one scratch dict per layer, all kept for the backward
    pass.  Recomputed (DESIGN.md §3.12): one fp32 checkpoint per layer input X[2i] (the final LayerNorm's input
    included), one attention-block output that every X[2i+1] aliases, and one layer scratch that every layer aliases,
    cut from one storage as wide as the widest layer kind; the backward pass re-runs each layer into it
    (Engine.recompute_layer).  Head buffers and backward temporaries are the same in both modes."""
    d, n, V, h = cfg['dim'], cfg['seq_len'], cfg['num_tokens'], cfg['heads']
    I, hid = cfg['heads'] * cfg['dim_head'], cfg['dim'] * cfg['ff_mult']
    half = hid // 2
    kinds = layer_kinds(cfg['depth'], cfg['global_mlp_depth'], cfg['ff_glu'])
    act = torch.bfloat16 if mixed_precision else torch.float32
    T = B * n
    allocated = []

    def new(shape, dtype):
        t = torch.empty(*shape, device=device, dtype=dtype)
        allocated.append(t)
        return t
    A = lambda *shape: new(shape, act)
    F = lambda *shape: new(shape, torch.float32)
    nl = len(kinds)
    b = dict(tok=new((T,), torch.int32), labels=new((T,), torch.int32))
    if not recompute:
        b['X'] = [F(T, d) for _ in range(2 * nl + 1)]            # residual stream at every LN input
        b['lay'] = []
        for kind in kinds:
            s = dict(mean1=F(T), rstd1=F(T), y1=A(T, d), qkv=A(T, 3 * I), att=A(T, I), lse=F(T, h),
                     mean2=F(T), rstd2=F(T), y2=A(T, d))
            if kind == 'glu':
                s.update(u=A(T, 2 * hid), hact=A(T, hid))
            else:
                s.update(u=A(T, hid), hact=A(T, hid))
            if kind == 'sgu':
                s.update(mean3=F(T), rstd3=F(T), gn=A(T, half), gp=A(T, half), sg=A(T, half), pj=A(T, half))
            b['lay'].append(s)
    else:
        ck, x_att = [F(T, d) for _ in range(nl + 1)], F(T, d)
        b['X'] = [x for c in ck[:-1] for x in (c, x_att)] + ck[-1:]
        common = dict(mean1=F(T), rstd1=F(T), y1=A(T, d), qkv=A(T, 3 * I), att=A(T, I), lse=F(T, h),
                      mean2=F(T), rstd2=F(T), y2=A(T, d))
        width = dict(glu=3 * hid, gelu=2 * hid, sgu=4 * hid)      # u, hact (and gn, gp, sg, pj) in act-dtype columns
        wide = A(T * max(width[k] for k in kinds))
        part = lambda col, w: wide[col * T:(col + w) * T].view(T, w)      # a contiguous [T, w] block: cuts by rows
        per_kind = dict(glu=dict(common, u=part(0, 2 * hid), hact=part(2 * hid, hid)),
                        gelu=dict(common, u=part(0, hid), hact=part(hid, hid)))
        if 'sgu' in kinds:
            per_kind['sgu'] = dict(common, u=part(0, hid), hact=part(hid, hid), mean3=F(T), rstd3=F(T),
                                   gn=part(2 * hid, half), gp=part(2 * hid + half, half), sg=part(3 * hid, half),
                                   pj=part(3 * hid + half, half))
        b['lay'] = [per_kind[k] for k in kinds]
    b.update(meanf=F(T), rstdf=F(T), yf=A(T, d), logits=F(T, V), dlogits=A(T, V), ce_w=F(T))
    # preference (DPO) head (train_step): B = 2 * pairs rows; allocated here so a captured step's pointers stay valid
    b.update(logp=F(T), seq_ll=F(B), seq_count=F(B), ref=F(B), stats=F(max(1, B // 2), 4), ce_scratch=F(1))
    # property head (train_step): pooled embedding and its gradient, predictions, targets, per-row losses
    C = L.PROPERTY_MAX_OUTPUTS
    b.update(emb=F(B, d), demb=F(B, d), pred=F(B * C), dpred=F(B * C), ptarget=F(B * C), prow_loss=F(B),
             pclass=new((B,), torch.int32))
    # backward temporaries (shared by all layers)
    b.update(dres=F(T, d))
    b.update(dres_lp=A(T, d) if mixed_precision else b['dres'], dy=A(T, d), dqkv=A(T, 3 * I), datt=A(T, I),
             delta=F(T, h), du=A(T, 2 * hid), dh_=A(T, hid))
    if 'sgu' in kinds:
        b.update(dpj=A(T, half), dsg=A(T, half), dgp=A(T, half), dgn=A(T, half))
    return b, sum(t.numel() * t.element_size() for t in allocated)


class ParamSpec:
    __slots__ = ('module', 'name', 'shape', 'decay', 'interleave', 'offset', 'stop', 'size')

    def __init__(self, module, name, shape, interleave=False):
        self.module, self.name, self.shape = module, name, tuple(shape)
        self.decay = len(shape) > 1                    # optax mask: tree_map(lambda x: x.ndim > 1) — train.py:113
        self.interleave = interleave
        self.size = int(np.prod(shape))
        self.offset = self.stop = -1                   # [offset, stop): the padded segment (set by Layout)


class Layout:
    """The engine layout of a flat fp32 buffer of haiku-shaped leaves: the ndim > 1 leaves first (the weight-decay mask
    is then one prefix), then the rest, each group in the order of `specs`; every segment starts on an ALIGN boundary;
    a GLU feed-forward input's columns (value | gate) are interleaved (value_j, gate_j), so both halves of a pair land
    in one GEMM tile.  Trees keep the order of `specs`.  Needs no device."""

    def __init__(self, specs):
        self.specs = list(specs)
        self.by_key = {(s.module, s.name): s for s in self.specs}
        off = 0
        for s in [s for s in self.specs if s.decay] + [s for s in self.specs if not s.decay]:
            s.offset = off
            off += (s.size + ALIGN - 1) // ALIGN * ALIGN
            s.stop = off
        self.size = off                                 # padded size of the buffer
        self.num_params = sum(s.size for s in self.specs)

    def span(self, specs):
        """[start, stop) of the padded segments of `specs` (contiguous when they are adjacent in the layout)"""
        return min(s.offset for s in specs), max(s.stop for s in specs)

    def seg(self, buf, module, name):
        s = self.by_key[(module, name)]
        return buf[s.offset:s.offset + s.size]

    def pack(self, tree):
        """haiku-shaped tree {module: {name: array}} (numpy or torch leaves) -> host float32 [size] in this layout"""
        host = np.zeros(self.size, np.float32)
        for s in self.specs:
            a = tree[s.module][s.name]
            a = (a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)).astype(np.float32)
            if a.shape != s.shape:
                raise L.ProgenError(f'{s.module}/{s.name}: expected shape {s.shape}, got {a.shape}')
            host[s.offset:s.offset + s.size] = (_interleave(a) if s.interleave else a).ravel()
        return host

    def unpack(self, buf):
        """a tensor in this layout -> haiku-shaped tree of float32 numpy arrays"""
        host = buf.detach().float().cpu().numpy()
        out = {}
        for s in self.specs:
            a = host[s.offset:s.offset + s.size].reshape(s.shape).copy()
            out.setdefault(s.module, {})[s.name] = _deinterleave(a) if s.interleave else a
        return out

    def shapes(self):
        """the shape tree {module: {name: shape}}"""
        out = {}
        for s in self.specs:
            out.setdefault(s.module, {})[s.name] = s.shape
        return out


def build_param_specs(cfg):
    """the Layout of the model's parameters"""
    d, V, n = cfg['dim'], cfg['num_tokens'], cfg['seq_len']
    inner = cfg['heads'] * cfg['dim_head']
    hid = d * cfg['ff_mult']
    specs = [ParamSpec(P + 'embed', 'embeddings', (V, d))]
    for i, kind in enumerate(layer_kinds(cfg['depth'], cfg['global_mlp_depth'], cfg['ff_glu'])):
        a = P + f'attn{i}/~/'
        specs += [ParamSpec(a + 'layer_norm', 'scale', (d,)),
                  ParamSpec(a + 'linear', 'w', (d, 3 * inner)),
                  ParamSpec(a + 'linear_1', 'w', (inner, d)), ParamSpec(a + 'linear_1', 'b', (d,))]
        f = P + f'ff{i}/~/'
        h_in = hid * 2 if kind == 'glu' else hid
        h_out = hid // 2 if kind == 'sgu' else hid
        glu = kind == 'glu'
        specs += [ParamSpec(f + 'layer_norm', 'scale', (d,)),
                  ParamSpec(f + 'linear', 'w', (d, h_in), interleave=glu), ParamSpec(f + 'linear', 'b', (h_in,), interleave=glu)]
        if kind == 'sgu':
            half = hid // 2
            specs += [ParamSpec(f + 'sgu/~/layer_norm', 'scale', (half,)),
                      ParamSpec(f + 'sgu', 'spatial_weights', (n, n)), ParamSpec(f + 'sgu', 'spatial_biases', (n, 1)),
                      ParamSpec(f + 'sgu/~/linear', 'w', (half, half)), ParamSpec(f + 'sgu/~/linear', 'b', (half,))]
        specs += [ParamSpec(f + 'linear_1', 'w', (h_out, d)), ParamSpec(f + 'linear_1', 'b', (d,))]
    specs += [ParamSpec(P + 'layer_norm', 'scale', (d,)),
              ParamSpec(P + 'linear', 'w', (d, V)), ParamSpec(P + 'linear', 'b', (V,))]
    return Layout(specs)


def _interleave(a):
    """[..., 2H] with columns (value | gate) -> columns (v0, g0, v1, g1, ...)"""
    H = a.shape[-1] // 2
    return np.stack((a[..., :H], a[..., H:]), axis=-1).reshape(a.shape)


def _deinterleave(a):
    return np.concatenate((a[..., 0::2], a[..., 1::2]), axis=-1)


class Acts:
    """One activation set: the buffers one forward pass runs on (B sequences of n positions, T = B * n token rows).
    `X` lists the residual stream at every LayerNorm input and `lay` one scratch dict per layer.  The training set keeps
    all of them (the backward pass reads them; in recompute mode the odd X and the layers alias one buffer each, see
    `training_set`) and its backward temporaries by name in `grad`; the inference set
    (`inplace`) repeats one residual buffer, updated in place, and one layer's scratch, and stores no GLU / GELU
    pre-activation (`u` is None)."""

    def __init__(self, B, n, tok, labels, X, lay, meanf, rstdf, yf, logits, inplace=False, rows=None, res=None, grad=None):
        self.B, self.n, self.T = B, n, B * n
        self.tok, self.labels, self.X, self.lay = tok, labels, X, lay
        self.meanf, self.rstdf, self.yf, self.logits = meanf, rstdf, yf, logits
        self.inplace = inplace
        self.rows = rows        # inference: [B, n+1] int32 staging of the input rows (one H2D copy per chunk)
        self.res = res          # inference: flat fp32 per-chunk results (see Engine.score)
        self.grad = grad        # training: {name: [T, ...] backward temporary}, shared by all layers

    def view(self, B, n):
        """the first B sequences of this set, cut to their first n positions (same memory): a ragged last chunk, a cut
        forward or a cut training step runs on the cached buffers.  `rows` is the contiguous (B, n+1) prefix of the
        staging buffer."""
        if (B, n) == (self.B, self.n):
            return self
        T = B * n
        cut = lambda t: None if t is None else t[:T]
        rows = None if self.rows is None else self.rows.view(-1)[:B * (n + 1)].view(B, n + 1)
        grad = None if self.grad is None else {k: cut(v) for k, v in self.grad.items()}
        return Acts(B, n, cut(self.tok), cut(self.labels), [cut(x) for x in self.X],
                    [{k: cut(v) for k, v in s.items()} for s in self.lay], cut(self.meanf), cut(self.rstdf), cut(self.yf),
                    cut(self.logits), self.inplace, rows, self.res, grad)


class Engine:
    def __init__(self, cfg, mixed_precision=False, device=None, recompute=False):
        L.require_device()
        self.cfg = cfg
        # recompute: the training set keeps one residual checkpoint per layer and the backward pass re-runs each layer's
        # forward from it (DESIGN.md §3.12); a way of running, not a property of the model
        self.recompute = bool(recompute)
        self.dev = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
        self.mp = bool(mixed_precision)
        self.act = torch.bfloat16 if self.mp else torch.float32
        self.act_dt = L.BF16 if self.mp else L.F32
        self.backend = L.BACKEND_TC if self.mp else L.BACKEND_SIMT
        self.kinds = layer_kinds(cfg['depth'], cfg['global_mlp_depth'], cfg['ff_glu'])
        # tensor-core (wgmma) attention kernels: bf16, dim_head 64, 64-aligned windows (checked below — no silent CUDA-core
        # fallback); the fp32 engine (mixed_precision=False) runs the exact CUDA-core kernels.  Two names for one flag
        # because bench.py reads both.
        self.attn_tc = self.attn_wgmma = self.mp
        d, n, w = cfg['dim'], cfg['seq_len'], cfg['window_size']
        self.d, self.n, self.w, self.V = d, n, w, cfg['num_tokens']
        self.h, self.dh = cfg['heads'], cfg['dim_head']
        self.I = self.h * self.dh
        self.hid = d * cfg['ff_mult']
        if n % w != 0:
            raise L.ProgenError('sequence length must be divisible by the window size')       # progen.py:80
        if self.dh not in (16, 32, 64, 128):
            raise L.ProgenError('dim_head must be one of 16/32/64/128')
        if d % 8 or self.I % 8 or self.V % 8:
            raise L.ProgenError('dim, heads*dim_head and num_tokens must be multiples of 8')
        if self.V > 384:
            raise L.ProgenError('num_tokens > 384 is not supported (embed_bwd keeps num_tokens x 32 fp32 bins in 48 KB of shared memory)')
        if self.mp and self.dh != 64:
            # the tensor-core attention kernels are built for dim_head 64; running another head size on the CUDA-core
            # kernel under mixed_precision would be a silent 10x slowdown, so it is refused (mixed_precision=False runs it)
            raise L.ProgenError(f'mixed_precision needs dim_head == 64 (got {self.dh}); use mixed_precision=False for other head sizes')
        if self.mp and w % 64:
            raise L.ProgenError(f'mixed_precision needs window_size % 64 == 0 (got {w}); use mixed_precision=False')
        if self.mp:
            bad = [k for k, v in dict(dim=d, inner=self.I, seq_len=n, num_tokens=self.V).items() if v % 64]
            if bad:
                raise L.ProgenError(f'mixed_precision (tensor-core path) needs {bad} to be multiples of 64')
        self.layout = build_param_specs(cfg)
        self.n_params_padded, self.num_params = self.layout.size, self.layout.num_params
        self.n_decay = self.layout.span([s for s in self.layout.specs if s.decay])[1]
        f32 = dict(device=self.dev, dtype=torch.float32)
        self.params = torch.zeros(self.n_params_padded, **f32)
        self.grads = torch.zeros(self.n_params_padded, **f32)
        self.params_lp = torch.zeros(self.n_params_padded, device=self.dev, dtype=torch.bfloat16) if self.mp else None
        self.wm = {}        # layer -> tril-masked compute copy of spatial_weights (act dtype)
        for i, kind in enumerate(self.kinds):
            if kind == 'sgu':
                self.wm[i] = torch.zeros(n, n, device=self.dev, dtype=self.act)
        # rotary tables: fixed_pos_embedding (progen.py:24-28), one (sin, cos) per frequency, computed in float64
        inv_freq = 1.0 / (10000 ** (np.arange(0, self.dh, 2, dtype=np.float64) / self.dh))
        ang = np.arange(n, dtype=np.float64)[:, None] * inv_freq[None, :]
        self.rot_sin = torch.tensor(np.sin(ang), **f32).contiguous()
        self.rot_cos = torch.tensor(np.cos(ang), **f32).contiguous()
        self.B = 0
        self.alloc_epoch = 0      # counts re-allocations of the training activations: a captured step holds for one epoch
        self.acts = None          # training activation set (ensure_batch)
        self._train_keys = ()     # the attributes ensure_batch set from training_set
        self.train_bytes = 0      # ... and the bytes they hold
        self.infer = None         # inference activation set (inference_acts), cached by row count
        self.loss = torch.zeros(1, device=self.dev)       # exists before the first batch: a rank without rows still reports 0
        self.loaded_token = None
        self.lora = None                  # lora.Adapters: the training set runs the adapted model with a frozen base
        self.teacher = None               # distillation (attach_teacher): a second Engine whose logits are the target
        self.dist = None                  # ... and the distillation head's buffers (ensure_distill)
        self.pol = None                   # policy-gradient head buffers (load_policy); its reference is self.teacher
        self.lib = L.load()
        self.num_sms = torch.cuda.get_device_properties(self.dev).multi_processor_count

    # ------------------------------------------------------------------------------------------ parameters
    def load_params(self, params):
        """haiku-shaped nested dict {module: {name: array}} (numpy or torch) -> flat engine layout on the device."""
        self.params.copy_(torch.from_numpy(self.layout.pack(params)))
        self.refresh_compute_copies()

    def export_params(self):
        return self.layout.unpack(self.params)

    def export_grads(self):
        return self.layout.unpack(self.base_grads())

    def base_grads(self):
        """the flat fp32 gradient of every parameter; released while adapters train (a LoRA Trainer) and allocated
        again, zeroed, by the next full-gradient path"""
        if self.grads is None:
            self.grads = torch.zeros(self.n_params_padded, device=self.dev, dtype=torch.float32)
        return self.grads

    def refresh_compute_copies(self):
        """bf16 mirror of all parameters + tril-masked SGU matrices; call after every parameter change."""
        st = L.stream()
        if self.mp:
            L.check(self.lib.progen_cast_f32(self.params.data_ptr(), self.params_lp.data_ptr(), L.BF16, self.n_params_padded, st),
                    'cast params')
        self.refresh_masked_copies()

    def refresh_masked_copies(self):
        st = L.stream()
        for i, wm in self.wm.items():
            src = self.Pf(P + f'ff{i}/~/sgu', 'spatial_weights')
            L.check(self.lib.progen_tril_cast(src.data_ptr(), wm.data_ptr(), self.act_dt, self.n, st), 'tril_cast')

    def W(self, module, name):
        """GEMM operand view of a parameter: bf16 mirror under mixed precision, fp32 master otherwise."""
        return self.layout.seg(self.params_lp if self.mp else self.params, module, name)

    def Pf(self, module, name):
        return self.layout.seg(self.params, module, name)

    def G(self, module, name):
        return self.layout.seg(self.base_grads(), module, name)

    # ------------------------------------------------------------------------------------------ workspaces
    def ensure_batch(self, B):
        """the training activation set (`training_set`) for B rows, in this engine's mode (resident or recompute);
        kept until B or the mode changes"""
        if B == self.B:
            return
        self.B = B
        self.alloc_epoch += 1                                       # activation buffers are re-allocated below: captured
                                                                    # CUDA graphs (Trainer.capture_graph) become invalid
        self.T = B * self.n
        self.acts = None
        for k in self._train_keys:                                  # release the old set before allocating the new one
            setattr(self, k, None)
        bufs, self.train_bytes = training_set(self.cfg, B, self.mp, self.recompute, self.dev)
        vars(self).update(bufs)                                     # self.X, self.lay, self.logits, self.dres, ...
        self._train_keys = tuple(bufs)
        # residue head (train_step): its B * n position buffers are sized for the head's outputs (ensure_residue)
        self.res_C, self.res = 0, None
        self.dist = None                                            # distillation head buffers (ensure_distill)
        self.pol = None                                             # policy-gradient head buffers (load_policy)
        grad = dict(dres=self.dres, dres_lp=self.dres_lp, dy=self.dy, dqkv=self.dqkv, datt=self.datt, delta=self.delta,
                    du=self.du, dh_=self.dh_, dlogits=self.dlogits, ce_w=self.ce_w, logp=self.logp)
        if 'sgu' in self.kinds:
            grad.update(dpj=self.dpj, dsg=self.dsg, dgp=self.dgp, dgn=self.dgn)
        self.acts = Acts(B, self.n, self.tok, self.labels, self.X, self.lay, self.meanf, self.rstdf, self.yf, self.logits,
                         grad=grad)

    def set_recompute(self, on):
        """switch the training set between resident and recomputed activations; a change re-allocates an existing set
        at once (advancing alloc_epoch, so captured steps are dropped before their next replay)"""
        on = bool(on)
        if on == self.recompute:
            return
        self.recompute = on
        if self.B:
            B, self.B = self.B, 0
            self.ensure_batch(B)

    def inference_acts(self, B):
        """Activation set of a forward pass that keeps no training state, for up to B sequences: one fp32 residual buffer
        [T, d] updated in place, one layer's scratch shared by every layer (no pre-activation store), the final LN output,
        the fp32 logits and the scoring outputs.  Allocated on first use and kept for later calls of the same or smaller
        row count, apart from the training set: `ensure_batch`, `alloc_epoch` and captured training graphs are untouched."""
        if self.infer is not None and self.infer.B >= B:
            return self.infer.view(B, self.n)
        self.infer = None                                       # release the smaller set before allocating the larger one
        n, d, I, hid, V = self.n, self.d, self.I, self.hid, self.V
        T = B * n
        dev, act = self.dev, self.act
        A = lambda *shape: torch.empty(*shape, device=dev, dtype=act)
        F = lambda *shape: torch.empty(*shape, device=dev, dtype=torch.float32)
        x = F(T, d)
        y, mean, rstd = A(T, d), F(T), F(T)
        s = dict(mean1=mean, rstd1=rstd, y1=y, qkv=A(T, 3 * I), att=A(T, I), lse=F(T, self.h), mean2=mean, rstd2=rstd, y2=y,
                 u=None, hact=A(T, hid))
        if 'sgu' in self.kinds:
            half = hid // 2
            gn, gp = A(T, half), A(T, half)
            # the gate output overwrites the normalised gate (dead once the spatial GEMM has read it) and the projection
            # overwrites the spatial GEMM output (dead once the gate has read it)
            s.update(mean3=F(T), rstd3=F(T), gn=gn, gp=gp, sg=gn, pj=gp)
        nl = len(self.kinds)
        self.infer = Acts(B, n, torch.empty(T, device=dev, dtype=torch.int32), torch.empty(T, device=dev, dtype=torch.int32),
                          [x] * (2 * nl + 1), [s] * nl, F(T), F(T), A(T, d), F(T, V), inplace=True,
                          rows=torch.empty(B, n + 1, device=dev, dtype=torch.int32), res=F(B * (2 + n + d)))
        return self.infer

    # ------------------------------------------------------------------------------------------ GEMM helpers
    def _mm(self, **kw):
        L.gemm(backend=self.backend, in_dtype=self.act_dt, **kw)

    def lora_fwd(self, x, K, module, N, acts):
        """adapters: u = x A of projection `module` (input x [T, K], N outputs; T from the training set or its view
        `acts`) -> the tail (u, s B) of its GEMM"""
        lo = self.lora
        if lo is None:
            return {}
        u, seg = lo.u[module][:acts.T], lo.layout.seg
        self.fwd_gemm(x, K, seg(lo.lp, module, 'lora_a'), lo.r, u, acts=acts)
        return dict(A2=u, lda2=lo.r, B2=seg(lo.lp, module, 'lora_b'), ldb2=N, K2=lo.r)

    def lora_bwd(self, x, K, module, dy, N, acts):
        """adapters: from the projection's output gradient dy [T, N], g' = s g = dy (s B)^T, dB += u^T dy (scaled by s
        after the backward pass), dA += x^T g' -> the tail (g', A^T) of its input-gradient GEMM"""
        lo = self.lora
        if lo is None:
            return {}
        seg = lo.layout.seg
        g, A = lo.g[:acts.T], seg(lo.lp, module, 'lora_a')
        self.dgrad_gemm(dy, N, seg(lo.lp, module, 'lora_b'), lo.r, g, acts=acts)
        self.wgrad_gemm(lo.u[module][:acts.T], lo.r, dy, N, seg(lo.grads, module, 'lora_b'), acts=acts)
        self.wgrad_gemm(x, K, g, lo.r, seg(lo.grads, module, 'lora_a'), acts=acts)
        return dict(A2=g, lda2=lo.r, B2=A, ldb2=lo.r, K2=lo.r)

    def fwd_gemm(self, x, K, w, N, out, epi=L.EPI_STORE, out_dtype=None, acts=None, **kw):
        """out[T,N] = x[T,K] @ w[K,N]  (w stored (in, out) like hk.Linear: MN-major B operand); T from `acts` (default:
        the training set)"""
        self._mm(M=(acts or self.acts).T, N=N, K=K, A=x, lda=K, B=w, ldb=N, b_mn=True, out=out, ldo=kw.pop('ldo', N), epi=epi,
                 out_dtype=self.act_dt if out_dtype is None else out_dtype, **kw)

    def dgrad_gemm(self, dy, N_out, w, K_in, out, epi=L.EPI_STORE, acts=None, **kw):
        """out[T,K_in] = dy[T,N_out] @ w[K_in,N_out]^T  (w rows are the output features: K-major B operand)"""
        self._mm(M=(acts or self.acts).T, N=K_in, K=N_out, A=dy, lda=N_out, B=w, ldb=N_out, out=out, ldo=kw.pop('ldo', K_in), epi=epi,
                 out_dtype=self.act_dt, **kw)

    def wgrad_gemm(self, x, K_in, dy, N_out, dw, acts=None):
        """dw[K_in,N_out] += x[T,K_in]^T @ dy[T,N_out]  (both operands MN-major, the token dimension is K)"""
        split = self.wgrad_split(K_in, N_out, acts) if self.backend == L.BACKEND_TC else 1
        self._mm(M=K_in, N=N_out, K=(acts or self.acts).T, A=x, lda=K_in, a_mn=True, B=dy, ldb=N_out, b_mn=True, out=dw, ldo=N_out,
                 epi=L.EPI_ACCUM, out_dtype=L.F32, split_k=split, atomic=split > 1)

    def wgrad_split(self, K_in, N_out, acts=None):
        """K split of a weight-gradient GEMM (one CTA per 128 x 128 output tile and K slice): the split in 1..8 whose CTAs
        fill the largest fraction of their waves over the SMs, the smallest such split on ties"""
        tiles = ((K_in + 127) // 128) * ((N_out + 127) // 128)
        fill = lambda s: tiles * s / (-(-tiles * s // self.num_sms) * self.num_sms)
        return max(range(1, min(8, max(1, (acts or self.acts).T // 64)) + 1), key=lambda s: (round(fill(s), 6), -s))

    def colsum(self, t, N, out, ld=None, acts=None):
        L.check(self.lib.progen_colsum(t.data_ptr(), N if ld is None else ld, L.dt(t), out.data_ptr(), (acts or self.acts).T, N,
                                       L.stream()), 'colsum')

    def ln_fwd(self, x, ldx, scale, y, ldy, mean, rstd, dcols, shift, acts=None):
        a = acts or self.acts
        L.check(self.lib.progen_ln_shift_fwd(x.data_ptr(), ldx, L.dt(x), scale.data_ptr(), y.data_ptr(), ldy, L.dt(y),
                                             mean.data_ptr(), rstd.data_ptr(), a.T, dcols, a.n, int(shift), L.stream()),
                'ln_fwd')

    # ------------------------------------------------------------------------------------------ forward
    def forward(self, ids):
        """ids: (B, n) integer array/tensor -> self.logits fp32 [T, V]; keeps everything the backward pass needs."""
        B = ids.shape[0]
        self.ensure_batch(B)
        self.tok.copy_(torch.as_tensor(ids).reshape(-1).to(device=self.dev, dtype=torch.int32), non_blocking=True)
        self._forward_device()
        return self.logits

    def prefill(self, ids, P, sink):
        """Inference forward of ids [Bs, n] that hands every layer's state to `sink(layer, name, buf, P)` instead of
        computing logits: name 'qkv' (the rotated q|k|v [T, 3 inner]) and 'y1' (the attention block's shifted LN output
        [T, d]) after the QKV GEMM, 'y2' (the feed-forward block's) after its LayerNorm, and in gMLP layers 'gn' (the
        normalised gate [T, hid/2]) after the spatial GEMM, before the gate overwrites it.  The sink must read what it
        needs before it returns (the inference set reuses its buffers across layers).  Causality makes positions < P and
        the shifted half of LN row P depend on ids[:, :P] alone.  Each row's result does not depend on the other rows."""
        Bs = ids.shape[0]
        if tuple(ids.shape[1:]) != (self.n,) or not 0 < P < self.n:
            raise L.ProgenError(f'prefill: ids must be (B, {self.n}) and 0 < P < {self.n}')
        acts = self.inference_acts(Bs)
        acts.tok.copy_(torch.as_tensor(ids).reshape(-1).to(device=self.dev, dtype=torch.int32))
        self._forward_device(acts, sink=lambda i, name, buf: sink(i, name, buf, P))

    def _forward_device(self, acts=None, sink=None, logits=True):
        """forward pass on activation set `acts` (default: the training set, which keeps what the backward pass reads)
        over its acts.n positions per row; with a `sink` (Engine.prefill) the layers' state goes to it and the logits
        head is skipped; `logits=False` stops after the final LayerNorm (acts.yf), for the property head.  Every mixing
        op is causal, so a forward on a view cut to the first n positions computes exactly those positions of the full
        one (DESIGN.md §3.6)."""
        acts = self.acts if acts is None else acts
        d, T = self.d, acts.T
        tail = self._lora_tail(acts)
        L.check(self.lib.progen_embed_fwd(acts.tok.data_ptr(), self.Pf(P + 'embed', 'embeddings').data_ptr(),
                                          acts.X[0].data_ptr(), T, d, self.V, L.stream()), 'embed_fwd')
        for i in range(len(self.kinds)):
            self._layer_forward(i, acts, tail, sink)
        if sink is not None:
            return
        # ---- to_logits (progen.py:219-222)
        xl = acts.X[-1]
        self.ln_fwd(xl, d, self.Pf(P + 'layer_norm', 'scale'), acts.yf, d, acts.meanf, acts.rstdf, d, False, acts=acts)
        if not logits:
            return
        self.fwd_gemm(acts.yf, d, self.W(P + 'linear', 'w'), self.V, acts.logits, bias=self.Pf(P + 'linear', 'b'), out_dtype=L.F32,
                      acts=acts)

    def _lora_tail(self, acts):
        """the forward's adapter tails on activation set `acts` (lora_fwd): adapters run on the training set (or its cut
        view) only"""
        lo = None if acts.inplace else self.lora
        if lo is None:
            return lambda *a: {}
        lo.activations(self.acts.T)
        return lambda *a: self.lora_fwd(*a, acts=acts)

    def _layer_forward(self, i, acts, tail, sink=None, through='all'):
        """layer i of the forward on activation set `acts`, from its input acts.X[2i]: with through='all' up to its
        output acts.X[2i+2]; with through='ff_in' (recompute_layer) it stops before the feed-forward output GEMM, the
        one launch that writes the next layer's input.  `tail` gives each projection's adapter tail (_lora_tail)."""
        lib, st, kind, s = self.lib, L.stream(), self.kinds[i], acts.lay[i]
        cfg, d, I, hid, T, n = self.cfg, self.d, self.I, self.hid, acts.T, acts.n
        shift = cfg['shift_tokens']
        a, f = P + f'attn{i}/~/', P + f'ff{i}/~/'
        # in place (inference): x0 = x1 = x2 is one buffer, and the residual epilogue without aux reads its output
        x0, x1, x2 = acts.X[2 * i], acts.X[2 * i + 1], acts.X[2 * i + 2]
        # ---- LocalAttention (progen.py:73-103)
        self.ln_fwd(x0, d, self.Pf(a + 'layer_norm', 'scale'), s['y1'], d, s['mean1'], s['rstd1'], d, shift, acts=acts)
        self.fwd_gemm(s['y1'], d, self.W(a + 'linear', 'w'), 3 * I, s['qkv'], epi=L.EPI_ROTARY, rot_sin=self.rot_sin,
                      rot_cos=self.rot_cos, seq_len=n, dim_head=self.dh, acts=acts, **tail(s['y1'], d, a + 'linear', 3 * I))
        if sink is not None:
            sink(i, 'qkv', s['qkv'])
            sink(i, 'y1', s['y1'])
        self.attn_fwd(s['qkv'], s['att'], s['lse'], acts=acts)
        self.fwd_gemm(s['att'], I, self.W(a + 'linear_1', 'w'), d, x1, epi=L.EPI_RESIDUAL, bias=self.Pf(a + 'linear_1', 'b'),
                      aux=None if acts.inplace else x0, ldaux=d, acts=acts, **tail(s['att'], I, a + 'linear_1', d))
        # ---- FeedForward (progen.py:131-149); s['u'] is None in the inference set: no pre-activation store
        self.ln_fwd(x1, d, self.Pf(f + 'layer_norm', 'scale'), s['y2'], d, s['mean2'], s['rstd2'], d, shift, acts=acts)
        if sink is not None:
            sink(i, 'y2', s['y2'])
        if kind == 'glu':
            self.fwd_gemm(s['y2'], d, self.W(f + 'linear', 'w'), 2 * hid, s['hact'], epi=L.EPI_GLU, ldo=hid, out2=s['u'],
                          ldo2=2 * hid, bias=self.Pf(f + 'linear', 'b'), acts=acts, **tail(s['y2'], d, f + 'linear', 2 * hid))
            last, last_k = s['hact'], hid
        else:
            self.fwd_gemm(s['y2'], d, self.W(f + 'linear', 'w'), hid, s['hact'], epi=L.EPI_GELU, out2=s['u'], ldo2=hid,
                          bias=self.Pf(f + 'linear', 'b'), acts=acts, **tail(s['y2'], d, f + 'linear', hid))
            last, last_k = s['hact'], hid
        if kind == 'sgu':
            half = hid // 2
            g = f + 'sgu'
            gate = s['hact'][:, half:]
            self.ln_fwd(gate, hid, self.Pf(g + '/~/layer_norm', 'scale'), s['gn'], half, s['mean3'], s['rstd3'], half, False,
                        acts=acts)
            # gate_b = tril(W) @ gn_b for every sequence b; masked K tiles are skipped (causal=1)
            self._mm(M=n, N=half, K=n, A=self.wm[i], lda=self.n, B=s['gn'], ldb=half, b_mn=True, out=s['gp'], ldo=half,
                     out_dtype=self.act_dt, batch=acts.B, b_batch_rows=n, d_batch_rows=n, causal=1)
            if sink is not None:
                sink(i, 'gn', s['gn'])
            L.check(lib.progen_sgu_gate_fwd(s['hact'].data_ptr(), hid, s['gp'].data_ptr(), half,
                                            self.Pf(g, 'spatial_biases').data_ptr(), s['sg'].data_ptr(), half, self.act_dt,
                                            T, half, n, st), 'sgu_gate_fwd')
            self.fwd_gemm(s['sg'], half, self.W(g + '/~/linear', 'w'), half, s['pj'], bias=self.Pf(g + '/~/linear', 'b'),
                          acts=acts)
            last, last_k = s['pj'], half
        if through == 'ff_in':
            return
        self.fwd_gemm(last, last_k, self.W(f + 'linear_1', 'w'), d, x2, epi=L.EPI_RESIDUAL, bias=self.Pf(f + 'linear_1', 'b'),
                      aux=None if acts.inplace else x1, ldaux=d, acts=acts, **tail(last, last_k, f + 'linear_1', d))

    def recompute_layer(self, i, acts=None):
        """re-run layer i's forward on the training set (or its cut view `acts`) from its checkpoint X[2i], up to the
        feed-forward output GEMM: its scratch and X[2i+1] (shared by every layer in recompute mode) and its adapters' u
        then hold what the forward wrote, bitwise (the same launches on the same inputs; DESIGN.md §3.12).  The
        feed-forward output adapter's u is kept per layer and is not re-run."""
        acts = self.acts if acts is None else acts
        self._layer_forward(i, acts, self._lora_tail(acts), through='ff_in')

    def attn_fwd(self, qkv, out, lse, acts=None):
        a = acts or self.acts
        B, n = a.B, a.n
        if self.attn_tc:
            L.check(self.lib.progen_local_attn_fwd_tc(qkv.data_ptr(), out.data_ptr(), lse.data_ptr(), B, n, self.w, self.h,
                                                      self.dh, L.stream()), 'local_attn_fwd')
            return
        L.check(self.lib.progen_local_attn_fwd_simt(qkv.data_ptr(), out.data_ptr(), lse.data_ptr(), self.act_dt, B, n,
                                                    self.w, self.h, self.dh, L.stream()), 'local_attn_fwd')

    def attn_bwd(self, qkv, out, dout, lse, dqkv, acts=None):
        """attention backward on the training set or its cut view `acts`; a cut that ends inside a window runs the
        `_cut_` entry point, every whole-window step the whole-window one"""
        a = acts or self.acts
        B, n, delta = a.B, a.n, a.grad['delta']
        lib = self.lib
        if self.attn_tc:
            fn = lib.progen_local_attn_bwd_tc if n % self.w == 0 else lib.progen_local_attn_bwd_cut_tc
            L.check(fn(qkv.data_ptr(), out.data_ptr(), dout.data_ptr(), lse.data_ptr(), dqkv.data_ptr(), delta.data_ptr(),
                       self.rot_sin.data_ptr(), self.rot_cos.data_ptr(), B, n, self.w, self.h, self.dh, L.stream()),
                    'local_attn_bwd')
            return     # rotary backward is fused into the kernel's epilogue
        fn = lib.progen_local_attn_bwd_simt if n % self.w == 0 else lib.progen_local_attn_bwd_cut_simt
        L.check(fn(qkv.data_ptr(), out.data_ptr(), dout.data_ptr(), lse.data_ptr(), dqkv.data_ptr(), delta.data_ptr(), self.act_dt,
                   B, n, self.w, self.h, self.dh, L.stream()), 'local_attn_bwd')

    # ------------------------------------------------------------------------------------------ scoring (inference)
    def _chunks(self, rows, batch_size, n):
        """The inference forward's chunks of rows (N >= 1, seq_len + 1), a host int32 tensor, batch_size rows at a time,
        each cut to its first n positions: yields (r0, acts), acts the (B, n) view of the inference set with the chunk's
        ids and labels in acts.tok / acts.labels, staged by one H2D copy of the contiguous (B, n + 1) block acts.rows."""
        full = self.inference_acts(min(batch_size, rows.shape[0]))
        for r0 in range(0, rows.shape[0], batch_size):
            chunk = rows[r0:r0 + batch_size, :n + 1]
            B = chunk.shape[0]
            acts = full.view(B, n)
            acts.rows.copy_(chunk)
            acts.tok.view(B, n).copy_(acts.rows[:, :-1])
            acts.labels.view(B, n).copy_(acts.rows[:, 1:])
            yield r0, acts

    def score(self, data, batch_size=64, tokens=False, embeddings=False, length=None):
        """data: (N, n+1) integer rows (ids = data[:, :-1], labels = data[:, 1:], as in loss_and_grad) -> dict of numpy
        arrays: log_likelihood [N] (sum of the label log-probabilities under the loss mask), num_tokens [N] (mask size);
        token_logp [N, n] with `tokens`; embedding [N, d] (masked mean of the final LayerNorm output) with `embeddings`.
        Runs the forward on the inference activation set, `batch_size` rows at a time: one H2D copy of the rows, the
        forward, progen_token_logprob (+ progen_masked_mean_pool) and one D2H copy of the results per chunk.
        `length` (default seq_len): run the forward over the first `length` positions of every row only, on a
        (B, length) view of the same activation set.  It must be seq_len or a multiple of CUT_ALIGN that covers every
        counted position of every row (`cut_length`); the results are then bitwise those of the full-length forward, and
        token_logp is zero beyond `length`."""
        rows = torch.as_tensor(np.asarray(data).astype(np.int32)) if not isinstance(data, torch.Tensor) else data
        rows = rows.to(device='cpu', dtype=torch.int32)
        if rows.dim() != 2 or rows.shape[1] != self.n + 1:
            raise L.ProgenError(f'score: rows must be (B, seq_len + 1 = {self.n + 1}), got {tuple(rows.shape)}')   # Q12
        if batch_size < 1:
            raise L.ProgenError(f'score: batch_size must be >= 1, got {batch_size}')
        N, n, d = rows.shape[0], self.n, self.d
        cut = n if length is None else check_length(rows[:, 1:].numpy(), length, 'score')
        out = dict(log_likelihood=np.zeros(N, np.float32), num_tokens=np.zeros(N, np.int64))
        if tokens:
            out['token_logp'] = np.zeros((N, n), np.float32)
        if embeddings:
            out['embedding'] = np.zeros((N, d), np.float32)
        if N == 0:
            return out
        lib, st = self.lib, L.stream()
        for r0, acts in self._chunks(rows, batch_size, cut):
            B, T, res = acts.B, acts.T, acts.res
            self._forward_device(acts)
            # results, packed for one D2H copy: seq_ll [B] | seq_count [B] | logp [T] | embedding [B, d]
            ll, cnt, lp, emb = res[:B], res[B:2 * B], res[2 * B:2 * B + T], res[2 * B + T:2 * B + T + B * d]
            L.check(lib.progen_token_logprob(acts.logits.data_ptr(), L.F32, acts.labels.data_ptr(), lp.data_ptr(), ll.data_ptr(),
                                             cnt.data_ptr(), B, cut, self.V, st), 'token_logprob')
            if embeddings:
                L.check(lib.progen_masked_mean_pool(acts.yf.data_ptr(), d, self.act_dt, acts.labels.data_ptr(), emb.data_ptr(),
                                                    B, cut, d, st), 'masked_mean_pool')
            used = 2 * B + (T + B * d if embeddings else T if tokens else 0)
            host = res[:used].cpu().numpy()
            out['log_likelihood'][r0:r0 + B] = host[:B]
            out['num_tokens'][r0:r0 + B] = host[B:2 * B].astype(np.int64)
            if tokens:
                out['token_logp'][r0:r0 + B, :cut] = host[2 * B:2 * B + T].reshape(B, cut)
            if embeddings:
                out['embedding'][r0:r0 + B] = host[2 * B + T:].reshape(B, d)
        return out

    # ------------------------------------------------------------------------------------------ loss + backward
    def loss_and_grad(self, data, global_batch=None, zero_grads=True):
        """data: (B, n+1) integer rows -> (device scalar loss, grads accumulated into self.grads).
        Mirrors utils.py:61-76: ids = data[:, :-1], labels = data[:, 1:], mean over rows of the masked CE.
        `global_batch` (DDP): scale by 1/global_batch so that a SUM all-reduce yields the global-mean gradient.
        The step runs at the rows' row_length (DESIGN.md §3.10)."""
        n = self.row_length(data)
        B = self.load_batch(data, n)
        self.train_step((), global_batch or B, zero_grads, length=n)
        return self.loss

    def row_length(self, data, length=None, what='training step'):
        """the row length a training step on rows `data` (B, n+1) runs at: check_length of host rows (None: their
        cut_length); rows on the device run at seq_len (their cut length would need a host sync)"""
        if isinstance(data, torch.Tensor) and data.is_cuda:
            if length not in (None, self.n):
                raise L.ProgenError(f'{what}: rows on the device run at seq_len ({self.n}), got length {length!r}')
            return self.n
        rows = np.asarray(data)
        if rows.ndim != 2 or rows.shape[1] != self.n + 1:
            raise L.ProgenError(f'{what}: rows must be (B, seq_len + 1 = {self.n + 1}), got {rows.shape}')
        return check_length(rows[:, 1:], length, what)

    def load_batch(self, data, length=None):
        """host (or device) rows (B, n+1) -> self.tok / self.labels, cut to their first `length` positions (default
        seq_len) in the layout of the training set's (B, length) view; returns B"""
        data = torch.as_tensor(np.asarray(data).astype(np.int32) if not isinstance(data, torch.Tensor) else data)
        B = data.shape[0]
        self.ensure_batch(B)
        n = self.n if length is None else length
        dd = data[:, :n + 1].to(device=self.dev, dtype=torch.int32, non_blocking=True)
        self.tok[:B * n].view(B, n).copy_(dd[:, :-1])
        self.labels[:B * n].view(B, n).copy_(dd[:, 1:])
        return B

    def train_step(self, objective, global_rows, zero_grads=True, backward=True, length=None):
        """forward + loss head + backward of one training objective on rows resident in self.tok / self.labels.
        `objective` (also the tail of Trainer's graph key) selects the loss head:
          ()                    the language-model loss: the masked cross entropy, mean over rows (utils.py:45-59);
          ('preference', beta)  the preference (DPO) loss (DESIGN.md §3.7) over the resident rows as pairs, rows 0..P-1
                                chosen and row i + P the rejected row of pair i, with their reference log-likelihoods in
                                self.ref (load_preference); self.stats [P, 4] holds each pair's (s(chosen), s(rejected),
                                z, loss);
          ('property', task)    the property head on the pooled embedding (DESIGN.md §3.9), task L.TASK_REGRESSION or
                                L.TASK_CLASSIFICATION, targets in self.ptarget / self.pclass (load_property); the
                                forward stops after the final LayerNorm.  Needs
                                adapters with a head (lora.Adapters with head_outputs): the base stays frozen;
          ('residue', task)     the same head at every position (DESIGN.md §3.11), mean over the labelled positions,
                                targets in self.res (load_residue); like 'property' otherwise.  The loss is the mean
                                over the micro-batch's own labelled positions: global_rows does not scale it.
          ('distill', tau, alpha)  distillation from the attached teacher (DESIGN.md §3.13): the teacher's forward on
                                the rows load_distill staged in its inference set, at teacher_length(length), then the
                                student's forward, progen_distill_head ((1 - alpha) tau^2 KL + alpha CE per row, mean over
                                rows; per-row (KL, CE) in self.dist['stats']) and the LM backward from dlogits.
          ('policy', beta)      the policy-gradient loss (DESIGN.md §3.14) on the spans and advantages load_policy staged:
                                with beta > 0 the attached reference's (self.teacher) forward first, as for 'distill',
                                then the policy's forward, progen_policy_head (per row the span mean of -A logp + beta KL,
                                per-row (logp, KL, N) in self.pol['stats']) and the LM backward from dlogits.
        The loss is scaled by 1/global_rows (the preference loss: 1/global pairs), so that a SUM all-reduce of the
        per-rank gradients is the global mean.  With adapters (self.lora) no base gradient is computed.
        `backward=False`: the forward and the loss only (a validation loss), no gradient.
        `length` (default seq_len): run on the first `length` positions of every row only, on the (B, length) view of
        the training set (DESIGN.md §3.10); it must cover every counted position of the rows (check_length).  Nothing
        is allocated per length."""
        lib, st, lo, d = self.lib, L.stream(), self.lora, self.d
        a = self.acts.view(self.B, self.n if length is None else int(length))
        g = a.grad
        kind = objective[0] if objective else None
        pairs = self.B // 2
        if kind == 'preference' and 2 * pairs != self.B:
            raise L.ProgenError(f'preference step: {pairs} pairs need {2 * pairs} resident rows, have {self.B}')
        if kind in ('property', 'residue') and (lo is None or not lo.head_outputs):
            raise L.ProgenError(f'{kind} step: needs adapters with a property head (the base stays frozen)')
        if kind == 'residue' and self.res_C != lo.head_outputs:
            raise L.ProgenError(f'residue step: no targets of a {lo.head_outputs}-output head are loaded (load_residue)')
        if not zero_grads and lo is not None:
            # the backward pass ends by scaling the whole B gradient by s (Adapters.scale_b_grads): an accumulated one
            # would be scaled twice
            raise L.ProgenError('adapters: gradients cannot accumulate across steps (zero_grads=False)')
        if kind == 'policy' and self.pol is None:
            raise L.ProgenError('policy step: no spans and advantages are loaded (load_policy)')
        if kind == 'distill' or (kind == 'policy' and objective[1] > 0):
            ta = self._teacher_view(a.B, a.n)
            self.teacher._forward_device(ta)
        self._forward_device(a, logits=kind not in ('property', 'residue'))
        if kind is None:
            self.loss.zero_()
        if zero_grads and backward:
            self.train_grads().zero_()
        if kind is None:
            L.check(lib.progen_ce_fwd_bwd(a.logits.data_ptr(), L.F32, a.labels.data_ptr(), g['ce_w'].data_ptr(),
                                          self.loss.data_ptr(), g['dlogits'].data_ptr() if backward else 0, self.act_dt,
                                          a.B, a.n, self.V, 1.0 / global_rows, st), 'ce_fwd_bwd')
        elif kind == 'preference':
            L.check(lib.progen_preference_head(a.logits.data_ptr(), L.F32, a.labels.data_ptr(), self.ref.data_ptr(),
                                               g['logp'].data_ptr(), self.seq_ll.data_ptr(), self.seq_count.data_ptr(),
                                               g['ce_w'].data_ptr(), self.stats.data_ptr(), self.loss.data_ptr(),
                                               self.ce_scratch.data_ptr(), g['dlogits'].data_ptr(), self.act_dt, pairs,
                                               a.n, self.V, objective[1], 1.0 / global_rows, st), 'preference_head')
        elif kind == 'residue':
            r, C = self.res, lo.head_outputs
            y, cls = (r['y'].data_ptr(), 0) if objective[1] == L.TASK_REGRESSION else (0, r['cls'].data_ptr())
            L.check(lib.progen_residue_head(a.yf.data_ptr(), d, self.act_dt, lo.head(lo.params, 'w').data_ptr(),
                                            lo.head(lo.params, 'b').data_ptr(), a.B, a.n, d, C, objective[1], y, cls,
                                            r['pred'].data_ptr(), r['loss'].data_ptr(), r['count'].data_ptr(),
                                            self.loss.data_ptr(), r['dpred'].data_ptr(), g['dy'].data_ptr(), d, st),
                    'residue_head')
            if backward:
                L.check(lib.progen_residue_head_wgrad(a.yf.data_ptr(), d, self.act_dt, r['dpred'].data_ptr(), y, cls, a.B,
                                                      a.n, d, C, r['ws'].data_ptr(), lo.head(lo.grads, 'w').data_ptr(),
                                                      lo.head(lo.grads, 'b').data_ptr(), st), 'residue_head_wgrad')
        elif kind == 'distill':
            dist = self.dist
            L.check(lib.progen_distill_head(a.logits.data_ptr(), L.F32, ta.logits.data_ptr(), ta.n, a.labels.data_ptr(),
                                            g['ce_w'].data_ptr(), dist['scratch'].data_ptr(), dist['stats'].data_ptr(),
                                            self.loss.data_ptr(), g['dlogits'].data_ptr(), self.act_dt, a.B, a.n, self.V,
                                            objective[1], objective[2], 1.0 / global_rows, st), 'distill_head')
        elif kind == 'policy':
            pol, beta = self.pol, objective[1]
            L.check(lib.progen_policy_head(a.logits.data_ptr(), L.F32, ta.logits.data_ptr() if beta > 0 else 0,
                                           ta.n if beta > 0 else a.n, a.labels.data_ptr(), pol['span'].data_ptr(),
                                           pol['adv'].data_ptr(), pol['scratch'].data_ptr(), pol['stats'].data_ptr(),
                                           self.loss.data_ptr(), g['dlogits'].data_ptr(), self.act_dt, a.B, a.n, self.V,
                                           beta, 1.0 / global_rows, st), 'policy_head')
        else:
            B, C, reg = a.B, lo.head_outputs, objective[1] == L.TASK_REGRESSION
            L.check(lib.progen_masked_mean_pool(a.yf.data_ptr(), d, self.act_dt, a.labels.data_ptr(),
                                                self.emb.data_ptr(), B, a.n, d, st), 'masked_mean_pool')
            L.check(lib.progen_property_head(self.emb.data_ptr(), lo.head(lo.params, 'w').data_ptr(),
                                             lo.head(lo.params, 'b').data_ptr(), B, d, C, objective[1],
                                             self.ptarget.data_ptr() if reg else 0, 0 if reg else self.pclass.data_ptr(),
                                             1.0 / global_rows, self.pred.data_ptr(), self.prow_loss.data_ptr(),
                                             self.loss.data_ptr(), self.dpred.data_ptr(), lo.head(lo.grads, 'w').data_ptr(),
                                             lo.head(lo.grads, 'b').data_ptr(), self.demb.data_ptr(), st), 'property_head')
        if not backward:
            return
        # the residue head has written d loss / d (final LayerNorm output) into g['dy'] itself
        if kind == 'property':
            L.check(lib.progen_masked_mean_pool_bwd(self.demb.data_ptr(), a.labels.data_ptr(), g['dy'].data_ptr(), d,
                                                    self.act_dt, a.B, a.n, d, st), 'masked_mean_pool_bwd')
        elif kind != 'residue':
            hw = P + 'linear'
            if lo is None:
                self.colsum(g['dlogits'], self.V, self.G(hw, 'b'), acts=a)
                self.wgrad_gemm(a.yf, d, g['dlogits'], self.V, self.G(hw, 'w'), acts=a)
            self.dgrad_gemm(g['dlogits'], self.V, self.W(hw, 'w'), d, g['dy'], acts=a)
        self._backward_body(a)

    def train_grads(self):
        """the flat gradient buffer a training step writes: the adapters' with adapters (the base is frozen)"""
        return self.base_grads() if self.lora is None else self.lora.grads

    def load_preference(self, rows, ref, length=None):
        """rows (2P, n+1): the chosen rows, then their rejected rows; ref [2P] float32: the reference log-likelihoods in
        the same order -> self.tok / self.labels (cut to `length` as in load_batch) / self.ref; returns P"""
        B = self.load_batch(rows, length)
        self.ref.copy_(torch.as_tensor(np.asarray(ref, np.float32)), non_blocking=True)
        return B // 2

    def preference_stats(self, pairs):
        """the last preference step's per-pair statistics as numpy float32 [pairs]"""
        st = self.stats[:pairs].cpu().numpy() if pairs else np.zeros((0, 4), np.float32)
        return dict(policy_chosen=st[:, 0].copy(), policy_rejected=st[:, 1].copy(), margin=st[:, 2].copy(),
                    loss=st[:, 3].copy())

    # ------------------------------------------------------------------------------------------ distillation
    def attach_teacher(self, teacher):
        """make Engine `teacher` (checked by distill.check_teacher) the target of 'distill' steps.  A teacher keeps only
        its parameters, their compute copies and its inference set: its base gradient and any training set are released
        (a later training step of its own allocates them again)."""
        self.teacher = teacher
        teacher.lora = None
        teacher.grads = None
        if teacher.B:
            teacher.alloc_epoch += 1
            teacher.B, teacher.acts, teacher.dist, teacher.pol, teacher.res_C, teacher.res = 0, None, None, None, 0, None
            for k in teacher._train_keys:
                setattr(teacher, k, None)
            teacher._train_keys, teacher.train_bytes = (), 0

    def _teacher_view(self, B, length):
        """the (B, teacher_length(length)) view of the teacher's inference set that load_distill filled"""
        from .distill import teacher_length
        t = self.teacher
        if t is None or t.infer is None or t.infer.B < B:
            raise L.ProgenError('no teacher or reference rows are loaded (attach_teacher, then load_distill or '
                                'load_policy)')
        return t.infer.view(B, teacher_length(length, t.n))

    def ensure_distill(self):
        """the distillation head's buffers for the training set's B rows: the per-position (KL, CE) scratch [2 B n] and
        the per-row stats [B, 2]; a cut step uses their prefix.  Kept until the batch size changes (ensure_batch)."""
        if self.dist is None:
            F = lambda *shape: torch.zeros(*shape, device=self.dev, dtype=torch.float32)
            self.dist = dict(scratch=F(2 * self.T), stats=F(self.B, 2))
        return self.dist

    def load_distill(self, data, length=None):
        """rows (B, n+1) -> the student's self.tok / self.labels as load_batch, and the same rows, zero-padded to the
        teacher's seq_len + 1, into the (B, teacher_length(length)) view of the teacher's inference set (allocated for B
        rows when it holds fewer); returns B"""
        B = self.load_batch(data, length)
        self.ensure_distill()
        self._stage_teacher(data, B, length)
        return B

    def _stage_teacher(self, data, B, length):
        """rows `data`, zero-padded to the attached teacher's seq_len + 1, into the (B, teacher_length(length)) view of
        its inference set (allocated for B rows when it holds fewer)"""
        from .distill import teacher_length
        t = self.teacher
        Lt = teacher_length(self.n if length is None else length, t.n)
        ta = t.inference_acts(B).view(B, Lt)
        rows = torch.as_tensor(np.asarray(data).astype(np.int32) if not isinstance(data, torch.Tensor) else data)
        k = min(Lt, rows.shape[1])
        tok = ta.tok.view(B, Lt)
        if k < Lt:
            tok.zero_()
        tok[:, :k].copy_(rows[:, :k].to(device=self.dev, dtype=torch.int32), non_blocking=True)

    def distill_stats(self, rows):
        """the last distillation step's per-row (KL, CE) as numpy float32 [rows] arrays"""
        if not rows or self.dist is None:
            return dict(kl=np.zeros(0, np.float32), ce=np.zeros(0, np.float32))
        st = self.dist['stats'][:rows].cpu().numpy()
        return dict(kl=st[:, 0].copy(), ce=st[:, 1].copy())

    # ------------------------------------------------------------------------------------------ policy gradient
    def load_policy(self, rows, span, advantage, length=None, reference=False):
        """rows (B, n+1) -> self.tok / self.labels as load_batch; span (B, 2) int32 and advantage [B] float32 (checked by
        policy.check_policy_batch) into the head's device buffers, allocated with the training set for its B rows; with
        `reference` (a step with beta > 0) the same rows into the attached reference's inference set, as load_distill
        does for a teacher.  Returns B."""
        B = self.load_batch(rows, length)
        if self.pol is None:
            F = lambda *shape: torch.zeros(*shape, device=self.dev, dtype=torch.float32)
            self.pol = dict(span=torch.zeros(self.B, 2, device=self.dev, dtype=torch.int32), adv=F(self.B),
                            scratch=F(2 * self.T), stats=F(self.B, 3))
        self.pol['span'][:B].copy_(torch.as_tensor(np.asarray(span, np.int32)), non_blocking=True)
        self.pol['adv'][:B].copy_(torch.as_tensor(np.asarray(advantage, np.float32)), non_blocking=True)
        if reference:
            self._stage_teacher(rows, B, length)
        return B

    def policy_stats(self, rows):
        """the last policy-gradient step's per-row statistics over each row's span as numpy [rows] arrays: logp (mean
        log-probability of the labels, float32), kl (mean exact KL to the reference, float32; 0 with beta = 0) and count
        (the span's positions, int64)"""
        if not rows or self.pol is None:
            return dict(logp=np.zeros(0, np.float32), kl=np.zeros(0, np.float32), count=np.zeros(0, np.int64))
        st = self.pol['stats'][:rows].cpu().numpy()
        return dict(logp=st[:, 0].copy(), kl=st[:, 1].copy(), count=st[:, 2].astype(np.int64))

    def ln_bwd_res(self, a, dy, x, scale, mean, rstd, dscale, shift, next_bias_grad=None):
        """LN(+shift) backward into the residual-gradient stream of the training set or its cut view `a`;
        `next_bias_grad` (+= column sums of the updated dres) is the bias gradient of the block that is differentiated
        next (its output bias sees exactly this dres)."""
        g = a.grad
        L.check(self.lib.progen_ln_shift_bwd(dy.data_ptr(), self.d, self.act_dt, x.data_ptr(), self.d, L.F32, scale.data_ptr(),
                                             mean.data_ptr(), rstd.data_ptr(), g['dres'].data_ptr(),
                                             g['dres_lp'].data_ptr() if self.mp else 0, self.d, L.ptr(dscale),
                                             L.ptr(next_bias_grad), a.T, self.d, a.n, int(shift), 1, L.stream()), 'ln_bwd')

    # ------------------------------------------------------------------------------------------ property head
    def load_property(self, rows, task, targets, length=None):
        """rows (B, n+1) and checked targets (regression: float32 [B, C]; classification: int32 [B]) -> self.tok /
        self.labels (cut to `length` as in load_batch) / self.ptarget or self.pclass; returns B"""
        B = self.load_batch(rows, length)
        t = torch.as_tensor(targets)
        if task == L.TASK_REGRESSION:
            self.ptarget[:t.numel()].copy_(t.reshape(-1), non_blocking=True)
        else:
            self.pclass.copy_(t, non_blocking=True)
        return B

    def property_stats(self, rows):
        """the last property step's predictions [rows, C] and per-row losses [rows] as numpy float32"""
        C = self.lora.head_outputs if self.lora is not None else 0
        if not rows or not C:
            return dict(prediction=np.zeros((0, C), np.float32), loss=np.zeros(0, np.float32))
        return dict(prediction=self.pred[:rows * C].view(rows, C).cpu().numpy(), loss=self.prow_loss[:rows].cpu().numpy())

    def predict(self, data, w, b, batch_size=64):
        """data: (N, n+1) integer rows; w [d, C], b [C] float32 head parameters -> (prediction [N, C], embedding [N, d])
        numpy float32.  Runs the inference forward cut to the rows' cut_length (the pooled embedding reads counted
        positions only, so it is bitwise the full-length one), without the logits GEMM, then progen_masked_mean_pool and
        progen_property_head without targets, batch_size rows at a time, one D2H copy per chunk."""
        rows = torch.as_tensor(np.asarray(data).astype(np.int32))
        N, d = rows.shape[0], self.d
        C = int(np.asarray(w).shape[1])
        out_p, out_e = np.zeros((N, C), np.float32), np.zeros((N, d), np.float32)
        if N == 0:
            return out_p, out_e
        hw = torch.tensor(np.asarray(w, np.float32), device=self.dev)
        hb = torch.tensor(np.asarray(b, np.float32), device=self.dev)
        res = torch.empty(min(batch_size, N) * (d + C), device=self.dev, dtype=torch.float32)
        lib, st = self.lib, L.stream()
        for r0, acts in self._chunks(rows, batch_size, cut_length(rows[:, 1:].numpy())):
            B = acts.B
            self._forward_device(acts, logits=False)
            emb, pred = res[:B * d], res[B * d:B * (d + C)]
            L.check(lib.progen_masked_mean_pool(acts.yf.data_ptr(), d, self.act_dt, acts.labels.data_ptr(), emb.data_ptr(),
                                                B, acts.n, d, st), 'masked_mean_pool')
            L.check(lib.progen_property_head(emb.data_ptr(), hw.data_ptr(), hb.data_ptr(), B, d, C, L.TASK_REGRESSION, 0, 0,
                                             1.0, pred.data_ptr(), 0, 0, 0, 0, 0, 0, st), 'property_head')
            host = res[:B * (d + C)].cpu().numpy()
            out_e[r0:r0 + B] = host[:B * d].reshape(B, d)
            out_p[r0:r0 + B] = host[B * d:].reshape(B, C)
        return out_p, out_e

    # ------------------------------------------------------------------------------------------ residue head
    def ensure_residue(self, C):
        """the residue head's buffers for the training set's B * n positions and a C-output head: targets y [B*n, C]
        (regression) and cls [B*n] (classification), pred and dpred [B*n, C], per-position loss [B*n], the count N and the
        wgrad workspace [B, (d + 1) C].  A cut step uses their (B, L) prefix, so nothing is allocated per length.  Kept
        until the batch size changes (ensure_batch) or a head with another C needs them; only that last re-allocation
        moves pointers a captured step holds, and it advances alloc_epoch as ensure_batch does."""
        if self.res_C == C:
            return self.res
        if self.res is not None:
            self.alloc_epoch += 1
        T, dev = self.T, self.dev
        F = lambda *shape: torch.empty(*shape, device=dev, dtype=torch.float32)
        self.res = dict(y=F(T * C), cls=torch.empty(T, device=dev, dtype=torch.int32), pred=F(T * C), dpred=F(T * C),
                        loss=F(T), count=torch.zeros(1, device=dev, dtype=torch.int32), ws=F(self.B * (self.d + 1) * C))
        self.res_C = C
        return self.res

    def load_residue(self, rows, task, targets, length=None):
        """rows (B, n+1) and checked per-position targets (property.check_residue_targets: regression float32 [B, n, C]
        with NaN where unlabelled, classification int32 [B, n] with -1) -> self.tok / self.labels and the residue
        targets, cut to their first `length` positions (default seq_len) in the layout of the (B, length) view; returns B.
        The engine's adapters (self.lora) carry the head."""
        B = self.load_batch(rows, length)
        n = self.n if length is None else length
        t = torch.as_tensor(np.ascontiguousarray(np.asarray(targets)[:, :n]))
        C = self.lora.head_outputs
        r = self.ensure_residue(C)
        if task == L.TASK_REGRESSION:
            r['y'][:B * n * C].view(B, n, C).copy_(t, non_blocking=True)
        else:
            r['cls'][:B * n].view(B, n).copy_(t, non_blocking=True)
        self.res_view = (B, n)
        return B

    def residue_stats(self, rows):
        """the last residue step's predictions [rows, seq_len, C] (regression values, or class logits) and per-position
        losses [rows, seq_len] (0 where unlabelled) as numpy float32; zero at positions beyond the step's row length"""
        C = self.res_C
        pred, loss = np.zeros((rows, self.n, C), np.float32), np.zeros((rows, self.n), np.float32)
        if rows and C:
            B, n = self.res_view
            pred[:, :n] = self.res['pred'][:B * n * C].view(B, n, C)[:rows].cpu().numpy()
            loss[:, :n] = self.res['loss'][:B * n].view(B, n)[:rows].cpu().numpy()
        return dict(prediction=pred, loss=loss)

    def predict_residues(self, data, w, b, length, batch_size=64):
        """data: (N, n+1) integer rows; w [d, C], b [C] float32 head parameters -> prediction [N, n, C] numpy float32 at
        every position (zero beyond `length`).  Runs the inference forward over the rows' first `length` positions
        (property.residue_length: it covers every position that holds a residue), without the logits GEMM, then
        progen_residue_head without targets, batch_size rows at a time, one D2H copy per chunk.  A position's prediction
        depends on its own row's ids only."""
        rows = torch.as_tensor(np.asarray(data).astype(np.int32))
        N, d = rows.shape[0], self.d
        C = int(np.asarray(w).shape[1])
        out = np.zeros((N, self.n, C), np.float32)
        if N == 0:
            return out
        hw = torch.tensor(np.asarray(w, np.float32), device=self.dev)
        hb = torch.tensor(np.asarray(b, np.float32), device=self.dev)
        res = torch.empty(min(batch_size, N) * length * C, device=self.dev, dtype=torch.float32)
        lib, st = self.lib, L.stream()
        for r0, acts in self._chunks(rows, batch_size, length):
            B = acts.B
            self._forward_device(acts, logits=False)
            L.check(lib.progen_residue_head(acts.yf.data_ptr(), d, self.act_dt, hw.data_ptr(), hb.data_ptr(), B, acts.n, d,
                                            C, L.TASK_REGRESSION, 0, 0, res.data_ptr(), 0, 0, 0, 0, 0, d, st),
                    'residue_head')
            out[r0:r0 + B, :length] = res[:B * length * C].cpu().numpy().reshape(B, length, C)
        return out

    def _backward_body(self, v):
        """the backward pass below the loss head (train_step) on the training set or its cut view `v` (B, n and T from
        it), from v.grad['dy'] = d loss / d (final LayerNorm output).
        With adapters (self.lora) the base is frozen: no base weight, bias, LayerNorm-scale, SGU or embedding
        gradient is computed, and every adapted projection's input gradient carries its adapter's tail (lora_bwd).
        In recompute mode every layer but the last is re-run (recompute_layer) before its backward."""
        lib, st = self.lib, L.stream()
        cfg, d, I, hid, T, n = self.cfg, self.d, self.I, self.hid, v.T, v.n
        shift = cfg['shift_tokens']
        lo = self.lora
        frozen = lo is not None
        G = (lambda module, name: None) if frozen else self.G
        tail = (lambda *a: self.lora_bwd(*a, acts=v)) if frozen else (lambda *a: {})
        mm = dict(acts=v)
        g_ = v.grad
        dres_lp, dy, dqkv, datt = g_['dres_lp'], g_['dy'], g_['dqkv'], g_['datt']
        hl = P + 'layer_norm'
        g_['dres'].zero_()
        nl = len(self.kinds)
        self.ln_bwd_res(v, dy, v.X[-1], self.Pf(hl, 'scale'), v.meanf, v.rstdf, G(hl, 'scale'), False,
                        next_bias_grad=G(P + f'ff{nl - 1}/~/linear_1', 'b'))
        for i in reversed(range(len(self.kinds))):
            if self.recompute and i < nl - 1:
                # the shared layer scratch still holds the last layer's forward; every other layer is re-run from its
                # checkpoint into it (its backward reads no buffer the re-run writes besides those)
                self.recompute_layer(i, v)
            kind, s = self.kinds[i], v.lay[i]
            a, f = P + f'attn{i}/~/', P + f'ff{i}/~/'
            x0, x1 = v.X[2 * i], v.X[2 * i + 1]
            # ---- FeedForward backward (d(proj_out bias) = colsum(dres) was produced by the previous LN backward)
            if kind == 'sgu':
                half = hid // 2
                g = f + 'sgu'
                dpj, dsg, dgp, dgn = g_['dpj'], g_['dsg'], g_['dgp'], g_['dgn']
                if not frozen:
                    self.wgrad_gemm(s['pj'], half, dres_lp, d, self.G(f + 'linear_1', 'w'), **mm)
                self.dgrad_gemm(dres_lp, d, self.W(f + 'linear_1', 'w'), half, dpj, **mm, **tail(s['pj'], half, f + 'linear_1', dres_lp, d))
                if not frozen:
                    self.colsum(dpj, half, self.G(g + '/~/linear', 'b'), **mm)
                    self.wgrad_gemm(s['sg'], half, dpj, half, self.G(g + '/~/linear', 'w'), **mm)
                self.dgrad_gemm(dpj, half, self.W(g + '/~/linear', 'w'), half, dsg, **mm)
                da = g_['dh_']                                           # gradient wrt gelu output a = [xs | gate], [T, hid]
                L.check(lib.progen_sgu_gate_bwd(dsg.data_ptr(), half, s['hact'].data_ptr(), hid, s['gp'].data_ptr(), half,
                                                self.Pf(g, 'spatial_biases').data_ptr(), da.data_ptr(), hid, dgp.data_ptr(),
                                                half, L.ptr(G(g, 'spatial_biases')), self.act_dt, T, half, n, st),
                        'sgu_gate_bwd')
                # the spatial matrices keep their leading dimension self.n; a cut step uses their top-left n x n block
                if not frozen:
                    # d spatial_weights = tril(sum_b dGp_b @ gn_b^T)
                    self._mm(M=n, N=n, K=half, A=dgp, lda=half, B=s['gn'], ldb=half, out=self.G(g, 'spatial_weights'),
                             ldo=self.n, epi=L.EPI_ACCUM, out_dtype=L.F32, batch=v.B, a_batch_rows=n, b_batch_rows=n,
                             batch_reduce=True, atomic=True, tril=True, tril_rows=n)
                # d gn_b = tril(W)^T @ dGp_b
                self._mm(M=n, N=half, K=n, A=self.wm[i], lda=self.n, a_mn=True, B=dgp, ldb=half, b_mn=True, out=dgn,
                         ldo=half, out_dtype=self.act_dt, batch=v.B, b_batch_rows=n, d_batch_rows=n, causal=2)
                gate = s['hact'][:, half:]
                L.check(lib.progen_ln_shift_bwd(dgn.data_ptr(), half, self.act_dt, gate.data_ptr(), hid, self.act_dt,
                                                self.Pf(g + '/~/layer_norm', 'scale').data_ptr(), s['mean3'].data_ptr(),
                                                s['rstd3'].data_ptr(), 0, da[:, half:].data_ptr(), hid,
                                                L.ptr(G(g + '/~/layer_norm', 'scale')), 0, T, half, n, 0, 0, st), 'ln_bwd_sgu')
                L.check(lib.progen_gelu_bwd(da.data_ptr(), s['u'].data_ptr(), self.act_dt, T * hid, st), 'gelu_bwd')
                du, n_in = da, hid
                if not frozen:
                    self.colsum(du, n_in, self.G(f + 'linear', 'b'), **mm)
            elif kind == 'glu':
                # the epilogue also adds the column sums of du into the proj_in bias gradient (interleaved like du)
                if not frozen:
                    self.wgrad_gemm(s['hact'], hid, dres_lp, d, self.G(f + 'linear_1', 'w'), **mm)
                self.dgrad_gemm(dres_lp, d, self.W(f + 'linear_1', 'w'), hid, g_['du'], epi=L.EPI_GLU_BWD, ldo=2 * hid,
                                aux=s['u'], ldaux=2 * hid, colsum=G(f + 'linear', 'b'), **mm,
                                **tail(s['hact'], hid, f + 'linear_1', dres_lp, d))
                du, n_in = g_['du'], 2 * hid
            else:
                if not frozen:
                    self.wgrad_gemm(s['hact'], hid, dres_lp, d, self.G(f + 'linear_1', 'w'), **mm)
                self.dgrad_gemm(dres_lp, d, self.W(f + 'linear_1', 'w'), hid, g_['dh_'], epi=L.EPI_GELU_BWD, aux=s['u'], ldaux=hid,
                                colsum=G(f + 'linear', 'b'), **mm, **tail(s['hact'], hid, f + 'linear_1', dres_lp, d))
                du, n_in = g_['dh_'], hid
            if not frozen:
                self.wgrad_gemm(s['y2'], d, du, n_in, self.G(f + 'linear', 'w'), **mm)
            self.dgrad_gemm(du, n_in, self.W(f + 'linear', 'w'), d, dy, **mm, **tail(s['y2'], d, f + 'linear', du, n_in))
            self.ln_bwd_res(v, dy, x1, self.Pf(f + 'layer_norm', 'scale'), s['mean2'], s['rstd2'], G(f + 'layer_norm', 'scale'), shift,
                            next_bias_grad=G(a + 'linear_1', 'b'))
            # ---- LocalAttention backward
            if not frozen:
                self.wgrad_gemm(s['att'], I, dres_lp, d, self.G(a + 'linear_1', 'w'), **mm)
            self.dgrad_gemm(dres_lp, d, self.W(a + 'linear_1', 'w'), I, datt, **mm, **tail(s['att'], I, a + 'linear_1', dres_lp, d))
            self.attn_bwd(s['qkv'], s['att'], datt, s['lse'], dqkv, **mm)
            if not self.attn_tc:
                L.check(lib.progen_rotary_bwd(dqkv.data_ptr(), 3 * I, self.act_dt, self.rot_sin.data_ptr(),
                                              self.rot_cos.data_ptr(), T, 3 * I, n, self.dh, st), 'rotary_bwd')
            if not frozen:
                self.wgrad_gemm(s['y1'], d, dqkv, 3 * I, self.G(a + 'linear', 'w'), **mm)
            self.dgrad_gemm(dqkv, 3 * I, self.W(a + 'linear', 'w'), d, dy, **mm, **tail(s['y1'], d, a + 'linear', dqkv, 3 * I))
            self.ln_bwd_res(v, dy, x0, self.Pf(a + 'layer_norm', 'scale'), s['mean1'], s['rstd1'], G(a + 'layer_norm', 'scale'), shift,
                            next_bias_grad=G(P + f'ff{i - 1}/~/linear_1', 'b') if i > 0 else None)
        if frozen:
            lo.scale_b_grads()
            return
        L.check(lib.progen_embed_bwd(v.tok.data_ptr(), g_['dres'].data_ptr(), self.G(P + 'embed', 'embeddings').data_ptr(),
                                     T, d, self.V, st), 'embed_bwd')
