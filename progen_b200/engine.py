"""Host-side orchestration of the ProGen forward / backward pass over the C-ABI kernels.

Mirrors `ProGenBase.__call__` (reference progen.py:224-233) and its gradient (`jax.value_and_grad`, utils.py:72),
batched over sequences (the reference's `vmap`, utils.py:67).  PyTorch provides device buffers and streams only.

Data layout in HBM (tokens are rows, T = B * seq_len):
  * residual stream: fp32 [T, d], one buffer per LayerNorm input (the residual epilogue of each GEMM writes the next
    one, so nothing is copied and every LN backward still has its input); the inference set (`Engine.score`) keeps one
    buffer and updates it in place;
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


def layer_kinds(depth, global_mlp_depth, ff_glu):
    """reference progen.py:210-212"""
    out = []
    for i in range(depth):
        use_gmlp = (depth - i) <= global_mlp_depth
        out.append('sgu' if use_gmlp else ('glu' if ff_glu else 'gelu'))
    return out


class ParamSpec:
    __slots__ = ('module', 'name', 'shape', 'decay', 'interleave', 'offset', 'size')

    def __init__(self, module, name, shape, interleave=False):
        self.module, self.name, self.shape = module, name, tuple(shape)
        self.decay = len(shape) > 1                    # optax mask: tree_map(lambda x: x.ndim > 1) — train.py:113
        self.interleave = interleave
        self.size = int(np.prod(shape))
        self.offset = -1


def build_param_specs(cfg):
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
    off = 0
    for s in [s for s in specs if s.decay] + [s for s in specs if not s.decay]:
        s.offset = off
        off += (s.size + ALIGN - 1) // ALIGN * ALIGN
    n_decay = sum((s.size + ALIGN - 1) // ALIGN * ALIGN for s in specs if s.decay)
    return specs, off, n_decay


def _interleave(a):
    """[..., 2H] with columns (value | gate) -> columns (v0, g0, v1, g1, ...)"""
    H = a.shape[-1] // 2
    return np.stack((a[..., :H], a[..., H:]), axis=-1).reshape(a.shape)


def _deinterleave(a):
    return np.concatenate((a[..., 0::2], a[..., 1::2]), axis=-1)


class Acts:
    """One activation set: the buffers one forward pass runs on (B sequences, T = B * seq_len token rows).
    `X` lists the residual stream at every LayerNorm input and `lay` one scratch dict per layer.  The training set keeps
    all of them (the backward pass reads them); the inference set (`inplace`) repeats one residual buffer, updated in
    place, and one layer's scratch, and stores no GLU / GELU pre-activation (`u` is None)."""

    def __init__(self, B, T, tok, labels, X, lay, meanf, rstdf, yf, logits, inplace=False, rows=None, res=None):
        self.B, self.T, self.tok, self.labels, self.X, self.lay = B, T, tok, labels, X, lay
        self.meanf, self.rstdf, self.yf, self.logits = meanf, rstdf, yf, logits
        self.inplace = inplace
        self.rows = rows        # inference: [B, n+1] int32 staging of the input rows (one H2D copy per chunk)
        self.res = res          # inference: flat fp32 per-chunk results (see Engine.score)

    def view(self, B, n):
        """the first B sequences of this set (same memory): a ragged last chunk runs on the cached buffers"""
        T = B * n
        cut = lambda t: None if t is None else t[:T]
        return Acts(B, T, cut(self.tok), cut(self.labels), [cut(x) for x in self.X],
                    [{k: cut(v) for k, v in s.items()} for s in self.lay], cut(self.meanf), cut(self.rstdf), cut(self.yf),
                    cut(self.logits), self.inplace, None if self.rows is None else self.rows[:B], self.res)


class Engine:
    def __init__(self, cfg, mixed_precision=False, device=None):
        L.require_device()
        self.cfg = cfg
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
        self.specs, self.n_params_padded, self.n_decay = build_param_specs(cfg)
        self.by_key = {(s.module, s.name): s for s in self.specs}
        self.num_params = sum(s.size for s in self.specs)
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
        self.acts = None          # training activation set (ensure_batch)
        self.infer = None         # inference activation set (inference_acts), cached by row count
        self.loss = torch.zeros(1, device=self.dev)       # exists before the first batch: a rank without rows still reports 0
        self.loaded_token = None
        self.on_layer_grads = None        # optional callback(layer_index) fired when a layer's weight gradients are final
        self.lora = None                  # lora.Adapters: the training set runs the adapted model with a frozen base
        self.lib = L.load()
        self.num_sms = torch.cuda.get_device_properties(self.dev).multi_processor_count

    def layer_grad_range(self, i):
        """[start, stop) of layer i's ndim>1 parameters inside the flat buffers (contiguous by construction)."""
        pre = (P + f'attn{i}/~/', P + f'ff{i}/~/')
        segs = [s for s in self.specs if s.decay and s.module.startswith(pre)]
        return min(s.offset for s in segs), max(s.offset + (s.size + ALIGN - 1) // ALIGN * ALIGN for s in segs)

    # ------------------------------------------------------------------------------------------ parameters
    def seg(self, buf, module, name):
        s = self.by_key[(module, name)]
        return buf[s.offset:s.offset + s.size]

    def load_params(self, params):
        """haiku-shaped nested dict {module: {name: array}} (numpy or torch) -> flat engine layout on the device."""
        host = np.zeros(self.n_params_padded, np.float32)
        for s in self.specs:
            a = params[s.module][s.name]
            a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
            a = a.astype(np.float32)
            if a.shape != s.shape:
                raise L.ProgenError(f'{s.module}/{s.name}: expected shape {s.shape}, got {a.shape}')
            if s.interleave:
                a = _interleave(a)
            host[s.offset:s.offset + s.size] = a.ravel()
        self.params.copy_(torch.from_numpy(host))
        self.refresh_compute_copies()

    def export_tree(self, buf):
        host = buf.detach().float().cpu().numpy()
        out = {}
        for s in self.specs:
            a = host[s.offset:s.offset + s.size].reshape(s.shape).copy()
            if s.interleave:
                a = _deinterleave(a)
            out.setdefault(s.module, {})[s.name] = a
        return out

    def export_params(self):
        return self.export_tree(self.params)

    def export_grads(self):
        return self.export_tree(self.base_grads())

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
            src = self.seg(self.params, P + f'ff{i}/~/sgu', 'spatial_weights')
            L.check(self.lib.progen_tril_cast(src.data_ptr(), wm.data_ptr(), self.act_dt, self.n, st), 'tril_cast')

    def W(self, module, name):
        """GEMM operand view of a parameter: bf16 mirror under mixed precision, fp32 master otherwise."""
        return self.seg(self.params_lp if self.mp else self.params, module, name)

    def Pf(self, module, name):
        return self.seg(self.params, module, name)

    def G(self, module, name):
        return self.seg(self.base_grads(), module, name)

    # ------------------------------------------------------------------------------------------ workspaces
    def ensure_batch(self, B):
        if B == self.B:
            return
        self.B = B
        self.alloc_epoch = getattr(self, 'alloc_epoch', 0) + 1      # activation buffers are re-allocated below: captured
                                                                    # CUDA graphs (Trainer.capture_graph) become invalid
        T = B * self.n
        self.T = T
        d, I, hid = self.d, self.I, self.hid
        dev, act = self.dev, self.act
        A = lambda *shape: torch.empty(*shape, device=dev, dtype=act)
        F = lambda *shape: torch.empty(*shape, device=dev, dtype=torch.float32)
        nl = len(self.kinds)
        self.tok = torch.empty(T, device=dev, dtype=torch.int32)
        self.labels = torch.empty(T, device=dev, dtype=torch.int32)
        self.X = [F(T, d) for _ in range(2 * nl + 1)]           # residual stream at every LN input
        self.lay = []
        for kind in self.kinds:
            s = dict(mean1=F(T), rstd1=F(T), y1=A(T, d), qkv=A(T, 3 * I), att=A(T, I), lse=F(T, self.h),
                     mean2=F(T), rstd2=F(T), y2=A(T, d))
            if kind == 'glu':
                s.update(u=A(T, 2 * hid), hact=A(T, hid))
            else:
                s.update(u=A(T, hid), hact=A(T, hid))
            if kind == 'sgu':
                half = hid // 2
                s.update(mean3=F(T), rstd3=F(T), gn=A(T, half), gp=A(T, half), sg=A(T, half), pj=A(T, half))
            self.lay.append(s)
        self.meanf, self.rstdf, self.yf = F(T), F(T), A(T, d)
        self.logits = F(T, self.V)
        self.dlogits = A(T, self.V)
        self.ce_w = F(T)
        # preference (DPO) head (preference_step_device): B = 2 * pairs rows; allocated here so a captured step's pointers
        # stay valid
        self.logp, self.seq_ll, self.seq_count, self.ref = F(T), F(B), F(B), F(B)
        self.stats, self.ce_scratch = F(max(1, B // 2), 4), F(1)
        # backward temporaries (shared by all layers)
        self.dres = F(T, d)
        self.dres_lp = A(T, d) if self.mp else self.dres
        self.dy = A(T, d)
        self.dqkv = A(T, 3 * I)
        self.datt = A(T, I)
        self.delta = F(T, self.h)
        self.du = A(T, 2 * hid)
        self.dh_ = A(T, hid)
        half = hid // 2
        if 'sgu' in self.kinds:
            self.dpj, self.dsg, self.dgp, self.dgn = A(T, half), A(T, half), A(T, half), A(T, half)
        self.acts = Acts(B, T, self.tok, self.labels, self.X, self.lay, self.meanf, self.rstdf, self.yf, self.logits)

    def inference_acts(self, B):
        """Activation set of a forward pass that keeps no training state, for up to B sequences: one fp32 residual buffer
        [T, d] updated in place, one layer's scratch shared by every layer (no pre-activation store), the final LN output,
        the fp32 logits and the scoring outputs.  Allocated on first use and kept for later calls of the same or smaller
        row count, apart from the training set: `ensure_batch`, `alloc_epoch` and captured training graphs are untouched."""
        if self.infer is not None and self.infer.B >= B:
            return self.infer if self.infer.B == B else self.infer.view(B, self.n)
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
        self.infer = Acts(B, T, torch.empty(T, device=dev, dtype=torch.int32), torch.empty(T, device=dev, dtype=torch.int32),
                          [x] * (2 * nl + 1), [s] * nl, F(T), F(T), A(T, d), F(T, V), inplace=True,
                          rows=torch.empty(B, n + 1, device=dev, dtype=torch.int32), res=F(B * (2 + n + d)))
        return self.infer

    # ------------------------------------------------------------------------------------------ GEMM helpers
    def _mm(self, **kw):
        L.gemm(backend=self.backend, in_dtype=self.act_dt, **kw)

    def lora_fwd(self, x, K, module, N):
        """adapters: u = x A of projection `module` (input x [T, K], N outputs) -> the tail (u, s B) of its GEMM"""
        lo = self.lora
        if lo is None:
            return {}
        u = lo.u[module]
        self.fwd_gemm(x, K, lo.seg(lo.lp, module, 'lora_a'), lo.r, u)
        return dict(A2=u, lda2=lo.r, B2=lo.seg(lo.lp, module, 'lora_b'), ldb2=N, K2=lo.r)

    def lora_bwd(self, x, K, module, dy, N):
        """adapters: from the projection's output gradient dy [T, N], g' = s g = dy (s B)^T, dB += u^T dy (scaled by s
        after the backward pass), dA += x^T g' -> the tail (g', A^T) of its input-gradient GEMM"""
        lo = self.lora
        if lo is None:
            return {}
        g, A = lo.g, lo.seg(lo.lp, module, 'lora_a')
        self.dgrad_gemm(dy, N, lo.seg(lo.lp, module, 'lora_b'), lo.r, g)
        self.wgrad_gemm(lo.u[module], lo.r, dy, N, lo.seg(lo.grads, module, 'lora_b'))
        self.wgrad_gemm(x, K, g, lo.r, lo.seg(lo.grads, module, 'lora_a'))
        return dict(A2=g, lda2=lo.r, B2=A, ldb2=lo.r, K2=lo.r)

    def fwd_gemm(self, x, K, w, N, out, epi=L.EPI_STORE, out_dtype=None, acts=None, **kw):
        """out[T,N] = x[T,K] @ w[K,N]  (w stored (in, out) like hk.Linear: MN-major B operand); T from `acts` (default:
        the training set)"""
        self._mm(M=(acts or self.acts).T, N=N, K=K, A=x, lda=K, B=w, ldb=N, b_mn=True, out=out, ldo=kw.pop('ldo', N), epi=epi,
                 out_dtype=self.act_dt if out_dtype is None else out_dtype, **kw)

    def dgrad_gemm(self, dy, N_out, w, K_in, out, epi=L.EPI_STORE, **kw):
        """out[T,K_in] = dy[T,N_out] @ w[K_in,N_out]^T  (w rows are the output features: K-major B operand)"""
        self._mm(M=self.T, N=K_in, K=N_out, A=dy, lda=N_out, B=w, ldb=N_out, out=out, ldo=kw.pop('ldo', K_in), epi=epi,
                 out_dtype=self.act_dt, **kw)

    def wgrad_gemm(self, x, K_in, dy, N_out, dw):
        """dw[K_in,N_out] += x[T,K_in]^T @ dy[T,N_out]  (both operands MN-major, the token dimension is K)"""
        split = self.wgrad_split(K_in, N_out) if self.backend == L.BACKEND_TC else 1
        self._mm(M=K_in, N=N_out, K=self.T, A=x, lda=K_in, a_mn=True, B=dy, ldb=N_out, b_mn=True, out=dw, ldo=N_out,
                 epi=L.EPI_ACCUM, out_dtype=L.F32, split_k=split, atomic=split > 1)

    def wgrad_split(self, K_in, N_out):
        """K split of a weight-gradient GEMM (one CTA per 128 x 128 output tile and K slice): the split in 1..8 whose CTAs
        fill the largest fraction of their waves over the SMs, the smallest such split on ties"""
        tiles = ((K_in + 127) // 128) * ((N_out + 127) // 128)
        fill = lambda s: tiles * s / (-(-tiles * s // self.num_sms) * self.num_sms)
        return max(range(1, min(8, max(1, self.T // 64)) + 1), key=lambda s: (round(fill(s), 6), -s))

    def colsum(self, t, N, out, ld=None):
        L.check(self.lib.progen_colsum(t.data_ptr(), N if ld is None else ld, L.dt(t), out.data_ptr(), self.T, N, L.stream()), 'colsum')

    def ln_fwd(self, x, ldx, scale, y, ldy, mean, rstd, dcols, shift, acts=None, seq_len=None):
        L.check(self.lib.progen_ln_shift_fwd(x.data_ptr(), ldx, L.dt(x), scale.data_ptr(), y.data_ptr(), ldy, L.dt(y),
                                             mean.data_ptr(), rstd.data_ptr(), (acts or self.acts).T, dcols,
                                             self.n if seq_len is None else seq_len, int(shift), L.stream()), 'ln_fwd')

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

    def _forward_device(self, acts=None, sink=None, length=None):
        """forward pass on activation set `acts` (default: the training set, which keeps what the backward pass reads);
        with a `sink` (Engine.prefill) the layers' state goes to it and the logits head is skipped.
        `length` (default seq_len): the positions per row, acts.T = acts.B * length.  Every mixing op is causal, so a
        forward cut to the first `length` positions computes exactly those positions of the full one (DESIGN.md §3.6)."""
        acts = self.acts if acts is None else acts
        lib, st = self.lib, L.stream()
        cfg, d, I, hid, T = self.cfg, self.d, self.I, self.hid, acts.T
        n = self.n if length is None else length
        if T != acts.B * n:
            raise L.ProgenError(f'forward: {T} token rows are not {acts.B} rows of length {n}')
        shift = cfg['shift_tokens']
        lo = self.lora if acts is self.acts else None       # adapters run on the training set only
        if lo is not None:
            lo.activations(T)
        tail = self.lora_fwd if lo is not None else (lambda *a: {})
        L.check(lib.progen_embed_fwd(acts.tok.data_ptr(), self.Pf(P + 'embed', 'embeddings').data_ptr(), acts.X[0].data_ptr(),
                                     T, d, self.V, st), 'embed_fwd')
        for i, kind in enumerate(self.kinds):
            s = acts.lay[i]
            a, f = P + f'attn{i}/~/', P + f'ff{i}/~/'
            # in place (inference): x0 = x1 = x2 is one buffer, and the residual epilogue without aux reads its output
            x0, x1, x2 = acts.X[2 * i], acts.X[2 * i + 1], acts.X[2 * i + 2]
            # ---- LocalAttention (progen.py:73-103)
            self.ln_fwd(x0, d, self.Pf(a + 'layer_norm', 'scale'), s['y1'], d, s['mean1'], s['rstd1'], d, shift, acts=acts, seq_len=n)
            self.fwd_gemm(s['y1'], d, self.W(a + 'linear', 'w'), 3 * I, s['qkv'], epi=L.EPI_ROTARY, rot_sin=self.rot_sin,
                          rot_cos=self.rot_cos, seq_len=n, dim_head=self.dh, acts=acts, **tail(s['y1'], d, a + 'linear', 3 * I))
            if sink is not None:
                sink(i, 'qkv', s['qkv'])
                sink(i, 'y1', s['y1'])
            self.attn_fwd(s['qkv'], s['att'], s['lse'], acts=acts, seq_len=n)
            self.fwd_gemm(s['att'], I, self.W(a + 'linear_1', 'w'), d, x1, epi=L.EPI_RESIDUAL, bias=self.Pf(a + 'linear_1', 'b'),
                          aux=None if acts.inplace else x0, ldaux=d, acts=acts, **tail(s['att'], I, a + 'linear_1', d))
            # ---- FeedForward (progen.py:131-149); s['u'] is None in the inference set: no pre-activation store
            self.ln_fwd(x1, d, self.Pf(f + 'layer_norm', 'scale'), s['y2'], d, s['mean2'], s['rstd2'], d, shift, acts=acts, seq_len=n)
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
                            acts=acts, seq_len=n)
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
            self.fwd_gemm(last, last_k, self.W(f + 'linear_1', 'w'), d, x2, epi=L.EPI_RESIDUAL, bias=self.Pf(f + 'linear_1', 'b'),
                          aux=None if acts.inplace else x1, ldaux=d, acts=acts, **tail(last, last_k, f + 'linear_1', d))
        if sink is not None:
            return
        # ---- to_logits (progen.py:219-222)
        xl = acts.X[-1]
        self.ln_fwd(xl, d, self.Pf(P + 'layer_norm', 'scale'), acts.yf, d, acts.meanf, acts.rstdf, d, False, acts=acts, seq_len=n)
        self.fwd_gemm(acts.yf, d, self.W(P + 'linear', 'w'), self.V, acts.logits, bias=self.Pf(P + 'linear', 'b'), out_dtype=L.F32,
                      acts=acts)

    def attn_fwd(self, qkv, out, lse, acts=None, seq_len=None):
        B = (acts or self.acts).B
        n = self.n if seq_len is None else seq_len
        if self.attn_tc:
            L.check(self.lib.progen_local_attn_fwd_tc(qkv.data_ptr(), out.data_ptr(), lse.data_ptr(), B, n, self.w, self.h,
                                                      self.dh, L.stream()), 'local_attn_fwd')
            return
        L.check(self.lib.progen_local_attn_fwd_simt(qkv.data_ptr(), out.data_ptr(), lse.data_ptr(), self.act_dt, B, n,
                                                    self.w, self.h, self.dh, L.stream()), 'local_attn_fwd')

    def attn_bwd(self, qkv, out, dout, lse, dqkv):
        if self.attn_tc:
            L.check(self.lib.progen_local_attn_bwd_tc(qkv.data_ptr(), out.data_ptr(), dout.data_ptr(), lse.data_ptr(), dqkv.data_ptr(),
                                                      self.delta.data_ptr(), self.rot_sin.data_ptr(), self.rot_cos.data_ptr(),
                                                      self.B, self.n, self.w, self.h, self.dh, L.stream()), 'local_attn_bwd')
            return     # rotary backward is fused into the kernel's epilogue
        L.check(self.lib.progen_local_attn_bwd_simt(qkv.data_ptr(), out.data_ptr(), dout.data_ptr(), lse.data_ptr(), dqkv.data_ptr(),
                                                    self.delta.data_ptr(), self.act_dt, self.B, self.n, self.w, self.h, self.dh,
                                                    L.stream()), 'local_attn_bwd')

    # ------------------------------------------------------------------------------------------ scoring (inference)
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
        cut = n if length is None else length
        if length is not None:
            if not isinstance(length, (int, np.integer)) or not (length == n or (0 < length < n and length % CUT_ALIGN == 0)):
                raise L.ProgenError(f'score: length must be seq_len ({n}) or a multiple of {CUT_ALIGN} below it, got {length!r}')
            if N and int(counted_length(rows[:, 1:].numpy()).max()) > length:
                raise L.ProgenError(f'score: length {length} cuts off counted positions (cut_length of these rows: '
                                    f'{cut_length(rows[:, 1:].numpy())})')
            cut = int(length)
        out = dict(log_likelihood=np.zeros(N, np.float32), num_tokens=np.zeros(N, np.int64))
        if tokens:
            out['token_logp'] = np.zeros((N, n), np.float32)
        if embeddings:
            out['embedding'] = np.zeros((N, d), np.float32)
        if N == 0:
            return out
        full = self.inference_acts(min(batch_size, N))
        lib, st = self.lib, L.stream()
        for r0 in range(0, N, batch_size):
            chunk = rows[r0:r0 + batch_size]
            B = chunk.shape[0]
            acts = full if B == full.B and cut == n else full.view(B, cut)
            T = acts.T
            # the rows staged as one contiguous (B, cut + 1) block: one H2D copy of what the cut forward reads
            staged = acts.rows if cut == n else full.rows.view(-1)[:B * (cut + 1)].view(B, cut + 1)
            staged.copy_(chunk if cut == n else chunk[:, :cut + 1])
            acts.tok.view(B, cut).copy_(staged[:, :-1])
            acts.labels.view(B, cut).copy_(staged[:, 1:])
            self._forward_device(acts, length=length)
            # results, packed for one D2H copy: seq_ll [B] | seq_count [B] | logp [T] | embedding [B, d]
            ll, cnt, lp, emb = full.res[:B], full.res[B:2 * B], full.res[2 * B:2 * B + T], full.res[2 * B + T:2 * B + T + B * d]
            L.check(lib.progen_token_logprob(acts.logits.data_ptr(), L.F32, acts.labels.data_ptr(), lp.data_ptr(), ll.data_ptr(),
                                             cnt.data_ptr(), B, cut, self.V, st), 'token_logprob')
            if embeddings:
                L.check(lib.progen_masked_mean_pool(acts.yf.data_ptr(), d, self.act_dt, acts.labels.data_ptr(), emb.data_ptr(),
                                                    B, cut, d, st), 'masked_mean_pool')
            used = 2 * B + (T + B * d if embeddings else T if tokens else 0)
            host = full.res[:used].cpu().numpy()
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
        `global_batch` (DDP): scale by 1/global_batch so that a SUM all-reduce yields the global-mean gradient."""
        B = self.load_batch(data)
        self.step_device(global_batch or B, zero_grads)
        return self.loss

    def load_batch(self, data):
        """host (or device) rows (B, n+1) -> self.tok / self.labels; returns B"""
        data = torch.as_tensor(np.asarray(data).astype(np.int32) if not isinstance(data, torch.Tensor) else data)
        B = data.shape[0]
        self.ensure_batch(B)
        dd = data.to(device=self.dev, dtype=torch.int32, non_blocking=True)
        self.tok.copy_(dd[:, :-1].reshape(-1))
        self.labels.copy_(dd[:, 1:].reshape(-1))
        return B

    def step_device(self, global_batch, zero_grads=True):
        """forward + loss + backward on tokens/labels already resident in self.tok / self.labels"""
        self._forward_device()
        lib, st = self.lib, L.stream()
        self.loss.zero_()
        self._check_zero_grads(zero_grads)
        if zero_grads:
            self.train_grads().zero_()
        L.check(lib.progen_ce_fwd_bwd(self.logits.data_ptr(), L.F32, self.labels.data_ptr(), self.ce_w.data_ptr(),
                                      self.loss.data_ptr(), self.dlogits.data_ptr(), self.act_dt, self.B, self.n, self.V,
                                      1.0 / global_batch, st), 'ce_fwd_bwd')
        self._backward_device()

    def _check_zero_grads(self, zero_grads):
        if not zero_grads and self.lora is not None:
            # the backward pass ends by scaling the whole B gradient by s (Adapters.scale_b_grads): an accumulated one
            # would be scaled twice
            raise L.ProgenError('adapters: gradients cannot accumulate across steps (zero_grads=False)')

    def train_grads(self):
        """the flat gradient buffer a training step writes: the adapters' with adapters (the base is frozen)"""
        return self.base_grads() if self.lora is None else self.lora.grads

    def load_preference(self, rows, ref):
        """rows (2P, n+1): the chosen rows, then their rejected rows; ref [2P] float32: the reference log-likelihoods in
        the same order -> self.tok / self.labels / self.ref; returns P"""
        B = self.load_batch(rows)
        self.ref.copy_(torch.as_tensor(np.asarray(ref, np.float32)), non_blocking=True)
        return B // 2

    def preference_step_device(self, pairs, beta, global_pairs, zero_grads=True):
        """forward + preference (DPO) head + backward on 2 * pairs rows already resident in self.tok / self.labels (rows
        0..P-1 chosen, row i + P the rejected row of pair i) and their reference log-likelihoods in self.ref.  The loss is
        the sum of the pair losses softplus(-z) over 1/global_pairs (DESIGN.md §3.7); self.stats [P, 4] holds each pair's
        (s(chosen), s(rejected), z, loss)."""
        if 2 * pairs != self.B:
            raise L.ProgenError(f'preference step: {pairs} pairs need {2 * pairs} resident rows, have {self.B}')
        self._check_zero_grads(zero_grads)
        self._forward_device()
        if zero_grads:
            self.train_grads().zero_()
        L.check(self.lib.progen_preference_head(self.logits.data_ptr(), L.F32, self.labels.data_ptr(), self.ref.data_ptr(),
                                                self.logp.data_ptr(), self.seq_ll.data_ptr(), self.seq_count.data_ptr(),
                                                self.ce_w.data_ptr(), self.stats.data_ptr(), self.loss.data_ptr(),
                                                self.ce_scratch.data_ptr(), self.dlogits.data_ptr(), self.act_dt, pairs, self.n,
                                                self.V, beta, 1.0 / global_pairs, L.stream()), 'preference_head')
        self._backward_device()

    def preference_stats(self, pairs):
        """the last preference step's per-pair statistics as numpy float32 [pairs]"""
        st = self.stats[:pairs].cpu().numpy() if pairs else np.zeros((0, 4), np.float32)
        return dict(policy_chosen=st[:, 0].copy(), policy_rejected=st[:, 1].copy(), margin=st[:, 2].copy(),
                    loss=st[:, 3].copy())

    def ln_bwd_res(self, dy, x, scale, mean, rstd, dscale, shift, next_bias_grad=None):
        """LN(+shift) backward into the residual-gradient stream; `next_bias_grad` (+= column sums of the updated dres) is
        the bias gradient of the block that is differentiated next (its output bias sees exactly this dres)."""
        L.check(self.lib.progen_ln_shift_bwd(dy.data_ptr(), self.d, self.act_dt, x.data_ptr(), self.d, L.F32, scale.data_ptr(),
                                             mean.data_ptr(), rstd.data_ptr(), self.dres.data_ptr(),
                                             self.dres_lp.data_ptr() if self.mp else 0, self.d, L.ptr(dscale),
                                             L.ptr(next_bias_grad), self.T, self.d, self.n, int(shift), 1, L.stream()), 'ln_bwd')

    def _backward_device(self):
        """With adapters (self.lora) the base is frozen: no base weight, bias, LayerNorm-scale, SGU or embedding
        gradient is computed, and every adapted projection's input gradient carries its adapter's tail (lora_bwd)."""
        lib, st = self.lib, L.stream()
        cfg, d, I, hid, T, n = self.cfg, self.d, self.I, self.hid, self.T, self.n
        shift = cfg['shift_tokens']
        lo = self.lora
        frozen = lo is not None
        G = (lambda module, name: None) if frozen else self.G
        tail = self.lora_bwd if frozen else (lambda *a: {})
        # ---- head
        hw, hl = P + 'linear', P + 'layer_norm'
        if not frozen:
            self.colsum(self.dlogits, self.V, self.G(hw, 'b'))
            self.wgrad_gemm(self.yf, d, self.dlogits, self.V, self.G(hw, 'w'))
        self.dgrad_gemm(self.dlogits, self.V, self.W(hw, 'w'), d, self.dy)
        self.dres.zero_()
        nl = len(self.kinds)
        self.ln_bwd_res(self.dy, self.X[-1], self.Pf(hl, 'scale'), self.meanf, self.rstdf, G(hl, 'scale'), False,
                        next_bias_grad=G(P + f'ff{nl - 1}/~/linear_1', 'b'))
        for i in reversed(range(len(self.kinds))):
            kind, s = self.kinds[i], self.lay[i]
            a, f = P + f'attn{i}/~/', P + f'ff{i}/~/'
            x0, x1 = self.X[2 * i], self.X[2 * i + 1]
            dres_lp = self.dres_lp
            # ---- FeedForward backward (d(proj_out bias) = colsum(dres) was produced by the previous LN backward)
            if kind == 'sgu':
                half = hid // 2
                g = f + 'sgu'
                if not frozen:
                    self.wgrad_gemm(s['pj'], half, dres_lp, d, self.G(f + 'linear_1', 'w'))
                self.dgrad_gemm(dres_lp, d, self.W(f + 'linear_1', 'w'), half, self.dpj, **tail(s['pj'], half, f + 'linear_1', dres_lp, d))
                if not frozen:
                    self.colsum(self.dpj, half, self.G(g + '/~/linear', 'b'))
                    self.wgrad_gemm(s['sg'], half, self.dpj, half, self.G(g + '/~/linear', 'w'))
                self.dgrad_gemm(self.dpj, half, self.W(g + '/~/linear', 'w'), half, self.dsg)
                da = self.dh_                                            # gradient wrt gelu output a = [xs | gate], [T, hid]
                L.check(lib.progen_sgu_gate_bwd(self.dsg.data_ptr(), half, s['hact'].data_ptr(), hid, s['gp'].data_ptr(), half,
                                                self.Pf(g, 'spatial_biases').data_ptr(), da.data_ptr(), hid, self.dgp.data_ptr(),
                                                half, L.ptr(G(g, 'spatial_biases')), self.act_dt, T, half, n, st),
                        'sgu_gate_bwd')
                if not frozen:
                    # d spatial_weights = tril(sum_b dGp_b @ gn_b^T)
                    self._mm(M=n, N=n, K=half, A=self.dgp, lda=half, B=s['gn'], ldb=half, out=self.G(g, 'spatial_weights'), ldo=n,
                             epi=L.EPI_ACCUM, out_dtype=L.F32, batch=self.B, a_batch_rows=n, b_batch_rows=n, batch_reduce=True,
                             atomic=True, tril=True, tril_rows=n)
                # d gn_b = tril(W)^T @ dGp_b
                self._mm(M=n, N=half, K=n, A=self.wm[i], lda=n, a_mn=True, B=self.dgp, ldb=half, b_mn=True, out=self.dgn,
                         ldo=half, out_dtype=self.act_dt, batch=self.B, b_batch_rows=n, d_batch_rows=n, causal=2)
                gate = s['hact'][:, half:]
                L.check(lib.progen_ln_shift_bwd(self.dgn.data_ptr(), half, self.act_dt, gate.data_ptr(), hid, self.act_dt,
                                                self.Pf(g + '/~/layer_norm', 'scale').data_ptr(), s['mean3'].data_ptr(),
                                                s['rstd3'].data_ptr(), 0, da[:, half:].data_ptr(), hid,
                                                L.ptr(G(g + '/~/layer_norm', 'scale')), 0, T, half, n, 0, 0, st), 'ln_bwd_sgu')
                L.check(lib.progen_gelu_bwd(da.data_ptr(), s['u'].data_ptr(), self.act_dt, T * hid, st), 'gelu_bwd')
                du, n_in = da, hid
                if not frozen:
                    self.colsum(du, n_in, self.G(f + 'linear', 'b'))
            elif kind == 'glu':
                # the epilogue also adds the column sums of du into the proj_in bias gradient (interleaved like du)
                if not frozen:
                    self.wgrad_gemm(s['hact'], hid, dres_lp, d, self.G(f + 'linear_1', 'w'))
                self.dgrad_gemm(dres_lp, d, self.W(f + 'linear_1', 'w'), hid, self.du, epi=L.EPI_GLU_BWD, ldo=2 * hid,
                                aux=s['u'], ldaux=2 * hid, colsum=G(f + 'linear', 'b'),
                                **tail(s['hact'], hid, f + 'linear_1', dres_lp, d))
                du, n_in = self.du, 2 * hid
            else:
                if not frozen:
                    self.wgrad_gemm(s['hact'], hid, dres_lp, d, self.G(f + 'linear_1', 'w'))
                self.dgrad_gemm(dres_lp, d, self.W(f + 'linear_1', 'w'), hid, self.dh_, epi=L.EPI_GELU_BWD, aux=s['u'], ldaux=hid,
                                colsum=G(f + 'linear', 'b'), **tail(s['hact'], hid, f + 'linear_1', dres_lp, d))
                du, n_in = self.dh_, hid
            if not frozen:
                self.wgrad_gemm(s['y2'], d, du, n_in, self.G(f + 'linear', 'w'))
            self.dgrad_gemm(du, n_in, self.W(f + 'linear', 'w'), d, self.dy, **tail(s['y2'], d, f + 'linear', du, n_in))
            self.ln_bwd_res(self.dy, x1, self.Pf(f + 'layer_norm', 'scale'), s['mean2'], s['rstd2'], G(f + 'layer_norm', 'scale'), shift,
                            next_bias_grad=G(a + 'linear_1', 'b'))
            # ---- LocalAttention backward
            if not frozen:
                self.wgrad_gemm(s['att'], I, dres_lp, d, self.G(a + 'linear_1', 'w'))
            self.dgrad_gemm(dres_lp, d, self.W(a + 'linear_1', 'w'), I, self.datt, **tail(s['att'], I, a + 'linear_1', dres_lp, d))
            self.attn_bwd(s['qkv'], s['att'], self.datt, s['lse'], self.dqkv)
            if not self.attn_tc:
                L.check(lib.progen_rotary_bwd(self.dqkv.data_ptr(), 3 * I, self.act_dt, self.rot_sin.data_ptr(),
                                              self.rot_cos.data_ptr(), T, 3 * I, n, self.dh, st), 'rotary_bwd')
            if not frozen:
                self.wgrad_gemm(s['y1'], d, self.dqkv, 3 * I, self.G(a + 'linear', 'w'))
            self.dgrad_gemm(self.dqkv, 3 * I, self.W(a + 'linear', 'w'), d, self.dy, **tail(s['y1'], d, a + 'linear', self.dqkv, 3 * I))
            self.ln_bwd_res(self.dy, x0, self.Pf(a + 'layer_norm', 'scale'), s['mean1'], s['rstd1'], G(a + 'layer_norm', 'scale'), shift,
                            next_bias_grad=G(P + f'ff{i - 1}/~/linear_1', 'b') if i > 0 else None)
            if self.on_layer_grads is not None:
                # every weight-matrix gradient of layer i is final: the DDP trainer starts its all-reduce here so the
                # transfer overlaps the backward pass of layers i-1 .. 0
                self.on_layer_grads(i)
        if frozen:
            lo.scale_b_grads()
            return
        L.check(lib.progen_embed_bwd(self.tok.data_ptr(), self.dres.data_ptr(), self.G(P + 'embed', 'embeddings').data_ptr(),
                                     T, d, self.V, st), 'embed_bwd')
