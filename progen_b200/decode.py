"""KV-cached sampler: the device-side equivalent of `progen_transformer.utils.sample` (utils.py:106-135).

The reference re-runs the whole model over the full padded sequence for every generated token; here `BatchDecoder`
consumes one position per step and keeps rotated K/V rows, the token-shift halves and the SGU gate history per layer
and sequence.  Every position of a launch runs inside ONE persistent kernel (`progen_decode_run`,
csrc/decode_persist.cu): the token loop, the sampler and the position counter stay on the device, and the loop never
synchronises with the host.  `BatchDecoder.sample` keeps the reference's quirks: top-k keeps k-1 logits and zeroes the
rest (Q6), `add_bos` adds the first sampled id to the last prime token (Q5), everything after the second pad is
cleared (Q7).  `BatchDecoder.generate` / `generate_queue` run the standard sampler with the settings of a `Sampling`."""
import ctypes as C
from dataclasses import dataclass

import numpy as np
import torch

from . import lib as L
from .engine import P, layer_kinds

_P, _I = C.c_void_p, C.c_int32


def integer(v, what, lo, hi):
    """v as an int; ProgenError unless it is an integer (not a bool) in [lo, hi]"""
    if isinstance(v, (bool, np.bool_)) or not isinstance(v, (int, np.integer)) or not lo <= int(v) <= hi:
        raise L.ProgenError(f'generate: {what} must be an integer in [{lo}, {hi}], got {v!r}')
    return int(v)


def prompt_ids(prompts, V, max_length):
    """each prompt as an int64 array; ProgenError unless it is 1-D, of integer ids in [1, V), and leaves a position to
    draw before max_length"""
    out = []
    for p in prompts:
        a = np.asarray(p)
        if a.ndim != 1 or (a.size and not np.issubdtype(a.dtype, np.integer)):
            raise L.ProgenError('generate: a prompt must be a string or a 1-D integer array')
        a = a.astype(np.int64)
        if a.size and (a.min() < 1 or a.max() >= V):
            raise L.ProgenError(f'generate: prompt ids must lie in [1, {V}) (0 is BOS / EOS)')
        if a.size + 1 >= max_length:
            raise L.ProgenError(f'generate: a prompt of {a.size} ids leaves nothing to generate before max_length {max_length}')
        out.append(a)
    return out


@dataclass(frozen=True, eq=False)
class Sampling:
    """The settings of the standard sampler (sampler 1 of csrc/decode_persist.cu) for one generate call, checked by
    `Sampling.check`; `ProGen.generate` documents each of them"""
    temperature: float
    top_k: int | None
    top_p: float | None
    seed: int
    logit_bias: np.ndarray | None                    # [V] float32
    min_new_tokens: int
    repetition_penalty: float
    repetition_window: int

    @classmethod
    def check(cls, V, n, min_new_max, keep_an_id, *, temperature=1.0, top_k=None, top_p=None, seed=0, logit_bias=None,
              min_new_tokens=0, repetition_penalty=1.0, repetition_window=0):
        """The settings for a model of V ids and seq_len n, or ProgenError before any device work.  The two rules the
        callers set: min_new_tokens lies in [0, min_new_max], and with keep_an_id logit_bias must leave some id of
        [1, V) allowed.  `ProGen.generate` passes max_length - 2 and True; `BatchDecoder` passes n and False, the
        kernel's own limits (min_new_tokens = n bans EOS for the whole row)."""
        seed = integer(seed, 'seed', 0, (1 << 64) - 1)
        top_k = None if top_k is None else integer(top_k, 'top_k', 1, V)
        try:
            temperature = float(temperature)
            top_p = None if top_p is None else float(top_p)
        except (TypeError, ValueError):
            raise L.ProgenError('generate: temperature and top_p must be numbers') from None
        if not (np.isfinite(temperature) and temperature >= 0.0):
            raise L.ProgenError(f'generate: temperature must be finite and >= 0, got {temperature}')
        if top_p is not None and not 0.0 < top_p <= 1.0:
            raise L.ProgenError(f'generate: top_p must lie in (0, 1], got {top_p}')
        min_new_tokens = integer(min_new_tokens, 'min_new_tokens', 0, min_new_max)
        repetition_window = integer(repetition_window, 'repetition_window', 0, n)
        try:
            repetition_penalty = float(repetition_penalty)
        except (TypeError, ValueError):
            raise L.ProgenError('generate: repetition_penalty must be a number') from None
        if not (np.isfinite(repetition_penalty) and repetition_penalty > 0.0):
            raise L.ProgenError(f'generate: repetition_penalty must be finite and > 0, got {repetition_penalty}')
        if logit_bias is not None:
            try:
                with np.errstate(over='ignore'):
                    logit_bias = np.asarray(logit_bias, np.float64).astype(np.float32)   # the kernel adds fp32
            except (TypeError, ValueError):
                raise L.ProgenError('generate: logit_bias must be an array of floats') from None
            if logit_bias.shape != (V,):
                raise L.ProgenError(f'generate: logit_bias must have shape ({V},), got {logit_bias.shape}')
            if np.isnan(logit_bias).any() or (logit_bias == np.inf).any():
                raise L.ProgenError('generate: logit_bias must not contain NaN or +inf (in float32)')
            if keep_an_id and not np.isfinite(logit_bias[1:]).any():
                raise L.ProgenError('generate: logit_bias bans every id in [1, V)')
        return cls(temperature, top_k, top_p, seed, logit_bias, min_new_tokens, repetition_penalty, repetition_window)


class DecodeLayer(C.Structure):
    _fields_ = [('kind', _I), ('_pad', _I)] + [(k, _P) for k in (
        'ln1_scale', 'wqkv_t', 'wo_t', 'bo', 'ln2_scale', 'win_t', 'bin', 'wout_t', 'bout', 'sgu_ln_scale', 'sgu_w', 'sgu_b',
        'sgu_proj_t', 'sgu_proj_b', 'kcache', 'vcache', 'shift1', 'shift2', 'gn_hist')]


class DecodeRun(C.Structure):
    _fields_ = [(k, _I) for k in ('n', 'd', 'heads', 'dim_head', 'inner', 'window', 'hid', 'V', 'depth', 'wdtype', 'shift_tokens',
                                  'top_k', 'B', 'pos0', 'nsteps', '_pad')] + \
               [(k, _P) for k in ('embed', 'lnf_scale', 'whead_t', 'bhead', 'rot_sin', 'rot_cos', 'layers', 'seq', 'start', 'noise',
                                  'logits_all', 'x', 'q', 'att', 'att_part', 'att_count', 'u', 'sg', 'pj', 'logits', 'grid_bar', 'prof')] + \
               [('sampler', _I), ('temperature', C.c_float), ('top_p', C.c_float), ('_pad1', _I), ('seed', C.c_uint64)] + \
               [(k, _P) for k in ('sample_id', 'token_logp', 'end', 'n_ended', 'steps_run', 'logit_bias')] + \
               [('repetition_penalty', C.c_float), ('repetition_window', _I), ('min_new_tokens', _I), ('_pad2', _I)] + \
               [(k, _P) for k in ('slot_row', 'slot_pos', 'next_row', 'done')] + [('num_rows', _I), ('max_length', _I)] + \
               [(k, _P) for k in ('position_bias', 'position_bias_table')] + [('position_bias_len', _I), ('_pad3', _I)] + \
               [('motif', _P)]


class MotifPattern(C.Structure):
    _fields_ = [(k, C.c_uint64) for k in ('optional', 'lead', 'last', 'anchors')]


class MotifDesc(C.Structure):
    """progen_motif_t: the device descriptor of the motif constraints (include/progen_b200.h, motif.py)"""
    _fields_ = [('num_patterns', _I), ('required', _I), ('need', _I * 65), ('_pad', _I), ('pattern', MotifPattern * 9),
                ('mask', _P), ('state', _P)]


class BatchDecoder:
    """Whole-generation decode in ONE persistent kernel (csrc/decode_persist.cu, `progen_decode_run`): B sequences advance
    in lock step, the weights stream once per position for all of them, the token loop / sampler / position stay on the
    device.  B = 1 is the reference's `sample` (utils.py:106-135) with every quirk kept (Q5 add_bos off-by-one, Q6 top-k
    keeps k-1 and zeroes the rest, Q7 truncation after the second pad); B > 1 decodes several primes at once — each
    sequence keeps its own prime and samples from its own `start` position on."""

    def __init__(self, config, params, batch=1, weights_dtype=torch.float32, keep_logits=False, device=None):
        L.require_device()
        self.lib = L.load()
        self.cfg = cfg = config
        self.dev = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
        self.B = B = int(batch)
        if not 1 <= B <= 64:
            raise L.ProgenError('BatchDecoder: 1 <= batch <= 64')
        d, n = cfg['dim'], cfg['seq_len']
        I = cfg['heads'] * cfg['dim_head']
        hid = d * cfg['ff_mult']
        # the shapes progen_decode_run accepts, refused here before any device buffer is allocated
        limits = [(cfg['dim_head'] in (8, 16, 32, 64), f"dim_head in {{8, 16, 32, 64}} (got {cfg['dim_head']})"),
                  (hid % 256 == 0, f"dim * ff_mult a multiple of 256 (got {hid})"),
                  (d % 8 == 0 and I % 8 == 0, f'dim and heads * dim_head multiples of 8 (got {d}, {I})'),
                  (max(d, I, hid) <= 8192, f'dim, heads * dim_head and dim * ff_mult <= 8192 (got {d}, {I}, {hid})'),
                  (cfg['num_tokens'] % 2 == 0 and cfg['num_tokens'] <= 512, f"an even num_tokens <= 512 (got {cfg['num_tokens']})"),
                  (1 <= cfg['window_size'] <= 512, f"window_size <= 512 (got {cfg['window_size']})")]
        for ok, what in limits:
            if not ok:
                raise L.ProgenError(f'BatchDecoder: the persistent decode kernel needs {what}')
        self.n, self.V = n, cfg['num_tokens']
        self.keep = []
        f32 = lambda a: self._hold(torch.tensor(np.ascontiguousarray(np.asarray(a, np.float32)), device=self.dev))
        wt = lambda a: self._hold(torch.tensor(np.ascontiguousarray(np.asarray(a, np.float32).T), device=self.dev).to(weights_dtype).contiguous())
        zeros = lambda *s, dtype=torch.float32: self._hold(torch.zeros(*s, device=self.dev, dtype=dtype))
        # (module, name) -> (the decoder's buffer of that parameter, whether it holds the transpose): load_weights
        self.leaves = {}

        def leaf(module, name, transposed, a=None):
            ptr = (wt if transposed else f32)(params[module][name] if a is None else a)
            self.leaves[(module, name)] = (self.keep[-1], transposed)
            return ptr
        kinds = layer_kinds(cfg['depth'], cfg['global_mlp_depth'], cfg['ff_glu'])
        layers = (DecodeLayer * len(kinds))()
        self.state = []
        self.caches = []                                  # per layer: name -> the cache tensor of the layer table
        for i, kind in enumerate(kinds):
            a, f = P + f'attn{i}/~/', P + f'ff{i}/~/'
            Lr = layers[i]
            self.caches.append({})
            Lr.kind = {'glu': 0, 'gelu': 1, 'sgu': 2}[kind]
            Lr.ln1_scale = leaf(a + 'layer_norm', 'scale', False)
            Lr.wqkv_t = leaf(a + 'linear', 'w', True)
            Lr.wo_t = leaf(a + 'linear_1', 'w', True)
            Lr.bo = leaf(a + 'linear_1', 'b', False)
            Lr.ln2_scale = leaf(f + 'layer_norm', 'scale', False)
            Lr.win_t = leaf(f + 'linear', 'w', True)
            Lr.bin = leaf(f + 'linear', 'b', False)
            Lr.wout_t = leaf(f + 'linear_1', 'w', True)
            Lr.bout = leaf(f + 'linear_1', 'b', False)
            if kind == 'sgu':
                g = f + 'sgu'
                Lr.sgu_ln_scale = leaf(g + '/~/layer_norm', 'scale', False)
                Lr.sgu_w = leaf(g, 'spatial_weights', False)
                Lr.sgu_b = leaf(g, 'spatial_biases', False, np.asarray(params[g]['spatial_biases']).reshape(-1))
                Lr.sgu_proj_t = leaf(g + '/~/linear', 'w', True)
                Lr.sgu_proj_b = leaf(g + '/~/linear', 'b', False)
                Lr.gn_hist = self._state(zeros(B, n, hid // 2), 'gn_hist')
            Lr.kcache = self._state(zeros(B, n, I), 'kcache')           # [B, heads, n, dim_head]
            Lr.vcache = self._state(zeros(B, n, I), 'vcache')
            Lr.shift1 = self._state(zeros(B, 2, d // 2), 'shift1')
            Lr.shift2 = self._state(zeros(B, 2, d // 2), 'shift2')
        # the kernel reads the layer table from DEVICE memory
        raw = np.frombuffer(bytes(layers), dtype=np.uint8).copy()
        self.layers_dev = torch.from_numpy(raw).to(self.dev)
        m = self.m = DecodeRun()
        m.n, m.d, m.heads, m.dim_head, m.inner, m.window, m.hid, m.V, m.depth = n, d, cfg['heads'], cfg['dim_head'], I, \
            cfg['window_size'], hid, self.V, len(kinds)
        m.wdtype = L.BF16 if weights_dtype == torch.bfloat16 else L.F32
        m.shift_tokens = int(cfg['shift_tokens'])
        m.B = B
        m.embed = leaf(P + 'embed', 'embeddings', False)
        m.lnf_scale = leaf(P + 'layer_norm', 'scale', False)
        m.whead_t = leaf(P + 'linear', 'w', True)
        m.bhead = leaf(P + 'linear', 'b', False)
        inv_freq = 1.0 / (10000 ** (np.arange(0, cfg['dim_head'], 2, dtype=np.float64) / cfg['dim_head']))
        ang = np.arange(n, dtype=np.float64)[:, None] * inv_freq[None, :]
        m.rot_sin, m.rot_cos = f32(np.sin(ang)), f32(np.cos(ang))
        m.layers = self.layers_dev.data_ptr()
        self.seq = torch.zeros(B, n, device=self.dev, dtype=torch.int32)
        self.start = torch.zeros(B, device=self.dev, dtype=torch.int32)
        m.seq, m.start = self.seq.data_ptr(), self.start.data_ptr()
        self.logits_all = torch.zeros(B, n, self.V, device=self.dev) if keep_logits else None
        m.logits_all = self.logits_all.data_ptr() if keep_logits else 0
        self.noise = None
        m.noise = 0
        ks = (2 * cfg['window_size'] + 31) // 32
        m.x, m.q, m.att = zeros(B, d), zeros(B, I), zeros(B, I)
        m.att_part = zeros(B, cfg['heads'], ks, cfg['dim_head'] + 4)
        self.att_count = torch.zeros(B * cfg['heads'], device=self.dev, dtype=torch.int32)
        m.att_count = self.att_count.data_ptr()
        m.u, m.sg, m.pj, m.logits = zeros(B, hid), zeros(8, B, hid // 2), zeros(B, hid // 2), zeros(B, self.V)
        self.grid_bar = torch.zeros(1, device=self.dev, dtype=torch.int32)
        m.grid_bar = self.grid_bar.data_ptr()
        m.repetition_penalty = 1.0                        # constraints off

    def load_weights(self, engine, lora=None):
        """Rewrite the decoder's weights in place from an Engine of the same config (progen_decode_load_weight): every
        parameter from its fp32 master copy, or with `lora` (lora.Adapters on that engine, whose base is frozen) only
        the adapted projections, as W + s A B.  Allocates nothing: the caches and the device layer table keep their
        pointers.  The weights then equal those of a decoder built from `engine.export_params()` (with lora: from the
        float32, no-FMA W + s A B of the float32 leaves)."""
        from .lora import adapter_modules
        lib, st = self.lib, L.stream()
        lay = engine.layout
        adapted = None if lora is None else {m for m, _, _, _ in adapter_modules(self.cfg)}
        for (module, name), (t, transposed) in self.leaves.items():
            if adapted is not None and not (name == 'w' and module in adapted):
                continue
            spec = lay.by_key[(module, name)]
            fan_in, fan_out = spec.shape if transposed else (1, spec.size)
            a = b = 0
            rank, scale = 0, 1.0
            if adapted is not None:
                la = lora.layout
                a, b = la.seg(lora.params, module, 'lora_a').data_ptr(), la.seg(lora.params, module, 'lora_b').data_ptr()
                rank, scale = lora.r, lora.scale
            L.check(lib.progen_decode_load_weight(lay.seg(engine.params, module, name).data_ptr(), a, b, rank, scale,
                                                  fan_in, fan_out, int(spec.interleave), t.data_ptr(), L.dt(t), st),
                    f'decode_load_weight {module}/{name}')

    def _hold(self, t):
        self.keep.append(t)
        return t.data_ptr()

    def _state(self, ptr, name):
        self.state.append(self.keep[-1])
        self.caches[-1][name] = self.keep[-1]
        return ptr

    def reset(self):
        for t in self.state:
            t.zero_()
        self.att_count.zero_()

    def prefill(self, engine, prompts):
        """Reset, then fill the caches of rows 0 .. len(prompts) - 1 for positions < P from ONE inference forward of
        `engine` (an Engine with this decoder's config and parameters) over the distinct prompts, each laid out as
        `generate` lays it out, [0 (BOS), prompt, 0...].  Every prompt must have the same length P; returns P, to pass to
        `generate(prompts, prefilled=P)` with the same prompts.  P = 0 (empty prompts) prefills nothing.  The caches then
        hold the forward's arithmetic (bf16 activations under mixed precision) rather than this kernel's."""
        if not 1 <= len(prompts) <= self.B:
            raise L.ProgenError(f'prefill: 1 <= prompts <= {self.B}')
        seq0, starts = self._rows(prompts, self.n)
        if len(set(starts.tolist())) != 1:
            raise L.ProgenError('prefill: every prompt must have the same length')
        keys = ('num_tokens', 'dim', 'seq_len', 'depth', 'window_size', 'global_mlp_depth', 'heads', 'dim_head', 'ff_mult',
                'ff_glu', 'shift_tokens')
        if any(engine.cfg[k] != self.cfg[k] for k in keys):
            raise L.ProgenError('prefill: the engine and the decoder have different model configurations')
        self.reset()
        P = int(starts[0]) - 1
        if P == 0:
            return 0
        distinct, row_map = {}, []
        for row in seq0:
            row_map.append(distinct.setdefault(row.tobytes(), len(distinct)))
        ids = np.stack([np.frombuffer(k, np.int32) for k in distinct])
        engine.prefill(ids, P, self._prefill_sink(torch.tensor(row_map, dtype=torch.int32, device=self.dev), len(distinct)))
        return P

    def _prefill_sink(self, row_map, nsrc):
        """Engine.prefill sink: row b of every cache takes forward row row_map[b] (progen_gather_rows_f32)"""
        cfg, n = self.cfg, self.n
        h, dh, half_d = cfg['heads'], cfg['dim_head'], cfg['dim'] // 2
        I = h * dh

        def gather(buf, row0, rows, col0, groups, cols, dst, b_stride, g_stride, row_stride):
            L.check(self.lib.progen_gather_rows_f32(buf.data_ptr(), buf.stride(0), L.dt(buf), nsrc, n, row_map.data_ptr(),
                                                    row_map.numel(), row0, rows, col0, groups, cols, dst, b_stride, g_stride,
                                                    row_stride, L.stream()), 'gather_rows_f32')

        def sink(i, name, buf, P):
            c = self.caches[i]
            if name == 'qkv':                             # k, v rows 0..P-1 (rotated) -> [B, heads, n, dim_head]
                for sec, cache in ((1, c['kcache']), (2, c['vcache'])):
                    gather(buf, 0, P, sec * I, h, dh, cache.data_ptr(), h * n * dh, n * dh, dh)
            elif name in ('y1', 'y2') and cfg['shift_tokens']:
                # LN row P after the shift: its first half is position P-1's, the half the kernel reads at P (slot P & 1)
                st = c['shift1' if name == 'y1' else 'shift2']
                gather(buf, P, 1, 0, 1, half_d, st.data_ptr() + (P & 1) * half_d * 4, 2 * half_d, 0, 0)
            elif name == 'gn':                            # normalised gate rows 0..P-1 -> [B, n, hid/2]
                gh = c['gn_hist']
                gather(buf, 0, P, 0, 1, gh.shape[-1], gh.data_ptr(), n * gh.shape[-1], 0, gh.shape[-1])
        return sink

    def profile_barriers(self, pos0, nsteps):
        """Run, recording clock64 at entry / exit of every grid barrier of the LAST step on CTA 0 and the last CTA.
        Returns an int64 array [2, events, 2] (events = barriers of one step)."""
        prof = torch.zeros(2 * 160 * 2 + 160 * 8, device=self.dev, dtype=torch.int64)
        self.m.prof = prof.data_ptr()
        try:
            self.run(pos0, nsteps)
            torch.cuda.synchronize()
        finally:
            self.m.prof = 0
        raw = prof.cpu().numpy()
        p = raw[:640].reshape(2, 160, 2)
        ev = int((p[0, :, 0] != 0).sum())
        self.last_marks = raw[640:].reshape(160, 8)[:ev]      # clock64 inside CTA 0's phases (0 = not recorded)
        return p[:, :ev]

    def run(self, pos0, nsteps, m=None):
        """launch the struct m (default self.m, the reference sampler's) for positions pos0 .. pos0 + nsteps - 1"""
        m = self.m if m is None else m
        self.grid_bar.zero_()
        m.pos0, m.nsteps = int(pos0), int(nsteps)
        L.check(self.lib.progen_decode_run(C.byref(m), L.stream()), 'decode_run')

    def sample(self, primes, length=None, top_k=None, add_bos=False, greedy=True, seed=0):
        """utils.py:106-135 for every prime of `primes` (a list of integer arrays, or one array for B = 1).
        Returns (ids [B, length] numpy int64, generated tokens counted over all sequences, device seconds)."""
        length = self.n if length is None else length
        assert length == self.n, 'the gMLP layers pin the sequence length (progen.py:175-181)'
        single = not isinstance(primes, (list, tuple))
        primes = [primes] if single else list(primes)
        assert len(primes) == self.B, f'expected {self.B} primes'
        seq0 = np.zeros((self.B, length), np.int32)
        starts = np.zeros(self.B, np.int32)
        for b, pr in enumerate(primes):
            pr = np.asarray(pr).astype(np.int64)
            sp = pr.shape[-1]
            pad_right = length - sp
            padding = (0, pad_right) if not add_bos else (1, pad_right - 1)
            seq0[b] = np.pad(pr, padding)
            starts[b] = sp                               # curr_pos starts at the prime length (utils.py:113)
        self.reset()
        self.seq.copy_(torch.as_tensor(seq0))
        self.start.copy_(torch.as_tensor(starts))
        self.m.top_k = int(top_k) if top_k is not None else 0
        if greedy:
            self.m.noise = 0
        else:
            g = torch.Generator(device=self.dev).manual_seed(int(seed))
            u = torch.rand(self.B, self.n, self.V, generator=g, device=self.dev)
            self.noise = -torch.log(-torch.log(u + 1e-20) + 1e-20)                # utils.py:102-104
            self.m.noise = self.noise.data_ptr()
        # The reference draws the token at curr_pos from logits[curr_pos - 1]; a prime of length 0 (sample.py's default
        # --prime '') starts at curr_pos = 0 and reads logits[-1] of the all-pad sequence — a full forward the cached step
        # cannot express, so position 0 is never sampled here (documented divergence for the empty prime).
        first = int(max(0, starts.min() - 1))
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        if first > 0:
            self.run(0, first)                           # prefill: only advances the caches (no sequence samples before its start)
        e0.record()
        self.run(first, length - 1 - first)              # positions first .. length-2: the last one writes seq[length-1]
        e1.record()
        torch.cuda.synchronize()
        seq = self.seq.cpu().numpy().astype(np.int64)
        after_eos = np.cumsum(seq == 0, axis=-1) > 1                               # utils.py:132-133
        out = seq * ~after_eos
        generated = int(sum(length - max(int(s), 1) for s in starts))
        return (out[0] if single else out), generated, e0.elapsed_time(e1) / 1e3

    def _rows(self, prompts, max_length):
        """-> (seq0 [R, n] int32: [0 (BOS), prompt, 0...] per prompt, starts [R] int32: 1 + prompt length), checked by
        `prompt_ids`"""
        ids = prompt_ids(prompts, self.V, max_length)
        seq0 = np.zeros((len(ids), self.n), np.int32)
        for b, a in enumerate(ids):
            seq0[b, 1:1 + len(a)] = a
        return seq0, np.array([1 + len(a) for a in ids], np.int32)

    def generate(self, prompts, *, temperature=1.0, top_k=None, top_p=None, seed=0, sample_ids=None, max_length=None,
                 logit_bias=None, min_new_tokens=0, repetition_penalty=1.0, repetition_window=0, position_bias=None,
                 prefilled=0, motif=None):
        """The standard sampler (sampler 1 of csrc/decode_persist.cu) for up to B prompts (integer arrays of ids in [1, V)).
        Each row is laid out as training data is, [0 (BOS), prompt..., 0...], and draws positions 1 + len(prompt) ..
        max_length - 1 until it samples EOS (id 0).  Row b uses the Philox stream sample_ids[b] (default b); the
        attention and SGU work splits are planned for the largest launch of the batch tile's class (1, 8 or 64 rows), so
        a row's result depends on (seed, its sample id) and that class, not on the other rows of the launch.  Fewer prompts than B run on a prefix of the caches.
        Constraints, applied to the logits of every draw before the filter (progen_b200.h, DESIGN.md §3.3): the ids present
        in the last `repetition_window` positions (0: all since BOS) have positive logits divided and negative ones
        multiplied by `repetition_penalty`; `logit_bias` ([V] floats, -inf bans an id) is added; EOS is banned for the
        first `min_new_tokens` draws of a row.  They do not change token_logp, the unfiltered model's log-probability.
        The settings are checked as `ProGen.generate` checks them (`Sampling.check`), except that min_new_tokens may be
        up to n and logit_bias may ban every id of [1, V).
        position_bias = (tables [Tb, Lb, V] float32, table_of_row [R] ints in [-1, Tb)): the draw of a row's generated
        offset j (0 = its first generated token) adds tables[table_of_row[r], j] to the logits after logit_bias and
        before the EOS ban, for j < Lb (-1: no table; -inf bans an id at that offset).
        prefilled = P > 0: `prefill` has filled the caches of these prompts for positions < P (P <= every prompt's
        length), so the caches are not reset and the kernel starts at position P instead of 0.
        motif: a motif.Motif (required / avoided PROSITE patterns), applied after every other adjustment: each row's
        state starts at zero (nothing generated) and the kernel bans the ids that break the patterns (progen_b200.h).
        Returns a dict of numpy arrays: ids [R, n] int64, token_logp [R, n] float32 (log p(ids[t] | ids[:t]) at drawn t,
        else 0), end [R] int32 (position of the EOS, n if none), start [R] int32; and steps_run (positions the last
        launch consumed before every row had ended, or its full length), device_s (that launch's device time) and
        prefill_s (device time of the launch that consumed the prompt positions before it, 0 when there was none)."""
        if not 1 <= len(prompts) <= self.B:
            raise L.ProgenError(f'generate: 1 <= prompts <= {self.B}')
        s = Sampling.check(self.V, self.n, self.n, False, temperature=temperature, top_k=top_k, top_p=top_p, seed=seed,
                           logit_bias=logit_bias, min_new_tokens=min_new_tokens, repetition_penalty=repetition_penalty,
                           repetition_window=repetition_window)
        return self._generate(prompts, s, sample_ids, max_length, position_bias, prefilled=prefilled, motif=motif)

    def generate_queue(self, prompts, *, slots=None, temperature=1.0, top_k=None, top_p=None, seed=0, sample_ids=None,
                       max_length=None, logit_bias=None, min_new_tokens=0, repetition_penalty=1.0, repetition_window=0,
                       position_bias=None, motif=None):
        """`generate` for Q = len(prompts) rows on `slots` (default min(B, Q), 2 <= slots <= min(B, Q)) sequences of ONE
        persistent launch: the rows form a queue, and a slot whose row ends (EOS, or position max_length - 1) takes the
        next row, which starts at position 0 with its prompt decoded like generated positions (csrc/decode_persist.cu,
        progen_b200.h).  A row's bits depend on its seed, sample id, prompt, the class of `slots` (2-8 or 9-64) and
        the GPU's SM count, not on its slot or the other rows, so each row equals what `generate` gives it in a launch of
        that class; the launch merely has no slot waiting for its longest row.  position_bias's table_of_row is indexed
        by queue row ([Q]), and so is the motif state.  Returns the dict of `generate` over the Q rows; steps_run is the
        positions the launch ran and prefill_s is 0."""
        Q = len(prompts)
        slots = min(self.B, Q) if slots is None else int(slots)
        if not 2 <= slots <= min(self.B, Q):
            raise L.ProgenError(f'generate_queue: 2 <= slots <= min(batch {self.B}, rows {Q})')
        s = Sampling.check(self.V, self.n, self.n, False, temperature=temperature, top_k=top_k, top_p=top_p, seed=seed,
                           logit_bias=logit_bias, min_new_tokens=min_new_tokens, repetition_penalty=repetition_penalty,
                           repetition_window=repetition_window)
        return self._generate(prompts, s, sample_ids, max_length, position_bias, slots=slots, motif=motif)

    def _generate(self, prompts, s, sample_ids, max_length, position_bias, prefilled=0, slots=None, motif=None):
        """One sampler-1 launch with the checked settings s (a Sampling).  slots None: row b runs on sequence b, after a
        launch that consumes the prompt positions from `prefilled` on; else the rows form the queue of `slots` sequences.
        It launches a copy of self.m with this call's buffers and sampler fields, so self.m keeps what `sample` runs."""
        n, dev, R = self.n, self.dev, len(prompts)
        max_length = n if max_length is None else integer(max_length, 'max_length', 2, n)
        seq0, starts = self._rows(prompts, max_length)
        sids = np.arange(R, dtype=np.int64) if sample_ids is None else np.asarray(sample_ids, np.int64).reshape(-1)
        if sids.shape != (R,):
            raise L.ProgenError('generate: one sample id per prompt')
        first = int(starts.min()) - 1                     # the first drawn position is start; it reads the logits of start - 1
        if not 0 <= int(prefilled) <= first:
            raise L.ProgenError(f'generate: prefilled must lie in [0, {first}] (the shortest prompt length)')
        prefilled = int(prefilled)
        position_bias = self._position_bias(position_bias, R)
        to_dev = lambda a: torch.as_tensor(a).to(dev)
        seq, start, sample_id = to_dev(seq0), to_dev(starts), to_dev(sids)
        token_logp = torch.zeros(R, n, device=dev, dtype=torch.float32)
        end = torch.full((R,), n, device=dev, dtype=torch.int32)
        counters = torch.tensor([0, 0, slots or 0, 0], device=dev, dtype=torch.int32)   # [n_ended, steps_run, next_row, done]
        m = DecodeRun.from_buffer_copy(self.m)
        m.B = R if slots is None else slots
        m.seq, m.start, m.sample_id, m.token_logp, m.end = (t.data_ptr() for t in (seq, start, sample_id, token_logp, end))
        c = counters.data_ptr()
        m.n_ended, m.steps_run = c, c + 4
        m.sampler, m.temperature, m.seed = 1, s.temperature, s.seed
        m.top_k, m.top_p = s.top_k or 0, 1.0 if s.top_p is None else s.top_p
        m.repetition_penalty, m.repetition_window, m.min_new_tokens = s.repetition_penalty, s.repetition_window, s.min_new_tokens
        if s.logit_bias is not None:                      # the device copies below live until the launch has synchronised
            bias = to_dev(s.logit_bias)
            m.logit_bias = bias.data_ptr()
        if position_bias is not None:
            tables, table_of_row = map(to_dev, position_bias)
            m.position_bias, m.position_bias_table = tables.data_ptr(), table_of_row.data_ptr()
            m.position_bias_len = tables.shape[1]
        m.max_length = max_length
        if motif is not None:                             # descriptor, masks and per-row state: one zeroed device block
            desc = self._motif_descriptor(motif, R)
            m.motif = desc.data_ptr()
        if slots is None:
            pre = (prefilled, first - prefilled)          # prefill: only advances the caches
            main = (first, max_length - 1 - first)        # positions first .. max_length - 2 (the last writes max_length - 1)
        else:
            slot_row = torch.arange(slots, device=dev, dtype=torch.int32)
            slot_pos = torch.zeros(slots, device=dev, dtype=torch.int32)
            m.next_row, m.done = c + 8, c + 12
            m.slot_row, m.slot_pos, m.num_rows = slot_row.data_ptr(), slot_pos.data_ptr(), R
            # while rows wait in the queue every slot is busy, and a row consumes at most max_length - 1 positions
            pre, main = (0, 0), (0, -(-R * (max_length - 1) // slots) + max_length - 1)
        if not prefilled:
            self.reset()                                  # (a queue row needs token-shift slot 0 zero at position 0)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        ev[0].record()
        if pre[1] > 0:
            self.run(*pre, m)
        ev[1].record()
        self.run(*main, m)
        ev[2].record()
        torch.cuda.synchronize()
        cnt = counters.cpu().numpy()
        if slots is not None and cnt[3] != R:
            raise L.ProgenError(f'generate_queue: {cnt[3]} of {R} rows retired in {cnt[1]} steps')
        return dict(ids=seq.cpu().numpy().astype(np.int64), token_logp=token_logp.cpu().numpy(), end=end.cpu().numpy(),
                    start=starts, steps_run=int(cnt[1]), device_s=ev[1].elapsed_time(ev[2]) / 1e3,
                    prefill_s=ev[0].elapsed_time(ev[1]) / 1e3 if pre[1] > 0 else 0.0)

    def _motif_descriptor(self, motif, rows):
        """progen_motif_t for `rows` rows in one device buffer: the descriptor, the masks [P, V] and the zeroed state
        [rows, P + 1] behind it"""
        mask, pat, need = motif.descriptor_arrays()
        P = len(pat)
        if not 1 <= P <= 9 or mask.shape != (P, self.V):
            raise L.ProgenError(f'generate: a motif needs 1 to 9 patterns over {self.V} ids')
        head = (C.sizeof(MotifDesc) + 15) // 16 * 16
        buf = torch.zeros(head + mask.nbytes + rows * (P + 1) * 8, dtype=torch.uint8, device=self.dev)
        d = MotifDesc()
        d.num_patterns, d.required = P, int(motif.required)
        d.need[:] = need.tolist()
        for k in range(P):
            d.pattern[k].optional, d.pattern[k].lead, d.pattern[k].last, d.pattern[k].anchors = (int(v) for v in pat[k])
        d.mask, d.state = buf.data_ptr() + head, buf.data_ptr() + head + mask.nbytes
        host = np.zeros(head + mask.nbytes, np.uint8)
        host[:C.sizeof(MotifDesc)] = np.frombuffer(bytes(d), np.uint8)
        host[head:] = np.frombuffer(np.ascontiguousarray(mask, np.uint64).tobytes(), np.uint8)
        buf[:head + mask.nbytes].copy_(torch.from_numpy(host))
        return buf

    def _position_bias(self, position_bias, rows):
        """checks position_bias of generate / generate_queue (`rows` rows); -> (float32 tables, int32 map) or None"""
        if position_bias is None:
            return None
        n = self.n
        try:
            tables, table_of_row = position_bias
            tables = np.ascontiguousarray(np.asarray(tables, np.float32))
            table_of_row = np.asarray(table_of_row)
        except (TypeError, ValueError):
            raise L.ProgenError('generate: position_bias must be a pair (tables [Tb, Lb, V], table_of_row [rows])') from None
        if tables.ndim != 3 or tables.shape[0] < 1 or not 1 <= tables.shape[1] <= n or tables.shape[2] != self.V:
            raise L.ProgenError(f'generate: position_bias tables must have shape [Tb >= 1, 1..{n}, {self.V}], '
                                f'got {tables.shape}')
        if np.isnan(tables).any() or (tables == np.inf).any():
            raise L.ProgenError('generate: position_bias tables must not contain NaN or +inf')
        if table_of_row.shape != (rows,) or (rows and not np.issubdtype(table_of_row.dtype, np.integer)):
            raise L.ProgenError(f'generate: position_bias needs one integer table index per row ({rows})')
        if rows and (table_of_row.min() < -1 or table_of_row.max() >= tables.shape[0]):
            raise L.ProgenError(f'generate: position_bias table indices must lie in [-1, {tables.shape[0]})')
        return tables, table_of_row.astype(np.int32)
