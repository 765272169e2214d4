"""`ProGen` — the drop-in for `progen_transformer.ProGen` (reference progen.py:235-243).

Same constructor keywords (including the accepted-and-ignored `attn_dim`, `clamp_gate`), and an object with
`.init(rng, seq) -> params` and `.apply(params, rng, seq) -> logits`, where `params` is the haiku-shaped nested dict
`{module_path: {name: array}}` of the reference (SURVEY §8(b)), so reference checkpoints and oracle parameters
interchange.  Everything below `.apply` runs as sm_90a kernels behind the C ABI (include/progen_b200.h).

Beyond the reference surface: `.apply` also accepts a batch (B, n); `.loss_and_grad(params, data)` is the fused
equivalent of `value_and_grad(get_loss_fn(model))` (utils.py:61-93) and `.preference_loss_and_grad` its preference
(DPO) twin over chosen / rejected pairs; `.trainer(...)` owns device-resident training
state (parameters, Adam moments, apply_every accumulator) for the train.py loop; `.score(params, data)` is an
inference-only forward returning per-sequence log-likelihoods (and optionally per-token log-probabilities and pooled
embeddings); `.score_variants` / `.mutational_scan` score substitutions against a wild type on that forward, cut to the
positions that count.
"""
import numpy as np
import torch

from . import lib as L
from .engine import Engine, build_param_specs, P


def _trunc_normal(rng, shape, std):
    r = rng.standard_normal(int(np.prod(shape)))
    bad = np.abs(r) > 2.0
    while bad.any():
        r[bad] = rng.standard_normal(int(bad.sum()))
        bad = np.abs(r) > 2.0
    return (r.reshape(shape) * std).astype(np.float32)


def _seed(rng):
    """an int seed, or the last element of a key-like array (a jax PRNGKey) -> int"""
    return int(rng) if isinstance(rng, (int, np.integer)) else int(np.asarray(rng).ravel()[-1])


def _batch_size(batch_size, what):
    """batch_size checked as an integer >= 1 -> int"""
    if isinstance(batch_size, (bool, np.bool_)) or not isinstance(batch_size, (int, np.integer)) or batch_size < 1:
        raise L.ProgenError(f'{what}: batch_size must be an integer >= 1, got {batch_size!r}')
    return int(batch_size)


def plan_launches(lengths, batch_size, by_length=False):
    """The decoder launches of `ProGen.generate` for N = len(lengths) rows (lengths[r]: row r's prompt length).
    Returns a list of (rows, real): rows is an int64 array of row indices, whose first `real` entries are the launch's rows
    in row order and the rest padding.  Launches take up to per_launch = min(batch_size, N) rows; by_length (forward
    prefill) runs only rows of one prompt length together, so every launch starts at the prefilled position of all its
    rows.  A ragged launch is padded with copies of its last row (same prompt and stream, so it ends when that row does)
    up to the smallest size of per_launch's class (1, 2-8 or 9-64 rows), which runs the same GEMV formulation and work
    split as the full launches: a row's result depends only on the class, not on which rows share its launch."""
    lengths = np.asarray(lengths, np.int64)
    N = len(lengths)
    per_launch = min(batch_size, N)
    min_rows = 9 if per_launch > 8 else (2 if per_launch > 1 else 1)
    groups = [np.flatnonzero(lengths == v) for v in np.unique(lengths)] if by_length else [np.arange(N)]
    out = []
    for g in groups:
        for c0 in range(0, len(g), per_launch):
            rows = g[c0:c0 + per_launch].astype(np.int64)
            pad = max(0, min_rows - len(rows))
            out.append((np.concatenate([rows, np.full(pad, rows[-1], np.int64)]), len(rows)))
    return out


# `ProGen.generate` feeds at most this many rows per slot to one queue launch: it bounds the launch's [rows, seq_len] ids
# and log-probabilities in device memory and the time one launch holds the GPU
QUEUE_ROWS_PER_SLOT = 64
# ... and position-bias tables (`generate(position_bias=, fixed=)`) of at most this many bytes: one [seq_len, V] table is
# 1 MiB at seq_len 1024 and V 256, and a queue launch of distinct prompts could otherwise hold thousands of them
QUEUE_TABLE_BYTES = 256 << 20


def plan_queue(n_rows, batch_size, row_table=None, table_bytes=0):
    """The queue launches of `ProGen.generate` (prefill='decode') for n_rows rows: -> (slots, chunks), slots =
    min(batch_size, n_rows) sequences per launch and chunks a list of int64 arrays of row indices in row order, each run
    as the queue of one launch.  Rows are split into the fewest chunks of at most QUEUE_ROWS_PER_SLOT * slots rows, of
    near-equal size, so every chunk holds at least `slots` rows.  With row_table ([n_rows] ints: each row's position
    table, -1 = none) and table_bytes (the bytes of one table), a chunk is further cut, in row order, before the row
    whose table would take its distinct tables past QUEUE_TABLE_BYTES, but never below `slots` rows (a last piece that
    short joins the one before it).  None when slots < 2: the single-stream kernel keeps one launch per row
    (`plan_launches`)."""
    slots = min(batch_size, n_rows)
    if slots < 2:
        return None
    k = -(-n_rows // (QUEUE_ROWS_PER_SLOT * slots))
    chunks = [c.astype(np.int64) for c in np.array_split(np.arange(n_rows), k)]
    if row_table is None or table_bytes <= 0:
        return slots, chunks
    row_table = np.asarray(row_table, np.int64)
    cap = max(1, QUEUE_TABLE_BYTES // table_bytes)           # distinct tables per launch
    out = []
    for c in chunks:
        pieces, cur, seen = [], [], set()
        for r in c.tolist():
            t = int(row_table[r])
            if t >= 0 and t not in seen and len(seen) >= cap and len(cur) >= slots:
                pieces.append(cur)
                cur, seen = [], set()
            cur.append(r)
            if t >= 0:
                seen.add(t)
        if pieces and len(cur) < slots:
            pieces[-1] += cur
        else:
            pieces.append(cur)
        out += [np.asarray(q, np.int64) for q in pieces]
    return slots, out


def plan_generate(lengths, batch_size, prefill='decode', row_table=None, table_bytes=0):
    """The decoder launches of `ProGen.generate` for N = len(lengths) rows: a list of (rows, real, slots).  With
    prefill='decode' and at least two rows per launch each chunk of `plan_queue` is the queue of one launch on `slots`
    sequences (real = len(rows)); otherwise the launches of `plan_launches` keep rows fixed to sequences (slots None)."""
    queue = plan_queue(len(lengths), batch_size, row_table, table_bytes) if prefill == 'decode' else None
    if queue is not None:
        slots, chunks = queue
        return [(c, len(c), slots) for c in chunks]
    return [(rows, real, None) for rows, real in plan_launches(lengths, batch_size, by_length=prefill == 'forward')]


def _per_prompt(arg, n_prompts, what, single):
    """`arg` for every prompt: one value (single(arg) true) for all, or a list with one entry (or None) per prompt"""
    if arg is None:
        return [None] * n_prompts
    if single(arg):
        return [arg] * n_prompts
    if not isinstance(arg, (list, tuple)) or len(arg) != n_prompts:
        raise L.ProgenError(f'generate: {what} must be one value for every prompt or a list of {n_prompts} (one per prompt)')
    return list(arg)


def position_tables(starts, V, n, max_length, position_bias=None, fixed=None, logit_bias=None, min_new_tokens=0):
    """The position tables of `ProGen.generate` for prompts whose first generated position is starts[i] (1 + prompt
    length).  position_bias: None, a [T, V] array for every prompt, or a list of one array or None per prompt; fixed:
    None, a dict {k: residue} for every prompt, or a list of one dict or None per prompt (k: 1-based generated offset;
    residue: one character, encoded like training text, or an id in [1, V)).  A prompt's table row j is the bias of its
    generated offset j + 1: its position_bias row (0 past its end) plus, for fixed residues, 0 at the fixed id and -inf
    elsewhere at offset k, and -inf on EOS at every offset before its last fixed offset.  Checked, with ProgenError naming
    the prompt and the offset: offsets in [1, max_length - starts[i]], residues in the vocabulary, and every reachable
    offset keeps a candidate (an id with logit_bias + row finite; EOS not counted at offsets <= min_new_tokens).
    Returns (tables, prompt_table): the distinct tables (float32 [L, V], L <= n; equal tables stored once) and an int64
    array with each prompt's table index (-1: none)."""
    from .data import encode_tokens
    P = len(starts)
    biases = _per_prompt(position_bias, P, 'position_bias', lambda a: not isinstance(a, (list, tuple)))
    fixes = _per_prompt(fixed, P, 'fixed', lambda a: isinstance(a, dict))
    lb = np.zeros(V, np.float32) if logit_bias is None else np.asarray(logit_bias, np.float32)
    tables, index, prompt_table = [], {}, np.full(P, -1, np.int64)
    for i in range(P):
        reach = max_length - int(starts[i])              # generated offsets 1 .. reach fit before max_length
        b, f = biases[i], fixes[i]
        rows = None
        if b is not None:
            try:
                with np.errstate(over='ignore'):
                    rows = np.asarray(b, np.float64).astype(np.float32)
            except (TypeError, ValueError):
                raise L.ProgenError(f'generate: position_bias of prompt {i} must be an array of floats') from None
            if rows.ndim != 2 or not 1 <= rows.shape[0] <= n or rows.shape[1] != V:
                raise L.ProgenError(f'generate: position_bias of prompt {i} must have shape [T, {V}] with 1 <= T <= {n}, '
                                    f'got {rows.shape}')
            if np.isnan(rows).any() or (rows == np.inf).any():
                raise L.ProgenError(f'generate: position_bias of prompt {i} must not contain NaN or +inf (in float32)')
        if f is not None:
            if not isinstance(f, dict):
                raise L.ProgenError(f'generate: fixed of prompt {i} must be a dict {{offset: residue}} or None')
            ids = {}
            for k, res in f.items():
                if isinstance(k, (bool, np.bool_)) or not isinstance(k, (int, np.integer)) or not 1 <= int(k) <= reach:
                    raise L.ProgenError(f'generate: fixed offset {k!r} of prompt {i} must be an integer in [1, {reach}] '
                                        f'(1-based, reachable before max_length {max_length})')
                if isinstance(res, str) and len(res) == 1:
                    c = encode_tokens(res)[0]
                elif isinstance(res, (int, np.integer)) and not isinstance(res, (bool, np.bool_)):
                    c = int(res)
                else:
                    raise L.ProgenError(f'generate: fixed residue at offset {k} of prompt {i} must be one character or an id')
                if not 1 <= c < V:
                    raise L.ProgenError(f'generate: fixed residue {res!r} at offset {k} of prompt {i} is outside the '
                                        f'vocabulary (ids in [1, {V}))')
                ids[int(k)] = c
            if ids:
                last = max(ids)
                fx = np.zeros((last, V), np.float32)
                fx[:, 0] = -np.inf                       # no EOS before the last fixed residue
                for k, c in ids.items():
                    fx[k - 1] = -np.inf
                    fx[k - 1, c] = 0.0
                if rows is None:
                    rows = fx
                else:
                    L_ = max(len(rows), last)
                    t = np.zeros((L_, V), np.float32)
                    t[:len(rows)] = rows
                    t[:last] += fx
                    rows = t
        if rows is None:
            continue
        for j in range(min(len(rows), reach)):
            ok = np.isfinite(lb + rows[j])
            if j < min_new_tokens:
                ok[0] = False
            if not ok.any():
                raise L.ProgenError(f'generate: prompt {i} has no id left to draw at generated offset {j + 1} (the logit '
                                    f'bias, position bias, fixed residues and min_new_tokens together ban every id)')
        key = (rows.shape, rows.tobytes())
        if key not in index:
            index[key] = len(tables)
            tables.append(rows)
        prompt_table[i] = index[key]
    return tables, prompt_table


def launch_tables(tables, row_table, rows):
    """position_bias of one decoder launch over `rows` (row indices), for BatchDecoder.generate / generate_queue: the
    distinct tables its rows use, stacked and zero-padded to the longest (a zero row changes no logit), and each launch
    row's index into them.  None when no row has a table."""
    t = np.asarray(row_table, np.int64)[np.asarray(rows, np.int64)]
    used = np.unique(t[t >= 0])
    if used.size == 0:
        return None
    Lb = max(len(tables[u]) for u in used)
    stack = np.zeros((len(used), Lb, tables[used[0]].shape[1]), np.float32)
    for i, u in enumerate(used):
        stack[i, :len(tables[u])] = tables[u]
    return stack, np.where(t >= 0, np.searchsorted(used, t), -1).astype(np.int32)


class ProGen:
    def __init__(self, *, num_tokens, dim, seq_len, depth, window_size=256, global_mlp_depth=2, heads=8, dim_head=64,
                 ff_mult=4, ff_glu=True, attn_dim=None, clamp_gate=True, shift_tokens=True, mixed_precision=False,
                 mixed_precision_policy=None, recompute=False):
        # attn_dim / clamp_gate are accepted and ignored, exactly like the reference (progen.py:201-202)
        # recompute (DESIGN.md §3.12): training steps keep one residual checkpoint per layer and re-run each layer's
        # forward in the backward pass; a way of running, so it is not part of `config` (nor of checkpoints)
        self.config = dict(num_tokens=num_tokens, dim=dim, seq_len=seq_len, depth=depth, window_size=window_size,
                           global_mlp_depth=global_mlp_depth, heads=heads, dim_head=dim_head, ff_mult=ff_mult,
                           ff_glu=ff_glu, attn_dim=attn_dim, clamp_gate=clamp_gate, shift_tokens=shift_tokens)
        assert seq_len % window_size == 0, 'sequence length must be divisible by the window size'   # progen.py:80
        self.mixed_precision = bool(mixed_precision)
        self._recompute = bool(recompute)
        self._engine = None
        self._loaded = None
        self._gen_decoder = self._gen_params = None

    # ---- engine (created lazily so that constructing a model does not need a GPU; using it does)
    @property
    def engine(self):
        if self._engine is None:
            self._engine = Engine(self.config, self.mixed_precision, recompute=self._recompute)
        return self._engine

    @property
    def recompute(self):
        """whether training steps recompute activations (DESIGN.md §3.12); setting it re-allocates the engine's training
        activations"""
        return self._recompute

    @recompute.setter
    def recompute(self, on):
        self._recompute = bool(on)
        if self._engine is not None:
            self._engine.set_recompute(on)

    def param_shapes(self):
        return build_param_specs(self.config).shapes()

    # ---- reference surface
    def init(self, rng, seq=None):
        """`model.init(rng, seq)` (train.py:130-131).  `rng` may be an int seed or a key-like array.  Distributions are the
        haiku defaults the reference relies on: Linear w ~ TruncatedNormal(1/sqrt(fan_in)), b = 0; Embed ~
        TruncatedNormal(1); LayerNorm scale = 1; SGU spatial_weights ~ U(+-1e-3/n), spatial_biases = 1 (progen.py:172-176)."""
        g = np.random.default_rng(_seed(rng))
        n = self.config['seq_len']
        out = {}
        for module, names in self.param_shapes().items():
            out[module] = {}
            for name, shape in names.items():
                if name == 'embeddings':
                    a = _trunc_normal(g, shape, 1.0)
                elif name == 'w':
                    a = _trunc_normal(g, shape, shape[0] ** -0.5)
                elif name == 'spatial_weights':
                    a = g.uniform(-1e-3 / n, 1e-3 / n, shape).astype(np.float32)
                elif name in ('scale', 'spatial_biases'):
                    a = np.ones(shape, np.float32)
                else:
                    a = np.zeros(shape, np.float32)
                out[module][name] = a
        return out

    def _ensure_loaded(self, params):
        self.engine.lora = None                  # every path but the adapted training step runs the plain model
        if self._loaded is not params:
            self.engine.load_params(params)
            self._loaded = params

    def apply(self, params, rng, seq):
        """`model.apply(params, rng, seq)`; `rng` is accepted and unused (no dropout — SURVEY Q11).
        seq: (n,) or (B, n) integers -> fp32 logits (n, V) or (B, n, V) as a torch CUDA tensor."""
        seq_t = torch.as_tensor(np.asarray(seq).astype(np.int64) if not isinstance(seq, torch.Tensor) else seq)
        single = seq_t.dim() == 1
        ids = seq_t.reshape(1, -1) if single else seq_t
        if ids.shape[-1] != self.config['seq_len']:
            raise L.ProgenError(f"sequence length {ids.shape[-1]} != constructor seq_len {self.config['seq_len']}")  # Q12
        self._ensure_loaded(params)
        logits = self.engine.forward(ids).view(ids.shape[0], ids.shape[1], -1)
        return logits[0].clone() if single else logits.clone()

    __call__ = apply

    def loss_and_grad(self, params, data, *, adapters=None, lora_alpha=None):
        """Fused `loss, grads = value_and_grad(batched_loss_fn)(params, key, data)` (utils.py:61-76).
        data: (B, n+1) integers.  Returns (python float loss, haiku-shaped dict of numpy fp32 gradients).
        With `adapters` (a tree of `init_adapters`' shape; lora_alpha default: its rank) the loss is the adapted
        model's, the base is frozen, and the gradients are the adapters' (a tree of the same shape)."""
        self._ensure_loaded(params)
        lo = None if adapters is None else self._attach_adapters(adapters, lora_alpha)
        loss = self.engine.loss_and_grad(data)
        return float(loss.item()), self.engine.export_grads() if lo is None else lo.layout.unpack(lo.grads)

    # ---- low-rank adapters (DESIGN.md §3.8)
    def init_adapters(self, rng, rank, *, alpha=None):
        """Initial low-rank adapters {module: {'lora_a': A [in, r], 'lora_b': B [r, out]}} on the QKV, attention output,
        feed-forward in and feed-forward out projections of every layer (gMLP layers included): A ~
        TruncatedNormal(1/sqrt(in)) from `rng` (an int seed or key-like array, as in `init`), B = 0, so the adapted model
        starts as the base model.  rank: an integer multiple of 8 in [8, 64]; alpha (finite, > 0; default rank) is only
        checked here: pass it as lora_alpha wherever the adapters are used, s = alpha / rank."""
        from .lora import check_rank_alpha, init_adapters
        rank, _ = check_rank_alpha(rank, alpha)
        return init_adapters(self.config, _seed(rng), rank)

    def merge_adapters(self, params, adapters, *, lora_alpha=None):
        """params with every adapted weight W replaced by W + s A B (s = lora_alpha / rank, default 1), computed on the
        host in float64 and cast to float32.  `apply`, `score`, `generate` and the other inference paths run on it."""
        from .lora import check_adapters, check_rank_alpha, merge_adapters
        rank, alpha = check_rank_alpha(check_adapters(self.config, adapters), lora_alpha)
        return merge_adapters(params, adapters, alpha / rank)

    def _attach_adapters(self, adapters, lora_alpha, head=None):
        """validate `adapters` and make them (with a checked property `head`: and it) the engine's training-set adapters
        -> lora.Adapters"""
        from .lora import HEAD, Adapters, check_adapters, check_rank_alpha
        rank, alpha = check_rank_alpha(check_adapters(self.config, adapters), lora_alpha)
        C = 0 if head is None else int(np.asarray(head[HEAD]['b']).shape[0])
        eng = self.engine
        lo = getattr(self, '_adapters', None)
        if lo is None or lo.r != rank or lo.alpha != alpha or lo.head_outputs != C:
            lo = self._adapters = Adapters(eng, rank, alpha, head_outputs=C)
        lo.load(adapters, head)
        eng.lora = lo
        return lo

    def preference_loss_and_grad(self, params, chosen, rejected, ref_chosen, ref_rejected, *, beta=0.1):
        """The preference (DPO, Rafailov et al. 2023) twin of `loss_and_grad`.  Pair i is (chosen[i], rejected[i]), each a
        (P, n+1) integer row of the `collate` / `loss_and_grad` contract; ref_chosen / ref_rejected [P] are the rows'
        log-likelihoods under the frozen reference parameters, as `score` returns them.  With s(x) the policy's
        log-likelihood (what `score` reports, bitwise), z_i = beta * ((s(c_i) - ref_c_i) - (s(r_i) - ref_r_i)) and
        loss = mean_i softplus(-z_i).  Inputs are checked before any device work (ProgenError).
        Returns (python float loss, haiku-shaped dict of numpy fp32 gradients, stats), stats a dict of float32 [P] arrays:
        policy_chosen, policy_rejected (s), margin (z) and loss (each pair's)."""
        from .preference import check_pairs
        rows, ref, beta, _ = check_pairs(chosen, rejected, ref_chosen, ref_rejected, beta, None, self.config['seq_len'])
        self._ensure_loaded(params)
        eng = self.engine
        n = eng.row_length(rows)                        # one cut length over all 2P rows (DESIGN.md §3.10)
        P = eng.load_preference(rows, ref, n)
        eng.train_step(('preference', beta), P, length=n)
        return float(eng.loss.item()), eng.export_grads(), eng.preference_stats(P)

    def distill_loss_and_grad(self, params, data, *, teacher, teacher_params, temperature=2.0, alpha=0.5, adapters=None,
                              lora_alpha=None):
        """Loss and gradients of distilling `teacher` (another ProGen with the same vocabulary and a seq_len at least
        this model's, run on `teacher_params`) into this model (DESIGN.md §3.13).  data: (B, n+1) integer rows of the
        `collate` contract.  Per counted position t (the loss mask of `loss_and_grad`), with s this model's logits and z
        the teacher's: KL_t = KL(softmax(z / tau) || softmax(s / tau)) and CE_t = -log_softmax(s)[label_t]; per row, KL_b
        and CE_b their means over the counted positions; loss = mean_b [(1 - alpha) tau^2 KL_b + alpha CE_b], tau =
        `temperature` (finite, > 0), alpha in [0, 1].  alpha = 1 is the `loss_and_grad` loss.  The teacher's forward runs
        in the same step, on its inference set; it keeps no gradient or training state.  With `adapters` (lora_alpha as
        in `loss_and_grad`) the student's base is frozen.  Inputs are checked before any device work (ProgenError).
        Returns (python float loss, gradients (the adapters' with adapters), stats), stats a dict of float32 [B] arrays
        kl and ce (each row's KL_b and CE_b)."""
        from .distill import check_objective, check_teacher
        check_teacher(self, teacher, 'distill_loss_and_grad')
        tau, alpha = check_objective(temperature, alpha, 'distill_loss_and_grad')
        self._ensure_loaded(params)
        lo = None if adapters is None else self._attach_adapters(adapters, lora_alpha)
        teacher._ensure_loaded(teacher_params)
        eng = self.engine
        eng.attach_teacher(teacher.engine)
        n = eng.row_length(data, what='distill_loss_and_grad')
        B = eng.load_distill(data, n)
        eng.train_step(('distill', tau, alpha), B, length=n)
        grads = eng.export_grads() if lo is None else lo.layout.unpack(lo.grads)
        return float(eng.loss.item()), grads, eng.distill_stats(B)

    def policy_loss_and_grad(self, params, samples_or_rows, advantages, *, reference=None, reference_params=None,
                             beta=0.04, span=None, adapters=None, lora_alpha=None):
        """Loss and gradients of one group-relative policy-gradient step (GRPO / RLOO style) with an exact KL to a frozen
        reference (DESIGN.md §3.14).  samples_or_rows: `generate`'s dict (rows and spans by `policy.samples_to_rows`), or
        (B, n+1) integer rows of the `collate` contract with `span` (B, 2) giving each row's label positions lo <= t < hi.
        advantages [B]: one float per row (e.g. `policy.group_advantages` of rewards).  Per position t of row b's span,
        with pi = softmax of this model's logits and rho the reference's: logp_t = log pi[label_t] and KL_t = KL(pi || rho)
        exactly (a sum over the vocabulary); L_b = mean over the span of (-A_b logp_t + beta KL_t); loss = mean_b L_b.
        With beta > 0 `reference` (another ProGen, checked as a distillation teacher; with adapters normally a model on
        the base params) runs its forward on `reference_params` in the same step; with beta = 0 it is not needed.  With
        `adapters` (lora_alpha as in `loss_and_grad`) the base is frozen.  Inputs are checked before any device work
        (ProgenError naming the row).  Returns (python float loss, gradients (the adapters' with adapters), stats), stats
        a dict of [B] arrays: logp and kl (each row's span means, float32) and count (its span length, int64)."""
        from .distill import check_teacher
        from .policy import check_policy_batch, samples_to_rows
        what = 'policy_loss_and_grad'
        if isinstance(samples_or_rows, dict):
            if span is not None:
                raise L.ProgenError(f'{what}: samples carry their spans; pass span= only with rows')
            rows, span = samples_to_rows(samples_or_rows)
        else:
            rows = samples_or_rows
            if span is None:
                raise L.ProgenError(f'{what}: rows need span= (the label positions each row is trained on)')
        rows, span, adv, beta, B = check_policy_batch(rows, span, advantages, beta, None, self.config['seq_len'], what)
        if beta > 0:
            check_teacher(self, reference, what)
            if reference_params is None:
                raise L.ProgenError(f'{what}: a reference needs reference_params')
        self._ensure_loaded(params)
        lo = None if adapters is None else self._attach_adapters(adapters, lora_alpha)
        eng = self.engine
        if beta > 0:
            reference._ensure_loaded(reference_params)
            eng.attach_teacher(reference.engine)
        n = eng.row_length(rows, what=what)
        eng.load_policy(rows, span, adv, n, reference=beta > 0)
        eng.train_step(('policy', beta), B, length=n)
        grads = eng.export_grads() if lo is None else lo.layout.unpack(lo.grads)
        return float(eng.loss.item()), grads, eng.policy_stats(B)

    def score(self, params, data, *, batch_size=64, return_tokens=False, return_embeddings=False):
        """Log-likelihood of sequences under the model, without keeping any training state.
        data: (B, n+1) integer rows, the contract of `loss_and_grad` and `data.collate`: ids = data[:, :-1] are fed to the
        model, labels = data[:, 1:] are scored.  A label counts when it is not pad, plus the first pad (the end of the
        sequence, quirk Q8: utils.py:54-56), so for a sequence of L residues the positions 0..L count.  Labels outside
        [0, num_tokens) are clamped, as in the training loss.

        Returns a dict of numpy arrays:
          log_likelihood [B] float32: sum over the counted positions of log softmax(logits)[label];
          num_tokens [B] int64: number of counted positions;
          token_logp [B, n] float32 and token_mask [B, n] bool (with return_tokens): per-position log-probability (0 where
            not counted) and the mask;
          embedding [B, d] float32 (with return_embeddings): mean over the counted positions of the final-LayerNorm output,
            the input of the logits head.
        Per row, -log_likelihood / num_tokens is exactly the reference's `cross_entropy` (utils.py:45-59), the quantity
        whose batch mean is the training loss.  `batch_size` rows run per forward pass; results do not depend on it."""
        rows = torch.as_tensor(np.asarray(data).astype(np.int64) if not isinstance(data, torch.Tensor) else data)
        if rows.dim() != 2 or rows.shape[-1] != self.config['seq_len'] + 1:
            raise L.ProgenError(f"score: rows must be (B, seq_len + 1 = {self.config['seq_len'] + 1}), got {tuple(rows.shape)}")  # Q12
        self._ensure_loaded(params)
        out = self.engine.score(rows, batch_size=batch_size, tokens=return_tokens, embeddings=return_embeddings)
        if return_tokens:
            labels = rows[:, 1:].cpu().numpy()
            pad = labels == 0
            out['token_mask'] = ~pad | ((np.cumsum(pad, axis=-1) == 1) & pad)
        return out

    def score_variants(self, params, wild_type, mutations, *, prefix='', batch_size=64, return_tokens=False):
        """Zero-shot variant effects: log p(variant) - log p(wild type) under the model, for each mutation set.

        wild_type: residue string.  prefix: optional prompt / tag string placed before the residues (e.g.
        '[Tax=Mammalia] #').  Each row is `data.collate([prefix + residues], seq_len)`, exactly what `score` receives.
        mutations: non-empty list of ProteinGym-style sets, 'A23G', 'A23G:K45R', or '' for the wild type; positions are
        1-based over the residues (not the prefix).  Rejected with ProgenError naming the set: a wild-type letter that does
        not match, a position out of range or cut off by seq_len, the same position twice in one set, a new letter that
        is not one printable ASCII character.  Identity substitutions (A23A) are allowed.

        The wild type and every variant run through the scoring forward cut to L = min(seq_len, counted length rounded up
        to 128) positions: every mixing op is causal, so positions < L depend on ids < L only, and the cut forward
        computes them bitwise as the full-length one does (DESIGN.md §3.6).  The wild type is scored once per call.

        Returns a dict:
          delta [M] float64: sum over positions of (variant - wild type) token log-probabilities, in float64, so
            identical positions cancel exactly (0.0 for '' and for identity substitutions);
          log_likelihood [M] float32 and num_tokens [M] int64: as `score` reports them for the variant rows;
          wt_log_likelihood (float32): `score`'s log-likelihood of the wild-type row;
          token_logp [M, seq_len] float32 (with return_tokens): as `score` reports it (zero beyond L).
        Rows run batch_size at a time; results do not depend on batch_size or on the other sets in the call."""
        from .engine import cut_length
        from .variants import parse_mutations, variant_rows
        n = self.config['seq_len']
        subs = parse_mutations(wild_type, mutations, n, prefix)
        batch_size = _batch_size(batch_size, 'score_variants')
        rows = variant_rows(wild_type, subs, n, prefix)
        length = cut_length(rows[:, 1:])
        self._ensure_loaded(params)
        sc = self.engine.score(rows, batch_size=batch_size, tokens=True, length=length)
        lp = sc['token_logp'][:, :length].astype(np.float64)
        out = dict(delta=(lp[1:] - lp[0]).sum(axis=-1), log_likelihood=sc['log_likelihood'][1:],
                   num_tokens=sc['num_tokens'][1:], wt_log_likelihood=sc['log_likelihood'][0])
        if return_tokens:
            out['token_logp'] = sc['token_logp'][1:]
        return out

    def mutational_scan(self, params, wild_type, *, positions=None, alphabet='ACDEFGHIKLMNPQRSTVWY', prefix='', batch_size=64):
        """Deep mutational scan: every single substitution at `positions` (1-based, default every residue) to each letter
        of `alphabet`, scored by `score_variants` in one call.  Returns a dict: delta [P, |alphabet|] float64 (0.0 at
        the wild-type letter, which is not run), positions [P] int64, alphabet, wt_log_likelihood."""
        from .variants import check_scan, scan_sets
        pos = check_scan(wild_type, positions, alphabet)
        sets, index = scan_sets(wild_type, pos, alphabet)
        delta = np.zeros(index.shape, np.float64)
        if sets:
            res = self.score_variants(params, wild_type, sets, prefix=prefix, batch_size=batch_size)
            delta[index >= 0] = res['delta'][index[index >= 0]]
            wt = res['wt_log_likelihood']
        else:                          # an alphabet of the wild-type letter alone: nothing to run but the wild type
            wt = self.score_variants(params, wild_type, [''], prefix=prefix, batch_size=batch_size)['wt_log_likelihood']
        return dict(delta=delta, positions=pos, alphabet=alphabet, wt_log_likelihood=wt)

    def generate(self, params, prompts, *, num_samples=1, temperature=1.0, top_k=None, top_p=None, max_length=None, seed=0,
                 batch_size=64, logit_bias=None, min_new_tokens=0, repetition_penalty=1.0, repetition_window=0,
                 prefill='decode', position_bias=None, fixed=None, require=None, avoid=None):
        """Sample sequences with the standard sampler of the persistent decode kernel (temperature, top-k with ties kept,
        nucleus top-p, in-kernel Philox Gumbel noise; csrc/decode_persist.cu), stopping each sequence at its EOS.
        Unlike the reference sampler (utils.sample, sample.py), a prompt is laid out as training data is: BOS (0), the
        prompt, then the generated residues; an empty prompt draws its first residue from the BOS logits.

        prompts: a string, or a list of strings (encoded like training text) or of integer id arrays (ids in [1, V)).
        Rows are prompt-major: row i * num_samples + j is sample j of prompt i and draws from Philox stream (seed, row).
        Rows run min(batch_size, N) (<= 64) at a time in one persistent kernel.  With prefill='decode' and at least two
        rows per launch, the rows form a queue (up to QUEUE_ROWS_PER_SLOT per slot and launch): a row that ends hands its
        slot to the next row, so a launch does not wait for its longest row.  The kernel's arithmetic depends on the
        class of the launch size, 1, 2-8 or 9-64 rows, and on the GPU's SM count, but not on the size within the class,
        the slot or the other rows: on one GPU model a row is bitwise the same for every batch_size of the same class and
        every chunking (with forward prefill a ragged last chunk is padded to the class).  Rows of different classes agree
        to fp32 round-off, so ids can differ where a draw is that close.  max_length (default seq_len) bounds BOS + prompt
        + generated tokens;
        temperature 0 is greedy (first maximal logit; top_k / top_p ignored), and so is a positive temperature so small
        that the largest logit divided by it overflows float32 (e.g. 1e-39).

        Constraints, applied in the kernel to the logits of every draw, in this order, before top-k / temperature / top-p
        (DESIGN.md §3.3):
          repetition_penalty θ (finite, > 0; 1 = off) and repetition_window W (integer in [0, seq_len]; 0 = the whole
            row): each id present at least once among the last W positions before the draw (prompt and generated, BOS
            excluded) has its logit l divided by θ if l > 0, else multiplied by θ;
          logit_bias: None or V floats added to the logits; -inf bans an id, +inf and NaN are rejected, and some id in
            [1, V) must stay allowed (EOS, id 0, may be banned);
          min_new_tokens (integer in [0, max_length - 2]): the first min_new_tokens generated tokens of a row are never
            EOS.  A row whose prompt leaves fewer positions before max_length simply runs to max_length unfinished.
          position_bias (after logit_bias, before the min_new_tokens EOS ban): None, a float array [T, V] (1 <= T <=
            seq_len) for every prompt, or a list with one array or None per prompt.  Row j is added to the logits of
            generated token j + 1, whatever the prompt's length; -inf bans an id at that offset; offsets past T are
            unconstrained.
          fixed: None, a dict {k: residue} for every prompt, or a list with one dict or None per prompt: generated token k
            (1-based, at position start + k - 1) is `residue`, one character encoded like training text or an id in
            [1, V).  It becomes position-bias rows (`position_tables`): 0 at the id and -inf elsewhere at offset k, and
            -inf on EOS at every earlier offset, so no row ends before its last fixed residue; added to the prompt's
            position_bias.  Offsets a prompt cannot reach before max_length, residues outside the vocabulary, and any
            reachable offset left with no candidate (say a fixed residue banned by logit_bias) raise ProgenError naming
            the prompt and the offset; an offset that allows only EOS ends the row there.
          require / avoid (after every adjustment above): None or one PROSITE pattern that a row's generated tokens
            t_1..t_L (before EOS, or up to max_length) must contain, and None, one pattern or a list of at most 8 that
            they must not contain; the same for every prompt, the prompt not matched (`motif.Pattern`: elements
            separated by '-', a letter, x, [..] or {..} with an optional (n) or (n,m) repeat, '<' / '>' anchor at t_1 /
            t_L, at most 64 positions).  A residue is drawn only if the required pattern can still be completed before
            max_length, EOS only once it is met, and no residue or EOS that completes an avoided pattern (a '>'-anchored
            one: at the row's end).  A row whose other constraints leave no candidate ends with EOS unmet.  Refused
            before anything runs: a malformed pattern, a mandatory position of the required one that logit_bias bans
            entirely, and a prompt that leaves fewer positions than its shortest match.
        Only the ids whose adjusted logit is not -inf can be drawn.  token_logp and log_likelihood do not see the
        constraints: they stay the unfiltered model's at temperature 1, comparable with `score`.  With position tables a
        row's bits depend only on (seed, row), its prompt, its table and the launch class, not on the other rows' tables
        or on how the rows are split into launches (QUEUE_TABLE_BYTES bounds the tables of one launch).

        prefill: how the positions before the first draw (BOS and the prompt but its last id) reach the decoder's caches.
          'decode' (default): the decode kernel consumes them one position at a time, as it does generated positions.
          'forward': one inference forward (the engine that `score` runs) over the distinct prompts of a launch fills the
            caches, and the decode kernel starts at the last prompt id.  Faster for long prompts and for many samples of
            one prompt; the caches carry the forward's arithmetic, so with mixed_precision (bf16 activations in the
            forward, fp32 in the decoder) the results differ from 'decode' by round-off.  A launch then holds rows of one
            prompt length only, so a row's result still depends only on (seed, row), the prompt and the launch class.
          An empty prompt has nothing to prefill: both modes are the same there.

        Returns a dict of numpy arrays over the N = len(prompts) * num_samples rows:
          tokens [N, seq_len] int64: BOS, prompt, generated tokens, EOS, zeros;
          start [N] int64: position of the first generated token (1 + prompt length);
          length [N] int64: generated tokens, EOS included;
          finished [N] bool: an EOS was drawn before max_length;
          log_likelihood [N] float64: sum of token_logp over the generated positions;
          token_logp [N, seq_len] float32: log p(tokens[t] | tokens[:t]) under the unfiltered model (temperature 1) at
            generated t, 0 elsewhere — the quantity `score` reports;
          prompt_index [N] int64;
          motif_match [N] bool (with require or avoid): the row's generated tokens contain the required pattern and
            none of the avoided ones, replayed on the host."""
        return self._generate(lambda batch: self._generate_decoder(params, batch), params, prompts,
                              num_samples=num_samples, temperature=temperature, top_k=top_k, top_p=top_p,
                              max_length=max_length, seed=seed, batch_size=batch_size, logit_bias=logit_bias,
                              min_new_tokens=min_new_tokens, repetition_penalty=repetition_penalty,
                              repetition_window=repetition_window, prefill=prefill, position_bias=position_bias,
                              fixed=fixed, require=require, avoid=avoid)

    def _generate(self, decoder, params, prompts, *, num_samples=1, temperature=1.0, top_k=None, top_p=None,
                  max_length=None, seed=0, batch_size=64, logit_bias=None, min_new_tokens=0, repetition_penalty=1.0,
                  repetition_window=0, prefill='decode', position_bias=None, fixed=None, require=None, avoid=None):
        """`generate` on the BatchDecoder `decoder(rows per launch)` returns (`Trainer.generate`: the trainer's own);
        `params` are what forward prefill runs on"""
        from .data import encode_tokens
        from .decode import Sampling, integer, prompt_ids
        cfg = self.config
        V, n = cfg['num_tokens'], cfg['seq_len']
        if not isinstance(prefill, str) or prefill not in ('decode', 'forward'):
            raise L.ProgenError(f"generate: prefill must be 'decode' or 'forward', got {prefill!r}")
        max_length = n if max_length is None else integer(max_length, 'max_length', 2, n)
        num_samples = integer(num_samples, 'num_samples', 1, 1 << 40)
        batch_size = integer(batch_size, 'batch_size', 1, 64)
        sampling = Sampling.check(V, n, max_length - 2, True, temperature=temperature, top_k=top_k, top_p=top_p, seed=seed,
                                  logit_bias=logit_bias, min_new_tokens=min_new_tokens,
                                  repetition_penalty=repetition_penalty, repetition_window=repetition_window)
        if isinstance(prompts, (str, bytes)):
            prompts = [prompts]
        if not isinstance(prompts, (list, tuple)) or len(prompts) == 0:
            raise L.ProgenError('generate: prompts must be a string or a non-empty list of strings or id arrays')
        ids = prompt_ids([encode_tokens(p.decode() if isinstance(p, bytes) else p) if isinstance(p, (str, bytes)) else p
                          for p in prompts], V, max_length)
        tables, prompt_table = position_tables([1 + len(a) for a in ids], V, n, max_length, position_bias, fixed,
                                               sampling.logit_bias, sampling.min_new_tokens)
        motif = None
        if require is not None or avoid is not None:
            from .motif import Motif
            motif = Motif(require, avoid, V, sampling.logit_bias)
            motif.check_reach([1 + len(a) for a in ids], max_length)
        N = len(ids) * num_samples
        rows = [ids[r // num_samples] for r in range(N)]
        row_table = prompt_table[np.arange(N) // num_samples]
        dec = decoder(min(batch_size, N))
        if prefill == 'forward':
            self._ensure_loaded(params)
        out = dict(tokens=np.zeros((N, n), np.int64), start=np.zeros(N, np.int64), end=np.zeros(N, np.int64),
                   token_logp=np.zeros((N, n), np.float32))
        table_bytes = max((t.nbytes for t in tables), default=0)
        for sids, real, slots in plan_generate([len(a) for a in rows], batch_size, prefill, row_table, table_bytes):
            chunk = [rows[r] for r in sids]
            P = dec.prefill(self.engine, chunk) if prefill == 'forward' else 0
            res = dec._generate(chunk, sampling, sids, max_length, launch_tables(tables, row_table, sids), prefilled=P,
                                slots=slots, motif=motif)
            for k, key in (('tokens', 'ids'), ('token_logp', 'token_logp'), ('start', 'start'), ('end', 'end')):
                out[k][sids[:real]] = res[key][:real]
        end = out.pop('end')
        out['finished'] = end < max_length
        out['length'] = np.where(out['finished'], end + 1, max_length) - out['start']
        out['log_likelihood'] = out['token_logp'].astype(np.float64).sum(axis=-1)
        out['prompt_index'] = np.arange(N, dtype=np.int64) // num_samples
        if motif is not None:
            gen = out['length'] - out['finished']
            out['motif_match'] = motif.matches([out['tokens'][i, s:s + g] for i, (s, g) in enumerate(zip(out['start'], gen))])
        return out

    def _generate_decoder(self, params, batch):
        """The BatchDecoder of `generate`, kept across calls with the same parameters (like `_ensure_loaded`); rebuilt when
        a call needs more rows per launch than it holds."""
        import torch
        from .decode import BatchDecoder
        dec = self._gen_decoder
        if dec is None or self._gen_params is not params or dec.B < batch:
            self._gen_decoder = None
            dec = BatchDecoder(self.config, params, batch=batch,
                               weights_dtype=torch.bfloat16 if self.mixed_precision else torch.float32)
            self._gen_decoder, self._gen_params = dec, params
        return dec

    def trainer(self, params, *, adapters=None, lora_alpha=None, head=None, task=None, teacher=None, teacher_params=None,
                reference=None, reference_params=None, **optim_kwargs):
        """Device-resident training state over `params` (train.py's loop).  With `adapters` only the adapters train
        (the base stays bitwise unchanged); lora_alpha as in `loss_and_grad`.  With a property `head` (`init_head`) and
        its `task` ('regression' | 'classification') the adapters and the head train together through
        `Trainer.property_step` (per-sequence labels) or `Trainer.residue_step` (per-residue labels).  With a `teacher`
        (another ProGen, as in `distill_loss_and_grad`) and its `teacher_params`, `Trainer.distill_step` distils it into
        this model.  With a `reference` (another ProGen, as in `policy_loss_and_grad`) and its `reference_params`,
        `Trainer.policy_step` takes policy-gradient steps with a KL to it; `Trainer.generate` samples from the weights
        being trained."""
        from .trainer import Trainer
        return Trainer(self, params, adapters=adapters, lora_alpha=lora_alpha, head=head, task=task, teacher=teacher,
                       teacher_params=teacher_params, reference=reference, reference_params=reference_params,
                       **optim_kwargs)

    # ---- property fine-tuning (DESIGN.md §3.9)
    def init_head(self, rng, num_outputs):
        """An initial property head {'property_head': {'w': [dim, C], 'b': [C]}} on the pooled embedding: w ~
        TruncatedNormal(1/sqrt(dim)) from `rng` (an int seed or key-like array, as in `init`), b = 0.  num_outputs C in
        [1, 64]: the regression outputs, or the classes (>= 2) of a classification head."""
        from .property import init_head
        return init_head(self.config['dim'], _seed(rng), num_outputs)

    def property_loss_and_grad(self, params, rows, targets, *, adapters, head, task, lora_alpha=None):
        """Loss and gradients of property fine-tuning: the head on the pooled embedding of the adapted model (the
        embedding `score(..., return_embeddings=True)` returns: the mean of the final LayerNorm output over the counted
        positions).  rows: (B, n+1) integer rows of the `collate` contract; task 'regression' (targets float [B, C]; loss
        = sum_b sum_c (p - y)^2 / (C B)) or 'classification' (targets class indices [B]; loss = mean cross entropy).
        The base is frozen.  Inputs are checked before any device work (ProgenError).
        Returns (python float loss, adapter gradients, head gradients, predictions [B, C] numpy float32: the regression
        values or the class logits)."""
        from .lora import check_adapters, check_rank_alpha
        from .property import check_head, check_rows, check_targets, check_task
        code = check_task(task)
        C = check_head(self.config, head, task)
        check_rank_alpha(check_adapters(self.config, adapters), lora_alpha)
        r = check_rows(rows, self.config['seq_len'], 'property_loss_and_grad')
        if r.shape[0] < 1:
            raise L.ProgenError('property_loss_and_grad: needs at least one row')
        y = check_targets(targets, task, C, r.shape[0], 'property_loss_and_grad')
        self._ensure_loaded(params)
        lo = self._attach_adapters(adapters, lora_alpha, head)
        eng = self.engine
        n = eng.row_length(r)
        B = eng.load_property(r, code, y, n)
        eng.train_step(('property', code), B, length=n)
        grads, hgrads = lo.split(lo.layout.unpack(lo.grads))
        return float(eng.loss.item()), grads, hgrads, eng.property_stats(B)['prediction']

    def predict(self, params, head, data, *, batch_size=64):
        """Property predictions of sequences: the head on the pooled embedding, on the inference forward (like `score`;
        pass merged parameters for a fine-tuned model: `merge_adapters`, `checkpoint.package_params`).  data: (N, n+1)
        integer rows of the `collate` contract.  The forward is cut to the rows' counted length rounded up to 128
        (`engine.cut_length`): the embedding reads counted positions only, so it is bitwise the full-length one.
        Returns a dict of numpy float32 arrays: prediction [N, C] (regression values, or class logits) and embedding
        [N, d] (bitwise `score(..., return_embeddings=True)['embedding']`).  Results do not depend on batch_size."""
        from .lora import HEAD
        from .property import check_head, check_rows
        check_head(self.config, head)
        batch_size = _batch_size(batch_size, 'predict')
        r = check_rows(data, self.config['seq_len'], 'predict')
        self._ensure_loaded(params)
        pred, emb = self.engine.predict(r, head[HEAD]['w'], head[HEAD]['b'], batch_size=batch_size)
        return dict(prediction=pred, embedding=emb)

    # ---- per-residue fine-tuning (DESIGN.md §3.11)
    def residue_loss_and_grad(self, params, rows, targets, *, adapters, head, task, lora_alpha=None):
        """Loss and gradients of per-residue fine-tuning: the property head (`init_head`) applied at every position to
        the adapted model's final LayerNorm output h[b, t], p[b, t] = h[b, t] W + b.  rows: (B, n+1) integer rows of the
        `collate` contract; the input at position t >= 1 is residue t - 1, so targets are indexed by position:
        regression float [B, n, C] (or [B, n] when C == 1; NaN in every output marks an unlabelled position), loss =
        sum over labelled (b, t) of sum_c (p - y)^2 / (C N); classification class indices [B, n] (-1: unlabelled), loss
        = the mean cross entropy over the N labelled positions.  Position 0 (BOS) and pad inputs hold no residue and
        must stay unlabelled.  ProGen is causal: h[b, t] has seen residues 0..t-1 only, so labels that depend on
        downstream context are harder for it than for a bidirectional model.  The base is frozen.  Inputs are checked
        before any device work (ProgenError names the first offending (row, position)).
        Returns (python float loss, adapter gradients, head gradients, predictions [B, n, C] numpy float32: the
        regression values or the class logits at every position, zero beyond the step's row length)."""
        from .lora import check_adapters, check_rank_alpha
        from .property import check_head, check_residue_targets, check_rows, check_task, residue_length
        code = check_task(task)
        C = check_head(self.config, head, task)
        check_rank_alpha(check_adapters(self.config, adapters), lora_alpha)
        r = check_rows(rows, self.config['seq_len'], 'residue_loss_and_grad')
        if r.shape[0] < 1:
            raise L.ProgenError('residue_loss_and_grad: needs at least one row')
        y, labelled = check_residue_targets(r, targets, task, C, 'residue_loss_and_grad')
        n = residue_length(r, labelled, None, 'residue_loss_and_grad')
        self._ensure_loaded(params)
        lo = self._attach_adapters(adapters, lora_alpha, head)
        eng = self.engine
        B = eng.load_residue(r, code, y, n)
        eng.train_step(('residue', code), B, length=n)
        grads, hgrads = lo.split(lo.layout.unpack(lo.grads))
        return float(eng.loss.item()), grads, hgrads, eng.residue_stats(B)['prediction']

    def predict_residues(self, params, head, data, *, batch_size=64):
        """Per-residue predictions: the head at every position of the inference forward (pass merged parameters for a
        fine-tuned model, as for `predict`).  data: (N, n+1) integer rows of the `collate` contract.  The forward is cut
        to the rows' counted length rounded up to 128.  Returns a dict: prediction [N, n, C] float32 (regression values,
        or class logits; 0 where no residue is) and mask [N, n] bool, the positions that hold residues (position t holds
        residue t - 1).  A position's prediction depends on its own row only: results do not depend on batch_size."""
        from .lora import HEAD
        from .property import check_head, check_rows, residue_length, residue_positions
        check_head(self.config, head)
        batch_size = _batch_size(batch_size, 'predict_residues')
        r = check_rows(data, self.config['seq_len'], 'predict_residues')
        mask = residue_positions(r)
        length = residue_length(r, mask, None, 'predict_residues')
        self._ensure_loaded(params)
        pred = self.engine.predict_residues(r, head[HEAD]['w'], head[HEAD]['b'], length, batch_size=batch_size)
        pred[~mask] = 0.0
        return dict(prediction=pred, mask=mask)
