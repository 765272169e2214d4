"""Device-resident training state for the train.py loop: parameters, gradients, Adam moments and the apply_every
accumulator live in flat fp32 buffers; one `step(data)` is one iteration of the reference's inner loop
(train.py:186-190): loss+grads, optim.update, apply_updates.

With low-rank adapters (`adapters=`) the same state exists for the adapter buffer only: the base parameters are frozen
and bitwise unchanged, and clip / AdamW / apply_every run over the adapters (weight decay on every A and B).  A property
head (`head=`, `task=`) joins that buffer: `property_step` trains adapters and head together on per-sequence labels
(DESIGN.md §3.9), `residue_step` on per-residue labels (§3.11).  With a frozen `reference=` model `policy_step` takes
policy-gradient steps on the model's own samples (§3.14), which `generate` draws from the weights being trained."""
import weakref

import torch

from . import lib as L
from . import parallel as PAR


class Trainer:
    overlap = False         # exists only because bench.py reads it: the gradient exchange is never overlapped

    def __init__(self, model, params, learning_rate=2e-4, weight_decay=1e-3, max_grad_norm=0.5, grad_accum_every=4,
                 b1=0.9, b2=0.999, eps=1e-8, optim_state=None, data_parallel=True, cuda_graph=False, adapters=None,
                 lora_alpha=None, head=None, task=None, teacher=None, teacher_params=None, reference=None,
                 reference_params=None):
        self.model = model
        if (teacher is not None or teacher_params is not None) and (reference is not None or reference_params is not None):
            raise L.ProgenError('trainer: pass a teacher (distill_step) or a reference (policy_step), not both')
        for other, other_params, name in ((teacher, teacher_params, 'teacher'), (reference, reference_params, 'reference')):
            if other is not None or other_params is not None:
                from .distill import check_teacher
                check_teacher(model, other, 'trainer')
                if other_params is None:
                    raise L.ProgenError(f'trainer: a {name} needs {name}_params')
        self.task = None
        if head is not None or task is not None:
            from .property import check_head, check_task
            if adapters is None:
                raise L.ProgenError('a property head trains with adapters on the frozen base: pass adapters= '
                                    '(full-parameter property fine-tuning is not supported)')
            if head is None or task is None:
                raise L.ProgenError('property fine-tuning needs both head= and task=')
            self.task = check_task(task)
            C = check_head(model.config, head, task)
        self.eng = model.engine
        self.eng.load_params(params)
        model._loaded = None
        # distillation (distill_step) or the policy step's reference: that engine keeps its parameters and inference
        # set only, in the engine's teacher slot
        self.teacher, self.reference = teacher, reference
        for other, other_params in ((teacher, teacher_params), (reference, reference_params)):
            if other is not None:
                other._ensure_loaded(other_params)
                self.eng.attach_teacher(other.engine)
        self._decoder, self._decoder_count = None, None   # generate: one decoder, refreshed after every step
        self.lora = None
        if adapters is not None:
            from .lora import Adapters, check_adapters, check_rank_alpha
            rank, alpha = check_rank_alpha(check_adapters(model.config, adapters), lora_alpha)
            self.lora = Adapters(self.eng, rank, alpha, head_outputs=C if head is not None else 0)
            self.lora.load(adapters, head)
        # the flat buffers the optimizer owns: (their layout, parameters, ndim > 1 prefix, bf16 mirror or None);
        # gradients: self.G
        if self.lora is None:
            e = self.eng
            self.layout, self.P, self.n_decay, self.P_lp = e.layout, e.params, e.n_decay, e.params_lp
        else:
            lo = self.lora
            self.layout, self.P, self.n_decay, self.P_lp = lo.layout, lo.params, lo.layout.size, None
            self.eng.grads = None                  # nothing reads or writes the base gradient while adapters train
        n = self.layout.size
        self.lr, self.wd, self.max_norm, self.every = learning_rate, weight_decay, max_grad_norm, grad_accum_every
        self.b1, self.b2, self.eps = b1, b2, eps
        z = lambda: torch.zeros(n, device=self.eng.dev, dtype=torch.float32)
        self.m, self.v, self.acc = z(), z(), z()
        self.count = 0                                     # host copy of the Adam count, for optim_state()
        # AdamDevState (count | bc1, bc2 | emit, pad): progen_adamw_step advances it on the device, eager or replayed
        self._adam_state = torch.zeros(4, dtype=torch.int64, device=self.eng.dev)
        self.ws = torch.empty(L.load().progen_optim_workspace_floats(), device=self.eng.dev)
        self.gnorm_sq = torch.zeros(1, device=self.eng.dev)
        self.rank, self.world = PAR.world() if data_parallel else (0, 1)
        # captured steps by (key, row length): the key is (rows, global_rows) + objective; all of them hold for one
        # batch size and one alloc_epoch.  _graph / _graph_key / _graph_length: the most recently installed one.
        self._graphs, self._graph_epoch = {}, 0
        self._installed, self._graph_key, self._graph_length = None, None, None
        # the teacher's inference set at the last capture (a weak reference): a distill step's graph reads it, and
        # inference_acts re-allocates it without advancing alloc_epoch
        self._graph_teacher = None
        # cuda_graph=True: the second eager step of one (key, row length) is captured and replayed from then on
        self._auto_graph, self._eager_runs = bool(cuda_graph), {}
        self.skip_allreduce = False                       # bench.py: "step without the exchange" for comm_exposed_ms
        if optim_state is not None:
            self.load_optim_state(optim_state)

    @property
    def _graph(self):
        """the most recently installed captured step, or None"""
        return self._installed

    @_graph.setter
    def _graph(self, g):
        """`_graph = None` drops every captured step (before the communicator they reference goes away, or to step
        eagerly)"""
        if g is not None:
            raise L.ProgenError('install a captured step with capture_graph')
        self._graphs, self._eager_runs = {}, {}
        self._installed, self._graph_key, self._graph_length = None, None, None

    @property
    def G(self):
        """the flat gradient the optimizer reads: the adapters', or every parameter's"""
        return self.eng.base_grads() if self.lora is None else self.lora.grads

    # ---- one micro-step of train.py:186-190
    def step(self, data, sync_loss=False, global_batch=None, length=None):
        """data: this rank's rows, (b, n+1) integers; `global_batch` = rows of the UNSHARDED batch (utils.py:83-91: the
        masked mean divides by the real row count, so ragged shards — 5 rows over 2 ranks = 3 + 2, or ranks with no rows
        at all — must all scale by 1/5).  Without it the shards are assumed equal.  Returns the device scalar loss
        (global mean when sync_loss).
        `length`: the row length the step runs at (DESIGN.md §3.10).  None: the rows' `engine.cut_length` in a single
        process, seq_len under data parallelism (every rank must run one length: pass the cut_length of the global
        batch); rows on the device run at seq_len.  Otherwise seq_len or a multiple of 128 below it that covers every
        counted position of the rows (ProgenError before any device work)."""
        rows = data.shape[0]
        gb = int(global_batch) if global_batch is not None else rows * self.world
        n = self._length(data, length, 'step')
        return self._step(rows, gb, (), lambda: self.eng.load_batch(data, n), sync_loss, n)

    def step_resident(self, global_batch=None, sync_loss=False):
        """same, on tokens/labels already copied into engine.tok / engine.labels (bench: inputs resident in HBM), at
        seq_len"""
        return self._step(self.eng.B, global_batch or self.eng.B * self.world, (), None, sync_loss, self.eng.n)

    def _length(self, rows, length, what):
        """the row length of a step on `rows` (see `step`)"""
        if length is None and self.world > 1:
            length = self.eng.n
        return self.eng.row_length(rows, length, what)

    def _step(self, rows, global_rows, objective, load, sync_loss, length):
        """One micro-step of `objective` (Engine.train_step) on `rows` rows at row length `length`, then the optimizer
        update.  `load()` makes the rows resident (None: they are); its H2D copies stay outside the graph.  A captured
        graph of (key, length), key = (rows, global_rows) + objective, replays; otherwise the step runs eagerly, and
        with cuda_graph=True the second eager step of one (key, length) is captured for the next one to replay."""
        eng = self.eng
        eng.lora = self.lora
        if rows == 0:
            # a rank without rows (batch smaller than the world): zero contribution, but every collective is joined
            self.G.zero_()
            eng.loss.zero_()
            return self._eager_update(sync_loss)
        key = (rows, global_rows) + objective
        self._drop_graph_unless(rows)
        if load is not None:
            load()
        g = self._graphs.get((key, length))
        if g is not None:
            return self._replay(sync_loss, g)
        eng.train_step(objective, global_rows, length=length)
        loss = self._eager_update(sync_loss)
        if self._auto_graph:
            runs = self._eager_runs[(key, length)] = self._eager_runs.get((key, length), 0) + 1
            if runs >= 2:
                # capture does not execute: eng.loss still holds this step's value
                self.capture_graph(rows, global_rows, objective=objective, length=length)
        return loss

    # ---- CUDA graph of the whole step: forward, loss, backward, (gradient all-reduce), norm, AdamW, masked copies
    def capture_graph(self, batch_rows, global_batch=None, install=True, objective=(), length=None):
        """Capture one training step for batches of `batch_rows` rows into a CUDA graph; later `step` / `step_resident`
        calls with that shape replay it.  The step-dependent optimizer scalars live on the device
        (`progen_adamw_step`), so the graph is identical for every step.  Under data parallelism the NCCL all-reduce
        of the gradient buffer is part of the graph (issued on the capture stream between backward and the norm).  Call
        after at least one eager step of the same shape (kernel attributes, tensor maps, buffers and the NCCL communicator
        must exist before capture).  `install=False` returns the graph without making it the one `step` replays.
        `objective` (Engine.train_step) selects the loss: ('preference', beta) captures the step `preference_step`
        replays, with batch_rows = 2 * pairs and global_batch = the global pair count.  `length` (default seq_len): the
        row length of the captured step; one graph is kept per (key, length), and a step replays the one of its own."""
        gb = global_batch or batch_rows * self.world
        length = self.eng.n if length is None else int(length)
        eng = self.eng
        eng.lora = self.lora
        eng.ensure_batch(batch_rows)
        self._drop_graph_unless(batch_rows)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            eng.train_step(objective, gb, length=length)
            self._allreduce_grads()
            self._update()
        if install:
            key = (batch_rows, gb) + objective
            self._graphs[(key, length)] = g
            self._installed, self._graph_key, self._graph_length, self._graph_epoch = g, key, length, eng.alloc_epoch
            t = eng.teacher
            self._graph_teacher = None if t is None or t.infer is None else weakref.ref(t.infer)
        return g

    # ---- preference (DPO) fine-tuning
    def preference_step(self, chosen, rejected, ref_chosen, ref_rejected, beta=0.1, sync_loss=False, global_pairs=None,
                        length=None):
        """One micro-step of preference (DPO) fine-tuning on this rank's pairs: the loss and gradient of
        `ProGen.preference_loss_and_grad`, then the same clip / AdamW / apply_every update as `step`.  chosen / rejected:
        (P, n+1) integer rows; ref_chosen / ref_rejected [P]: their log-likelihoods under the frozen reference (`score`).
        Data parallel: give each rank `parallel.shard_rows(P_global, rank, world)` of the pairs and global_pairs =
        P_global (default: equal shards, P * world); a rank without pairs contributes zeros but joins the all-reduce.
        With cuda_graph=True the step is captured after two eager steps of one (P, global_pairs, beta) and replayed from
        then on.  Returns the device scalar loss (global mean when sync_loss); `preference_stats()` has the per-pair
        statistics.  `length` as in `step`, over the chosen and rejected rows together."""
        from .preference import check_pairs
        gp = global_pairs
        if gp is None and self.world > 1:
            gp = len(chosen) * self.world
        rows, ref, beta, gp = check_pairs(chosen, rejected, ref_chosen, ref_rejected, beta, gp, self.eng.n,
                                          what='preference_step', allow_empty=True)
        n = self._length(rows, length, 'preference_step')             # one length over all 2P rows
        P = rows.shape[0] // 2
        self._pref_pairs = P
        return self._step(2 * P, gp, ('preference', beta), lambda: self.eng.load_preference(rows, ref, n), sync_loss, n)

    # ---- property fine-tuning (a head on the pooled embedding, adapters on the frozen base)
    def property_step(self, rows, targets, sync_loss=False, length=None):
        """One micro-step of property fine-tuning: the loss and gradients of `ProGen.property_loss_and_grad` over the
        adapters and the head, then one clip / AdamW / apply_every update of both (weight decay on every trained
        parameter).  rows: (B, n+1) integer rows; targets: regression float [B, C], classification class indices [B].
        With cuda_graph=True the step is captured after two eager steps of one batch size and replayed from then on.
        Single process only.  Returns the device scalar loss; `property_stats()` has the predictions and per-row losses.
        `length` as in `step`."""
        from .property import check_rows, check_targets
        if self.task is None:
            raise L.ProgenError('property_step: this trainer has no property head (model.trainer(..., head=, task=))')
        if self.world > 1:
            raise L.ProgenError('property_step: data-parallel property fine-tuning is not supported; run one process '
                                '(data_parallel=False or without torchrun)')
        task = 'regression' if self.task == L.TASK_REGRESSION else 'classification'
        r = check_rows(rows, self.eng.n, 'property_step')
        B = r.shape[0]
        if B < 1:
            raise L.ProgenError('property_step: needs at least one row')
        y = check_targets(targets, task, self.lora.head_outputs, B, 'property_step')
        n = self._length(r, length, 'property_step')
        self._prop_rows = B
        return self._step(B, B, ('property', self.task), lambda: self.eng.load_property(r, self.task, y, n), sync_loss, n)

    # ---- per-residue fine-tuning (the same head at every position, DESIGN.md §3.11)
    def residue_step(self, rows, targets, sync_loss=False, length=None):
        """One micro-step of per-residue fine-tuning: the loss and gradients of `ProGen.residue_loss_and_grad` over the
        adapters and the head, then one clip / AdamW / apply_every update of both.  rows: (B, n+1) integer rows;
        targets per position (`property.check_residue_targets`): regression float [B, n, C] (NaN: unlabelled),
        classification class indices [B, n] (-1: unlabelled).  With cuda_graph=True the step is captured after two eager
        steps of one (batch size, row length) and replayed from then on.  Single process only.  Returns the device scalar
        loss; `residue_stats()` has the predictions and per-position losses.  `length` as in `step`; it must also cover
        every labelled position."""
        from .property import check_residue_targets, check_rows, residue_length
        if self.task is None:
            raise L.ProgenError('residue_step: this trainer has no property head (model.trainer(..., head=, task=))')
        if self.world > 1:
            raise L.ProgenError('residue_step: data-parallel residue fine-tuning is not supported; run one process '
                                '(data_parallel=False or without torchrun)')
        task = 'regression' if self.task == L.TASK_REGRESSION else 'classification'
        r = check_rows(rows, self.eng.n, 'residue_step')
        B = r.shape[0]
        if B < 1:
            raise L.ProgenError('residue_step: needs at least one row')
        y, labelled = check_residue_targets(r, targets, task, self.lora.head_outputs, 'residue_step')
        n = residue_length(r, labelled, length, 'residue_step')
        self._res_rows = B
        return self._step(B, B, ('residue', self.task), lambda: self.eng.load_residue(r, self.task, y, n), sync_loss, n)

    # ---- distillation (a teacher's per-position distribution as the target, DESIGN.md §3.13)
    def distill_step(self, rows, temperature, alpha, sync_loss=False, global_batch=None, length=None):
        """One micro-step of distillation from the trainer's teacher (model.trainer(..., teacher=, teacher_params=)): the
        loss and gradient of `ProGen.distill_loss_and_grad`, then the same clip / AdamW / apply_every update as `step`.
        rows: this rank's (b, n+1) integer rows; global_batch, sync_loss and `length` as in `step` (the teacher runs at
        `distill.teacher_length(length)`).  Data parallel: every rank holds its own teacher; a rank without rows joins the
        all-reduce.  With cuda_graph=True the step, the teacher's forward included, is captured after two eager steps of
        one (rows, global_batch, temperature, alpha, length) and replayed from then on.  Returns the device scalar loss;
        `distill_stats()` has the per-row statistics."""
        from .distill import check_objective
        if self.teacher is None:
            raise L.ProgenError('distill_step: this trainer has no teacher (model.trainer(..., teacher=, teacher_params=))')
        tau, alpha = check_objective(temperature, alpha, 'distill_step')
        b = rows.shape[0]
        gb = int(global_batch) if global_batch is not None else b * self.world
        n = self._length(rows, length, 'distill_step')
        self._distill_rows = b
        return self._step(b, gb, ('distill', tau, alpha), lambda: self.eng.load_distill(rows, n), sync_loss, n)

    def distill_stats(self):
        """this rank's per-row statistics of its last `distill_step` as numpy float32 [b] arrays: kl (KL_b) and ce (CE_b)"""
        return self.eng.distill_stats(getattr(self, '_distill_rows', 0))

    def evaluate_distill(self, data, temperature, alpha, length=None):
        """validation of distillation: the distillation loss of rows `data` (forward and head only); `distill_stats()`
        then has their per-row KL and CE"""
        from .distill import check_objective
        if self.teacher is None:
            raise L.ProgenError('evaluate_distill: this trainer has no teacher')
        tau, alpha = check_objective(temperature, alpha, 'evaluate_distill')
        eng = self.eng
        n = self._length(data, length, 'evaluate_distill')
        eng.lora = self.lora
        B = eng.load_distill(data, n)
        self._drop_graph_unless(B)
        self._distill_rows = B
        eng.train_step(('distill', tau, alpha), B, backward=False, length=n)
        return eng.loss

    # ---- policy gradient on the model's own samples (DESIGN.md §3.14)
    def policy_step(self, rows, span, advantages, beta, sync_loss=False, global_rows=None, length=None):
        """One micro-step of policy-gradient fine-tuning: the loss and gradient of `ProGen.policy_loss_and_grad` on this
        rank's rows (b, n+1), their spans (b, 2) and advantages [b] (`policy.samples_to_rows`, `group_advantages`), with
        the KL to the trainer's reference (model.trainer(..., reference=, reference_params=); needed when beta > 0),
        then the same clip / AdamW / apply_every update as `step`.  global_rows (default b * world) scales the loss, so
        that the all-reduced gradient is the global mean; a rank without rows contributes zeros and joins the
        all-reduce.  sync_loss and `length` as in `step`.  With cuda_graph=True the step, the reference's forward
        included, is captured after two eager steps of one (rows, global_rows, beta, length) and replayed from then on.
        Returns the device scalar loss; `policy_stats()` has the per-row statistics."""
        from .policy import check_policy_batch
        b = len(rows)
        gr = global_rows if global_rows is not None else (b * self.world if b else None)
        rows, span, adv, beta, gr = check_policy_batch(rows, span, advantages, beta, gr, self.eng.n, 'policy_step',
                                                       allow_empty=True)
        if beta > 0 and self.reference is None:
            raise L.ProgenError('policy_step: beta > 0 needs a reference (model.trainer(..., reference=, '
                                'reference_params=))')
        n = self._length(rows, length, 'policy_step')
        self._policy_rows = b
        return self._step(b, gr, ('policy', beta), lambda: self.eng.load_policy(rows, span, adv, n, reference=beta > 0),
                          sync_loss, n)

    def policy_stats(self):
        """this rank's per-row statistics of its last `policy_step` as numpy [b] arrays: logp and kl (span means,
        float32) and count (span lengths, int64)"""
        return self.eng.policy_stats(getattr(self, '_policy_rows', 0))

    def generate(self, prompts, **kw):
        """`ProGen.generate` (same arguments and return dict) from the weights this trainer is updating: with adapters the
        model `adapters()` describes on the frozen base, otherwise `params()`.  One decoder per trainer, rebuilt only when
        a call needs more rows per launch than it holds; its weights are rewritten on the device
        (BatchDecoder.load_weights) when the trainer has stepped since the last call, with no host copy of any weight.
        prefill='forward' is refused: the engine's inference forward does not apply adapters."""
        if kw.get('prefill', 'decode') != 'decode':
            raise L.ProgenError("Trainer.generate: only prefill='decode' runs on the trained weights")
        return self.model._generate(self._generate_decoder, None, prompts, **kw)

    def _generate_decoder(self, batch):
        """the trainer's BatchDecoder for `batch` rows per launch, holding the current weights"""
        from .decode import BatchDecoder
        dec = self._decoder
        if dec is None or dec.B < batch:
            self._decoder = None
            dec = BatchDecoder(self.model.config, self.params(), batch=batch,
                               weights_dtype=torch.bfloat16 if self.model.mixed_precision else torch.float32)
            self._decoder, self._decoder_count = dec, None
        if self._decoder_count != self.count:
            dec.load_weights(self.eng, self.lora)
            self._decoder_count = self.count
        return dec

    def residue_stats(self):
        """the last `residue_step`'s predictions [B, n, C] (regression values, or class logits) and per-position losses
        [B, n] (0 where unlabelled) as numpy float32"""
        return self.eng.residue_stats(getattr(self, '_res_rows', 0))

    def property_stats(self):
        """the last `property_step`'s predictions [B, C] (regression values, or class logits) and per-row losses [B] as
        numpy float32"""
        return self.eng.property_stats(getattr(self, '_prop_rows', 0))

    def head(self):
        """the trained property head {'property_head': {'w', 'b'}} (None without one)"""
        if self.lora is None or not self.lora.head_outputs:
            return None
        return self.lora.split(self.layout.unpack(self.lora.params))[1]

    def preference_stats(self):
        """this rank's statistics of its last `preference_step` as numpy float32 [P] arrays: policy_chosen and
        policy_rejected (the policy's log-likelihoods s), margin (z) and loss (each pair's softplus(-z))"""
        return self.eng.preference_stats(getattr(self, '_pref_pairs', 0))

    def _allreduce_grads(self):
        """SUM of the per-rank gradients (each already scaled by 1/global_rows): the reference's pmap mean, utils.py:78-91"""
        if self.world <= 1 or self.skip_allreduce:
            return
        import torch.distributed as dist
        dist.all_reduce(self.G, op=dist.ReduceOp.SUM)

    def _eager_update(self, sync_loss):
        """the rest of an eager step after the backward pass: the gradient exchange, the logged loss, the optimizer"""
        self._allreduce_grads()
        if sync_loss and self.world > 1:
            PAR.allreduce_scalar_(self.eng.loss)
        self.count += 1
        self._update()
        return self.eng.loss

    def _update(self):
        """norm, AdamW with the device-side count, masked copies: the same launches eagerly and in a captured graph"""
        lib, st = L.load(), L.stream()
        n = self.P.numel()
        L.check(lib.progen_grad_sqnorm(self.G.data_ptr(), n, self.ws.data_ptr(), self.gnorm_sq.data_ptr(), st), 'grad_sqnorm')
        L.check(lib.progen_adamw_step(self.P.data_ptr(), L.ptr(self.P_lp), self.G.data_ptr(),
                                      self.m.data_ptr(), self.v.data_ptr(), self.acc.data_ptr(), n,
                                      self.n_decay, self.gnorm_sq.data_ptr(), self.lr, self.b1, self.b2, self.eps, self.wd,
                                      self.max_norm, self.every, self._adam_state.data_ptr(), st), 'adamw_step')
        self._refresh()                                    # every step (a no-op recompute between emits): keeps the graph static

    def _refresh(self):
        """the compute copies of what the optimizer changed"""
        if self.lora is None:
            self.eng.refresh_masked_copies()
        else:
            self.lora.refresh()

    def _drop_graph_unless(self, batch_rows):
        """a different batch size re-allocates the engine's activation buffers: the captured pointers would dangle"""
        if self._graph is not None and (batch_rows != self._graph_key[0] or
                                        self.eng.alloc_epoch != self._graph_epoch or self._teacher_moved()):
            self._graph = None                             # (model.apply / sampling with another batch size re-allocates too)

    def _teacher_moved(self):
        """the teacher's inference set is not the one the captured steps were recorded on (a larger `score` call on the
        teacher re-allocated it)"""
        ref = self._graph_teacher
        return ref is not None and ref() is not getattr(self.eng.teacher, 'infer', None)

    def _replay(self, sync_loss=False, graph=None):
        """replay `graph` (default: the most recently installed one)"""
        (graph or self._installed).replay()
        self.count += 1
        if sync_loss and self.world > 1:
            PAR.allreduce_scalar_(self.eng.loss)           # logged loss only; the next replay zeroes it again
        return self.eng.loss

    def evaluate(self, data, length=None):
        """validation loss (train.py:207-211): forward + loss only; `length` as in `step`"""
        eng = self.eng
        n = self._length(data, length, 'evaluate')
        eng.lora = self.lora
        B = eng.load_batch(data, n)
        self._drop_graph_unless(B)
        eng.train_step((), B, backward=False, length=n)
        return eng.loss

    # ---- checkpoint interchange (haiku-shaped trees, train.py:196-202)
    def params(self):
        """the base parameters (with adapters: unchanged by training)"""
        return self.eng.export_params()

    def adapters(self):
        """the trained adapters, a tree of `ProGen.init_adapters`' shape (None without adapters)"""
        return None if self.lora is None else self.lora.split(self.layout.unpack(self.lora.params))[0]

    def optim_state(self):
        """{count, mu, nu, acc, every}: trees of the parameters (with adapters: of the adapters) the optimizer owns"""
        u = self.layout.unpack
        return dict(count=self.count, mu=u(self.m), nu=u(self.v), acc=u(self.acc), every=self.every)

    def load_optim_state(self, st):
        """a state of `optim_state`'s form -> the optimizer; ProgenError names a leaf of the wrong shape"""
        if not (isinstance(st, dict) and {'count', 'mu', 'nu', 'acc'} <= set(st)):
            # e.g. an optax chain state from a reference checkpoint: only `params` interchange (checkpoint.py)
            import warnings
            warnings.warn('optim_state is not a progen_b200 Trainer state (reference / optax checkpoint?): optimizer state re-initialised')
            return
        host = [self.layout.pack(st[k]) for k in ('mu', 'nu', 'acc')]
        self.count = int(st['count'])
        self._adam_state[0] = self.count
        for buf, h in zip((self.m, self.v, self.acc), host):
            buf.copy_(torch.from_numpy(h))
