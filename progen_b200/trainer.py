"""Device-resident training state for the train.py loop: parameters, gradients, Adam moments and the apply_every
accumulator live in flat fp32 buffers; one `step(data)` is one iteration of the reference's inner loop
(train.py:186-190): loss+grads, optim.update, apply_updates.

With low-rank adapters (`adapters=`) the same state exists for the adapter buffer only: the base parameters are frozen
and bitwise unchanged, and clip / AdamW / apply_every run over the adapters (weight decay on every A and B)."""
import os

import numpy as np
import torch

from . import lib as L
from . import parallel as PAR


class Trainer:
    def __init__(self, model, params, learning_rate=2e-4, weight_decay=1e-3, max_grad_norm=0.5, grad_accum_every=4,
                 b1=0.9, b2=0.999, eps=1e-8, optim_state=None, data_parallel=True, cuda_graph=False, adapters=None,
                 lora_alpha=None):
        self.model = model
        self.eng = model.engine
        self.eng.load_params(params)
        model._loaded = None
        self.lora = None
        if adapters is not None:
            from .lora import Adapters, check_adapters, check_rank_alpha
            rank, alpha = check_rank_alpha(check_adapters(model.config, adapters), lora_alpha)
            self.lora = Adapters(self.eng, rank, alpha)
            self.lora.load(adapters)
        # the flat buffers the optimizer owns: (parameters, size, ndim > 1 prefix, bf16 mirror or None); gradients: self.G
        if self.lora is None:
            e = self.eng
            self.P, n, self.n_decay, self.P_lp = e.params, e.n_params_padded, e.n_decay, e.params_lp
        else:
            lo = self.lora
            self.P, n, self.n_decay, self.P_lp = lo.params, lo.n_padded, lo.n_padded, None
            self.eng.grads = None                  # nothing reads or writes the base gradient while adapters train
        self.eng.lora = self.lora
        self.lr, self.wd, self.max_norm, self.every = learning_rate, weight_decay, max_grad_norm, grad_accum_every
        self.b1, self.b2, self.eps = b1, b2, eps
        z = lambda: torch.zeros(n, device=self.eng.dev, dtype=torch.float32)
        self.m, self.v, self.acc = z(), z(), z()
        self.count = 0
        self.ws = torch.empty(L.load().progen_optim_workspace_floats(), device=self.eng.dev)
        self.gnorm_sq = torch.zeros(1, device=self.eng.dev)
        self.rank, self.world = PAR.world() if data_parallel else (0, 1)
        self._works, self._done = [], []
        self._graph, self._graph_key, self._graph_epoch, self._adam_state = None, None, 0, None
        # cuda_graph=True: after two eager steps of one batch shape the step is captured and replayed from then on
        self._auto_graph, self._eager_key, self._eager_run = bool(cuda_graph), None, 0
        self._bucket, self._bucket_layers = None, max(1, int(os.environ.get('PROGEN_DDP_BUCKET_LAYERS', '3')))
        # Gradient exchange (world > 1).  Default: ONE SUM all-reduce of the whole flat buffer after the backward pass, on
        # the compute stream, inside the captured CUDA graph.  Overlapping per-layer buckets with the backward pass lets the
        # NCCL kernels take SMs from the backward kernels and needs eager launches.  PROGEN_DDP_OVERLAP=1 selects that mode
        # (eager launches only) for models whose gradient is large enough to make the transfer itself matter.
        self.overlap = os.environ.get('PROGEN_DDP_OVERLAP', '0') == '1'
        if self.overlap and self.lora is not None:
            raise L.ProgenError('PROGEN_DDP_OVERLAP=1 does not support adapters: their gradient is one small buffer, '
                                'all-reduced once per step')
        self.skip_allreduce = False                       # bench.py: "step without the exchange" for comm_exposed_ms
        if self.world > 1 and self.overlap:
            # overlap: a layer's weight gradients are all-reduced (async, NCCL's stream) as soon as its backward is done
            self.eng.on_layer_grads = self._reduce_layer
        if optim_state is not None:
            self.load_optim_state(optim_state)

    @property
    def G(self):
        """the flat gradient the optimizer reads: the adapters', or every parameter's"""
        return self.eng.base_grads() if self.lora is None else self.lora.grads

    # ---- one micro-step of train.py:186-190
    def step(self, data, sync_loss=False, global_batch=None):
        """data: this rank's rows, (b, n+1) integers; `global_batch` = rows of the UNSHARDED batch (utils.py:83-91: the
        masked mean divides by the real row count, so ragged shards — 5 rows over 2 ranks = 3 + 2, or ranks with no rows
        at all — must all scale by 1/5).  Without it the shards are assumed equal.  Returns the device scalar loss
        (global mean when sync_loss)."""
        rows = data.shape[0]
        gb = int(global_batch) if global_batch is not None else (rows * self.world if self.world > 1 else rows)
        self.eng.lora = self.lora
        if rows == 0:
            # a rank without rows (batch smaller than the world): zero contribution, but every collective is joined
            self.G.zero_()
            self.eng.loss.zero_()
            return self._update(sync_loss)
        self._drop_graph_unless(rows)
        if self._graph is not None and self._graph_key == (rows, gb):
            self.eng.load_batch(data)                      # H2D copies stay outside the graph
            return self._replay(sync_loss)
        self.eng.loss_and_grad(data, global_batch=gb)
        loss = self._update(sync_loss)
        if self._auto_graph and not self.overlap:
            key = (data.shape[0], gb)
            self._eager_run = self._eager_run + 1 if key == self._eager_key else 1
            self._eager_key = key
            if self._eager_run >= 2:
                self.capture_graph(data.shape[0], gb)      # capture does not execute: eng.loss still holds this step's value
                self._eager_run = 0
        return loss

    def step_resident(self, global_batch=None, sync_loss=False):
        """same, on tokens/labels already copied into engine.tok / engine.labels (bench: inputs resident in HBM)"""
        gb = global_batch or self.eng.B * self.world
        self.eng.lora = self.lora
        self._drop_graph_unless(self.eng.B)
        if self._graph is not None and self._graph_key == (self.eng.B, gb):
            return self._replay(sync_loss)
        self.eng.step_device(gb)
        return self._update(sync_loss)

    # ---- CUDA graph of the whole step: forward, loss, backward, (gradient all-reduce), norm, AdamW, masked copies
    def capture_graph(self, batch_rows, global_batch=None, install=True):
        """Capture one training step for batches of `batch_rows` rows into a CUDA graph; later `step` / `step_resident`
        calls with that shape replay it.  The step-dependent optimizer scalars live on the device
        (`progen_adamw_step_dev`), so the graph is identical for every step.  Under data parallelism the NCCL all-reduce
        of the gradient buffer is part of the graph (issued on the capture stream between backward and the norm).  Call
        after at least one eager step of the same shape (kernel attributes, tensor maps, buffers and the NCCL communicator
        must exist before capture).  `install=False` returns the graph without making it the one `step` replays."""
        gb = global_batch or batch_rows * self.world
        return self._capture(batch_rows, (batch_rows, gb), lambda: self.eng.step_device(gb), install)

    def _capture(self, batch_rows, key, step_device, install=True):
        """capture step_device() + gradient exchange + optimizer for batches of `batch_rows` rows; `key` is what a later
        step must match to replay it"""
        if self.world > 1 and self.overlap:
            raise L.ProgenError('capture_graph: PROGEN_DDP_OVERLAP=1 launches its bucketed all-reduces eagerly')
        eng = self.eng
        eng.lora = self.lora
        eng.ensure_batch(batch_rows)
        if self._adam_state is None:
            self._adam_state = torch.zeros(4, dtype=torch.int64, device=eng.dev)   # AdamDevState: count | bc1, bc2 | emit, pad
        self._adam_state[0] = self.count
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            step_device()
            self._allreduce_grads()
            self._update_captured()
        if install:
            self._graph, self._graph_key, self._graph_epoch = g, key, getattr(eng, 'alloc_epoch', 0)
        return g

    # ---- preference (DPO) fine-tuning
    def preference_step(self, chosen, rejected, ref_chosen, ref_rejected, beta=0.1, sync_loss=False, global_pairs=None):
        """One micro-step of preference (DPO) fine-tuning on this rank's pairs: the loss and gradient of
        `ProGen.preference_loss_and_grad`, then the same clip / AdamW / apply_every update as `step`.  chosen / rejected:
        (P, n+1) integer rows; ref_chosen / ref_rejected [P]: their log-likelihoods under the frozen reference (`score`).
        Data parallel: give each rank `parallel.shard_rows(P_global, rank, world)` of the pairs and global_pairs =
        P_global (default: equal shards, P * world); a rank without pairs contributes zeros but joins the all-reduce.
        With cuda_graph=True the step is captured after two eager steps of one (P, global_pairs, beta) and replayed from
        then on.  Returns the device scalar loss (global mean when sync_loss); `preference_stats()` has the per-pair
        statistics."""
        from .preference import check_pairs
        gp = global_pairs
        if gp is None and self.world > 1:
            gp = len(chosen) * self.world
        rows, ref, beta, gp = check_pairs(chosen, rejected, ref_chosen, ref_rejected, beta, gp, self.eng.n,
                                          what='preference_step', allow_empty=True)
        P = rows.shape[0] // 2
        self._pref_pairs = P
        self.eng.lora = self.lora
        if P == 0:
            self.G.zero_()
            self.eng.loss.zero_()
            return self._update(sync_loss)
        key = (2 * P, gp, 'preference', beta)
        self._drop_graph_unless(2 * P)
        if self._graph is not None and self._graph_key == key:
            self.eng.load_preference(rows, ref)            # H2D copies stay outside the graph
            return self._replay(sync_loss)
        self.eng.load_preference(rows, ref)
        self.eng.preference_step_device(P, beta, gp)
        loss = self._update(sync_loss)
        if self._auto_graph and not self.overlap:
            self._eager_run = self._eager_run + 1 if key == self._eager_key else 1
            self._eager_key = key
            if self._eager_run >= 2:
                self._capture(2 * P, key, lambda: self.eng.preference_step_device(P, beta, gp))
                self._eager_run = 0
        return loss

    def preference_stats(self):
        """this rank's statistics of its last `preference_step` as numpy float32 [P] arrays: policy_chosen and
        policy_rejected (the policy's log-likelihoods s), margin (z) and loss (each pair's softplus(-z))"""
        return self.eng.preference_stats(getattr(self, '_pref_pairs', 0))

    def _allreduce_grads(self):
        """SUM of the per-rank gradients (each already scaled by 1/global_rows): the reference's pmap mean, utils.py:78-91"""
        if self.world <= 1 or self.skip_allreduce:
            return
        import torch.distributed as dist
        if self.overlap:
            self._finish_allreduce()
        else:
            dist.all_reduce(self.G, op=dist.ReduceOp.SUM)

    def _update_captured(self):
        eng, lib, st = self.eng, L.load(), L.stream()
        n = self.P.numel()
        L.check(lib.progen_grad_sqnorm(self.G.data_ptr(), n, self.ws.data_ptr(), self.gnorm_sq.data_ptr(), st), 'grad_sqnorm')
        L.check(lib.progen_adamw_step_dev(self.P.data_ptr(), L.ptr(self.P_lp), self.G.data_ptr(),
                                          self.m.data_ptr(), self.v.data_ptr(), self.acc.data_ptr(), n,
                                          self.n_decay, self.gnorm_sq.data_ptr(), self.lr, self.b1, self.b2, self.eps, self.wd,
                                          self.max_norm, self.every, self._adam_state.data_ptr(), st), 'adamw_step_dev')
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
                                        getattr(self.eng, 'alloc_epoch', 0) != self._graph_epoch):
            self._graph, self._graph_key = None, None      # (model.apply / sampling with another batch size re-allocates too)

    def _replay(self, sync_loss=False):
        self._graph.replay()
        self.count += 1
        if sync_loss and self.world > 1:
            PAR.allreduce_scalar_(self.eng.loss)           # logged loss only; the next replay zeroes it again
        return self.eng.loss

    def _reduce_layer(self, i):
        """Layer i's backward is done (layers arrive in descending order).  Consecutive layers are merged into one
        bucket of `PROGEN_DDP_BUCKET_LAYERS` layers (default 3): every NCCL kernel holds SMs while it waits for the slowest
        rank, and the statically partitioned persistent kernels running beside it end late by that long, so fewer, larger
        all-reduces cost less than one per layer."""
        import torch.distributed as dist
        a, b = self.eng.layer_grad_range(i)
        if self._bucket is None:
            self._bucket = [a, b, 0]
        assert b == self._bucket[0] or (a, b) == tuple(self._bucket[:2]), 'layer gradient ranges must be adjacent'
        self._bucket[0] = min(self._bucket[0], a)
        self._bucket[2] += 1
        if self._bucket[2] >= self._bucket_layers or i == 0:
            lo, hi, _ = self._bucket
            self._works.append(dist.all_reduce(self.eng.grads[lo:hi], op=dist.ReduceOp.SUM, async_op=True))
            self._done.append((lo, hi))
            self._bucket = None

    def _finish_allreduce(self):
        """everything the per-layer reductions did not cover: embedding (final only at the very end of backward), head,
        and the small ndim<=1 section; then wait for the overlapped ones"""
        eng = self.eng
        lo = min((a for a, _ in self._done), default=eng.n_params_padded)
        hi = max((b for _, b in self._done), default=eng.n_params_padded)
        if self._done:
            PAR.allreduce_sum_(eng.grads[:lo])
            PAR.allreduce_sum_(eng.grads[hi:])
        else:
            PAR.allreduce_sum_(eng.grads)
        for w in self._works:
            w.wait()
        self._works, self._done = [], []

    def _update(self, sync_loss):
        eng, lib, st = self.eng, L.load(), L.stream()
        if self.world > 1:
            self._allreduce_grads()
            if sync_loss:
                PAR.allreduce_scalar_(eng.loss)
        self.count += 1
        if self._adam_state is not None:
            self._adam_state[0] = self.count               # keep the device-side count in step with eager steps
        emit = int(self.count % self.every == 0)
        n = self.P.numel()
        L.check(lib.progen_grad_sqnorm(self.G.data_ptr(), n, self.ws.data_ptr(), self.gnorm_sq.data_ptr(), st), 'grad_sqnorm')
        L.check(lib.progen_adamw_step(self.P.data_ptr(), L.ptr(self.P_lp), self.G.data_ptr(),
                                      self.m.data_ptr(), self.v.data_ptr(), self.acc.data_ptr(), n, self.n_decay,
                                      self.gnorm_sq.data_ptr(), self.lr, self.b1, self.b2, self.eps, self.wd, self.max_norm,
                                      self.count, emit, st), 'adamw_step')
        if emit:
            self._refresh()
        return eng.loss

    def evaluate(self, data):
        """validation loss (train.py:207-211): forward + loss only"""
        eng = self.eng
        d = torch.as_tensor(np.asarray(data).astype(np.int32) if not isinstance(data, torch.Tensor) else data)
        self._drop_graph_unless(d.shape[0])
        eng.lora = self.lora
        eng.ensure_batch(d.shape[0])
        dd = d.to(device=eng.dev, dtype=torch.int32)
        eng.tok.copy_(dd[:, :-1].reshape(-1))
        eng.labels.copy_(dd[:, 1:].reshape(-1))
        eng._forward_device()
        eng.loss.zero_()
        L.check(L.load().progen_ce_fwd_bwd(eng.logits.data_ptr(), L.F32, eng.labels.data_ptr(), eng.ce_w.data_ptr(), eng.loss.data_ptr(),
                                           0, eng.act_dt, eng.B, eng.n, eng.V, 1.0 / d.shape[0], L.stream()), 'ce_fwd')
        return eng.loss

    # ---- checkpoint interchange (haiku-shaped trees, train.py:196-202)
    def params(self):
        """the base parameters (with adapters: unchanged by training)"""
        return self.eng.export_params()

    def adapters(self):
        """the trained adapters, a tree of `ProGen.init_adapters`' shape (None without adapters)"""
        return None if self.lora is None else self.lora.export_tree(self.lora.params)

    def optim_state(self):
        """{count, mu, nu, acc, every}: trees of the parameters (with adapters: of the adapters) the optimizer owns"""
        e = self.eng if self.lora is None else self.lora
        return dict(count=self.count, mu=e.export_tree(self.m), nu=e.export_tree(self.v), acc=e.export_tree(self.acc),
                    every=self.every)

    def load_optim_state(self, st):
        e = self.eng if self.lora is None else self.lora
        if not (isinstance(st, dict) and {'count', 'mu', 'nu', 'acc'} <= set(st)):
            # e.g. an optax chain state from a reference checkpoint: only `params` interchange (checkpoint.py)
            import warnings
            warnings.warn('optim_state is not a progen_b200 Trainer state (reference / optax checkpoint?): optimizer state re-initialised')
            return
        self.count = int(st['count'])
        for buf, tree in ((self.m, st['mu']), (self.v, st['nu']), (self.acc, st['acc'])):
            host = np.zeros(self.P.numel(), np.float32)
            for s in e.specs:
                a = np.asarray(tree[s.module][s.name], np.float32)
                if s.interleave:
                    from .engine import _interleave
                    a = _interleave(a)
                host[s.offset:s.offset + s.size] = a.ravel()
            buf.copy_(torch.from_numpy(host))
