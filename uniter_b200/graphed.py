"""Host-free training step: forward + backward (+ gradient exchange, + optimizer) replayed from a
CUDA graph per batch-shape bucket.

Why.  At the reference's batch sizes one step is a few milliseconds of GPU work spread over ~250
kernels; enqueueing them from Python (autograd glue, ctypes marshalling, allocator) costs about as
much host time as the GPU needs to run them, so the step is host-bound (SURVEY.md §7 step 8; the
thing replaced is the per-op Python of model/layer.py:159-170 and the training loop around it,
train_vqa.py:183-229).  A captured graph is enqueued with ONE driver call.

What makes the step capturable here:
  * every kernel of libub200 takes shapes from host-known lengths (`register_lengths`), never
    from data on the device, and launches on the capturing stream;
  * dropout streams are offset by a DEVICE counter (`rng_offset_dev`) that the graph itself bumps
    at the start of every replay, so replays draw fresh masks;
  * every parameter's .grad is a fixed view of the gradient arena (uniter_b200.arena): the kernels
    write into the same addresses in every graph, whatever the bucket;
  * the token count is padded to a bucket (`token_bucket`, default 128 rows = one GEMM row tile) with
    ONE dummy sequence (see model._prefix_pack_host): identical results, bit for bit, and one graph
    serves every batch of the bucket.  The key of a graph is
    (tensor shapes of the batch, padded token count, attention max-seqlen bucket, accumulate flag,
    library mode).
  * the library's deterministic mode follows torch.use_deterministic_algorithms at stage() time
    (uniter_b200._lib.select_mode): warm-up and capture run in it, and a graph only replays in the
    mode it was captured in.

Usage:
    step = GraphedStep(model, lambda b: model(b).sum() * b["mlm_inv_n"])
    loss = step(host_batch, lens)          # host_batch: dict of (pinned) CPU tensors; lens: per-sample
                                           # valid lengths of host_batch["attn_masks"] (prefix masks)
`loss` is a static device tensor, overwritten by the next call of the same bucket.
"""
import numpy as np
import torch

from . import _lib
from . import model as _model
from .arena import GradArena


def _round_up(v, m):
    return (v + m - 1) // m * m


class _Bucket(object):
    __slots__ = ("graph", "graphs", "ship_after", "inputs", "meta_dev", "meta_offs", "loss", "T_pad", "maxseq",
                 "n_replays", "launches", "mode")


class GraphedStep(object):
    def __init__(self, module, loss_fn, token_bucket=128, reducer=None, optimizer=None,
                 optimizer_kwargs=None, zero_all_grads=False, mask_key="attn_masks", warmup=2,
                 reducer_mode="split", loss_scaler=None, loss_ids=None):
        """module: the root nn.Module (its parameters' gradients go to one arena);
        loss_fn(batch_on_device) -> scalar loss (runs the forward);
        reducer: optional GradientReducer.  reducer_mode "split" (default): the step is captured as a
        CHAIN of graphs cut where a slice of the gradient arena becomes final (after the task head +
        top layer group, after every further layer group, after the embedding backward); on replay each
        slice's NCCL all-reduce is issued eagerly on the reducer's side stream right after its graph and
        overlaps the next graph; the tail graph (never-touched gradients zeroed, optimizer) runs after
        the last all-reduce.  "in-graph": the reducer's exchange is captured inside the ONE graph of the
        step — what GradientReducer(transport="peer") is built for (its exchange is memcpy + kernel nodes);
        with the NCCL transport this mode and "split" hung in earlier measurements because capture warm-ups
        executed collectives the other ranks did not take part in (fixed: captures are local now), and
        were not re-measured since.
        optimizer: optional FusedAdamW stepped inside the (tail) graph; zero_all_grads: see
        GradArena.begin_step(zero_all=...).
        loss_scaler: optional DynamicLossScaler (fp16): the step back-propagates
        loss_scaler.scale(loss, id) and the optimizer unscales by, and updates, entry `id` — all from
        device memory, so replays follow the current scale and a change of scale never re-captures;
        the returned loss stays unscaled.  loss_ids: {tag: id} (e.g. one scaler per pre-training task,
        pretrain.py:230-233); without it every step uses id 0."""
        if loss_scaler is not None and "grad_scale" in (optimizer_kwargs or {}):
            raise ValueError("GraphedStep: give either loss_scaler or optimizer_kwargs['grad_scale'], not both")
        self.module = module
        self.loss_fn = loss_fn
        self.token_bucket = int(token_bucket)
        self.reducer = reducer
        self.reducer_mode = reducer_mode if reducer is not None else "none"
        self.optimizer = optimizer
        self.optimizer_kwargs = optimizer_kwargs or {}
        self.loss_scaler = loss_scaler
        self.loss_ids = dict(loss_ids) if loss_ids is not None else None
        self.zero_all = bool(zero_all_grads)
        self.mask_key = mask_key
        self.warmup = int(warmup)
        self.arena = GradArena.attach(module)
        self.device = self.arena.device
        self.buckets = {}
        self.pool = None
        self.rng_counter = torch.zeros(1, device=self.device, dtype=torch.int64)
        # the step is captured on a HIGH-priority stream: kernel nodes inherit it, side-stream work forked
        # inside the step (the reducer's gradient exchange, priority 0) yields SMs to the step's own kernels
        self._cap_stream = torch.cuda.Stream(device=self.device, priority=-1)
        self._meta_pinned = {}
        self.captures = 0

    # ------------------------------------------------------------------ keys / buffers
    def _key(self, host_batch, lens, accumulate, tag=None, step_optimizer=True):
        T = int(sum(lens))
        T_pad = max(_round_up(T, self.token_bucket), self.token_bucket)
        maxseq = _round_up(max(max(lens), 1, T_pad - T), 128)
        sig = tuple((k, tuple(v.shape), str(v.dtype)) for k, v in sorted(host_batch.items())
                    if torch.is_tensor(v))
        # the library mode the step runs in (torch.use_deterministic_algorithms) and, for a bucket whose
        # attention backward has no fixed-order form, the warn_only decision (raises, or warns and gives 0:
        # the encoder node then runs in the default mode, as in an eager step, the rest of the step in the
        # step's mode).  Both are part of the key, so a change of torch's flags captures a new graph
        # instead of replaying one of the other mode.
        long_decision = _lib.select_mode(maxseq)
        mode = _lib.select_mode()
        return (sig, T_pad, maxseq, bool(accumulate), tag, self._steps_optimizer(step_optimizer), mode,
                long_decision), T_pad, maxseq

    def _steps_optimizer(self, step_optimizer):
        return self.optimizer is not None and bool(step_optimizer)

    def _loss_id(self, tag):
        if self.loss_ids is None:
            return 0
        if tag not in self.loss_ids:
            raise KeyError("GraphedStep: no loss id for tag %r (loss_ids has %s)" % (tag, sorted(self.loss_ids)))
        return int(self.loss_ids[tag])

    def _fill_meta(self, bk, lens, L):
        """Packing bookkeeping of this batch -> the bucket's static device buffer (one H2D)."""
        host, offs, _ = _model._prefix_pack_host(lens, L, bk.T_pad)
        n = host.numel()
        slot = self._meta_pinned.get(n)
        if slot is None:
            slot = [torch.empty(n, dtype=torch.int32).pin_memory() for _ in range(4)] + [0]
            self._meta_pinned[n] = slot
        i = slot[4]
        slot[4] = (i + 1) % 4
        slot[i].copy_(host)
        bk.meta_dev.copy_(slot[i], non_blocking=True)
        return offs

    # ------------------------------------------------------------------ the captured region
    def _run(self, bk, accumulate, tag=None, step_optimizer=True):
        with _lib.library_mode(bk.mode):
            return self._run_in_mode(bk, accumulate, tag, step_optimizer)

    def _run_in_mode(self, bk, accumulate, tag, step_optimizer):
        self.rng_counter.add_(64)                       # fresh dropout masks for this replay
        self.arena.begin_step(accumulate=accumulate, zero_all=self.zero_all)
        _model._RNG_GRAPH["dev"] = self.rng_counter
        _model._RNG_GRAPH["call"] = 0
        try:
            loss = self.loss_fn(bk.inputs) if tag is None else self.loss_fn(bk.inputs, tag)
            opt_kwargs = self.optimizer_kwargs
            to_backward = loss
            if self.loss_scaler is not None:
                # the scale is a device scalar read by the graph: every micro-batch of an accumulation
                # window carries the same scale, which moves only at the optimizer step (apex delay_unscale)
                lid = self._loss_id(tag)
                to_backward = self.loss_scaler.scale(loss, lid)
                opt_kwargs = dict(opt_kwargs, grad_scale=self.loss_scaler, loss_id=lid)
            if self.reducer is not None:
                self.reducer.backward_and_reduce(to_backward)
            else:
                to_backward.backward()
            self.arena.finish_step()          # parameters this step never touched: exactly zero
            if self.optimizer is not None and step_optimizer:
                self.optimizer.step(**opt_kwargs)
        finally:
            _model._RNG_GRAPH["dev"] = None
            self.arena.end_step_mode()
        return loss.detach()

    def _capture(self, key, host_batch, lens, T_pad, maxseq, accumulate, tag=None, step_optimizer=True):
        bk = _Bucket()
        bk.T_pad, bk.maxseq, bk.n_replays, bk.mode = T_pad, maxseq, 0, key[-2]
        dev = self.device
        bk.inputs = {k: torch.empty(v.shape, dtype=v.dtype, device=dev)
                     for k, v in host_batch.items() if torch.is_tensor(v)}
        for k, v in host_batch.items():
            if torch.is_tensor(v):
                bk.inputs[k].copy_(v, non_blocking=True)
        mask = bk.inputs[self.mask_key]
        B, L = mask.shape
        host, offs, _ = _model._prefix_pack_host(lens, L, T_pad)
        bk.meta_dev = torch.empty(host.numel(), dtype=torch.int32, device=dev)
        bk.meta_offs = self._fill_meta(bk, lens, L)
        meta = _model._meta_from_buffer(bk.meta_dev, bk.meta_offs, B, L, T_pad, maxseq, None, True)
        _model._meta_store(mask, meta)            # forward() finds the static bookkeeping on this tensor
        # warm-up on a side stream (allocator, cudaFuncSetAttribute, TMA descriptor cache), then capture
        # (the warm-up runs are REAL steps: an accumulating step would add its gradients several times
        #  and an optimizer would move the weights, so the arena is restored and the optimizer only
        #  prepares its device tables)
        # A capture must be a purely LOCAL event: ranks see different batches, so they meet new buckets
        # (new shapes of the padded masked-token lists, new token counts) at different steps and in
        # different numbers.  The warm-up therefore runs WITHOUT the reducer — a warm-up step that
        # all-reduced would be a collective the other ranks do not take part in (NCCL: hang; peer
        # exchange: ranks pair up different calls) — and the capture itself executes nothing.
        saved = self.arena.flat.clone() if accumulate else None
        opt, self.optimizer = self.optimizer, None
        red, self.reducer = self.reducer, None
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(self.warmup):
                self._run(bk, accumulate, tag, step_optimizer)
            if saved is not None:
                self.arena.flat.copy_(saved)
        torch.cuda.current_stream().wait_stream(s)
        self.optimizer = opt
        self.reducer = red
        if red is not None:
            red.reset_step_state()        # the warm-up forwards were not followed by a reduce()
        if opt is not None:
            opt.prepare()
        if self.pool is None:
            self.pool = torch.cuda.graph_pool_handle()
        lib = _lib.load()
        lib.ub200_launch_count.restype = __import__("ctypes").c_ulonglong
        n0 = lib.ub200_launch_count()
        if self.reducer_mode == "split":
            self._capture_split(bk, accumulate, tag, step_optimizer)
        else:
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, pool=self.pool, stream=self._cap_stream):
                bk.loss = self._run(bk, accumulate, tag, step_optimizer)
            bk.graphs, bk.ship_after = [g], [[]]
        bk.launches = int(lib.ub200_launch_count() - n0)     # libub200 kernels inside one replay
        bk.graph = bk.graphs[0]
        self.buckets[key] = bk
        self.captures += 1
        return bk

    def _capture_split(self, bk, accumulate, tag, step_optimizer=True):
        """Capture the step as a chain of graphs, cut wherever the reducer reports that ranges of the
        arena are final (reducer._split_cb).  No NCCL call happens during the capture; on replay the
        ranges recorded for a cut are all-reduced right after the graph that ends there."""
        import gc
        graphs, ship = [], []
        state = {"g": None}

        def begin():
            g = torch.cuda.CUDAGraph()
            g.capture_begin(pool=self.pool)
            state["g"] = g

        def cut(ranges, final=False):
            state["g"].capture_end()
            graphs.append(state["g"])
            ship.append(list(ranges))
            begin()                       # (after the final cut: the tail — zeroing, optimizer)

        torch.cuda.synchronize()
        gc.collect()
        cap = torch.cuda.Stream()
        cap.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(cap):
            begin()
            self.reducer._split_cb = cut
            try:
                # the cuts end / begin captures from inside autograd's backward: keep it on this thread
                with torch.autograd.set_multithreading_enabled(False):
                    bk.loss = self._run(bk, accumulate, tag, step_optimizer)
            finally:
                self.reducer._split_cb = None
                state["g"].capture_end()
                graphs.append(state["g"])
                ship.append([])
        torch.cuda.current_stream().wait_stream(cap)
        bk.graphs, bk.ship_after = graphs, ship

    def replay(self, bk):
        """Enqueue one step of a staged bucket (see stage())."""
        if self.optimizer is not None:
            self.optimizer.sync_lr()          # the captured step reads the learning rates from the device
        if len(bk.graphs) == 1:
            bk.graphs[0].replay()
        else:
            red = self.reducer
            last = len(bk.graphs) - 1
            for k, g in enumerate(bk.graphs):
                if k == last:
                    red.reduce()              # nothing left to ship: waits for the slices in flight
                g.replay()
                if bk.ship_after[k]:
                    red.ship(bk.ship_after[k])
        bk.n_replays += 1
        return bk.loss

    # ------------------------------------------------------------------ public
    def stage(self, host_batch, lens, accumulate=False, tag=None, step_optimizer=True):
        """Copy a batch (pinned host tensors, or device tensors prefetched on a copy stream) into its
        bucket's static inputs (async, current stream) and return the bucket; capture the bucket's
        graph first if it is new.  `tag` (e.g. the pre-training task) becomes part of the bucket key and
        is passed to loss_fn(batch, tag).  step_optimizer=False: the step ends after the backward (the
        micro-batches of an accumulation window before its last one); it has its own graph."""
        key, T_pad, maxseq = self._key(host_batch, lens, accumulate, tag, step_optimizer)
        bk = self.buckets.get(key)
        if bk is None:
            bk = self._capture(key, host_batch, lens, T_pad, maxseq, accumulate, tag,
                               self._steps_optimizer(step_optimizer))
        for k, v in host_batch.items():
            if torch.is_tensor(v):
                bk.inputs[k].copy_(v, non_blocking=True)
        mask = bk.inputs[self.mask_key]
        self._fill_meta(bk, lens, mask.size(1))
        return bk

    def __call__(self, batch, lens, accumulate=False, tag=None, step_optimizer=True):
        if self.arena._stale:
            raise RuntimeError("GraphedStep: parameters of the module were replaced after this step was built "
                               "(e.g. by init_type_embedding / init_word_embedding); build a new GraphedStep")
        return self.replay(self.stage(batch, lens, accumulate, tag, step_optimizer))
