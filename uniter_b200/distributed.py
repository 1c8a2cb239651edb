"""Data-parallel plumbing over torch.distributed (NCCL on H100 / NVLink 4; gloo for CPU tests).

Replaces the Horovod path of the reference (utils/distributed.py):
  * `all_reduce_and_rescale_tensors(grads, 1.0)` (:16-43; call sites train_vqa.py:193-199,
    pretrain.py:302-308) — copy every grad into one flat buffer, `hvd.allreduce_` (Horovod 0.16.4
    default = AVERAGE over ranks), copy back — becomes `GradientReducer`: every parameter's .grad
    already IS a view of one flat arena (uniter_b200.arena.GradArena: task head | pooler | encoder
    layers | embedding front-end, i.e. the order in which the backward pass finishes them), so the
    exchange is a handful of in-place all-reduces of arena slices with no copy-in / copy-out,
    issued on a side stream while the backward of the earlier layers is still running.
  * `broadcast_tensors(params, 0)` (:100-148; train_vqa.py:147) becomes `broadcast_parameters`.
One process per GPU; the path shards by samples only (pure data parallelism, SURVEY.md §8e).
"""
import torch
import torch.distributed as dist

from .arena import GradArena


def _avg_all_reduce(t, async_op=False, group=None):
    """Mean over the ranks of `group`.  NCCL reduces with AVG directly; gloo (CPU tests) sums then
    divides."""
    if dist.get_backend(group) == "nccl":
        return dist.all_reduce(t, op=dist.ReduceOp.AVG, async_op=async_op, group=group)
    dist.all_reduce(t, op=dist.ReduceOp.SUM, async_op=False, group=group)
    t.div_(dist.get_world_size(group))
    return None


def _capped_nccl_group(max_ctas):
    """A second NCCL communicator whose collectives use at most `max_ctas` CTAs, so that the
    overlapped all-reduce and the persistent GEMM / row kernels (which leave exactly that many SMs
    free, ub200_set_sm_reserve) do not fight over SMs.  None if this torch build cannot cap it."""
    try:
        opts = dist.ProcessGroupNCCL.Options()
        opts.config.max_ctas = int(max_ctas)
        opts.config.min_ctas = min(int(max_ctas), 4)
        return dist.new_group(backend="nccl", pg_options=opts)
    except Exception:     # older torch / NCCL without per-communicator config
        return None


class PeerExchange(object):
    """All-reduce (mean) of slices of one flat 16-bit buffer over NVLink peer memory, without NCCL:
    ub200_peer_allreduce of csrc/peer.cu.  Construction is collective: every rank maps every other
    rank's buffer, staging buffer and signal block with cudaIpc (handles travel through
    torch.distributed's object all-gather).  `all_reduce(lo, hi)` only enqueues a handful of memcpy /
    kernel nodes on the current stream — no host synchronisation, capturable in a CUDA graph; every
    rank must issue the same sequence of calls.  Replaces hvd.allreduce_ of utils/distributed.py:16-43."""

    def __init__(self, flat, group=None, max_count=None, timeout_ms=0):
        import ctypes as C
        from . import _lib
        self.lib = _lib.load()
        self.flat = flat
        self.group = group
        self.rank = dist.get_rank(group)
        self.world = dist.get_world_size(group)
        if self.world > _lib.MAX_PEERS:
            raise RuntimeError("PeerExchange supports up to %d ranks of one NVSwitch domain" % _lib.MAX_PEERS)
        self.dtype = _lib.dtype_code(flat.dtype)
        self.timeout_ms = int(timeout_ms)
        n = int(max_count or flat.numel())
        self.stage_bytes = int(self.lib.ub200_peer_stage_bytes(n, self.world))
        fb = int(self.lib.ub200_peer_flags_bytes())
        # one allocation per rank: [staging | signal block]; large enough to be its own cudaMalloc
        # segment of the caching allocator (an allocation can be opened once per process)
        self.ws = torch.zeros(max(self.stage_bytes, 32 << 20) + fb, dtype=torch.uint8, device=flat.device)
        self._flags_off = self.ws.numel() - fb
        torch.cuda.synchronize(flat.device)

        def export(t):
            h = (C.c_char * 64)()
            off = C.c_int64(0)
            _lib.check(self.lib.ub200_peer_ipc_export(C.c_void_p(t.data_ptr()), h, C.byref(off)))
            return bytes(h.raw), int(off.value)

        mine = (export(flat), export(self.ws))
        if mine[0][0] == mine[1][0]:
            raise RuntimeError("PeerExchange: the buffer and the workspace share one allocation")
        everyone = [None] * self.world
        dist.all_gather_object(everyone, mine, group=group)
        self._mapped = []
        self.buf, self.stage, self.flags = [], [], []
        for q, ((hb, ob), (hw, ow)) in enumerate(everyone):
            if q == self.rank:
                b, w = flat.data_ptr(), self.ws.data_ptr()
            else:
                pb, pw = C.c_void_p(), C.c_void_p()
                _lib.check(self.lib.ub200_peer_ipc_open(hb, C.byref(pb)))
                _lib.check(self.lib.ub200_peer_ipc_open(hw, C.byref(pw)))
                self._mapped += [pb.value, pw.value]
                b, w = pb.value + ob, pw.value + ow
            self.buf.append(b)
            self.stage.append(w)
            self.flags.append(w + self._flags_off)
        self._args = {}
        self.calls = 0
        dist.barrier(group=group)          # every signal block is zeroed and mapped before the first kernel

    def _make(self, lo, hi, max_ctas):
        import ctypes as C
        from . import _lib
        a = _lib.PeerAllreduceArgs()
        for q in range(self.world):
            a.buf[q], a.stage[q] = self.buf[q], self.stage[q]
            a.flags[q] = C.cast(C.c_void_p(self.flags[q]), C.POINTER(C.c_uint32))
        a.rank, a.world = self.rank, self.world
        a.offset, a.count = lo, hi - lo
        a.stage_bytes = self.stage_bytes
        a.dtype, a.max_ctas = self.dtype, int(max_ctas)
        a.scale = 1.0 / self.world
        a.timeout_ms = self.timeout_ms
        return a

    def all_reduce(self, lo, hi, max_ctas=-1):
        """flat[lo:hi] <- mean over ranks, in place, on the current stream (lo, hi multiples of 8).
        max_ctas < 0 (default): the copy engines move the bytes over NVLink (memcpy nodes), the SMs only
        run the flag barriers and the local reduction — nothing competes with the backward it overlaps;
        0: a push kernel + a reduce kernel of short-lived CTAs; > 0: one persistent kernel of that many CTAs."""
        from . import _lib
        key = (lo, hi, max_ctas)
        a = self._args.get(key)
        if a is None:
            a = self._args[key] = self._make(lo, hi, max_ctas)
        with _lib.library_mode(_lib.select_mode()):
            _lib.check(self.lib.ub200_peer_allreduce(a, _lib.current_stream()))
        self.calls += 1

    def error_word(self):
        """0, or (call number << 4 | phase) of the first flag wait that expired on this rank (host read)."""
        w = self.ws[self._flags_off:].view(torch.int32)
        return int(w[19].item())

    def close(self):
        for p in self._mapped:
            self.lib.ub200_peer_ipc_close(p)
        self._mapped = []


def broadcast_parameters(model, root=0):
    """Rank `root`'s parameters and buffers -> every rank (startup only)."""
    works = []
    seen = set()
    for t in list(model.parameters()) + list(model.buffers()):
        if id(t) in seen:
            continue
        seen.add(id(t))
        works.append(dist.broadcast(t.data, src=root, async_op=True))
    for w in works:
        w.wait()


class GradientReducer:
    """Average gradients over ranks: in-place all-reduce of slices of the model's gradient arena."""

    def __init__(self, model, overlap_chunks=4, sm_reserve=0, transport="nccl", peer_ctas=-1,
                 peer_tail_ctas=-1):
        """`overlap_chunks` > 1: the encoder layers are all-reduced in that many groups (top group
        first, together with the task-head / pooler slice, which is final by then) while the backward
        of the earlier layers still runs; only the embedding front-end slice is reduced after the
        backward.  `sm_reserve` > 0: during that overlap the library's persistent kernels leave
        `sm_reserve` SMs to the collective, and the collective runs on a communicator capped to the
        same number of CTAs (must be called by all ranks).  Default 0: reserving SMs
        costs the backward more than it gains the collective.
        `transport` "peer": the slices are exchanged by the library's own NVLink peer-memory kernel
        (PeerExchange; `peer_ctas` / `peer_tail_ctas` select its form for the slices shipped while the
        backward runs / after it: < 0 copy engines + local reduction, 0 short-lived CTAs, > 0 one persistent
        kernel of that many CTAs) instead of NCCL — no host involvement, so the whole step including the
        exchange is one CUDA graph."""
        self.model = model
        self.arena = GradArena.attach(model)
        self.encoders = self.arena.encoders
        self.sm_reserve = int(sm_reserve)
        self._group = None
        self._lib = None
        nccl = dist.is_initialized() and dist.get_backend() == "nccl"
        if self.sm_reserve > 0 and overlap_chunks > 1 and nccl:
            self._group = _capped_nccl_group(self.sm_reserve)
            from . import _lib
            self._lib = _lib.load()
        self.overlap_chunks = overlap_chunks
        self.transport = transport
        self.peer = None
        self.peer_ctas, self.peer_tail_ctas = int(peer_ctas), int(peer_tail_ctas)
        if transport == "peer":
            if not (nccl and self.arena.flat.is_cuda):
                raise RuntimeError("transport='peer' needs an initialised NCCL process group on CUDA devices")
            self.peer = PeerExchange(self.arena.flat)
        self._pending = []
        self._done = []               # element ranges of the arena already shipped in this step
        # created up front: the first use may be inside a CUDA-graph capture
        # (lowest priority: GraphedStep captures the step itself on a high-priority stream, so the block
        #  scheduler places the backward's CTAs first and the exchange's CTAs fill what is left)
        self._comm_stream = torch.cuda.Stream(priority=0) if self.arena.flat.is_cuda else None
        self._reserved = False
        self._bwd_seen = {}
        self._tail = False             # shipping what is left after the backward (nothing to overlap)
        self._peer_inflight = False
        # GraphedStep (split mode) sets this while it CAPTURES a step: instead of issuing NCCL, the
        # reducer reports which arena ranges become final at this point of the backward
        self._split_cb = None

    def _emit(self, ranges, final=False):
        ranges = [(lo, hi) for lo, hi in ranges if hi > lo]
        if self._split_cb is not None:
            self._split_cb(ranges, final)
            self._done += ranges
        else:
            for lo, hi in ranges:
                self._ship(lo, hi)

    def ship(self, ranges):
        """Issue the all-reduces of these arena ranges now (side stream, after everything enqueued on the
        current stream so far): the replay side of a step captured in split mode."""
        for lo, hi in ranges:
            self._ship(lo, hi)

    # ---- overlap: called by _EncoderStack.backward after the kernels of layers [lo, hi) are enqueued
    def _ship(self, lo, hi):
        if hi <= lo:
            return
        if self._comm_stream is None:
            self._comm_stream = torch.cuda.Stream()
        ev = torch.cuda.Event()
        ev.record()
        if self._lib is not None and not self._reserved:
            self._lib.ub200_set_sm_reserve(self.sm_reserve)   # launches after this point
            self._reserved = True
        with torch.cuda.stream(self._comm_stream):
            self._comm_stream.wait_event(ev)
            if self.peer is not None:
                self.peer.all_reduce(lo, hi, self.peer_tail_ctas if self._tail else self.peer_ctas)
                self._peer_inflight = True
            else:
                self._pending.append(_avg_all_reduce(self.arena.flat[lo:hi], async_op=True, group=self._group))
        self._done.append((lo, hi))

    def _on_chunk(self, enc, lo, hi):
        # an encoder that ran several forwards in this step (model/nlvr2.py runs the same encoder on
        # two images) accumulates all of them into the same slices: only the LAST backward may ship
        n = self._bwd_seen.get(id(enc), 0)
        NL = enc.config.num_hidden_layers
        if hi == NL:
            n += 1
            self._bwd_seen[id(enc)] = n
        if n < getattr(enc, "_fwd_since_reduce", 1):
            return
        ei = self.encoders.index(enc)
        _, ep = enc._ensure_arena()
        ranges = []
        if hi == NL:
            # everything downstream of the encoder output (task head, pooler) has finished its backward
            h_lo, h_hi = self.arena.segments["head"]
            p_lo, p_hi = self.arena.segments["enc%d.pooler" % ei]
            if ei == 0 and len(self.encoders) == 1 and h_hi == p_lo:
                self.arena.fold_foreign_range(h_lo, p_hi)
                ranges.append((h_lo, p_hi))
        ranges.append((ep["layer0"] + lo * ep["per_layer"], ep["layer0"] + hi * ep["per_layer"]))
        self._emit(ranges)

    def reduce(self):
        """Ship whatever part of the arena has not been shipped yet, then wait for everything."""
        self.arena.fold_foreign()
        rest, pos = [], 0
        for lo, hi in sorted(self._done):
            if lo > pos:
                rest.append((pos, lo))
            pos = max(pos, hi)
        if pos < self.arena.numel:
            rest.append((pos, self.arena.numel))
        if self._split_cb is not None:          # capturing in split mode: report, issue nothing
            self._emit(rest, final=True)
            self._done = []
            self._bwd_seen = {}
            for enc in self.encoders:
                enc._fwd_since_reduce = 0
            return
        works = self._pending
        self._pending = []
        cuda = self.arena.flat.is_cuda
        self._tail = True
        try:
            for lo, hi in rest:
                if cuda and self._comm_stream is not None and (self._done or self.peer is not None):
                    self._ship(lo, hi)
                else:
                    works.append(_avg_all_reduce(self.arena.flat[lo:hi], async_op=cuda, group=self._group))
        finally:
            self._tail = False
        if self._peer_inflight:           # join: the current stream continues after the last exchange kernel
            torch.cuda.current_stream().wait_stream(self._comm_stream)
            self._peer_inflight = False
        works += self._pending
        self._pending = []
        self._done = []
        self._bwd_seen = {}
        for enc in self.encoders:
            enc._fwd_since_reduce = 0
        for w in works:
            if w is not None:
                w.wait()

    def reset_step_state(self):
        """Forget what this step has shipped / how many forwards each encoder ran since the last reduce().
        GraphedStep calls it before capturing a step: its warm-up steps run without the reducer (a capture
        must not communicate), so the per-step counters that reduce() normally clears are stale."""
        self._pending = []
        self._done = []
        self._bwd_seen = {}
        self._tail = False
        for enc in self.encoders:
            enc._fwd_since_reduce = 0

    def backward_and_reduce(self, loss):
        """loss.backward() with the gradients all-reduced slice by slice while the rest of the
        backward is still running (replaces the non-overlapped Horovod call of
        train_vqa.py:193-199), then the remaining slices."""
        overlap = self.overlap_chunks > 1 and dist.get_backend() == "nccl"
        if overlap:
            for enc in self.encoders:
                enc._bwd_chunk_hook = self._on_chunk
                enc._bwd_chunks = self.overlap_chunks
        try:
            loss.backward()
        finally:
            for enc in self.encoders:
                enc._bwd_chunk_hook = None
            if self._reserved:
                self._lib.ub200_set_sm_reserve(0)
                self._reserved = False
        self.reduce()
