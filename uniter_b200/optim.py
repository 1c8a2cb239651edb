"""Fused multi-tensor AdamW with fp32 master weights on libub200 (SURVEY.md §8f-2).

Replaces, for 16-bit models on an H100, what the reference assembles from three pieces:

* ``optim/adamw.py:43-103`` — the AdamW update itself (bias-corrected step size; decoupled weight
  decay ``p -= lr * wd * p`` applied AFTER the Adam update);
* apex ``amp`` O2 (``train_vqa.py:152,190-192``) — fp32 master copies of the fp16 parameters,
  master-gradient copy + unscale before the step, master -> model copy after it;
* ``torch.nn.utils.clip_grad_norm_(amp.master_params(optimizer), grad_norm)``
  (``train_vqa.py:223-226``).

Here: ONE kernel computes the global gradient norm (``ub200_grad_sumsq``) and ONE kernel does
unscale + clip + Adam + decay + 16-bit refresh for every parameter (``ub200_adamw_step``); the clip
coefficient is read from device memory, so a step never synchronises with the host.  The
encoder-layer gradients are read in place from the flat gradient arena (right where the NCCL
all-reduce left them).

Same surface as the reference optimizer: ``param_groups`` (list of dicts with ``params``, ``lr``,
``weight_decay``, ``betas``, ``eps``, ``correct_bias``) that the training loop mutates
(``train_vqa.py:207-214``), ``step()``, ``zero_grad()``, ``state_dict()`` / ``load_state_dict()``;
``build_optimizer`` groups parameters by name exactly as ``optim/misc.py:14-22``.
"""
import ctypes as C
import math

import torch

from . import _lib


def build_optimizer(model, opts):
    """optim/misc.py:12-37: no weight decay for names containing 'bias', 'LayerNorm.bias',
    'LayerNorm.weight'; betas / lr from opts (only the 'adamw' branch exists here)."""
    param_optimizer = list(model.named_parameters())
    no_decay = ["bias", "LayerNorm.bias", "LayerNorm.weight"]
    groups = [
        {"params": [p for n, p in param_optimizer if not any(nd in n for nd in no_decay)],
         "weight_decay": opts.weight_decay},
        {"params": [p for n, p in param_optimizer if any(nd in n for nd in no_decay)],
         "weight_decay": 0.0},
    ]
    if getattr(opts, "optim", "adamw") != "adamw":
        raise ValueError("invalid optimizer (libub200 implements adamw)")
    return FusedAdamW(groups, lr=opts.learning_rate, betas=tuple(opts.betas))


def scaler_table(entries):
    """Host image of a ub200_loss_scaler table: one (scale, unskipped, window, max_scale, min_scale)
    tuple per loss id -> float32 [n, 8] (the int32 fields are stored bit-cast, read them through
    .view(torch.int32)).  inv_scale starts at 1 / scale."""
    arr = (_lib.LossScalerEntry * len(entries))()
    for e, (scale, unskipped, window, max_scale, min_scale) in zip(arr, entries):
        e.scale, e.unskipped, e.inv_scale = scale, unskipped, 1.0 / scale
        e.window, e.max_scale, e.min_scale = window, max_scale, min_scale or 0.0
    raw = bytearray(C.string_at(C.addressof(arr), C.sizeof(arr)))
    return torch.frombuffer(raw, dtype=torch.float32).view(len(entries), C.sizeof(_lib.LossScalerEntry) // 4)


class DynamicLossScaler(object):
    """apex amp's dynamic loss scaler (``LossScaler``, dynamic mode; train_vqa.py:152,189-199), one
    entry per loss id like pre-training's ``num_losses=len(task2scaler)`` (pretrain.py:230-233), held
    in DEVICE memory at a fixed address (``self.table``, the C ABI's ``ub200_loss_scaler`` array).

    ``scale(loss, k)`` multiplies by the device scalar, ``FusedAdamW.step(grad_scale=scaler,
    loss_id=k)`` unscales by it and moves it after the overflow check, all on the device: a step
    never reads the scale on the host, so it can be captured in a CUDA graph and replayed while the
    scale changes.  Policy (apex): an overflowed step is skipped and halves the scale (not below
    `min_scale`, if given); after `scale_window` clean steps in a row the scale doubles, up to
    `max_scale`."""

    def __init__(self, num_losses=1, init_scale=2.**16, scale_window=2000, max_scale=2.**24, min_scale=None,
                 device=None):
        if num_losses < 1:
            raise ValueError("DynamicLossScaler: num_losses must be >= 1")
        if not init_scale > 0 or not max_scale > 0 or scale_window < 1:
            raise ValueError("DynamicLossScaler: need init_scale > 0, max_scale > 0 and scale_window >= 1")
        self.num_losses = int(num_losses)
        self.policy = (int(scale_window), float(max_scale), None if not min_scale else float(min_scale))
        host = scaler_table([(float(init_scale), 0) + self.policy] * self.num_losses)
        self.table = host.to(device if device is not None else torch.device("cuda", torch.cuda.current_device()))
        self._scales = [self.table[k, 0] for k in range(self.num_losses)]     # 0-d views, built once

    def _check_id(self, loss_id):
        if not 0 <= loss_id < self.num_losses:
            raise IndexError("DynamicLossScaler: loss_id %d out of range [0, %d)" % (loss_id, self.num_losses))

    def scale(self, loss, loss_id=0):
        """loss * current scale of `loss_id`, in fp32, as a device op (no host read)."""
        self._check_id(loss_id)
        return loss.float() * self._scales[loss_id]

    def loss_scale(self, loss_id=0):
        """Current scale of `loss_id` (host read: synchronises; for logging)."""
        self._check_id(loss_id)
        return float(self.table[loss_id, 0].item())

    def unskipped(self, loss_id=0):
        self._check_id(loss_id)
        return int(self.table.view(torch.int32)[loss_id, 1].item())

    def state_dict(self):
        """What apex's ``amp.state_dict()`` stores: {'loss_scaler<k>': {'loss_scale', 'unskipped'}}."""
        rows = self.table.cpu()
        ints = rows.view(torch.int32)
        return {"loss_scaler%d" % k: {"loss_scale": float(rows[k, 0]), "unskipped": int(ints[k, 1])}
                for k in range(self.num_losses)}

    def load_state_dict(self, sd):
        if len(sd) != self.num_losses:
            raise ValueError("DynamicLossScaler: state_dict has %d loss scalers, this one %d"
                             % (len(sd), self.num_losses))
        entries = [(float(sd["loss_scaler%d" % k]["loss_scale"]), int(sd["loss_scaler%d" % k]["unskipped"]))
                   + self.policy for k in range(self.num_losses)]
        self.table.copy_(scaler_table(entries))        # in place: the table keeps its address


def _owned_ranges(params):
    """For each parameter, the element ranges [lo, hi) of its storage that its own segment updates.

    Parameters may share storage: UniterForImageTextRetrieval.init_output() makes rank_output.weight and
    .bias views of row 1 of itm_output's.  Every element of model storage is updated by ONE segment per
    step, that of the innermost parameter covering it (of parameters with the same range, the first
    listed), so no two CTAs of one launch write the same address, and a view's elements follow the view's
    own gradient and moments.  The covering parameter's gradient over those elements is not used, and
    they are left out of its share of the gradient norm.  Storage that two parameters share only in part
    has no single owner and is refused."""
    spans = [(p.data_ptr(), p.data_ptr() + p.numel() * p.element_size(), p.element_size()) for p in params]
    out = []
    for i, (lo, hi, es) in enumerate(spans):
        holes = []
        for j, (lo2, hi2, es2) in enumerate(spans):
            if j == i or hi2 <= lo or hi <= lo2:
                continue
            inside, around = lo <= lo2 and hi2 <= hi, lo2 <= lo and hi <= hi2
            if not (inside or around) or es2 != es or (lo2 - lo) % es:
                raise RuntimeError("FusedAdamW: parameters %d and %d share storage in part; give each shared "
                                   "element one parameter" % (i, j))
            if inside and ((lo2, hi2) != (lo, hi) or j < i):
                holes.append(((lo2 - lo) // es, (hi2 - lo) // es))
        ranges, cur = [], 0
        for a, b in sorted(holes):
            if a > cur:
                ranges.append((cur, a))
            cur = max(cur, b)
        n = (hi - lo) // es
        if cur < n:
            ranges.append((cur, n))
        out.append(ranges)
    return out


class FusedAdamW(object):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-6, weight_decay=0.0,
                 correct_bias=True):
        if lr < 0.0:
            raise ValueError("Invalid learning rate: {} - should be >= 0.0".format(lr))
        if not 0.0 <= betas[0] < 1.0:
            raise ValueError("Invalid beta parameter: {} - should be in [0.0, 1.0[".format(betas[0]))
        if not 0.0 <= betas[1] < 1.0:
            raise ValueError("Invalid beta parameter: {} - should be in [0.0, 1.0[".format(betas[1]))
        if not 0.0 <= eps:
            raise ValueError("Invalid epsilon value: {} - should be >= 0.0".format(eps))
        defaults = dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, correct_bias=correct_bias)
        params = list(params)
        if params and not isinstance(params[0], dict):
            params = [{"params": params}]
        self.param_groups = []
        seen = set()
        for g in params:
            g = dict(g)
            g["params"] = [p for p in g["params"] if not (id(p) in seen or seen.add(id(p)))]
            for k, v in defaults.items():
                g.setdefault(k, v)
            self.param_groups.append(g)
        self.state = {}          # id(param) -> dict(step_offset, master, exp_avg, exp_avg_sq)
        self._tables = None      # device-resident segment table + bookkeeping (see _build_tables)
        self._dev_state = None   # int32 [4] on the device: step, found_inf, skipped, pad (ub200_adam_state)
        self._lr_dev = None
        self._lr_pinned = None
        self.last_sumsq = None   # device scalar: sum of squares of the (scaled) gradients

    # ------------------------------------------------------------------ state
    def _init_state(self, p, step_now):
        st = self.state.get(id(p))
        if st is None:
            st = dict(step_offset=step_now)
            self.state[id(p)] = st
        if "master" not in st:           # e.g. a reference AdamW train_state: step / exp_avg / exp_avg_sq only
            st["master"] = p.detach().float().clone()
        for k in ("exp_avg", "exp_avg_sq"):
            t = st.get(k)
            if t is None:
                st[k] = torch.zeros(p.shape, device=p.device, dtype=torch.float32)
            elif t.dtype != torch.float32 or not t.is_contiguous() or t.device != p.device:
                st[k] = t.to(device=p.device, dtype=torch.float32).contiguous()
        m = st["master"]
        if m.dtype != torch.float32 or not m.is_contiguous() or m.device != p.device:
            st["master"] = m.to(device=p.device, dtype=torch.float32).contiguous()
        return st

    def zero_grad(self, set_to_none=True):
        for g in self.param_groups:
            for p in g["params"]:
                if set_to_none:
                    p.grad = None
                elif p.grad is not None:
                    p.grad.zero_()

    def _applied_steps(self):
        """Optimizer steps actually applied so far (reads the device counter: synchronises)."""
        return int(self._dev_state[0].item()) if self._dev_state is not None else 0

    @property
    def found_inf(self):
        """Device int32 scalar: 1 iff the last step() saw a non-finite gradient norm and was skipped
        (what apex's dynamic loss scaler reads to lower the scale) — no host synchronisation."""
        return None if self._dev_state is None else self._dev_state[1]

    def skipped_steps(self):
        return int(self._dev_state[2].item()) if self._dev_state is not None else 0

    def state_dict(self):
        packed, idx = {}, 0
        groups = []
        applied = self._applied_steps()
        for g in self.param_groups:
            ids = []
            for p in g["params"]:
                st = self.state.get(id(p))
                if st is not None:
                    d = {k: (v.clone() if torch.is_tensor(v) else v) for k, v in st.items() if k != "step_offset"}
                    d["step"] = applied - st.get("step_offset", 0)
                    packed[idx] = d
                ids.append(idx)
                idx += 1
            groups.append({k: (ids if k == "params" else v) for k, v in g.items()})
        return {"state": packed, "param_groups": groups}

    def load_state_dict(self, sd):
        """Accepts its own state_dict and a reference AdamW one (optim/adamw.py: step / exp_avg /
        exp_avg_sq, possibly 16-bit, no master): masters are rebuilt from the parameters and the
        moments cast to contiguous fp32 on first use (_init_state)."""
        idx = 0
        steps = []
        loaded = []
        for g, sg in zip(self.param_groups, sd["param_groups"]):
            for k, v in sg.items():
                if k != "params":
                    g[k] = v
            for p in g["params"]:
                st = sd["state"].get(idx)
                if st is not None:
                    d = {k: (v.to(p.device).clone() if torch.is_tensor(v) else v) for k, v in st.items()}
                    steps.append(int(d.pop("step", 0)))
                    loaded.append((p, d, steps[-1]))
                idx += 1
        top = max(steps) if steps else 0
        for p, d, stp in loaded:
            d["step_offset"] = top - stp
            self.state[id(p)] = d
        self._tables = None
        if loaded:
            dev = loaded[0][0].device
            if dev.type == "cuda":
                self._dev_state = torch.tensor([top, 0, 0, 0], device=dev, dtype=torch.int32)

    # ------------------------------------------------------------------ device tables
    def _table_key(self):
        key = []
        for gi, g in enumerate(self.param_groups):
            key.append((gi, g["weight_decay"], bool(g["correct_bias"]), tuple(g["betas"]), g["eps"]))
            for p in g["params"]:
                if p.grad is not None:
                    key.append((id(p), p.grad.data_ptr(), p.data_ptr(), p.grad.dtype, p.dtype))
        return tuple(key)

    def _build_tables(self, key):
        """Segment table (one entry per range of a parameter with a gradient that the parameter owns, see
        _owned_ranges: one per parameter unless parameters share storage), CTA prefix sums, per-group
        learning rates and the optimizer state counters, all in DEVICE memory at fixed addresses, so
        that a step is three launches with constant arguments (capturable in a CUDA graph).  Rebuilt
        only when the set of (parameter, gradient buffer) pairs changes."""
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError("FusedAdamW: the set of gradients changed inside a CUDA-graph capture; run one "
                               "eager step() first (GraphedStep's warm-up does)")
        lib = _lib.load()
        chunk = lib.ub200_adam_chunk()
        segs, starts, keep = [], [0], []
        dev = None
        betas = eps = None
        for g in self.param_groups:
            for p in g["params"]:
                if p.grad is not None:
                    dev = p.device
        if dev is None:
            return None
        if self._dev_state is None or self._dev_state.device != dev:
            self._dev_state = torch.zeros(4, device=dev, dtype=torch.int32)
        step_now = self._applied_steps()
        with_grad = []
        for gi, g in enumerate(self.param_groups):
            b1, b2 = g["betas"]
            if betas is None:
                betas, eps = (b1, b2), g["eps"]
            elif (b1, b2) != betas or g["eps"] != eps:
                raise ValueError("FusedAdamW: betas / eps must be the same in every param group")
            for p in g["params"]:
                if p.grad is None:
                    continue
                if not p.is_cuda:
                    raise RuntimeError("FusedAdamW runs on CUDA parameters only (no CPU fallback)")
                if p.grad.is_sparse:
                    raise RuntimeError("Adam does not support sparse gradients")
                if not p.is_contiguous() or not p.grad.is_contiguous():
                    raise RuntimeError("FusedAdamW needs contiguous parameters and gradients")
                with_grad.append((gi, g, p))
        owned = _owned_ranges([p for _, _, p in with_grad])
        for (gi, g, p), ranges in zip(with_grad, owned):
            st = self._init_state(p, step_now)
            ge, me = p.grad.element_size(), p.element_size()
            for lo, hi in ranges:
                segs.append(_lib.AdamSegment(
                    grad=p.grad.data_ptr() + lo * ge, master=st["master"].data_ptr() + lo * 4,
                    exp_avg=st["exp_avg"].data_ptr() + lo * 4, exp_avg_sq=st["exp_avg_sq"].data_ptr() + lo * 4,
                    model=p.data_ptr() + lo * me, n=hi - lo,
                    step_size=0.0, lr_wd=0.0,
                    grad_dtype=_lib.dtype_code(p.grad.dtype, allow_f32=True),
                    model_dtype=_lib.dtype_code(p.dtype, allow_f32=True),
                    weight_decay=float(g["weight_decay"]), group=gi, step_offset=int(st["step_offset"]),
                    flags=1 if g["correct_bias"] else 0))
                starts.append(starts[-1] + (hi - lo + chunk - 1) // chunk)
            keep.append(p.grad)
        if not segs:
            return None
        nseg, nblocks = len(segs), starts[-1]
        arr = (_lib.AdamSegment * nseg)(*segs)
        host = torch.frombuffer(bytearray(C.string_at(C.addressof(arr), C.sizeof(arr))), dtype=torch.uint8)
        segs_dev = host.pin_memory().to(dev, non_blocking=True)
        starts_dev = torch.tensor(starts, dtype=torch.int32).pin_memory().to(dev, non_blocking=True)
        self._lr_dev = torch.zeros(len(self.param_groups), device=dev, dtype=torch.float32)
        self._lr_pinned = [torch.zeros(len(self.param_groups), dtype=torch.float32).pin_memory() for _ in range(4)]
        self._lr_slot = 0
        self._lr_events = [None] * 4
        self._lr_last = None
        self.last_sumsq = torch.zeros(1, device=dev, dtype=torch.float32)
        # one fp32 partial per block: the fixed-order sum of squares of the deterministic mode
        sumsq_ws = torch.empty(max(_lib.load().ub200_grad_sumsq_workspace_bytes(nblocks) // 4, 1), device=dev,
                               dtype=torch.float32)
        self._tables = dict(key=key, segs=segs_dev, starts=starts_dev, nseg=nseg, nblocks=nblocks,
                            betas=betas, eps=eps, keep=keep, sumsq_ws=sumsq_ws)
        return self._tables

    def prepare(self):
        """Build the device tables for the current set of gradients without stepping (GraphedStep calls
        this before capturing a step that contains the optimizer)."""
        key = self._table_key()
        if self._tables is None or self._tables["key"] != key:
            self._build_tables(key)
        self.sync_lr()

    def sync_lr(self):
        """Ship param_groups[*]['lr'] to the device (the training loop mutates it every step,
        train_vqa.py:207-214).  step() does this itself except inside a CUDA-graph capture: a captured
        step reads the learning rate from device memory, so call sync_lr() before each replay."""
        if self._lr_dev is None:
            return
        lrs = [float(g["lr"]) for g in self.param_groups]
        if lrs == self._lr_last:
            return
        k = self._lr_slot
        self._lr_slot = (k + 1) % len(self._lr_pinned)
        if self._lr_events[k] is not None:
            self._lr_events[k].synchronize()
        self._lr_pinned[k].copy_(torch.tensor(lrs, dtype=torch.float32))
        self._lr_dev.copy_(self._lr_pinned[k], non_blocking=True)
        ev = self._lr_events[k] or torch.cuda.Event()
        ev.record()
        self._lr_events[k] = ev
        self._lr_last = lrs

    # ------------------------------------------------------------------ step
    @torch.no_grad()
    def step(self, grad_scale=1.0, max_grad_norm=-1.0, loss_id=0):
        """One optimizer step over every parameter that has a gradient: global gradient norm
        (always — it is also the overflow detector), device-side bookkeeping, fused update.

        grad_scale: the loss scale the gradients carry (they are multiplied by 1 / grad_scale), or a
        DynamicLossScaler whose entry `loss_id` scaled the loss: the unscale factor is then read from
        device memory and the scaler is updated on the device after the overflow check;
        max_grad_norm > 0: clip the global norm of the unscaled gradients like ``clip_grad_norm_``
        (the norm itself stays on the device: ``self.last_sumsq``).  A non-finite norm (fp16
        overflow) SKIPS the step on the device — masters, moments, weights and the step count stay
        untouched and ``self.found_inf`` is set — like apex's dynamic loss scaler does.
        Under torch.use_deterministic_algorithms the gradient norm is summed in a fixed order."""
        with _lib.library_mode(_lib.select_mode()):
            return self._step(grad_scale, max_grad_norm, loss_id)

    def _step(self, grad_scale, max_grad_norm, loss_id):
        lib = _lib.load()
        if isinstance(grad_scale, DynamicLossScaler):
            return self._step_scaled(lib, grad_scale, int(loss_id), max_grad_norm)
        key = self._table_key()
        T = self._tables
        if T is None or T["key"] != key:
            T = self._build_tables(key)
            if T is None:
                return None
        if not torch.cuda.is_current_stream_capturing():
            self.sync_lr()
        stream = _lib.current_stream()
        self.last_sumsq.zero_()
        self._grad_sumsq(lib, T, stream)
        _lib.check(lib.ub200_adam_prep(self.last_sumsq.data_ptr(), self._dev_state.data_ptr(), stream))
        clip = max_grad_norm is not None and max_grad_norm > 0
        _lib.check(lib.ub200_adamw_step(T["segs"].data_ptr(), T["starts"].data_ptr(), T["nseg"], T["nblocks"],
                                        T["betas"][0], T["betas"][1], T["eps"], 1.0 / float(grad_scale),
                                        float(max_grad_norm) if clip else -1.0, self.last_sumsq.data_ptr(),
                                        self._dev_state.data_ptr(), self._lr_dev.data_ptr(), stream))
        return None

    def _grad_sumsq(self, lib, T, stream):
        ws = T["sumsq_ws"]
        _lib.check(lib.ub200_grad_sumsq_ws(T["segs"].data_ptr(), T["starts"].data_ptr(), T["nseg"], T["nblocks"],
                                           self.last_sumsq.data_ptr(), ws.data_ptr(), ws.numel() * 4, stream))

    def _step_scaled(self, lib, scaler, loss_id, max_grad_norm):
        scaler._check_id(loss_id)
        key = self._table_key()
        T = self._tables
        if T is None or T["key"] != key:
            T = self._build_tables(key)
            if T is None:
                return None
        if scaler.table.device != self._dev_state.device:
            raise RuntimeError("FusedAdamW: the loss scaler lives on %s, the parameters on %s"
                               % (scaler.table.device, self._dev_state.device))
        if not torch.cuda.is_current_stream_capturing():
            self.sync_lr()
        stream = _lib.current_stream()
        self.last_sumsq.zero_()
        self._grad_sumsq(lib, T, stream)
        _lib.check(lib.ub200_adam_prep_scaled(self.last_sumsq.data_ptr(), self._dev_state.data_ptr(),
                                              scaler.table.data_ptr(), loss_id, stream))
        clip = max_grad_norm is not None and max_grad_norm > 0
        _lib.check(lib.ub200_adamw_step_scaled(T["segs"].data_ptr(), T["starts"].data_ptr(), T["nseg"],
                                               T["nblocks"], T["betas"][0], T["betas"][1], T["eps"],
                                               float(max_grad_norm) if clip else -1.0, self.last_sumsq.data_ptr(),
                                               self._dev_state.data_ptr(), self._lr_dev.data_ptr(),
                                               scaler.table.data_ptr(), loss_id, stream))
        return None
