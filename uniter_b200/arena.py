"""One flat gradient arena for every parameter under a root module.

Replaces the flat-buffer round trip of the reference's gradient exchange
(utils/distributed.py:16-43: copy every grad into one buffer -> hvd.allreduce_ -> copy back):
here every parameter's ``.grad`` IS a view of one flat 16-bit buffer for its whole life, the
library's wgrad / scatter / column-sum kernels write (or accumulate) straight into those views,
and the data-parallel reducer all-reduces slices of the buffer in place.

Layout (element offsets, every segment 16-byte aligned), in the order the backward pass
completes them so that the reducer can ship a slice as soon as it is final:

    [ head : parameters outside any UniterModel (task heads), named_parameters order      ]
    [ per UniterModel:  pooler | encoder layers 0..NL-1 (library layout) | front-end       ]

* encoder layer l (``ub200_layer_grads``): dWqkv[3H,H] dWo[H,H] dW1[I,H] dW2[H,I] then the small
  gradients in ``SmallLayout`` order (dbqkv dbo dln1_g dln1_b db1 db2 dln2_g dln2_b);
* front-end: word_embeddings[V,H] img_linear.weight[H,D] mask_embedding[2,D] then the small
  section in the order of the fp32 staging buffer of ``_EmbedFront.backward`` (one conversion
  launch): position[P,H] ln_txt(g,b) | token_type[Ty,H] | ln_out(g,b) ln_img(g,b) ln_pos(g,b)
  img_linear.bias pos_linear.bias pos_linear.weight[H,7]  (text-only | shared | image-only).

Write protocol.  A library writer calls ``claim(params)`` before touching the views of a group of
parameters; it returns whether to ACCUMULATE (the views already hold partial gradients of the
current step) or to OVERWRITE.  "Current step" is defined in one of two ways:
  * implicit (the reference's loop: ``optimizer.zero_grad()`` then backward): a parameter whose
    ``.grad`` is None is fresh; the writer attaches the view as ``.grad``;
  * explicit (``begin_step()``; used by GraphedStep, where ``.grad`` can never be None because the
    captured graph needs fixed addresses): every library-managed parameter is marked fresh and the
    autograd-managed slices are zeroed (autograd then accumulates in place).
"""
import torch


def _align8(n):
    return (n + 7) // 8 * 8


class GradArena(object):
    def __init__(self, root):
        from .model import UniterModel
        self.root = root
        self.encoders = [m for m in root.modules() if isinstance(m, UniterModel)]
        enc_param_ids = set()
        for e in self.encoders:
            if e.encoder.layer[0].attention.self.query.weight.is_cuda:
                e._weight_table()                               # re-home q/k/v, validate dtype
            enc_param_ids.update(id(p) for p in e.parameters())
        seen, head = set(), []
        for name, p in root.named_parameters():
            if id(p) in seen or id(p) in enc_param_ids:
                continue
            seen.add(id(p))
            head.append((name, p))
        ref = self.encoders[0].encoder.layer[0].attention.self.query.weight if self.encoders \
            else next(root.parameters())
        self.dtype, self.device = ref.dtype, ref.device
        for name, p in head:
            if p.dtype != self.dtype or p.device != self.device:
                raise RuntimeError("GradArena: parameter %s is %s on %s, the encoder is %s on %s — convert "
                                   "the whole module with .to(device, dtype) first"
                                   % (name, p.dtype, p.device, self.dtype, self.device))
        # ---------------------------------------------------------------- plan
        off = 0
        plan = []                                  # (param, offset, numel)
        self.segments = {}                         # name -> (lo, hi) element range
        lo = off
        for name, p in head:
            plan.append((p, off, p.numel()))
            off += _align8(p.numel())
        self.segments["head"] = (lo, off)
        self._enc_plans = []
        for ei, e in enumerate(self.encoders):
            ep = e._plan_arena(off)                # dict: plan entries, segments, total
            plan += ep["plan"]
            for k, v in ep["segments"].items():
                self.segments["enc%d.%s" % (ei, k)] = v
            off = ep["end"]
            self._enc_plans.append(ep)
        self.numel = off
        self.flat = torch.zeros(max(off, 8), device=self.device, dtype=self.dtype)
        # ---------------------------------------------------------------- views
        self._views = {}
        self._offsets = {}
        self.managed = set()                       # ids of parameters whose grads the library writes
        for p, o, n in plan:
            v = self.flat[o:o + n].view(p.shape)
            self._views[id(p)] = v
            self._offsets[id(p)] = o
            p._ub_grad_view = v
            p._ub_arena = self
        for e, ep in zip(self.encoders, self._enc_plans):
            e._bind_arena(self, ep)
        self.step_mode = False
        self._fresh = set()
        # the planned parameters themselves: their ids key the views, so none of them may be freed and
        # its id reused by another tensor while this arena exists
        self._planned = [p for p, _, _ in plan]
        self._stale = False
        root._ub_arena = self

    # ------------------------------------------------------------------ lookup
    @staticmethod
    def of(module):
        """The arena a module was attached to (searching up is the caller's job), or None."""
        return getattr(module, "_ub_arena", None)

    @staticmethod
    def attach(root):
        a = getattr(root, "_ub_arena", None)
        if a is not None and a._still_valid():
            return a
        return GradArena(root)

    @staticmethod
    def for_params(root, sentinel):
        """The arena `sentinel` (a parameter under `root`) currently lives in; a new arena over
        `root` when it has none (or a stale one, e.g. after .half())."""
        a = getattr(sentinel, "_ub_arena", None)
        if a is None or not a._still_valid() or id(sentinel) not in a._views or \
                a._views[id(sentinel)].dtype != sentinel.dtype:
            a = GradArena(root)
        return a

    def invalidate(self):
        """Mark this arena as describing a parameter set that no longer exists (a parameter was replaced,
        e.g. by the VCR head's init_type_embedding / init_word_embedding).  The next backward builds a
        fresh arena; a GraphedStep built over this one refuses to run."""
        self._stale = True

    def _still_valid(self):
        if self._stale:
            return False
        for e in self.encoders:
            p = e.encoder.layer[0].attention.self.query.weight
            if p.dtype != self.dtype or p.device != self.device:
                return False
        return True

    def view(self, p):
        v = self._views.get(id(p))
        if v is None or v.shape != p.shape:
            raise RuntimeError("GradArena: a parameter of shape %s has no view in this gradient arena (was it "
                               "replaced after the arena was built?)" % (tuple(p.shape),))
        return v

    def segment(self, name):
        lo, hi = self.segments[name]
        return self.flat[lo:hi]

    def mark_managed(self, params):
        self.managed.update(id(p) for p in params)

    # ------------------------------------------------------------------ write protocol
    def _is_live(self, p):
        v = self._views[id(p)]
        if self.step_mode:
            return id(p) not in self._fresh
        g = p.grad
        if g is None:
            return False
        if g.data_ptr() == v.data_ptr():
            return True
        v.copy_(g)                 # a foreign gradient tensor (autograd assigned it first): fold it in
        return True

    def claim(self, params):
        """About to write the gradients of `params` as one group.  Returns True when the group must
        ACCUMULATE; fresh members of an accumulating group are zeroed first.  Attaches the views."""
        params = [p for p in params if p is not None and p.requires_grad]
        live = [self._is_live(p) for p in params]
        acc = any(live)
        for p, l in zip(params, live):
            v = self._views[id(p)]
            if acc and not l:
                v.zero_()
            if p.grad is None or p.grad.data_ptr() != v.data_ptr():
                p.grad = v
            self._fresh.discard(id(p))
        return acc

    def begin_step(self, accumulate=False, zero_all=False):
        """Explicit step protocol: call before the forward of every (micro-)step.
        accumulate=False: library-managed gradients will be overwritten by their first writer, the
        autograd-managed slices are zeroed now; every parameter's .grad is (re)attached.
        zero_all=True: zero the WHOLE arena and let every writer accumulate — needed when autograd
        also contributes to library-managed parameters (e.g. the reference's torch MLM decoder tied to
        the word embeddings)."""
        self.step_mode = True
        all_ids = list(self._views.keys())
        if accumulate:
            self._fresh = set()          # after the window's first step every view is live (or zero)
        if not accumulate:
            if zero_all:
                self.flat.zero_()
                self._fresh = set()
            else:
                self._fresh = set(i for i in all_ids if i in self.managed)
                self._zero_unmanaged()
        for p in self._params():
            v = self._views[id(p)]
            if p.requires_grad and (p.grad is None or p.grad.data_ptr() != v.data_ptr()):
                p.grad = v

    def finish_step(self):
        """Explicit protocol, after the backward: library-managed parameters that no writer claimed in
        this step (a head the step's task does not use, the mask embedding without img_masks, ...)
        still hold whatever an earlier step left in their views — zero them, so that every .grad is
        either this step's gradient or exactly zero (their .grad cannot be None: fixed addresses)."""
        if not self.step_mode:
            return
        for p in self._params():
            if id(p) in self._fresh:
                self._views[id(p)].zero_()
        self._fresh = set()

    def end_step_mode(self):
        self.step_mode = False
        self._fresh = set()

    def _params(self):
        seen = set()
        for p in self.root.parameters():
            if id(p) not in seen:
                seen.add(id(p))
                yield p

    def _zero_unmanaged(self):
        """Zero the autograd-managed views (contiguous runs are merged into single memsets)."""
        runs = []
        for p in self._params():
            if id(p) in self.managed:
                continue
            v = self._views[id(p)]
            lo = (v.data_ptr() - self.flat.data_ptr()) // self.flat.element_size()
            hi = lo + _align8(v.numel())
            if runs and runs[-1][1] == lo:
                runs[-1][1] = hi
            else:
                runs.append([lo, hi])
        for lo, hi in runs:
            self.flat[lo:min(hi, self.flat.numel())].zero_()

    def fold_foreign_range(self, lo, hi):
        """fold_foreign() restricted to parameters whose views start inside [lo, hi)."""
        n = 0
        for p in self._params():
            g = p.grad
            if g is None or not (lo <= self._offsets[id(p)] < hi):
                continue
            v = self._views[id(p)]
            if g.data_ptr() != v.data_ptr():
                v.copy_(g)
                p.grad = v
                n += 1
        return n

    def fold_foreign(self):
        """Implicit protocol: gradients autograd allocated itself (.grad was None when it ran) are
        copied into their views and re-pointed, so that the whole model's gradient is the flat buffer
        (what the reducer / the fused optimizer read).  Returns the number of tensors folded."""
        n = 0
        for p in self._params():
            g = p.grad
            if g is None:
                continue
            v = self._views[id(p)]
            if g.data_ptr() != v.data_ptr():
                v.copy_(g)
                p.grad = v
                n += 1
        return n
