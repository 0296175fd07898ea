"""Adam over flat buffers (the `optimizer.step()` of run_model.py:101-109, torch.optim.Adam semantics).

`FlatAdam(params, lr, groups=...)` re-homes the parameters it is given in ONE contiguous fp32 buffer (every
`p.data` becomes a view of it -- names, shapes, `state_dict()` and `load_state_dict()` are unchanged) and keeps
buffers of the same layout next to it: the gradients `g`, Adam's `m` and `v`, and a bf16 mirror of the parameters.
One `fira_adam_flat` launch updates everything (csrc/optim.cu) and refreshes the mirror.  What the layout buys:

  * the step is ONE memory-bound kernel instead of torch's multi-tensor launches over 264 tensors;
  * the bf16 GEMM operands of the throughput mode are views of the mirror: no per-step cast kernels;
  * `groups` of parameters laid out back to back (q|k, q|k|v, the 12 cross-attention k|v projections) make the
    concatenated weights of the fused projections plain views (`cat_rows`): no per-step `torch.cat`;
  * backward passes write parameter gradients straight into views of `g` (`grad_dest`), so neither the optimizer nor
    the data-parallel all-reduce needs a packing pass: the all-reduce runs on `g` itself.

`max_grad_norm=c` clips the gradient's global norm before Adam (torch.nn.utils.clip_grad_norm_) and skips steps whose
gradient is not finite, on the device (csrc/optim.cu): a float64 sum of squares per buffer, one finalize kernel, then
the Adam launch scaled by the coefficient.  `ClipGroup(optims)` takes one norm over several instances (the two halves
of engine.GraphedTrainStep's pair); a FlatAdam alone is a group of one.
"""
import weakref

import torch

from . import _lib

ALIGN = 64          # elements: every tensor starts on a 256-byte (fp32) / 128-byte (bf16) boundary


class _Slot:
    __slots__ = ("owner", "off", "numel")

    def __init__(self, owner, off, numel):
        self.owner, self.off, self.numel = weakref.ref(owner), off, numel


_SLOTS = {}          # (data_ptr, numel) of a re-homed parameter or of a cat_rows view -> _Slot


def _lookup(t):
    key = (t.data_ptr(), t.numel())
    s = _SLOTS.get(key)
    if s is None:
        return None, None
    o = s.owner()
    if o is None or o.p.data_ptr() + 4 * s.off != key[0]:
        del _SLOTS[key]                                       # the optimizer is gone: the address means nothing any more
        return None, None
    return o, s


def mirror_of(t):
    """bf16 view of a re-homed parameter / cat_rows view while the mirror is fresh, else None"""
    o, s = _lookup(t)
    if o is None or not o.fresh:
        return None
    return o.p16[s.off:s.off + s.numel].view(t.shape)


def grad_dest(ts, shape):
    """A NEW view, of shape `shape`, of the flat gradient buffer over the parameters `ts` (which must lie back to back
    in one FlatAdam layout), or None.  Backward passes write gradients there and hand (slices of) the view to autograd,
    which adopts them as `.grad` -- no copy, no packing pass.  The buffer was zero-filled by zero_grad().  Each span is
    handed out once per zero_grad(): a second backward before the next zero_grad() gets None, allocates as usual and lets
    autograd accumulate."""
    o0, s0 = _lookup(ts[0])
    if o0 is None or not o0.direct:
        return None
    off = s0.off
    for t in ts:
        o, s = _lookup(t)
        if o is not o0 or s.off != off:
            return None
        off += s.numel
    if s0.off in o0.handed:
        return None
    o0.handed.add(s0.off)
    return o0.g[s0.off:off].view(shape)


def cat_rows(ts):
    """torch.cat(ts, 0) -- as a zero-copy view when the tensors are adjacent parameters of one flat buffer"""
    o0, s0 = _lookup(ts[0])
    if o0 is not None:
        off = s0.off
        for t in ts:
            o, s = _lookup(t)
            if o is not o0 or s.off != off or t.shape[1:] != ts[0].shape[1:]:
                break
            off += s.numel
        else:
            n = off - s0.off
            view = o0.p[s0.off:off].view((sum(t.shape[0] for t in ts),) + tuple(ts[0].shape[1:]))
            _SLOTS[(view.data_ptr(), n)] = _Slot(o0, s0.off, n)
            return view
    return torch.cat(ts, 0)


def plan_layout(params, groups=()):
    """Offsets (in elements) of `params` inside one flat buffer and the buffer length: the members of every group whose
    parameters are all present lie back to back, in the group's order; every group / ungrouped tensor starts on an
    ALIGN-element boundary; the length is a multiple of ALIGN.  Pure host logic (works on any tensors)."""
    mine = {id(p) for p in params}
    order, seen = [], set()
    for grp in groups:                                   # adjacency groups first, members back to back
        if all(id(p) in mine for p in grp) and not any(id(p) in seen for p in grp):
            order.append(list(grp))
            seen.update(id(p) for p in grp)
    for p in params:
        if id(p) not in seen:
            order.append([p])
            seen.add(id(p))
    offs, off = {}, 0
    for grp in order:
        off = (off + ALIGN - 1) // ALIGN * ALIGN
        for p in grp:
            if len(grp) > 1 and p.numel() % 8:
                raise ValueError("FlatAdam: grouped parameters must have a multiple of 8 elements")
            offs[id(p)] = off
            off += p.numel()
    return [offs[id(p)] for p in params], (off + ALIGN - 1) // ALIGN * ALIGN


def check_ema_decay(d):
    """d as a float; ValueError unless 0 < d < 1 (finite)"""
    try:
        d = float(d)
    except (TypeError, ValueError):
        raise ValueError(f"ema_decay must be a number in (0, 1), got {d!r}")
    if not 0.0 < d < 1.0:
        raise ValueError(f"ema_decay must be a number in (0, 1), got {d!r}")
    return d


def check_max_grad_norm(c):
    """c as a float; ValueError unless 0 < c <= inf (inf: the norm is monitored and non-finite steps are skipped, but
    no step is clipped)"""
    try:
        c = float(c)
    except (TypeError, ValueError):
        raise ValueError(f"max_grad_norm must be a positive number or inf, got {c!r}")
    if not c > 0.0:                                          # NaN fails the comparison
        raise ValueError(f"max_grad_norm must be a positive number or inf, got {c!r}")
    return c


CLIP_NORM, CLIP_COEF, CLIP_TAKEN, CLIP_CLIPPED, CLIP_SKIPPED = range(5)       # FIRA_CLIP_* (include/fira_b200.h)


class ClipGroup:
    """One global gradient norm over the FlatAdam instances `optims` (all built with the same max_grad_norm c).  Per step:
    `sumsq(o)` for every member once its gradients are final (any order, any stream), then `finish()`: the finalize
    kernel (norm, coefficient, skip flag, counters, every member's step counter) and every member's clipped Adam launch.
    `step()` does all of it in one go.  `grad_norm`, `clipped` and `skipped` are device scalars (float64 views of the
    state), read without a synchronisation inside the step.  Members must share `grad_scale` (or have none)."""

    def __init__(self, optims):
        optims = list(optims)
        if not optims or not all(isinstance(o, FlatAdam) for o in optims):
            raise ValueError("ClipGroup: needs FlatAdam instances")
        cs = {o.max_grad_norm for o in optims}
        if None in cs or len(cs) != 1:
            raise ValueError(f"ClipGroup: every member needs the same max_grad_norm, got {[o.max_grad_norm for o in optims]}")
        self.members = optims
        self.max_grad_norm = cs.pop()
        dev = optims[0].p.device
        counts = [_lib.lib().fira_grad_sumsq_blocks(o.n) for o in optims]
        self.partials = torch.zeros(sum(counts), dtype=torch.float64, device=dev)
        self._slot, off = {}, 0
        for o, k in zip(optims, counts):
            self._slot[id(o)] = self.partials[off:off + k]
            off += k
        self.state = torch.tensor([0.0, 1.0, 1.0, 0.0, 0.0], dtype=torch.float64, device=dev)
        # the members' step counters, advanced by the finalize kernel on a taken step only
        self.steps = torch.tensor([o.step_t.data_ptr() for o in optims], dtype=torch.int64, device=dev)
        for o in optims:
            o.clip = self

    @property
    def grad_norm(self):
        """the last step's gradient norm sqrt(sum g^2) / grad_scale (non-finite on a skipped step)"""
        return self.state[CLIP_NORM]

    @property
    def clipped(self):
        """steps whose gradient was scaled down (coefficient < 1)"""
        return self.state[CLIP_CLIPPED]

    @property
    def skipped(self):
        """steps skipped because the gradient was not finite"""
        return self.state[CLIP_SKIPPED]

    def sumsq(self, o):
        """member o's gradients are final: gather them into its flat buffer and launch its sum of squares"""
        o.gather_grads()
        o.direct = False                                      # g now holds this step's gradients
        slot = self._slot[id(o)]
        _lib.call("fira_grad_sumsq", o.g.data_ptr(), o.n, slot.data_ptr(), torch.cuda.current_stream().cuda_stream)

    def finish(self):
        """every member's sumsq() is done (on this stream or joined into it): finalize, then every clipped Adam launch"""
        scale = self.members[0].grad_scale
        if any(o.grad_scale is not scale for o in self.members):
            raise RuntimeError("ClipGroup: the members must share grad_scale")
        stream = torch.cuda.current_stream().cuda_stream
        _lib.call("fira_grad_clip_finalize", self.partials.data_ptr(), self.partials.numel(),
                  scale.data_ptr() if scale is not None else None, self.max_grad_norm, self.state.data_ptr(),
                  self.steps.data_ptr(), len(self.members), stream)
        for o in self.members:
            o._adam_clip(self.state)

    def step(self):
        for o in self.members:
            self.sumsq(o)
        self.finish()


class _EmaMirror:
    """The EMA buffer of one FlatAdam as the owner of a shadow model's parameters (ema_model): `p` is the EMA, `p16` its
    own bf16 mirror, refreshed on demand by ensure_fresh -- what mirror_of / cat_rows look up.  `moved()` marks the mirror
    stale and bumps `decoder.weights_epoch` of every shadow model, so weight caches keyed on weights_key re-read."""

    def __init__(self, opt):
        self.p, self.n = opt.ema, opt.n
        self.p16 = torch.zeros(self.n, dtype=torch.bfloat16, device=opt.ema.device)
        self.fresh = False
        self.direct = False                                   # never a gradient destination (grad_dest)
        self.models = weakref.WeakSet()

    def sync_mirror(self):
        _lib.call("fira_cast_bf16", self.p.data_ptr(), self.p16.data_ptr(), self.n, torch.cuda.current_stream().cuda_stream)
        self.fresh = True

    def moved(self):
        self.fresh = False
        for m in self.models:
            m.decoder.weights_epoch = getattr(m.decoder, "weights_epoch", 0) + 1


class FlatAdam:
    """torch.optim.Adam(params, lr, betas, eps) on flat buffers; `step()` is one kernel launch (capturable).
    ema_decay: keep `ema`, the exponential moving average of the parameters, updated in the same launch (None = off).
    max_grad_norm: clip the gradient's global norm to it and skip non-finite steps (None = off; see ClipGroup): `step()`
    is then three launches, and `clip` the group this instance belongs to."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, groups=(), ema_decay=None, max_grad_norm=None):
        self.params = [p for p in params if p.requires_grad]
        if not self.params:
            raise ValueError("FlatAdam: no parameters")
        dev = self.params[0].device
        if dev.type != "cuda":
            raise _lib.FiraLibraryError("FlatAdam: parameters must live on a CUDA device (no CPU path)")
        self.lr, self.betas, self.eps = float(lr), (float(betas[0]), float(betas[1])), float(eps)
        self.offsets, self.n = plan_layout(self.params, groups)
        f32 = dict(dtype=torch.float32, device=dev)
        self.p = torch.zeros(self.n, **f32)
        self.g = torch.zeros(self.n, **f32)
        self.m = torch.zeros(self.n, **f32)
        self.v = torch.zeros(self.n, **f32)
        self.p16 = torch.zeros(self.n, dtype=torch.bfloat16, device=dev)
        self.step_t = torch.zeros((), **f32)
        self.grad_scale = None                                # device fp32 scalar: gradients are divided by it
        self.fresh = False                                    # the bf16 mirror equals the parameters
        self.direct = False                                   # g is zero-filled and may be written by backward passes
        self.handed = set()
        with torch.no_grad():
            for p, o in zip(self.params, self.offsets):
                view = self.p[o:o + p.numel()].view(p.shape)
                view.copy_(p.data)
                p.data = view
                _SLOTS[(view.data_ptr(), p.numel())] = _Slot(self, o, p.numel())
        self.gviews = [self.g[o:o + p.numel()].view(p.shape) for p, o in zip(self.params, self.offsets)]
        self.sync_mirror()
        self.ema_decay = None if ema_decay is None else check_ema_decay(ema_decay)
        self.ema = None if ema_decay is None else torch.empty_like(self.p)
        self._ema_mirror = None                               # created by ema_model
        if self.ema is not None:
            self.reset_ema()
        self.max_grad_norm = None if max_grad_norm is None else check_max_grad_norm(max_grad_norm)
        self.clip = None
        if self.max_grad_norm is not None:
            ClipGroup([self])

    def reset_ema(self):
        """ema <- the parameters"""
        self.ema.copy_(self.p)
        self.ema_moved()

    def ema_moved(self):
        """The EMA moved (step(), a graph replay of a captured step(), load_state_dict): shadow models re-read it."""
        if self._ema_mirror is not None:
            self._ema_mirror.moved()

    def ema_mirror(self):
        if self.ema is None:
            raise ValueError("FlatAdam: no EMA (built without ema_decay)")
        if self._ema_mirror is None:
            self._ema_mirror = _EmaMirror(self)
        return self._ema_mirror

    def sync_mirror(self):
        """bf16 mirror <- parameters (after load_state_dict / any update that did not go through step())"""
        _lib.call("fira_cast_bf16", self.p.data_ptr(), self.p16.data_ptr(), self.n, torch.cuda.current_stream().cuda_stream)
        self.fresh = True

    # ------------------------------------------------------------------ torch.optim surface
    def zero_grad(self, set_to_none=True):
        """`.grad = None` for every parameter and ONE zero-fill of the flat gradient buffer: backward passes then write
        (or atomically accumulate) their results into it directly (grad_dest)"""
        for p in self.params:
            p.grad = None
        self.g.zero_()
        self.direct = True
        self.handed.clear()

    def gather_grads(self):
        """Gradients the backward did not write into `g` itself (ops.grad_dest) are copied there; returns how many."""
        src, dst = [], []
        base = self.p.data_ptr()
        for p, gv, o in zip(self.params, self.gviews, self.offsets):
            if p.data_ptr() != base + 4 * o:
                raise RuntimeError("FlatAdam: a parameter no longer lives in the flat buffer (model.to()/deepcopy after the "
                                   "optimizer was built?) -- build the optimizer after moving the model")
            if p.grad is None:
                raise RuntimeError("FlatAdam.step: a parameter received no gradient (torch.optim.Adam would skip it; "
                                   "leave dead parameters out of the optimizer instead)")
            if p.grad.data_ptr() != gv.data_ptr():
                src.append(p.grad.reshape(gv.shape))
                dst.append(gv)
        if src:
            torch._foreach_copy_(dst, src)
        return len(src)

    @property
    def grad_norm(self):
        return None if self.clip is None else self.clip.grad_norm

    @property
    def clipped(self):
        return None if self.clip is None else self.clip.clipped

    @property
    def skipped(self):
        return None if self.clip is None else self.clip.skipped

    def _adam_clip(self, state):
        _lib.call("fira_adam_flat_clip", self.p.data_ptr(), self.g.data_ptr(), self.m.data_ptr(), self.v.data_ptr(),
                  self.p16.data_ptr(), self.n, self.lr, self.betas[0], self.betas[1], self.eps, self.step_t.data_ptr(),
                  self.grad_scale.data_ptr() if self.grad_scale is not None else None,
                  self.ema.data_ptr() if self.ema is not None else None,
                  self.ema_decay if self.ema is not None else 0.0, state.data_ptr(),
                  torch.cuda.current_stream().cuda_stream)
        self.fresh = True
        if self.ema is not None:
            self.ema_moved()

    def step(self):
        if self.clip is not None:
            if len(self.clip.members) > 1:
                raise RuntimeError("FlatAdam.step: this optimizer shares a ClipGroup; step the group")
            self.clip.step()
            return
        self.gather_grads()
        self.direct = False                                   # g now holds this step's gradients
        self.step_t.add_(1.0)
        _lib.call("fira_adam_flat", self.p.data_ptr(), self.g.data_ptr(), self.m.data_ptr(), self.v.data_ptr(),
                  self.p16.data_ptr(), self.n, self.lr, self.betas[0], self.betas[1], self.eps, self.step_t.data_ptr(),
                  self.grad_scale.data_ptr() if self.grad_scale is not None else None,
                  self.ema.data_ptr() if self.ema is not None else None,
                  self.ema_decay if self.ema is not None else 0.0, torch.cuda.current_stream().cuda_stream)
        self.fresh = True
        if self.ema is not None:
            self.ema_moved()

    def _state_views(self, buf):
        return [buf[o:o + p.numel()].view(p.shape) for p, o in zip(self.params, self.offsets)]

    def state_dict(self):
        sd = {"step": float(self.step_t.item()), "lr": self.lr, "betas": self.betas, "eps": self.eps,
              "exp_avg": [t.clone() for t in self._state_views(self.m)],
              "exp_avg_sq": [t.clone() for t in self._state_views(self.v)]}
        if self.ema is not None:
            sd["ema"] = [t.clone() for t in self._state_views(self.ema)]
            sd["ema_decay"] = self.ema_decay
        return sd

    def load_state_dict(self, sd):
        self.step_t.fill_(float(sd["step"]))
        for dst, src in zip(self._state_views(self.m), sd["exp_avg"]):
            dst.copy_(src)
        for dst, src in zip(self._state_views(self.v), sd["exp_avg_sq"]):
            dst.copy_(src)
        if self.ema is not None and "ema" in sd:
            self.ema_decay = check_ema_decay(sd["ema_decay"])
            for dst, src in zip(self._state_views(self.ema), sd["ema"]):
                dst.copy_(src)
            self.ema_moved()


def attach(model, optims):
    """Tell `model` which FlatAdam instances own its parameters: TransModel.forward refreshes a stale bf16 mirror
    before it runs, and load_state_dict marks the mirrors stale."""
    model._flat_optims = list(optims)
    if not getattr(model, "_flat_hooked", False):
        model._flat_hooked = True

        def _stale(module, incompatible_keys):
            for o in getattr(module, "_flat_optims", ()):
                o.fresh = False
        model.register_load_state_dict_post_hook(_stale)


def ensure_fresh(model):
    for o in getattr(model, "_flat_optims", ()):
        if not o.fresh:
            o.sync_mirror()


def eager_step(model, optimizer, loss_fn):
    """One eager training step: model.train(), optimizer.zero_grad(), loss_fn() -> (loss, ...), loss.backward(),
    optimizer.step() -> what loss_fn returned.  Then the decoder's weights_epoch is bumped: a FlatAdam step writes the
    parameters through a raw kernel that moves neither their version counters nor their addresses, and the decoding
    loops' cached weight operands (decode_loop.loop_for) must re-read them."""
    model.train()
    optimizer.zero_grad()
    out = loss_fn()
    out[0].backward()
    optimizer.step()
    model.decoder.weights_epoch = getattr(model.decoder, "weights_epoch", 0) + 1
    return out


def ema_model(model, optims):
    """The EMA weights of `optims` (FlatAdam instances built with ema_decay that own `model`'s live parameters: one, or
    both halves of engine.GraphedTrainStep's pair) as a TransModel: built from `model.args`, in eval mode, no parameter
    requires grad.  Its live parameters are zero-copy views of the EMA buffers -- they follow every step -- and its dead
    parameters (and buffers) are copies of `model`'s.  state_dict() gives the reference's 338 keys, so torch.save of it
    is a checkpoint like best_model.pt.  ValueError if a live parameter is owned by no optimizer with an EMA."""
    from .model import TransModel
    owned = [o for o in optims if isinstance(o, FlatAdam) and o.ema is not None]
    dead = {id(p) for p in model.dead_parameters()}
    homes = []                                                # per parameter: None (dead) or (optimizer, slot)
    for name, p in model.named_parameters():
        if id(p) in dead:
            homes.append(None)
            continue
        o, s = _lookup(p)
        if o is None or not any(o is x for x in owned):
            raise ValueError(f"ema_model: live parameter {name} is owned by no optimizer with an EMA")
        homes.append((o, s))
    shadow = TransModel(model.args).to(model.out_fc.weight.device)
    shadow.set_precision(model.precision)
    mirrors = []
    with torch.no_grad():
        for home, p, q in zip(homes, model.parameters(), shadow.parameters()):
            if home is None:
                q.copy_(p)
                continue
            o, s = home
            mirror = o.ema_mirror()
            view = o.ema[s.off:s.off + s.numel].view(p.shape)
            q.data = view
            _SLOTS[(view.data_ptr(), s.numel)] = _Slot(mirror, s.off, s.numel)
            if not any(mirror is x for x in mirrors):
                mirrors.append(mirror)
        for b, c in zip(model.buffers(), shadow.buffers()):
            c.copy_(b)
    shadow.eval()
    shadow.requires_grad_(False)
    for mirror in mirrors:
        mirror.models.add(shadow)
    attach(shadow, mirrors)
    return shadow
