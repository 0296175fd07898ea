"""CUDA-graph training engine: the whole step (zero grads -> TransModel forward -> backward ->
[all-reduce] -> Adam) is captured once per input shape and replayed, so the ~700 launches of a step
cost one cudaGraphLaunch instead of ~700 Python/ctypes round trips (the bf16 step is launch-bound
otherwise).

What makes the path capturable
  * every kernel is launched on the current stream through the C ABI, with caller-owned buffers
    (they come from the graph's private pool during capture) and no host synchronisation;
  * inputs live in STATIC device buffers (ids, labels, CSR arrays with a fixed edge capacity -- the
    kernels only walk rowptr ranges, so the tail of col/val is never read);
  * dropout masks are keyed by `seed + *seed_ctr`; the graph bumps the device counter on every replay,
    so replays draw fresh masks although the host-side seed is frozen into the graph;
  * TMA tensor maps are kernel parameters, rebuilt at capture time for the pooled buffers;
  * weight-gradient work and weight preparation run on a forked stream = parallel graph branches.
Batches whose padding was trimmed by the loader (data.PackedBatchLoader / trim_batch_host) come in a few
distinct (batch, n_code, n_sub, n_ast) shapes: one graph per shape, one shared optimizer.  The graphs are
replayed strictly one after the other on one stream and nothing produced inside one is read after the
next has started (losses are copied to static scalars inside the graph, gradients are consumed by the
optimizer inside the graph or right after the replay), so all of them capture into ONE memory pool: device
memory is the maximum over the shapes, not the sum (FIRA_GRAPH_PRIVATE_POOLS=1 gives each graph its own).
N > 1: forward/backward graph, eager NCCL all-reduce of ONE flat gradient buffer, optimizer graph
(same numerics as parallel.DataParallelStep).
An optimizer factory that builds optim.FlatAdam(..., ema_decay=d) gets the weights' moving average in every mode: each
captured optimizer step is a fira_adam_flat launch, which updates the EMA too.  `ema_model()` is the EMA as a model;
every replay marks it stale.  Under data parallelism every rank updates the same EMA from the same parameters.
An optimizer factory that builds optim.FlatAdam(..., max_grad_norm=c) clips the gradient's global norm over BOTH halves
of the optimizer pair (one optim.ClipGroup) and skips steps whose gradient is not finite, inside the captured work:
  * overlap: the head/decoder half's sum of squares runs on the side stream while the encoder backward runs; after the
    join, the encoder half's sum of squares, the finalize and both Adam launches (Adam can no longer hide behind the
    encoder backward: it needs the whole norm);
  * one optimizer (FIRA_OPT_OVERLAP=0, or N > 1 without the split): sum of squares -> finalize -> Adam, at the end of the
    graph or in the optimizer graph after the all-reduce;
  * split: half A's all-reduce and sum of squares still run behind graph B; half B's all-reduce is followed by its sum
    of squares, the finalize and both Adam launches.
`grad_norm`, `clipped` and `skipped` are the group's device scalars.  A skipped step changes no buffer and captures
nothing new.
"""
import os

import torch
import torch.distributed as dist

from . import optim as _optim
from .graph import PackedEdges
from .optim import FlatAdam
from .packed import PackedBatch
from .parallel import FlatGradBucket

ID_KEYS = ("sou", "tar", "mark", "ast_change", "tar_label", "sub_token")


class _Captured:
    """Static buffers + graph of one input shape."""

    def __init__(self, shapes, B, n_nodes, cap, dev):
        self.ids = {k: torch.zeros((B, n), dtype=torch.int64, device=dev) for k, n in zip(ID_KEYS, shapes)}
        self.rowptr = torch.zeros(B * n_nodes + 1, dtype=torch.int32, device=dev)
        self.col = torch.zeros(cap, dtype=torch.int32, device=dev)
        self.val = torch.zeros(cap, dtype=torch.float32, device=dev)
        self.B, self.n_nodes, self.cap = B, n_nodes, cap
        self.graph = None
        self.grads = None


class _CapturedPacked:
    """Static device copy of a per-commit packed batch shape (packed.PackedBatch) + its graph."""

    def __init__(self, pb, cap, dev):
        def z(t, n=None):
            return torch.zeros(t.shape if n is None else (n,), dtype=t.dtype, device=dev)
        t = {k: z(getattr(pb, k)) for k in PackedBatch.FIELDS if k not in ("col", "val")}
        t["col"], t["val"] = z(pb.col, cap), z(pb.val, cap)
        self.pb = PackedBatch(pb.B, pb.Rc, pb.Rs, pb.Ra, pb.S, pb.T, cap, pb.chunks, pb.Rv, pb.Rt, **t)
        self.B, self.cap = pb.B, cap
        self.graph = None
        self.grads = None
        self.packed = True

    def copy_from(self, pb):
        for k in PackedBatch.FIELDS:
            src, dst = getattr(pb, k), getattr(self.pb, k)
            if k in ("col", "val"):
                dst[:src.numel()].copy_(src, non_blocking=True)
            else:
                dst.copy_(src, non_blocking=True)


class _OptimizerPair:
    """the two optimizers of the overlapped step behind the one-optimizer interface callers use (step / state_dict)"""

    def __init__(self, pair):
        self.pair = pair

    def step(self):
        clip = getattr(self.pair[0], "clip", None)
        if clip is not None:                         # one norm over both halves
            clip.step()
            return
        for o in self.pair:
            o.step()

    def zero_grad(self, set_to_none=True):
        for o in self.pair:
            o.zero_grad(set_to_none=set_to_none)

    def state_dict(self):
        return [o.state_dict() for o in self.pair]


class GraphedTrainStep:
    def __init__(self, model, batch_size, optimizer_factory, edge_capacity=None, group=None, split=None):
        self.model, self.B, self.group = model, batch_size, group          # B: the largest batch (sizes the CSR capacity)
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        # split: capture the step as TWO graphs -- (A) forward + head/decoder backward down to the encoder memory,
        # (B) encoder backward -- so that the all-reduce of the head/decoder gradients (3/4 of the bytes) runs on a
        # communication stream WHILE graph B replays.  Default: on for N > 1 (FIRA_DP_OVERLAP=0 restores the single
        # graph + one flat all-reduce); split=True on one GPU exercises the same two-graph path without NCCL (tests).
        self.split = (self.world > 1 and os.environ.get("FIRA_DP_OVERLAP", "1") != "0") if split is None else bool(split)
        self.comm = None
        self._stash = None
        self.flat_a = self.flat_b = None
        self.params_a = self.params_b = None
        # one GPU: two optimizers (head/decoder parameters, encoder parameters) so that the first can step while the
        # encoder backward still runs (FIRA_OPT_OVERLAP=0: one optimizer at the end of the graph)
        self.opt_factory = optimizer_factory
        self.opt_pair = None
        self.opt_stream = None
        self.opt_overlap = self.world == 1 and not self.split and os.environ.get("FIRA_OPT_OVERLAP", "1") != "0"
        self.dev = next(model.parameters()).device
        self.cap = edge_capacity or batch_size * 4096
        self.n_global = torch.ones(1, dtype=torch.float32, device=self.dev)     # global token count (all ranks)
        self.seed_ctr = torch.zeros(1, dtype=torch.int64, device=self.dev)
        model.encoder.seed_ctr = model.decoder.seed_ctr = self.seed_ctr
        self.bucket = FlatGradBucket(model.live_parameters())
        # the overlapped modes train with TWO optimizers (head/decoder parameters | encoder parameters) found by the
        # first split backward; the single optimizer of the other modes is built right away
        self.two_opts = self.opt_overlap or (self.split and os.environ.get("FIRA_DP_TWO_OPTS", "1") != "0")
        self.optimizer = None if self.two_opts else optimizer_factory(self.bucket.params)
        self.flat_optims = []
        self._note_optimizers()
        self.loss_sum = torch.zeros((), dtype=torch.float32, device=self.dev)
        self.n_local = torch.zeros((), dtype=torch.int64, device=self.dev)
        self.captured = {}
        self.cur = None
        self.opt_ready = False
        self.graph_opt = None
        self.static_flat = None
        self.pool = None                     # graph memory pool shared by every captured shape
        self._ema = None                     # optim.ema_model of the optimizers, built by ema_model()

    def _note_optimizers(self):
        """optim.FlatAdam instances own the parameters' storage, their flat gradient buffers and the bf16 mirror"""
        opts = list(self.opt_pair) if self.opt_pair is not None else ([self.optimizer] if self.optimizer is not None else [])
        self.flat_optims = [o for o in opts if isinstance(o, FlatAdam)]
        if self.flat_optims:
            _optim.attach(self.model, self.flat_optims)

    def ema_model(self):
        """The moving average of the weights kept by the optimizers (FlatAdam with ema_decay) as a TransModel in eval mode
        (optim.ema_model), built once: its parameters are views of the EMA buffers, so it follows every step.  The
        optimizers exist after the first step(), not before."""
        if self._ema is None:
            if not self.opt_ready:
                raise RuntimeError("GraphedTrainStep.ema_model: the optimizers exist after the first step()")
            self._ema = _optim.ema_model(self.model, self.flat_optims)
        return self._ema

    @property
    def clip(self):
        """the optim.ClipGroup of the optimizers (FlatAdam with max_grad_norm), or None (no clipping, or before the first
        step() in the modes that build their optimizers then)"""
        for o in self.flat_optims:
            if o.clip is not None:
                return o.clip
        return None

    @property
    def grad_norm(self):
        """device float64 scalar: the last step's global gradient norm (non-finite on a skipped step); None without
        clipping"""
        return None if self.clip is None else self.clip.grad_norm

    @property
    def clipped(self):
        return None if self.clip is None else self.clip.clipped

    @property
    def skipped(self):
        return None if self.clip is None else self.clip.skipped

    def _ema_moved(self):
        """a replay moved the EMA behind Python's back: the shadow model's bf16 mirror and weight caches are stale"""
        for o in self.flat_optims:
            if o.ema is not None:
                o.ema_moved()

    def _cap_stream(self):
        """Capture stream of the step graphs: HIGH priority, so that the kernels of the main chain (the critical path:
        forward, input gradients) carry a higher launch priority than the weight-gradient / preparation work on the
        default-priority side streams that runs next to them (FIRA_MAIN_PRIORITY=0: default priority)."""
        if getattr(self, "_cap_s", None) is None:
            hi = os.environ.get("FIRA_MAIN_PRIORITY", "1") != "0"
            self._cap_s = torch.cuda.Stream(priority=-1) if hi else torch.cuda.Stream()
        return self._cap_s

    def _zero(self):
        self.bucket.zero()
        for o in self.flat_optims:
            o.zero_grad()                  # one zero-fill of the flat gradient buffer; backward writes into it directly

    # ------------------------------------------------------------------ data
    @staticmethod
    def _split(batch):
        src = dict(zip(("sou", "tar", "attr", "mark", "ast_change", "edges", "tar_label", "sub_token"), batch))
        e = src["edges"]
        csr = (e.rowptr, e.col, e.val) if isinstance(e, PackedEdges) else e
        return src, csr

    def load(self, batch):
        """batch: [sou, tar, attr, mark, ast_change, edges, tar_label, sub_token]; `edges` a PackedEdges or a
        host/device (rowptr, col, val) triple.  Copies into the static buffers of the batch's shape
        (async when the sources are pinned) and makes that shape current."""
        if isinstance(batch, PackedBatch):
            if batch.nnz > self.cap:
                raise ValueError(f"batch has {batch.nnz} edges, graph capacity is {self.cap}")
            key = ("packed",) + batch.shape_key
            c = self.captured.get(key)
            if c is None:
                c = self.captured[key] = _CapturedPacked(batch, self.cap, self.dev)
            c.copy_from(batch)
            self.cur = c
            return c
        src, (rowptr, col, val) = self._split(batch)
        shapes = tuple(int(src[k].shape[1]) for k in ID_KEYS)
        B = int(src["sou"].shape[0])
        n_nodes = shapes[0] + shapes[3] + shapes[5]
        if rowptr.numel() != B * n_nodes + 1:
            raise ValueError("adjacency does not match the id tensors (rows != B * (n_code + n_sub + n_ast))")
        if col.numel() > self.cap:
            raise ValueError(f"batch has {col.numel()} edges, graph capacity is {self.cap}")
        c = self.captured.get((B,) + shapes)
        if c is None:               # a new (batch, n_code, n_sub, n_ast) shape, e.g. the short last batch of an epoch
            c = self.captured[(B,) + shapes] = _Captured(shapes, B, n_nodes, self.cap, self.dev)
        for k in ID_KEYS:
            c.ids[k].copy_(src[k], non_blocking=True)
        c.rowptr.copy_(rowptr, non_blocking=True)
        c.col[:col.numel()].copy_(col, non_blocking=True)
        c.val[:val.numel()].copy_(val, non_blocking=True)
        self.cur = c
        return c

    @staticmethod
    def _static_batch(c, B):
        edges = PackedEdges(c.rowptr, c.col, c.val, B, c.n_nodes, True)     # fresh wrapper: no cached rowsum
        i = c.ids
        return [i["sou"], i["tar"], None, i["mark"], i["ast_change"], edges, i["tar_label"], i["sub_token"]]

    # ------------------------------------------------------------------ the step
    def _forward_backward(self, c):
        self.seed_ctr.add_(1)
        self._zero()
        if getattr(c, "packed", False):
            loss_sum, n_tok = self.model.forward_packed(c.pb, "train")
        else:
            loss_sum, n_tok = self.model(*self._static_batch(c, c.B), "train")
        self.loss_sum.copy_(loss_sum.detach())
        self.n_local.copy_(n_tok)
        denom = self.n_global.squeeze(0) if self.world > 1 else n_tok.to(torch.float32)
        (loss_sum / denom).backward()

    # ------------------------------------------------------------------ split step (gradient all-reduce overlap)
    def _split_memory(self, memory):
        leaf = memory.detach().requires_grad_(True)
        self._stash = (memory, leaf)
        return leaf

    def _phase_a(self, c):
        """forward + backward of the head and the decoder; stops at the encoder memory (a leaf for this pass)"""
        self.model._memory_hook = self._split_memory
        try:
            self._forward_backward(c)
        finally:
            self.model._memory_hook = None

    def _phase_b(self):
        """encoder backward from the memory gradient phase A left on the leaf"""
        memory, leaf = self._stash
        # drop the reference BEFORE anything else can run: a stashed autograd graph keeps the parameters' AccumulateGrad
        # nodes alive, and a later (captured) forward would re-use nodes bound to the stream of THIS pass
        self._stash = None
        memory.backward(leaf.grad)

    def _bind_flat(self, c, which, params):
        """After a capture: gradients the captured backward left OUTSIDE the optimizers' flat buffers (none when every
        producer wrote through ops._gdest) are listed for an eager copy per replay; `.grad` of every parameter is then
        pointed at its slice of the flat buffer, which is what the captured optimizer step reads."""
        pairs = []
        for o in self.flat_optims:
            ids = {id(p) for p in params}
            for p, gv in zip(o.params, o.gviews):
                if id(p) in ids:
                    if p.grad.data_ptr() != gv.data_ptr():
                        pairs.append((gv, p.grad.reshape(gv.shape)))
                    p.grad = gv
        setattr(c, "copy_" + which, pairs)

    @staticmethod
    def _copy_pairs(pairs):
        if pairs:
            torch._foreach_copy_([d for d, _ in pairs], [s for _, s in pairs])

    def _capture_split(self, c):
        flat = bool(self.flat_optims)
        c.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(c.graph, pool=self.pool, stream=self._cap_stream()):
            self._phase_a(c)
        if self.params_a is None:
            self.params_a = [p for p in self.bucket.params if p.grad is not None]
            ids = {id(p) for p in self.params_a}
            self.params_b = [p for p in self.bucket.params if id(p) not in ids]
        c.grads_a = [p.grad for p in self.params_a]
        c.graph_b = torch.cuda.CUDAGraph()
        with torch.cuda.graph(c.graph_b, pool=self.pool, stream=self._cap_stream()):
            self._phase_b()
        c.grads_b = [p.grad for p in self.params_b]
        assert all(g is not None for g in c.grads_a + c.grads_b), "a live parameter received no gradient"
        if self.comm is None:
            self.comm = torch.cuda.Stream()
        if flat:
            # optim.FlatAdam: the backward wrote the gradients into the optimizers' flat buffers, which are all-reduced
            # in place; two optimizers, so that Adam of the head/decoder parameters also runs behind graph B
            self._bind_flat(c, "a", self.params_a)
            self._bind_flat(c, "b", self.params_b)
            if self.graph_opt is None:
                clip = self.clip
                self.graph_opt = []
                for k, o in enumerate(self.opt_pair):
                    g = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(g):
                        if clip is None:
                            o.step()
                        else:                             # A: its sum of squares; B: its sum of squares + both Adams
                            clip.sumsq(o)
                            if k == len(self.opt_pair) - 1:
                                clip.finish()
                    self.graph_opt.append(g)
            return
        if self.flat_a is None:
            self.flat_a = torch.cat([g.reshape(-1) for g in c.grads_a])
            self.flat_b = torch.cat([g.reshape(-1) for g in c.grads_b])
        for flat_buf, params in ((self.flat_a, self.params_a), (self.flat_b, self.params_b)):
            off = 0
            for p in params:
                p.grad = flat_buf[off:off + p.numel()].view_as(p)
                off += p.numel()
        if self.graph_opt is None:
            self.graph_opt = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.graph_opt):
                self.optimizer.step()

    def _replay_split(self, c):
        cur = torch.cuda.current_stream()
        flat = bool(self.flat_optims)
        c.graph.replay()
        self.comm.wait_stream(cur)
        with torch.cuda.stream(self.comm):               # head/decoder gradients: all-reduce (+ Adam) behind graph B
            if flat:
                self._copy_pairs(c.copy_a)
                if self.world > 1:
                    dist.all_reduce(self.opt_pair[0].g, group=self.group)
                self.graph_opt[0].replay()
            else:
                torch.cat([g.reshape(-1) for g in c.grads_a], out=self.flat_a)
                if self.world > 1:
                    dist.all_reduce(self.flat_a, group=self.group)
        c.graph_b.replay()
        self.comm.wait_stream(cur)
        with torch.cuda.stream(self.comm):
            if flat:
                self._copy_pairs(c.copy_b)
                if self.world > 1:
                    dist.all_reduce(self.opt_pair[1].g, group=self.group)
                self.graph_opt[1].replay()
            else:
                torch.cat([g.reshape(-1) for g in c.grads_b], out=self.flat_b)
                if self.world > 1:
                    dist.all_reduce(self.flat_b, group=self.group)
        cur.wait_stream(self.comm)
        if not flat:
            self.graph_opt.replay()

    def _count_tokens_eager(self, c):
        if self.world > 1:
            lab = c.pb.label if getattr(c, "packed", False) else c.ids["tar_label"][:, 1:]     # packed labels are shifted
            self.n_global.copy_((lab != 0).sum().to(torch.float32).reshape(1))
            dist.all_reduce(self.n_global, group=self.group)

    def _make_pair(self, c):
        """find the two parameter groups with one split backward, then build the two optimizers"""
        self._phase_a(c)
        pa = [p for p in self.bucket.params if p.grad is not None]
        ids = {id(p) for p in pa}
        pb = [p for p in self.bucket.params if id(p) not in ids]
        self._phase_b()
        self.params_a, self.params_b = pa, pb
        self.opt_pair = (self.opt_factory(pa), self.opt_factory(pb))
        if any(getattr(o, "max_grad_norm", None) is not None for o in self.opt_pair):
            _optim.ClipGroup(self.opt_pair)            # one norm over both halves (ValueError unless both clip alike)
        self.optimizer = _OptimizerPair(self.opt_pair)
        self._note_optimizers()
        if self.opt_overlap:
            self.opt_stream = torch.cuda.Stream()

    def _eager_step(self, c):
        """A normal (uncaptured) training step: initialises the optimizer state and all lazy CUDA state."""
        self._count_tokens_eager(c)
        if self.two_opts and self.opt_pair is None:
            self._make_pair(c)             # the gradients of this pass predate the optimizers' flat buffers: discard them
            self._zero()
        self._forward_backward(c)
        if self.world > 1:
            if self.flat_optims:
                for o in self.flat_optims:
                    o.gather_grads()
                    dist.all_reduce(o.g, group=self.group)
                    for p, gv in zip(o.params, o.gviews):
                        p.grad = gv
            else:
                self.bucket.all_reduce(self.group)
        self.optimizer.step()
        self.opt_ready = True

    def _capture(self, c):
        """Warm the shape up with one forward/backward whose gradients are discarded, then capture."""
        self._stash = None
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            # no collective here: ranks meet new shapes at different steps, so the number of NCCL calls per step
            # must not depend on whether a rank is capturing (n_global keeps its previous value; the result of
            # this warm-up pass is discarded)
            self._forward_backward(c)
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        self._zero()
        if self.pool is None and os.environ.get("FIRA_GRAPH_PRIVATE_POOLS", "0") != "1":
            self.pool = torch.cuda.graph_pool_handle()
        if self.split:
            return self._capture_split(c)
        c.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(c.graph, pool=self.pool, stream=self._cap_stream()):
            if self.world == 1 and self.opt_overlap:
                # ONE graph, two branches: Adam on the head/decoder parameters (3/4 of the bytes, memory-bound, nothing
                # else could hide it at the end of the step) runs on a side stream WHILE the encoder backward runs
                clip = self.clip
                self._phase_a(c)
                cur = torch.cuda.current_stream()
                self.opt_stream.wait_stream(cur)
                with torch.cuda.stream(self.opt_stream):
                    if clip is None:
                        self.opt_pair[0].step()
                    else:                                  # clipping: only this half's share of the norm runs here
                        clip.sumsq(self.opt_pair[0])
                self._phase_b()
                cur.wait_stream(self.opt_stream)
                if clip is None:
                    self.opt_pair[1].step()
                else:
                    clip.sumsq(self.opt_pair[1])
                    clip.finish()
            else:
                self._forward_backward(c)
                if self.world == 1:
                    self.optimizer.step()
        if self.world > 1:
            # the captured backward always writes the same pool tensors; pack them into ONE static flat buffer
            # (eager concat + NCCL all-reduce) and let the captured optimizer read views of that buffer
            c.grads = [p.grad for p in self.bucket.params]
            if self.static_flat is None:
                self.static_flat = torch.cat([g.reshape(-1) for g in c.grads])
            off = 0
            for p in self.bucket.params:
                p.grad = self.static_flat[off:off + p.numel()].view_as(p)
                off += p.numel()
            if self.graph_opt is None:
                self.graph_opt = torch.cuda.CUDAGraph()
                with torch.cuda.graph(self.graph_opt):        # private pool: Adam's temporaries live across shapes
                    self.optimizer.step()

    def capture(self, warmup=None):
        """Make sure the current shape is ready to replay (kept for callers that want to pay the capture
        cost up front); performs real training steps only for the very first batch."""
        c = self.cur
        if not self.opt_ready:
            self._eager_step(c)
        if c.graph is None:
            self._capture(c)
        return self

    def step(self, batch=None):
        """One training step on `batch` (or on what was load()ed).  Returns the device scalars (sum of the
        local NLL, local token count); nothing synchronises once the shape's graph exists."""
        c = self.load(batch) if batch is not None else self.cur
        if not self.opt_ready:
            self._eager_step(c)                       # first step of the run: eager
            return self.loss_sum, self.n_local
        if c.graph is None:
            self._capture(c)
        for o in self.flat_optims:                    # parameters set from outside (load_state_dict): refresh the bf16 mirror
            if not o.fresh:
                o.sync_mirror()
        self._count_tokens_eager(c)
        if self.split:
            self._replay_split(c)
            self.model.decoder.weights_epoch = getattr(self.model.decoder, "weights_epoch", 0) + 1
            self._ema_moved()
            return self.loss_sum, self.n_local
        c.graph.replay()
        # graph replays update the parameters without touching their autograd version counters: tell weight caches
        # keyed on those (incremental.IncrementalDecoder) that the weights moved
        self.model.decoder.weights_epoch = getattr(self.model.decoder, "weights_epoch", 0) + 1
        if self.world > 1:
            torch.cat([g.reshape(-1) for g in c.grads], out=self.static_flat)
            dist.all_reduce(self.static_flat, group=self.group)
            self.graph_opt.replay()
        self._ema_moved()
        return self.loss_sum, self.n_local
