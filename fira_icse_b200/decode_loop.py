"""The on-device decoding loop shared by seeded sampling (sample.py) and n-best beam search (beam.nbest).

Per batch the encoder, the cross-attention K/V of the memory and LinearSource(memory) run once (`start`).  The N rows
of a commit (samples or beam slots) are the N query rows of an incremental.IncrementalDecoder.  Per position:
newest decoder row -> out_fc -> target projection and gate -> copy scores (`head`), then the decoder's own kernel,
which writes the next input tokens straight into the decoder's token buffer (`position`, defined by each decoder).
A position is captured once into a CUDA graph and replayed for every later batch of the same shape; the loop reads
back nothing but an all-finished flag, once every POLL_EVERY positions.
"""
import weakref

import torch

from . import ops
from ._lib import call
from .incremental import IncrementalDecoder

D = ops.D
POLL_EVERY = 8            # positions between two reads of the all-finished flag


def _weights_key(model):
    ps = list(model.parameters())
    return (getattr(model.decoder, "weights_epoch", 0),) + tuple(p._version for p in ps) + tuple(p.data_ptr() for p in ps)


class PositionLoop:
    """Static buffers and captured position graphs of one (model, B, N, tar_len, S, precision).

    Subclasses define position(t, *cfg) (head(t), then their own launches; every launch on the current stream) and
    unfinished(t) (a device bool: some row still decodes after t positions)."""

    def __init__(self, model, B, N, T, S):
        self.model, self.B, self.N, self.T, self.S = model, B, N, T, S
        self.inc = IncrementalDecoder(model.decoder, B, N, T, S, graphs=False)   # its launches go into our graphs
        self.pr = ops.Prec(self.inc.be.bf16)
        self.dev = dev = model.out_fc.weight.device
        R = self.R = B * N
        tdt = self.inc.be.tdt
        self.V = model.vocab_size
        self.ldl = ops._ld_logits(self.V)
        self.mem_mask = torch.zeros((B, S), dtype=torch.uint8, device=dev)
        self.copy_src = torch.zeros((B, S), dtype=torch.int32, device=dev)
        self.src = torch.empty((B * S, D), dtype=tdt, device=dev)
        self.logits = torch.empty((R, self.ldl), dtype=tdt, device=dev)
        self.tgt = torch.empty((R, D), dtype=tdt, device=dev)
        self.gl = torch.empty((R, 2), dtype=torch.float32, device=dev)
        self.sc = torch.empty((B, N, S), dtype=torch.float32, device=dev)
        self.graphs = {}

    def start(self, memory, mem_mask, copy_src, start_id, pad_id):
        inc = self.inc
        inc.start(memory, mem_mask)
        mem2 = memory.contiguous().to(inc.be.tdt).view(self.B * self.S, D)
        self.pr.linear(mem2, self.model.copy_net.LinearSource.weight, out=self.src)     # once per batch, not per row
        self.mem_mask.copy_(mem_mask)
        self.copy_src.copy_(copy_src)
        inc.tok[:self.R].fill_(start_id)
        inc.tok_mask[:, 0].fill_(int(start_id != pad_id))

    def head(self, t):
        """logits, copy scores and gate logits of decoder row t (every launch on the current stream: capturable)."""
        m, pr, B, N, S = self.model, self.pr, self.B, self.N, self.S
        cn = m.copy_net
        x = self.inc.advance(t)                                                  # [R, D]
        pr.linear(x, m.out_fc.weight, m.out_fc.bias, out=self.logits, ld_out=self.ldl)
        pr.linear(x, cn.LinearTarget.weight, out=self.tgt)
        ops.linear(x.float() if pr.bf16 else x, cn.LinearProb.weight, cn.LinearProb.bias, out=self.gl)   # fp32 gate
        p = ops._ptr
        call("fira_copy_scores_fwd", p(self.src), p(self.tgt), p(cn.LinearRes.weight), p(cn.LinearRes.bias),
             p(self.mem_mask), None, p(self.sc), B, N, S, D, pr.code, ops._stream())

    def run(self, cfg):
        """Positions 0..T-2 (fewer once every row has finished) -> the number of positions run."""
        t = 0
        while t < self.T - 1:
            if t and t % POLL_EVERY == 0 and not bool(self.unfinished(t)):
                break
            g = self.graphs.get((cfg, t))
            if g is not None:
                g.replay()
            else:
                self.position(t, *cfg)                         # this batch's result (and the warm-up of a capture) ...
                torch.cuda.synchronize()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):                      # ... and the same launches recorded for later batches
                    self.position(t, *cfg)
                self.graphs[(cfg, t)] = g
            t += 1
        return t


_LOOPS = weakref.WeakKeyDictionary()          # model -> {(class, B, N, T, S, precision): (weights key, loop)}


def loop_for(cls, model, B, N, T, S):
    """The cached `cls` instance of this shape; rebuilt (fresh operand copies and graphs) when the weights changed."""
    store = _LOOPS.setdefault(model, {})
    key = (cls, B, N, T, S, model.precision)
    wkey = _weights_key(model)
    if key not in store or store[key][0] != wkey:
        store[key] = (wkey, cls(model, B, N, T, S))
    return store[key][1]
