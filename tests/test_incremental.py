"""Cache bookkeeping of the KV-cached beam decoder (fira_icse_b200.incremental) on CPU.

The product backend launches CUDA kernels; here a torch backend (test infrastructure, below) is injected so
that the incremental evaluation -- token feeding, pad masks, cache writes, beam reordering -- can be compared
with the oracle's full 30-position decoder without a GPU.  The same path on the CUDA backend -- its kernels at the
decoding shapes, strides and row paddings, captured graphs, weight refreshes, shared buffers and the position loop's
head -- is checked against float64 by tests/test_gpu_incremental.py, and the end-to-end id parity by
tests/test_gpu_cli.py."""
import math

import torch
import torch.nn.functional as Fn

import fira_oracle as O
from fira_testlib import reference_args


class TorchBackend:
    tdt = torch.float32

    def weight(self, W):
        return W.detach()

    def embed(self, ids_i32, table, pos_row, out):
        out.copy_(table[ids_i32.long()] + pos_row)
        return out

    def linear(self, x, Wop, b, relu=False, out=None):
        y = x @ Wop.t() + b
        y = torch.relu(y) if relu else y
        if out is not None:
            out.copy_(y)
            return out
        return y

    def attention(self, q, k, v, key_mask, B, H, Lq, Lk):
        d = q.shape[1] // H
        Q = q.reshape(B, Lq, H, d).transpose(1, 2)
        K = k.reshape(B, Lk, H, d).transpose(1, 2)
        V = v.reshape(B, Lk, H, d).transpose(1, 2)
        s = (Q @ K.transpose(-1, -2)) / math.sqrt(d)
        s = s.masked_fill(key_mask.view(B, 1, 1, Lk) == 0, -1e9)
        return (torch.softmax(s, -1) @ V).transpose(1, 2).reshape(B * Lq, H * d)

    def layer_norm(self, z, resid, gamma, beta):
        return Fn.layer_norm(z + resid, (z.shape[1],), gamma, beta, 1e-5)


def test_incremental_rows_equal_full_decoder_under_beam_reordering():
    from fira_icse_b200.incremental import IncrementalDecoder
    from fira_icse_b200.modules import Decoder
    torch.manual_seed(5)
    args = reference_args(vocab_size=200)
    dec = Decoder(args, 0).eval()
    with torch.no_grad():
        for p in dec.parameters():                      # LayerNorm weights/biases away from (1, 0)
            if p.dim() == 1:
                p.add_(0.1 * torch.randn_like(p))
    sd = {"decoder." + k: v.detach() for k, v in dec.state_dict().items()}
    B, K, T, S, steps = 2, 3, args.tar_len, 11, 7
    memory = torch.randn(B, S, 256)
    mem_mask = torch.rand(B, S) > 0.3
    mem_mask[:, 0] = True
    inc = IncrementalDecoder(dec, B, K, T, S, backend=TorchBackend()).start(memory, mem_mask)
    assert inc.Rp == 128 and not inc.use_graphs
    seq = torch.zeros(B, K, T, dtype=torch.long)
    seq[:, :, 0] = 1
    g = torch.Generator().manual_seed(9)
    with torch.no_grad():
        for t in range(steps):
            got = inc.step(seq[:, :, t].reshape(B * K), t, 0).clone()
            full = O.decoder(sd, seq.view(B * K, T), memory.repeat_interleave(K, 0), mem_mask.repeat_interleave(K, 0)[:, None, None, :],
                             seq.view(B * K, T) != 0)
            assert torch.allclose(got, full[:, t], atol=2e-5, rtol=1e-5), t
            # re-rank: every new beam continues a random old beam of the same commit and appends a token
            src = torch.randint(0, K, (B, K), generator=g)
            seq = seq[torch.arange(B).unsqueeze(1), src]
            seq[:, :, t + 1] = torch.randint(0 if t == 3 else 3, 200, (B, K), generator=g)   # step 3 may append pad (0)
            inc.reorder((torch.arange(B).unsqueeze(1) * K + src).reshape(-1))
    # a second batch on the same instance starts from clean caches
    inc.start(memory.flip(0), mem_mask.flip(0))
    assert int(inc.tok_mask.sum()) == 0 and float(inc.kv_self.abs().sum()) == 0.0
    # parameters updated in place (a training step between two evaluations): the prepared weights follow
    with torch.no_grad():
        for p in dec.parameters():
            p.mul_(1.05)
    sd2 = {"decoder." + k: v.detach() for k, v in dec.state_dict().items()}
    inc.start(memory, mem_mask)
    tok = torch.full((B * K,), 1, dtype=torch.long)
    with torch.no_grad():
        got = inc.step(tok, 0, 0).clone()
        seq0 = torch.zeros(B * K, T, dtype=torch.long)
        seq0[:, 0] = 1
        full = O.decoder(sd2, seq0, memory.repeat_interleave(K, 0), mem_mask.repeat_interleave(K, 0)[:, None, None, :],
                         seq0 != 0)
    assert torch.allclose(got, full[:, 0], atol=2e-5, rtol=1e-5)
