"""`Model.py` surface of the reference (CopyNet, TransModel) on the CUDA path.

    model = TransModel(args)                  # args as run_model.py:27-56
    loss_sum, n_tok = model(sou, tar, attr, mark, ast_change, edge, tar_label, sub_token, 'train')
    ids = model(..., 'dev')                   # argmax over the 25,020-wide dual-copy distribution

`edge` is the reference's dense [B,650,650] float tensor (any float dtype) OR a
fira_icse_b200.graph.PackedEdges (what the packed loader emits).  Sub-modules `encoder`,
`decoder`, `out_fc`, `copy_net` are individually callable, as the reference's beam loop
requires (run_model.py:204,256,257,259).
"""
import os

import torch
import torch.nn as nn

from . import ops
from . import optim as _optim
from .modules import Decoder, Encoder, _i32, _u8


class _OutFc(nn.Linear):
    """nn.Linear whose forward runs on fira_gemm_f32 (Model.py:34,54)."""

    def forward(self, x):
        return ops.LinearFn.apply(x, self.weight, self.bias)


class CopyNet(nn.Module):
    """Model.py:7-20.  forward(source, target) -> (pointer scores [B,T,S], gate [B,T,2])."""

    def __init__(self, args):
        super().__init__()
        self.embedding_size = args.embedding_dim
        self.LinearSource = nn.Linear(self.embedding_size, self.embedding_size, bias=False)
        self.LinearTarget = nn.Linear(self.embedding_size, self.embedding_size, bias=False)
        self.LinearRes = nn.Linear(self.embedding_size, 1)
        self.LinearProb = nn.Linear(self.embedding_size, 2)

    def flat_params(self):
        return [self.LinearSource.weight, self.LinearTarget.weight, self.LinearRes.weight, self.LinearRes.bias,
                self.LinearProb.weight, self.LinearProb.bias]

    def forward(self, source, traget):
        scores = ops.CopyScoresFn.apply(source, traget, self.LinearSource.weight, self.LinearTarget.weight,
                                        self.LinearRes.weight, self.LinearRes.bias)
        gate_logits = ops.LinearFn.apply(traget, self.LinearProb.weight, self.LinearProb.bias)
        # [B,T,2] two-way softmax: 60 floats per commit, not worth a kernel outside the fused head
        return scores, torch.softmax(gate_logits, dim=-1)


class TransModel(nn.Module):
    """Model.py:24-86."""

    def __init__(self, args):
        super().__init__()
        self.embedding_dim = args.embedding_dim
        self.vocab_size = args.vocab_size
        self.sou_len = args.sou_len
        self.sub_token_len = args.sub_token_len
        self.encoder = Encoder(args, pad_token_id=0)
        self.decoder = Decoder(args, pad_token_id=0)
        self.out_fc = _OutFc(args.embedding_dim, args.vocab_size)
        self.gate_fc = nn.Linear(args.embedding_dim, 1)   # dead upstream too (Model.py:35)
        self.copy_net = CopyNet(args)
        self._memory_hook = None      # engine.GraphedTrainStep(split=True): cuts the autograd graph at the encoder memory
        self.set_precision(os.environ.get("FIRA_PRECISION", "fp32"))

    def set_precision(self, precision):
        """'fp32' (parity mode, default) or 'bf16' (throughput mode: bf16 activations, wgmma GEMMs)."""
        if precision not in ("fp32", "bf16"):
            raise ValueError("precision must be 'fp32' or 'bf16'")
        self.precision = precision
        self.encoder.bf16 = self.decoder.bf16 = precision == "bf16"
        return self

    def dead_parameters(self):
        return self.encoder.dead_parameters() + list(self.gate_fc.parameters())

    def live_parameters(self):
        dead = {id(p) for p in self.dead_parameters()}
        return [p for p in self.parameters() if id(p) not in dead]

    def flat_groups(self):
        """Parameters optim.FlatAdam should lay out back to back, so that the concatenated weights of the fused
        projections (q|k of a Combination, q|k|v of a self-attention, the 12 cross-attention k|v projections) and the
        (weight, bias) pair of every LayerNorm are single views of its flat buffers."""
        g = []
        for comb, gcn in zip(self.encoder.combination_list2, self.encoder.gcn_list):
            l = comb.linear_layers
            g += [[l[0].weight, l[1].weight], [l[0].bias, l[1].bias], [comb.layernorm.weight, comb.layernorm.bias],
                  [gcn.layernorm.weight, gcn.layernorm.bias]]
        dec = self.decoder
        for a, c, f in zip(dec.attention_list, dec.cross_attention_list, dec.feed_forward_list):
            g += [[a.fc_q.weight, a.fc_k.weight, a.fc_v.weight], [a.fc_q.bias, a.fc_k.bias, a.fc_v.bias],
                  [a.layernorm.weight, a.layernorm.bias], [c.layernorm.weight, c.layernorm.bias],
                  [f.layernorm.weight, f.layernorm.bias]]
        g.append([t for c in dec.cross_attention_list for t in (c.fc_k.weight, c.fc_v.weight)])
        g.append([t for c in dec.cross_attention_list for t in (c.fc_k.bias, c.fc_v.bias)])
        return g

    @staticmethod
    def shifted_label(tar_label):
        """Model.py:71-79: labels shifted left by one with a trailing 0."""
        pad = torch.zeros((tar_label.shape[0], 1), dtype=tar_label.dtype, device=tar_label.device)
        return torch.cat((tar_label[:, 1:], pad), dim=1)

    def forward_packed(self, pb, stage="train"):
        """The same computation on a per-commit PACKED batch (fira_icse_b200.packed.PackedBatch on this device, what
        PackedBatchLoader(packed=True) emits): node rows = the real nodes of every commit, no 210/160/280 padding
        (Dataset.py:80-94).  Loss, token count and gradients equal forward() on the padded batch; 'dev' ids number
        copy positions by the commit's own memory rows (V + m, m < code rows + sub-token rows)."""
        bf16 = self.precision == "bf16"
        if bf16:
            _optim.ensure_fresh(self)
        self.decoder.prefetch_weights()
        pf_head = ops.prefetch_head(bf16, self.out_fc.weight, self.copy_net.LinearSource.weight,
                                    self.copy_net.LinearTarget.weight)
        memory = self.encoder.encode_memory_packed(pb)                       # [1, Rc + Rs, D]
        if self._memory_hook is not None:
            memory = self._memory_hook(memory)
        want_ids = stage != "train"
        dec = self.decoder(pb.tar, memory, pb.mem_mask, pb.tar_mask, packed=pb, label=None if want_ids else pb.label)
        loss_sum, _, ids = ops.HeadFn.apply(want_ids, bf16, pf_head, memory, dec, pb.mem_mask, pb.label.view(-1),
                                            self.out_fc.weight, self.out_fc.bias, *self.copy_net.flat_params(), pb)
        if stage == "train":
            return loss_sum, (pb.label != 0).sum()
        elif stage == "dev" or stage == "test":
            return ids.long()
        raise ValueError(f"unknown stage {stage!r}")

    def forward(self, sou, tar, attr, mark, ast_change, edge, tar_label, sub_token, stage="train"):
        dev = self.out_fc.weight.device
        sou, tar, mark, ast_change, tar_label, sub_token = (
            t.to(dev, non_blocking=True) for t in (sou, tar, mark, ast_change, tar_label, sub_token))
        mem_mask = torch.cat((sou != 0, sub_token != 0), dim=1)
        bf16 = self.precision == "bf16"
        if bf16:
            _optim.ensure_fresh(self)            # parameters re-homed by optim.FlatAdam: bf16 mirror up to date
        self.decoder.prefetch_weights()          # decoder / head weight preparation overlaps with the encoder
        pf_head = ops.prefetch_head(bf16, self.out_fc.weight, self.copy_net.LinearSource.weight,
                                    self.copy_net.LinearTarget.weight) if sou.is_cuda else None
        memory = self.encoder.encode_memory(sou, mark, ast_change, edge, sub_token)
        if self._memory_hook is not None:
            memory = self._memory_hook(memory)
        dec = self.decoder(tar, memory, mem_mask, tar != 0)
        label = self.shifted_label(tar_label)
        want_ids = stage != "train"
        loss_sum, _, ids = ops.HeadFn.apply(want_ids, bf16, pf_head, memory, dec, _u8(mem_mask),
                                            _i32(label).view(-1),
                                            self.out_fc.weight, self.out_fc.bias, *self.copy_net.flat_params())
        if stage == "train":
            return loss_sum, (label != 0).sum()
        elif stage == "dev" or stage == "test":
            return ids.long()
        raise ValueError(f"unknown stage {stage!r}")
