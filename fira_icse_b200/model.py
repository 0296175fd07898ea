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
from types import SimpleNamespace

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
        # the constructor arguments as a plain attribute (no state_dict entry; a namespace, so deepcopy and pickle work
        # whatever type the caller used): optim.ema_model builds a twin from them.  Attributes win over mapping keys:
        # run_model.py's DotDict gets vocab_size by attribute assignment after it was built
        fields = dict(args) if isinstance(args, dict) else {}
        fields.update(getattr(args, "__dict__", {}))
        self.args = SimpleNamespace(**fields)
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

    def _prefetch(self):
        """Brings the bf16 mirror of parameters re-homed by optim.FlatAdam up to date, then starts the decoder's and the
        head's weight preparation, which overlaps with the encoder -> the head's prefetch (None off CUDA)."""
        bf16 = self.precision == "bf16"
        if bf16:
            _optim.ensure_fresh(self)
        self.decoder.prefetch_weights()
        if not self.out_fc.weight.is_cuda:
            return None
        return ops.prefetch_head(bf16, self.out_fc.weight, self.copy_net.LinearSource.weight,
                                 self.copy_net.LinearTarget.weight)

    def teacher_forced(self, sou, tar, mark, ast_change, edge, sub_token, pad_id=0, repeat=1):
        """The padded batch's teacher-forced pass up to the head, in the model's current mode and under autograd ->
        (head prefetch, memory [B', S, D], copy mask [B', S] = cat(sou != pad_id, sub_token != 0), decoder output
        [B', T, D] of tar masked by tar != pad_id), what head() takes.  The inputs are moved to the model's device.
        repeat = N > 1 replicates memory and mask N-fold along the batch (commit b -> rows b*N .. b*N + N-1; the
        encoder's gradient is the sum over the copies): tar then holds B' = B*N rows."""
        dev = self.out_fc.weight.device
        sou, tar, mark, ast_change, sub_token = (
            t.to(dev, non_blocking=True) for t in (sou, tar, mark, ast_change, sub_token))
        mem_mask = torch.cat((sou != pad_id, sub_token != 0), dim=1)
        pf_head = self._prefetch()
        memory = self.encoder.encode_memory(sou, mark, ast_change, edge, sub_token)
        if self._memory_hook is not None:
            memory = self._memory_hook(memory)
        if repeat > 1:
            def rep(x):
                return x.unsqueeze(1).expand(x.shape[0], repeat, *x.shape[1:]).reshape(-1, *x.shape[1:])
            memory, mem_mask = rep(memory), rep(mem_mask)
        return pf_head, memory, mem_mask, self.decoder(tar, memory, mem_mask, tar != pad_id)

    def head(self, pf_head, memory, mem_mask, dec, label, want_ids=False, pk=None, seq_weight=None, teacher=None,
             sparse=None):
        """ops.HeadFn on this model's head weights -> (loss_sum, per-position nll [B, T], argmax ids or None).  label:
        the shifted labels [B, T]; the objectives as HeadFn documents them."""
        return ops.HeadFn.apply(want_ids, self.precision == "bf16", pf_head, memory, dec, _u8(mem_mask),
                                _i32(label).view(-1), self.out_fc.weight, self.out_fc.bias,
                                *self.copy_net.flat_params(), pk, seq_weight, teacher, sparse)

    @staticmethod
    def _result(stage, loss_sum, ids, label):
        if stage == "train":
            return loss_sum, (label != 0).sum()
        elif stage == "dev" or stage == "test":
            return ids.long()
        raise ValueError(f"unknown stage {stage!r}")

    def forward_packed(self, pb, stage="train"):
        """The same computation on a per-commit PACKED batch (fira_icse_b200.packed.PackedBatch on this device, what
        PackedBatchLoader(packed=True) emits): node rows = the real nodes of every commit, no 210/160/280 padding
        (Dataset.py:80-94).  Loss, token count and gradients equal forward() on the padded batch; 'dev' ids number
        copy positions by the commit's own memory rows (V + m, m < code rows + sub-token rows)."""
        pf_head = self._prefetch()
        memory = self.encoder.encode_memory_packed(pb)                       # [1, Rc + Rs, D]
        if self._memory_hook is not None:
            memory = self._memory_hook(memory)
        want_ids = stage != "train"
        dec = self.decoder(pb.tar, memory, pb.mem_mask, pb.tar_mask, packed=pb, label=None if want_ids else pb.label)
        loss_sum, _, ids = self.head(pf_head, memory, pb.mem_mask, dec, pb.label, want_ids=want_ids, pk=pb)
        return self._result(stage, loss_sum, ids, pb.label)

    def forward(self, sou, tar, attr, mark, ast_change, edge, tar_label, sub_token, stage="train"):
        tar_label = tar_label.to(self.out_fc.weight.device, non_blocking=True)
        pf_head, memory, mem_mask, dec = self.teacher_forced(sou, tar, mark, ast_change, edge, sub_token)
        label = self.shifted_label(tar_label)
        loss_sum, _, ids = self.head(pf_head, memory, mem_mask, dec, label, want_ids=stage != "train")
        return self._result(stage, loss_sum, ids, label)
