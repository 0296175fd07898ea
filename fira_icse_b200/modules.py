"""nn.Module surface of the reference's gnn_transformer.py / combination_layer.py, re-hosted on
libfira_b200.

Every class keeps the reference's name, constructor signature, parameter names, shapes and
REGISTRATION ORDER (so `torch.manual_seed(0)` initialisation is bit-identical and the 338-key
state_dict interchanges with reference checkpoints, SURVEY.md 9.1) -- including the three dead
blocks `encoder.lstm`, `encoder.combination_list1` and `gate_fc`.  The sub-modules are parameter
containers: the arithmetic runs in the fused Encoder/Decoder autograd Functions of ops.py, which
launch the CUDA kernels.  There is no CPU execution path.
"""
import math

import torch
import torch.nn as nn

from . import ops
from .graph import PackedEdges


def position_encoding(length, dmodel):
    """Sin/cos table of gnn_transformer.py:10-19 (pair j uses exponent 2j/dmodel for both), fp32."""
    inv = [10000 ** (2 * j / dmodel) for j in range(dmodel // 2)]
    rows = []
    for i in range(length):
        row = [0.0] * dmodel
        for j, f in enumerate(inv):
            a = i / f
            row[2 * j] = math.sin(a)
            row[2 * j + 1] = math.cos(a)
        rows.append(row)
    return torch.tensor(rows)


def _i32(t):
    return t.to(torch.int32).contiguous()


def _u8(t):
    return t.to(torch.uint8).contiguous()


class _KernelBacked(nn.Module):
    """Parameter container.  Inside the model its arithmetic is executed by the enclosing fused Function
    (ops.EncoderFn / DecoderFn); called on its own, `forward` runs the same CUDA kernels block by block with the
    reference's signature (fira_icse_b200/blocks.py), so the class is a drop-in by itself too."""


class CombinationLayer(_KernelBacked):
    """combination_layer.py:6-17 (parameter-free gate); fused into fira_comb_gate_fwd/bwd."""

    def forward(self, query, key, value, dropout=None):
        from . import blocks
        return blocks.combination_layer_forward(query, key, value, dropout)


class Combination(_KernelBacked):
    """gnn_transformer.py:176-205."""

    def __init__(self, h, d_model, dropout_rate=0.1):
        super().__init__()
        assert d_model % h == 0
        self.d_k = d_model // h
        self.h = h
        self.linear_layers = nn.ModuleList([nn.Linear(d_model, d_model) for _ in range(3)])
        self.output_linear = nn.Linear(d_model, d_model)
        self.combination = CombinationLayer()
        self.dropout = nn.Dropout(p=dropout_rate)
        self.layernorm = nn.LayerNorm(d_model)

    def flat_params(self):
        l = self.linear_layers
        return [l[0].weight, l[0].bias, l[1].weight, l[1].bias, l[2].weight, l[2].bias,
                self.output_linear.weight, self.output_linear.bias, self.layernorm.weight, self.layernorm.bias]

    def forward(self, query, key, value, mask=None):
        from . import blocks
        return blocks.combination_forward(self, query, key, value, mask)


class GCN(_KernelBacked):
    """gnn_transformer.py:64-86."""

    def __init__(self, dmodel, dropout_rate=0.1):
        super().__init__()
        self.dmodel = dmodel
        self.fc1 = nn.Linear(dmodel, dmodel)
        self.fc2 = nn.Linear(dmodel, dmodel)
        self.dropout = nn.Dropout(dropout_rate)
        self.layernorm = nn.LayerNorm(dmodel)

    def flat_params(self):
        return [self.fc1.weight, self.fc1.bias, self.fc2.weight, self.fc2.bias,
                self.layernorm.weight, self.layernorm.bias]

    def forward(self, graph_em, edge, code_len, sub_token_len, ast_change_len):
        from . import blocks
        return blocks.gcn_forward(self, graph_em, edge, code_len, sub_token_len, ast_change_len)


class Attention(_KernelBacked):
    """gnn_transformer.py:124-161."""

    def __init__(self, dmodel, num_head, dropout_rate=0.1):
        super().__init__()
        self.fc_q = nn.Linear(dmodel, dmodel)
        self.fc_k = nn.Linear(dmodel, dmodel)
        self.fc_v = nn.Linear(dmodel, dmodel)
        self.fc_o = nn.Linear(dmodel, dmodel)
        self.layernorm = nn.LayerNorm(dmodel)
        self.dropout = nn.Dropout(dropout_rate)
        self.num_head = num_head
        assert dmodel % self.num_head == 0
        self.dhead = dmodel // self.num_head

    def flat_params(self):
        return [self.fc_q.weight, self.fc_q.bias, self.fc_k.weight, self.fc_k.bias, self.fc_v.weight,
                self.fc_v.bias, self.fc_o.weight, self.fc_o.bias, self.layernorm.weight, self.layernorm.bias]

    def forward(self, query, key, value, mask):
        from . import blocks
        return blocks.attention_forward(self, query, key, value, mask)


class FeedForward(_KernelBacked):
    """gnn_transformer.py:163-174."""

    def __init__(self, dmodel, dropout_rate=0.1):
        super().__init__()
        self.fc1 = nn.Linear(dmodel, 4 * dmodel)
        self.fc2 = nn.Linear(4 * dmodel, dmodel)
        self.dropout = nn.Dropout(dropout_rate)
        self.layernorm = nn.LayerNorm(dmodel)

    def flat_params(self):
        return [self.fc1.weight, self.fc1.bias, self.fc2.weight, self.fc2.bias,
                self.layernorm.weight, self.layernorm.bias]

    def forward(self, input_em):
        from . import blocks
        return blocks.feed_forward_forward(self, input_em)


def _run_cfg(module, stream_base=0):
    return {"training": module.training, "seed": ops.make_seed() if module.training else 0,
            "stream_base": stream_base, "heads": module.num_head, "bf16": bool(getattr(module, "bf16", False)),
            "seed_ctr": getattr(module, "seed_ctr", None)}


class Encoder(nn.Module):
    """gnn_transformer.py:21-62.  forward(...) -> (code rows [B,210,D], sub-token rows [B,160,D])."""

    def __init__(self, args, pad_token_id):
        super().__init__()
        self.dropout_rate = args.dropout_rate
        self.sou_len = args.sou_len
        self.att_len = args.att_len
        self.ast_change_len = args.ast_change_len
        self.sub_token_len = args.sub_token_len
        self.embedding_dim = args.embedding_dim
        self.num_head = args.num_head
        self.pad_token_id = pad_token_id
        if args.embedding_dim != ops.D:
            raise ValueError("fira_icse_b200 kernels are specialised for embedding_dim == 256")
        self.embedding = nn.Embedding(num_embeddings=args.vocab_size, embedding_dim=args.embedding_dim,
                                      padding_idx=pad_token_id)
        self.ast_change_embedding = nn.Embedding(num_embeddings=args.ast_change_vocab_size,
                                                 embedding_dim=args.embedding_dim, padding_idx=pad_token_id)
        self.pos_encode = position_encoding(args.sou_len, self.embedding_dim)
        self.mark_embedding = nn.Embedding(num_embeddings=4, embedding_dim=args.embedding_dim, padding_idx=0)
        # dead in the reference forward, kept for checkpoint compatibility (gnn_transformer.py:40-41)
        self.lstm = nn.LSTM(input_size=args.embedding_dim, hidden_size=args.embedding_dim, num_layers=3,
                            batch_first=True)
        self.combination_list1 = nn.ModuleList(
            [Combination(h=args.num_head, d_model=args.embedding_dim) for _ in range(6)])
        self.combination_list2 = nn.ModuleList(
            [Combination(h=args.num_head, d_model=args.embedding_dim) for _ in range(6)])
        self.gcn_list = nn.ModuleList([GCN(args.embedding_dim, dropout_rate=0.2) for _ in range(6)])

    def _pos(self, device):
        if self.pos_encode.device != device:
            self.pos_encode = self.pos_encode.to(device)
        return self.pos_encode

    def dead_parameters(self):
        """Parameters the forward never touches (never receive gradients; excluded from the DP reducer)."""
        return list(self.lstm.parameters()) + list(self.combination_list1.parameters())

    def encode_memory(self, input_token, mark, ast_change, edge, sub_token):
        """-> memory [B, sou_len + sub_token_len, D] = cat(code rows, sub-token rows) (Model.py:48)."""
        dev = self.embedding.weight.device
        if not isinstance(edge, PackedEdges):
            edge = PackedEdges.from_dense(edge.to(dev))
        cfg = _run_cfg(self)
        cfg.update(p_comb=self.combination_list2[0].dropout.p, p_gcn=self.gcn_list[0].dropout.p)
        lp = []
        for comb, gcn in zip(self.combination_list2, self.gcn_list):
            lp += comb.flat_params() + gcn.flat_params()
        return ops.EncoderFn.apply(cfg, _i32(input_token), _i32(mark), _i32(ast_change), _i32(sub_token), edge,
                                   self._pos(dev), self.embedding.weight, self.ast_change_embedding.weight,
                                   self.mark_embedding.weight, *lp)

    def encode_memory_packed(self, pb):
        """Packed batch (fira_icse_b200.packed.PackedBatch on this device) -> memory rows [1, Rc + Rs, D]: the code rows
        then the sub-token rows of every commit (commit b owns the two row ranges pb.ranges[b]).  The batch runs as ONE
        ragged graph through the same kernels (B = 1, segments = the three row blocks, global adjacency)."""
        dev = self.embedding.weight.device
        cfg = _run_cfg(self)
        cfg.update(p_comb=self.combination_list2[0].dropout.p, p_gcn=self.gcn_list[0].dropout.p, pos=pb.pos)
        lp = []
        for comb, gcn in zip(self.combination_list2, self.gcn_list):
            lp += comb.flat_params() + gcn.flat_params()
        edges = PackedEdges(pb.rowptr, pb.col, pb.val, 1, pb.rows, True)
        return ops.EncoderFn.apply(cfg, pb.code.view(1, -1), pb.mark.view(1, -1), pb.ast.view(1, -1), pb.sub.view(1, -1),
                                   edges, self._pos(dev), self.embedding.weight, self.ast_change_embedding.weight,
                                   self.mark_embedding.weight, *lp)

    def forward(self, input_token, sou_mask, attr, mark, ast_change, edge, sub_token):
        # `attr` and `sou_mask` are accepted and unused, exactly like gnn_transformer.py:45
        memory = self.encode_memory(input_token, mark, ast_change, edge, sub_token)
        n_code = input_token.shape[1]                 # == sou_len unless the loader trimmed the padding
        return memory[:, :n_code], memory[:, n_code:]


class Decoder(nn.Module):
    """gnn_transformer.py:88-122."""

    def __init__(self, args, pad_token_id):
        super().__init__()
        self.embedding_dim = args.embedding_dim
        self.num_head = args.num_head
        self.pad_token_id = pad_token_id
        self.embedding = nn.Embedding(num_embeddings=args.vocab_size, embedding_dim=args.embedding_dim)
        self.pos_encode = position_encoding(args.tar_len, self.embedding_dim)
        self.tar_mask_pos = torch.tril(torch.ones(args.tar_len, args.tar_len))
        self.attention_list = nn.ModuleList(
            [Attention(dmodel=args.embedding_dim, num_head=args.num_head) for _ in range(6)])
        self.cross_attention_list = nn.ModuleList(
            [Attention(dmodel=args.embedding_dim, num_head=args.num_head) for _ in range(6)])
        self.feed_forward_list = nn.ModuleList([FeedForward(args.embedding_dim) for _ in range(6)])

    def _flat(self):
        lp = []
        for a, c, f in zip(self.attention_list, self.cross_attention_list, self.feed_forward_list):
            lp += a.flat_params() + c.flat_params() + f.flat_params()
        return lp

    def prefetch_weights(self):
        """Start this decoder's weight preparation on the side stream (TransModel.forward calls it before
        the encoder so that it overlaps with the encoder); the next forward() consumes it."""
        dev = self.embedding.weight.device
        if dev.type == "cuda":
            self._prefetched = ops.prefetch_decoder(bool(getattr(self, "bf16", False)), self._flat(), dev)

    def forward(self, output_token, input_em, sou_mask, tar_mask_pad, packed=None, label=None):
        """packed: a packed.PackedBatch -- `input_em` is then the [1, Rc + Rs, D] memory-row matrix of
        Encoder.encode_memory_packed and `sou_mask` the [B, S] mask over each commit's own memory rows.
        label (packed training batches): the shifted labels [B, T]; the bf16 mode then computes the gradient on the rows
        before each commit's last label only, and the output rows after it are zero (ops.DecoderFn)"""
        dev = self.embedding.weight.device
        if self.pos_encode.device != dev:
            self.pos_encode = self.pos_encode.to(dev)
        cfg = _run_cfg(self)
        cfg.update(p_dec=self.attention_list[0].dropout.p, prefetch=getattr(self, "_prefetched", None), packed=packed,
                   label=None if label is None else _i32(label))
        self._prefetched = None
        lp = self._flat()
        return ops.DecoderFn.apply(cfg, _i32(output_token), input_em, _u8(sou_mask), _u8(tar_mask_pad),
                                   self.pos_encode, self.embedding.weight, *lp)
