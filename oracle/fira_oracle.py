"""CPU oracle for the FIRA hot path  --  TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs
may import this file.  The product (fira_icse_b200) never does, and fails loudly when
its CUDA library is missing.

It is a functional torch-CPU restatement (fp32, or fp64 on request) of the reference
algorithm, operating on a plain ``state_dict`` with the reference's 338 key names.  It
does what the reference does, the way the reference does it -- dense 650x650 adjacency
``bmm``, materialised copy tensor, materialised B x 30 x 25020 distribution -- so that
timing it is a fair stand-in for the reference CPU path, and so that its autograd
gradients are the gradient reference for the CUDA backward kernels.

Pinned against the unmodified reference by tests/test_oracle_golden.py using
tests/golden/model_first128.npz (made by tests/golden/make_golden.py from
/root/reference at commit 77b9a6a) and tests/golden/model_edge.npz (DataSet extremes and
crafted truncation commits, tests/golden/make_golden_edge.py).

Reference sites restated here (relative to /root/reference):
  position table .......... gnn_transformer.py:10-19
  Encoder.forward ......... gnn_transformer.py:45-62
  Combination(+Layer) ..... gnn_transformer.py:192-205, combination_layer.py:7-17
  GCN.forward ............. gnn_transformer.py:74-86
  Decoder.forward ......... gnn_transformer.py:108-122
  Attention.forward ....... gnn_transformer.py:137-161
  FeedForward.forward ..... gnn_transformer.py:170-174
  CopyNet.forward ......... Model.py:15-20
  TransModel.forward ...... Model.py:38-86
"""
import math

import torch
import torch.nn.functional as F

N_LAYERS = 6
LN_EPS = 1e-5


def position_table(length, dim, dtype=torch.float32):
    """sin/cos table; pair j shares the exponent 2j/dim (gnn_transformer.py:10-19)."""
    i = torch.arange(length, dtype=torch.float64).unsqueeze(1)
    j = torch.arange(dim // 2, dtype=torch.float64).unsqueeze(0)
    ang = i / torch.pow(torch.tensor(10000.0, dtype=torch.float64), 2.0 * j / dim)
    tab = torch.stack((torch.sin(ang), torch.cos(ang)), dim=-1).reshape(length, dim)
    return tab.to(dtype)


def _lin(sd, prefix, x):
    return F.linear(x, sd[prefix + ".weight"], sd.get(prefix + ".bias"))


def _ln(sd, prefix, x):
    return F.layer_norm(x, (x.shape[-1],), sd[prefix + ".weight"], sd[prefix + ".bias"], LN_EPS)


def _drop(x, p, training, masks=None, sid=0, rows=None):
    """dropout; with `masks` (a callable (stream id, row index tensor) -> bool keep mask [..., 256]) the given mask
    instead of torch's: x * keep / (1 - p32), p32 the fp32 value of p.  rows: the row index of every row of x
    (default: the flat row number over x's leading dims)."""
    if not (training and p > 0):
        return x
    if masks is None:
        return F.dropout(x, p, training)
    if rows is None:
        rows = torch.arange(x.numel() // x.shape[-1]).view(x.shape[:-1])
    keep = torch.as_tensor(masks(sid, rows)).reshape(x.shape)
    p32 = float(torch.tensor(p, dtype=torch.float32))
    return x * keep.to(x.dtype) / (1.0 - p32)


def combination(sd, prefix, x, mark_em, heads, p, training, masks=None, sid=0, rows=None):
    """Per-element two-way gate between key and value (combination_layer.py:7-17)
    wrapped by three input linears, an output linear, residual and post-LN
    (gnn_transformer.py:192-205).  masks: the gate's dropout uses stream `sid`, the LayerNorm's `sid + 1`."""
    dk = x.shape[-1] // heads
    q = _lin(sd, prefix + ".linear_layers.0", x)
    k = _lin(sd, prefix + ".linear_layers.1", x)
    v = _lin(sd, prefix + ".linear_layers.2", mark_em)
    pair_logits = torch.stack((q * k, q * v), dim=-1) / math.sqrt(dk)
    w = torch.softmax(pair_logits, dim=-1)
    mixed = w[..., 0] * k + w[..., 1] * v
    mixed = _drop(mixed, p, training, masks, sid, rows)
    y = _lin(sd, prefix + ".output_linear", mixed)
    return _ln(sd, prefix + ".layernorm", _drop(y, p, training, masks, sid + 1, rows) + x)


def gcn(sd, prefix, nodes, adj, p, training, masks=None, sid=2, rows=None):
    """LN(dropout(fc2(A @ fc1(H))) + H), dense batched adjacency (gnn_transformer.py:74-86)."""
    x = _lin(sd, prefix + ".fc1", nodes)
    x = torch.bmm(adj.to(x.dtype), x)
    x = _lin(sd, prefix + ".fc2", x)
    return _ln(sd, prefix + ".layernorm", _drop(x, p, training, masks, sid, rows) + nodes)


def encoder(sd, sou, mark, ast_change, adj, sub_token, *, heads=8, training=False,
            p_comb=0.1, p_gcn=0.2, collect=None, masks=None, stream_base=0):
    """gnn_transformer.py:45-62.  Returns (code rows [B,210,D], sub-token rows [B,160,D]).
    masks: dropout masks of the CUDA kernels -- layer i draws stream stream_base + 8 i + {0, 1, 2} (gate, Combination
    LayerNorm, GCN LayerNorm); code rows are numbered b * n_code + j, node rows segment-major (code rows of every
    commit, then sub-token rows, then AST rows)."""
    emb = sd["encoder.embedding.weight"]
    B, n_code, n_sub = sou.shape[0], sou.shape[1], sub_token.shape[1]
    n_ast = ast_change.shape[1]
    seg = torch.cat((torch.arange(B * n_code).view(B, n_code), B * n_code + torch.arange(B * n_sub).view(B, n_sub),
                     B * (n_code + n_sub) + torch.arange(B * n_ast).view(B, n_ast)), dim=1)
    code = emb[sou] + position_table(n_code, emb.shape[1], emb.dtype)
    mark_em = sd["encoder.mark_embedding.weight"][mark]
    ast = sd["encoder.ast_change_embedding.weight"][ast_change]
    sub = emb[sub_token]
    for i in range(N_LAYERS):
        sid = stream_base + 8 * i
        code = combination(sd, f"encoder.combination_list2.{i}", code, mark_em, heads, p_comb, training, masks, sid)
        nodes = torch.cat((code, sub, ast), dim=1)
        nodes = gcn(sd, f"encoder.gcn_list.{i}", nodes, adj, p_gcn, training, masks, sid + 2, seg)
        code, sub, ast = nodes[:, :n_code], nodes[:, n_code:n_code + n_sub], nodes[:, n_code + n_sub:]
        if collect is not None:
            collect.append(nodes)
    return code, sub


def attention(sd, prefix, query, memory, mask, heads, p, training, masks=None, sid=0, rows=None):
    """Post-LN multi-head attention, mask fill -1e9, no dropout on the weights
    (gnn_transformer.py:137-161).  mask broadcasts to [B, heads, Lq, Lk]."""
    B, Lq, D = query.shape
    Lk = memory.shape[1]
    dh = D // heads
    q = _lin(sd, prefix + ".fc_q", query).view(B, Lq, heads, dh).transpose(1, 2)
    k = _lin(sd, prefix + ".fc_k", memory).view(B, Lk, heads, dh).transpose(1, 2)
    v = _lin(sd, prefix + ".fc_v", memory).view(B, Lk, heads, dh).transpose(1, 2)
    score = torch.matmul(q, k.transpose(-2, -1)) / math.sqrt(dh)
    if mask.dim() < 4:
        mask = mask.unsqueeze(1).unsqueeze(1)
    score = score.masked_fill(mask == 0, -1e9)
    ctx = torch.matmul(torch.softmax(score, dim=-1), v)
    ctx = ctx.transpose(1, 2).reshape(B, Lq, D)
    y = _lin(sd, prefix + ".fc_o", ctx)
    return _ln(sd, prefix + ".layernorm", _drop(y, p, training, masks, sid, rows) + query)


def feed_forward(sd, prefix, x, p, training, masks=None, sid=2, rows=None):
    """gnn_transformer.py:170-174."""
    y = _lin(sd, prefix + ".fc2", F.relu(_lin(sd, prefix + ".fc1", x)))
    return _ln(sd, prefix + ".layernorm", _drop(y, p, training, masks, sid, rows) + x)


def decoder(sd, tar, memory, mem_mask, tar_pad_mask, *, heads=8, training=False, p=0.1, masks=None, stream_base=0):
    """gnn_transformer.py:108-122.  Self-attention keys are masked by pad AND causal.
    masks: layer i draws stream stream_base + 64 + 8 i + {0, 1, 2} (self-attention, cross-attention, FFN), rows b * T + t."""
    emb = sd["decoder.embedding.weight"]
    T = tar.shape[1]
    x = emb[tar] + position_table(T, emb.shape[1], emb.dtype)
    causal = torch.tril(torch.ones(T, T, dtype=torch.bool))
    self_mask = tar_pad_mask[:, None, None, :] & causal[None, None]
    for i in range(N_LAYERS):
        sid = stream_base + 64 + 8 * i
        x = attention(sd, f"decoder.attention_list.{i}", x, x, self_mask, heads, p, training, masks, sid)
        x = attention(sd, f"decoder.cross_attention_list.{i}", x, memory, mem_mask, heads, p, training, masks, sid + 1)
        x = feed_forward(sd, f"decoder.feed_forward_list.{i}", x, p, training, masks, sid + 2)
    return x


def copy_net(sd, memory, tar_em):
    """Pointer scores and 2-way gate (Model.py:15-20); materialises [B,T,S,D] like the reference."""
    src = F.linear(memory, sd["copy_net.LinearSource.weight"])
    tgt = F.linear(tar_em, sd["copy_net.LinearTarget.weight"])
    scores = _lin(sd, "copy_net.LinearRes", torch.tanh(src.unsqueeze(1) + tgt.unsqueeze(2))).squeeze(-1)
    gate = torch.softmax(_lin(sd, "copy_net.LinearProb", tar_em), dim=-1)
    return scores, gate


def output_distribution(sd, memory, mem_mask, dec):
    """[g0 * softmax(out_fc) || g1 * softmax(masked copy)] then log(clamp) (Model.py:54-69)."""
    gen = torch.softmax(_lin(sd, "out_fc", dec), dim=-1)
    scores, gate = copy_net(sd, memory, dec)
    scores = scores.masked_fill(mem_mask.unsqueeze(1) == 0, -1e9)
    ptr = torch.softmax(scores, dim=-1)
    dist = torch.cat((gate[..., 0:1] * gen, gate[..., 1:2] * ptr), dim=-1)
    return torch.log(dist.clamp(min=1e-10, max=1.0)), dist


def shifted_labels(tar_label):
    """Labels shifted left with a trailing 0 (Model.py:71-79)."""
    pad = torch.zeros(tar_label.shape[0], 1, dtype=tar_label.dtype)
    return torch.cat((tar_label, pad), dim=-1)[:, 1:].long()


def forward(sd, sou, tar, attr, mark, ast_change, edge, tar_label, sub_token, stage="train",
            training=False, detail=None, masks=None):
    """TransModel.forward (Model.py:38-86).  `attr` is accepted and ignored, as upstream.
    masks: callable (stream id, row index tensor) -> keep mask [..., 256]; dropout then applies the masks the CUDA
    kernels draw (tests/philox_rule.py) instead of torch's."""
    sou_mask = sou != 0
    code, sub = encoder(sd, sou, mark, ast_change, edge, sub_token, training=training, masks=masks)
    memory = torch.cat((code, sub), dim=1)
    mem_mask = torch.cat((sou_mask, sub_token != 0), dim=1)
    dec = decoder(sd, tar, memory, mem_mask, tar != 0, training=training, masks=masks)
    logp, _ = output_distribution(sd, memory, mem_mask, dec)
    label = shifted_labels(tar_label)
    keep = label != 0
    nll = F.nll_loss(logp.reshape(-1, logp.shape[-1]), label.reshape(-1), reduction="none")
    nll = nll.masked_fill(~keep.reshape(-1), 0)
    if detail is not None:
        detail.update(memory=memory, decoder=dec, logp=logp, nll=nll.view_as(label), mem_mask=mem_mask)
    if stage == "train":
        return nll.sum(), keep.sum()
    return torch.argmax(logp, dim=-1)


def dense_adjacency(rows, cols, vals, n=650, dtype=torch.float64):
    """COO -> dense, duplicates summed, exactly what Dataset.py:340 `toarray()` hands the model."""
    a = torch.zeros(n, n, dtype=dtype)
    a.index_put_((torch.as_tensor(rows).long(), torch.as_tensor(cols).long()),
                 torch.as_tensor(vals).to(dtype), accumulate=True)
    return a


def random_state_dict(vocab_size=24650, ast_vocab_size=71, dim=256, seed=0):
    """Reference-shaped parameters (the live ones of SURVEY.md 9.1) with nn.Linear/nn.Embedding-style
    initial distributions -- for timing the oracle without touching any product code."""
    g = torch.Generator().manual_seed(seed)
    sd = {}

    def emb(name, n):
        sd[name] = torch.randn(n, dim, generator=g)

    def lin(name, out_f, in_f, bias=True):
        bound = 1.0 / math.sqrt(in_f)
        sd[name + ".weight"] = (torch.rand(out_f, in_f, generator=g) * 2 - 1) * bound
        if bias:
            sd[name + ".bias"] = (torch.rand(out_f, generator=g) * 2 - 1) * bound

    def ln(name):
        sd[name + ".weight"], sd[name + ".bias"] = torch.ones(dim), torch.zeros(dim)

    emb("encoder.embedding.weight", vocab_size)
    emb("encoder.ast_change_embedding.weight", ast_vocab_size)
    emb("encoder.mark_embedding.weight", 4)
    emb("decoder.embedding.weight", vocab_size)
    for i in range(N_LAYERS):
        c = f"encoder.combination_list2.{i}"
        for j in range(3):
            lin(f"{c}.linear_layers.{j}", dim, dim)
        lin(f"{c}.output_linear", dim, dim); ln(f"{c}.layernorm")
        gname = f"encoder.gcn_list.{i}"
        lin(f"{gname}.fc1", dim, dim); lin(f"{gname}.fc2", dim, dim); ln(f"{gname}.layernorm")
        for blk in ("attention_list", "cross_attention_list"):
            a = f"decoder.{blk}.{i}"
            for nm in ("fc_q", "fc_k", "fc_v", "fc_o"):
                lin(f"{a}.{nm}", dim, dim)
            ln(f"{a}.layernorm")
        f = f"decoder.feed_forward_list.{i}"
        lin(f"{f}.fc1", 4 * dim, dim); lin(f"{f}.fc2", dim, 4 * dim); ln(f"{f}.layernorm")
    lin("out_fc", vocab_size, dim)
    lin("copy_net.LinearSource", dim, dim, bias=False)
    lin("copy_net.LinearTarget", dim, dim, bias=False)
    lin("copy_net.LinearRes", 1, dim)
    lin("copy_net.LinearProb", 2, dim)
    return sd


def train_step(sd_params, optimizer, batch):
    """One reference training step (run_model.py:101-109): loss = sum/sum, backward, Adam."""
    loss_sum, n_tok = forward(sd_params, *batch, stage="train", training=True)
    loss = loss_sum / n_tok
    optimizer.zero_grad()
    loss.backward()
    optimizer.step()
    return float(loss.detach())
