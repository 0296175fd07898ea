"""The bf16 training step (bf16 activations, wgmma GEMMs, MMA attention, fira_decoder_fwd) against float64, element by
element and row by row (tests/bf16_bound.py), at the level of the autograd Functions and of the whole graphed step.

ops.EncoderFn, ops.DecoderFn and ops.HeadFn are called directly with cfg["bf16"] = True, so the checks see their Python
wiring as well as the kernels: which saved tensor feeds which product, the accumulate= flags, the dropout site of every
backward, the side-stream forks, the vocabulary-row slots, the `active` flags and the packed row ranges.  Each compares
the forward output and EVERY gradient the Function returns (inputs and parameters; the decoder's hoisted K/V weight
gradient comes back split into its per-layer parameters) with float64 autograd of the oracle's own blocks
(oracle/fira_oracle.py) on the same inputs:

  * inputs are bf16 values; the GEMM weights Prec.w hands the kernels are rounded to bf16 in the reference as well;
    biases, LayerNorm parameters, the value table of the Combination gate, the embeddings and the fp32 gate of the head
    stay float64.  The bf16 rounding of the merged GCN weight W2 W1 stays inside the bound;
  * dropout applies the masks the kernels draw (tests/philox_rule.py) through the oracle's `masks` hook.

Where the error comes from, per stage (u = 2^-8, one bf16 rounding):
  * HeadFn: dec and memory are exact bf16 inputs; the logits, the pointer-score projections src / tgt and the
    vocabulary-gradient d_logits are each rounded once to bf16 (a few u relative, before the fp32 softmax / tanh),
    d_dec accumulates in fp32.  The logits enter the softmax as a difference of O(1) numbers, so their rounding is an
    absolute error of ~u on every probability's exponent.
  * DecoderFn, one layer: ~10 roundings in a row -- the layer input, Q/K/V, attention's bf16 P (forward) and dS
    (backward) inside the MMA kernel, the context, the three output projections before their LayerNorms, the 1024-wide
    hidden layer, and the same again on the gradient path (dZ, dctx, dQKV, dHh).  LayerNorm renormalises each row, so
    the forward error stays at a few u; the backward of softmax turns the rounding of P and dS into an error relative
    to the row's gradient norm, the largest single term.  Six layers: the errors of the layers add.
  * EncoderFn, one layer: the gate input q|k, the gate output, Z of the Combination, the GCN aggregate A H, the merged
    weight W2 W1 and Z of the GCN layer, then the gradient path through the same points.  The GCN sums up to ~40
    neighbours per row, so an aggregate's rounding is relative to the sum, not to each term.
  * The whole step: the encoder's six layers feed the decoder's six layers and the head; the reference there keeps
    fp32 weights, so the weight rounding of Prec.w adds to it.
  * The decoder FFN's fc1 gradients also carry the ReLU gates bf16 decides differently from float64 (gate_allowance,
    ~2.5 % of the gates): without the allowance the one-layer fc1 error is ~2.3x the 2^-5 bound, with it < 0.1x.

Each eps below is the smallest power of two at least twice the worst error measured on an H100 SXM (80 GB, 700 W
power limit) -- the printed "[bf16 bound]" lines give it as a fraction of its bound (worst: head 0.38, one decoder
layer 0.51, six 0.41, one encoder layer 0.29, six 0.51, whole step 0.30).  A one-layer eps may not exceed 2^-5.  The
decoder on the live-row map and the graph replayed across batches reach 0.56 (one layer: the self-attention fc_q
gradient under dropout, whose loss gradient lives on 74 of 180 rows), 0.51 (six layers) and 0.52 (the whole-step
loss, 1.3e-4 relative), measured on the same card."""
import copy

import numpy as np
import pytest
import torch

import philox_rule as R
from bf16_bound import close, small, vanishing
from fira_testlib import golden_batch, seeded_model

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SEED = 20241016
V = 24650
D = 256
T = 30

EPS_HEAD = 2 ** -7
EPS_DEC = {1: 2 ** -5, 6: 2 ** -3}
EPS_ENC = {1: 2 ** -5, 6: 2 ** -4}
EPS_STEP = 2 ** -3                                  # the whole step: six encoder + six decoder layers + the head
LOSS_REL = 2 ** -12                                 # the whole-step loss, relative (measured worst 9.7e-5)
# the decoder cases scale every fc_q weight by Q_SCALE: at the initial weights the attention scores have a standard
# deviation of ~0.3, the softmax is nearly uniform and the query gradient dQ is ~1 % of the layer's input gradient,
# too small for any rounding bound to see it dropped; x8 gives scores of ~2.6, a peaked softmax as in a trained model
Q_SCALE = 8.0
RELU_TAU = 2 ** -5                                  # 8 bf16 roundings of the FFN pre-activation's scale

PACKED_INDEX = [100, 3, 77, 127, 64, 9]             # tests/test_gpu_packed.py
HEAD_INDEX = [0, 5, 9, 64, 77, 100]


@pytest.fixture(scope="module", autouse=True)
def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


@pytest.fixture(scope="module")
def model():
    m = seeded_model()                              # CPU: the parameters are copied to the device per test
    return m


def _names(model):
    return {id(p): k for k, p in model.named_parameters()}


def _leaves(model, tensors, rounded):
    """-> (names, device fp32 leaves, float64 state dict with the bf16-rounded GEMM weights where rounded(name))"""
    nm = _names(model)
    names = [nm[id(t)] for t in tensors]
    dev = [t.detach().to(DEV).clone().requires_grad_(True) for t in tensors]
    sd = {}
    for k, t in zip(names, tensors):
        v = t.detach().to(torch.bfloat16).double() if rounded(k) else t.detach().double()
        sd[k] = v.clone().requires_grad_(True)
    return names, dev, sd


def _bf16_randn(shape, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(shape, generator=g).to(torch.bfloat16).float()


def _check_grads(tag, names, leaves, sd, eps, rows=(), allow=None):
    """every parameter gradient against the reference; rows: names checked per row as well; allow: {name: element-wise
    allowance}"""
    worst = 0.0
    for k, t in zip(names, leaves):
        ref = sd[k].grad
        assert t.grad is not None, f"{tag} {k}: no gradient"
        if vanishing(k):
            pair = sd[k[:-len("bias")] + "weight"].grad
            worst = max(worst, small(f"{tag} {k}", t.grad, pair.abs().max().item(), eps))
            continue
        worst = max(worst, close(f"{tag} {k}", t.grad, ref, eps, rows=k in rows, allow=(allow or {}).get(k)))
    return worst


def _drop_masks(seed, p_of_sid):
    def masks(sid, rows):
        shape = tuple(rows.shape)
        k = R.keep_mask(seed, 0, sid, rows.reshape(-1).numpy(), p_of_sid(sid))
        return torch.from_numpy(k).view(*shape, R.D)
    return masks


def _packed(index, pad=False):
    from fira_icse_b200.packed import PackedSlot, PackedTables, pack_from_dataset, packed_needs
    from test_packed import GoldenSplit
    tables = PackedTables(GoldenSplit())
    pad_dims = None
    if pad:                                         # every segment padded to the staging capacity, 128 spare vocab slots
        cap = PackedSlot(len(index), tables.lens, tables.msg_len, 1, False).cap
        pad_dims = tuple(cap) + (packed_needs(tables, np.asarray(index), V)[4] + 128,)
    return pack_from_dataset(tables, np.asarray(index), V, pad_dims=pad_dims)


def _commit_rows(pk):
    """[B, S] index of commit b's memory position m in the packed memory rows (0 where masked) and the [B, S] mask"""
    rng = pk.ranges.cpu().numpy()
    B, S = pk.B, pk.S
    idx = np.zeros((B, S), np.int64)
    for b in range(B):
        c0, n0, s0, n1 = (int(x) for x in rng[b])
        idx[b, :n0] = c0 + np.arange(n0)
        idx[b, n0:n0 + n1] = s0 + np.arange(n1)
    return torch.from_numpy(idx), pk.mem_mask.cpu().bool()


# ============================================================================= HeadFn
HEAD_PARAMS = ("out_fc.weight", "out_fc.bias", "copy_net.LinearSource.weight", "copy_net.LinearTarget.weight",
               "copy_net.LinearRes.weight", "copy_net.LinearRes.bias", "copy_net.LinearProb.weight",
               "copy_net.LinearProb.bias")
HEAD_ROUNDED = ("out_fc.weight", "copy_net.LinearSource.weight", "copy_net.LinearTarget.weight")


def _edit_labels(label, mem_valid):
    """label [B, T] int: commit 0 gets a zero label inside its message, commit 1 no label at all, commit 2 copy labels
    only (valid memory positions of its own)"""
    label = label.clone()
    n0 = int((label[0] != 0).sum())
    assert n0 > 4
    label[0, 2] = 0
    label[1] = 0
    pos = torch.nonzero(mem_valid[2]).view(-1)
    label[2] = 0
    label[2, :10] = V + pos[torch.arange(10) * 7 % len(pos)]
    return label


@pytest.mark.parametrize("layout", ["padded", "packed", "packed_bucket"])
def test_head_fn_matches_float64(model, layout):
    from fira_icse_b200 import ops
    import fira_oracle as O
    pk = None
    if layout == "padded":
        parts = [golden_batch(i, i + 1) for i in HEAD_INDEX]
        sou, tar_label, sub = (torch.cat([p[k] for p in parts], 0) for k in (0, 6, 7))
        mem_valid = torch.cat((sou != 0, sub != 0), 1)
        label = _edit_labels(torch.cat((tar_label[:, 1:], torch.zeros_like(tar_label[:, :1])), 1), mem_valid)
        B, S = label.shape[0], mem_valid.shape[1]
        memory = _bf16_randn((B, S, D), 1)
        mem_mask_dev = mem_valid.to(torch.uint8).to(DEV)
        label_dev = label.to(torch.int32).reshape(-1).to(DEV)
    else:
        pk = _packed(HEAD_INDEX, pad=layout == "packed_bucket").to(DEV)
        idx, mem_valid = _commit_rows(pk)
        label = _edit_labels(pk.label.cpu().long(), mem_valid)
        pk.label.copy_(label.to(torch.int32))
        B, S = pk.B, pk.S
        memory = _bf16_randn((1, pk.mem_rows, D), 1)
        mem_mask_dev, label_dev = pk.mem_mask, pk.label.reshape(-1)
    names, params, sd = _leaves(model, [dict(model.named_parameters())[k] for k in HEAD_PARAMS],
                                lambda k: k in HEAD_ROUNDED)
    dec = _bf16_randn((B, T, D), 2)
    m_dev = memory.to(DEV).requires_grad_(True)
    d_dev = dec.to(DEV).requires_grad_(True)
    loss, nll, _ = ops.HeadFn.apply(False, True, None, m_dev, d_dev, mem_mask_dev, label_dev, *params, pk)
    loss.backward()
    torch.cuda.synchronize()

    m64 = memory.double().requires_grad_(True)
    d64 = dec.double().requires_grad_(True)
    mem_b = m64 if pk is None else m64[0][idx]
    logp, _ = O.output_distribution(sd, mem_b, mem_valid, d64)
    keep = label != 0
    ref_nll = -logp.gather(-1, label.unsqueeze(-1)).squeeze(-1) * keep
    ref_nll.sum().backward()
    eps, tag = EPS_HEAD, f"head/{layout}"
    close(f"{tag} loss", loss, ref_nll.sum(), eps)
    close(f"{tag} nll", nll.reshape(B, T), ref_nll, eps, rows=True)
    assert (nll.reshape(B, T).cpu()[~keep] == 0).all()
    close(f"{tag} d_dec", d_dev.grad, d64.grad, eps, rows=True)
    assert (d_dev.grad[1].abs().sum() == 0).item(), "a commit without labels has no gradient"
    close(f"{tag} d_memory", m_dev.grad, m64.grad, eps, rows=True)
    _check_grads(tag, names, params, sd, eps)


# ============================================================================= DecoderFn
DEC_BLOCKS = ("attention_list", "cross_attention_list", "feed_forward_list")


def _feed_forward(sd, prefix, x, p, training, masks=None, sid=2, rows=None, gates=None):
    """oracle.feed_forward, keeping (input, pre-activation, ReLU output, fc1 weight) in `gates` for the gate allowance"""
    import fira_oracle as O
    h = O._lin(sd, prefix + ".fc1", x)
    a = torch.relu(h)
    a.retain_grad()
    gates[prefix] = (x, h, a, sd[prefix + ".fc1.weight"])
    y = O._lin(sd, prefix + ".fc2", a)
    return O._ln(sd, prefix + ".layernorm", O._drop(y, p, training, masks, sid, rows) + x)


def record_gates(monkeypatch, gates):
    """make the oracle's decoder (oracle.forward / oracle.decoder) record its FFN gates into `gates`"""
    import functools
    import fira_oracle as O
    monkeypatch.setattr(O, "feed_forward", functools.partial(_feed_forward, gates=gates))


def gate_allowance(gates, tag):
    """bf16 evaluates each FFN pre-activation h = x W1^T + b1 with an error of a few roundings of its terms: about
    u sqrt(sum_k (x_k W1_jk)^2), u = 2^-8, from the bf16 input x (plus the error x carries from the layers before).  A
    ReLU gate whose float64 h lies within RELU_TAU = 8 u of that scale may open in the bf16 forward and stay shut in
    float64 (or the other way round); it then moves its whole term dA_ij x_i in or out of the column sums of the fc1
    gradients, a few per cent of the largest element and far above any rounding bound.  The fc1 checks allow the terms
    of exactly those gates: -> {param name: allowance}; prints the share of gates that get one."""
    out, n_amb, n_all = {}, 0, 0
    for prefix, (x, h, a, W) in gates.items():
        W = W.detach()
        x2, h2, dA = x.detach().reshape(-1, D), h.detach().reshape(-1, W.shape[0]), a.grad.reshape(-1, W.shape[0])
        amb = (h2.abs() <= RELU_TAU * ((x2 * x2) @ (W * W).t()).sqrt()).double()
        n_amb, n_all = n_amb + int(amb.sum()), n_all + amb.numel()
        out[prefix + ".fc1.weight"] = (amb * dA.abs()).t() @ x2.abs()
        out[prefix + ".fc1.bias"] = (amb * dA.abs()).sum(0)
    print(f"[bf16 bound] {tag}: {n_amb} of {n_all} ReLU gates ({100.0 * n_amb / max(n_all, 1):.2f} %) within the "
          f"rounding of h")
    return out


def _dec_ref(sd, tar, memory, mem_mask, tar_mask, L, p, masks, gates):
    """oracle.decoder with L layers"""
    import fira_oracle as O
    emb = sd["decoder.embedding.weight"]
    x = emb[tar] + O.position_table(T, D, emb.dtype)
    causal = torch.tril(torch.ones(T, T, dtype=torch.bool))
    self_mask = tar_mask[:, None, None, :] & causal[None, None]
    training = p > 0
    for i in range(L):
        sid = 64 + 8 * i
        x = O.attention(sd, f"decoder.attention_list.{i}", x, x, self_mask, 8, p, training, masks, sid)
        x = O.attention(sd, f"decoder.cross_attention_list.{i}", x, memory, mem_mask, 8, p, training, masks, sid + 1)
        x = _feed_forward(sd, f"decoder.feed_forward_list.{i}", x, p, training, masks, sid + 2, gates=gates)
    return x


# live rows of the six PACKED_INDEX commits with the map: none, one, 16 / 17 (the m16 edge), a label at t = T - 1,
# and the commit's own (-1)
LIVE_COUNTS = (0, 1, 16, 17, T, -1)


def _live_labels(pk, Rt):
    """edit pk.label to LIVE_COUNTS (a zero label inside the 17-row message) and set pk.Rt: "count" = the live rows,
    "r128" = rounded up to 128 (pad slots), "all" = B*T -> live [B, T] bool"""
    lab = pk.label.cpu().clone()
    for b, n in enumerate(LIVE_COUNTS):
        if n >= 0:
            lab[b, n:] = 0
            if n:
                lab[b, n - 1] = 5
    lab[3, 4] = 0
    pk.label.copy_(lab)
    nz = lab != 0
    tlen = torch.where(nz.any(1), T - nz.flip(1).int().argmax(1), torch.zeros(pk.B, dtype=torch.long))
    assert tlen.tolist()[:5] == [0, 1, 16, 17, T] and 0 < int(tlen[5]) < T and int(tlen[5]) not in (1, 16, 17)
    assert bool(pk.tar_mask.cpu()[tlen > 0, 0].all()), "a labelled commit's row 0 must be a valid key (DecoderFn)"
    n = int(tlen.sum())
    pk.Rt = {"count": n, "r128": -(-n // 128) * 128, "all": pk.B * T}[Rt]
    assert pk.Rt <= pk.B * T
    return torch.arange(T)[None, :] < tlen[:, None]


def _dec_cases():
    cases = [pytest.param(L, packed, p, None, id=f"{L}-{'packed' if packed else 'padded'}-p{p:g}")
             for L in (1, 6) for packed in (False, True) for p in (0.0, 0.1)]
    return cases + [pytest.param(L, True, p, live, id=f"{L}-packed-p{p:g}-live_{live}")
                    for L, live in ((1, "count"), (1, "r128"), (1, "all"), (6, "r128")) for p in (0.0, 0.1)]


@pytest.mark.parametrize("L,packed,p,live", _dec_cases())
def test_decoder_fn_matches_float64(model, L, packed, p, live):
    """live: the live-row map (cfg["label"], packed batches): the forward saves and the backward runs on the pk.Rt slots;
    the loss gradient is zero on the dead rows, whose output rows must be exactly zero"""
    from fira_icse_b200 import ops
    dm = model.decoder
    pk = None
    alive = None
    if packed:
        pk = _packed(PACKED_INDEX).to(DEV)
        if live is not None:
            alive = _live_labels(pk, live)
        idx, mem_valid = _commit_rows(pk)
        tar, tar_mask = pk.tar.cpu().long(), pk.tar_mask.cpu().bool()
        memory = _bf16_randn((1, pk.mem_rows, D), 3)
        B = pk.B
        args = (pk.tar, memory, pk.mem_mask, pk.tar_mask)
    else:
        sou, tar, _, _, _, _, _, sub = golden_batch(0, 6)
        mem_valid = torch.cat((sou != 0, sub != 0), 1)
        mem_valid[1] = False                        # a commit without a valid memory key
        tar = tar.clone()
        tar[2, 0] = 0                               # target row 0 of commit 2: no valid self-attention key
        tar_mask = tar != 0
        B = tar.shape[0]
        memory = _bf16_randn((B, mem_valid.shape[1], D), 3)
        args = (tar.to(torch.int32).to(DEV), memory, mem_valid.to(torch.uint8).to(DEV), tar_mask.to(torch.uint8).to(DEV))
    tensors = [dm.embedding.weight]
    for i in range(L):
        tensors += dm.attention_list[i].flat_params() + dm.cross_attention_list[i].flat_params() + \
            dm.feed_forward_list[i].flat_params()
    names, leaves, sd = _leaves(model, tensors, lambda k: ".fc" in k and k.endswith(".weight"))
    with torch.no_grad():                           # peaked attention (see Q_SCALE); a power of two keeps bf16 exact
        for k, t in zip(names, leaves):
            if k.endswith("fc_q.weight"):
                t.mul_(Q_SCALE)
                sd[k].mul_(Q_SCALE)
    cfg = {"training": p > 0, "seed": SEED, "stream_base": 0, "heads": 8, "bf16": True, "seed_ctr": None,
           "p_dec": p, "prefetch": None, "packed": pk}
    if alive is not None:
        cfg["label"] = pk.label
    m_dev = memory.to(DEV).requires_grad_(True)
    tar_dev, _, mm_dev, tm_dev = args
    out = ops.DecoderFn.apply(cfg, tar_dev, m_dev, mm_dev, tm_dev, dm.pos_encode.to(DEV), *leaves)
    g_out = _bf16_randn((B, T, D), 4)
    if alive is not None:
        g_out = g_out * alive[..., None]
    out.backward(g_out.to(DEV).to(out.dtype))
    torch.cuda.synchronize()

    m64 = memory.double().requires_grad_(True)
    mem_b = m64 if pk is None else m64[0][idx]
    masks = _drop_masks(SEED, lambda sid: p) if p > 0 else None
    gates = {}
    ref = _dec_ref(sd, tar, mem_b, mem_valid, tar_mask, L, p, masks, gates)
    ref.backward(g_out.double())
    eps, tag = EPS_DEC[L], f"decoder/L{L}/{'packed' if packed else 'padded'}/p{p}"
    if alive is not None:
        tag += f"/live_{live}(Rt={pk.Rt})"
        close(f"{tag} output", out.detach().cpu()[alive], ref[alive], eps, rows=True)
        assert bool((out.detach().cpu()[~alive] == 0).all()), "dead rows must be exactly zero"
    else:
        close(f"{tag} output", out, ref, eps, rows=True)
    close(f"{tag} d_memory", m_dev.grad, m64.grad, eps, rows=True)
    _check_grads(tag, names, leaves, sd, eps, rows=("decoder.embedding.weight",), allow=gate_allowance(gates, tag))


# ============================================================================= EncoderFn
def _enc_ref(sd, sou, mark, ast_change, adj, sub_token, L, p_comb, p_gcn, masks):
    """oracle.encoder with L layers -> memory = cat(code rows, sub-token rows)"""
    import fira_oracle as O
    emb = sd["encoder.embedding.weight"]
    B, n_code, n_sub, n_ast = sou.shape[0], sou.shape[1], sub_token.shape[1], ast_change.shape[1]
    seg = torch.cat((torch.arange(B * n_code).view(B, n_code), B * n_code + torch.arange(B * n_sub).view(B, n_sub),
                     B * (n_code + n_sub) + torch.arange(B * n_ast).view(B, n_ast)), dim=1)
    code = emb[sou] + O.position_table(n_code, D, emb.dtype)
    mark_em = sd["encoder.mark_embedding.weight"][mark]
    ast = sd["encoder.ast_change_embedding.weight"][ast_change]
    sub = emb[sub_token]
    training = p_comb > 0
    for i in range(L):
        sid = 8 * i
        code = O.combination(sd, f"encoder.combination_list2.{i}", code, mark_em, 8, p_comb, training, masks, sid)
        nodes = torch.cat((code, sub, ast), dim=1)
        nodes = O.gcn(sd, f"encoder.gcn_list.{i}", nodes, adj, p_gcn, training, masks, sid + 2, seg)
        code, sub, ast = nodes[:, :n_code], nodes[:, n_code:n_code + n_sub], nodes[:, n_code + n_sub:]
    return torch.cat((code, sub), 1)


ENC_EMB = ("encoder.embedding.weight", "encoder.ast_change_embedding.weight", "encoder.mark_embedding.weight")


@pytest.mark.parametrize("drop", [False, True], ids=["p0", "dropout"])
@pytest.mark.parametrize("fused", ["0", "1"], ids=["default_gcn", "fused_gcn"])
@pytest.mark.parametrize("packed", [False, True], ids=["padded", "packed"])
@pytest.mark.parametrize("L", [1, 6])
def test_encoder_fn_matches_float64(model, monkeypatch, L, packed, fused, drop):
    """padded: three golden commits, B = 3.  packed: the packed batch as Encoder.encode_memory_packed runs it (one
    ragged graph, B = 1, positions from pb.pos, the packed CSR), against the reference on the padded commits with its
    node rows mapped to the packed rows"""
    from fira_icse_b200 import PackedEdges, ops
    from fira_icse_b200.modules import _i32
    from test_gpu_train_dropout import model_masks, packed_row_map
    monkeypatch.setenv("FIRA_GCN_FUSED", fused)
    em = model.encoder
    index = PACKED_INDEX if packed else [0, 1, 2]
    parts = [golden_batch(i, i + 1) for i in index]
    sou, _, _, mark, ast, edge, _, sub = (torch.cat([q[k] for q in parts], 0) for k in range(8))
    B, n_code, n_sub = sou.shape[0], sou.shape[1], sub.shape[1]
    tensors = [em.embedding.weight, em.ast_change_embedding.weight, em.mark_embedding.weight]
    for i in range(L):
        tensors += em.combination_list2[i].flat_params() + em.gcn_list[i].flat_params()
    names, leaves, sd = _leaves(model, tensors, lambda k: k.endswith(("linear_layers.0.weight", "linear_layers.1.weight",
                                                                       "output_linear.weight")))
    p_comb, p_gcn = (0.1, 0.2) if drop else (0.0, 0.0)
    cfg = {"training": drop, "seed": SEED, "stream_base": 0, "heads": 8, "bf16": True, "seed_ctr": None,
           "p_comb": p_comb, "p_gcn": p_gcn}
    if packed:
        pb = _packed(index).to(DEV)
        cfg["pos"] = pb.pos
        edges = PackedEdges(pb.rowptr, pb.col, pb.val, 1, pb.rows, True)
        ids = (pb.code.view(1, -1), pb.mark.view(1, -1), pb.ast.view(1, -1), pb.sub.view(1, -1))
        row_map = packed_row_map(pb, B, (n_code, n_sub, ast.shape[1]))
        # memory position (b, m) of the reference -> its row of the packed memory (-1: padding the kernels drop)
        node = np.concatenate((np.arange(B)[:, None] * n_code + np.arange(n_code),
                               B * n_code + np.arange(B)[:, None] * n_sub + np.arange(n_sub)), 1)
        pmap = torch.from_numpy(row_map[node])
    else:
        edges = PackedEdges.from_dense(edge.to(DEV))
        ids = tuple(_i32(t.to(DEV)) for t in (sou, mark, ast, sub))
        row_map, pmap = None, torch.arange(B * (n_code + n_sub)).view(B, -1)
    out = ops.EncoderFn.apply(cfg, *ids, edges, em.pos_encode.to(DEV), *leaves)
    live = pmap >= 0
    g_rows = _bf16_randn((int(live.sum()), D), 5)
    g_out = torch.zeros(out.numel() // D, D)        # packed: no gradient reaches the rows of the segment padding
    g_out[pmap[live]] = g_rows
    out.backward(g_out.view(out.shape).to(DEV).to(out.dtype))
    torch.cuda.synchronize()

    masks = model_masks(SEED, SEED, row_map=row_map) if drop else None      # p_comb = 0.1, p_gcn = 0.2
    ref = _enc_ref(sd, sou, mark, ast, edge, sub, L, p_comb, p_gcn, masks)
    g_ref = torch.zeros(B, n_code + n_sub, D, dtype=torch.float64)
    g_ref[live] = g_rows.double()
    ref.backward(g_ref)
    for k in ENC_EMB:                               # padding_idx = 0 (gnn_transformer.py:36-39)
        sd[k].grad[0] = 0.0
    assert (leaves[2].grad[0] == 0).all(), "the mark-embedding padding row must be exactly zero"
    eps = EPS_ENC[L]
    tag = f"encoder/L{L}/{'packed' if packed else 'padded'}/gcn_fused{fused}/{'dropout' if drop else 'p0'}"
    close(f"{tag} output", out.reshape(-1, D)[pmap[live].to(DEV)], ref[live], eps, rows=True)
    _check_grads(tag, names, leaves, sd, eps, rows=ENC_EMB)


# ============================================================================= the whole step, as bench.py runs it
def test_graphed_packed_bf16_step_matches_oracle(monkeypatch):
    """bf16, packed batch, one GraphedTrainStep replay with optim.FlatAdam at lr = 0: the loss and every live
    parameter's gradient against the float64 oracle under the masks of the replay (seeds frozen at capture + the
    replay's counter)"""
    from fira_icse_b200 import FlatAdam, ops
    from fira_icse_b200.engine import GraphedTrainStep
    from test_gpu_train_dropout import SeedRecorder, model_masks, oracle, packed_row_map
    rec = SeedRecorder(ops.make_seed)
    monkeypatch.setattr(ops, "make_seed", rec)
    base = seeded_model()
    m = copy.deepcopy(base).to(DEV)
    m.train()
    m.set_precision("bf16")
    B = len(PACKED_INDEX)
    eng = GraphedTrainStep(m, B, lambda ps: FlatAdam(ps, lr=0.0, groups=m.flat_groups()), edge_capacity=32768)
    pb = _packed(PACKED_INDEX)
    eng.load(pb)
    eng.capture()
    se, sd = rec.seeds[-2:]                         # the forward recorded into the graph: encoder, then decoder
    ls, n = eng.step(pb)
    loss = (ls / n).item()
    ctr = int(eng.seed_ctr.item())
    assert eng.flat_optims, "the bench configuration trains with optim.FlatAdam"
    nm = _names(m)
    grads = {nm[id(p)]: g for o in eng.flat_optims for p, g in zip(o.params, o.gviews)}
    parts = [golden_batch(i, i + 1) for i in PACKED_INDEX]
    batch = [torch.cat([q[k] for q in parts], 0) for k in range(8)]
    row_map = packed_row_map(eng.cur.pb, B, (batch[0].shape[1], batch[7].shape[1], batch[4].shape[1]))
    gates = {}
    record_gates(monkeypatch, gates)
    ref_loss, ref_grads = oracle(base, batch, model_masks(se, sd, ctr=ctr, row_map=row_map))
    check_step("graphed/packed", loss, grads, ref_loss, ref_grads, gates)


# a second batch with PACKED_INDEX's shape key (packed_needs (1024, 512, 512, 256, 128, 128)) but 87 live target rows to
# its 49: one captured graph, other slot offsets and pad-slot counts
REPLAY_INDEX = [52, 95, 96, 1, 32, 18]


def test_graph_replays_across_batches_of_one_shape_key(monkeypatch):
    """bf16, packed, GraphedTrainStep with optim.FlatAdam at lr = 0: captured on batch A, then replayed on A, B, A.  The
    live-row map is computed inside the graph, so each replay must train on its own batch's slots: after every replay
    the loss and every gradient against the float64 oracle under that replay's masks"""
    from fira_icse_b200 import FlatAdam, ops
    from fira_icse_b200.engine import GraphedTrainStep
    from fira_icse_b200.packed import PackedTables, packed_needs
    from test_gpu_train_dropout import SeedRecorder, model_masks, oracle, packed_row_map
    from test_packed import GoldenSplit
    rec = SeedRecorder(ops.make_seed)
    monkeypatch.setattr(ops, "make_seed", rec)
    tables = PackedTables(GoldenSplit())
    pa, pb = _packed(PACKED_INDEX), _packed(REPLAY_INDEX)
    assert pa.shape_key == pb.shape_key
    assert packed_needs(tables, np.asarray(PACKED_INDEX), V) == packed_needs(tables, np.asarray(REPLAY_INDEX), V)
    assert tables.live_rows(np.asarray(PACKED_INDEX)) != tables.live_rows(np.asarray(REPLAY_INDEX))
    base = seeded_model()
    m = copy.deepcopy(base).to(DEV)
    m.train()
    m.set_precision("bf16")
    B = len(PACKED_INDEX)
    eng = GraphedTrainStep(m, B, lambda ps: FlatAdam(ps, lr=0.0, groups=m.flat_groups()), edge_capacity=32768)
    eng.load(pa)
    eng.capture()
    se, sd = rec.seeds[-2:]                         # the forward recorded into the graph: encoder, then decoder
    gates = {}
    record_gates(monkeypatch, gates)
    nm = _names(m)
    for name, index, pk in (("A", PACKED_INDEX, pa), ("B", REPLAY_INDEX, pb), ("A again", PACKED_INDEX, pa)):
        ls, n = eng.step(pk)
        loss = (ls / n).item()
        ctr = int(eng.seed_ctr.item())
        assert len(eng.captured) == 1 and eng.cur.graph is not None, "one graph for both batches"
        grads = {nm[id(p)]: g.detach().clone() for o in eng.flat_optims for p, g in zip(o.params, o.gviews)}
        parts = [golden_batch(i, i + 1) for i in index]
        batch = [torch.cat([q[k] for q in parts], 0) for k in range(8)]
        row_map = packed_row_map(eng.cur.pb, B, (batch[0].shape[1], batch[7].shape[1], batch[4].shape[1]))
        gates.clear()
        ref_loss, ref_grads = oracle(base, batch, model_masks(se, sd, ctr=ctr, row_map=row_map))
        check_step(f"graphed/replay {name}", loss, grads, ref_loss, ref_grads, gates)


def check_step(tag, loss, grads, ref_loss, ref_grads, gates, eps=EPS_STEP):
    """loss (relative LOSS_REL) and every gradient of one training step against the float64 oracle; gates: the FFN
    gates the oracle recorded (record_gates) for the fc1 allowance"""
    rel = abs(loss - ref_loss) / abs(ref_loss)
    print(f"[bf16 bound] {tag} loss: {rel / LOSS_REL:.3f} of {LOSS_REL} relative ({rel:.2e})")
    assert rel <= LOSS_REL, (loss, ref_loss)
    assert sorted(grads) == sorted(k for k, g in ref_grads.items() if g is not None)
    allow = gate_allowance(gates, tag)
    assert sorted(allow) == sorted(k for k in grads if k.startswith("decoder.feed_forward_list") and ".fc1." in k)
    for k, g in grads.items():
        ref = ref_grads[k]
        if vanishing(k):
            small(f"{tag} {k}", g, ref_grads[k[:-len("bias")] + "weight"].abs().max().item(), eps)
            continue
        close(f"{tag} {k}", g, ref, eps, rows=k.endswith("embedding.weight"), allow=allow.get(k))
