"""The KV-cached decoding position (incremental.IncrementalDecoder on CudaBackend, decode_loop.PositionLoop.head)
against float64, row by row (tests/bf16_bound.py).  Every decoder of the package runs its positions through this path,
on its own launches: gemm_tc / gemm_raw on rows padded to MIN_ROWS = 128, fira_attn_fwd with Lq = 1 over the strided
self-attention cache (ldk = ldv = 2D, key mask tok_mask), fira_attn_fwd with Lq = N slots per commit over kv_mem
(ldk = 6 * 2D), the cross K/V product of B*S rows, LayerNorm, the cache reorder and captured graphs whose static weight
copies are refreshed in place.

The reference is the oracle's decoder blocks (oracle/fira_oracle.py) and output head on the same inputs:
  * the memory is bf16-exact; in bf16 mode the float64 weights are the bf16-rounded GEMM operands where the kernels
    round them (the concatenated self-attention QKV, fc_o, the cross-attention fc_q / fc_o and K/V, the FFN, out_fc,
    LinearTarget, LinearSource); biases, LayerNorm parameters, the embedding table, LinearProb (an fp32 product of the
    bf16 row) and LinearRes stay float64;
  * every fc_q weight is scaled by Q_SCALE (a power of two, bf16-exact) so the attention is peaked and a misrouted key
    moves the row, and the LayerNorm weights and biases are moved away from (1, 0);
  * the decoder is causal, so the float64 decoder runs once on the final token histories of a case, and the row the
    kernels gave at position t is compared with the row of its descendant, found through the ancestor chain of the
    reorders.  At the positions where beams collapse the reference also runs on the histories of that moment, so the
    rows of lines that die there are checked as well.

Each eps is the smallest power of two at least twice the worst error measured on an H100 SXM (80 GB, 700 W power limit),
within the ceilings 2^-13 (fp32, the rtol = 1e-4 of the fp32 token-logprob tests), 2^-5 (bf16, one layer), 2^-3 (bf16,
six layers: the training-step decoder's EPS_DEC) and 2^-7 (the head: EPS_HEAD of tests/test_gpu_bf16_step.py).  The
printed "[bf16 bound]" lines give each check's worst error as a fraction of its bound; the worst measured:
  * decoder rows, fp32: one layer 0.19 of 2^-20, six layers 0.40 of 2^-19 (after an in-place weight update);
  * decoder rows, bf16: one layer 0.38 of 2^-7, six layers 0.45 of 2^-5 (the position loop after a weight update);
  * head triple and ensemble mixture: fp32 0.26 of 2^-19 (logits), bf16 0.46 of 2^-8 (copy scores).
The head triple (logits, copy scores at unmasked positions, gate logits) is compared with the float64 head of the rows
the loop's own decoder wrote, which are checked against the float64 decoder first: so its bound counts the head's own
roundings only -- in bf16 the logits rounded once and the LinearTarget / LinearSource projections rounded once before
the fp32 tanh -- and a misrouted commit or member in the head cannot hide inside the six layers' error.  Masked copy
positions must hold exactly 0, what fira_copy_scores_fwd writes where its src_mask is 0.

The negative controls perturb only the float64 reference -- two beams' parents swapped at one step, one commit's memory
mask shifted by one key, the position-table row of t - 1 used at t -- and assert that the same check fails."""
import copy

import numpy as np
import pytest
import torch
import torch.nn as nn

import fira_oracle as O
from bf16_bound import close
from fira_testlib import reference_args, seeded_model
from sample_rule import mixture

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
D = 256
T = 30
HEADS = 8
START, PAD = 1, 0
Q_SCALE = 8.0
EPS = {("fp32", 1): 2 ** -20, ("fp32", 6): 2 ** -19, ("bf16", 1): 2 ** -7, ("bf16", 6): 2 ** -5}
EPS_HEAD = {"fp32": 2 ** -19, "bf16": 2 ** -8}
# the GEMM operands the bf16 kernels round (Prec.w / CudaBackend.weight)
ROUNDED = (".fc_q.weight", ".fc_k.weight", ".fc_v.weight", ".fc_o.weight", ".fc1.weight", ".fc2.weight",
           "out_fc.weight", "copy_net.LinearTarget.weight", "copy_net.LinearSource.weight")


@pytest.fixture(scope="module", autouse=True)
def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


# ============================================================================= fixture and reference
def _sharpen(module, seed):
    """every fc_q weight x Q_SCALE, LayerNorm weights and biases moved away from (1, 0)"""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in module.named_parameters():
            if name.endswith("fc_q.weight"):
                p.mul_(Q_SCALE)
            elif ".layernorm." in name:
                p.add_(0.1 * torch.randn(p.shape, generator=g).to(p.device))
    return module


def _decoder(V, L, seed, precision):
    """a fira_icse_b200.modules.Decoder on the device with L layers"""
    from fira_icse_b200.modules import Decoder
    torch.manual_seed(seed)
    dec = Decoder(reference_args(vocab_size=V), PAD)
    if L < len(dec.attention_list):
        for k in ("attention_list", "cross_attention_list", "feed_forward_list"):
            setattr(dec, k, nn.ModuleList(getattr(dec, k)[:L]))
    dec = _sharpen(dec, seed).to(DEV).eval()
    dec.bf16 = precision == "bf16"
    return dec


def _model(V, seed, precision):
    """a TransModel on the device: seeded_model() at V = 24650, else seeded with `seed`; out_fc sharpened x4"""
    import fira_icse_b200 as F
    if V == 24650:
        m = copy.deepcopy(seeded_model())
    else:
        torch.manual_seed(seed)
        m = F.TransModel(reference_args(vocab_size=V))
    with torch.no_grad():
        m.out_fc.weight.mul_(4.0)
        m.out_fc.bias.mul_(4.0)
    _sharpen(m.decoder, seed)
    return m.to(DEV).eval().set_precision(precision)


def _ref_sd(module, bf16, prefix=""):
    """float64 state dict, the bf16-rounded GEMM operands in bf16 mode"""
    sd = {}
    for k, v in module.state_dict().items():
        v = v.detach().cpu()
        if bf16 and (prefix + k).endswith(ROUNDED):
            v = v.to(torch.bfloat16)
        sd[prefix + k] = v.double()
    return sd


def _memory(B, S, seed, empty=None):
    """bf16-exact memory [B, S, D] and a mask like cat(sou != pad, sub_token != 0): a code part and a sub-token part,
    each with a padded tail; commit `empty` has no valid key"""
    g = torch.Generator().manual_seed(seed)
    mem = torch.randn((B, S, D), generator=g).to(torch.bfloat16).double()
    a = max(1, S * 21 // 37)
    n_code = torch.randint(1, a + 1, (B,), generator=g)
    n_sub = torch.randint(0, S - a + 1, (B,), generator=g)
    mask = torch.cat((torch.arange(a)[None] < n_code[:, None], torch.arange(S - a)[None] < n_sub[:, None]), 1)
    if empty is not None:
        mask[empty] = False
    return mem, mask


def _dec_ref(sd, seq, memory, mem_mask, L, N, pos=None):
    """the oracle's decoder with L layers on token histories seq [B*N, Tn] (rows (commit, slot)) -> [B*N, Tn, D].  The
    N slots of a commit share its memory: cross-attention is row-wise, so their rows are one [N*Tn] query block."""
    R, Tn = seq.shape
    B = R // N
    emb = sd["decoder.embedding.weight"]
    pos = O.position_table(Tn, D, torch.float64) if pos is None else pos[:Tn]
    x = emb[seq] + pos
    causal = torch.tril(torch.ones(Tn, Tn, dtype=torch.bool))
    self_mask = (seq != PAD)[:, None, None, :] & causal[None, None]
    for i in range(L):
        x = O.attention(sd, f"decoder.attention_list.{i}", x, x, self_mask, HEADS, 0.0, False)
        x = O.attention(sd, f"decoder.cross_attention_list.{i}", x.reshape(B, N * Tn, D), memory, mem_mask, HEADS,
                        0.0, False).reshape(R, Tn, D)
        x = O.feed_forward(sd, f"decoder.feed_forward_list.{i}", x, 0.0, False)
    return x


def _head_ref(sd, memory, mem_mask, x, N):
    """the oracle's head on decoder rows x [B*N, Tn, D] -> logits [R, Tn, V], copy scores [R, Tn, S] (0 at masked
    positions), gate logits [R, Tn, 2], mixture P [R, Tn, V + S]"""
    R, Tn, _ = x.shape
    B, S = memory.shape[0], memory.shape[1]
    logits = O._lin(sd, "out_fc", x)
    xb = x.reshape(B, N * Tn, D)
    sc, _ = O.copy_net(sd, memory, xb)
    sc = sc.masked_fill(~mem_mask[:, None, :], 0.0).reshape(R, Tn, S)
    gl = O._lin(sd, "copy_net.LinearProb", x)
    _, P = O.output_distribution(sd, memory, mem_mask, xb)
    return logits, sc, gl, P.reshape(R, Tn, -1)


# ============================================================================= token histories and reorders
class Histories:
    """The host record of a decode: toks[t] = the token of every row at position t, srcs[t] = the reorder after
    position t (new row r continues old row srcs[t][r]).  Most reorders are permutations inside each commit; at
    COLLAPSE (N > 2) two slots of every commit continue one parent.  Slot N - 1 of commit 0 (N > 1) keeps its own line
    and appends pad at every position: its only valid self-attention key is position 0."""

    COLLAPSE = (9, 19)

    def __init__(self, B, N, V, seed):
        self.B, self.N, self.V = B, N, V
        self.g = torch.Generator().manual_seed(seed)
        self.toks, self.srcs = [torch.full((B * N,), START, dtype=torch.long)], []

    def reorder(self, t):
        B, N, g = self.B, self.N, self.g
        src = torch.stack([torch.randperm(N, generator=g) for _ in range(B)])
        if N > 1:
            src[0] = torch.cat((src[0][src[0] != N - 1], torch.tensor([N - 1])))
        if t in self.COLLAPSE and N > 2:
            src[:, 1] = src[:, 0]
        src = (torch.arange(B)[:, None] * N + src).reshape(-1)
        tok = torch.randint(3, self.V, (B * N,), generator=g)
        tok[torch.rand(B * N, generator=g) < 0.15] = PAD          # finished beams
        if N > 1:
            tok[N - 1] = PAD
        self.srcs.append(src)
        self.toks.append(tok)
        return src, tok

    def at(self, upto, srcs=None):
        """-> seq [R, upto + 1] = the histories of the rows at position `upto` (before its reorder), anc [R, upto + 1]
        = the row at position t of each one's ancestor.  srcs: other reorders (the negative controls)"""
        srcs = self.srcs if srcs is None else srcs
        R = self.B * self.N
        seq, anc = self.toks[0][:, None], torch.arange(R)[:, None]
        for t in range(1, upto + 1):
            s = srcs[t - 1]
            seq = torch.cat((seq[s], self.toks[t][:, None]), 1)
            anc = torch.cat((anc[s], torch.arange(R)[:, None]), 1)
        return seq, anc


def _mapped(got, anc):
    """got [Tn, R, ...] recorded per position -> the recorded rows along each row's ancestor chain [R, Tn, ...]"""
    Tn = anc.shape[1]
    return got[torch.arange(Tn)[None, :], anc]


def _decode_rows(inc, hist, memory, mem_mask):
    """start() a batch and step all T positions with hist's tokens and reorders -> the rows [T, R, D] (float64)"""
    inc.start(memory.float().to(DEV), mem_mask.to(DEV))
    got = []
    for t in range(T):
        if t:
            src, _ = hist.reorder(t - 1)
            inc.reorder(src.to(DEV))
        got.append(inc.step(hist.toks[t].to(DEV), t, PAD).to("cpu", torch.float64, copy=True))
    return torch.stack(got)


def _check_rows(tag, got, hist, sd, memory, mem_mask, L, eps, positions=None):
    """the recorded rows against the float64 decoder at `positions` (default: each collapse and the last one)"""
    worst = 0.0
    for upto in positions or [p for p in hist.COLLAPSE if hist.N > 2] + [T - 1]:
        seq, anc = hist.at(upto)
        ref = _dec_ref(sd, seq, memory, mem_mask, L, hist.N)
        worst = max(worst, close(f"{tag} rows 0..{upto}", _mapped(got, anc), ref, eps, rows=True))
    return worst


# ============================================================================= 1. decoder rows
ROW_CASES = [(1, 1, 370, None), (2, 3, 11, None), (4, 32, 370, None), (64, 5, 370, None), (3, 7, 45, 1)]


def _row_cases():
    out = []
    for B, N, S, empty in ROW_CASES:
        for prec in ("fp32", "bf16"):
            out.append(pytest.param(B, N, S, empty, prec, 6, id=f"{B}x{N}-S{S}-{prec}-L6"))
    for B, N, S, empty in (ROW_CASES[1], ROW_CASES[4]):
        for prec in ("fp32", "bf16"):
            out.append(pytest.param(B, N, S, empty, prec, 1, id=f"{B}x{N}-S{S}-{prec}-L1"))
    return out


@pytest.mark.parametrize("B,N,S,empty,prec,L", _row_cases())
def test_incremental_rows_match_float64(B, N, S, empty, prec, L):
    """B commits x N slots, memory length S: R = 1 (127 pad rows, cross-attention Lq = 1), a cross K/V product of 22
    rows, N = 32 = LQ_MAX with R = 128, R = 320, and a commit whose memory keys are all masked"""
    from fira_icse_b200.incremental import IncrementalDecoder
    V = 61
    dec = _decoder(V, L, 11 + L, prec)
    sd = _ref_sd(dec, prec == "bf16", "decoder.")
    memory, mask = _memory(B, S, B * 100 + S, empty)
    inc = IncrementalDecoder(dec, B, N, T, S)
    assert inc.Rp == max(128, B * N)
    hist = Histories(B, N, V, B * N + S)
    got = _decode_rows(inc, hist, memory, mask)
    _check_rows(f"incremental/{B}x{N}/S{S}/{prec}/L{L}", got, hist, sd, memory, mask, L, EPS[(prec, L)])


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
def test_negative_controls_fail_the_row_bound(prec):
    """the 3x7 case's rows against perturbed float64 references: each must fail the bound that the true reference
    passes (a) two beams' parents swapped at one step, (b) one commit's memory mask shifted by one key, (c) the position
    table's row t - 1 used at t"""
    from fira_icse_b200.incremental import IncrementalDecoder
    B, N, S, L, V = 3, 7, 45, 6, 61
    dec = _decoder(V, L, 17, prec)
    sd = _ref_sd(dec, prec == "bf16", "decoder.")
    memory, mask = _memory(B, S, 5, empty=1)
    hist = Histories(B, N, V, 23)
    got = _decode_rows(IncrementalDecoder(dec, B, N, T, S), hist, memory, mask)
    eps, tag = EPS[(prec, L)], f"control/{prec}"
    seq, anc = hist.at(T - 1)
    close(f"{tag} true reference", _mapped(got, anc), _dec_ref(sd, seq, memory, mask, L, N), eps, rows=True)
    # (a) commit 2's slots 0 and 1 swap parents after position 4
    srcs = list(hist.srcs)
    s = srcs[4].clone()
    s[2 * N], s[2 * N + 1] = srcs[4][2 * N + 1], srcs[4][2 * N]
    srcs[4] = s
    seq_a, anc_a = hist.at(T - 1, srcs)
    assert not torch.equal(seq_a, seq)
    # (b) commit 0's mask shifted by one key
    mask_b = mask.clone()
    mask_b[0] = torch.roll(mask[0], 1)
    # (c) position t - 1's table row at t
    pos = O.position_table(T, D, torch.float64)
    pos_c = torch.cat((pos[:1], pos[:-1]))
    for what, ref, a in (("(a) parents swapped", _dec_ref(sd, seq_a, memory, mask, L, N), anc_a),
                         ("(b) mask shifted", _dec_ref(sd, seq, memory, mask_b, L, N), anc),
                         ("(c) position t - 1", _dec_ref(sd, seq, memory, mask, L, N, pos_c), anc)):
        with pytest.raises(AssertionError):
            close(f"{tag} {what}", _mapped(got, a), ref, eps, rows=True)


# ============================================================================= 2. static buffers, graphs, weights
@pytest.mark.parametrize("prec", ["fp32", "bf16"])
def test_graphs_replay_new_batches_and_follow_weight_updates(prec):
    """graphs=True: batch 1 captures a graph per position; batch 2 (other memory, mask and tokens) replays them from
    clean caches; parameters updated in place (p.mul_) and written raw (p.data, no _version bump, then
    weights_epoch += 1 as engine.py / optim.py / scst.py do) give rows of the new weights from the same graphs"""
    from fira_icse_b200.incremental import IncrementalDecoder, weights_key
    B, N, S, L, V = 4, 8, 45, 6, 61
    bf16 = prec == "bf16"
    dec = _decoder(V, L, 29, prec)
    inc = IncrementalDecoder(dec, B, N, T, S, graphs=True)
    eps, tag = EPS[(prec, L)], f"graphs/{prec}"
    memory, mask = _memory(B, S, 1, empty=2)
    hist = Histories(B, N, V, 1)
    got = _decode_rows(inc, hist, memory, mask)
    _check_rows(f"{tag} batch 1 (captured)", got, hist, _ref_sd(dec, bf16, "decoder."), memory, mask, L, eps, [T - 1])
    graphs = dict(inc.graphs)
    assert sorted(graphs) == list(range(T))

    def replayed():
        assert inc.graphs == graphs, "no recapture"

    memory, mask = _memory(B, S, 2)
    inc.start(memory.float().to(DEV), mask.to(DEV))
    assert int(inc.tok_mask.sum()) == 0 and float(inc.kv_self.float().abs().sum()) == 0.0, "start() clears the caches"
    hist = Histories(B, N, V, 2)
    got = _decode_rows(inc, hist, memory, mask)
    replayed()
    _check_rows(f"{tag} batch 2 (replayed)", got, hist, _ref_sd(dec, bf16, "decoder."), memory, mask, L, eps)

    with torch.no_grad():                               # an optimizer step in place: _version moves
        for i, p in enumerate(dec.parameters()):
            p.mul_(1.0 + 0.03 * (1 + i % 5))
    hist = Histories(B, N, V, 3)
    got = _decode_rows(inc, hist, memory, mask)
    replayed()
    _check_rows(f"{tag} in-place update", got, hist, _ref_sd(dec, bf16, "decoder."), memory, mask, L, eps, [T - 1])

    key = weights_key(dec)
    for i, p in enumerate(dec.parameters()):            # a raw kernel write: neither _version nor the address moves
        p.data.mul_(1.0 - 0.02 * (1 + i % 3))
    assert weights_key(dec) == key
    dec.weights_epoch = getattr(dec, "weights_epoch", 0) + 1
    hist = Histories(B, N, V, 4)
    got = _decode_rows(inc, hist, memory, mask)
    replayed()
    _check_rows(f"{tag} raw write + weights_epoch", got, hist, _ref_sd(dec, bf16, "decoder."), memory, mask, L, eps,
                [T - 1])


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
def test_shared_token_buffer_and_mask(prec):
    """a second decoder with its own weights and memory reads the first one's token buffer and pad mask (share=); the
    owner reorders the mask, the member its cache only (tok_mask=False): each against its own float64 reference"""
    from fira_icse_b200.incremental import IncrementalDecoder
    B, N, S, L, V = 3, 7, 45, 6, 61
    bf16 = prec == "bf16"
    decs = [_decoder(V, L, 41, prec), _decoder(V, L, 43, prec)]
    owner = IncrementalDecoder(decs[0], B, N, T, S, graphs=True)
    member = IncrementalDecoder(decs[1], B, N, T, S, graphs=True, share=owner)
    assert member.tok is owner.tok and member.tok_mask is owner.tok_mask
    mems = [_memory(B, S, 7, empty=0), _memory(B, S, 8, empty=0)]
    mems[1] = (mems[1][0], mems[0][1])                  # one mask: the members decode one batch
    mask = mems[0][1]
    for inc, (mem, _) in zip((owner, member), mems):
        inc.start(mem.float().to(DEV), mask.to(DEV))
    hist = Histories(B, N, V, 9)
    got = ([], [])
    for t in range(T):
        if t:
            src, _ = hist.reorder(t - 1)
            owner.reorder(src.to(DEV))
            member.reorder(src.to(DEV), tok_mask=False)
        got[0].append(owner.step(hist.toks[t].to(DEV), t, PAD).to("cpu", torch.float64, copy=True))
        got[1].append(member.advance(t).to("cpu", torch.float64, copy=True))
    for i, (dec, (mem, _)) in enumerate(zip(decs, mems)):
        _check_rows(f"shared/{prec} decoder {i}", torch.stack(got[i]), hist, _ref_sd(dec, bf16, "decoder."), mem, mask,
                    L, EPS[(prec, L)], [T - 1])


def test_more_than_32_slots_is_refused():
    """N = 33 slots is a cross-attention with Lq = 33 > LQ_MAX: the library refuses the launch"""
    from fira_icse_b200._lib import FiraLibraryError
    from fira_icse_b200.incremental import IncrementalDecoder
    B, N, S = 1, 33, 11
    dec = _decoder(61, 1, 3, "fp32")
    memory, mask = _memory(B, S, 3)
    inc = IncrementalDecoder(dec, B, N, T, S).start(memory.float().to(DEV), mask.to(DEV))
    with pytest.raises(FiraLibraryError, match="Lq <= 32"):
        inc.step(torch.full((B * N,), START, dtype=torch.long, device=DEV), 0, PAD)
    torch.cuda.synchronize()


# ============================================================================= 3. the position loop's head inputs
def _loop_batch(loop, models, sds, graphs, B, N, S, V, seed, prec, tag):
    """start() one batch, write the teacher tokens, run head(t) through replay_or_capture and reorder; then every
    member's decoder rows against the float64 decoder, its triple against the float64 head of those rows, and for an
    ensemble the combined triple's mixture against the weighted mixture of the members' float64 mixtures"""
    from fira_icse_b200.incremental import replay_or_capture
    memory, mask = [], None
    for i in range(len(models)):
        mem, msk = _memory(B, S, seed + 17 * i, empty=B - 1 if B > 1 else None)
        memory.append(mem)
        mask = msk if mask is None else mask
    copy_src = torch.randint(3, V, (B, S))
    loop.start([m.float().to(DEV) for m in memory], mask.to(DEV), copy_src.to(DEV), START, PAD)
    hist = Histories(B, N, V, seed)
    inc = loop.inc
    R = B * N
    host = lambda x: x.to("cpu", torch.float64, copy=True)
    got = [([], [], [], []) for _ in loop.heads]
    comb = ([], [], [])
    for t in range(T):
        if t:
            src, _ = hist.reorder(t - 1)
            loop.reorder(src.to(DEV))
        inc.tok[:R].copy_(hist.toks[t].to(DEV))
        inc.tok_mask[:, t].copy_((hist.toks[t] != PAD).to(DEV))
        replay_or_capture(graphs, t, lambda: loop.head(t))
        for h, g in zip(loop.heads, got):
            for a, x in zip(g, (h.inc.out[:R], h.logits[:, :V], h.sc.reshape(R, S), h.gl)):
                a.append(host(x))
        if loop.ensemble:
            for a, x in zip(comb, (loop.logits[:, :V], loop.sc.reshape(R, S), loop.gl)):
                a.append(host(x))
    seq, anc = hist.at(T - 1)
    msk = mask.repeat_interleave(N, 0)[:, None, :].expand(R, T, S)
    Ps = []
    for i, (m, sd, mem, g) in enumerate(zip(models, sds, memory, got)):
        L = len(m.decoder.attention_list)
        x_g, lg_g, sc_g, gl_g = (_mapped(torch.stack(a), anc) for a in g)
        close(f"{tag} member {i} decoder rows", x_g, _dec_ref(sd, seq, mem, mask, L, N), EPS[(prec, L)], rows=True)
        lg, sc, gl, P = _head_ref(sd, mem, mask, x_g, N)
        Ps.append(P)
        assert bool((sc_g[~msk] == 0).all()), "masked copy positions: the kernel writes 0"
        close(f"{tag} member {i} logits", lg_g, lg, EPS_HEAD[prec], rows=True)
        close(f"{tag} member {i} copy scores", sc_g, sc, EPS_HEAD[prec], rows=True)
        close(f"{tag} member {i} gate logits", gl_g, gl, EPS_HEAD[prec], rows=True)
    if loop.ensemble:
        w = torch.tensor(loop.log_weights, dtype=torch.float64).exp()
        ref = sum(wi * P for wi, P in zip(w, Ps))
        lg_c, sc_c, gl_c = (_mapped(torch.stack(a), anc).numpy() for a in comb)
        mk = msk.numpy()
        got_P = torch.from_numpy(np.array([[mixture(lg_c[r, t], sc_c[r, t], gl_c[r, t], mk[r, t]) for t in range(T)]
                                           for r in range(R)]))
        keep = ref >= 1e-6
        close(f"{tag} ensemble log P (P >= 1e-6)", torch.where(keep, got_P.clamp(min=1e-300).log(), 0.0),
              torch.where(keep, ref.log(), 0.0), EPS_HEAD[prec], rows=True)


LOOP_CASES = [pytest.param("single", 24650, 2, 3, 370, id="single-V24650"),
              pytest.param("ensemble", 61, 3, 4, 45, id="ensemble2-V61")]


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("kind,V,B,N,S", LOOP_CASES)
def test_position_loop_head_matches_float64(kind, V, B, N, S, prec):
    """decode_loop.PositionLoop.head(t), captured, for one model at the real vocabulary (the logits pitch is padded) and
    for a two-member Ensemble (the _members pointer arrays and the shared mask).  Between two batches the weights are
    updated in place: loop_for returns the same loop with its weights refreshed, and the replayed graphs must give the
    head of the new weights"""
    from fira_icse_b200.decode_loop import PositionLoop, drop_loops, loop_for
    from fira_icse_b200.ensemble import Ensemble
    bf16 = prec == "bf16"
    models = [_model(V, 51, prec)] + ([_model(V, 53, prec)] if kind == "ensemble" else [])
    model = models[0] if kind == "single" else Ensemble(models, [1.0, 3.0])
    tag = f"loop/{kind}/{prec}"
    try:
        loop = loop_for(PositionLoop, model, B, N, T, S)
        graphs = {}
        _loop_batch(loop, models, [_ref_sd(m, bf16) for m in models], graphs, B, N, S, V, 61, prec, f"{tag} batch 1")
        assert sorted(graphs) == list(range(T))
        captured = dict(graphs)
        with torch.no_grad():
            for m in models:
                for i, p in enumerate(m.parameters()):
                    p.mul_(1.0 + 0.03 * (1 + i % 5))
        assert loop_for(PositionLoop, model, B, N, T, S) is loop
        _loop_batch(loop, models, [_ref_sd(m, bf16) for m in models], graphs, B, N, S, V, 67, prec,
                    f"{tag} batch 2 (new weights)")
        assert graphs == captured, "the head replays the graphs of batch 1"
    finally:
        drop_loops(models[0])
