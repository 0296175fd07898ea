"""fira_decoder_fwd (csrc/decoder_fwd.cu): the whole bf16 decoder forward in one launch, called through the C ABI on
seeded inputs with six layers.  Every output is checked against a float64 restatement of its own stage computed from the
kernel's saved inputs of that stage (the product from the saved layer input, attention from the saved q|k|v, LayerNorm
from the saved z and residual, ...), so the bound is one bf16 rounding of each result, as in tests/test_gpu_ops_bf16.py;
attention adds the bf16 rounding of P that its product consumes.  With dropout on, fira_ln_residual_fwd run on the
kernel's own z and residuals must reproduce every LayerNorm output: a wrong mask would show as O(1) errors.

Layouts: padded batches (T = 30 and 32; a commit without a valid memory key, a target row without a valid key) and
packed batches of golden commits and of a hand-made ragged layout (an empty sub-token range, a commit without a valid
key).  Outputs start as NaN, so an element the kernel does not write fails the comparison.

fira_decoder_fwd_rows (the live-row slot layout of the training step) runs on the same batches with maps from
fira_target_rows: every slot must be bit-equal to its row of the map-less run above, pad slots zero, the output zero
past each commit's last label and NaN for a live row without a slot, and nothing written past any buffer."""
import ctypes

import pytest
import torch

from test_gpu_ops_bf16 import BF, DEV, EPS, close16, st
from test_gpu_packed_kernels import hand_layout, real_layout

pytestmark = pytest.mark.gpu

D, H, DH, F, L = 256, 8, 32, 1024, 6
VOCAB = 500
NAMES = ("wqkv", "bqkv", "swo", "sbo", "slw", "slb", "cwq", "cbq", "cwo", "cbo", "clw", "clb",
         "w1", "b1", "w2", "b2", "flw", "flb")


@pytest.fixture(scope="module", autouse=True)
def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _g(seed):
    return torch.Generator().manual_seed(seed)


def layer_weights(seed):
    """the 18 tensors of fira_decoder_fwd's per-layer table: bf16 [out, in] weights, fp32 biases and LayerNorm"""
    g = _g(seed)
    shapes = {"wqkv": (3 * D, D), "swo": (D, D), "cwq": (D, D), "cwo": (D, D), "w1": (F, D), "w2": (D, F)}
    w = {}
    for n in NAMES:
        if n in shapes:
            w[n] = (torch.randn(*shapes[n], generator=g) / shapes[n][1] ** 0.5).to(BF).to(DEV)
        elif n.endswith("lw"):
            w[n] = (1.0 + 0.2 * torch.randn(D, generator=g)).to(DEV)
        else:
            w[n] = (0.1 * torch.randn({"bqkv": 3 * D, "b1": F}.get(n, D), generator=g)).to(DEV)
    return w


class Batch:
    """inputs of one call: target ids / mask [B, T], the hoisted K/V rows, and the keys of every commit"""

    def __init__(self, B, T, seed, layout=None, S=80):
        g = _g(seed)
        self.B, self.T = B, T
        self.tar = torch.randint(0, VOCAB, (B, T), generator=g, dtype=torch.int32).to(DEV)
        lens = torch.randint(1, T + 1, (B,), generator=g)
        lens[0] = T
        tm = (torch.arange(T)[None, :] < lens[:, None]).to(torch.uint8)
        tm[1, 0] = 0                                        # target row 0 of commit 1 has no valid key
        self.tar_mask = tm.to(DEV)
        self.emb = torch.randn(VOCAB, D, generator=g).to(DEV)
        self.pe = torch.randn(T + 3, D, generator=g).to(DEV)
        if layout is None:                                  # padded: keys b*S + s, mem_mask [B, S]
            mlen = torch.randint(1, S + 1, (B,), generator=g)
            mm = (torch.arange(S)[None, :] < mlen[:, None]) & (torch.rand(B, S, generator=g) > 0.2)
            mm[2] = False                                   # commit 2 has no valid key: uniform over all S
            self.mem_mask, self.S, self.ranges = mm.to(torch.uint8).to(DEV), S, None
            self.key_rows = [torch.arange(b * S, (b + 1) * S) for b in range(B)]
            R = B * S
        else:
            assert layout.B == B
            rg, _, mm = layout.dev()
            self.mem_mask, self.S, self.ranges = mm, layout.S, rg
            self.key_rows = [layout.rows(b) for b in range(B)]
            R = layout.R
        self.kv = (torch.randn(R, L * 2 * D, generator=g)).to(BF).to(DEV)
        self.w = [layer_weights(100 * seed + i) for i in range(L)]
        self.table = (ctypes.c_void_p * (18 * L))(*[w[n].data_ptr() for w in self.w for n in NAMES])

    def keys(self, b):
        """(global K/V rows, mask) of commit b's key list"""
        rows = self.key_rows[b].to(DEV)
        return rows, self.mem_mask[b, :len(rows)].bool()


def run(bt, p=0.0, seed=0, sid=64):
    from fira_icse_b200 import _lib
    B, T = bt.B, bt.T
    Mt = B * T
    nan = float("nan")

    def e(*shape, dtype=BF):
        return torch.full(shape, nan, dtype=dtype, device=DEV)
    o = {"X": e(L + 1, Mt, D), "qkv": e(L, Mt, 3 * D), "hh": e(L, Mt, F)}
    for n in ("ctx1", "z1", "x1", "q", "ctx2", "z2", "x2", "z3"):
        o[n] = e(L, Mt, D)
    for n in ("st1", "st2"):
        o[n] = e(L, B, H, T, 2, dtype=torch.float32)
    for n in ("ls1", "ls2", "ls3"):
        o[n] = e(L, 2, Mt, dtype=torch.float32)
    ptr = {k: v.data_ptr() for k, v in o.items()}
    _lib.call("fira_decoder_fwd", bt.tar.data_ptr(), bt.emb.data_ptr(), bt.pe.data_ptr(), bt.tar_mask.data_ptr(),
              bt.kv.data_ptr(), bt.kv.shape[1], bt.mem_mask.data_ptr(),
              bt.ranges.data_ptr() if bt.ranges is not None else None, bt.S, ctypes.addressof(bt.table), L,
              ptr["X"], ptr["qkv"], ptr["ctx1"], ptr["st1"], ptr["z1"], ptr["ls1"], ptr["x1"], ptr["q"], ptr["ctx2"],
              ptr["st2"], ptr["z2"], ptr["ls2"], ptr["x2"], ptr["hh"], ptr["z3"], ptr["ls3"], B, T, float(p), seed,
              None, sid, st())
    torch.cuda.synchronize()
    return o


def lin(x, w, b, relu=False):
    y = x.double() @ w.double().t() + b.double()
    return y.clamp_min(0.0) if relu else y


def ln(z, resid, gamma, beta):
    y = z.double() + resid.double()
    mean = y.mean(-1, keepdim=True)
    var = ((y - mean) ** 2).mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + 1e-5)
    return (y - mean) * rstd * gamma.double() + beta.double(), mean[:, 0], rstd[:, 0]


def within(out, ref, atol, what):
    """|out - ref| <= 2^-8 |ref| + atol element-wise"""
    out, ref = out.double(), ref.double()
    bad = ((out - ref).abs() > EPS * ref.abs() + atol) | out.isnan()
    assert not bad.any(), f"{what}: {int(bad.sum())} elements off, worst |diff| {(out - ref).abs().nan_to_num(1e30).max():.3e}"


def attention(q, k, v, allowed):
    """one commit, one head: q [T, 32], k / v [n, 32], allowed [T, n] -> ctx, (max in natural-log units, l)"""
    s = (q.double() @ k.double().t()) / DH ** 0.5
    s = s.masked_fill(~allowed, -1e9)
    m = s.max(-1, keepdim=True).values
    e = torch.exp(s - m)
    l = e.sum(-1, keepdim=True)
    return (e / l) @ v.double(), m[:, 0], l[:, 0]


def check_attention(ctx, stats, q, kvk, kvv, keys, B, T, what):
    """ctx [B*T, 256], stats [B, H, T, 2] against the restatement; P is rounded to bf16 before P V (2^-8 of max|v|).
    keys(b) -> (K/V rows of commit b's key list, allowed [T, n])"""
    for b in range(B):
        rows, allowed = keys(b)
        for h in range(H):
            c = slice(h * DH, (h + 1) * DH)
            qb = q[b * T:(b + 1) * T, c]
            kb, vb = kvk[rows][:, c], kvv[rows][:, c]
            ref, m, l = attention(qb, kb, vb, allowed)
            within(ctx[b * T:(b + 1) * T, c], ref, 2 ** -8 * vb.double().abs().max().item(), f"{what} ctx b{b} h{h}")
            within(stats[b, h, :, 0], m, 1e-5, f"{what} max b{b} h{h}")
            within(stats[b, h, :, 1], l, 0.0, f"{what} l b{b} h{h}")


def check_all(bt, o):
    B, T = bt.B, bt.T
    Mt = B * T
    x0 = bt.emb[bt.tar.long().view(-1)] + bt.pe[:T].repeat(B, 1)        # fp32 sum, then one rounding
    within(o["X"][0], x0.to(BF), 0.0, "embedding")
    causal = torch.tril(torch.ones(T, T, dtype=torch.bool, device=DEV))
    for i, w in enumerate(bt.w):
        X, qkv = o["X"][i], o["qkv"][i]
        close16(qkv, lin(X, w["wqkv"], w["bqkv"]), what=f"L{i} qkv")

        def self_keys(b):
            # a row without a valid key has every score at -1e9: uniform over all T keys, max -1e9, l = T
            allowed = causal & bt.tar_mask[b].bool()[None, :]
            return torch.arange(b * T, (b + 1) * T, device=DEV), allowed
        check_attention(o["ctx1"][i], o["st1"][i], qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:],
                        self_keys, B, T, f"L{i} self")
        close16(o["z1"][i], lin(o["ctx1"][i], w["swo"], w["sbo"]), what=f"L{i} z1")
        for site, (z, res, out, ls, g, be) in enumerate(((o["z1"][i], X, o["x1"][i], o["ls1"][i], w["slw"], w["slb"]),
                                                         (o["z2"][i], o["x1"][i], o["x2"][i], o["ls2"][i], w["clw"], w["clb"]),
                                                         (o["z3"][i], o["x2"][i], o["X"][i + 1], o["ls3"][i], w["flw"], w["flb"]))):
            ref, mean, rstd = ln(z, res, g, be)
            close16(out, ref, what=f"L{i} LayerNorm {site}")
            within(ls[0], mean, 1e-5 * mean.abs().max().item(), f"L{i} mean {site}")
            within(ls[1], rstd, 0.0, f"L{i} rstd {site}")
        close16(o["q"][i], lin(o["x1"][i], w["cwq"], w["cbq"]), what=f"L{i} q")

        def cross_keys(b):
            rows, valid = bt.keys(b)
            return rows, valid[None, :].expand(T, -1)      # no valid key: uniform over the commit's whole list
        kv = bt.kv[:, i * 2 * D:(i + 1) * 2 * D]
        check_attention(o["ctx2"][i], o["st2"][i], o["q"][i], kv[:, :D], kv[:, D:], cross_keys, B, T,
                        f"L{i} cross")
        close16(o["z2"][i], lin(o["ctx2"][i], w["cwo"], w["cbo"]), what=f"L{i} z2")
        close16(o["hh"][i], lin(o["x2"][i], w["w1"], w["b1"], relu=True), what=f"L{i} hh")
        close16(o["z3"][i], lin(o["hh"][i], w["w2"], w["b2"]), what=f"L{i} z3")
    assert not any(bool(t.isnan().any()) for t in o.values())
    assert o["X"].shape[1] == Mt


def _hand_no_valid_key():
    lay = hand_layout()
    lay.mask[1] = False                                      # the single-row commit: no valid key
    return lay


CASES = {
    "padded T=30": lambda: Batch(7, 30, 1),
    "padded T=32": lambda: Batch(7, 32, 2),
    "packed hand T=30": lambda: Batch(5, 30, 3, layout=_hand_no_valid_key()),
    "packed golden T=30": lambda: Batch(6, 30, 4, layout=real_layout([100, 3, 77, 127, 64, 9])),
}


@pytest.mark.parametrize("case", list(CASES))
def test_decoder_fwd_matches_float64(case):
    bt = CASES[case]()
    check_all(bt, run(bt))


def test_layouts_have_the_edge_cases():
    lay = _hand_no_valid_key()
    assert 0 in [n1 for *_, n1 in lay.ranges] and not bool(lay.mask[1].any())
    bt = Batch(7, 30, 1)
    assert not bool(bt.mem_mask[2].any()) and int(bt.tar_mask[1, 0]) == 0


# ------------------------------------------------------------------ the live-row slot layout (fira_decoder_fwd_rows)
SLOT_NAMES = ("qkv", "ctx1", "z1", "x1", "q", "ctx2", "z2", "x2", "hh", "z3")      # with X: the 11 bf16 tensors
GUARD = 64                      # elements after each buffer that no call may write
FILL = 3.0                      # their value (exact in bf16)


def target_map(label, R):
    """fira_target_rows on labels [B, T] -> device tlen [B], toff [B+1], trows [R] (-1: a pad slot)"""
    from fira_icse_b200 import _lib
    B, T = label.shape
    lab = torch.as_tensor(label, dtype=torch.int32).to(DEV)
    m = torch.full((2 * B + 1 + R,), 7, dtype=torch.int32, device=DEV)
    p = m.data_ptr()
    _lib.call("fira_target_rows", lab.data_ptr(), B, T, p, p + 4 * B, p + 4 * (2 * B + 1), R, st())
    torch.cuda.synchronize()
    return m[:B], m[B:2 * B + 1], m[2 * B + 1:]


def live_labels(bt, counts):
    """labels [B, T] whose commit b has counts[b] live rows, a zero label inside the longest message"""
    lab = torch.zeros(bt.B, bt.T, dtype=torch.int32)
    for b, n in enumerate(counts):
        lab[b, :n] = 5 + b
        assert n == 0 or int(bt.tar_mask[b, 0]) == 1, "a labelled commit's row 0 must be a valid key (DecoderFn)"
    lab[max(range(bt.B), key=lambda b: counts[b]), 2] = 0
    return lab


def run_rows(bt, tlen, toff, R, p=0.0, seed=0, sid=64):
    """fira_decoder_fwd_rows with the map (tlen, toff) and R slots: every buffer starts as NaN, followed by GUARD
    elements of FILL -> (outputs, guards)"""
    from fira_icse_b200 import _lib
    B, T = bt.B, bt.T
    o, guards = {}, {}

    def e(name, *shape, dtype=BF):
        n = 1
        for s in shape:
            n *= s
        buf = torch.full((n + GUARD,), float("nan"), dtype=dtype, device=DEV)
        buf[n:] = FILL
        o[name], guards[name] = buf[:n].view(*shape), buf[n:]
    e("X", L, R, D)
    e("out", B * T, D)
    e("qkv", L, R, 3 * D)
    e("hh", L, R, F)
    for n in ("ctx1", "z1", "x1", "q", "ctx2", "z2", "x2", "z3"):
        e(n, L, R, D)
    for n in ("st1", "st2"):
        e(n, L, B, H, T, 2, dtype=torch.float32)
    for n in ("ls1", "ls2", "ls3"):
        e(n, L, 2, R, dtype=torch.float32)
    ptr = {k: v.data_ptr() for k, v in o.items()}
    _lib.call("fira_decoder_fwd_rows", bt.tar.data_ptr(), bt.emb.data_ptr(), bt.pe.data_ptr(), bt.tar_mask.data_ptr(),
              bt.kv.data_ptr(), bt.kv.shape[1], bt.mem_mask.data_ptr(),
              bt.ranges.data_ptr() if bt.ranges is not None else None, bt.S, ctypes.addressof(bt.table), L,
              ptr["X"], ptr["out"], ptr["qkv"], ptr["ctx1"], ptr["st1"], ptr["z1"], ptr["ls1"], ptr["x1"], ptr["q"],
              ptr["ctx2"], ptr["st2"], ptr["z2"], ptr["ls2"], ptr["x2"], ptr["hh"], ptr["z3"], ptr["ls3"],
              tlen.data_ptr(), toff.data_ptr(), R, B, T, float(p), seed, None, sid, st())
    torch.cuda.synchronize()
    return o, guards


def check_slots(bt, full, o, guards, tlen, toff, trows):
    """the slot layout against the map-less run `full` (checked against float64 by test_decoder_fwd_matches_float64):
    slots bit-equal to their rows, pad slots zero, out = the last layer's rows / zero past tlen / NaN for a live row
    without a slot, st1 / st2 unchanged, nothing written past any buffer"""
    B, T = bt.B, bt.T
    R = trows.numel()
    nl = int(toff[B])
    rows = trows[:nl].long()
    assert bool((rows >= 0).all()) and bool((trows[nl:] == -1).all())
    saved = dict((n, full[n]) for n in SLOT_NAMES)
    saved["X"] = full["X"][:L]
    for n, t in saved.items():
        assert torch.equal(o[n][:, :nl], t[:, rows]), f"{n}: a slot differs from its row"
        assert bool((o[n][:, nl:] == 0).all()), f"{n}: a pad slot is not zero"
    for n in ("ls1", "ls2", "ls3"):
        assert torch.equal(o[n][:, :, :nl], full[n][:, :, rows]), f"{n}: a slot differs from its row"
    for n in ("st1", "st2"):
        assert torch.equal(o[n], full[n]), f"{n}: the [L, B, H, T, 2] statistics changed"
    tl, to = tlen.long().cpu(), toff.long().cpu()
    t_idx = torch.arange(T)
    slotted = (t_idx[None, :] < (to[1:] - to[:-1])[:, None]).view(-1).to(DEV)
    alive = (t_idx[None, :] < tl[:, None]).view(-1).to(DEV)
    last = full["X"][L]
    assert torch.equal(o["out"][slotted], last[slotted]), "out: a live row differs from the map-less output"
    assert bool((o["out"][~alive] == 0).all()), "out: a row past tlen is not zero"
    assert bool(o["out"][alive & ~slotted].isnan().all()), "out: a live row without a slot is not NaN"
    for n, g in guards.items():
        assert bool((g == FILL).all()), f"{n}: written past the end of the buffer"
    return R - nl


# case -> (live rows per commit, p): every case has empty, 1-row, 16 / 17-row and full-length commits
SLOT_CASES = {
    "padded T=30": ([30, 0, 1, 16, 17, 9, 29], 0.0),
    "padded T=30 dropout": ([30, 0, 1, 16, 17, 9, 29], 0.2),
    "padded T=32": ([32, 0, 17, 1, 16, 31, 3], 0.0),
    "packed hand T=30": ([30, 0, 17, 1, 16], 0.0),
}


@pytest.mark.parametrize("slots", ["exact", "pad", "short"])
@pytest.mark.parametrize("case", list(SLOT_CASES))
def test_decoder_fwd_rows_slot_layout(case, slots):
    """fira_decoder_fwd_rows on the same batch as fira_decoder_fwd: R = the live count, R with pad slots, and R below
    the live count (the commits past the last slot come up short)"""
    counts, p = SLOT_CASES[case]
    bt = CASES[case.replace(" dropout", "")]()
    full = run(bt, p=p, seed=77, sid=64)
    lab = live_labels(bt, counts)
    n = sum(counts)
    R = {"exact": n, "pad": min(n + 37, bt.B * bt.T), "short": n - 20}[slots]
    tlen, toff, trows = target_map(lab, R)
    assert tlen.tolist() == counts
    o, guards = run_rows(bt, tlen, toff, R, p=p, seed=77, sid=64)
    pad = check_slots(bt, full, o, guards, tlen, toff, trows)
    assert pad == {"exact": 0, "pad": R - n, "short": 0}[slots]
    if slots == "short":
        assert bool(o["out"].isnan().any())


def test_decoder_fwd_rows_bad_arguments():
    """tlen without toff, R = 0 and R > B*T with a map are refused with an error code, before any launch"""
    from fira_icse_b200 import _lib
    bt = CASES["padded T=30"]()
    B, T = bt.B, bt.T
    tlen, toff, _ = target_map(live_labels(bt, SLOT_CASES["padded T=30"][0]), B * T)
    X = torch.zeros(L, B * T, 4 * F, dtype=BF, device=DEV)
    f = torch.zeros(L, B, H, T, 2, device=DEV)
    x, s = X.data_ptr(), f.data_ptr()

    def call(tl, to, R):
        _lib.call("fira_decoder_fwd_rows", bt.tar.data_ptr(), bt.emb.data_ptr(), bt.pe.data_ptr(),
                  bt.tar_mask.data_ptr(), bt.kv.data_ptr(), bt.kv.shape[1], bt.mem_mask.data_ptr(), None, bt.S,
                  ctypes.addressof(bt.table), L, x, x, x, x, s, x, s, x, x, x, s, x, s, x, x, x, s, tl, to, R, B, T,
                  0.0, 0, None, 64, st())
    for tl, to, R in ((tlen.data_ptr(), None, B * T), (None, toff.data_ptr(), B * T),
                      (tlen.data_ptr(), toff.data_ptr(), 0), (tlen.data_ptr(), toff.data_ptr(), B * T + 1)):
        with pytest.raises(_lib.FiraLibraryError, match="tlen and toff"):
            call(tl, to, R)
    torch.cuda.synchronize()
    assert bool((X == 0).all()) and bool((f == 0).all())


@pytest.mark.parametrize("case", ["padded T=30", "packed hand T=30"])
def test_decoder_fwd_dropout_masks(case):
    """p = 0.2: the LayerNorm block run on the kernel's own z and residual with the same key reproduces each output"""
    from fira_icse_b200 import _lib
    bt = CASES[case]()
    seed, sid, p = 1234, 64, 0.2
    o = run(bt, p=p, seed=seed, sid=sid)
    Mt = bt.B * bt.T
    for i, w in enumerate(bt.w):
        for site, (z, res, out, g, be) in enumerate(((o["z1"][i], o["X"][i], o["x1"][i], w["slw"], w["slb"]),
                                                     (o["z2"][i], o["x1"][i], o["x2"][i], w["clw"], w["clb"]),
                                                     (o["z3"][i], o["x2"][i], o["X"][i + 1], w["flw"], w["flb"]))):
            ref = torch.empty_like(out)
            stats = torch.empty(2, Mt, device=DEV)
            _lib.call("fira_ln_residual_fwd", z.data_ptr(), res.data_ptr(), g.data_ptr(), be.data_ptr(), ref.data_ptr(),
                      ref.data_ptr(), Mt, stats.data_ptr(), stats.data_ptr() + 4 * Mt, Mt, D, p, seed, None,
                      sid + 8 * i + site, 1, st())
            torch.cuda.synchronize()
            close16(out, ref.double(), what=f"L{i} dropout LayerNorm {site}")
            nodrop, _, _ = ln(z, res, g, be)
            assert (out.double() - nodrop).abs().max().item() > 0.1       # the masks did drop something
