"""bf16 attention on the tensor cores (attn_mma_fwd/bwd_kernel, attention.cu) against a float64 restatement of
gnn_transformer.py:144-156 on the same bf16-rounded inputs: the packed form (two key row ranges per commit), the
incremental-decoding form (few query rows, no statistics), causal rows without a valid key, and key counts beyond
any fixed chunk budget.  Tolerances as in test_gpu_ops_bf16.py: P is rounded to bf16 before P.V (2^-8 of the
largest output), the backward consumes bf16 P / dS and the bf16 forward output (2^-6).  The packed form also runs on
the FFMA kernels (fp32 parity mode at the fp32 bounds of test_gpu_ops.py, bf16 with FIRA_ATTN_TC=0), and all three
kernels must reproduce the padded entry points bit for bit on the same keys.  fira_attn_bwd_rows, the backward on the
training step's live-row slots, is checked against float64 over the live query rows alone."""
import math

import pytest
import torch

from test_gpu_ops import close
from test_gpu_ops_bf16 import BF, DEV, close16, rnd16, rnd32, st

pytestmark = pytest.mark.gpu

H, DH = 8, 32
D = H * DH


@pytest.fixture(scope="module", autouse=True)
def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _ref(q, k, v, mask, causal):
    """q [Lq, D], k / v [L, D] (float64, autograd leaves or views of them), mask [L] bool -> [Lq, D]"""
    Lq, L = q.shape[0], k.shape[0]
    Q, K, V = (x.reshape(-1, H, DH).transpose(0, 1) for x in (q, k, v))
    m = mask[None, None, :].expand(H, Lq, L)
    if causal:
        m = m & torch.tril(torch.ones(Lq, L, dtype=torch.bool, device=DEV))[None]
    s = (Q @ K.transpose(-1, -2) / math.sqrt(DH)).masked_fill(~m, -1e9)
    return (torch.softmax(s, -1) @ V).transpose(0, 1).reshape(Lq, D)


# (code rows, sub-token rows, mask rule): a long first range, an empty second range, no valid key at all,
# a commit whose keys are all valid, ranges that straddle a 64-key block boundary
PACKED_SPEC = [(150, 27, "rand"), (100, 0, "rand"), (40, 12, "none"), (7, 3, "all"), (61, 70, "rand")]
SENTINEL = 3.0


def _packed_layout(spec=PACKED_SPEC):
    """-> ranges [B][4], mask [B, pitch] bool, pitch, kv_rows; rows outside every range lie between and after them"""
    B = len(spec)
    pitch = max(a + b for a, b, _ in spec) + 5
    gm = torch.Generator().manual_seed(7)
    ranges, mask = [], torch.zeros(B, pitch, dtype=torch.bool)
    row = 3                                                   # rows outside every range must stay untouched
    code_rows = []
    for b, (n0, n1, rule) in enumerate(spec):
        code_rows.append(row)
        row += n0 + 2
    sub_rows = []
    for b, (n0, n1, rule) in enumerate(spec):
        sub_rows.append(row)
        row += n1 + 1
    kv_rows = row + 4
    for b, (n0, n1, rule) in enumerate(spec):
        ranges.append([code_rows[b], n0, sub_rows[b], n1])
        L = n0 + n1
        if rule == "rand":
            mask[b, :L] = torch.rand(L, generator=gm) > 0.3
        elif rule == "all":
            mask[b, :L] = True
    return ranges, mask, pitch, kv_rows


def _key_rows(r):
    s0, n0, s1, n1 = r
    return torch.cat([torch.arange(s0, s0 + n0), torch.arange(s1, s1 + n1)])


def _packed_inputs(dtype, B, Lq, kv_rows):
    if dtype == 1:
        return rnd16(B * Lq, D, seed=1), rnd16(kv_rows, 2 * D, seed=2), rnd16(B * Lq, D, seed=4)
    return rnd32(B * Lq, D, seed=1), rnd32(kv_rows, 2 * D, seed=2), rnd32(B * Lq, D, seed=4)


def _run_attn(q, kv, go, mask, dtype, ranges=None, Lk=None):
    """fwd + bwd through fira_attn_packed_* (ranges given; keys = rows of kv) or fira_attn_* (padded: commit b's keys at
    rows b*Lk ..) -> ctx, stats, dq, dkv (dkv starts as SENTINEL)"""
    from fira_icse_b200 import _lib
    B, pitch = mask.shape
    Lq = q.shape[0] // B
    vo = kv.data_ptr() + D * kv.element_size()
    mask_u8 = mask.to(torch.uint8).to(DEV)
    ctx = torch.empty(B * Lq, D, device=DEV, dtype=q.dtype)
    stats = torch.empty(B, H, Lq, 2, device=DEV)
    dq = torch.empty_like(q)
    dkv = torch.full_like(kv, SENTINEL)
    dvo = dkv.data_ptr() + D * dkv.element_size()
    if ranges is not None:
        rg = torch.tensor(ranges, dtype=torch.int32, device=DEV)
        _lib.call("fira_attn_packed_fwd", q.data_ptr(), D, kv.data_ptr(), 2 * D, vo, 2 * D, rg.data_ptr(), kv.shape[0],
                  mask_u8.data_ptr(), pitch, 1, ctx.data_ptr(), D, stats.data_ptr(), B, H, Lq, DH, dtype, st())
        _lib.call("fira_attn_packed_bwd", q.data_ptr(), D, kv.data_ptr(), 2 * D, vo, 2 * D, rg.data_ptr(), kv.shape[0],
                  mask_u8.data_ptr(), pitch, 1, ctx.data_ptr(), go.data_ptr(), D, stats.data_ptr(), dq.data_ptr(), D,
                  dkv.data_ptr(), 2 * D, dvo, 2 * D, B, H, Lq, DH, dtype, st())
    else:
        _lib.call("fira_attn_fwd", q.data_ptr(), D, kv.data_ptr(), 2 * D, vo, 2 * D, mask_u8.data_ptr(), 0, ctx.data_ptr(),
                  D, stats.data_ptr(), B, H, Lq, Lk, DH, dtype, st())
        _lib.call("fira_attn_bwd", q.data_ptr(), D, kv.data_ptr(), 2 * D, vo, 2 * D, mask_u8.data_ptr(), 0, ctx.data_ptr(),
                  go.data_ptr(), D, stats.data_ptr(), dq.data_ptr(), D, dkv.data_ptr(), 2 * D, dvo, 2 * D, B, H, Lq, Lk, DH,
                  dtype, st())
    torch.cuda.synchronize()
    return ctx, stats, dq, dkv


def _check_packed_against_float64(dtype):
    """the packed spec through fira_attn_packed_fwd / _bwd against _ref per commit (a commit without a valid key:
    uniform over its own rows); rows outside every range untouched, masked keys exactly zero gradient"""
    Lq = 30
    ranges, mask, pitch, kv_rows = _packed_layout()
    B = len(ranges)
    q, kv, go = _packed_inputs(dtype, B, Lq, kv_rows)
    ctx, stats, dq, dkv = _run_attn(q, kv, go, mask, dtype, ranges=ranges)

    qd = q.double().requires_grad_(True)
    kvd = kv.double().requires_grad_(True)
    outs, touched = [], torch.zeros(kv_rows, dtype=torch.bool)
    for b, (s0, n0, s1, n1) in enumerate(ranges):
        idx = _key_rows(ranges[b]).to(DEV)
        touched[idx.cpu()] = True
        keys = kvd[idx]
        outs.append(_ref(qd[b * Lq:(b + 1) * Lq], keys[:, :D], keys[:, D:], mask[b, :n0 + n1].to(DEV), False))
    ref = torch.cat(outs)
    ref.backward(go.double())
    if dtype == 1:
        # tensor cores: P is rounded to bf16 before P.V; FFMA: fp32 P, one rounding of the output -- the MMA bounds
        # hold for both
        close16(ctx, ref, glob=2.0 ** -8, what="packed attention fwd")
        close16(dq, qd.grad, glob=2.0 ** -6, what="packed attention dq")
        close16(dkv[touched], kvd.grad[touched.to(DEV)], glob=2.0 ** -6, what="packed attention dkv")
    else:                                                     # the fp32 bounds of test_gpu_ops.test_attention_fwd_bwd
        close(ctx, ref, rtol=2e-5, atol=1e-5)
        close(dq, qd.grad, rtol=5e-5, atol=1e-5)
        close(dkv[touched], kvd.grad[touched.to(DEV)], rtol=5e-5, atol=1e-5)
    assert (dkv[~touched.to(DEV)] == SENTINEL).all(), "rows outside every range were written"
    for b, (s0, n0, s1, n1) in enumerate(ranges):
        if PACKED_SPEC[b][2] == "none":
            continue
        dead = _key_rows(ranges[b])[~mask[b, :n0 + n1]]
        assert (dkv[dead.to(DEV)] == 0).all(), "masked keys must get exactly zero gradient"


def test_attention_packed_ranges():
    _check_packed_against_float64(1)


@pytest.mark.parametrize("dtype", [0, 1], ids=["fp32", "bf16"])
def test_attention_packed_ranges_ffma(dtype, monkeypatch):
    """the FFMA kernels on the packed spec: fp32 (parity mode), and bf16 with the tensor-core kernels switched off"""
    monkeypatch.setenv("FIRA_ATTN_TC", "0")
    _check_packed_against_float64(dtype)


@pytest.mark.parametrize("kernel", ["ffma_fp32", "ffma_bf16", "mma"])
def test_attention_packed_equals_padded(kernel, monkeypatch):
    """Packed and padded layouts hold the same valid keys in the same order, and none of the kernels uses atomics:
    ctx, stats, dq and dk / dv of every real key row are bit for bit those of fira_attn_fwd / _bwd on the keys scattered
    into a [B, pitch] layout whose mask is 0 beyond the commit's rows.  A commit without a valid key is the documented
    difference: the padded layout is uniform over all `pitch` keys, the packed one over the commit's own rows (pinned
    against float64 in test_attention_packed_ranges*), so it is left out here."""
    dtype = 0 if kernel == "ffma_fp32" else 1
    monkeypatch.setenv("FIRA_ATTN_TC", "1" if kernel == "mma" else "0")
    Lq = 30
    ranges, mask, pitch, kv_rows = _packed_layout()
    B = len(ranges)
    q, kv, go = _packed_inputs(dtype, B, Lq, kv_rows)
    ctx, stats, dq, dkv = _run_attn(q, kv, go, mask, dtype, ranges=ranges)
    kvp = rnd16(B * pitch, 2 * D, seed=9).to(kv.dtype)        # filler beyond each commit's keys (masked)
    for b in range(B):
        idx = _key_rows(ranges[b]).to(DEV)
        kvp[b * pitch:b * pitch + len(idx)] = kv[idx]
    ctxp, statsp, dqp, dkvp = _run_attn(q, kvp, go, mask, dtype, Lk=pitch)
    compared = 0
    for b in range(B):
        if not mask[b].any():
            continue
        idx = _key_rows(ranges[b]).to(DEV)
        rows = slice(b * Lq, (b + 1) * Lq)
        assert torch.equal(ctx[rows], ctxp[rows]), f"ctx of commit {b}"
        assert torch.equal(stats[b], statsp[b]), f"stats of commit {b}"
        assert torch.equal(dq[rows], dqp[rows]), f"dq of commit {b}"
        assert torch.equal(dkv[idx], dkvp[b * pitch:b * pitch + len(idx)]), f"dk / dv of commit {b}"
        compared += 1
    assert compared == B - 1


@pytest.mark.parametrize("Lq,Lk,causal", [(5, 30, 0), (1, 30, 0), (17, 700, 0), (30, 30, 1)])
def test_attention_padded_shapes(Lq, Lk, causal):
    """Lq < 30 with stats = NULL (incremental decoding), Lk far above 384, causal rows whose keys are all padded"""
    from fira_icse_b200 import _lib
    B = 4
    q = rnd16(B * Lq, D, seed=11)
    kv = rnd16(B * Lk, 2 * D, seed=12)
    gm = torch.Generator().manual_seed(13)
    mask = torch.rand(B, Lk, generator=gm) > 0.4
    mask[0] = True
    if causal:
        mask[1, :4] = False                                   # rows 0..3 of commit 1: no valid key (uniform)
    else:
        mask[2] = False                                       # one commit without a valid key
    mask_u8 = mask.to(torch.uint8).to(DEV)
    ctx = torch.empty(B * Lq, D, device=DEV, dtype=BF)
    _lib.call("fira_attn_fwd", q.data_ptr(), D, kv.data_ptr(), 2 * D, kv.data_ptr() + 2 * D, 2 * D, mask_u8.data_ptr(),
              causal, ctx.data_ptr(), D, None, B, H, Lq, Lk, DH, 1, st())
    qd = q.double().requires_grad_(True)
    kvd = kv.double().requires_grad_(True)
    ref = torch.cat([_ref(qd[b * Lq:(b + 1) * Lq], kvd[b * Lk:(b + 1) * Lk, :D], kvd[b * Lk:(b + 1) * Lk, D:],
                          mask[b].to(DEV), causal) for b in range(B)])
    close16(ctx, ref, glob=2.0 ** -8, what="attention fwd (no stats)")
    # the same shapes through the backward, with statistics
    stats = torch.empty(B, H, Lq, 2, device=DEV)
    _lib.call("fira_attn_fwd", q.data_ptr(), D, kv.data_ptr(), 2 * D, kv.data_ptr() + 2 * D, 2 * D, mask_u8.data_ptr(),
              causal, ctx.data_ptr(), D, stats.data_ptr(), B, H, Lq, Lk, DH, 1, st())
    close16(ctx, ref, glob=2.0 ** -8, what="attention fwd")
    go = rnd16(B * Lq, D, seed=14)
    dq, dkv = torch.empty_like(q), torch.empty_like(kv)
    _lib.call("fira_attn_bwd", q.data_ptr(), D, kv.data_ptr(), 2 * D, kv.data_ptr() + 2 * D, 2 * D, mask_u8.data_ptr(),
              causal, ctx.data_ptr(), go.data_ptr(), D, stats.data_ptr(), dq.data_ptr(), D, dkv.data_ptr(), 2 * D,
              dkv.data_ptr() + 2 * D, 2 * D, B, H, Lq, Lk, DH, 1, st())
    ref.backward(go.double())
    close16(dq, qd.grad, glob=2.0 ** -6, what="attention dq")
    close16(dkv, kvd.grad, glob=2.0 ** -6, what="attention dkv")


# ------------------------------------------------------------------ the backward on live-row slots (fira_attn_bwd_rows)
# layout -> (T, key ranges, live query rows per commit): counts at the m16 edge (1, 15, 16, 17) and the LQ_MAX edge
# (a fully live 32-row commit), a commit without live rows inside the batch and one last (its CTAs zero the pad rows)
SLOT_LAYOUTS = {
    "T30": (30, PACKED_SPEC + [(33, 64, "rand")], [17, 30, 1, 0, 15, 16]),
    "T32_empty_last": (32, PACKED_SPEC, [32, 16, 1, 17, 0]),
}


def _slots(counts, T, pad):
    """-> qoff [B+1], trows [R] (row b*T + t of each slot, -1 for the pad slots) for live rows t < counts[b]"""
    qoff = [0]
    for n in counts:
        qoff.append(qoff[-1] + n)
    trows = [b * T + t for b, n in enumerate(counts) for t in range(n)] + [-1] * pad
    return qoff, torch.tensor(trows, device=DEV)


@pytest.mark.parametrize("pad", [0, 21], ids=["R_exact", "R_pad"])
@pytest.mark.parametrize("layout", list(SLOT_LAYOUTS))
@pytest.mark.parametrize("causal", [1, 0], ids=["self", "cross"])
def test_attention_backward_on_slots_against_float64(causal, layout, pad):
    """forward on every row (fira_attn_fwd causal over tar_mask / fira_attn_packed_fwd), then the live rows gathered into
    slots qoff[b] + t and fira_attn_bwd_rows against float64 autograd over those rows alone.  Causal keys are the commit's
    slots, cross keys its packed ranges.  dq and the causal dk / dv start as NaN, the cross dk / dv as SENTINEL: every key
    row of every range is written (a commit without live rows: exactly zero), masked keys get exactly zero, rows outside
    the ranges stay SENTINEL, pad slots come back zero"""
    from fira_icse_b200 import _lib
    T, spec, counts = SLOT_LAYOUTS[layout]
    B = len(counts)
    qoff, trows = _slots(counts, T, pad)
    qoff_d = torch.tensor(qoff, dtype=torch.int32, device=DEV)
    nl, R = qoff[B], qoff[B] + pad
    tm = torch.ones(B, T, dtype=torch.uint8, device=DEV)
    tm[0, 5] = 0                                              # a masked key among commit 0's live rows
    for b, n in enumerate(counts):
        tm[b, n + 2:] = 0                                     # padding past the message (never a live row's key)
    ranges, mask, pitch, kv_rows = _packed_layout(spec)
    stats = torch.empty(B, H, T, 2, device=DEV)
    ctx = torch.empty(B * T, D, device=DEV, dtype=BF)
    if causal:
        qkv = rnd16(B * T, 3 * D, seed=21)
        _lib.call("fira_attn_fwd", qkv.data_ptr(), 3 * D, qkv[:, D:].data_ptr(), 3 * D, qkv[:, 2 * D:].data_ptr(),
                  3 * D, tm.data_ptr(), 1, ctx.data_ptr(), D, stats.data_ptr(), B, H, T, T, DH, 1, st())
        q = qkv[:, :D]
    else:
        q, kv = rnd16(B * T, D, seed=22), rnd16(kv_rows, 2 * D, seed=23)
        rg = torch.tensor(ranges, dtype=torch.int32, device=DEV)
        mask_u8 = mask.to(torch.uint8).to(DEV)
        _lib.call("fira_attn_packed_fwd", q.data_ptr(), D, kv.data_ptr(), 2 * D, kv[:, D:].data_ptr(), 2 * D,
                  rg.data_ptr(), kv_rows, mask_u8.data_ptr(), pitch, 1, ctx.data_ptr(), D, stats.data_ptr(), B, H, T,
                  DH, 1, st())
    idx, padm = trows.clamp(min=0), (trows < 0)[:, None]

    def gather(x):
        return x[idx].masked_fill(padm, 0).contiguous()
    q_s, ctx_s = gather(q), gather(ctx)
    go_s = rnd16(R, D, seed=24).masked_fill(padm, 0).contiguous()
    nan = float("nan")
    dq_s = torch.full((R, D), nan, device=DEV, dtype=BF)
    if causal:
        qkv_s = gather(qkv)
        dqkv_s = torch.full((R, 3 * D), nan, device=DEV, dtype=BF)
        _lib.call("fira_attn_bwd_rows", qkv_s.data_ptr(), 3 * D, qkv_s[:, D:].data_ptr(), 3 * D,
                  qkv_s[:, 2 * D:].data_ptr(), 3 * D, None, tm.data_ptr(), T, 1, qoff_d.data_ptr(), R,
                  ctx_s.data_ptr(), go_s.data_ptr(), D, stats.data_ptr(), dqkv_s.data_ptr(), 3 * D,
                  dqkv_s[:, D:].data_ptr(), 3 * D, dqkv_s[:, 2 * D:].data_ptr(), 3 * D, B, H, T, DH, 1, st())
        dq_s = dqkv_s[:, :D]
    else:
        dkv = torch.full_like(kv, SENTINEL)
        _lib.call("fira_attn_bwd_rows", q_s.data_ptr(), D, kv.data_ptr(), 2 * D, kv[:, D:].data_ptr(), 2 * D,
                  rg.data_ptr(), mask_u8.data_ptr(), pitch, 0, qoff_d.data_ptr(), R, ctx_s.data_ptr(), go_s.data_ptr(),
                  D, stats.data_ptr(), dq_s.data_ptr(), D, dkv.data_ptr(), 2 * D, dkv[:, D:].data_ptr(), 2 * D,
                  B, H, T, DH, 1, st())
    torch.cuda.synchronize()

    # float64 autograd over the live query rows only
    qd = q_s.double().requires_grad_(True)
    outs = []
    if causal:
        kvd = qkv_s[:, D:].double().requires_grad_(True)
        for b in range(B):
            s = slice(qoff[b], qoff[b + 1])
            if qoff[b + 1] > qoff[b]:
                outs.append(_ref(qd[s], kvd[s, :D], kvd[s, D:], tm[b, :qoff[b + 1] - qoff[b]].bool(), True))
    else:
        kvd = kv.double().requires_grad_(True)
        for b in range(B):
            keys = kvd[_key_rows(ranges[b]).to(DEV)]
            s0, n0, s1, n1 = ranges[b]
            if qoff[b + 1] > qoff[b]:
                outs.append(_ref(qd[qoff[b]:qoff[b + 1]], keys[:, :D], keys[:, D:], mask[b, :n0 + n1].to(DEV), False))
    torch.cat(outs).backward(go_s[:nl].double())

    assert not dq_s.isnan().any(), "dq: a slot was not written"
    close16(dq_s[:nl], qd.grad[:nl], glob=2.0 ** -6, what="slot attention dq")
    assert (dq_s[nl:] == 0).all(), "dq: a pad slot is not zero"
    if causal:
        dkv_s = dqkv_s[:, D:]
        assert not dkv_s.isnan().any(), "dk / dv: a slot was not written"
        close16(dkv_s[:nl], kvd.grad[:nl], glob=2.0 ** -6, what="slot attention causal dk / dv")
        assert (dkv_s[nl:] == 0).all(), "dk / dv: a pad slot is not zero"
        dead = [qoff[b] + t for b in range(B) for t in range(qoff[b + 1] - qoff[b]) if not tm[b, t]]
        assert dead and (dkv_s[dead] == 0).all(), "masked keys must get exactly zero gradient"
        return
    touched = torch.zeros(kv_rows, dtype=torch.bool)
    for b in range(B):
        rows = _key_rows(ranges[b])
        touched[rows] = True
        n0, n1 = ranges[b][1], ranges[b][3]
        if qoff[b + 1] == qoff[b]:
            assert (dkv[rows.to(DEV)] == 0).all(), f"commit {b} has no live row: its keys must get exactly zero"
        elif spec[b][2] != "none":
            assert (dkv[rows[~mask[b, :n0 + n1]].to(DEV)] == 0).all(), "masked keys must get exactly zero gradient"
    td = touched.to(DEV)
    close16(dkv[td], kvd.grad[td], glob=2.0 ** -6, what="slot attention cross dk / dv")
    assert (dkv[~td] == SENTINEL).all(), "rows outside every range were written"
