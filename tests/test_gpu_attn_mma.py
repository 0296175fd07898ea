"""bf16 attention on the tensor cores (attn_mma_fwd/bwd_kernel, attention.cu) against a float64 restatement of
gnn_transformer.py:144-156 on the same bf16-rounded inputs: the packed form (two key row ranges per commit), the
incremental-decoding form (few query rows, no statistics), causal rows without a valid key, and key counts beyond
any fixed chunk budget.  Tolerances as in test_gpu_ops_bf16.py: P is rounded to bf16 before P.V (2^-8 of the
largest output), the backward consumes bf16 P / dS and the bf16 forward output (2^-6)."""
import math

import pytest
import torch

from test_gpu_ops_bf16 import BF, DEV, close16, rnd16, st

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


def test_attention_packed_ranges():
    from fira_icse_b200 import _lib
    Lq = 30
    # (code rows, sub-token rows, mask rule): a long first range, an empty second range, no valid key at all,
    # a commit whose keys are all valid, ranges that straddle a 64-key block boundary
    spec = [(150, 27, "rand"), (100, 0, "rand"), (40, 12, "none"), (7, 3, "all"), (61, 70, "rand")]
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
    rg = torch.tensor(ranges, dtype=torch.int32, device=DEV)
    mask_u8 = mask.to(torch.uint8).to(DEV)
    q = rnd16(B * Lq, D, seed=1)
    kv = rnd16(kv_rows, 2 * D, seed=2)
    ctx = torch.empty(B * Lq, D, device=DEV, dtype=BF)
    stats = torch.empty(B, H, Lq, 2, device=DEV)
    _lib.call("fira_attn_packed_fwd", q.data_ptr(), D, kv.data_ptr(), 2 * D, kv.data_ptr() + 2 * D, 2 * D, rg.data_ptr(),
              kv_rows, mask_u8.data_ptr(), pitch, 1, ctx.data_ptr(), D, stats.data_ptr(), B, H, Lq, DH, 1, st())
    go = rnd16(B * Lq, D, seed=4)
    dq = torch.empty_like(q)
    sentinel = 3.0
    dkv = torch.full_like(kv, sentinel)
    _lib.call("fira_attn_packed_bwd", q.data_ptr(), D, kv.data_ptr(), 2 * D, kv.data_ptr() + 2 * D, 2 * D, rg.data_ptr(),
              kv_rows, mask_u8.data_ptr(), pitch, 1, ctx.data_ptr(), go.data_ptr(), D, stats.data_ptr(), dq.data_ptr(), D,
              dkv.data_ptr(), 2 * D, dkv.data_ptr() + 2 * D, 2 * D, B, H, Lq, DH, 1, st())
    torch.cuda.synchronize()

    qd = q.double().requires_grad_(True)
    kvd = kv.double().requires_grad_(True)
    outs, touched = [], torch.zeros(kv_rows, dtype=torch.bool)
    for b, (s0, n0, s1, n1) in enumerate(ranges):
        idx = torch.cat([torch.arange(s0, s0 + n0), torch.arange(s1, s1 + n1)]).to(DEV)
        touched[idx.cpu()] = True
        keys = kvd[idx]
        outs.append(_ref(qd[b * Lq:(b + 1) * Lq], keys[:, :D], keys[:, D:], mask[b, :n0 + n1].to(DEV), False))
    ref = torch.cat(outs)
    close16(ctx, ref, glob=2.0 ** -8, what="packed attention fwd")
    ref.backward(go.double())
    close16(dq, qd.grad, glob=2.0 ** -6, what="packed attention dq")
    close16(dkv[touched], kvd.grad[touched.to(DEV)], glob=2.0 ** -6, what="packed attention dkv")
    assert (dkv[~touched.to(DEV)] == sentinel).all(), "rows outside every range were written"
    for b, (s0, n0, s1, n1) in enumerate(ranges):
        if spec[b][2] == "none":
            continue
        dead = torch.cat([torch.arange(s0, s0 + n0), torch.arange(s1, s1 + n1)])[~mask[b, :n0 + n1]]
        assert (dkv[dead.to(DEV)] == 0).all(), "masked keys must get exactly zero gradient"


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
