"""The training step's decoder on the live target rows only, the rows before each commit's last label (ops.DecoderFn with
cfg["label"]): fira_target_rows against numpy, the LayerNorm backward's slot twin against the row-layout kernel, the
embedding backward through the map against float64, and DecoderFn with the map against DecoderFn without it on a
packed golden batch (the attention backward on slots: tests/test_gpu_attn_mma.py).  The map only
moves rows to other slots, so a live row's forward values are the same, and the gradients agree to the bf16 rounding of
GEMM tiles that now hold other rows."""
import copy

import numpy as np
import pytest
import torch

from bf16_bound import close, small
from fira_testlib import seeded_model
from test_packed import GoldenSplit, V

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
D, H, T = 256, 8, 30


def _st():
    return torch.cuda.current_stream().cuda_stream


def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _target_rows_np(label, cap):
    B, T_ = label.shape
    nz = label != 0
    tlen = np.where(nz.any(1), T_ - np.argmax(nz[:, ::-1], axis=1), 0).astype(np.int32)
    off = np.concatenate(([0], np.cumsum(tlen)))
    toff = np.minimum(off, cap).astype(np.int32)
    trows = np.full(cap, -1, np.int32)
    for b in range(B):
        for t in range(tlen[b]):
            if off[b] + t < cap:
                trows[off[b] + t] = b * T_ + t
    return tlen, toff, trows


def _target_rows_dev(label, cap):
    from fira_icse_b200 import _lib
    B, T_ = label.shape
    lab = torch.as_tensor(label, dtype=torch.int32, device=DEV)
    out = torch.full((2 * B + 1 + cap,), 7, dtype=torch.int32, device=DEV)
    p = out.data_ptr()
    _lib.call("fira_target_rows", lab.data_ptr(), B, T_, p, p + 4 * B, p + 4 * (2 * B + 1), cap, _st())
    torch.cuda.synchronize()
    o = out.cpu().numpy()
    return o[:B], o[B:2 * B + 1], o[2 * B + 1:]


def _labels(B, rng):
    lab = np.zeros((B, T), np.int32)
    for b in range(B):
        n = int(rng.integers(0, T))
        lab[b, :n] = rng.integers(1, V + 40, n)
    lab[0, :9] = rng.integers(1, V, 9)
    lab[0, 9:] = 0
    lab[0, 3] = 0                                   # a zero label inside a message: still live
    lab[1] = 0                                      # a commit without labels
    lab[2, :12] = V + rng.integers(0, 40, 12)       # a commit with copy labels only
    lab[2, 12:] = 0
    return lab


@pytest.mark.parametrize("B", [3, 64])
def test_target_rows_match_numpy(B):
    _need_cuda()
    lab = _labels(B, np.random.default_rng(B))
    n = int(_target_rows_np(lab, B * T)[0].sum())
    for cap in (B * T, n, -(-n // 128) * 128, max(1, n - 5)):     # every row, exact, the 128 bound, a count above cap
        got, want = _target_rows_dev(lab, cap), _target_rows_np(lab, cap)
        for g, w, what in zip(got, want, ("tlen", "toff", "trows")):
            assert np.array_equal(g, w), (cap, what)
    assert _target_rows_dev(lab, B * T)[0][1] == 0 and _target_rows_dev(lab, B * T)[0][0] == 9


def test_target_rows_at_a_128_edge():
    _need_cuda()
    lab = np.zeros((8, T), np.int32)
    lab[:4, :T - 1] = 5                             # 4 x 29 + 12 = 128 live rows
    lab[4, 11] = V + 1
    for cap in (128, 127):
        got, want = _target_rows_dev(lab, cap), _target_rows_np(lab, cap)
        assert all(np.array_equal(g, w) for g, w in zip(got, want)), cap
    assert _target_rows_dev(lab, 127)[1][-1] == 127             # the commit past the slots comes up short


def _map(lab, cap):
    lab_d = torch.as_tensor(lab, dtype=torch.int32, device=DEV)
    B = lab.shape[0]
    m = torch.empty((2 * B + 1 + cap,), dtype=torch.int32, device=DEV)
    p = m.data_ptr()
    from fira_icse_b200 import _lib
    _lib.call("fira_target_rows", lab_d.data_ptr(), B, T, p, p + 4 * B, p + 4 * (2 * B + 1), cap, _st())
    return m[B:2 * B + 1], m[2 * B + 1:]


@pytest.mark.parametrize("dtype", [0, 1], ids=["fp32", "bf16"])
def test_embedding_backward_through_the_map_against_float64(dtype):
    """fira_embed_rows_bwd_rows: slot r adds its gradient row to the embedding row of token ids[rows_map[r]], against a
    float64 index_add over the live slots.  Pad slots (-1), one token id in many slots (atomic adds onto one row), and a
    slot whose gradient row is exactly zero (skipped: the only slot of its token, whose row must stay exactly zero).  The
    adds happen in fp32 in any order: |g - r| <= 2^-20 sum |terms| per element"""
    _need_cuda()
    from fira_icse_b200 import _lib
    B, Vt = 24, 96
    lab = _labels(B, np.random.default_rng(13))
    n = int(_target_rows_np(lab, B * T)[0].sum())
    R = -(-n // 128) * 128
    assert R > n, "the map needs pad slots"
    _, trows = _map(lab, R)
    g = torch.Generator().manual_seed(17)
    ids = torch.randint(1, Vt - 1, (B * T,), generator=g, dtype=torch.int32)       # Vt - 1: only the zero slot
    ids[::3] = 7                                              # one token in a third of the rows
    tr = trows.cpu().long()
    live = tr[tr >= 0]
    zero_slot = int(torch.nonzero(tr >= 0)[len(live) // 2])
    ids[tr[zero_slot]] = Vt - 1                               # the zero-gradient slot's token appears nowhere else
    d_out = torch.randn(R, D, generator=g)
    d_out[zero_slot] = 0.0
    d_out = d_out.to(torch.bfloat16 if dtype else torch.float32)
    d_emb = torch.zeros(Vt, D, device=DEV)
    ids_d, d_out_d = ids.to(DEV), d_out.to(DEV)
    _lib.call("fira_embed_rows_bwd_rows", ids_d.data_ptr(), trows.data_ptr(), d_out_d.data_ptr(), d_emb.data_ptr(), R,
              D, dtype, _st())
    torch.cuda.synchronize()
    slots = torch.nonzero(tr >= 0).view(-1)
    terms = d_out.double()[slots]
    tok = ids[tr[slots]].long()
    ref = torch.zeros(Vt, D, dtype=torch.float64).index_add_(0, tok, terms)
    mag = torch.zeros(Vt, D, dtype=torch.float64).index_add_(0, tok, terms.abs())
    got = d_emb.cpu().double()
    err = (got - ref).abs()
    bound = 2.0 ** -20 * mag
    assert bool((err <= bound).all()), f"{int((err > bound).sum())} elements off, worst {(err - bound).max():.3e}"
    assert int((tok == 7).sum()) > 64, "one row takes many atomic adds"
    assert bool((got[Vt - 1] == 0).all()), "the zero-gradient slot's row"
    untouched = torch.ones(Vt, dtype=torch.bool)
    untouched[tok] = False
    assert bool((got[untouched] == 0).all()), "a row no live slot names was written"


@pytest.mark.parametrize("p", [0.0, 0.1])
def test_layernorm_backward_on_slots_matches_rows(p):
    """fira_ln_residual_bwd_rows == fira_ln_residual_bwd on the gathered rows; the dropout mask follows the row"""
    _need_cuda()
    from fira_icse_b200 import _lib
    B = 16
    lab = _labels(B, np.random.default_rng(7))
    n = int(_target_rows_np(lab, B * T)[0].sum())
    R = -(-n // 128) * 128
    _, trows = _map(lab, R)
    M = B * T
    g = torch.Generator().manual_seed(11)
    bf = dict(dtype=torch.bfloat16, device=DEV)
    z, res, dout = (torch.randn(M, D, generator=g).to(**bf) for _ in range(3))
    gamma, beta = torch.randn(D, generator=g).to(DEV), torch.randn(D, generator=g).to(DEV)
    stats = torch.empty((2, M), dtype=torch.float32, device=DEV)
    y = torch.empty((M, D), **bf)
    _lib.call("fira_ln_residual_fwd", z.data_ptr(), res.data_ptr(), gamma.data_ptr(), beta.data_ptr(), y.data_ptr(),
              y.data_ptr(), M, stats[0].data_ptr(), stats[1].data_ptr(), M, D, float(p), 42, None, 3, 1, _st())
    idx, pad = trows.clamp(min=0).long(), trows < 0

    def slots(x, dim0=True):
        return x[idx].masked_fill(pad[:, None], 0).contiguous() if dim0 else x[:, idx].contiguous()
    dz, dr = torch.empty_like(z), torch.empty_like(z)
    dgb = torch.zeros((2, D), dtype=torch.float32, device=DEV)
    live = torch.zeros(M, dtype=torch.bool, device=DEV)
    live[trows[trows >= 0].long()] = True
    dout_live = (dout * live[:, None]).contiguous()
    _lib.call("fira_ln_residual_bwd", dout_live.data_ptr(), dout_live.data_ptr(), M, z.data_ptr(), res.data_ptr(),
              stats[0].data_ptr(), stats[1].data_ptr(), gamma.data_ptr(), dz.data_ptr(), dr.data_ptr(), 0,
              dgb[0].data_ptr(), dgb[1].data_ptr(), M, D, float(p), 42, None, 3, 1, _st())
    z_s, r_s, d_s, st_s = slots(z), slots(res), slots(dout), slots(stats, False)
    dz_s, dr_s = torch.full_like(z_s, float("nan")), torch.full_like(z_s, float("nan"))
    dgb_s = torch.zeros((2, D), dtype=torch.float32, device=DEV)
    _lib.call("fira_ln_residual_bwd_rows", d_s.data_ptr(), d_s.data_ptr(), R, z_s.data_ptr(), r_s.data_ptr(),
              st_s[0].data_ptr(), st_s[1].data_ptr(), gamma.data_ptr(), dz_s.data_ptr(), dr_s.data_ptr(), 0,
              dgb_s[0].data_ptr(), dgb_s[1].data_ptr(), trows.data_ptr(), R, D, float(p), 42, None, 3, 1, _st())
    torch.cuda.synchronize()
    assert torch.equal(dz_s, slots(dz)) and torch.equal(dr_s, slots(dr))        # pad slots: zeros
    close("layernorm d_gamma / d_beta", dgb_s, dgb, 2 ** -16)


def _decoder_run(model, pb, memory, g_out, p, label):
    from fira_icse_b200 import ops
    dm = model.decoder
    leaves = [t.detach().clone().requires_grad_(True) for t in [dm.embedding.weight] + dm._flat()]
    cfg = {"training": p > 0, "seed": 1234, "stream_base": 0, "heads": 8, "bf16": True, "seed_ctr": None, "p_dec": p,
           "prefetch": None, "packed": pb, "label": label}
    m = memory.clone().requires_grad_(True)
    out = ops.DecoderFn.apply(cfg, pb.tar, m, pb.mem_mask, pb.tar_mask, dm.pos_encode.to(DEV), *leaves)
    out.backward(g_out)
    torch.cuda.synchronize()
    return out.detach(), [m.grad] + [t.grad for t in leaves]


@pytest.mark.parametrize("p", [0.0, 0.1])
def test_decoder_on_live_rows_matches_every_row(p):
    """DecoderFn with the live-row map == without it: live output rows bit-equal, dead rows zero, every gradient within
    the 6-layer bf16 bound (tests/test_gpu_bf16_step.py), given a loss gradient that is zero on the dead rows"""
    _need_cuda()
    from fira_icse_b200.packed import PackedTables, pack_from_dataset
    model = copy.deepcopy(seeded_model()).to(DEV).set_precision("bf16")
    index = np.arange(0, 64)
    pb = pack_from_dataset(PackedTables(GoldenSplit()), index, V).to(DEV)
    lab = pb.label.cpu().numpy().copy()
    assert pb.Rt < pb.B * pb.T
    g = torch.Generator().manual_seed(2)
    memory = torch.randn((1, pb.mem_rows, D), generator=g).to(torch.bfloat16).to(DEV)
    tlen = _target_rows_np(lab, pb.B * T)[0]
    live = torch.as_tensor(np.arange(T)[None, :] < tlen[:, None]).to(DEV)
    g_out = (torch.randn((pb.B, T, D), generator=g).to(DEV) * live[..., None]).to(torch.bfloat16)
    out_all, g_all = _decoder_run(model, pb, memory, g_out, p, None)
    out_map, g_map = _decoder_run(model, pb, memory, g_out, p, pb.label)
    assert torch.equal(out_map[live], out_all[live])
    assert (out_map[~live] == 0).all()
    for i, (a, b) in enumerate(zip(g_map, g_all)):
        if b is None:
            assert a is None
            continue
        if i >= 2 and (i - 2) % 26 in (3, 13):     # fc_k.bias: zero in exact arithmetic, round-off on both sides
            small(f"decoder gradient {i}", a, g_all[i - 1].abs().max().item(), 2 ** -3)
            continue
        close(f"decoder gradient {i}", a.float(), b.float(), 2 ** -3, rows=b.dim() == 2)
