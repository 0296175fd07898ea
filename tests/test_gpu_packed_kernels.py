"""Kernels of the per-commit packed batch (fira_icse_b200/packed.py) called directly through the C ABI on seeded
inputs: the packed copy scores (fira_copy_scores_packed_fwd / _bwd), the segment-padding clear (fira_zero_pad_rows) and
the encoder input with explicit positions (fira_embed_nodes_pos_fwd), in fp32 and bf16.  Each is compared with a
float64 restatement of the same operation over each commit's own rows, and with the padded-layout kernel whose
results it must reproduce bit for bit.  Bounds are those of the padded kernels: tests/test_gpu_ops.py (fp32) and
tests/test_gpu_ops_bf16.py (bf16).

Two kinds of layout: real packed batches of golden commits (default buckets, and enlarged buckets so every segment
ends in padding), and a hand-made ragged one with an empty sub-token range, a single-row commit, commits that cross the
32-row slices of the copy kernels and the 64-key blocks of attention, a pitch far above every commit's row count, and
sentinel rows after each segment that no kernel but fira_zero_pad_rows may write."""
import numpy as np
import pytest
import torch

from test_gpu_ops import close
from test_gpu_ops_bf16 import BF, DEV, close16, rnd16, rnd32, st
from test_packed import GoldenSplit, V

pytestmark = pytest.mark.gpu

D = 256
SENT = 5.0                 # sentinel of rows a kernel must not write


@pytest.fixture(scope="module", autouse=True)
def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


class Layout:
    """Memory rows of a packed batch: ranges[b] = (first code row, code rows, first sub-token row (global), sub-token
    rows), off [3, B + 1] = row offsets of each commit inside the three segments, mask [B, S] (1 = real, unmasked
    memory position), pitch S, segment sizes Rc / Rs (memory rows = Rc + Rs)."""

    def __init__(self, ranges, off, mask, S, Rc, Rs, label=None):
        self.ranges = [tuple(int(x) for x in r) for r in np.asarray(ranges).reshape(-1, 4)]
        self.off = torch.as_tensor(np.asarray(off), dtype=torch.int32).reshape(3, -1)
        self.mask = torch.as_tensor(np.asarray(mask)).to(torch.bool)
        self.S, self.Rc, self.Rs = int(S), int(Rc), int(Rs)
        self.B = len(self.ranges)
        self.label = label

    @property
    def R(self):
        return self.Rc + self.Rs

    def rows(self, b):
        """global memory rows of commit b, in memory-position order"""
        s0, n0, s1, n1 = self.ranges[b]
        return torch.cat([torch.arange(s0, s0 + n0), torch.arange(s1, s1 + n1)])

    def covered(self):
        c = torch.zeros(self.R, dtype=torch.bool)
        for b in range(self.B):
            c[self.rows(b)] = True
        return c

    def padding(self):
        """the segment padding: rows [off[0][B], Rc) and [Rc + off[1][B], Rc + Rs)"""
        p = torch.zeros(self.R, dtype=torch.bool)
        p[int(self.off[0, self.B]):self.Rc] = True
        p[self.Rc + int(self.off[1, self.B]):] = True
        return p

    def dev(self):
        return (torch.tensor(self.ranges, dtype=torch.int32, device=DEV), self.off.to(DEV),
                self.mask.to(torch.uint8).to(DEV))


# (code rows, sub-token rows): an empty sub-token range, a single memory row, memory positions across the 32-row
# slices and the 64-key blocks, a long code range
HAND = [(40, 0), (1, 0), (29, 45), (100, 27), (61, 70)]


def hand_layout(pad=True):
    B = len(HAND)
    off = np.zeros((3, B + 1), np.int32)
    off[0, 1:] = np.cumsum([n0 for n0, _ in HAND])
    off[1, 1:] = np.cumsum([n1 for _, n1 in HAND])
    off[2, 1:] = np.cumsum([3 + 5 * b for b in range(B)])
    Rc = int(off[0, B]) + (25 if pad else 0)
    Rs = int(off[1, B]) + (18 if pad else 0)
    ranges = [(off[0, b], n0, Rc + off[1, b], n1) for b, (n0, n1) in enumerate(HAND)]
    S = 192                                                  # every commit has <= 131 rows
    g = torch.Generator().manual_seed(17)
    mask = torch.zeros(B, S, dtype=torch.bool)
    for b, (n0, n1) in enumerate(HAND):
        mask[b, :n0 + n1] = torch.rand(n0 + n1, generator=g) > 0.3
        mask[b, 0] = True
    return Layout(ranges, off, mask, S, Rc, Rs)


def real_layout(index, bucket=False):
    from fira_icse_b200.packed import PackedTables, pack_from_dataset
    t = PackedTables(GoldenSplit())
    pb = pack_from_dataset(t, np.asarray(index), V)
    if bucket:                                               # more empty rows at the end of every segment
        pb = pack_from_dataset(t, np.asarray(index), V, pad_dims=(pb.Rc + 1024, pb.Rs + 512, pb.Ra + 512, pb.S + 64))
    return Layout(pb.ranges.numpy(), pb.off.numpy(), pb.mem_mask.numpy(), pb.S, pb.Rc, pb.Rs,
                  label=pb.label.numpy().copy())


@pytest.fixture(scope="module")
def layouts():
    return {"hand": hand_layout(), "nopad": hand_layout(pad=False), "real": real_layout([100, 3, 77, 127, 64, 9]),
            "real_bucket": real_layout(np.arange(40, 46), bucket=True)}


def test_layouts_are_what_the_tests_assume(layouts):
    h, r = layouts["hand"], layouts["real_bucket"]
    n = [n0 + n1 for _, n0, _, n1 in h.ranges]
    assert 0 in [n1 for *_, n1 in h.ranges] and 1 in n and max(n) + 60 <= h.S
    assert any(k > 64 for k in n)
    assert h.padding().sum() == 25 + 18 and not layouts["nopad"].padding().any()
    assert not (h.covered() & h.padding()).any() and bool((h.covered() | h.padding()).all())
    for L in (layouts["real"], r):
        assert bool((L.covered() ^ L.padding()).all())      # a real batch: every row is a commit's row or padding
    assert int(r.off[0, r.B]) < r.Rc and int(r.off[1, r.B]) < r.Rs


# ------------------------------------------------------------------------------------ copy scores
def _rnd(dtype, *shape, seed):
    return rnd16(*shape, seed=seed) if dtype else rnd32(*shape, seed=seed)


@pytest.mark.parametrize("dtype", [0, 1], ids=["fp32", "bf16"])
@pytest.mark.parametrize("kind,T", [("hand", 30), ("hand", 32), ("real", 30), ("real_bucket", 30)])
def test_copy_scores_packed(layouts, kind, T, dtype):
    """sc[b,t,s] = b_res + sum_d w_res[d] tanh(src[row(b,s)] + tgt[b,t]) over commit b's own rows, against float64 with
    autograd; skipped positions (row_mask, src_mask, s >= the commit's rows) exactly 0; d_src rows outside every range
    untouched until fira_zero_pad_rows clears the segment padding; and bit for bit the padded kernels
    fira_copy_scores_fwd / _bwd on the same rows scattered into a [B, S, 256] source (scores and d_src are fixed-order
    sums; d_tgt / d_w / d_b use atomics and are held to the float64 bounds)."""
    from fira_icse_b200 import _lib
    L = layouts[kind]
    B, S, R = L.B, L.S, L.R
    rg, off, srcm = L.dev()
    src, tgt = _rnd(dtype, R, D, seed=1), _rnd(dtype, B * T, D, seed=2)
    w, bres = rnd32(1, D, seed=3, scale=0.2), rnd32(1, seed=4)
    g = torch.Generator().manual_seed(5)
    if L.label is not None:
        rowm = torch.from_numpy(L.label >= V)                # the step's row mask: rows whose label is a copy label
    else:
        rowm = torch.rand(B, T, generator=g) > 0.5
    rowm[1] = False                                          # a commit without an active target row
    active = torch.rand(B, T, generator=g) > 0.4
    active[2] = False                                        # a commit without gradient
    rowm_u8, act_u8 = rowm.to(torch.uint8).to(DEV), active.to(torch.uint8).to(DEV)
    dsc = rnd32(B, T, S, seed=6)                             # also in inactive rows and beyond each commit's rows
    dsc[:, :, 5] = 0                                         # exact zeros inside active rows are skipped too

    sc = torch.full((B, T, S), 7.0, device=DEV)
    _lib.call("fira_copy_scores_packed_fwd", src.data_ptr(), tgt.data_ptr(), w.data_ptr(), bres.data_ptr(), rg.data_ptr(),
              srcm.data_ptr(), rowm_u8.data_ptr(), sc.data_ptr(), B, T, S, D, dtype, st())

    sd, td, wd, bd = (x.double().requires_grad_(True) for x in (src, tgt, w, bres))
    ref = torch.zeros(B, T, S, dtype=torch.float64, device=DEV)
    keep = torch.zeros(B, T, S, dtype=torch.bool)
    loss = torch.zeros((), dtype=torch.float64, device=DEV)
    for b in range(B):
        idx = L.rows(b)
        n = len(idx)
        sb = (torch.tanh(sd[idx.to(DEV)][None] + td[b * T:(b + 1) * T][:, None]) * wd.view(1, 1, D)).sum(-1) + bd
        ref[b, :, :n] = sb.detach()
        keep[b, :, :n] = rowm[b][:, None] & L.mask[b, :n][None]
        loss = loss + (sb * dsc[b, :, :n].double() * active[b].to(DEV)[:, None]).sum()
    keep = keep.to(DEV)
    assert (sc[~keep] == 0).all(), "skipped positions must be exactly 0"
    if dtype:
        close16(sc[keep], ref[keep], rel=1e-4, glob=1e-5, what="packed copy scores")
    else:
        close(sc[keep], ref[keep], rtol=1e-5, atol=1e-5)

    loss.backward()
    d_src = torch.full((R, D), SENT, device=DEV, dtype=src.dtype)
    d_tgt = torch.zeros(B * T, D, device=DEV)
    d_w, d_b = torch.zeros(1, D, device=DEV), torch.zeros(1, device=DEV)
    cov, pad = L.covered().to(DEV), L.padding().to(DEV)
    if L.label is not None:                                  # HeadFn.backward: clear the padding, then the product
        _lib.call("fira_zero_pad_rows", d_src.data_ptr(), D, D, off.data_ptr(), B, L.Rc, L.Rs, dtype, st())
    _lib.call("fira_copy_scores_packed_bwd", src.data_ptr(), tgt.data_ptr(), w.data_ptr(), dsc.data_ptr(),
              act_u8.data_ptr(), rg.data_ptr(), d_src.data_ptr(), d_tgt.data_ptr(), d_w.data_ptr(), d_b.data_ptr(),
              B, T, S, D, dtype, st())
    if L.label is None:
        assert (d_src[~cov] == SENT).all(), "rows outside every range were written"
        _lib.call("fira_zero_pad_rows", d_src.data_ptr(), D, D, off.data_ptr(), B, L.Rc, L.Rs, dtype, st())
    assert (d_src[pad] == 0).all() and (d_src[~cov & ~pad] == SENT).all()
    if dtype:
        close16(d_src[cov], sd.grad[cov], what="packed copy d_src")
        for out, r, what in ((d_tgt, td.grad, "d_tgt"), (d_w, wd.grad, "d_w"), (d_b, bd.grad, "d_b")):
            close16(out, r, rel=1e-4, glob=1e-4, what="packed copy " + what)
    else:
        close(d_src[cov], sd.grad[cov], rtol=5e-5, atol=1e-5)
        close(d_tgt, td.grad, rtol=5e-5, atol=1e-4)
        close(d_w, wd.grad, rtol=5e-5, atol=1e-4)
        close(d_b, bd.grad, rtol=5e-5, atol=1e-4)

    # the padded kernels on the same rows: commit b's rows at b*S + s, other rows filler (masked in the forward; their
    # score gradient is 0, as the mixture backward leaves it)
    srcp = _rnd(dtype, B * S, D, seed=9)
    dscp = dsc.clone()
    for b in range(B):
        idx = L.rows(b).to(DEV)
        srcp[b * S:b * S + len(idx)] = src[idx]
        dscp[b, :, len(idx):] = 0
    scp = torch.full((B, T, S), 7.0, device=DEV)
    _lib.call("fira_copy_scores_fwd", srcp.data_ptr(), tgt.data_ptr(), w.data_ptr(), bres.data_ptr(), srcm.data_ptr(),
              rowm_u8.data_ptr(), scp.data_ptr(), B, T, S, D, dtype, st())
    assert torch.equal(scp, sc), "packed scores differ from the padded kernel's"
    d_srcp = torch.full((B * S, D), SENT, device=DEV, dtype=src.dtype)
    d_tgtp = torch.zeros(B * T, D, device=DEV)
    d_wp, d_bp = torch.zeros(1, D, device=DEV), torch.zeros(1, device=DEV)
    _lib.call("fira_copy_scores_bwd", srcp.data_ptr(), tgt.data_ptr(), w.data_ptr(), dscp.data_ptr(), act_u8.data_ptr(),
              d_srcp.data_ptr(), d_tgtp.data_ptr(), d_wp.data_ptr(), d_bp.data_ptr(), B, T, S, D, dtype, st())
    for b in range(B):
        idx = L.rows(b).to(DEV)
        assert torch.equal(d_srcp[b * S:b * S + len(idx)], d_src[idx]), f"d_src of commit {b} differs from the padded kernel's"
    if dtype:
        for out, r, what in ((d_tgtp, td.grad, "d_tgt"), (d_wp, wd.grad, "d_w"), (d_bp, bd.grad, "d_b")):
            close16(out, r, rel=1e-4, glob=1e-4, what="padded copy " + what)
    else:
        close(d_tgtp, td.grad, rtol=5e-5, atol=1e-4)
        close(d_wp, wd.grad, rtol=5e-5, atol=1e-4)
        close(d_bp, bd.grad, rtol=5e-5, atol=1e-4)


def test_copy_scores_packed_argument_errors(layouts):
    """T_len above 32 and a null `ranges` are refused before anything is launched"""
    from fira_icse_b200 import _lib
    L = layouts["hand"]
    B, S, T = L.B, L.S, 33
    rg, _, srcm = L.dev()
    src, tgt = rnd32(L.R, D, seed=1), rnd32(B * T, D, seed=2)
    w, bres = rnd32(1, D, seed=3), rnd32(1, seed=4)
    sc, dsc = torch.zeros(B, T, S, device=DEV), torch.zeros(B, T, S, device=DEV)
    act = torch.ones(B * T, dtype=torch.uint8, device=DEV)
    d_src, d_tgt = torch.zeros_like(src), torch.zeros_like(tgt)
    d_w, d_b = torch.zeros(1, D, device=DEV), torch.zeros(1, device=DEV)
    for t, ranges in ((33, rg.data_ptr()), (30, None)):
        with pytest.raises(_lib.FiraLibraryError):
            _lib.call("fira_copy_scores_packed_fwd", src.data_ptr(), tgt.data_ptr(), w.data_ptr(), bres.data_ptr(), ranges,
                      srcm.data_ptr(), None, sc.data_ptr(), B, t, S, D, 0, st())
        with pytest.raises(_lib.FiraLibraryError):
            _lib.call("fira_copy_scores_packed_bwd", src.data_ptr(), tgt.data_ptr(), w.data_ptr(), dsc.data_ptr(),
                      act.data_ptr(), ranges, d_src.data_ptr(), d_tgt.data_ptr(), d_w.data_ptr(), d_b.data_ptr(),
                      B, t, S, D, 0, st())
    torch.cuda.synchronize()
    assert (sc == 0).all() and (d_src == 0).all()


# ------------------------------------------------------------------------------------ segment padding
@pytest.mark.parametrize("dtype", [0, 1], ids=["fp32", "bf16"])
@pytest.mark.parametrize("kind,ld,width", [("hand", 256, 256), ("hand", 264, 136), ("nopad", 256, 256),
                                           ("real", 3072, 3072), ("real_bucket", 256, 256), ("real_bucket", 520, 512)])
def test_zero_pad_rows(layouts, kind, ld, width, dtype):
    """rows [off[0][B], Rc) and [Rc + off[1][B], Rc + Rs) become exactly 0 in columns < width; every other element
    keeps its value (ld = 3072: the decoder's dKV, 6 layers x [K | V])"""
    from fira_icse_b200 import _lib
    L = layouts[kind]
    _, off, _ = L.dev()
    g = torch.Generator().manual_seed(3)
    x = (torch.rand(L.R, ld, generator=g) + 1.0).to(BF if dtype else torch.float32).to(DEV)     # no zero anywhere
    exp = x.clone()
    pad = L.padding().to(DEV)
    exp[pad, :width] = 0
    _lib.call("fira_zero_pad_rows", x.data_ptr(), ld, width, off.data_ptr(), L.B, L.Rc, L.Rs, dtype, st())
    assert torch.equal(x, exp)
    assert bool(pad.any()) == (kind != "nopad")


# ------------------------------------------------------------------------------------ encoder input
@pytest.mark.parametrize("dtype", [0, 1], ids=["fp32", "bf16"])
def test_embed_nodes_pos(dtype):
    """code row r = emb[sou[r]] + pe[pos[r]] for any position (one fp32 add, rounded once to bf16), sub-token and
    AST/edit rows = their embeddings at their global row of out_rest; with pos = r % n_code the padded kernel
    fira_embed_nodes_fwd bit for bit"""
    from fira_icse_b200 import _lib
    dt = BF if dtype else torch.float32
    gm = torch.Generator().manual_seed(0)
    V, VA = 500, 71
    emb, aemb, pe = rnd32(V, D, seed=1), rnd32(VA, D, seed=2), rnd32(210, D, seed=3)

    def ids(n, hi):
        return torch.randint(0, hi, (n,), generator=gm, dtype=torch.int32)

    n0, n1, n2 = 300, 104, 72                            # one ragged "graph" (B = 1) as a packed batch passes it
    sou, sub, ast, pos = ids(n0, V), ids(n1, V), ids(n2, VA), ids(n0, 210)
    pos[:4] = torch.tensor([209, 0, 209, 17], dtype=torch.int32)
    sou, sub, ast, pos = (t.to(DEV) for t in (sou, sub, ast, pos))
    xc = torch.full((n0, D), SENT, device=DEV, dtype=dt)
    rest = torch.full((n0 + n1 + n2, D), SENT, device=DEV, dtype=dt)
    _lib.call("fira_embed_nodes_pos_fwd", sou.data_ptr(), pos.data_ptr(), sub.data_ptr(), ast.data_ptr(), emb.data_ptr(),
              aemb.data_ptr(), pe.data_ptr(), xc.data_ptr(), rest.data_ptr(), 1, n0, n1, n2, D, dtype, st())
    assert torch.equal(xc, (emb[sou.long()] + pe[pos.long()]).to(dt))
    assert torch.equal(rest[n0:n0 + n1], emb[sub.long()].to(dt))
    assert torch.equal(rest[n0 + n1:], aemb[ast.long()].to(dt))
    assert (rest[:n0] == SENT).all()

    B, n0, n1, n2 = 3, 96, 40, 56
    sou, sub, ast = (t.to(DEV) for t in (ids(B * n0, V), ids(B * n1, V), ids(B * n2, VA)))
    pos = (torch.arange(B * n0, dtype=torch.int32) % n0).to(DEV)
    R = B * (n0 + n1 + n2)
    outs = []
    for with_pos in (True, False):
        xc = torch.full((B * n0, D), SENT, device=DEV, dtype=dt)
        rest = torch.full((R, D), SENT, device=DEV, dtype=dt)
        if with_pos:
            _lib.call("fira_embed_nodes_pos_fwd", sou.data_ptr(), pos.data_ptr(), sub.data_ptr(), ast.data_ptr(),
                      emb.data_ptr(), aemb.data_ptr(), pe.data_ptr(), xc.data_ptr(), rest.data_ptr(), B, n0, n1, n2, D,
                      dtype, st())
        else:
            _lib.call("fira_embed_nodes_fwd", sou.data_ptr(), sub.data_ptr(), ast.data_ptr(), emb.data_ptr(),
                      aemb.data_ptr(), pe.data_ptr(), xc.data_ptr(), rest.data_ptr(), B, n0, n1, n2, D, dtype, st())
        outs.append((xc, rest))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
