"""PackedBatch.Rt: the live target rows of a packed batch (before each commit's last label) rounded up to one GEMM row
tile, at least Rv, capped at B*T, and part of the graph shape key (host only)."""
import numpy as np
import pytest

from fira_icse_b200.packed import VOCAB_ROW_BUCKET, PackedTables, pack_from_dataset, packed_needs
from test_packed import GoldenSplit, V


def _live(lab):
    nz = lab != 0
    return int(np.where(nz.any(1), lab.shape[1] - np.argmax(nz[:, ::-1], axis=1), 0).sum())


def test_packed_batch_bounds_its_live_rows():
    t = PackedTables(GoldenSplit())
    for index in ([5], [100, 3, 77, 127, 64, 9], list(range(64))):
        pb = pack_from_dataset(t, np.asarray(index), V)
        lab = pb.label.numpy()
        n = _live(lab)
        assert t.live_rows(index) == n
        assert pb.Rt == min(max(-(-max(n, 1) // VOCAB_ROW_BUCKET) * VOCAB_ROW_BUCKET, pb.Rv), pb.B * pb.T)
        assert n <= pb.Rt and pb.Rv <= pb.Rt <= pb.B * pb.T
        assert packed_needs(t, np.asarray(index), V)[4:] == (pb.Rv, pb.Rt)
        assert pb.Rt in pb.shape_key and pb.to("cpu").Rt == pb.Rt


def test_gather_takes_a_larger_live_row_bound_and_rejects_a_smaller_one():
    t = PackedTables(GoldenSplit())
    index = np.arange(40)
    a = pack_from_dataset(t, index, V)
    assert a.Rt < a.B * a.T
    b = pack_from_dataset(t, index, V, pad_dims=(a.Rc, a.Rs, a.Ra, a.S, a.Rv, a.Rt + VOCAB_ROW_BUCKET))
    assert b.Rt == min(a.Rt + VOCAB_ROW_BUCKET, a.B * a.T) and b.shape_key != a.shape_key
    c = pack_from_dataset(t, index, V, pad_dims=(a.Rc, a.Rs, a.Ra, a.S, a.Rt))     # Rt of a 5-tuple: at least Rv
    assert c.Rv == c.Rt == a.Rt
    with pytest.raises(ValueError):
        pack_from_dataset(t, index, V, pad_dims=(a.Rc, a.Rs, a.Ra, a.S, a.Rv, a.Rt - VOCAB_ROW_BUCKET))


def test_loader_shape_budget_covers_the_live_rows():
    """PackedBatchLoader's shape policy chooses Rt with the other rows: max_shapes bounds the (Rc, Rs, Ra, S, Rv, Rt)
    shapes, and every emitted batch has one of them"""
    from fira_icse_b200.data import PackedBatchLoader
    from fira_icse_b200.synth import SynthDataset
    Vs = 24650
    ds = SynthDataset(0, 512, Vs, 71)
    free = PackedBatchLoader(ds, 64, Vs, packed=True, pin=False)
    capped = PackedBatchLoader(ds, 64, Vs, packed=True, pin=False, max_shapes=2)
    for ld in (free, capped):
        dims = set()
        for pb in ld:
            assert _live(pb.label.numpy()) <= pb.Rt and pb.Rv <= pb.Rt <= pb.B * pb.T
            dims.add((pb.Rc, pb.Rs, pb.Ra, pb.S, pb.Rv, pb.Rt))
        assert dims == set(ld.dims_used)
    assert len({s[5] for s in free.dims_used}) > 1 and len(capped.dims_used) < len(free.dims_used)


def test_bench_batches_need_two_shapes():
    """the four 64-commit batches of SynthDataset(0, 256): (Rv, Rt) = (512, 640) x 3 and (384, 512)"""
    from fira_icse_b200.synth import SynthDataset
    Vs = 24650
    t = PackedTables(SynthDataset(0, 256, Vs, 71))
    got = sorted(packed_needs(t, np.arange(64 * i, 64 * (i + 1)), Vs)[4:] for i in range(4))
    assert got == [(384, 512), (512, 640), (512, 640), (512, 640)]
