"""PackedBatch.Rv: the vocabulary-label target rows of a packed batch rounded up to one GEMM row tile, capped at B*T,
and part of the graph shape key (host only)."""
import numpy as np
import pytest

from fira_icse_b200.packed import VOCAB_ROW_BUCKET, PackedTables, pack_from_dataset
from test_packed import GoldenSplit, V


def test_packed_batch_bounds_its_vocabulary_rows():
    t = PackedTables(GoldenSplit())
    for index in ([5], [100, 3, 77, 127, 64, 9], list(range(64))):
        pb = pack_from_dataset(t, np.asarray(index), V)
        lab = pb.label.numpy()
        n = int(((lab > 0) & (lab < V)).sum())
        assert pb.Rv == min(-(-max(n, 1) // VOCAB_ROW_BUCKET) * VOCAB_ROW_BUCKET, pb.B * pb.T)
        assert n <= pb.Rv <= pb.B * pb.T
        assert pb.shape_key[-1] == pb.Rv and pb.to("cpu").Rv == pb.Rv


def test_loader_shape_budget_covers_the_vocabulary_rows():
    """PackedBatchLoader's shape policy (max_shapes) chooses Rv together with the segment rows: every emitted batch has one
    of the loader's recorded (Rc, Rs, Ra, S, Rv) shapes"""
    from fira_icse_b200.data import PackedBatchLoader
    from fira_icse_b200.synth import SynthDataset
    Vs = 24650
    ds = SynthDataset(0, 512, Vs, 71)
    free = PackedBatchLoader(ds, 64, Vs, packed=True, pin=False)
    capped = PackedBatchLoader(ds, 64, Vs, packed=True, pin=False, max_shapes=2)
    for ld in (free, capped):
        dims = set()
        for pb in ld:
            lab = pb.label.numpy()
            n = int(((lab > 0) & (lab < Vs)).sum())
            assert n <= pb.Rv <= pb.B * pb.T
            dims.add((pb.Rc, pb.Rs, pb.Ra, pb.S, pb.Rv))
        assert dims == set(ld.shapes)
    assert len({s[4] for s in free.shapes}) > 1 and len(capped.shapes) < len(free.shapes)


def test_gather_takes_a_larger_vocabulary_row_bound():
    t = PackedTables(GoldenSplit())
    index = np.arange(8)
    a = pack_from_dataset(t, index, V)
    b = pack_from_dataset(t, index, V, pad_dims=(a.Rc, a.Rs, a.Ra, a.S, a.Rv + VOCAB_ROW_BUCKET))
    assert b.Rv == min(a.Rv + VOCAB_ROW_BUCKET, a.B * a.T) and np.array_equal(a.label.numpy(), b.label.numpy())
    lab = a.label.numpy()
    if int(((lab > 0) & (lab < V)).sum()) > 0:
        with pytest.raises(ValueError):
            pack_from_dataset(t, index, V, pad_dims=(a.Rc, a.Rs, a.Ra, a.S, 0))
