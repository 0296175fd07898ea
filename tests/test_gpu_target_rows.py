"""The training step's vocabulary projection on the vocabulary-label rows only (ops.HeadFn, want_argmax false):
fira_vocab_rows against numpy, and the compacted head against the full-row head (the argmax path, which keeps one
logits row per target row) on padded and packed golden batches.  fp32 parity mode: per-row losses and the logits of
the vocabulary rows are bit-equal, the gradients differ only by the order of their sums.  bf16 mode: fira_gemm_bf16_tc
starts each CTA's k loop at a k-block that depends on its tile (FIRA_GEMM_ROTATE), so a row moved to another tile sums
its logits in another order: they agree to one bf16 rounding."""
import copy

import numpy as np
import pytest
import torch

from fira_testlib import golden_batch, seeded_model
from test_packed import GoldenSplit, V

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _vocab_rows_np(label, V, cap):
    vslot = np.full(label.shape, -1, np.int32)
    rows = np.flatnonzero((label > 0) & (label < V))
    vslot[rows] = np.arange(len(rows))
    vrows = np.full(cap, -1, np.int32)
    vrows[:len(rows)] = rows
    return vslot, vrows


def _vocab_rows_dev(label, V, cap):
    from fira_icse_b200 import _lib
    lab = torch.as_tensor(label, dtype=torch.int32, device=DEV)
    vslot = torch.full((len(label),), 7, dtype=torch.int32, device=DEV)
    vrows = torch.full((cap,), 7, dtype=torch.int32, device=DEV)
    _lib.call("fira_vocab_rows", lab.data_ptr(), len(label), V, vslot.data_ptr(), vrows.data_ptr(), cap,
              torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return vslot.cpu().numpy(), vrows.cpu().numpy()


def _labels(B, T, rng):
    lab = np.zeros((B, T), np.int32)
    for b in range(B):
        n = int(rng.integers(0, T + 1))
        lab[b, :n] = rng.integers(1, V + 40, n)                 # vocabulary and copy labels
    lab[0, 3] = 0                                               # a zero label inside a message
    lab[1] = 0                                                  # a commit without labels
    lab[2, :12] = V + rng.integers(0, 40, 12)                   # a commit with copy labels only
    lab[2, 12:] = 0
    return lab.reshape(-1)


@pytest.mark.parametrize("B", [3, 64])
def test_vocab_rows_match_numpy(B):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    lab = _labels(B, 30, np.random.default_rng(B))
    for cap in (len(lab), max(1, int(((lab > 0) & (lab < V)).sum()))):
        got, want = _vocab_rows_dev(lab, V, cap), _vocab_rows_np(lab, V, cap)
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]), cap


def test_vocab_rows_count_at_a_bucket_edge():
    """exactly 128 vocabulary rows: every slot of a 128-row bucket used, none left over"""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from fira_icse_b200.packed import VOCAB_ROW_BUCKET
    lab = np.zeros(1920, np.int32)
    perm = np.random.default_rng(5).permutation(1920)
    lab[perm[:VOCAB_ROW_BUCKET]] = 17
    lab[perm[VOCAB_ROW_BUCKET:VOCAB_ROW_BUCKET + 40]] = V + 3
    got, want = _vocab_rows_dev(lab, V, VOCAB_ROW_BUCKET), _vocab_rows_np(lab, V, VOCAB_ROW_BUCKET)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
    assert (got[1] >= 0).all()


@pytest.fixture(scope="module")
def model():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    m = copy.deepcopy(seeded_model()).to(DEV)
    m.eval()
    return m


def _head_inputs(model, packed, index):
    """(memory, dec, mem_mask, label, pk) of TransModel.forward / forward_packed, without gradient history"""
    from fira_icse_b200.modules import _i32, _u8
    with torch.no_grad():
        model.decoder.prefetch_weights()
        if packed:
            from fira_icse_b200.packed import PackedTables, pack_from_dataset
            pb = pack_from_dataset(PackedTables(GoldenSplit()), np.asarray(index), V).to(DEV)
            memory = model.encoder.encode_memory_packed(pb)
            dec = model.decoder(pb.tar, memory, pb.mem_mask, pb.tar_mask, packed=pb)
            return memory, dec, pb.mem_mask, pb.label.reshape(-1), pb
        parts = [golden_batch(i, i + 1) for i in index]
        sou, tar, _, mark, ast_change, edge, tar_label, sub_token = [torch.cat([p[k] for p in parts], 0).to(DEV)
                                                                       for k in range(8)]
        memory = model.encoder.encode_memory(sou, mark, ast_change, edge, sub_token)
        dec = model.decoder(tar, memory, torch.cat((sou != 0, sub_token != 0), 1), tar != 0)
        label = _i32(model.shifted_label(tar_label)).reshape(-1)
        return memory, dec, _u8(torch.cat((sou != 0, sub_token != 0), 1)), label, None


def _head(model, bf16, full_rows, memory, dec, mem_mask, label, pk):
    from fira_icse_b200 import ops
    params = [model.out_fc.weight, model.out_fc.bias, *model.copy_net.flat_params()]
    for p in params:
        p.grad = None
    m = memory.detach().clone().requires_grad_()
    d = dec.detach().clone().requires_grad_()
    loss, nll, _ = ops.HeadFn.apply(full_rows, bf16, None, m, d, mem_mask, label, *params, pk)
    loss.backward()
    torch.cuda.synchronize()
    return loss.item(), nll.clone(), d.grad.clone(), m.grad.clone(), [p.grad.clone() for p in params]


@pytest.mark.parametrize("packed", [False, True])
@pytest.mark.parametrize("bf16", [False, True])
def test_head_on_vocab_rows_equals_full_rows(model, packed, bf16):
    m = copy.deepcopy(model).set_precision("bf16" if bf16 else "fp32")
    index = [100, 3, 77, 127, 64, 9, 0, 5]
    memory, dec, mem_mask, label, pk = _head_inputs(m, packed, index)
    lab = label.cpu().numpy()
    n_vocab = int(((lab > 0) & (lab < V)).sum())
    assert 0 < n_vocab < len(lab)
    if pk is not None:
        assert pk.Rv == min(-(-n_vocab // 128) * 128, len(lab))
    l_full, nll_full, dd_full, dm_full, g_full = _head(m, bf16, True, memory, dec, mem_mask, label, pk)
    l_v, nll_v, dd_v, dm_v, g_v = _head(m, bf16, False, memory, dec, mem_mask, label, pk)
    if bf16:
        assert (nll_v - nll_full).abs().max().item() <= 2e-2 and abs(l_v - l_full) <= 1e-3 * abs(l_full)
    else:
        assert torch.equal(nll_v, nll_full) and abs(l_v - l_full) <= 1e-6 * abs(l_full)
    tol = 2e-2 if bf16 else 1e-5
    # LinearRes.bias (index 5) vanishes in exact arithmetic (softmax shift invariance): its gradient is round-off noise
    for name, a, b in [("d_dec", dd_v, dd_full), ("d_memory", dm_v, dm_full)] + \
            [(f"param {i}", a, b) for i, (a, b) in enumerate(zip(g_v, g_full)) if i != 5]:
        scale = b.abs().max().item()
        assert (a.float() - b.float()).abs().max().item() <= tol * scale + 1e-9, name


@pytest.mark.parametrize("bf16", [False, True])
def test_vocab_row_logits_are_the_full_rows(model, bf16):
    """the compacted out_fc product gives each vocabulary row the full product's bits (fp32) or to one bf16 rounding"""
    from fira_icse_b200 import ops
    from fira_icse_b200._lib import FIRA_BF16, FIRA_F32
    pr = ops.Prec(bf16)
    torch.manual_seed(0)
    Mt, cap, D = 1920, 512, 256
    dec = torch.randn(Mt, D, device=DEV).to(pr.tdt)
    lab = torch.zeros(Mt, dtype=torch.int32, device=DEV)
    rows = torch.randperm(Mt, device=DEV)[:400]
    lab[rows] = torch.randint(1, V, (400,), dtype=torch.int32, device=DEV)
    W, b = model.out_fc.weight, model.out_fc.bias
    ldl = ops._ld_logits(V)
    full = pr.linear(dec, W, b, out=pr.empty((Mt, ldl), DEV), ld_out=ldl)
    vslot = torch.empty(Mt, dtype=torch.int32, device=DEV)
    vrows = torch.empty(cap, dtype=torch.int32, device=DEV)
    st = ops._stream()
    ops.call("fira_vocab_rows", lab.data_ptr(), Mt, V, vslot.data_ptr(), vrows.data_ptr(), cap, st)
    dec_v = pr.empty((cap, D), DEV)
    ops.call("fira_gather_rows", dec.data_ptr(), D, vrows.data_ptr(), dec_v.data_ptr(), D, cap, D,
             FIRA_BF16 if bf16 else FIRA_F32, st)
    part = pr.linear(dec_v, W, b, out=pr.empty((cap, ldl), DEV), ld_out=ldl)
    torch.cuda.synchronize()
    r = vrows[:400].long()
    assert torch.equal(r.sort().values, rows.sort().values)
    if bf16:
        assert torch.allclose(part[:400, :V].float(), full[r, :V].float(), rtol=2 ** -7, atol=1e-5)
    else:
        assert torch.equal(part[:400, :V], full[r, :V])
    assert (dec_v[400:] == 0).all()
