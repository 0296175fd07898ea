"""n-best beam search on the GPU: fira_pointer_mix_beam_step against the float64 restatement (tests/beam_rule.py), and
fira_icse_b200.beam.nbest end to end (the reference beam goldens, the existing beam search's K beams, log-probabilities
= the training NLL, length-penalised scores, static buffers across batches)."""
import copy
import os

import numpy as np
import pytest
import torch

from beam_rule import candidates, step
from fira_testlib import GOLDEN, golden_batch, seeded_model
from sample_rule import mixture
from test_gpu_sample import _check_bookkeeping, _head_nll, _inputs, _model, _teacher_forced, _teacher_forced_nll, _vocab

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module", autouse=True)
def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


# ------------------------------------------------------------------ one step of the kernel
def _state(gen, B, K, T, pos, V, pad):
    """slot state in half pos & 1: commit 0 at its first position (slot 0 alone), commit 1 live and finished slots,
    later commits live; histories filled with distinct values"""
    R = B * K
    L = -torch.rand(R, generator=gen, dtype=torch.float64).float() * 6
    n = torch.randint(1, pos + 2, (R,), generator=gen, dtype=torch.int32)
    status = torch.zeros(R, dtype=torch.uint8)
    status[1:K] = 2
    L[0], n[0] = 0.0, 1
    if B > 1:
        status[K:2 * K:2] = 1
    seq = torch.randint(3, V, (R, T), generator=gen, dtype=torch.int32)
    raw = torch.randint(3, V, (R, T), generator=gen, dtype=torch.int32)
    tlp = -torch.rand((R, T), generator=gen)
    seq[:, pos + 1:] = pad
    raw[:, pos + 1:] = pad
    tlp[:, pos + 1:] = 0
    return L, n, status, seq, raw, tlp


def _step(logits, sc, gl, mem_mask, copy_src, K, V, alpha, state, pos, T, eos, pad=0):
    from fira_icse_b200 import ops
    from fira_icse_b200._lib import FIRA_BF16, FIRA_F32, call
    R, S = logits.shape[0], sc.shape[-1]
    L, n, status, seq, raw, tlp = state
    h = pos & 1
    i32 = dict(dtype=torch.int32, device=DEV)
    bufs = dict(seq=torch.full((2, R, T), -7, **i32), raw=torch.full((2, R, T), -7, **i32),
                tlp=torch.full((2, R, T), 9.0, device=DEV), length=torch.full((2, R), -7, **i32),
                lp=torch.full((2, R), 9.0, device=DEV), score=torch.full((2, R), 9.0, device=DEV),
                status=torch.full((2, R), 7, dtype=torch.uint8, device=DEV))
    bufs["seq"][h], bufs["raw"][h], bufs["tlp"][h] = seq.to(DEV), raw.to(DEV), tlp.to(DEV)
    bufs["length"][h], bufs["lp"][h], bufs["status"][h] = n.to(DEV), L.to(DEV), status.to(DEV)
    bufs["score"][h] = (L / torch.pow((5.0 + (n - 1).float()) / 6.0, alpha)).to(DEV)
    parent = torch.full((R,), -1, dtype=torch.int64, device=DEV)
    nxt = torch.full((R,), -1, **i32)
    work = torch.zeros(R * K, dtype=torch.int64, device=DEV)
    P = ops._ptr
    call("fira_pointer_mix_beam_step", P(logits), logits.stride(0), P(sc), P(gl), P(mem_mask), P(copy_src), float(alpha),
         eos, pad, P(work), P(bufs["seq"]), P(bufs["raw"]), P(bufs["tlp"]), P(bufs["length"]), P(bufs["lp"]),
         P(bufs["score"]), P(bufs["status"]), P(parent), P(nxt), T, pos, R // K, K, V, S,
         FIRA_BF16 if logits.dtype == torch.bfloat16 else FIRA_F32, ops._stream())
    torch.cuda.synchronize()
    out = {k: v[1 - h].cpu() for k, v in bufs.items()}
    out["score_in"] = bufs["score"][h].cpu()
    return out, parent.cpu(), nxt.cpu()


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("V,S", [(24650, 370), (61, 13)])
def test_kernel_step_matches_float64_rule(dtype, V, S):
    gen = torch.Generator().manual_seed(V + S + (dtype == torch.bfloat16))
    B, T, pos, pad = 3, 8, 3, 0
    C = V + S
    compared = near = 0
    for K in (1, 3, 5, 8, 16):
        R = B * K
        logits, sc, gl, mem_mask, copy_src = _inputs(gen, B, K, V, S, dtype)   # planted ties, masked copies at 40.0
        if K > 1:                                     # exact ties across rows: slots 0 and 1 of the last commit
            logits[(B - 1) * K + 1] = logits[(B - 1) * K]
            sc[B - 1, 1] = sc[B - 1, 0]
            gl[(B - 1) * K + 1] = gl[(B - 1) * K]
        x = logits.float().cpu().numpy()[:, :V].astype(np.float64)
        scn, gln, mk = sc.cpu().numpy().reshape(R, S), gl.cpu().numpy(), mem_mask.cpu().numpy()
        Pm = np.stack([mixture(x[r], scn[r], gln[r], mk[r // K]) for r in range(R)])
        eos = 3                                       # a planted top token: some slots finish
        for alpha in (0.0, 0.6, 1.5):
            state = _state(gen, B, K, T, pos, V, pad)
            L, n, status, seq, raw, tlp = state
            if K > 1:
                L[(B - 1) * K + 1] = L[(B - 1) * K]
                n[(B - 1) * K + 1] = n[(B - 1) * K]
            out, parent, nxt = _step(logits, sc, gl, mem_mask, copy_src, K, V, alpha, state, pos, T, eos, pad)
            Ld, nd = L.double().numpy(), (n - 1).double().numpy()         # n: generated tokens = length - 1
            for b in range(B):
                rows = slice(b * K, (b + 1) * K)
                st = status[rows].numpy()
                ref, gap = step(Ld[rows], nd[rows], st, Pm[rows], mk[b], V, K, alpha)
                table = {(c[2], c[3]): c[0] for c in candidates(Ld[rows], nd[rows], st, Pm[rows], mk[b], V, K, alpha)}
                for k in range(K):
                    r = b * K + k
                    i = int(parent[r]) - b * K
                    assert 0 <= i < K
                    carried = st[i] == 1                      # a finished slot only ever proposes itself
                    j = C if carried else int(out["raw"][r, pos + 1])
                    assert (i, j) in table, (b, k, i, j)
                    if (i, j) != ref[k][:2]:                  # only across a float64 near-tie of fp32 rounding size
                        near += 1
                        d = abs(table[(i, j)] - ref[k][4]) / max(1e-30, abs(ref[k][4]))
                        assert d <= 1e-6, (dtype, V, K, alpha, b, k, (i, j), ref[k][:2], d)
                    compared += 1
                    p = b * K + i
                    # histories follow the parent; a grown slot has its new token at pos + 1
                    assert torch.equal(out["seq"][r, :pos + 1], seq[p, :pos + 1])
                    assert torch.equal(out["raw"][r, :pos + 1], raw[p, :pos + 1])
                    assert torch.equal(out["tlp"][r, :pos + 1], tlp[p, :pos + 1])
                    assert (out["seq"][r, pos + 2:] == pad).all() and (out["tlp"][r, pos + 2:] == 0).all()
                    if carried:
                        assert out["status"][r] == 1 and out["lp"][r] == L[p] and nxt[r] == pad
                        assert out["seq"][r, pos + 1] == pad and out["score"][r] == out["score_in"][p]
                        continue
                    tok = j if j < V else int(copy_src[b, j - V])
                    assert j < V or mk[b, j - V], "masked copy position selected"
                    assert out["seq"][r, pos + 1] == tok and nxt[r] == tok
                    assert out["length"][r] == n[p] + 1 and out["status"][r] == int(tok == eos)
                    lp = out["tlp"][r, pos + 1]
                    assert out["lp"][r] == torch.tensor(L[p].item(), dtype=torch.float32) + lp      # one fp32 add
                    want = out["lp"][r].double() / ((5.0 + n[p].double()) / 6.0) ** alpha
                    assert abs(out["score"][r].double() - want) <= 1e-6 * abs(want) + 1e-12
                scores = out["score"][b * K:(b + 1) * K]
                assert (scores[1:] <= scores[:-1]).all()
            # every selected lp is -nll of fira_pointer_mix_nll_fwd for that label on the parent's row
            grown = out["status"] != 1
            grown |= out["seq"][:, pos + 1] != pad
            par = parent.to(DEV)
            lab = torch.where(grown, out["raw"][:, pos + 1], torch.zeros_like(out["raw"][:, pos + 1]))
            nll = _head_nll(logits[par].contiguous(), sc.view(R, S)[par].view(B, K, S).contiguous(), gl[par].contiguous(),
                            mem_mask, lab.numpy(), K, V)
            live = lab.numpy() != 0
            np.testing.assert_allclose(out["tlp"][:, pos + 1].numpy()[live], -nll[live], rtol=1e-6, atol=0)
    assert near <= 0.02 * compared, (near, compared)


# ------------------------------------------------------------------ end to end
def _nbest(m, b, **kw):
    from fira_icse_b200.beam import nbest
    v = _vocab()
    return nbest(m, b[0], b[3], b[4], b[5].to(DEV), b[7], start_id=v["<start>"], eos_id=v["<eos>"], pad_id=v["<pad>"],
                 **kw)


def _beam(m, b, K):
    from fira_icse_b200.beam import beam_search
    v = _vocab()
    return beam_search(m, b[0], b[3], b[4], b[5].to(DEV), b[7], beam_size=K, tar_len=30, start_id=v["<start>"],
                       eos_id=v["<eos>"], pad_id=v["<pad>"], mode="graph")


def _check(out, v):
    _check_bookkeeping(out, v)
    last = out.seq.gather(2, (out.length - 1).unsqueeze(-1)).squeeze(-1)
    assert torch.equal(out.finished, last == v["<eos>"])
    assert torch.isfinite(out.score).all() and (out.score[:, 1:] <= out.score[:, :-1]).all()


@pytest.mark.parametrize("golden", ["beam_first16.npz", "beam5_first16.npz"])
def test_alpha0_best_hypothesis_matches_reference_beam_goldens(golden):
    gold = np.load(os.path.join(GOLDEN, golden))
    m = _model("fp32")
    bs = int(gold["batch"])
    for lo in range(0, gold["beam_ids"].shape[0], bs):
        b = golden_batch(lo, lo + bs)
        out = _nbest(m, b, beam_size=int(gold["beam"]))
        _check(out, _vocab())
        for i in range(bs):
            ref = gold["beam_ids"][lo + i]
            ref = ref[ref >= 0]
            mine = out.seq[i, 0, :out.length[i, 0]].cpu().numpy()
            assert np.array_equal(mine, ref), (lo + i, mine, ref)


@pytest.mark.parametrize("K", [3, 5])
def test_k_list_equals_beam_search(K):
    m = _model("fp32")
    b = golden_batch(0, 16)
    out = _nbest(m, b, beam_size=K)
    seq, length, prob = _beam(m, b, K)
    assert torch.equal(out.length, length)
    for i in range(seq.shape[0]):
        for k in range(K):
            assert torch.equal(out.seq[i, k, :length[i, k]], seq[i, k, :length[i, k]]), (i, k)
    torch.testing.assert_close(out.logprob, torch.log(prob), rtol=0, atol=1e-4)


def _tf_logprob_check(m, b, out, precision):
    rep = _teacher_forced(m, b, out)
    with torch.no_grad():
        nll = _teacher_forced_nll(m, rep, m.shifted_label(rep[6]).to(torch.int32).view(-1))
    got = -out.token_logprob.view(-1, out.seq.shape[2])[:, 1:].cpu()
    ref = nll[:, :-1].cpu()
    live = rep[6][:, 1:].cpu() != 0
    if precision == "fp32":
        torch.testing.assert_close(got[live], ref[live], rtol=1e-4, atol=1e-6)
    else:
        d = (got[live] - ref[live]).abs()                 # incremental vs full bf16 decoder (test_gpu_sample.py)
        assert d.median().item() <= 5e-2 and d.max().item() <= 0.5


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_token_logprob_is_the_teacher_forced_nll_on_the_sharpened_model(precision):
    m = _model(precision)
    b = golden_batch(8, 16)
    out = _nbest(m, b, beam_size=3)
    _check(out, _vocab())
    _tf_logprob_check(m, b, out, precision)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_unscaled_model_where_probability_products_underflow(precision):
    m = copy.deepcopy(seeded_model()).to(DEV).eval().set_precision(precision)
    b = golden_batch(0, 8)
    out = _nbest(m, b, beam_size=3)
    _check(out, _vocab())
    if precision == "fp32":
        _, _, prob = _beam(m, b, 3)
        assert (prob == 0).any()                          # the reference's product ranking has lost these commits
        assert (out.logprob < -104).any()                 # log of the smallest fp32 subnormal is about -103.3
    _tf_logprob_check(m, b, out, precision)


@pytest.mark.parametrize("alpha", [0.6, 1.5])
def test_length_penalised_scores(alpha):
    m = _model("fp32")
    b = golden_batch(0, 16)
    out = _nbest(m, b, beam_size=5, length_penalty=alpha)
    _check(out, _vocab())
    want = out.logprob.double() / ((5.0 + (out.length - 1).double()) / 6.0) ** alpha
    torch.testing.assert_close(out.score.double(), want, rtol=1e-6, atol=0)


def test_static_buffers_are_reset_between_batches():
    m = _model("fp32")
    a, b = golden_batch(0, 8), golden_batch(8, 16)
    first = _nbest(m, a, beam_size=3)
    other = _nbest(m, b, beam_size=3)
    again = _nbest(m, a, beam_size=3)
    assert not torch.equal(first.seq, other.seq)
    assert torch.equal(first.seq, again.seq) and torch.equal(first.raw, again.raw)
    torch.testing.assert_close(first.logprob, again.logprob, rtol=0, atol=1e-4)
