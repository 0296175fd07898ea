"""Nearest-neighbour decoding on the GPU: fira_knn_search and fira_pointer_mix_knn against the float64 rule
(tests/knn_rule.py), a one-word datastore end to end, retrieval of a datastore's own entries, every decoder with a
KNNModel, graph reuse and run-time lam / tau, and `run_model.py datastore` + `test` with FIRA_KNN."""
import json
import math
import os

import numpy as np
import pytest
import torch

from fira_testlib import golden_batch, reference_args
from knn_rule import mix, neighbour_q
from test_gpu_cli import _run_model, _test_lines, trained  # noqa: F401  (the trained-model fixture)
from test_gpu_sample import _head_nll, _inputs, _model, _sample, _vocab
from test_gpu_prefix import _score

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module", autouse=True)
def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


@pytest.fixture(autouse=True)
def _drop_new_loops():
    """the decoding-loop cache keeps every model's loops and graphs until the process ends: drop this test's"""
    from fira_icse_b200 import decode_loop
    before = {id(m) for m in decode_loop._LOOPS.keys()}
    yield
    for m in [m for m in decode_loop._LOOPS.keys() if id(m) not in before]:
        del decode_loop._LOOPS[m]
    torch.cuda.empty_cache()


def _store(keys, words=None, V=100):
    from fira_icse_b200.knn import Datastore
    N = keys.shape[0]
    kb = keys.to(torch.bfloat16).contiguous()
    words = torch.zeros(N, dtype=torch.int32, device=DEV) if words is None else words
    return Datastore(kb, kb.float().square().sum(1), words, torch.zeros((N, 2), dtype=torch.int32, device=DEV),
                     vocab_size=V, precision="fp32", fingerprint="test")


def _reference(q, keys, m):
    """float64 (d [R, N] top-m smallest, as (idx, d) sorted by (d, i)) and |q|, over bf16-rounded operands, on the GPU"""
    qd, kd = q.to(torch.bfloat16).double(), keys.to(torch.bfloat16).double()
    kn = kd.square().sum(1)
    out_i, out_d = [], []
    for r0 in range(0, qd.shape[0], 128):
        qq = qd[r0:r0 + 128]
        d = qq.square().sum(1, keepdim=True) + kn[None, :] - 2.0 * qq @ kd.T
        v, i = torch.topk(d, m, dim=1, largest=False)
        out_i.append(i.cpu().numpy()); out_d.append(v.cpu().numpy())
    idx, d = np.concatenate(out_i), np.concatenate(out_d)
    order = np.lexsort((idx, d), axis=1)
    return np.take_along_axis(idx, order, 1), np.take_along_axis(d, order, 1), qd.norm(dim=1).cpu().numpy()


def _tol(qnorm, kmax):
    """|fp32 d - float64 d|: 256 exact bf16 products summed in fp32, |q|^2, the norm and the fma, each within
    ~264 ulp of (|q| + |key|)^2"""
    return 264 * 2.0 ** -24 * (qnorm + kmax) ** 2


def _check_search(q, keys, k, idx, dist):
    N = keys.shape[0]
    m = min(N, k + 32)
    ridx, rd, qn = _reference(q, keys, m)
    kmax = float(keys.to(torch.bfloat16).double().norm(dim=1).max())
    kd = keys.to(torch.bfloat16).double()
    qd = q.to(torch.bfloat16).double()
    idx, dist = idx.cpu().numpy(), dist.cpu().numpy()
    for r in range(q.shape[0]):
        tol = _tol(qn[r], kmax)
        own = (qd[r] - kd[torch.from_numpy(idx[r]).to(DEV)]).square().sum(1).cpu().numpy()    # float64 d of the ids
        assert np.all(np.abs(dist[r] - own) <= tol + 1e-6 * np.abs(own)), (r, dist[r], own, tol)
        assert len(set(idx[r].tolist())) == k
        kth = rd[r, k - 1]
        assert np.all(own <= kth + 2 * tol), r                             # a valid k-nearest set under the bound
        must = set(ridx[r][rd[r] < kth - 2 * tol].tolist())
        assert must <= set(idx[r].tolist()), r
        for j in range(k):                                                 # exact ids outside near-ties
            lo = rd[r, j - 1] if j else -np.inf
            hi = rd[r, j + 1] if j + 1 < m else np.inf
            if rd[r, j] - lo > 2 * tol and hi - rd[r, j] > 2 * tol:
                assert idx[r, j] == ridx[r, j], (r, j)


def _search_case(N, R, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    keys = torch.randn((N, 256), generator=g, device=DEV)
    src = torch.randint(0, N, (R,), generator=g, device=DEV)
    q = keys[src] + 0.3 * torch.randn((R, 256), generator=g, device=DEV)
    q[0] = keys[N // 2]                                                    # a planted exact copy: d ~ 0
    if N >= 16:
        keys[7] = keys[3]                                                  # duplicate keys: the tie goes to index 3
        keys[N - 1] = keys[3]
        if R > 1:
            q[1] = keys[3] + 0.01 * torch.randn(256, generator=g, device=DEV)
    return keys, q, src


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("k", [1, 8, 64])
@pytest.mark.parametrize("R", [1, 3, 384, 2048])
@pytest.mark.parametrize("N", ["k", 1000, 2 ** 20 + 37])
def test_search_matches_float64(N, R, k, dtype):
    from fira_icse_b200.knn import search
    N = k if N == "k" else N
    keys, q, _ = _search_case(N, R, seed=N + R + k)
    store = _store(keys)
    idx, dist = search(store, q.to(dtype), k)
    _check_search(q, keys, k, idx, dist)
    i0 = idx[0].tolist()
    assert i0[0] == N // 2 or torch.equal(store.keys[i0[0]], store.keys[N // 2]), i0
    assert abs(float(dist[0, 0])) <= _tol(float(q[0].norm()), float(keys.norm(dim=1).max()))
    if N >= 16 and R > 1 and k >= 3:
        i1 = idx[1].tolist()
        assert i1[:3] == [3, 7, N - 1], i1                                  # bit-identical d: index order
        assert dist[1, 0] == dist[1, 1] == dist[1, 2]
    if R == 384:                                                           # row independence: bit for bit
        for r in (0, 1, 200, 383):
            i1, d1 = search(store, q[r:r + 1].to(dtype), k)
            assert torch.equal(i1[0], idx[r]) and torch.equal(d1[0], dist[r]), r
        i2, d2 = search(store, q.flip(0).to(dtype), k)
        assert torch.equal(i2.flip(0), idx) and torch.equal(d2.flip(0), dist)


def test_search_repeats_bit_for_bit():
    from fira_icse_b200.knn import search
    keys, q, _ = _search_case(50_000, 700, seed=5)
    store = _store(keys)
    a = search(store, q, 64)
    b = search(store, q, 64)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


# ------------------------------------------------------------------ the combine

def _combine(logits, sc, gl, mem_mask, idx, dist, words, k, lam, tau, N, V):
    from fira_icse_b200 import ops
    from fira_icse_b200._lib import FIRA_BF16, FIRA_F32, call
    R, S = logits.shape[0], sc.shape[-1]
    B = R // N
    ld = ops._ld_logits(V)
    out = torch.full((R, ld), float("nan"), dtype=torch.float32, device=DEV)
    sco = torch.empty((B, N, S), dtype=torch.float32, device=DEV)
    glo = torch.empty((R, 2), dtype=torch.float32, device=DEV)
    params = torch.tensor([lam, tau], dtype=torch.float32, device=DEV)
    p = ops._ptr
    call("fira_pointer_mix_knn", p(logits), logits.stride(0), p(sc), p(gl), p(mem_mask), p(idx), p(dist), p(words), k,
         p(params), p(out), ld, p(sco), p(glo), B, N, V, S,
         FIRA_BF16 if logits.dtype == torch.bfloat16 else FIRA_F32, ops._stream())
    torch.cuda.synchronize()
    return out, sco, glo


def _mixture64(x, c, gl, mask, V):
    """float64 P [R, V + S] of a triple, with the masked copy positions at -1e9 (Model.py:54-86)"""
    x = x[:, :V].double()
    c = c.reshape(x.shape[0], -1).double()
    c = torch.where(mask.bool(), c, torch.full_like(c, -1e9))
    g = torch.softmax(gl.double(), 1)
    return torch.cat((g[:, :1] * torch.softmax(x, 1), g[:, 1:] * torch.softmax(c, 1)), 1)


# relative to max(1, |log P'|): x' is rounded once to fp32 and the step kernels' softmax of it adds its own fp32 rounding.
# Measured on an H100 over every case below: at most 3.5e-7; the bound keeps a 5x margin.
LOG_TOL = 2e-6


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("V,S", [(24650, 370), (40, 9)])
def test_combine_matches_float64(dtype, V, S):
    B, N, k = 6, 2, 16
    gen = torch.Generator().manual_seed(V + S)
    logits, sc, gl, mem_mask, _ = _inputs(gen, B, N, V, S, dtype)
    R = B * N
    gl[1] = torch.tensor([-200.0, 0.0], device=DEV)                        # g0 = 0 in fp32
    gl[2] = torch.tensor([0.0, -200.0], device=DEV)                        # g1 = 0 in fp32
    Nst = 500
    words = torch.randint(0, V, (Nst,), generator=gen).to(torch.int32).to(DEV)
    idx = torch.stack([torch.randperm(Nst, generator=gen)[:k] for _ in range(R)]).to(torch.int32).to(DEV)
    dist = torch.sort(torch.rand((R, k), generator=gen) * 50, 1).values.to(DEV)
    idx[3] = idx[3, 0]                                                      # every neighbour the same entry
    idx[4, : k // 2] = idx[4, 0]                                            # repeated words
    wm = words.clone()
    wm[idx[5].long()] = 7 % V                                               # all neighbours on one word
    mm = mem_mask
    ref_rows = []
    for lam, tau in ((0.25, 10.0), (0.9, 1e-3), (0.01, 1e6)):              # extreme tau
        for wv in (words, wm):
            out, sco, glo = _combine(logits, sc, gl, mm, idx, dist, wv, k, lam, tau, N, V)
            assert bool(torch.isfinite(out[:, :V]).all())                  # P' = 0 is -1e9, never -inf
            P = _mixture64(logits.float(), sc, gl, mm.repeat_interleave(N, 0), V).cpu().numpy()
            Pn = _mixture64(out, sco, glo, mm.repeat_interleave(N, 0), V).cpu().numpy()
            for r in range(R):
                q = neighbour_q(wv.cpu().numpy()[idx[r].cpu().numpy()], dist[r].cpu().double().numpy(), tau, V)
                Pr = mix(P[r], q, lam, V)
                live = Pr > 1e-30
                assert np.all(Pn[r][~live] < 1e-30)
                lp, lr = np.log(Pn[r][live]), np.log(Pr[live])
                err = np.max(np.abs(lp - lr) / np.maximum(1.0, np.abs(lr)))
                ref_rows.append(err)
                assert err <= LOG_TOL, (lam, tau, r, err)
            # the NLL kernel on the output reads -log P'
            lab = np.array([1 + (r * 131) % (V + S - 1) for r in range(R)])           # label 0 carries no loss
            rows_mask = mm.repeat_interleave(N, 0).cpu().numpy()
            lab = np.where((lab < V) | (rows_mask[np.arange(R), np.clip(lab - V, 0, S - 1)] != 0), lab, 3)
            nll = _head_nll(out, sco, glo, mm, lab, N, V)
            want = -np.log(np.clip(Pn[np.arange(R), lab], 1e-10, 1.0))
            assert np.allclose(nll, want, rtol=2e-6, atol=2e-6), (nll, want)
    print(f"[knn combine] max relative error of log P' = {max(ref_rows):.3g}")


# ------------------------------------------------------------------ end to end

def _datastore(m, lo=0, hi=16):
    from fira_icse_b200.knn import build_datastore
    v = _vocab()
    return build_datastore(m, [golden_batch(lo, hi)], first_index=lo, start_id=v["<start>"], eos_id=v["<eos>"],
                           pad_id=v["<pad>"], unk_id=v["<unkm>"])


# bf16: the decoder's split-K products add fp32 partials atomically in no fixed order, so two runs of the same bf16
# model differ (test_gpu_ensemble.py; measured on an H100 here too: up to ~0.2 in a token's log-probability).  The kNN
# score and the plain score it is compared with are separate runs, so bf16 uses the bound of the other bf16 decoding
# tests: median <= 5e-2, max <= 0.5.  log((1 - lam) e^lp + lam [w]) is 1-Lipschitz in lp, so the bound carries over.
BF16_MEDIAN, BF16_MAX = 5e-2, 0.5


def _one_word(m, ds, b):
    """the commits' most frequent word w and a datastore over ds's keys whose every entry carries w"""
    from fira_icse_b200.knn import Datastore
    lab = b[6][:, :30].to(DEV)
    v = _vocab()
    body = lab[:, 1:][(lab[:, 1:] < m.vocab_size) & (lab[:, 1:] != v["<pad>"]) & (lab[:, 1:] != v["<eos>"])]
    w = int(torch.mode(body).values)
    return w, Datastore(ds.keys, ds.norms, torch.full_like(ds.words, w), ds.source, vocab_size=ds.vocab_size,
                        precision=ds.precision, fingerprint=ds.fingerprint)


def _check_one_word(knn, plain, b, w, lam, precision):
    """score with a one-word datastore: log((1 - lam) e^lp + lam [label == w]) per token, lp the plain model's"""
    lab = b[6][:, :30].to(DEV)
    T = plain.token_logprob.shape[1]
    hit = lab[:, :T] == w
    pos = torch.arange(T, device=DEV)[None, :]
    tok = (pos >= 1) & (pos < knn.length[:, None])
    lk = knn.token_logprob.double()
    assert (hit & tok).sum() >= 3
    assert bool((lk[hit & tok] >= math.log(lam) - 1e-5).all())           # P' >= lam on w, <= 1 - lam elsewhere
    assert bool((lk[~hit & tok] <= math.log(1 - lam) + 1e-5).all())
    lp = plain.token_logprob.double()
    want = torch.log(torch.clamp((1 - lam) * torch.exp(lp) + lam * hit.double(), 1e-10, 1.0))
    live = tok & (lp > -22.0)
    assert live.sum() > 10
    err = (lk - want).abs()[live]
    if precision == "fp32":
        assert float(err.max()) <= 1e-4, float(err.max())
    else:
        assert err.median().item() <= BF16_MEDIAN and err.max().item() <= BF16_MAX, err.max()


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_one_word_datastore_score(precision):
    """every entry carries word w, so q is one-hot on w whatever the search returns"""
    from fira_icse_b200.knn import KNNModel
    m = _model(precision)
    ds = _datastore(m)
    b = golden_batch(0, 16)
    w, one = _one_word(m, ds, b)
    plain = _score(m, b)
    lam = 0.3
    knn = _score(KNNModel(m, one, k=8, temperature=5.0, lam=lam), b)
    _check_one_word(knn, plain, b, w, lam, "fp32" if precision == "fp32" else "bf16")


def test_loops_follow_the_datastore_over_shared_keys():
    """two datastores over one keys tensor (and norms) with other words get their own loops: decoding with the first
    and then with the second follows the second's words; drop_loops releases one datastore's loops or all of them"""
    from fira_icse_b200 import decode_loop
    from fira_icse_b200.knn import KNNModel
    m = _model("fp32")
    ds = _datastore(m)
    b = golden_batch(0, 16)
    w, one = _one_word(m, ds, b)
    assert one.keys is ds.keys and one.norms is ds.norms
    lam = 0.3
    plain = _score(m, b)
    _score(KNNModel(m, ds, k=8, temperature=5.0, lam=lam), b)
    knn = _score(KNNModel(m, one, k=8, temperature=5.0, lam=lam), b)
    _check_one_word(knn, plain, b, w, lam, "fp32")
    loops = decode_loop._LOOPS[m]
    stores = {e[2].store for e in loops.values() if getattr(e[2], "knn", False)}
    assert stores == {ds, one}
    decode_loop.drop_loops(KNNModel(m, one, k=8))
    assert {e[2].store for e in loops.values() if getattr(e[2], "knn", False)} == {ds}
    decode_loop.drop_loops(m)
    assert m not in decode_loop._LOOPS


def test_retrieval_of_own_entries(trained):  # noqa: F811
    from fira_icse_b200 import TransModel
    from fira_icse_b200.knn import KNNModel, build_datastore, search
    d = trained[0]
    vocab = json.load(open(d / "DataSet" / "word_vocab.json"))
    ast = json.load(open(d / "DataSet" / "ast_change_vocab.json"))
    m = TransModel(reference_args(len(vocab), len(ast)))
    m.load_state_dict(torch.load(d / "best_model.pt", map_location="cpu"))
    m = m.to(DEV).eval()
    ids = dict(start_id=vocab["<start>"], eos_id=vocab["<eos>"], pad_id=vocab["<pad>"], unk_id=vocab["<unkm>"])
    ds = build_datastore(m, [golden_batch(lo, lo + 32) for lo in range(0, 128, 32)], first_index=0, **ids)
    idx, dist = search(ds, ds.keys, 2)
    first = idx[:, 0].cpu()
    ar = torch.arange(ds.N)
    same = first == ar
    keys = ds.keys.cpu()
    eq = (~same) & (first < ar) & (keys[first] == keys[ar]).all(1)
    assert bool((same | eq).all())
    # k = 1, lam close to 1, small tau: a commit's own reference gets at least log lam wherever its own entry is the
    # nearest by a margin (the nearest key with another word is far)
    lam = 0.98
    kw = KNNModel(m, ds, k=1, temperature=0.01, lam=lam)
    kd = ds.keys.double()
    full = kd.square().sum(1)[:, None] + kd.square().sum(1)[None, :] - 2 * kd @ kd.T
    other = torch.where(ds.words[:, None] != ds.words[None, :], full, torch.full_like(full, float("inf")))
    margin = other.min(1).values / kd.square().sum(1).clamp(min=1e-6)
    good = (margin > 0.05).cpu()
    src = ds.source.cpu()
    b = golden_batch(0, 32)
    from fira_icse_b200.sample import score
    s = score(kw, b[0], b[3], b[4], b[5].to(DEV), b[7], b[6], start_id=ids["start_id"], eos_id=ids["eos_id"],
              pad_id=ids["pad_id"])
    tlp = s.token_logprob.cpu()
    lab = b[6]
    checked = 0
    for e in range(ds.N):
        cb, t = int(src[e, 0]), int(src[e, 1])
        if cb >= 32 or not good[e] or t + 1 >= tlp.shape[1] or int(lab[cb, t + 1]) >= ds.vocab_size:
            continue
        assert float(tlp[cb, t + 1]) >= math.log(lam) - 1e-4, (e, cb, t, float(tlp[cb, t + 1]))
        checked += 1
    assert checked > 50, checked


def _ids():
    v = _vocab()
    return dict(start_id=v["<start>"], eos_id=v["<eos>"], pad_id=v["<pad>"])


def test_decoders_with_knn_model():
    from fira_icse_b200 import decode_loop
    from fira_icse_b200.beam import nbest
    from fira_icse_b200.knn import KNNModel
    from fira_icse_b200.mbr import mbr
    m = _model("fp32")
    b = golden_batch(0, 16)
    plain_before = _sample(m, b, num_samples=2, seed=4)
    ds = _datastore(m)
    km = KNNModel(m, ds, k=8)
    s = _sample(km, b, num_samples=3, seed=1, top_p=0.9, no_repeat_ngram=2, min_length=2)
    assert (s.length >= 2).all()
    # a sample's score equals its logprob (the finished samples: score needs <eos>)
    done = (s.raw[:, 0] == _ids()["eos_id"]).any(1).cpu()
    assert done.sum() >= 4
    bb = [x[done] if torch.is_tensor(x) else x for x in b]
    bb[6] = s.raw[:, 0].cpu()[done]
    sc = _score(km, bb)
    # the score runs its own loop (one sample per commit): fp32 rounding differs in the last bits, summed over 30 tokens
    assert torch.allclose(sc.logprob, s.logprob[done.to(DEV), 0], rtol=1e-4, atol=5e-3), (sc.logprob, s.logprob)
    g = b[0], b[3], b[4], b[5].to(DEV), b[7]
    h = nbest(km, *g, beam_size=4, groups=2, diversity=0.5, **_ids())
    assert h.seq.shape[:2] == (16, 4)
    con = torch.zeros((16, 1, 1), dtype=torch.long)
    con[:, 0, 0] = 25
    h = nbest(km, *g, beam_size=3, constraints=con, **_ids())
    assert h.seq.shape[:2] == (16, 3)
    pre = torch.zeros((16, 2), dtype=torch.long)
    pre[:, 0] = 25
    mb = mbr(km, *g, num_samples=4, prefix=pre, **_ids())
    assert (mb.seq[:, 1] == 25).all()
    # a second batch of the same shape replays the position graphs, and new lam / tau take effect without recapture:
    # every loop and every captured graph is still the same object afterwards
    _score(KNNModel(m, ds, k=8, lam=0.25), b)                               # the B = 16 score loop, captured
    loop = decode_loop._LOOPS[m]
    snap = {key: (e[2], dict(e[2].graphs)) for key, e in loop.items()}
    assert any(getattr(lp, "knn", False) and lp.N == 1 for lp, _ in snap.values())      # score's loop is captured
    b2 = golden_batch(16, 32)
    _sample(km, b2, num_samples=3, seed=1, top_p=0.9, no_repeat_ngram=2, min_length=2)
    a = _score(KNNModel(m, ds, k=8, lam=0.25), b2)
    c = _score(KNNModel(m, ds, k=8, lam=0.6, temperature=2.0), b2)
    assert not torch.equal(a.token_logprob, c.token_logprob)
    a2 = _score(KNNModel(m, ds, k=8, lam=0.25), b2)
    # the fp32 decoder's own replays of one batch agree to ~1e-5 per token (measured on an H100), not bit for bit
    assert torch.allclose(a.token_logprob, a2.token_logprob, rtol=0.0, atol=1e-4)
    for key, (lp, graphs) in snap.items():
        assert loop[key][2] is lp, key
        for gk, g in graphs.items():
            assert lp.graphs[gk] is g, (key, gk)
    # a plain model's outputs are unchanged by the kNN loops in the same process
    plain_after = _sample(m, b, num_samples=2, seed=4)
    assert torch.equal(plain_before.seq, plain_after.seq)
    assert torch.allclose(plain_before.token_logprob, plain_after.token_logprob, rtol=0.0, atol=1e-4)


def test_refusals_on_gpu():
    from fira_icse_b200.beam import beam_search
    from fira_icse_b200.knn import KNNModel
    m = _model("fp32")
    km = KNNModel(m, _datastore(m), k=4)
    b = golden_batch(0, 4)
    with pytest.raises(TypeError, match="KNNModel"):
        beam_search(km, b[0], b[3], b[4], b[5].to(DEV), b[7], beam_size=3, **_ids())
    m2 = _model("fp32")
    with torch.no_grad():
        m2.out_fc.bias += 1.0
    with pytest.raises(ValueError, match="fingerprint"):
        KNNModel(m2, km.datastore)


def test_run_model_datastore_then_test(trained):  # noqa: F811
    d, base, _ = trained
    r = _run_model("datastore", d, base)
    assert "datastore:" in r.stdout and os.path.isfile(d / "datastore.pt")
    n_test, lines = _test_lines(trained, "output_fira_samples_knn4", FIRA_DECODE="sample", FIRA_SAMPLES="2",
                                FIRA_KNN="datastore.pt", FIRA_KNN_K="4")
    assert len(lines) == 2 * n_test + 1 and lines[-1] == ""
    n_test, lines = _test_lines(trained, "output_fira_nbest_knn8", FIRA_DECODE="nbest", FIRA_KNN="datastore.pt")
    assert len(lines) == 3 * n_test + 1
