"""Prefix-constrained decoding on the GPU: the three `_prefix` step entry points against their twins and against
fira_pointer_mix_nll_fwd on random inputs, and `prefix=` / sample.score end to end on the sharpened golden model
(teacher-forced NLL, self-consistency, reference prefixes, no prefix), and `run_model.py test` with FIRA_PREFIX_WORDS."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from fira_testlib import ROOT, golden_batch, load_raw_golden
from test_gpu_cli import _run_model, trained  # noqa: F401  (the trained-model fixture)
from test_gpu_nbest import _check, _nbest, _state
from test_gpu_sample import (_check_bookkeeping, _head_nll, _inputs, _model, _sample, _teacher_forced,
                             _teacher_forced_nll, _vocab)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
DTYPES = [torch.float32, torch.bfloat16]


@pytest.fixture(scope="module", autouse=True)
def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _code(x):
    from fira_icse_b200._lib import FIRA_BF16, FIRA_F32
    return FIRA_BF16 if x.dtype == torch.bfloat16 else FIRA_F32


def _prefix(B, T, forced, pos):
    """prefix [B, T] and prefix_len [B] on the device: commit b forced at `pos` with label forced[b] (None = free)"""
    pre = torch.zeros((B, T), dtype=torch.int32)
    n = torch.zeros(B, dtype=torch.int32)
    for b, j in enumerate(forced):
        if j is not None:
            pre[b, :pos + 1] = 4
            pre[b, pos] = j
            n[b] = pos + 1 + b % 2                        # the prefix may go on after pos
        else:
            n[b] = pos if b % 2 else 0                    # ended exactly at pos, or no prefix at all
    return pre.to(DEV), n.to(DEV)


# ------------------------------------------------------------------ sampler step
def _sample_step(inputs, N, V, pos, T, prefix=None, uniforms=None, seed=0, eos=-1, pad=0, k=0, p=1.0):
    """one fira_pointer_mix_sample[_prefix] step at `pos` from a fixed mid-decode state -> every written buffer"""
    from fira_icse_b200 import ops
    from fira_icse_b200._lib import call
    logits, sc, gl, mem_mask, copy_src = inputs
    R, S = logits.shape[0], sc.shape[-1]
    gen = torch.Generator().manual_seed(pos)
    i32 = dict(dtype=torch.int32, device=DEV)
    o = dict(nxt=torch.full((R,), -7, **i32), seq=torch.full((R, T), -7, **i32), raw=torch.full((R, T), -7, **i32),
             tlp=torch.full((R, T), 9.0, device=DEV), msk=torch.full((R, T), 7, dtype=torch.uint8, device=DEV),
             fin=torch.zeros(R, dtype=torch.uint8, device=DEV), length=torch.full((R,), pos + 1, **i32),
             lp=(-torch.rand(R, generator=gen) * 5).to(DEV))
    o["fin"][1] = 1                                       # a finished row pads whatever its commit's prefix says
    o["lp0"] = o["lp"].clone()                            # the state before the step
    seed_t = torch.tensor([seed], dtype=torch.int64, device=DEV)
    first_t = torch.tensor([3], **i32)
    P = ops._ptr
    args = [P(logits), logits.stride(0), P(sc), P(gl), P(mem_mask), P(copy_src), P(seed_t), P(first_t), P(uniforms),
            1.0, int(k), float(p), eos, pad, P(o["nxt"]), P(o["seq"]), P(o["raw"]), P(o["tlp"]), P(o["msk"]), T, pos,
            P(o["fin"]), P(o["length"]), P(o["lp"]), R // N, N, V, S, _code(logits), ops._stream()]
    if prefix is None:
        call("fira_pointer_mix_sample", *args)
    else:
        call("fira_pointer_mix_sample_prefix", *args, P(prefix[0]), T, P(prefix[1]))
    torch.cuda.synchronize()
    return {key: v.cpu() for key, v in o.items()}


def _rows_equal(a, b, rows):
    for key in a:
        assert torch.equal(a[key][rows], b[key][rows]), key


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("philox", [False, True])
def test_sample_prefix_len_zero_and_free_commits_match_the_twin(dtype, philox):
    gen = torch.Generator().manual_seed(11 + philox)
    B, N, V, S, T, pos = 4, 4, 24650, 370, 8, 3
    inputs = _inputs(gen, B, N, V, S, dtype)
    for k, p in ((0, 1.0), (5, 0.9)):
        u = None if philox else torch.rand(B * N, generator=gen).to(DEV)
        kw = dict(uniforms=u, seed=77, k=k, p=p)
        twin = _sample_step(inputs, N, V, pos, T, **kw)
        zero = (torch.zeros((B, T), dtype=torch.int32, device=DEV), torch.zeros(B, dtype=torch.int32, device=DEV))
        _rows_equal(_sample_step(inputs, N, V, pos, T, prefix=zero, **kw), twin, slice(None))
        mixed = _prefix(B, T, [5, None, V, None], pos)               # commits 0 and 2 forced at pos
        got = _sample_step(inputs, N, V, pos, T, prefix=mixed, **kw)
        for b in (1, 3):
            _rows_equal(got, twin, slice(b * N, (b + 1) * N))


@pytest.mark.parametrize("dtype", DTYPES)
def test_forced_sample_rows_write_the_label_with_the_training_nll(dtype):
    gen = torch.Generator().manual_seed(23)
    B, N, V, S, T, pos, eos = 3, 4, 24650, 370, 8, 2, 7
    inputs = _inputs(gen, B, N, V, S, dtype)
    logits, sc, gl, mem_mask, copy_src = inputs
    s_copy = int(mem_mask[2].nonzero()[-1])                          # an unmasked copy position of commit 2
    labels = [11, eos, V + s_copy]                                    # vocabulary, <eos>, copy
    pre = _prefix(B, T, labels, pos)
    got = _sample_step(inputs, N, V, pos, T, prefix=pre, uniforms=torch.zeros(B * N, device=DEV), eos=eos)
    nll = _head_nll(logits, sc, gl, mem_mask, np.repeat(np.array(labels), N), N, V)
    c = pos + 1
    for r in range(B * N):
        if r == 1:                                                    # finished: pad, nothing counted
            assert got["seq"][r, c] == 0 and got["raw"][r, c] == 0 and got["tlp"][r, c] == 0
            assert got["length"][r] == pos + 1 and got["fin"][r] == 1 and got["lp"][r] == got["lp0"][r]
            continue
        j = labels[r // N]
        tok = j if j < V else int(copy_src[r // N, j - V])
        assert got["raw"][r, c] == j and got["seq"][r, c] == tok and got["nxt"][r] == tok
        assert got["msk"][r, c] == int(tok != 0)
        assert got["tlp"][r, c].item() == np.float32(-nll[r]), (r, got["tlp"][r, c].item(), -nll[r])   # bit for bit
        assert got["lp"][r] == got["lp0"][r] + got["tlp"][r, c]                                           # one fp32 add
        assert got["length"][r] == pos + 2 and got["fin"][r] == int(tok == eos)


# ------------------------------------------------------------------ n-best and diverse steps
def _beam_step(inputs, K, V, state, pos, T, G=None, prefix=None, alpha=0.6, diversity=0.5, eos=3, pad=0):
    """one (diverse, G given) beam step from `state` with or without a prefix -> the written half and the outputs"""
    from fira_icse_b200 import ops
    from fira_icse_b200._lib import call
    logits, sc, gl, mem_mask, copy_src = inputs
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
    chosen = torch.full((R,), -7, **i32)
    work = torch.zeros(R * K, dtype=torch.int64, device=DEV)
    work_lp = torch.zeros(R * K, dtype=torch.float32, device=DEV)
    P = ops._ptr
    args = [P(logits), logits.stride(0), P(sc), P(gl), P(mem_mask), P(copy_src), float(alpha), eos, pad, P(work),
            P(bufs["seq"]), P(bufs["raw"]), P(bufs["tlp"]), P(bufs["length"]), P(bufs["lp"]), P(bufs["score"]),
            P(bufs["status"]), P(parent), P(nxt), T, pos, R // K, K, V, S]
    if G is not None:
        args += [G, float(diversity), P(chosen), P(work_lp)]
    args += [_code(logits), ops._stream()]
    name = "fira_pointer_mix_beam_step" if G is None else "fira_pointer_mix_diverse_beam_step"
    if prefix is None:
        call(name, *args)
    else:
        call(name + "_prefix", *args, P(prefix[0]), T, P(prefix[1]))
    torch.cuda.synchronize()
    out = {k: v[1 - h].cpu() for k, v in bufs.items()}
    out.update(parent=parent.cpu(), nxt=nxt.cpu())
    if G is not None:
        out["chosen"] = chosen.cpu()
    return out


def _first_position(state, K, Kg):
    """commit 0 at position 0: the first slot of every group alone live, L = 0, length 1"""
    L, n, status, seq, raw, tlp = state
    status[:K] = 2
    status[:K:Kg], L[:K:Kg], n[:K:Kg] = 0, 0.0, 1
    return state


CONFIGS = [(1, None), (3, None), (5, None), (16, None), (4, 1), (4, 2), (4, 4), (6, 3), (16, 16)]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("K,G", CONFIGS)
def test_beam_prefix_len_zero_and_free_commits_match_the_twin(dtype, K, G):
    gen = torch.Generator().manual_seed(K * 31 + (G or 0) + (dtype == torch.bfloat16))
    B, V, S, T, pos = 3, 24650, 370, 8, 3
    Kg = K // (G or 1)
    inputs = _inputs(gen, B, K, V, S, dtype)
    state = _first_position(_state(gen, B, K, T, pos, V, 0), K, Kg)
    twin = _beam_step(inputs, K, V, state, pos, T, G)
    zero = (torch.zeros((B, T), dtype=torch.int32, device=DEV), torch.zeros(B, dtype=torch.int32, device=DEV))
    _rows_equal(_beam_step(inputs, K, V, state, pos, T, G, prefix=zero), twin, slice(None))
    got = _beam_step(inputs, K, V, state, pos, T, G, prefix=_prefix(B, T, [9, None, None], pos))
    for b in (1, 2):
        _rows_equal(got, twin, slice(b * K, (b + 1) * K))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("K,G", CONFIGS)
def test_forced_beam_commit_grows_its_live_slots_with_the_label(dtype, K, G):
    gen = torch.Generator().manual_seed(K * 37 + (G or 0) + (dtype == torch.bfloat16))
    B, V, S, T, pos, alpha = 3, 24650, 370, 8, 3, 0.6
    Kg = K // (G or 1)
    inputs = _inputs(gen, B, K, V, S, dtype)
    logits, sc, gl, mem_mask, copy_src = inputs
    state = _first_position(_state(gen, B, K, T, pos, V, 0), K, Kg)
    L, n, status, seq, raw, tlp = state
    s_copy = int(mem_mask[0].nonzero()[-1])
    for j in (17, V + s_copy):                                        # a vocabulary label and a copy label
        got = _beam_step(inputs, K, V, state, pos, T, G, prefix=_prefix(B, T, [j, None, None], pos), alpha=alpha)
        tok = j if j < V else int(copy_src[0, j - V])
        nll = _head_nll(logits, sc, gl, mem_mask, np.full(B * K, j), K, V)
        for k in range(K):
            assert got["parent"][k] == k                                # every slot's parent is itself
            if k % Kg == 0:                                             # the live slot of its group grows with j
                c = pos + 1
                assert got["raw"][k, c] == j and got["seq"][k, c] == tok and got["nxt"][k] == tok
                assert got["tlp"][k, c].item() == np.float32(-nll[k]), (k, j)      # bit for bit -nll
                assert got["lp"][k] == torch.tensor(L[k].item()) + got["tlp"][k, c]
                assert got["length"][k] == n[k] + 1 and got["status"][k] == 0
                want = got["lp"][k].double() / ((5.0 + n[k].double()) / 6.0) ** alpha
                assert abs(got["score"][k].double() - want) <= 1e-6 * abs(want) + 1e-12
                assert torch.equal(got["raw"][k, :c], raw[k, :c]) and torch.equal(got["seq"][k, :c], seq[k, :c])
                if G is not None:
                    assert got["chosen"][k] == tok
            else:                                                       # the others carried inactive
                assert got["status"][k] == 2 and got["nxt"][k] == 0
                assert torch.equal(got["raw"][k], raw[k]) and torch.equal(got["seq"][k], seq[k])
                if G is not None:
                    assert got["chosen"][k] == -1


# ------------------------------------------------------------------ end to end
def _eos_prefix(lab, k, eos):
    """the first k labels after <start>, never <eos> (zeros from a message's end on)"""
    pre = lab[:, 1:1 + k].clone()
    return pre.masked_fill((pre == eos).long().cumsum(1) > 0, 0)


def _score(m, b, **kw):
    from fira_icse_b200.sample import score
    v = _vocab()
    return score(m, b[0], b[3], b[4], b[5].to(DEV), b[7], b[6], start_id=v["<start>"], eos_id=v["<eos>"],
                 pad_id=v["<pad>"], **kw)


def _tokens(b, lab, V):
    """labels -> vocabulary ids through the commit's own sou / sub_token"""
    copy_src = torch.cat((b[0], b[7]), 1).to(lab.device)
    return torch.where(lab >= V, copy_src.gather(1, (lab - V).clamp(min=0)), lab)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_score_is_the_teacher_forced_nll(precision):
    m = _model(precision)
    b = golden_batch(0, 16)
    v = _vocab()
    out = _score(m, b)
    lab = b[6]
    n_msg = (lab[:, 1:] == v["<eos>"]).int().argmax(1) + 1                       # labels up to and including <eos>
    assert torch.equal(out.length.cpu(), n_msg + 1)
    tf = _teacher_forced(m, b, type("O", (), dict(seq=b[1].unsqueeze(1).to(DEV), raw=lab.unsqueeze(1).to(DEV)))())
    with torch.no_grad():
        nll = _teacher_forced_nll(m, tf, m.shifted_label(tf[6]).to(torch.int32).view(-1))
    got, ref = -out.token_logprob[:, 1:].cpu(), nll[:, :-1].cpu()
    live = torch.arange(29).unsqueeze(0) < n_msg.unsqueeze(1)
    assert (got[~live] == 0).all() and (out.token_logprob[:, 0] == 0).all()
    if precision == "fp32":
        torch.testing.assert_close(got[live], ref[live], rtol=1e-4, atol=1e-6)
    else:
        d = (got[live] - ref[live]).abs()                 # incremental vs full bf16 decoder (test_gpu_sample.py)
        assert d.median().item() <= 5e-2 and d.max().item() <= 0.5
    torch.testing.assert_close(out.logprob.cpu(), out.token_logprob.sum(1).cpu(), rtol=1e-5, atol=1e-5)
    with pytest.raises(ValueError, match="<eos>"):
        _score(m, b, tar_len=4)                           # messages longer than 2 labels: no <eos> within tar_len


@pytest.mark.parametrize("seed", [3, 8])
def test_sample_reproduces_itself_from_its_own_prefix(seed):
    m = _model("fp32")
    b = golden_batch(0, 16)
    ref = _sample(m, b, num_samples=1, seed=seed)
    for k in (1, 3, 5):
        out = _sample(m, b, num_samples=1, seed=seed, prefix=ref.raw[:, 0, 1:1 + k])   # <eos> last at most, 0 after
        assert torch.equal(out.seq, ref.seq) and torch.equal(out.raw, ref.raw), k
        # two decoder runs over the same tokens: the split-K fp32 atomics leave the sums ~1e-6 apart (relative)
        torch.testing.assert_close(out.logprob, ref.logprob, rtol=1e-5, atol=1e-5)


def test_nbest_beam_1_reproduces_itself_from_its_own_prefix():
    m = _model("fp32")
    b = golden_batch(0, 16)
    v = _vocab()
    ref = _nbest(m, b, beam_size=1, length_penalty=0.6)
    for k in (1, 3, 5):
        out = _nbest(m, b, beam_size=1, length_penalty=0.6, prefix=_eos_prefix(ref.raw[:, 0], k, v["<eos>"]))
        assert torch.equal(out.seq, ref.seq) and torch.equal(out.raw, ref.raw), k
        # two decoder runs over the same tokens: the split-K fp32 atomics leave the sums ~1e-6 apart (relative)
        torch.testing.assert_close(out.logprob, ref.logprob, rtol=1e-5, atol=1e-5)
        torch.testing.assert_close(out.score, ref.score, rtol=1e-5, atol=1e-5)


DECODERS = {
    "sample": dict(num_samples=4, seed=5),
    "nbest3": dict(beam_size=3),
    "nbest5": dict(beam_size=5, length_penalty=0.6),
    "diverse": dict(beam_size=4, groups=2, diversity=0.5),
    "mbr": dict(num_samples=4, seed=5),
}


def _decode(name, m, b, **kw):
    from fira_icse_b200.mbr import mbr
    v = _vocab()
    kw = dict(DECODERS[name], **kw)
    if name == "mbr":
        return mbr(m, b[0], b[3], b[4], b[5].to(DEV), b[7], start_id=v["<start>"], eos_id=v["<eos>"],
                   pad_id=v["<pad>"], **kw)
    return (_sample if name == "sample" else _nbest)(m, b, **kw)


@pytest.mark.parametrize("name", list(DECODERS))
def test_reference_prefixes(name):
    m = _model("fp32")
    b = golden_batch(0, 16)
    v = _vocab()
    V = m.vocab_size
    pre = _eos_prefix(b[6], 3, v["<eos>"])
    out = _decode(name, m, b, prefix=pre)
    hyp = out.samples if name == "mbr" else out
    if name in ("sample", "mbr"):
        _check_bookkeeping(hyp, v)
    else:
        _check(hyp, v)
    sc = _score(m, b)
    n = (pre != 0).sum(1)
    assert (n > 0).all()
    toks = _tokens(b, pre, V).to(DEV)
    for c in range(pre.shape[0]):
        P = int(n[c])
        raw, seq = hyp.raw[c, :, 1:1 + P].cpu(), hyp.seq[c, :, 1:1 + P]
        assert (raw == pre[c, :P]).all() and (seq == toks[c, :P]).all(), c
        torch.testing.assert_close(hyp.token_logprob[c, :, 1:1 + P],
                                   sc.token_logprob[c, 1:1 + P].expand(raw.shape[0], P), rtol=1e-4, atol=1e-5)
        if name == "mbr":
            assert (out.seq[c, 1:1 + P] == toks[c, :P]).all(), c


@pytest.mark.parametrize("name", list(DECODERS))
def test_zero_prefix_is_no_prefix(name):
    m = _model("fp32")
    b = golden_batch(0, 8)
    none = _decode(name, m, b)
    zero = _decode(name, m, b, prefix=torch.zeros((8, 5), dtype=torch.int64))
    assert torch.equal(none.seq, zero.seq)
    if name != "mbr":
        assert torch.equal(none.raw, zero.raw)


def test_prefix_errors_raise_before_any_device_work():
    m = _model("fp32")
    b = golden_batch(0, 4)
    v = _vocab()
    with pytest.raises(ValueError, match="<eos>"):
        _nbest(m, b, beam_size=3, prefix=torch.tensor([[5, v["<eos>"]]] * 4))
    with pytest.raises(ValueError, match="shape"):
        _sample(m, b, prefix=torch.ones((3, 2), dtype=torch.int64))


# ------------------------------------------------------------------ run_model.py test
def _expected_words(d, n_words):
    """each test commit's first n reference words as run_model.py writes them (deanonymised), in test order"""
    import run_model
    from fira_icse_b200.data import build_commit
    raw = load_raw_golden()
    vocab = raw["word_vocab"]
    r_vocab = {i: w for w, i in vocab.items()}
    upper = set(raw["VOCAB_UPPER_CASE"])
    out = []
    for i in json.load(open(d / "all_index"))["test"]:
        tar = build_commit(raw["raw"], i, vocab, raw["ast_change_vocab"], upper)["tar"]
        ids = tar[1:tar.index(vocab["<eos>"])][:n_words]
        out.append(run_model.deanonymise(run_model.ids_to_text(ids, r_vocab), raw["raw"]["variable"][i]))
    return out


@pytest.mark.parametrize("mode,name,per,fields", [("nbest", "output_fira_nbest_prefix2", 3, 2),
                                                  ("sample", "output_fira_samples_prefix2", 2, 1)])
def test_run_model_prefix_words(trained, mode, name, per, fields):  # noqa: F811
    d, base, _ = trained
    env = dict(base, FIRA_DECODE=mode, FIRA_PREFIX_WORDS="2", FIRA_BEAM="3", FIRA_SAMPLES="2")
    r = _run_model("test", d, env)
    assert "mean sentence bleu" in r.stdout
    lines = open(d / "OUTPUT" / name).read().split("\n")
    want = _expected_words(d, 2)
    assert len(lines) == per * len(want) + 1 and lines[-1] == ""
    for c, words in enumerate(want):
        for ln in lines[per * c:per * (c + 1)]:
            msg = ln.split("\t", fields)[fields].split()
            assert msg[:len(words)] == words, (c, ln, words)


def test_run_model_beam_rejects_a_prefix(trained):  # noqa: F811
    d, base, _ = trained
    r = subprocess.run([sys.executable, os.path.join(ROOT, "run_model.py"), "test"], cwd=d,
                       env=dict(base, FIRA_DECODE="beam", FIRA_PREFIX_WORDS="2"), capture_output=True, text=True,
                       timeout=900)
    assert r.returncode != 0 and "FIRA_PREFIX_WORDS applies to FIRA_DECODE=sample, nbest and mbr" in r.stderr
