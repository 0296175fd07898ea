"""Self-critical fine-tuning on the GPU: fira_bleu_reward against the float64 rule (tests/scst_rule.py), the weighted head
backward against the unweighted kernel and float64 autograd, the gradient pass against the sampler's own
log-probabilities and the float64 oracle, the decoding loop after an optimizer step, and `run_model.py finetune`."""
import copy
import os

import numpy as np
import pytest
import torch

from bf16_bound import close
from fira_testlib import golden_batch, load_raw_golden, seeded_model
from scst_rule import rewards as rule_rewards
from test_gpu_mbr import _candidates

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
START, EOS, PAD = 2, 1, 0
TOL = 1e-12
V = 24650
D = 256
FIRA_ERR_SHAPE = 1


@pytest.fixture(scope="module", autouse=True)
def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _vocab_ids():
    v = load_raw_golden()["word_vocab"]
    return dict(start_id=v["<start>"], eos_id=v["<eos>"], pad_id=v["<pad>"])


# ============================================================================= fira_bleu_reward
def _references(rng, B, T, ld):
    """<start>, words of the 5-id vocabulary with start / pad ids mid-message, <eos> (none in every fifth row), then ids
    the rule never reads"""
    ref = rng.integers(3, 8, (B, ld))
    ref[:, 0] = START
    for b in range(B):
        L = int(rng.integers(1, T))
        if rng.random() < 0.3:
            ref[b, 1 + rng.integers(0, L)] = rng.choice([START, PAD])
        if b % 5 != 4:
            ref[b, L] = EOS
    return torch.from_numpy(ref)


def _kernel(seq, length, ref, T):
    from fira_icse_b200 import scst
    assert seq.shape[2] == T
    r, a = scst.rewards(seq.to(DEV), length.to(DEV), ref.to(DEV), start_id=START, eos_id=EOS, pad_id=PAD)
    torch.cuda.synchronize()
    return r.cpu().numpy(), a.cpu().numpy()


@pytest.mark.parametrize("B", [0, 1, 48])
@pytest.mark.parametrize("N", [2, 5, 32])
def test_reward_kernel_matches_float64_rule(B, N):
    rng = np.random.default_rng(1000 + 10 * N + B)
    for T in (32, 30, 2):
        seq, length = _candidates(rng, B, N, T, T)
        ref = _references(rng, B, T, T + 3)
        if B > 2:
            seq[1, 0, :T], length[1, 0] = ref[1, :T], T          # a sample that copies its reference
            seq[2, :, 1:T] = seq[2, :, 1:T] % 2 + 3               # two ids only: repeated n-grams everywhere
        r, a = _kernel(seq, length, ref, T)
        assert r.shape == (B, N) and a.shape == (B, N)
        for b in range(B):
            rr, ra = rule_rewards(seq[b].tolist(), length[b].tolist(), ref[b].tolist(), START, EOS, PAD)
            np.testing.assert_allclose(r[b], np.array(rr), rtol=0, atol=TOL)
            np.testing.assert_allclose(a[b], np.array(ra), rtol=0, atol=TOL)
            if b % 8 == 2:                                        # _candidates: every sample of the commit the same
                assert (a[b] == 0).all()


def test_reward_kernel_all_equal_and_exact_copies():
    T, N = 12, 4
    ref = torch.tensor([[START, 5, 6, 7, 5, 6, 7, 8, EOS] + [PAD] * 3] * 2)
    seq = ref.unsqueeze(1).repeat(1, N, 1)
    length = torch.full((2, N), 9)
    seq[1, 2:] = torch.tensor([START, 9, 9, EOS] + [PAD] * 8)
    length[1, 2:] = 4
    r, a = _kernel(seq, length, ref, T)
    assert (r[0] == 1.0).all() and (a[0] == 0.0).all()
    assert (r[1, :2] == 1.0).all() and (r[1, 2:] == 0.0).all()
    np.testing.assert_array_equal(a[1], [2.0 / 3.0, 2.0 / 3.0, -2.0 / 3.0, -2.0 / 3.0])


def test_reward_kernel_shape_errors():
    from fira_icse_b200 import _lib
    lib = _lib.lib()
    s = torch.zeros((2, 4, 32), dtype=torch.int32, device=DEV)
    n = torch.ones((2, 4), dtype=torch.int32, device=DEV)
    out = torch.zeros((2, 4), dtype=torch.float64, device=DEV)
    p = lambda t: t.data_ptr()
    st = torch.cuda.current_stream().cuda_stream
    call = lambda ld, ldr, B, N, T: lib.fira_bleu_reward(p(s), p(n), ld, p(s), ldr, START, EOS, PAD, p(out), p(out), B,
                                                         N, T, st)
    assert call(32, 32, 2, 4, 32) == 0
    assert call(32, 32, 0, 4, 32) == 0
    for args in ((32, 32, 2, 1, 32), (32, 32, 2, 33, 32), (33, 33, 2, 4, 33), (32, 32, 2, 4, 1), (30, 32, 2, 4, 32),
                 (32, 30, 2, 4, 32), (32, 32, -1, 4, 32)):
        assert call(*args) == FIRA_ERR_SHAPE, args
    torch.cuda.synchronize()


# ============================================================================= weighted head backward
HEAD_PARAMS = ("out_fc.weight", "out_fc.bias", "copy_net.LinearSource.weight", "copy_net.LinearTarget.weight",
               "copy_net.LinearRes.weight", "copy_net.LinearRes.bias", "copy_net.LinearProb.weight",
               "copy_net.LinearProb.bias")
HEAD_ROUNDED = ("out_fc.weight", "copy_net.LinearSource.weight", "copy_net.LinearTarget.weight")
EPS_HEAD = 2 ** -7                                   # tests/test_gpu_bf16_step.py


def _head_inputs(bf16):
    """six golden commits: labels (a zero label mid-message, an all-copy row), bf16-exact memory and decoder rows"""
    parts = [golden_batch(i, i + 1) for i in (0, 5, 9, 64, 77, 100)]
    sou, tar_label, sub = (torch.cat([p[k] for p in parts], 0) for k in (0, 6, 7))
    mem_valid = torch.cat((sou != 0, sub != 0), 1)
    label = torch.cat((tar_label[:, 1:], torch.zeros_like(tar_label[:, :1])), 1)
    label[0, 2] = 0
    pos = torch.nonzero(mem_valid[2]).view(-1)
    label[2] = 0
    label[2, :10] = V + pos[torch.arange(10) * 7 % len(pos)]
    B, S = label.shape[0], mem_valid.shape[1]
    g = torch.Generator().manual_seed(7)
    memory = torch.randn((B, S, D), generator=g).to(torch.bfloat16).float()
    dec = torch.randn((B, label.shape[1], D), generator=g).to(torch.bfloat16).float()
    return memory, dec, mem_valid, label


def _run_head(bf16, weight, memory, dec, mem_valid, label):
    from fira_icse_b200 import ops
    model = seeded_model()
    params = [dict(model.named_parameters())[k].detach().to(DEV).clone().requires_grad_(True) for k in HEAD_PARAMS]
    m = memory.to(DEV).requires_grad_(True)
    d = dec.to(DEV).requires_grad_(True)
    w = None if weight is None else weight.to(DEV, torch.float32)
    loss, nll, _ = ops.HeadFn.apply(False, bf16, None, m, d, mem_valid.to(torch.uint8).to(DEV),
                                    label.to(torch.int32).reshape(-1).to(DEV), *params, None, w)
    loss.backward()
    torch.cuda.synchronize()
    return loss, nll, m.grad, d.grad, [p.grad for p in params]


@pytest.mark.parametrize("bf16", [False, True], ids=["fp32", "bf16"])
def test_unit_weights_are_bit_identical_in_the_kernel(bf16):
    """fira_pointer_mix_nll_bwd_rows_weighted with weights 1.0 writes exactly what fira_pointer_mix_nll_bwd_rows writes"""
    from fira_icse_b200 import ops
    from fira_icse_b200._lib import call
    g = torch.Generator().manual_seed(3)
    memory, dec, mem_valid, label = _head_inputs(bf16)
    B, T = label.shape
    S = mem_valid.shape[1]
    R, ld = B * T, ops._ld_logits(V)
    dt = torch.bfloat16 if bf16 else torch.float32
    code = 1 if bf16 else 0
    logits = (torch.randn((R, ld), generator=g) * 3).to(DEV, dt)
    sc = torch.randn((B, T, S), generator=g).to(DEV)
    gl = torch.randn((R, 2), generator=g).to(DEV)
    mm = mem_valid.to(torch.uint8).to(DEV)
    lab = label.to(torch.int32).reshape(-1).to(DEV)
    stats = torch.empty((R, 8), device=DEV)
    nll = torch.empty(R, device=DEV)
    p = ops._ptr
    st = ops._stream()
    call("fira_pointer_mix_nll_fwd_rows", p(logits), ld, p(sc), p(gl), p(mm), p(lab), None, p(stats), p(nll), None, R,
         T, V, S, code, st)
    up = torch.tensor([0.37], device=DEV)
    ones = torch.ones(B, device=DEV)
    outs = []
    for weighted in (False, True):
        dl = torch.full((R, ld), 7.0, device=DEV, dtype=dt)
        dsc = torch.full((B, T, S), 7.0, device=DEV)
        dgl = torch.full((R, 2), 7.0, device=DEV)
        act = torch.full((R,), 7, dtype=torch.uint8, device=DEV)
        args = (p(logits), ld, p(sc), p(mm), p(lab), None, None, 0, p(stats), p(up), p(dl), p(dsc), p(dgl), p(act), R,
                T, V, S, code, st)
        if weighted:
            call("fira_pointer_mix_nll_bwd_rows_weighted", *args, p(ones))
        else:
            call("fira_pointer_mix_nll_bwd_rows", *args)
        outs.append((dl[:, :V], dsc, dgl, act))
    torch.cuda.synchronize()
    for a, b in zip(*outs):
        assert torch.equal(a, b)
    assert int(outs[0][3].sum()) > 0                             # the copy rows are active


@pytest.mark.parametrize("bf16", [False, True], ids=["fp32", "bf16"])
def test_unit_weights_match_the_unweighted_head(bf16):
    inputs = _head_inputs(bf16)
    B = inputs[3].shape[0]
    ref = _run_head(bf16, None, *inputs)
    one = _run_head(bf16, torch.ones(B), *inputs)
    assert torch.equal(ref[1], one[1])                           # the per-position NLL is the same forward
    names = ["loss", "d_memory", "d_dec"] + list(HEAD_PARAMS)
    for k, a, b in zip(names, [ref[0], ref[2], ref[3]] + ref[4], [one[0], one[2], one[3]] + one[4]):
        if k == "copy_net.LinearRes.bias":                       # zero in exact arithmetic: round-off only
            continue
        # the products accumulate with split-K atomics: equal up to fp32 summation order
        a, b = a.detach(), b.detach()
        assert float((a - b).abs().max()) <= 1e-5 * float(a.abs().max()), k


WEIGHTS = torch.tensor([0.7, -1.3, 0.0, 2.1, -0.4, 0.0])


def _head_reference(memory, dec, mem_valid, label, weight, rounded):
    import fira_oracle as O
    model = seeded_model()
    named = dict(model.named_parameters())
    sd = {k: (named[k].detach().to(torch.bfloat16).double() if rounded and k in HEAD_ROUNDED else
              named[k].detach().double()).requires_grad_(True) for k in HEAD_PARAMS}
    m64 = memory.double().requires_grad_(True)
    d64 = dec.double().requires_grad_(True)
    logp, _ = O.output_distribution(sd, m64, mem_valid, d64)
    keep = label != 0
    nll = -logp.gather(-1, label.unsqueeze(-1)).squeeze(-1) * keep
    loss = (weight.double().unsqueeze(1) * nll).sum()
    loss.backward()
    return loss, nll, m64.grad, d64.grad, [sd[k].grad for k in HEAD_PARAMS]


def test_weighted_head_fp32_matches_float64():
    inputs = _head_inputs(False)
    loss, nll, dm, dd, dp = _run_head(False, WEIGHTS, *inputs)
    rl, rn, rdm, rdd, rdp = _head_reference(*inputs, WEIGHTS, rounded=False)
    assert abs(loss.item() - rl.item()) <= 1e-4 * float((WEIGHTS.double().abs().unsqueeze(1) * rn).sum())
    for what, g, r in [("nll", nll.view_as(rn), rn), ("d_memory", dm, rdm), ("d_dec", dd, rdd)] + \
            [(k, g, r) for k, g, r in zip(HEAD_PARAMS, dp, rdp)]:
        g, r = g.detach().cpu().double(), r.detach().double()
        if what == "copy_net.LinearRes.bias":                   # zero in exact arithmetic (softmax shift invariance)
            assert float(g.abs().max()) <= 1e-4 * float(rdp[HEAD_PARAMS.index("copy_net.LinearRes.weight")].abs().max())
            continue
        err = float((g - r).abs().max())
        assert err <= 1e-4 * float(r.abs().max()), (what, err, float(r.abs().max()))
    for b in np.flatnonzero(WEIGHTS.numpy() == 0):              # a zero-weight sequence takes no gradient at all
        assert float(dd[b].abs().max()) == 0.0


def test_weighted_head_bf16_matches_float64():
    inputs = _head_inputs(True)
    loss, nll, dm, dd, dp = _run_head(True, WEIGHTS, *inputs)
    rl, rn, rdm, rdd, rdp = _head_reference(*inputs, WEIGHTS, rounded=True)
    close("scst head nll", nll.view_as(rn), rn, EPS_HEAD, rows=True)
    close("scst head d_dec", dd, rdd, EPS_HEAD, rows=True)
    close("scst head d_memory", dm, rdm, EPS_HEAD, rows=True)
    for k, g, r in zip(HEAD_PARAMS, dp, rdp):
        if k == "copy_net.LinearRes.bias":
            continue
        close(f"scst head {k}", g, r, EPS_HEAD)
    for b in np.flatnonzero(WEIGHTS.numpy() == 0):
        assert float(dd[b].abs().max()) == 0.0


# ============================================================================= the gradient pass
def _model(precision):
    from test_gpu_sample import _model as sharpened
    return sharpened(precision)


def _samples(m, b, N=4, seed=11):
    from fira_icse_b200.sample import sample
    return sample(m, b[0], b[3], b[4], b[5].to(DEV), b[7], num_samples=N, top_p=0.95, seed=seed, **_vocab_ids())


def test_teacher_forced_nll_of_the_samples_is_the_samplers_logprob():
    from fira_icse_b200 import scst
    m = _model("fp32")
    b = [t.to(DEV) for t in golden_batch(0, 8)]
    s = _samples(m, b)
    B, N, T = s.seq.shape
    with torch.no_grad():
        _, nll = scst.policy_loss(m, b, s.seq, s.raw, torch.ones(B * N, device=DEV))
    nll = nll.view(B, N, T).cpu()
    tlp = s.token_logprob.cpu()
    np.testing.assert_allclose(nll[..., :T - 1].numpy(), -tlp[..., 1:].numpy(), rtol=0, atol=1e-4)
    assert (nll[..., T - 1] == 0).all()


def _replicated(b, s):
    """the padded batch repeated per sample with the samples as tar / tar_label (CPU, for the oracle)"""
    N, T = s.seq.shape[1], s.seq.shape[2]
    rep = [x.repeat_interleave(N, 0) for x in b]
    rep[1] = s.seq.reshape(-1, T).cpu()
    rep[6] = s.raw.reshape(-1, T).cpu()
    return rep


def _step_grads(m, b, s, weight):
    from fira_icse_b200 import scst
    m.zero_grad(set_to_none=True)
    loss, _ = scst.policy_loss(m, [t.to(DEV) for t in b], s.seq, s.raw, weight.to(DEV, torch.float32))
    loss.backward()
    torch.cuda.synchronize()
    return loss.item(), {k: p.grad for k, p in m.named_parameters() if p.grad is not None}


def _oracle_step(m, b, s, weight):
    import fira_oracle as O
    sd = {k: v.detach().cpu().double().requires_grad_(v.is_floating_point()) for k, v in m.state_dict().items()}
    detail = {}
    rep = _replicated(b, s)
    O.forward(sd, *rep, stage="train", detail=detail)
    terms = weight.double().unsqueeze(1) * detail["nll"]
    loss = terms.sum()
    loss.backward()
    return loss.item(), {k: v.grad for k, v in sd.items() if v.requires_grad}, float(terms.abs().sum())


def _plain(precision):
    """the seeded model (not sharpened: the bf16 bounds of tests/test_gpu_bf16_step.py hold at its scale)"""
    return copy.deepcopy(seeded_model()).to(DEV).eval().set_precision(precision)


def test_whole_step_gradients_fp32_match_float64():
    m = _plain("fp32")
    b = golden_batch(0, 3)
    s = _samples(m, [t.to(DEV) for t in b])
    B, N = s.seq.shape[:2]
    w = torch.tensor([0.4, -0.9, 0.0, 1.3, -0.2, 0.8, 0.0, -1.1, 0.5, 0.3, -0.6, 0.9])[:B * N] / (B * N)
    loss, grads = _step_grads(m, b, s, w)
    ref_loss, ref, scale = _oracle_step(m, b, s, w)
    assert abs(loss - ref_loss) <= 1e-4 * scale
    assert sorted(grads) == sorted(k for k, g in ref.items() if g is not None)
    for k, g in grads.items():
        r = ref[k].numpy()
        scale = float(np.abs(r).max())
        if k.endswith("fc_k.bias") or k == "copy_net.LinearRes.bias":
            assert float(g.abs().max()) < 1e-6, k
            continue
        np.testing.assert_allclose(g.cpu().numpy(), r, rtol=5e-3, atol=1e-7 + 5e-4 * scale, err_msg=k)


def test_whole_step_gradients_bf16_match_float64(monkeypatch):
    from test_gpu_bf16_step import check_step, record_gates
    m = _plain("bf16")
    b = golden_batch(0, 3)
    s = _samples(m, [t.to(DEV) for t in b])
    B, N = s.seq.shape[:2]
    w = torch.linspace(0.2, 1.0, B * N) / (B * N)     # one sign: the loss is no cancellation of large terms
    loss, grads = _step_grads(m, b, s, w)
    gates = {}
    record_gates(monkeypatch, gates)
    ref_loss, ref, _ = _oracle_step(m, b, s, w)
    check_step("scst/padded", loss, grads, ref_loss, ref, gates)


# ============================================================================= the decoding loop after a step
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_sampling_after_a_step_uses_the_new_weights_without_recapture(precision):
    from fira_icse_b200 import TransModel, optim, scst
    from fira_icse_b200.decode_loop import _LOOPS
    from fira_testlib import reference_args
    m = _model(precision)
    b = [t.to(DEV) for t in golden_batch(0, 8)]
    kw = dict(num_samples=4, top_p=0.95, seed=3, **_vocab_ids())
    opt = optim.FlatAdam(m.live_parameters(), lr=1e-3, groups=m.flat_groups())
    optim.attach(m, [opt])
    from fira_icse_b200.sample import sample
    before = sample(m, b[0], b[3], b[4], b[5], b[7], **kw)
    (key, (_, _, loop)), = _LOOPS[m].items()
    graphs = dict(loop.graphs)
    assert graphs
    step = scst.scst_step(m, opt, b, tar_len=30, **kw)
    assert np.isfinite(step.loss) and 0.0 <= step.reward <= 1.0 and step.advantage >= 0.0
    m.eval()
    after = sample(m, b[0], b[3], b[4], b[5], b[7], **kw)
    assert _LOOPS[m][key][2] is loop and loop.graphs.keys() == graphs.keys()
    assert all(loop.graphs[k] is g for k, g in graphs.items())
    fresh = TransModel(reference_args())
    fresh.load_state_dict({k: v.cpu() for k, v in m.state_dict().items()})
    fresh = fresh.to(DEV).eval().set_precision(precision)
    ref = sample(fresh, b[0], b[3], b[4], b[5], b[7], **kw)
    # the step moves token log-probabilities by O(1) (a stale operand would show that much); two decodings of the same
    # weights differ by split-K summation order only.  bf16 carries that as larger noise, which can flip a near-tie draw
    # (about a fifth of the rows here):
    # compare each row up to its first differing draw
    T = after.seq.shape[-1]
    differ = (after.seq != ref.seq) | (after.raw != ref.raw)
    first = torch.where(differ.any(-1), differ.float().argmax(-1), torch.full_like(differ[..., 0], T, dtype=torch.long))
    if precision == "fp32":
        assert bool((first == T).all())
    agree = torch.arange(T, device=DEV) < first.unsqueeze(-1)
    assert float(agree.float().mean()) >= 0.5
    # bf16: the bound tests/test_gpu_sample.py gives two bf16 decodings of the sharpened model (measured here: 0.27)
    tol = 1e-4 if precision == "fp32" else 0.5
    np.testing.assert_allclose(after.token_logprob[agree].cpu().numpy(), ref.token_logprob[agree].cpu().numpy(), rtol=0,
                               atol=tol)
    if step.advantage > 0:                                                # the step moved the model
        assert not torch.equal(after.token_logprob, before.token_logprob)


# ============================================================================= CLI
@pytest.fixture(scope="module")
def trained(tmp_path_factory):
    from fira_testlib import ROOT
    from test_data import _write_dataset
    from test_gpu_cli import _run_model
    d = tmp_path_factory.mktemp("cli_scst")
    _write_dataset(str(d), load_raw_golden())
    env = dict(os.environ, PYTHONPATH=ROOT, FIRA_EPOCHS="1", FIRA_BATCH="16", FIRA_MAX_BATCHES="3",
               FIRA_WORKERS="0", FIRA_TEST_BATCH="4")
    _run_model("train", d, env)
    return d, env


def test_run_model_finetune_then_test(trained):
    from test_gpu_cli import _run_model
    d, env = trained
    base = open(d / "best_model.pt", "rb").read()
    r = _run_model("finetune", d, dict(env, FIRA_MAX_BATCHES="2", FIRA_SAMPLES="4"))
    assert "scst epoch: 0 batch: 0/" in r.stdout and "best dev bleu" in r.stdout
    assert open(d / "best_model.pt", "rb").read() == base
    sd = torch.load(d / "best_model_scst.pt", map_location="cpu")
    assert len(sd) == 338 and sorted(sd) == sorted(torch.load(d / "best_model.pt", map_location="cpu"))
    r = _run_model("test", d, dict(env, FIRA_CHECKPOINT="best_model_scst.pt"))
    assert "mean sentence bleu" in r.stdout
    assert os.path.getsize(d / "OUTPUT" / "output_fira") > 0
