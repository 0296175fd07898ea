"""The exponential moving average of the weights on the device: fira_adam_flat with `ema` (bit-identical Adam, the EMA
against ema_rule), optim.FlatAdam(ema_decay) against torch.optim.Adam plus a float64 EMA and its state_dict round trip,
the EMA of every GraphedTrainStep mode against the float64 recurrence over the parameters' trajectory, the shadow model
(optim.ema_model / GraphedTrainStep.ema_model) against freshly loaded copies of its weights, and `run_model.py train`
with FIRA_EMA."""
import copy
import gc
import json
import os

import numpy as np
import pytest
import torch

import ema_rule
from fira_testlib import ROOT, golden_batch, load_raw_golden, reference_args, seeded_model

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
LR, B1, B2, EPS = 1e-3, 0.9, 0.999, 1e-8


@pytest.fixture(scope="module", autouse=True)
def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    yield
    # hand the engines' graph pools and the decoding loops' buffers back to the device before the next module: later
    # modules start training subprocesses of their own on this GPU
    gc.collect()
    torch.cuda.empty_cache()


# ============================================================================= the kernel
def _adam_flat(p, g, m, v, p16, t, scale, ema=None, d=0.0, ema_ptr=None):
    from fira_icse_b200 import _lib
    _lib.call("fira_adam_flat", p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), p16.data_ptr(), p.numel(), LR, B1,
              B2, EPS, t.data_ptr(), scale.data_ptr() if scale is not None else None,
              ema_ptr if ema_ptr is not None else (ema.data_ptr() if ema is not None else None), d,
              torch.cuda.current_stream().cuda_stream)


@pytest.mark.parametrize("n", [8 * 1001, 8 * 300_001])         # a partial last block; more than one grid-stride pass
@pytest.mark.parametrize("scaled", [False, True])
def test_kernel_ema_keeps_adam_bits_and_follows_the_rule(n, scaled):
    gen = torch.Generator(device=DEV).manual_seed(n + scaled)
    f32 = dict(dtype=torch.float32, device=DEV)
    p = torch.randn(n, generator=gen, **f32)
    g = torch.randn(n, generator=gen, **f32) * 3.0
    m = torch.randn(n, generator=gen, **f32) * 0.1
    v = torch.rand(n, generator=gen, **f32) * 0.01
    e = p + torch.randn(n, generator=gen, **f32) * 0.01
    t = torch.tensor(7.0, **f32)
    scale = torch.tensor(37.0, **f32) if scaled else None
    d = 0.999
    bufs = {}
    for with_ema in (False, True):
        b = dict(p=p.clone(), m=m.clone(), v=v.clone(), p16=torch.empty(n, dtype=torch.bfloat16, device=DEV),
                 e=e.clone())
        _adam_flat(b["p"], g, b["m"], b["v"], b["p16"], t, scale, b["e"] if with_ema else None, d if with_ema else 0.0)
        bufs[with_ema] = b
    torch.cuda.synchronize()
    off, on = bufs[False], bufs[True]
    for k in ("p", "m", "v", "p16"):
        assert torch.equal(off[k].view(torch.int32 if k != "p16" else torch.int16),
                           on[k].view(torch.int32 if k != "p16" else torch.int16)), k
    assert torch.equal(off["e"], e)                                    # no ema: the buffer is not touched
    p_new = on["p"].cpu().double().numpy()
    ref = ema_rule.ema(e.cpu().double().numpy(), p_new, d)
    got = on["e"].cpu().double().numpy()
    ulp = np.spacing(np.abs(ref).astype(np.float32)).astype(np.float64)
    assert np.all(np.abs(got - ref) <= 2 * ulp), np.max(np.abs(got - ref) / ulp)
    # and Adam itself against the float64 rule, loosely (the kernel's own fp32 roundings)
    p64, _, _ = ema_rule.adam(p.cpu().numpy(), g.cpu().numpy(), m.cpu().numpy(), v.cpu().numpy(), 7.0, LR, B1, B2, EPS,
                              37.0 if scaled else None)
    np.testing.assert_allclose(p_new, p64, rtol=1e-6, atol=1e-6)


def test_kernel_ema_argument_checks():
    from fira_icse_b200._lib import FiraLibraryError
    f32 = dict(dtype=torch.float32, device=DEV)
    n = 64
    p, g, m, v, e = (torch.zeros(n + 8, **f32) for _ in range(5))
    p16 = torch.zeros(n, dtype=torch.bfloat16, device=DEV)
    t = torch.tensor(1.0, **f32)
    for d in (0.0, 1.0, -0.5, 1.5, float("nan"), float("inf")):
        with pytest.raises(FiraLibraryError, match="ema_decay"):
            _adam_flat(p[:n], g[:n], m[:n], v[:n], p16, t, None, e[:n], d)
    with pytest.raises(FiraLibraryError, match="alignment"):
        _adam_flat(p[:n], g[:n], m[:n], v[:n], p16, t, None, d=0.9, ema_ptr=e.data_ptr() + 4)
    assert torch.equal(p, torch.zeros_like(p)) and torch.equal(e, torch.zeros_like(e))       # nothing was launched


# ============================================================================= FlatAdam
def _params(seed):
    g = torch.Generator().manual_seed(seed)
    shapes = [(256, 256), (256,), (256, 256), (256,), (1024, 256), (1024,), (2,), (1,), (1, 256), (333, 256), (24650,)]
    return [torch.nn.Parameter(torch.randn(s, generator=g).to(DEV)) for s in shapes]


def _grads(step, params):
    g = torch.Generator().manual_seed(100 + step)
    return [torch.randn(p.shape, generator=g).to(DEV) for p in params]


def _set_grads(params, grads):
    for q, gr in zip(params, grads):
        q.grad = gr.clone()


def test_flat_adam_ema_matches_torch_adam_and_float64_ema():
    from fira_icse_b200.optim import FlatAdam
    d = 0.9
    ref, mine, plain = _params(0), _params(0), _params(0)
    opt_ref = torch.optim.Adam(ref, lr=LR)
    opt = FlatAdam(mine, lr=LR, groups=[[mine[0], mine[2]], [mine[1], mine[3]]], ema_decay=d)
    opt_plain = FlatAdam(plain, lr=LR, groups=[[plain[0], plain[2]], [plain[1], plain[3]]])
    assert torch.equal(opt.ema, opt.p)                                # the average starts at the parameters
    ema64 = [p.detach().cpu().double().numpy() for p in ref]
    dd, c = ema_rule.ema_coefficients(d)
    for step in range(20):
        grads = _grads(step, ref)
        _set_grads(ref, grads)
        _set_grads(mine, grads)
        _set_grads(plain, grads)
        opt_ref.step()
        opt.step()
        opt_plain.step()
        ema64 = [dd * e + c * p.detach().cpu().double().numpy() for e, p in zip(ema64, ref)]
    torch.cuda.synchronize()
    assert torch.equal(opt.p, opt_plain.p) and torch.equal(opt.m, opt_plain.m) and torch.equal(opt.v, opt_plain.v)
    assert torch.equal(opt.p16, opt_plain.p16)                        # the EMA changes no bit of Adam
    sd = opt.state_dict()
    for p, q, e64, e in zip(ref, mine, ema64, sd["ema"]):
        torch.testing.assert_close(q.data, p.data, rtol=2e-6, atol=2e-7)
        np.testing.assert_allclose(e.cpu().double().numpy(), e64, rtol=2e-6, atol=2e-7)


def test_flat_adam_ema_state_dict_roundtrip_is_bit_exact():
    from fira_icse_b200.optim import FlatAdam
    a = _params(1)
    groups = lambda ps: [[ps[0], ps[2]], [ps[1], ps[3]]]               # noqa: E731
    opt_a = FlatAdam(a, lr=LR, groups=groups(a), ema_decay=0.9)
    for step in range(10):
        _set_grads(a, _grads(step, a))
        opt_a.step()
    sd = opt_a.state_dict()
    assert sd["ema_decay"] == 0.9 and len(sd["ema"]) == len(a)
    b = [torch.nn.Parameter(q.detach().clone()) for q in a]
    opt_b = FlatAdam(b, lr=LR, groups=groups(b), ema_decay=0.5)
    opt_b.load_state_dict(sd)
    assert opt_b.ema_decay == 0.9
    for step in range(10, 20):
        grads = _grads(step, a)
        _set_grads(a, grads)
        _set_grads(b, grads)
        opt_a.step()
        opt_b.step()
    torch.cuda.synchronize()
    for k in ("p", "m", "v", "ema", "p16", "step_t"):
        assert torch.equal(getattr(opt_a, k), getattr(opt_b, k)), k


def test_flat_adam_without_ema_keeps_its_state_dict():
    from fira_icse_b200.optim import FlatAdam
    a = _params(2)
    opt = FlatAdam(a, lr=LR)
    assert opt.ema is None
    assert list(opt.state_dict()) == ["step", "lr", "betas", "eps", "exp_avg", "exp_avg_sq"]
    with pytest.raises(ValueError, match="ema_decay"):
        FlatAdam(_params(3), lr=LR, ema_decay=1.0)


# ============================================================================= the engine
def _hosts():
    from fira_icse_b200.packed import PackedTables, pack_from_dataset
    from test_packed import GoldenSplit, V
    tables = PackedTables(GoldenSplit())
    eight = [pack_from_dataset(tables, np.arange(lo, lo + 8), V) for lo in (0, 16)]
    six = [pack_from_dataset(tables, np.arange(lo, lo + 6), V) for lo in (40, 64)]
    assert eight[0].shape_key != six[0].shape_key
    return [eight[0], six[0], eight[1], six[1]]


def _engine(mode, monkeypatch, d, precision="bf16"):
    from fira_icse_b200.engine import GraphedTrainStep
    from fira_icse_b200.optim import FlatAdam
    if mode == "single_opt":
        monkeypatch.setenv("FIRA_OPT_OVERLAP", "0")
    else:
        monkeypatch.delenv("FIRA_OPT_OVERLAP", raising=False)
    m = copy.deepcopy(seeded_model()).to(DEV)
    m.train()
    m.set_precision(precision)
    init = {id(p): p.detach().cpu().double() for p in m.parameters()}
    eng = GraphedTrainStep(m, 8, lambda ps: FlatAdam(ps, lr=LR, groups=m.flat_groups(), ema_decay=d),
                           edge_capacity=65536, split=True if mode == "split" else None)
    return m, eng, init


def _flat(eng, name):
    return torch.cat([getattr(o, name) for o in eng.flat_optims]).cpu().double().numpy()


@pytest.mark.parametrize("mode", ["overlap", "single_opt", "split"])
def test_engine_ema_is_the_recurrence_over_the_trajectory(mode, monkeypatch):
    """every replay's fira_adam_flat launches update the EMA: after each step the flat parameters are copied to the host,
    and the final EMA equals e_k = d e_{k-1} + fl32(c p_k) from e_0 = the initial parameters"""
    d = 0.9
    m, eng, init = _engine(mode, monkeypatch, d)
    hosts = [pb.to(DEV) for pb in _hosts()]
    steps = 10
    e = scale = None
    for k in range(steps):
        ls, nt = eng.step(hosts[k % len(hosts)])
        assert np.isfinite((ls / nt).item())
        if e is None:                                             # the optimizers exist now: lay e_0 out like them
            parts = []
            for o in eng.flat_optims:
                x = torch.zeros(o.n, dtype=torch.float64)
                for p, off in zip(o.params, o.offsets):
                    x[off:off + p.numel()] = init[id(p)].reshape(-1)
                parts.append(x)
            e = torch.cat(parts).numpy()
            scale = np.abs(e)
        p = _flat(eng, "p")
        e = ema_rule.ema(e, p, d)
        scale = np.maximum(scale, np.abs(p))
    assert len(eng.captured) >= 2 and (len(eng.flat_optims) == (1 if mode == "single_opt" else 2))
    got = _flat(eng, "ema")
    err = np.abs(got - e)
    tol = (steps + 1) * 2.0 ** -24 * (np.abs(e) + scale)
    assert np.all(err <= tol), float(np.max(err / np.maximum(tol, 1e-300)))
    moved = np.abs(got - _flat(eng, "p"))                         # the average lags the parameters
    assert float(moved.max()) > 1e-5


# ============================================================================= the shadow model
def _fresh(shadow, precision):
    from fira_icse_b200 import TransModel
    f = TransModel(reference_args())
    f.load_state_dict({k: v.cpu() for k, v in shadow.state_dict().items()})
    return f.to(DEV).eval().set_precision(precision)


def _dev_and_loss(model, b):
    with torch.no_grad():
        ids = model(*b, "dev")
        ls, nt = model(*b, "train")
    return ids, (ls / nt).item()


def test_shadow_model_follows_the_graphed_steps(monkeypatch):
    from fira_icse_b200 import decode_loop, optim
    from fira_icse_b200.sample import score
    m, eng, _ = _engine("overlap", monkeypatch, 0.5)
    hosts = [pb.to(DEV) for pb in _hosts()]
    with pytest.raises(RuntimeError, match="first step"):
        eng.ema_model()
    for k in range(4):
        eng.step(hosts[k % len(hosts)])
    shadow = eng.ema_model()
    assert eng.ema_model() is shadow                                # built once
    keys = list(m.state_dict())
    assert list(shadow.state_dict()) == keys and len(keys) == 338
    assert not shadow.training and shadow.precision == "bf16"
    assert not any(p.requires_grad for p in shadow.parameters())
    spans = [(o.ema.data_ptr(), o.ema.data_ptr() + 4 * o.n) for o in eng.flat_optims]
    live = {id(p) for p in m.live_parameters()}
    for (name, p), q in zip(m.named_parameters(), shadow.parameters()):
        if id(p) in live:
            assert any(lo <= q.data_ptr() < hi for lo, hi in spans), name
        else:
            assert torch.equal(q, p) and q.data_ptr() != p.data_ptr(), name
    kv = optim.cat_rows([t for c in shadow.decoder.cross_attention_list for t in (c.fc_k.weight, c.fc_v.weight)])
    assert kv.data_ptr() == shadow.decoder.cross_attention_list[0].fc_k.weight.data_ptr()     # one view of the EMA

    raw = load_raw_golden()
    vocab = raw["word_vocab"]
    ids = dict(tar_len=30, start_id=vocab["<start>"], eos_id=vocab["<eos>"], pad_id=vocab["<pad>"])
    b = [t.to(DEV) for t in golden_batch(0, 8)]
    losses = []
    for rnd in range(2):
        got_ids, got_loss = _dev_and_loss(shadow, b)
        ref_ids, ref_loss = _dev_and_loss(_fresh(shadow, "bf16"), b)
        assert torch.equal(got_ids, ref_ids), (rnd, float((got_ids != ref_ids).float().mean()))
        assert abs(got_loss - ref_loss) <= 5e-3 * abs(ref_loss), (rnd, got_loss, ref_loss)
        losses.append(got_loss)
        for k in range(4):                                          # the shadow must follow these steps
            eng.step(hosts[k % len(hosts)])
    assert abs(losses[1] - losses[0]) > 5e-3 * abs(losses[0]), losses      # the comparison above could see a stale model

    # sample.score keeps weight caches keyed on weights_key: score, step, score again against a freshly loaded model
    shadow.set_precision("fp32")
    before = score(shadow, b[0], b[3], b[4], b[5], b[7], b[6], **ids)
    for k in range(4):
        eng.step(hosts[k % len(hosts)])
    after = score(shadow, b[0], b[3], b[4], b[5], b[7], b[6], **ids)
    fresh = _fresh(shadow, "fp32")
    ref = score(fresh, b[0], b[3], b[4], b[5], b[7], b[6], **ids)
    assert torch.equal(after.length, ref.length)
    np.testing.assert_allclose(after.logprob.cpu().numpy(), ref.logprob.cpu().numpy(), rtol=0, atol=1e-3)
    assert float((after.logprob - before.logprob).abs().max()) > 1e-2
    # decoding loops hold their models (decode_loop._LOOPS): release them, with their captured graphs
    decode_loop.drop_loops(shadow)
    decode_loop.drop_loops(fresh)


def test_ema_model_needs_an_ema_for_every_live_parameter():
    from fira_icse_b200 import optim
    from fira_icse_b200.optim import FlatAdam
    m = copy.deepcopy(seeded_model()).to(DEV)
    live = m.live_parameters()
    half = len(live) // 2
    o1 = FlatAdam(live[:half], lr=LR, ema_decay=0.9)
    o2 = FlatAdam(live[half:], lr=LR)
    with pytest.raises(ValueError, match="no optimizer with an EMA"):
        optim.ema_model(m, [o1, o2])
    shadow = optim.ema_model(m, [o1, FlatAdam(live[half:], lr=LR, ema_decay=0.9)])
    for p, q in zip(m.parameters(), shadow.parameters()):
        assert torch.equal(p, q)                                    # no step yet: the average is the weights


# ============================================================================= run_model.py train
def _train_dir(tmp_path_factory, name, **extra):
    from test_data import _write_dataset
    from test_gpu_cli import _run_model
    d = tmp_path_factory.mktemp(name)
    _write_dataset(str(d), load_raw_golden())
    env = dict(os.environ, PYTHONPATH=ROOT, FIRA_EPOCHS="16", FIRA_BATCH="16", FIRA_MAX_BATCHES="1",
               FIRA_WORKERS="0", FIRA_TEST_BATCH="4")
    env.pop("FIRA_EMA", None)
    env.update(extra)
    return d, env, _run_model("train", d, env)


def test_run_model_train_with_ema_then_test(tmp_path_factory):
    from test_gpu_cli import _run_model
    d, env, _ = _train_dir(tmp_path_factory, "cli_ema", FIRA_EMA="0.99")
    for f in ("best_model.pt", "best_model_ema.pt", "OUTPUT/dev_output", "OUTPUT/dev_output_ema"):
        assert os.path.exists(d / f), f
    lines = open(d / "OUTPUT" / "train_process").read().splitlines()
    assert [ln for ln in lines if ln.startswith("epoch: 15 batch: 0 dev bleu:")], lines
    assert [ln for ln in lines if ln.startswith("ema epoch: 15 batch: 0 dev bleu:")], lines
    n_valid = len(json.load(open(d / "all_index"))["valid"])
    assert len(open(d / "OUTPUT" / "dev_output_ema").read().splitlines()) == n_valid
    sd = torch.load(d / "best_model_ema.pt", map_location="cpu")
    raw_sd = torch.load(d / "best_model.pt", map_location="cpu")
    assert list(sd) == list(raw_sd) and len(sd) == 338
    assert any(not torch.equal(sd[k], raw_sd[k]) for k in sd)        # the average is not the trained weights
    env_test = dict(env, FIRA_DECODE="nbest", FIRA_CHECKPOINT="best_model_ema.pt")
    env_test.pop("FIRA_EMA")
    r = _run_model("test", d, env_test)
    assert "mean sentence bleu" in r.stdout
    n_test = len(json.load(open(d / "all_index"))["test"])
    assert len(open(d / "OUTPUT" / "output_fira_nbest").read().splitlines()) == 3 * n_test


def test_run_model_train_without_ema_writes_no_ema_file(tmp_path_factory):
    d, _, _ = _train_dir(tmp_path_factory, "cli_no_ema")
    assert os.path.exists(d / "best_model.pt") and os.path.exists(d / "OUTPUT" / "dev_output")
    assert not os.path.exists(d / "best_model_ema.pt") and not os.path.exists(d / "OUTPUT" / "dev_output_ema")
    assert not any(ln.startswith("ema") for ln in open(d / "OUTPUT" / "train_process").read().splitlines())
