"""The training step with dropout ON against the float64 oracle run with the masks the kernels draw (tests/philox_rule.py
through the oracle's `masks` hook): fp32 parity mode on padded and packed batches (loss and every live parameter's full
gradient), the bf16 mode with the default and the fused GCN layer, CUDA-graph replays (seed + the replay's counter),
and the blocks.py module surface.  The seeds are the ones ops.make_seed hands out, recorded by a fixture of this file."""
import copy

import numpy as np
import pytest
import torch

import philox_rule as R
from fira_testlib import golden_batch, seeded_model

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
P_ENC, P_GCN, P_DEC = 0.1, 0.2, 0.1                 # Combination / GCN / decoder dropout of the reference model
SEED = 20240607
PADDED = (0, 8)
PACKED_INDEX = [100, 3, 77, 127, 64, 9]             # tests/test_gpu_packed.py
_ORACLE = {}


@pytest.fixture(scope="module", autouse=True)
def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


class SeedRecorder:
    """ops.make_seed, recording every seed it hands out (in call order)"""

    def __init__(self, make_seed):
        self.make_seed, self.seeds = make_seed, []

    def __call__(self):
        s = self.make_seed()
        self.seeds.append(s)
        return s


@pytest.fixture
def seeds(monkeypatch):
    from fira_icse_b200 import ops
    rec = SeedRecorder(ops.make_seed)
    monkeypatch.setattr(ops, "make_seed", rec)
    return rec


def model_masks(enc_seed, dec_seed, ctr=0, row_map=None):
    """the oracle's `masks` for one TransModel forward: encoder streams < 64 (GCN LayerNorm: site 2, p = 0.2) keyed by the
    encoder's seed, decoder streams keyed by the decoder's; row_map maps the oracle's padded node rows to the kernels'
    rows (-1: a padding node the kernels do not hold -- its mask reaches no real row)"""
    def masks(sid, rows):
        shape = tuple(rows.shape)
        r = rows.reshape(-1).numpy()
        if sid < R.DEC_OFFSET:
            seed, p = enc_seed, (P_GCN if sid % R.LAYER_STRIDE == R.ENC_SITE["gcn_ln"] else P_ENC)
            if row_map is not None:
                r = row_map[r]
        else:
            seed, p = dec_seed, P_DEC
        k = R.keep_mask(seed, ctr, sid, np.maximum(r, 0), p)
        k[r < 0] = True
        return torch.from_numpy(k).view(*shape, R.D)
    return masks


def packed_row_map(pb, B, n):
    """segment-major padded node row -> row of the packed buffer (packed.PackedBatch.off), -1 for dropped padding"""
    off = pb.off.cpu().numpy()
    base = (0, pb.Rc, pb.Rc + pb.Rs)
    out = []
    for s in range(3):
        for b in range(B):
            j = np.arange(n[s])
            u = off[s][b + 1] - off[s][b]
            out.append(np.where(j < u, base[s] + off[s][b] + j, -1))
    return np.concatenate(out)


def oracle(model, batch, masks, key=None, grad=True):
    """float64 oracle loss (and gradients by autograd on a float64 copy of the state dict) under `masks`"""
    import fira_oracle as O
    if key is not None and key in _ORACLE:
        return _ORACLE[key]
    sd = {k: v.detach().cpu().double().requires_grad_(grad) for k, v in model.state_dict().items()}
    with torch.set_grad_enabled(grad):
        loss_sum, n_tok = O.forward(sd, *batch, stage="train", training=True, masks=masks)
        loss = loss_sum / n_tok
        if grad:
            loss.backward()
    grads = {}
    if grad:
        for k, v in sd.items():
            g = v.grad
            if g is not None and k in ("encoder.embedding.weight", "encoder.ast_change_embedding.weight",
                                       "encoder.mark_embedding.weight"):
                g = g.clone()
                g[0] = 0.0                               # padding_idx = 0 (gnn_transformer.py:36-39)
            grads[k] = g
    res = (float(loss.detach()), grads)
    if key is not None:
        _ORACLE[key] = res
    return res


def run_model(model, fn, seeds):
    """one training forward + backward; -> (loss, {name: grad}, (encoder seed, decoder seed))"""
    model.zero_grad(set_to_none=True)
    n0 = len(seeds.seeds)
    torch.manual_seed(SEED)                             # the same seeds for every precision mode
    ls, nt = fn()
    (ls / nt).backward()
    torch.cuda.synchronize()
    drawn = seeds.seeds[n0:]
    assert len(drawn) == 2, drawn                       # one seed per encoder forward, one per decoder forward
    return (ls / nt).item(), {k: p.grad for k, p in model.named_parameters() if p.grad is not None}, tuple(drawn)


def check_fp32(model, loss, grads, ref_loss, ref_grads):
    """the bounds of test_gpu_model.py::test_gradients_match_reference, on every element"""
    assert abs(loss - ref_loss) <= 1e-4 * abs(ref_loss), (loss, ref_loss)
    assert sorted(grads) == sorted(k for k, g in ref_grads.items() if g is not None)
    for p in model.dead_parameters():
        assert p.grad is None
    worst = 0.0
    for k, g in grads.items():
        ref = ref_grads[k]
        norm = ref.norm().item()
        g = g.double().cpu()
        if norm < 1e-7:                 # fc_k.bias, LinearRes.bias: zero in exact arithmetic (softmax shift invariance)
            assert g.norm().item() < 1e-6, k
            continue
        err = abs(g.norm().item() - norm) / norm
        worst = max(worst, err)
        assert err <= 5e-4, (k, err)
        bound = 1e-7 + 5e-4 * norm + 5e-3 * ref.abs()
        over = (g - ref).abs() - bound
        assert not (over > 0).any(), f"{k}: {int((over > 0).sum())} of {g.numel()} elements off, worst {over.max():.3e}"
    print("worst gradient-norm rel err", worst)


def _padded_batch(lo, hi):
    return golden_batch(lo, hi)


@pytest.fixture(scope="module")
def base_model():
    m = copy.deepcopy(seeded_model()).to(DEV)
    m.train()
    return m


def test_fp32_padded_matches_oracle_with_the_kernels_masks(base_model, seeds):
    batch = _padded_batch(*PADDED)
    dev = [b.to(DEV) for b in batch]
    loss, grads, (se, sd) = run_model(base_model, lambda: base_model(*dev, "train"), seeds)
    ref_loss, ref_grads = oracle(base_model, batch, model_masks(se, sd), key=("padded", se, sd))
    check_fp32(base_model, loss, grads, ref_loss, ref_grads)


def test_fp32_packed_matches_oracle_with_the_kernels_masks(base_model, seeds):
    from fira_icse_b200.packed import PackedTables, pack_from_dataset
    from test_packed import GoldenSplit, V
    pb = pack_from_dataset(PackedTables(GoldenSplit()), np.asarray(PACKED_INDEX), V).to(DEV)
    parts = [golden_batch(i, i + 1) for i in PACKED_INDEX]
    batch = [torch.cat([p[k] for p in parts], 0) for k in range(8)]
    loss, grads, (se, sd) = run_model(base_model, lambda: base_model.forward_packed(pb, "train"), seeds)
    B = len(PACKED_INDEX)
    row_map = packed_row_map(pb, B, (batch[0].shape[1], batch[7].shape[1], batch[4].shape[1]))
    ref_loss, ref_grads = oracle(base_model, batch, model_masks(se, sd, row_map=row_map))
    check_fp32(base_model, loss, grads, ref_loss, ref_grads)


@pytest.mark.parametrize("fused", ["0", "1"], ids=["default_gcn", "fused_gcn"])
def test_bf16_tracks_oracle_with_the_kernels_masks(base_model, seeds, monkeypatch, fused):
    """the loss and every gradient element (embedding gradients also row by row) within the whole-step bound of
    tests/test_gpu_bf16_step.py; the exact masks of the bf16 kernels are checked in tests/test_gpu_dropout_rule.py"""
    from test_gpu_bf16_step import check_step, record_gates
    monkeypatch.setenv("FIRA_GCN_FUSED", fused)
    m = copy.deepcopy(base_model).set_precision("bf16")
    batch = _padded_batch(*PADDED)
    dev = [b.to(DEV) for b in batch]
    loss, grads, (se, sd) = run_model(m, lambda: m(*dev, "train"), seeds)
    gates = {}
    record_gates(monkeypatch, gates)                    # a fresh oracle run: it records the FFN gates of the allowance
    ref_loss, ref_grads = oracle(base_model, batch, model_masks(se, sd))
    check_step(f"padded/gcn_fused{fused}", loss, grads, ref_loss, ref_grads, gates)


def test_graph_replays_use_seed_plus_replay_counter(seeds):
    """each replay of the captured step keys its masks by the seeds frozen into the graph at capture plus the device
    counter the replay bumped (engine.GraphedTrainStep._forward_backward adds 1 before the forward): the loss of two
    replays and the gradients of the first against the oracle under those masks"""
    from fira_icse_b200 import PackedEdges
    from fira_icse_b200.engine import GraphedTrainStep
    m = copy.deepcopy(seeded_model()).to(DEV)
    m.train()
    eng = GraphedTrainStep(m, 4, lambda ps: torch.optim.Adam(ps, lr=0.0, fused=True, capturable=True))
    batch = golden_batch(0, 4)
    b = golden_batch(0, 4, dense_edge=False)
    b[5] = PackedEdges.from_coo_lists(b[5], 650, DEV)
    b = [x.to(DEV) if torch.is_tensor(x) else x for x in b]
    eng.load(b)
    eng.capture()
    se, sd = seeds.seeds[-2:]                           # the forward recorded into the graph: encoder, then decoder
    losses = []
    for rep in range(2):
        ls, n = eng.step(b)
        loss = (ls / n).item()
        ctr = int(eng.seed_ctr.item())
        ref, ref_grads = oracle(m, batch, model_masks(se, sd, ctr=ctr), grad=rep == 0)
        assert abs(loss - ref) <= 1e-4 * abs(ref), (ctr, loss, ref)
        if rep == 0:                                    # lr = 0: the parameters stay those of the oracle's state dict
            grads = {k: p.grad for k, p in m.named_parameters() if p.grad is not None}
            check_fp32(m, loss, grads, ref, ref_grads)
        losses.append(loss)
    assert abs(losses[0] - losses[1]) > 1e-3 * abs(losses[0]), losses     # the check can tell the masks apart


# ------------------------------------------------------------------------------------ blocks.py in train mode
def _block_masks(seed_by_sid, p):
    def masks(sid, rows):
        shape = tuple(rows.shape)
        k = R.keep_mask(seed_by_sid[sid], 0, sid, rows.reshape(-1).numpy(), p)
        return torch.from_numpy(k).view(*shape, R.D)
    return masks


def _sd64(module, prefix="m"):
    return {f"{prefix}.{k}": v.detach().cpu().double().requires_grad_(True) for k, v in module.state_dict().items()}


def _check_block(out, ref, inputs, refs, sd, module, prefix="m"):
    """forward and the gradients of the inputs and parameters (fp32 kernels against float64)"""
    def close(a, b, what):
        a, b = a.detach().double().cpu(), b.detach().double()
        err, scale = (a - b).abs().max().item(), b.abs().max().item()
        assert err <= 1e-5 + 1e-4 * scale, f"{what}: max err {err:.3e}, scale {scale:.3e}"
    close(out, ref, "output")
    g = torch.randn(out.shape, generator=torch.Generator().manual_seed(9))
    out.backward(g.to(DEV))
    ref.backward(g.double())
    for i, (x, xr) in enumerate(zip(inputs, refs)):
        close(x.grad, xr.grad, f"input {i} gradient")
    for k, p in module.named_parameters():
        close(p.grad, sd[f"{prefix}.{k}"].grad, f"{k} gradient")


def _leaf(t):
    return t.to(DEV).requires_grad_(True), t.double().requires_grad_(True)


def test_blocks_train_mode_match_oracle_blocks(seeds):
    import fira_oracle as O
    from fira_icse_b200.blocks import combination_layer_forward
    from fira_icse_b200.modules import GCN, Attention, Combination, FeedForward
    torch.manual_seed(3)
    g = torch.Generator().manual_seed(4)
    B, L, Lk = 3, 47, 29

    # Combination: gate (stream 0) and LayerNorm (stream 1) each draw their own seed
    m = Combination(8, 256).to(DEV).train()
    x, x64 = _leaf(torch.randn(B, L, 256, generator=g))
    v, v64 = _leaf(torch.randn(B, L, 256, generator=g))
    n0 = len(seeds.seeds)
    out = m(x, x, v)
    s = seeds.seeds[n0:]
    assert len(s) == 2
    sd = _sd64(m)
    ref = O.combination(sd, "m", x64, v64, 8, 0.1, True, masks=_block_masks({0: s[0], 1: s[1]}, 0.1), sid=0)
    _check_block(out, ref, (x, v), (x64, v64), sd, m)

    # GCN on real commits (the block keeps the reference's (b, node) row order: rows b * 650 + j), stream 2, p = 0.2
    m = GCN(256, dropout_rate=0.2).to(DEV).train()
    adj = golden_batch(0, 2)[5]
    h, h64 = _leaf(torch.randn(2, 650, 256, generator=g))
    n0 = len(seeds.seeds)
    parts = m(h, adj.to(DEV), 210, 160, 280)
    s = seeds.seeds[n0:]
    assert len(s) == 1
    out = torch.cat(parts, 1)
    sd = _sd64(m)
    ref = O.gcn(sd, "m", h64, adj, 0.2, True, masks=_block_masks({2: s[0]}, 0.2), sid=2)
    _check_block(out, ref, (h,), (h64,), sd, m)

    # Attention with a key-padding mask (decoder-length queries: the fp32 attention kernel takes Lq <= 32), stream 0
    m = Attention(256, 8).to(DEV).train()
    q, q64 = _leaf(torch.randn(B, 30, 256, generator=g))
    mem, mem64 = _leaf(torch.randn(B, Lk, 256, generator=g))
    key_mask = torch.rand(B, Lk, generator=g) > 0.3
    key_mask[:, 0] = True
    n0 = len(seeds.seeds)
    out = m(q, mem, mem, key_mask.to(DEV))
    s = seeds.seeds[n0:]
    sd = _sd64(m)
    ref = O.attention(sd, "m", q64, mem64, key_mask, 8, 0.1, True, masks=_block_masks({0: s[0]}, 0.1), sid=0)
    _check_block(out, ref, (q, mem), (q64, mem64), sd, m)

    # FeedForward, stream 2
    m = FeedForward(256).to(DEV).train()
    x, x64 = _leaf(torch.randn(B, L, 256, generator=g))
    n0 = len(seeds.seeds)
    out = m(x)
    s = seeds.seeds[n0:]
    sd = _sd64(m)
    ref = O.feed_forward(sd, "m", x64, 0.1, True, masks=_block_masks({2: s[0]}, 0.1), sid=2)
    _check_block(out, ref, (x,), (x64,), sd, m)

    # CombinationLayer with 32-wide heads: 8 heads share one 256-wide kernel row (stream 0); 7 x 5 heads pad the last row
    drop = torch.nn.Dropout(0.1).train()
    q, q64 = _leaf(torch.randn(7, 5, 32, generator=g))
    k, k64 = _leaf(torch.randn(7, 5, 32, generator=g))
    v, v64 = _leaf(torch.randn(7, 5, 32, generator=g))
    n0 = len(seeds.seeds)
    out = combination_layer_forward(q, k, v, drop)
    s = seeds.seeds[n0:]
    assert len(s) == 1
    n = 35
    rows = -(-n // 8)
    keep = torch.from_numpy(R.keep_mask(s[0], 0, 0, rows, 0.1)).view(-1, 32)[:n].view(7, 5, 32)
    w = torch.softmax(torch.stack((q64 * k64, q64 * v64), -1) / np.sqrt(32), -1)
    ref = (w[..., 0] * k64 + w[..., 1] * v64) * keep / (1 - float(np.float32(0.1)))
    _check_block(out, ref, (q, k, v), (q64, k64, v64), {}, torch.nn.Module())
