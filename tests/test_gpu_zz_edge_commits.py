"""Whole-path parity on the GPU for the edge-case fixture (tests/golden/make_golden_edge.py): the DataSet's extreme
commits and crafted commits that reach the truncation branches, against the outputs of the unmodified reference
(tests/golden/model_edge.npz); fp32 parity mode, 1e-4 relative."""
import numpy as np
import pytest
import torch

from fira_testlib import seeded_model

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
RTOL = 1e-4


@pytest.fixture(scope="module")
def model():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import copy
    m = copy.deepcopy(seeded_model()).to(DEV)
    m.eval()
    return m


def test_loss_matches_reference_on_extreme_and_truncated_commits(model):
    """tests/golden/make_golden_edge.py: longest diff, most AST / edit / sub-token nodes, commits without AST nodes,
    edit nodes or sub-tokens, and crafted commits cut by the 210 / 30 truncation; reference outputs in model_edge.npz"""
    import os
    import fira_oracle as O
    from fira_testlib import GOLDEN, load_edge_golden
    _, g = load_edge_golden()
    ref = np.load(os.path.join(GOLDEN, "model_edge.npz"))
    n = len(g["sou"])
    t = lambda k: torch.from_numpy(g[k].astype(np.int64)).to(DEV)
    ptr = g["edge_ptr"]
    dense = torch.stack([O.dense_adjacency(g["edge_row"][ptr[i]:ptr[i + 1]], g["edge_col"][ptr[i]:ptr[i + 1]],
                                           g["edge_val"][ptr[i]:ptr[i + 1]]) for i in range(n)]).to(DEV)   # input only
    batch = [t("sou"), t("tar"), t("attr"), t("mark"), t("ast_change"), dense, t("tar_label"), t("sub_token")]
    with torch.no_grad():
        loss_sum, n_tok = model(*batch, "train")
        one = [model(*[b[i:i + 1] for b in batch], "train")[0].item() for i in range(n)]
        ids = model(*batch, "dev").cpu().numpy()
    assert int(n_tok) == int(ref["mask_sum"])
    assert abs(loss_sum.item() - float(ref["loss_sum"])) <= RTOL * float(ref["loss_sum"])
    np.testing.assert_allclose(np.array(one), ref["loss_per_commit"], rtol=RTOL)
    # argmax ids: identical to the reference, except at positions that are TIES at fp32 resolution in the fp32
    # reference distribution itself (random-initialised weights give near-uniform rows): there the log-probability
    # of the id picked here must equal the reference's top-1 log-probability to within fp32 round-off of the
    # 25,020-wide softmax (|logp| ~ 10, one ulp ~ 1e-6)
    bad = np.argwhere(ids != ref["argmax_ids"])
    if len(bad):
        sd = {k: v.detach().cpu() for k, v in model.state_dict().items()}
        detail = {}
        with torch.no_grad():
            O.forward(sd, *[b.cpu() for b in batch], stage="train", detail=detail)
        logp = detail["logp"]
        for i, t in bad:
            gap = float(logp[i, t, int(ref["argmax_ids"][i, t])] - logp[i, t, int(ids[i, t])])
            assert abs(gap) <= 4e-6, f"commit {i} position {t}: not a tie (log-prob gap {gap:.3e})"
    assert len(bad) <= 2, "argmax ids differ from the reference at more than two (tied) positions"
