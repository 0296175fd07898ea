"""wgmma / TMA GEMM (fira_gemm_bf16_tc) against torch on the same bf16-rounded operands.
bf16 x bf16 products are exact in fp32, so only the fp32 summation order differs: tolerance 1e-4."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module", autouse=True)
def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def rnd(*shape, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*shape, generator=g).to(DEV).to(torch.bfloat16)


def close(a, b, rtol=1e-4):
    a, b = a.double(), b.double()
    err = (a - b).abs().max().item()
    assert err <= rtol * b.abs().max().item() + 1e-6, f"max err {err:.3e} (ref scale {b.abs().max().item():.3e})"


@pytest.mark.parametrize("M,N,K", [(128, 256, 256), (128, 64, 64), (1000, 256, 256), (41600, 256, 256),
                                   (1920, 1024, 256), (1920, 256, 1024), (300, 72, 200), (257, 3072, 256),
                                   (1920, 24650, 256)])
def test_kmajor_forward(M, N, K):
    from fira_icse_b200 import ops as o
    x, W = rnd(M, K, seed=1), rnd(N, K, seed=2)
    b = torch.randn(N, device=DEV)
    ref = x.float() @ W.float().T
    ldc = (N + 7) // 8 * 8
    c = torch.full((M, ldc), 3.0, device=DEV)
    o.gemm_tc(x, K, 1, W, K, 1, c, ldc, M, N, K)
    close(c[:, :N], ref)
    assert (c[:, N:] == 3.0).all()
    c16 = torch.empty((M, ldc), device=DEV, dtype=torch.bfloat16)
    o.gemm_tc(x, K, 1, W, K, 1, c16, ldc, M, N, K, bias=b, relu=True)
    close(c16[:, :N].float(), torch.relu(ref + b), rtol=1e-2)


def test_rank1_and_splitk():
    from fira_icse_b200 import ops as o
    M, N, K = 700, 256, 512
    x, W = rnd(M, K, seed=1), rnd(N, K, seed=2)
    b, rs, rc = torch.randn(N, device=DEV), torch.randn(M, device=DEV), torch.randn(N, device=DEV)
    ref = x.float() @ W.float().T + b + rs[:, None] * rc[None]
    c = torch.empty((M, N), device=DEV)
    o.gemm_tc(x, K, 1, W, K, 1, c, N, M, N, K, bias=b, rs=rs, rc=rc)
    close(c, ref)
    for s in (2, 3, 8):
        c = torch.full((M, N), 9.0, device=DEV)
        o.gemm_tc(x, K, 1, W, K, 1, c, N, M, N, K, bias=b, rs=rs, rc=rc, splits=s)
        close(c, ref)


@pytest.mark.parametrize("rows,N,K", [(1000, 256, 256), (41600, 256, 256), (1920, 1024, 256), (333, 72, 136),
                                      (1920, 512, 256)])
def test_mnmajor_weight_grad_and_input_grad(rows, N, K):
    """dW[N,K] = dY[rows,N]^T X[rows,K] (both operands MN-major, split over rows) and
    dX[rows,K] = dY[rows,N] W[N,K] (A K-major, B MN-major)."""
    from fira_icse_b200 import ops as o
    dy, x, W = rnd(rows, N, seed=1), rnd(rows, K, seed=2), rnd(N, K, seed=3)
    dW = torch.empty((N, K), device=DEV)
    o.gemm_tc(dy, N, 0, x, K, 0, dW, K, N, K, rows)
    close(dW, dy.float().T @ x.float())
    dW2 = torch.empty((N, K), device=DEV)
    o.gemm_tc(dy, N, 0, x, K, 0, dW2, K, N, K, rows, splits=37)
    close(dW2, dy.float().T @ x.float())
    dx = torch.empty((rows, K), device=DEV, dtype=torch.bfloat16)
    o.gemm_tc(dy, N, 1, W, K, 0, dx, K, rows, K, N)
    close(dx.float(), dy.float() @ W.float(), rtol=1e-2)


@pytest.mark.parametrize("rows,N,K,ld", [(1000, 256, 256, 256), (1920, 1024, 256, 1024), (333, 72, 136, 72), (1920, 768, 256, 768),
                                         (1920, 24650, 256, 24704), (11000, 3072, 256, 3072), (77, 256, 1024, 256)])
def test_weight_grad_with_folded_bias_grad(rows, N, K, ld):
    """fira_gemm_bf16_tc_dbias: dW = dY^T X and db += colsum(dY) from the same launch (dY tiles summed in shared memory)"""
    from fira_icse_b200 import ops as o
    dy = torch.zeros((rows, ld), device=DEV, dtype=torch.bfloat16)
    dy[:, :N] = rnd(rows, N, seed=1)
    x = rnd(rows, K, seed=2)
    pr = o.Prec(True)
    ref_w, ref_b = dy[:, :N].float().T @ x.float(), dy[:, :N].float().sum(0)
    for _ in range(2):                                   # the second pass checks nothing is left behind in the buffers
        dW = torch.full((N, K), 7.0, device=DEV)
        db = torch.zeros(N, device=DEV)
        pr.linear_dw(dy, ld, x, K, rows, N, K, out=dW, dbias=db)
        close(dW, ref_w)
        close(db, ref_b)


@pytest.mark.parametrize("rows,K,split,rank1,p", [(1920, 256, None, False, 0.0), (1920, 1024, None, False, 0.1), (300, 256, None, False, 0.0),
                                                  (11000, 256, 3500, True, 0.2), (333, 256, 100, True, 0.0), (128, 256, 0, False, 0.0)])
def test_gemm_ln_fused_equals_gemm_then_layernorm(rows, K, split, rank1, p):
    """fira_gemm_ln_fwd (one launch) against fira_gemm_bf16_tc + fira_ln_residual_fwd (the sequence it replaces): same z,
    same dropout masks, same statistics, same normalised rows in both outputs"""
    from fira_icse_b200 import ops as o
    D = 256
    x, W = rnd(rows, K, seed=1), rnd(D, K, seed=2) * 0.1
    resid = rnd(rows, D, seed=3)
    g = torch.Generator().manual_seed(4)
    b, gamma, beta = (torch.randn(D, generator=g).to(DEV) for _ in range(3))
    rs = torch.randn(rows, generator=g).to(DEV) if rank1 else None
    rc = torch.randn(D, generator=g).to(DEV) if rank1 else None
    pr = o.Prec(True)
    sp = rows if split is None else split
    seed, sid = 1234, 7

    def run(fused):
        o.FUSE_GEMM_LN = fused
        outA = torch.full((max(sp, 1), D), 5.0, device=DEV, dtype=torch.bfloat16)
        outB = torch.full((rows, D), 5.0, device=DEV, dtype=torch.bfloat16) if split is not None else outA
        z, st = pr.linear_ln(x, W.to(torch.bfloat16), b, resid, gamma, beta, outA, outB, sp, rows, p, seed, sid, rs=rs, rc=rc)
        torch.cuda.synchronize()
        return z.float(), st.clone(), outA.float(), outB.float()
    try:
        z1, s1, a1, b1 = run(True)
        z0, s0, a0, b0 = run(False)
    finally:
        o.FUSE_GEMM_LN = True
    close(z1, z0, rtol=1e-2)
    torch.testing.assert_close(s1, s0, rtol=2e-2, atol=2e-2)
    if sp > 0:
        close(a1[:sp], a0[:sp], rtol=2e-2)
    if split is not None:
        close(b1[sp:], b0[sp:], rtol=2e-2)
        assert (b1[:sp // 32 * 32] == 5.0).all()       # rows below the split's 32-row slab are not written to outB
    if split is not None and sp > 0:
        assert a1.shape[0] == sp


@pytest.mark.parametrize("rows,N,K", [(1920, 256, 1024), (300, 72, 200), (128, 64, 64)])
def test_input_grad_through_relu(rows, N, K):
    """fira_gemm_bf16_tc_dx_relu: dx = relu'(h) * (dy W) in one launch == the product followed by fira_relu_bwd"""
    from fira_icse_b200 import ops as o
    dy, W = rnd(rows, N, seed=1), rnd(N, K, seed=2)
    h = torch.relu(rnd(rows, K, seed=3))
    pr = o.Prec(True)
    try:
        o.FUSE_DX_RELU = True
        a = pr.linear_dx_relu(dy, N, W, rows, h).float()
        o.FUSE_DX_RELU = False
        b = pr.linear_dx_relu(dy, N, W, rows, h).float()
    finally:
        o.FUSE_DX_RELU = True
    ref = (dy.float() @ W.float()) * (h > 0)
    close(a, ref, rtol=1e-2)
    close(b, ref, rtol=1e-2)
    assert ((a == 0) == (b == 0)).all()
