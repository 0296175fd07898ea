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


# ------------------------------------------------------------------------------------ accumulating / register epilogue
def _c0(ab, c_dtype, seed):
    """an existing C: odd rows nearly cancel A B (there C0 + A B is far smaller than A B, so an epilogue that rounds A B
    before adding C0, or drops C0, is off by much more than one rounding of the sum), even rows are independent of it"""
    g = torch.Generator().manual_seed(seed)
    noise = torch.randn(ab.shape, generator=g, dtype=torch.float64).to(DEV)
    c0 = noise * ab.abs().max() / 4
    c0[1::2] = -ab[1::2] + noise[1::2] * 0.01
    return c0.to(c_dtype)


def close_acc(out, ref, ab, c16):
    """|out - ref| <= e |ref| + 1e-4 max|AB| + 1e-6 element-wise, ref = C0 + A B (+ terms) in float64 on the stored
    operands.  1e-4 max|AB| is this file's fp32 summation bound; e = 2^-8 for bf16 C (the sum is rounded to bf16 once:
    2^-9 of it, 2^-8 leaves room for the fp32 error it carries -- the convention of test_gpu_ops_bf16.close16), 2^-22
    for fp32 C (the fp32 adds of C0, bias and rank-1 term)."""
    out, ref = out.double(), ref.double()
    bound = (2.0 ** -8 if c16 else 2.0 ** -22) * ref.abs() + 1e-4 * ab.abs().max().item() + 1e-6
    bad = (out - ref).abs() > bound
    assert not bad.any(), f"{int(bad.sum())} elements off, worst {((out - ref).abs() - bound).max().item():.3e} over the bound"


def _dx_operands(M, N, K, seed=1):
    """the linear_dx form: A = dY [M, K] K-major, B = W [K, N] MN-major stored with a leading dimension of ceil8(N)"""
    ldw = (N + 7) // 8 * 8
    A = rnd(M, K, seed=seed)
    Wst = torch.zeros(K, ldw, device=DEV, dtype=torch.bfloat16)
    Wst[:, :N] = rnd(K, N, seed=seed + 1)
    return A, Wst, ldw, A.double() @ Wst[:, :N].double()


@pytest.mark.parametrize("M,N,K,c16,ldc,terms", [
    # pr.linear_dx(..., accumulate=True) of the training step, bf16 C and fp32 C
    (1920, 256, 1024, True, 256, ""), (1920, 256, 768, True, 256, ""), (3000, 256, 512, True, 256, ""),
    (1920, 256, 1024, False, 256, ""), (3000, 256, 512, False, 256, ""),
    # tails: rows; 72 columns (vector path, partial tile); 300 columns, ldc = 300 (bf16: scalar path)
    (333, 256, 1024, True, 256, ""), (1920, 72, 256, True, 72, ""), (1920, 300, 512, True, 300, ""),
    (333, 300, 256, False, 300, ""),
    # fp32 C with ldc % 4 != 0 (scalar path)
    (333, 300, 256, False, 301, ""), (1920, 256, 768, False, 257, ""),
    # bias and rank-1 terms with accumulate
    (1920, 256, 1024, True, 256, "bias"), (333, 300, 512, True, 300, "rank1"), (700, 72, 256, False, 75, "bias+rank1"),
])
def test_accumulate_input_grad(M, N, K, c16, ldc, terms):
    """C = C0 + A B (+ bias, + rs rc) with accumulate=1 on A K-major x B MN-major; columns >= N of C untouched"""
    from fira_icse_b200 import ops as o
    A, Wst, ldw, ab = _dx_operands(M, N, K)
    g = torch.Generator().manual_seed(7)
    b = torch.randn(N, generator=g).to(DEV) if "bias" in terms else None
    rs = torch.randn(M, generator=g).to(DEV) if "rank1" in terms else None
    rc = torch.randn(N, generator=g).to(DEV) if "rank1" in terms else None
    cdt = torch.bfloat16 if c16 else torch.float32
    C = torch.full((M, ldc), 3.0, device=DEV, dtype=cdt)
    C[:, :N] = _c0(ab, cdt, seed=5)
    C0 = C.clone()
    o.gemm_tc(A, K, 1, Wst, ldw, 0, C, ldc, M, N, K, bias=b, rs=rs, rc=rc, accumulate=True)
    ref = C0[:, :N].double() + ab
    if b is not None:
        ref += b.double()
    if rs is not None:
        ref += rs.double()[:, None] * rc.double()[None]
    close_acc(C[:, :N], ref, ab, c16)
    assert torch.equal(C[:, N:], C0[:, N:])


@pytest.mark.parametrize("N,ldc_pad", [(300, 304), (260, 264), (5, 8)])
def test_bf16_register_epilogue_without_accumulate(N, ldc_pad):
    """bf16 C with ldc = N (not a multiple of 8) takes the register epilogue without accumulation: one rounding of
    A B + bias, bit for bit what the TMA-store epilogue writes for the same product into C with ldc_pad (a multiple of
    8); neither writes a column past N (N = 300: the tail shares a TMA box with full chunks, 260: the tail starts a box,
    5: fewer than 8 columns, register epilogue both times)"""
    from fira_icse_b200 import ops as o
    M, K = 333, 512
    A, Wst, ldw, ab = _dx_operands(M, N, K)
    b = torch.randn(N, generator=torch.Generator().manual_seed(7)).to(DEV)
    c = torch.full((M + 1, N), 3.0, device=DEV, dtype=torch.bfloat16)
    o.gemm_tc(A, K, 1, Wst, ldw, 0, c, N, M, N, K, bias=b)
    close_acc(c[:M], ab + b.double(), ab, True)
    assert (c[M] == 3.0).all()
    cp = torch.full((M, ldc_pad), 3.0, device=DEV, dtype=torch.bfloat16)
    o.gemm_tc(A, K, 1, Wst, ldw, 0, cp, ldc_pad, M, N, K, bias=b)
    assert torch.equal(c[:M], cp[:, :N])
    assert (cp[:, N:] == 3.0).all(), "columns past N were written"


@pytest.mark.parametrize("splits,ldc", [(1, 256), (2, 256), (8, 256), (2, 257), (8, 259)])
def test_accumulate_split_k_bias_once(splits, ldc):
    """fp32 C, accumulate=1, split-K: no zero-fill, the partials add onto C0, bias and rank-1 term land once (first
    split only); ldc % 4 != 0 takes the scalar atomics"""
    from fira_icse_b200 import ops as o
    M, N, K = 700, 256, 1024
    A, Wst, ldw, ab = _dx_operands(M, N, K)
    g = torch.Generator().manual_seed(7)
    b, rs, rc = torch.randn(N, generator=g).to(DEV), torch.randn(M, generator=g).to(DEV), torch.randn(N, generator=g).to(DEV)
    C = torch.full((M, ldc), 3.0, device=DEV)
    C[:, :N] = _c0(ab, torch.float32, seed=5)
    C0 = C.clone()
    o.gemm_tc(A, K, 1, Wst, ldw, 0, C, ldc, M, N, K, bias=b, rs=rs, rc=rc, accumulate=True, splits=splits)
    ref = C0[:, :N].double() + ab + b.double() + rs.double()[:, None] * rc.double()[None]
    close_acc(C[:, :N], ref, ab, False)
    assert torch.equal(C[:, N:], C0[:, N:])


@pytest.mark.parametrize("c16", [True, False])
def test_relu_with_accumulate(c16):
    """relu applies to the product before it is accumulated: C += relu(A B + bias) (include/fira_b200.h)"""
    from fira_icse_b200 import ops as o
    M, N, K = 333, 256, 512
    A, Wst, ldw, ab = _dx_operands(M, N, K)
    b = torch.randn(N, generator=torch.Generator().manual_seed(7)).to(DEV)
    cdt = torch.bfloat16 if c16 else torch.float32
    C = _c0(ab, cdt, seed=5)
    C0 = C.clone()
    o.gemm_tc(A, K, 1, Wst, ldw, 0, C, N, M, N, K, bias=b, relu=True, accumulate=True)
    close_acc(C, C0.double() + torch.relu(ab + b.double()), ab, c16)
