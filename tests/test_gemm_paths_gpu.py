"""GPU: the strided fp32 GEMM (ops.sgemm) at PointWiseMLP's wide shapes and on every path of the wgmma 3xTF32 kernel,
per element against float64:  |C - C64| <= 1e-5 * (|A| |B|)_mn,  plus the max-normalised bar of test_gemm_gpu.py.

The tensor-core kernel's path is chosen on the host from the operands' strides and alignment (staging modes AV / BV,
gemm_tc.cuh:403-407), the tile width (WN 96 / 160, gemm_tc.cuh:408-412), the transposed orientation (swap,
gemm.cu:274) and, per output tile, the epilogue branch (gemm_tc.cuh:324-365).  tc_path() restates those predicates;
every case below states the path it is meant to take, and test_tc_cases_cover_every_path (CPU) asserts that the
table reaches each of them.
"""
import pytest
import torch

TOL = 1e-5
ALGOS = [0, 1, 2]  # CL3D_GEMM_AUTO, CL3D_GEMM_FFMA, CL3D_GEMM_TC3X
BM, BK, MAXN = 128, 16, 160     # kTcBM, kTcBK, kTcMaxN (gemm_tc.cuh:37-38)


def _cdiv(a, b):
    return -(-a // b)


def _padded(C):
    return (C + 7) & ~7


def _tile_n(N):                       # gemm_tc.cuh:111
    return MAXN if N >= MAXN else _cdiv(N, 32) * 32


def _tc_cost(M, N):                   # gemm.cu:263-266
    return _cdiv(M, BM) * _cdiv(N, MAXN) * (BM + _tile_n(N))


def tc_path(M, N, K, sa, sb, a_al, b_al, splitk, ldc, c_al):
    """(swap, AV, BV, WN, epilogue branches of the first warp's rows over all column tiles) of the tensor-core kernel
    for C (M x N, row stride ldc) = A (M x K, element strides sa = (m, k)) @ B (K x N, strides sb = (k, n));
    *_al: the operand / output address is 16-byte aligned.  Branches: 1 flat contiguous copy, 2 float4 rows,
    3 transposed (unit row stride), 4 scalar."""
    swap = M <= 256 and _tc_cost(N, M) < _tc_cost(M, N)           # gemm.cu:274
    if swap:
        (M, N), (sa, sb), (a_al, b_al), (sc_m, sc_n) = (N, M), ((sb[1], sb[0]), (sa[1], sa[0])), (b_al, a_al), (1, ldc)
    else:
        sc_m, sc_n = ldc, 1
    kps = _cdiv(_cdiv(K, splitk), BK) * BK                          # gemm.cu:283-285
    splits = _cdiv(K, kps)
    kal = K % 4 == 0 and kps % 4 == 0                              # gemm_tc.cuh:403-407
    av = 1 if (sa[1] == 1 and a_al and sa[0] % 4 == 0 and kal) else \
        2 if (sa[0] == 1 and a_al and sa[1] % 4 == 0 and M % 4 == 0) else 0
    bv = 1 if (sb[0] == 1 and b_al and sb[1] % 4 == 0 and kal) else \
        2 if (sb[1] == 1 and b_al and sb[0] % 4 == 0 and N % 4 == 0) else 0
    wn = 96 if _tile_n(N) <= 96 else MAXN                          # gemm_tc.cuh:408-412
    branches = set()
    for n0 in range(0, N, MAXN):                                   # gemm_tc.cuh:313-365, warp 0 (rows m0 ..)
        ncol = min(min(MAXN, _cdiv(N - n0, 32) * 32), N - n0)
        if splits > 1:
            sm, sn, al = N, 1, (n0 + 0) % 4 == 0 and N % 4 == 0   # partial tiles [z][M][N], 256-byte aligned base
        else:
            sm, sn = sc_m, sc_n
            al = c_al and (n0 * sc_n) % 4 == 0
        if sn == 1 and sm == ncol and ncol % 4 == 0 and al:
            branches.add(1)
        elif sn == 1 and sm % 4 == 0 and ncol % 4 == 0 and al:
            branches.add(2)
        elif sm == 1:
            branches.add(3)
        else:
            branches.add(4)
    return swap, av, bv, wn, frozenset(branches)


def _operand(rows, cols, layout, off, g, cuda):
    """(rows x cols) matrix X stored with X[r][c] = buf[off + r*s0 + c*s1]: layout "row" (s1 = 1, row pitch
    cols + 4), "col" (s0 = 1, column pitch rows + 4) -> (base tensor at `off`, (s0, s1), dense float64 copy)"""
    s = (cols + 4, 1) if layout == "row" else (1, rows + 4)
    n = (rows - 1) * s[0] + (cols - 1) * s[1] + 1
    buf = torch.randn(off + n + 8, generator=g).to(cuda)
    base = buf[off:]
    dense = torch.as_strided(base, (rows, cols), s).double()
    return base, s, dense


def _check(out, A, B, N):
    ref = A @ B
    bound = A.abs() @ B.abs()
    err = (out[:, :N].double() - ref).abs()
    worst = float((err / bound.clamp(min=1e-30)).max())
    assert (err <= TOL * bound).all(), f"per element: worst {worst}"
    assert float(err.max()) <= TOL * max(1.0, float(ref.abs().max()))
    return worst


# (M, N, K, A layout, B layout, A offset, B offset, split-K, ldc - N, output offset) -> intended path
TC_CASES = [
    # staging modes: row-major operands take float4 along k (1), column-major float4 along the rows (2), an
    # odd storage offset forces scalar loads (0)
    ((1000, 80, 64, "row", "col", 0, 0, 1, 0, 0), (False, 1, 1, 96, {1})),
    ((1000, 80, 64, "col", "row", 0, 0, 1, 0, 0), (False, 2, 2, 96, {1})),
    ((1000, 80, 64, "row", "row", 1, 0, 1, 0, 0), (False, 0, 2, 96, {1})),
    ((1000, 80, 64, "col", "col", 0, 1, 1, 0, 0), (False, 2, 0, 96, {1})),
    ((1000, 80, 64, "row", "col", 1, 1, 1, 0, 0), (False, 0, 0, 96, {1})),
    ((1000, 80, 61, "row", "col", 0, 0, 1, 0, 0), (False, 0, 0, 96, {1})),     # K % 4 != 0: no float4 along k
    # tile widths: N in 32..96, 97..160, and N > 160 with a narrow last tile (336 = 2 x 160 + 16)
    ((700, 32, 40, "row", "col", 0, 0, 1, 0, 0), (False, 1, 1, 96, {1})),
    ((700, 152, 40, "row", "col", 0, 0, 1, 0, 0), (False, 1, 1, 160, {1})),
    ((700, 336, 40, "row", "col", 0, 0, 1, 0, 0), (False, 1, 1, 160, {2})),
    ((700, 330, 40, "col", "row", 0, 0, 1, 6, 0), (False, 2, 0, 160, {2, 4})),  # N % 4 != 0: last tile scalar
    # epilogue: padded rows (ldc > N), a misaligned output view, an odd row pitch
    ((700, 120, 48, "row", "col", 0, 0, 1, 8, 0), (False, 1, 1, 160, {2})),
    ((700, 120, 48, "row", "col", 0, 0, 1, 0, 1), (False, 1, 1, 160, {4})),
    ((700, 120, 48, "row", "col", 0, 0, 1, 3, 0), (False, 1, 1, 160, {4})),
    # swap (short M: C^T = B^T A^T is staged), transposed epilogue; with split-K the partial tiles are row-major
    ((144, 80, 5000, "col", "row", 0, 0, 1, 0, 0), (True, 2, 2, 160, {3})),
    ((144, 80, 5000, "col", "row", 0, 0, 40, 0, 0), (True, 2, 2, 160, {1})),
    ((144, 80, 4000, "col", "row", 1, 0, 31, 0, 0), (True, 2, 0, 160, {1})),
    # split-K without swap, partial tiles of several column tiles
    ((1000, 336, 2048, "row", "col", 0, 0, 16, 0, 0), (False, 1, 1, 160, {2})),
    ((600, 90, 2000, "col", "col", 0, 0, 8, 0, 0), (False, 2, 1, 96, {4})),     # N % 4 != 0
]


def _tc_id(c):
    (M, N, K, la, lb, oa, ob, sk, dl, oc), _ = c
    return f"M{M}-N{N}-K{K}-{la}{oa}-{lb}{ob}-sk{sk}-ldc+{dl}-c{oc}"


def _case_path(case):
    M, N, K, la, lb, oa, ob, sk, dl, oc = case
    sa = (K + 4, 1) if la == "row" else (1, M + 4)
    sb = (N + 4, 1) if lb == "row" else (1, K + 4)
    return tc_path(M, N, K, sa, sb, oa % 4 == 0, ob % 4 == 0, sk, N + dl, oc % 4 == 0)


def test_tc_cases_cover_every_path():
    paths = [_case_path(c) for c, _ in TC_CASES]
    for (c, want), got in zip(TC_CASES, paths):
        assert got == (want[0], want[1], want[2], want[3], frozenset(want[4])), (c, got)
    assert {p[1] for p in paths} == {0, 1, 2} and {p[2] for p in paths} == {0, 1, 2}
    assert {p[3] for p in paths} == {96, MAXN}
    assert {p[0] for p in paths} == {False, True}
    assert set().union(*(p[4] for p in paths)) == {1, 2, 3, 4}
    assert any(c[1] > MAXN and c[1] % MAXN < 32 for c, _ in TC_CASES)              # a narrow last tile
    assert {c[7] > 1 for c, _ in TC_CASES} == {False, True}
    # the PointWiseMLP products below: their un-split products at C >= 576 leave AUTO to the FMA kernel (k > 512)
    assert [_padded(C + 3) > 512 for C in PW_WIDTHS] == [False, True, True]


@pytest.mark.gpu
@pytest.mark.parametrize("case", TC_CASES, ids=_tc_id)
def test_tc_path_matches_f64(cuda, case):
    from closerlook3d_b200 import ops
    (M, N, K, la, lb, oa, ob, sk, dl, oc), _ = case
    g = torch.Generator().manual_seed(M * 7 + N * 3 + K + oa + 2 * ob + sk)
    a, sa, A = _operand(M, K, la, oa, g, cuda)
    b, sb, Bm = _operand(K, N, lb, ob, g, cuda)
    ldc = N + dl
    obuf = torch.full((oc + M * ldc + 64,), float("nan"), device=cuda)
    out = obuf[oc:oc + M * ldc].view(M, ldc)
    got = ops.sgemm(a, sa[0], sa[1], b, sb[0], sb[1], M, N, K, out=out, ldc=ldc, splitk=sk, algo=ops.GEMM_TC3X)
    torch.cuda.synchronize()
    assert got.data_ptr() == out.data_ptr()
    worst = _check(out, A, Bm, N)
    # nothing outside the M x N block of the output view is written
    assert torch.isnan(obuf[:oc]).all() and torch.isnan(obuf[oc + M * ldc:]).all()
    if dl:
        assert torch.isnan(out[:, N:]).all()
    print(f"\nGEMM tc {_tc_id((case[0], None))}: {worst:.2e}")


# --------------------------------------------------------------------------------------------------------------
# the three products of the fused PointWiseMLP (pwmlp.py:28, 68, 71) at the network's wide layers
# --------------------------------------------------------------------------------------------------------------
PW_WIDTHS = [288, 576, 1152]
PW_POINTS = {288: 2 * 1152, 576: 2 * 1152, 1152: 2 * 304}     # B * N of the layer (supports of the strided block)


@pytest.mark.gpu
@pytest.mark.parametrize("algo", ALGOS)
@pytest.mark.parametrize("product", ["forward", "weight_grad", "feature_grad"])
@pytest.mark.parametrize("C", PW_WIDTHS)
def test_pwmlp_products_at_wide_layers(cuda, C, product, algo):
    from closerlook3d_b200 import ops
    P = PW_POINTS[C]
    Cout, Cp, Cpa = C, _padded(C), _padded(C + 3)
    Cop = _padded(Cout)
    g = torch.Generator().manual_seed(C + P)
    fa = torch.randn(P, Cpa, generator=g).to(cuda)            # [f | xyz/r | 0] rows
    wcat = torch.randn(2 * Cop, Cpa, generator=g).to(cuda)
    grad_ab = torch.randn(P, 2 * Cop, generator=g).to(cuda)
    if product == "forward":        # AB = fa @ wcat^T  (pwmlp.py:28)
        out = ops.sgemm(fa, Cpa, 1, wcat, 1, Cpa, P, 2 * Cop, Cpa, algo=algo)
        worst = _check(out, fa.double(), wcat.double().t(), 2 * Cop)
    elif product == "weight_grad":  # d/dwcat = grad_AB^T @ fa, split-K  (pwmlp.py:67-68)
        splitk = max(1, min(1024, P // 128))
        out = ops.sgemm(grad_ab, 1, 2 * Cop, fa, Cpa, 1, 2 * Cop, Cpa, P, splitk=splitk, algo=algo)
        worst = _check(out, grad_ab.double().t(), fa.double(), Cpa)
    else:                           # d/dfeat = grad_AB @ wcat[:, :Cp]  (pwmlp.py:71)
        out = ops.sgemm(grad_ab, 2 * Cop, 1, wcat, Cpa, 1, P, Cp, 2 * Cop, ldc=Cp, algo=algo)
        assert out.shape == (P, Cp)
        worst = _check(out, grad_ab.double(), wcat[:, :Cp].double(), Cp)
    print(f"\nGEMM pwmlp C={C} {product} algo={algo}: {worst:.2e}")
