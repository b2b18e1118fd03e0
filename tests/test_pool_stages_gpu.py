"""GPU: the fused max-pool (pool.cu: gather_max_fwd_kernel, gather_max_bwd_kernel, gather_max_bwd_csr_kernel), the
decoder's nearest upsampling and the grouping it runs on (core.cu: group_points*, the 16-bit convert_kernel) at the
stage shapes the shipped networks run, against float64.

Reference: the reference's own composition (pt_utils.py:195-201) in float64 on the GPU -- f64_ext.group_points, then
F.max_pool2d over K -- and its backward by autograd; nearest upsampling is group_points with K = 1.  max_pool2d sends
the gradient to the FIRST maximal slot, the rule pool.cu follows, so ties between distinct neighbours pin it.  The
library is called at the operator level (ops.gather_max / gather_max_grad, ops.group_points / group_points_grad) over
the indices of its own search (pt_utils.neighbors, ops.nearest_query; checked bit for bit by other tests), which
isolates the pooling kernels from the search.

Bars.  A max and a gather are exact: the forward equals the float64 result cast to the features' dtype.  Backward, per
element: |got - ref| <= u |ref| + 1e-6 S, S = the same float64 backward applied to |grad_out| (the magnitudes routed
to that element), u = 0 in fp32, 2^-8 in bf16, 2^-11 in fp16 (the library accumulates in fp32 and rounds once).  A
gradient sent to the wrong slot is an O(S) error.  Every backward runs in the default mode (fp32 atomics) and in
deterministic mode (gather form over the transposed lists).
"""
import pytest
import torch
import torch.nn.functional as F

from closerlook3d_b200 import synth

GRAD_TOL = 1e-6
UNIT = {torch.float32: 0.0, torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}

# MaskedMaxPool of each strided bottleneck: (C, N, M, K) = (the block's input width, the previous stage's points,
# npoints[s], nsamples[s]) of backbone.model_config; the widths are width * 2^s (backbone.ResNet, width 144).
POOL_S3DIS = [(144, 15000, 4096, 26), (288, 4096, 1152, 31), (576, 1152, 304, 38), (1152, 304, 88, 41)]
POOL_S3DIS_X2 = [(2 * C, N, M, K) for C, N, M, K in POOL_S3DIS]        # width x2 (BASELINE c5: PosPool sin_cos)
POOL_MODELNET = [(144, 10000, 2048, 20), (288, 2048, 512, 31), (576, 512, 128, 38), (1152, 128, 32, 36)]
POOL_SHAPENETPART = [(144, 2048, 1280, 11), (288, 1280, 768, 25), (576, 768, 192, 37), (1152, 192, 64, 36)]
# PartNet (10000 -> 5120/1024/384/64, K = 23/38/42/40) reaches no launch shape the tables above do not
# (test_case_tables_reach_every_path), so it is not run.
POOL_TABLES = {"s3dis": POOL_S3DIS, "s3dis_x2": POOL_S3DIS_X2, "modelnet": POOL_MODELNET,
               "shapenetpart": POOL_SHAPENETPART}

# SceneSegHeadResNet's nearest upsampling up0..up3: (C, N, M) = (the coarse stage's width, its points, the fine
# stage's points) -- res5 -> res4 carries 16 * width channels, then the decoder's up_conv outputs 4, 2, 1 x width.
UP_S3DIS = [(2304, 88, 304), (576, 304, 1152), (288, 1152, 4096), (144, 4096, 15000)]
UP_S3DIS_X2 = [(2 * C, N, M) for C, N, M in UP_S3DIS]
UP_TABLES = {"s3dis": UP_S3DIS, "s3dis_x2": UP_S3DIS_X2}

LOW = (torch.bfloat16, torch.float16)


def _ends(table):
    """the narrowest and the widest stage"""
    return [min(table), max(table)]


POOL_CASES = ([(name, s, torch.float32) for name, t in POOL_TABLES.items() for s in t]
              + [(name, s, dt) for name, t in POOL_TABLES.items() for s in _ends(t) for dt in LOW])
UP_CASES = ([(name, s, torch.float32) for name, t in UP_TABLES.items() for s in t]
            + [(name, s, dt) for name, t in UP_TABLES.items() for s in _ends(t) for dt in LOW])

# small shapes at the edges of the launch arithmetic: (C, N, M, K, B, features)
#   features: "randn"; "ties" = floor(4|x|) / 4, many distinct neighbours share the maximum; "relu" = max(x, 0)
EDGE_CASES = [
    (12, 700, 33, 5, 2, "randn"),      # forward CI = 1, a partial warp, an M tail of one query
    (40, 700, 31, 3, 1, "ties"),       # CI = 2, one partial tile
    (72, 700, 1, 1, 3, "randn"),       # CI = 3, K = 1, M = 1
    (100, 700, 33, 2, 3, "relu"),      # CI = 4 in one chunk of 104 padded channels
    (130, 700, 64, 255, 2, "ties"),    # two forward chunks, the second 8 wide; K = 255 (the largest)
    (130, 2500, 31, 5, 1, "relu"),
    (12, 700, 33, 255, 1, "relu"),
    (1815, 700, 33, 5, 1, "randn"),    # the widest backward in one chunk: 32 x 1816 floats = the 227 KB opt-in
    (1816, 700, 40, 6, 2, "ties"),     # the narrowest in two: chunks of 928 and 888 channels
]


def _dt_id(dt):
    return str(dt).replace("torch.", "")


def _features(feats, kind):
    if kind == "ties":
        return torch.floor(4 * feats.abs()) / 4
    if kind == "relu":
        return feats.clamp(min=0)
    return feats


def _check_fwd(out, ref, dtype, tag):
    want = ref.detach().to(dtype)
    ndiff = int((out != want).sum())
    print(f"\n{tag}: forward {ndiff} of {out.numel()} elements differ")
    assert out.dtype == dtype and out.shape == want.shape
    assert torch.equal(out, want), f"{tag}: {ndiff} forward elements differ"


def _check_bwd(got, ref, S, dtype, tag):
    """|got - ref| <= u |ref| + GRAD_TOL * S per element; prints the worst ratio to the bar"""
    err = (got.double() - ref).abs()
    bar = UNIT[dtype] * ref.abs() + GRAD_TOL * S
    worst = float((err / bar.clamp(min=1e-300)).max())
    bad = err > bar
    print(f"{tag}: worst |err| / bar {worst:.2e}")
    assert got.dtype == dtype and got.shape == ref.shape
    assert not bad.any(), f"{tag}: {int(bad.sum())} elements over the bar, first (b,c,n) {bad.nonzero()[0].tolist()}"


def _both_modes(fn):
    """fn() in the default mode and under torch.use_deterministic_algorithms(True) -> [(mode, result)]"""
    prev = torch.are_deterministic_algorithms_enabled()
    res = []
    try:
        for det in (False, True):
            torch.use_deterministic_algorithms(det)
            res.append(("deterministic" if det else "default", fn()))
    finally:
        torch.use_deterministic_algorithms(prev)
    return res


def _f64_grads(ref, f64, gout):
    """autograd of the float64 reference: (d/df for grad_out, the same backward of |grad_out| = S)"""
    g64 = gout.double()
    (ref_g,) = torch.autograd.grad(ref, f64, g64, retain_graph=True)
    (S,) = torch.autograd.grad(ref, f64, g64.abs())
    return ref_g, S


def run_pool(cuda, C, N, M, K, B=2, dtype=torch.float32, kind="randn", seed=None, tag=""):
    """ops.gather_max / gather_max_grad over the library's ball query against the float64 composition"""
    from closerlook3d_b200 import ops, pt_utils
    from oracle import f64_ext
    torch.cuda.reset_peak_memory_stats()
    seed = 9000 + C + N + M + K if seed is None else seed
    d = synth.make_cloud_batch(B, N, C, seed)                  # padded clouds: padded rows repeat valid ones
    r = synth.ball_radius(N, K)
    g = torch.Generator().manual_seed(seed + 1)
    q = (d["xyz"][:, :M] + 0.1 * r * torch.randn(B, M, 3, generator=g)).contiguous()
    qm = torch.ones(B, M, dtype=torch.int32)
    qm[:, M - M // 8:] = 0                                     # queries with mask 0: the max ignores masks
    xyz, mask = d["xyz"].to(cuda), d["mask"].to(cuda)
    nl = pt_utils.neighbors(q.to(cuda), xyz, qm.to(cuda), mask, r, K).wait()
    idx = nl.idx
    pt_utils.clear_neighbor_cache()
    feats = _features(d["features"], kind).to(cuda, dtype)

    out, arg = ops.gather_max(feats, idx)
    f64 = feats.double().requires_grad_(True)
    ref = F.max_pool2d(f64_ext.group_points(f64, idx), kernel_size=[1, K]).squeeze(-1)
    _check_fwd(out, ref, dtype, tag)

    gout = torch.randn(B, C, M, generator=torch.Generator().manual_seed(seed + 2)).to(cuda, dtype)
    ref_g, S = _f64_grads(ref, f64, gout)
    del ref
    for mode, got in _both_modes(lambda: ops.gather_max_grad(gout, idx, arg, N)):
        _check_bwd(got, ref_g, S, dtype, f"{tag} backward {mode}")
    print(f"{tag}: peak {torch.cuda.max_memory_allocated() / 2**30:.2f} GiB")


def run_upsample(cuda, C, N, M, B=2, dtype=torch.float32, seed=None, tag=""):
    """nearest upsampling (MaskedUpsample(mode='nearest')): ops.group_points / group_points_grad with K = 1 over
    ops.nearest_query against the float64 gather"""
    from closerlook3d_b200 import ops
    from oracle import f64_ext
    torch.cuda.reset_peak_memory_stats()
    seed = 9500 + C + N + M if seed is None else seed
    coarse = synth.make_cloud_batch(B, N, C, seed)
    fine = synth.make_cloud_batch(B, M, 1, seed + 1)           # its padded rows are queries with mask 0
    xyz, mask = coarse["xyz"].to(cuda), coarse["mask"].to(cuda)
    up_xyz, up_mask = fine["xyz"].to(cuda), fine["mask"].to(cuda)
    idx, _ = ops.nearest_query(up_xyz, xyz, up_mask, mask)
    idx = idx.unsqueeze(-1).contiguous()                       # (B,M,1)
    feats = coarse["features"].to(cuda, dtype)

    out = ops.group_points(feats, idx)[..., 0]
    f64 = feats.double().requires_grad_(True)
    ref = f64_ext.group_points(f64, idx)[..., 0]
    _check_fwd(out, ref, dtype, tag)

    gout = torch.randn(B, C, M, generator=torch.Generator().manual_seed(seed + 2)).to(cuda, dtype)
    ref_g, S = _f64_grads(ref, f64, gout)
    del ref
    g4 = gout.unsqueeze(-1).contiguous()
    for mode, got in _both_modes(lambda: ops.group_points_grad(g4, idx, N)):
        _check_bwd(got, ref_g, S, dtype, f"{tag} backward {mode}")
    print(f"{tag}: peak {torch.cuda.max_memory_allocated() / 2**30:.2f} GiB")


@pytest.mark.gpu
@pytest.mark.parametrize("net,shape,dtype", POOL_CASES,
                         ids=[f"{n}-C{s[0]}-N{s[1]}-M{s[2]}-K{s[3]}-{_dt_id(dt)}" for n, s, dt in POOL_CASES])
def test_max_pool_stage_matches_f64(cuda, net, shape, dtype):
    C, N, M, K = shape
    run_pool(cuda, C, N, M, K, dtype=dtype, tag=f"POOL {net} C={C} N={N} M={M} K={K} {_dt_id(dtype)}")


@pytest.mark.gpu
@pytest.mark.parametrize("net,shape,dtype", UP_CASES,
                         ids=[f"{n}-C{s[0]}-N{s[1]}-M{s[2]}-{_dt_id(dt)}" for n, s, dt in UP_CASES])
def test_nearest_upsample_stage_matches_f64(cuda, net, shape, dtype):
    C, N, M = shape
    run_upsample(cuda, C, N, M, dtype=dtype, tag=f"UP {net} C={C} N={N} M={M} {_dt_id(dtype)}")


@pytest.mark.gpu
@pytest.mark.parametrize("C,N,M,K,B,kind", EDGE_CASES, ids=[f"C{c[0]}-M{c[2]}-K{c[3]}-B{c[4]}-{c[5]}" for c in EDGE_CASES])
def test_max_pool_edges_match_f64(cuda, C, N, M, K, B, kind):
    run_pool(cuda, C, N, M, K, B=B, kind=kind, tag=f"POOL-EDGE C={C} N={N} M={M} K={K} B={B} {kind}")


@pytest.mark.gpu
@pytest.mark.parametrize("C,N,M,B", [(12, 300, 33, 1), (130, 300, 1, 3), (100, 500, 31, 3)],
                         ids=["C12-M33-B1", "C130-M1-B3", "C100-M31-B3"])
def test_nearest_upsample_edges_match_f64(cuda, C, N, M, B):
    run_upsample(cuda, C, N, M, B=B, tag=f"UP-EDGE C={C} N={N} M={M} B={B}")


@pytest.mark.gpu
def test_max_pool_rejects_k_256_on_the_host(cuda):
    from closerlook3d_b200 import ops
    feats = torch.randn(1, 16, 300, device=cuda)
    idx = torch.randint(0, 300, (1, 8, 256), dtype=torch.int32, device=cuda)
    with pytest.raises(RuntimeError, match="cl3d_gather_max_fwd: bad arguments"):
        ops.gather_max(feats, idx)
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_masked_upsample_max_module_matches_f64(cuda):
    """MaskedUpsample(mode='max') through autograd at the decoder's res4 -> res3 stage (C = 576, 304 -> 1152 points,
    nsample = nsamples[2] = 38)"""
    from closerlook3d_b200 import pt_utils
    from closerlook3d_b200.pt_utils import MaskedUpsample
    from oracle import f64_ext
    B, C, N, M, K = 2, 576, 304, 1152, 38
    torch.cuda.reset_peak_memory_stats()
    coarse = synth.make_cloud_batch(B, N, C, 77)
    fine = synth.make_cloud_batch(B, M, 1, 78)
    xyz, mask, feats = coarse["xyz"].to(cuda), coarse["mask"].to(cuda), coarse["features"].to(cuda)
    up_xyz, up_mask = fine["xyz"].to(cuda), fine["mask"].to(cuda)
    r = synth.ball_radius(N, K)
    gout = torch.randn(B, C, M, generator=torch.Generator().manual_seed(79)).to(cuda)
    pt_utils.clear_neighbor_cache()
    idx = pt_utils.neighbors(up_xyz, xyz, up_mask, mask, r, K).wait().idx
    f64 = feats.double().requires_grad_(True)
    ref = F.max_pool2d(f64_ext.group_points(f64, idx), kernel_size=[1, K]).squeeze(-1)
    ref_g, S = _f64_grads(ref, f64, gout)
    tag = f"UP-MAX module C={C} N={N} M={M} K={K}"

    def step():
        f = feats.clone().requires_grad_(True)
        out = MaskedUpsample(r, K, mode="max")(up_xyz, xyz, up_mask, mask, f)
        out.backward(gout)
        return out.detach(), f.grad

    for mode, (out, grad) in _both_modes(step):
        _check_fwd(out, ref, torch.float32, f"{tag} {mode}")
        _check_bwd(grad, ref_g, S, torch.float32, f"{tag} backward {mode}")
    pt_utils.clear_neighbor_cache()
    print(f"{tag}: peak {torch.cuda.max_memory_allocated() / 2**30:.2f} GiB")


@pytest.mark.gpu
def test_width_x2_scene_network_trains(cuda):
    """one training step of the width x2 scene-segmentation network (PosPool sin_cos avg, width 288) in the default
    mode: its layer4 max-pool runs at C = 2304, whose backward stages its channels in two chunks"""
    from closerlook3d_b200 import backbone as bb, pt_utils
    cfg = bb.model_config("scene_segmentation", "pospool", pospool=dict(position_embedding="sin_cos", reduction="avg"))
    cfg.width = 288
    cfg.radius, cfg.sampleDl = 0.06, 0.03                      # stage settings of test_model_gpu._cfg
    cfg.npoints = [1024, 320, 96, 32]
    cfg.nsamples = [16, 18, 20, 18, 16]
    cfg.num_classes = 9
    assert cfg.width * 8 == 2304                               # layer4's strided block input
    torch.cuda.reset_peak_memory_stats()
    torch.manual_seed(5)
    model, criterion = bb.build_scene_segmentation(cfg)
    model.init_weights()
    model = model.to(cuda).train()
    B, N = 2, 3000
    d = synth.make_cloud_batch(B, N, cfg.input_features_dim, 31)
    xyz, mask, feats = d["xyz"].to(cuda), d["mask"].to(cuda), d["features"].to(cuda)
    target = torch.randint(0, cfg.num_classes, (B, N), generator=torch.Generator().manual_seed(32)).to(cuda)
    pt_utils.clear_neighbor_cache()
    assert not torch.are_deterministic_algorithms_enabled()
    loss = criterion(model(xyz, mask, feats), target, mask.float())
    loss.backward()
    torch.cuda.synchronize()
    pt_utils.clear_neighbor_cache()
    assert torch.isfinite(loss), float(loss)
    for name, p in model.named_parameters():
        assert p.grad is not None, f"no gradient for {name}"
        assert torch.isfinite(p.grad).all(), f"non-finite gradient in {name}"
    print(f"\nNET width x2 loss {float(loss):.4f}: peak {torch.cuda.max_memory_allocated() / 2**30:.2f} GiB")


# --------------------------------------------------------------------------------------------------------------
# CPU: the launch rules of pool.cu, restated, and the paths the case tables above reach
# --------------------------------------------------------------------------------------------------------------
def _cdiv(a, b):
    return -(-a // b)


def _padded(C):
    return (C + 7) & ~7


MAX_DYN_SMEM = 227 * 1024      # kMaxDynSmem (common.cuh)


def pool_fwd_instance(C):
    """cl3d_gather_max_fwd: CI = min(ceil(Cp / 32), 4) channels per lane, gridDim.y chunks of 32 CI padded
    channels -> (CI, gridDim.y, padded width of the last chunk)"""
    Cp = _padded(C)
    ci = min(_cdiv(Cp, 32), 4)
    n = _cdiv(Cp, 32 * ci)
    return ci, n, Cp - (n - 1) * 32 * ci


def pool_bwd_chunks(C):
    """cl3d_gather_max_bwd (default mode): one chunk of C channels while 32 x (C + 1) floats fit in the opt-in shared
    memory, else the fewest equal chunks that fit, rounded up to 32 channels -> (gridDim.y, chunk)"""
    if 32 * (C + 1) * 4 <= MAX_DYN_SMEM:
        return 1, C
    most = (MAX_DYN_SMEM // (32 * 4) - 1) // 32 * 32
    chunk = _cdiv(_cdiv(C, _cdiv(C, most)), 32) * 32
    return _cdiv(C, chunk), chunk


def test_case_tables_reach_every_path():
    from closerlook3d_b200.backbone import PART_DATASETS, model_config
    # the tables are the shipped configurations' stages
    for table, task, ds in ((POOL_S3DIS, "scene_segmentation", None), (POOL_MODELNET, "classification", None),
                            (POOL_SHAPENETPART, "multi_part_segmentation", "shapenetpart")):
        c = model_config(task, dataset=ds) if ds else model_config(task)
        pts = [c.num_points] + list(c.npoints)
        assert [(N, M, K) for _, N, M, K in table] == list(zip(pts[:-1], pts[1:], c.nsamples[:4]))
        assert [C for C, _, _, _ in table] == [c.width << s for s in range(4)]
    s3 = model_config("scene_segmentation")
    pts = [s3.num_points] + list(s3.npoints)
    assert [(N, M) for _, N, M in UP_S3DIS] == list(zip(pts[:0:-1], pts[-2::-1]))
    assert [C for C, _, _ in UP_S3DIS] == [16 * s3.width, 4 * s3.width, 2 * s3.width, s3.width]
    assert {C for C, _, _, _ in POOL_S3DIS_X2} == {288, 576, 1152, 2304}

    pool = [s for _, s, _ in POOL_CASES] + [c[:4] for c in EDGE_CASES]
    fwd = [pool_fwd_instance(C) for C, _, _, _ in pool]
    assert {ci for ci, _, _ in fwd} == {1, 2, 3, 4}                          # every forward instance
    assert any(n > 1 and last < 32 * ci for ci, n, last in fwd)             # a partial last chunk
    assert any(n > 1 and last == 8 for ci, n, last in fwd)                  # ... 8 channels wide
    assert any(C % 32 for C, _, _, _ in pool)                               # partial warps
    assert {K % 4 for _, _, _, K in pool} == {0, 1, 2, 3}                   # every tail of the 4-row unroll
    assert {1, 255} <= {K for _, _, _, K in pool}
    assert any(M % 32 for _, _, M, _ in pool) and 1 in {M for _, _, M, _ in pool}   # M tails
    # the backward: every width-144 stage in one chunk (the launch it always had), C = 2304 in more than one
    assert all(pool_bwd_chunks(C) == (1, C) for t in (POOL_S3DIS, POOL_MODELNET, POOL_SHAPENETPART)
               for C, _, _, _ in t)
    assert max(pool_bwd_chunks(C)[0] for C, _, _, _ in pool) > 1
    assert pool_bwd_chunks(1815) == (1, 1815) and pool_bwd_chunks(1816) == (2, 928)
    assert pool_bwd_chunks(2304) == (2, 1152)
    assert {1815, 1816} <= {C for C, _, _, _ in pool}                       # both sides of the one-chunk limit
    # PartNet's stages reach nothing new: CI 4, widths, K % 4 and tile-aligned M all appear above
    pn = PART_DATASETS["partnet"]
    pts = [pn["num_points"]] + pn["npoints"]
    for s in range(4):
        C, M, K = 144 << s, pts[s + 1], pn["nsamples"][s]
        assert C in {c for c, _, _, _ in pool} and M % 32 == 0 and K % 4 in {K2 % 4 for _, _, _, K2 in pool}
