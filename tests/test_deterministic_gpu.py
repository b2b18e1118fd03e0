"""Deterministic mode (torch.use_deterministic_algorithms(True)): canonical transposed lists, and bit-for-bit
repeatable fused LocalAggregation, max-pool, upsample and grouping steps, whatever the stream overlap, the
neighbour cache, a CUDA-graph replay or other work on the GPU."""
import copy
import importlib.util
import os

import numpy as np
import pytest
import torch

from closerlook3d_b200 import ops, pt_utils, synth
from closerlook3d_b200.config import baseline_config, la_config

pytestmark = pytest.mark.gpu


def canonical_lists(idx, ncount, N):
    """numpy: every list in ascending q*K + k (the stable argsort of the slots' support indices)"""
    B, M, K = idx.shape
    off = np.zeros((B, N + 1), np.int32)
    ent = np.full((B, M * K), -1, np.int32)
    for b in range(B):
        e = np.arange(M * K)
        keep = np.ones(M * K, bool) if ncount is None else (e % K) < np.repeat(ncount[b], K)
        e, j = e[keep], idx[b].reshape(-1)[keep]
        ent[b, :len(e)] = e[np.argsort(j, kind="stable")]
        off[b, 1:] = np.cumsum(np.bincount(j, minlength=N))
    return off, ent


@pytest.fixture
def det():
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(False)


def _clouds(kind, B, N, M, K, seed):
    d = synth.make_cloud_batch(B, N, 8, seed)
    xyz, mask = d["xyz"], d["mask"]
    r = synth.ball_radius(N, K)
    if kind == "coincident":       # every query picks the same K lowest indices: K lists of M entries each
        xyz = torch.zeros_like(xyz) + 0.5
    if M == N:
        return xyz, xyz, mask, mask, r
    g = torch.Generator().manual_seed(seed + 1)
    q = (xyz[:, :M] + 0.1 * r * torch.randn(B, M, 3, generator=g)).contiguous()
    qm = torch.ones(B, M, dtype=torch.int32)
    qm[:, M - M // 8:] = 0
    return q, xyz, qm, mask, r


def _check_lists(off, ent, want_off, want_ent):
    off, ent = off.cpu().numpy(), ent.cpu().numpy()
    assert np.array_equal(off, want_off)
    for b in range(off.shape[0]):
        n = off[b, -1]
        assert np.array_equal(ent[b, :n], want_ent[b, :n])


@pytest.mark.parametrize("kind,B,N,M,K", [
    ("random", 2, 1500, 1500, 16),       # brute force search (AUTO), padded clouds
    ("random", 2, 6000, 6000, 26),       # grid search
    ("random", 2, 6000, 1500, 26),       # strided layer, masked queries
    ("coincident", 1, 3000, 3000, 32),   # lists of 3000 entries: the grid-wide pass
])
@pytest.mark.parametrize("algo", [0, 1, 2])   # CL3D_BQ_AUTO, BRUTE, GRID
def test_lists_are_canonical(cuda, det, kind, B, N, M, K, algo):
    q, s, qm, sm, r = [t.to(cuda) if torch.is_tensor(t) else t for t in _clouds(kind, B, N, M, K, 5)]
    for slots in ("counted", "all"):
        idx, _, ncount, (off, ent) = ops.ball_query(q, s, qm, sm, r, K, algo=algo, csr=slots, deterministic=True)
        _, _, _, (off0, _) = ops.ball_query(q, s, qm, sm, r, K, algo=algo, csr=slots, deterministic=False)
        assert torch.equal(off, off0)
        nc = ncount.cpu().numpy() if slots == "counted" else None
        want = canonical_lists(idx.cpu().numpy(), nc, N)
        _check_lists(off, ent, *want)
        # the stand-alone builder gives the same lists
        off2, ent2 = ops.build_csr(idx, ncount if slots == "counted" else None, N, deterministic=True)
        off3, _ = ops.build_csr(idx, ncount if slots == "counted" else None, N, deterministic=False)
        assert torch.equal(off2, off3)
        _check_lists(off2, ent2, *want)
    if kind == "coincident":
        assert int((off[:, 1:] - off[:, :-1]).max()) > 1024   # longer than the one-warp path takes


# ---------------------------------------------------------------------------------------------------------------
# repeatability of the fused LocalAggregation modules
# ---------------------------------------------------------------------------------------------------------------
FAMILIES = [
    ("pospool", dict(pospool=dict(position_embedding="xyz", reduction="avg")), 66),
    ("pospool", dict(pospool=dict(position_embedding="xyz", reduction="sum")), 66),
    ("pospool", dict(pospool=dict(position_embedding="xyz", reduction="max")), 66),
    ("pospool", dict(pospool=dict(position_embedding="sin_cos", reduction="avg")), 72),
    ("pospool", dict(pospool=dict(position_embedding="sin_cos", reduction="sum")), 72),
    ("pospool", dict(pospool=dict(position_embedding="sin_cos", reduction="max")), 72),
    ("adaptive_weight", dict(adaptive_weight=dict(weight_type="dp", num_mlps=1, shared_channels=1,
                                                  reduction="avg")), 64),
    ("adaptive_weight", dict(adaptive_weight=dict(weight_type="dp", num_mlps=1, shared_channels=1,
                                                  reduction="max")), 64),
    ("pseudo_grid", dict(), 40),      # pg3 range
    ("pseudo_grid", dict(), 72),      # pg2 range
    ("pseudo_grid", dict(), 136),     # above 128: channel chunks
    ("pointwisemlp", dict(pointwisemlp=dict(feature_type="dp_fi_df", num_mlps=1, reduction="max")), 72),
]
PWMLP = FAMILIES[-1]


def _module(cuda, la, over, C, N, K):
    from closerlook3d_b200.local_aggregation_operators import LocalAggregation
    torch.manual_seed(3)
    np.random.seed(3)
    return LocalAggregation(C, C, synth.ball_radius(N, K), K, la_config(la, **over)).to(cuda).train()


def _state(mod):
    return [b.detach().clone() for b in mod.buffers()]


def _eager(mod, sd, b, gout):
    mod.load_state_dict(sd)
    for p in mod.parameters():
        p.grad = None
    f = b["features"].clone().requires_grad_(True)
    out = mod(b["xyz"], b["xyz"], b["mask"], b["mask"], f)
    out.backward(gout)
    torch.cuda.synchronize()
    return [out.detach().clone(), f.grad.clone()] + [p.grad.clone() for p in mod.parameters()] + _state(mod)


def _busy_matmul(cuda):
    """a large matmul queued on a second stream, running beside the step"""
    st = torch.cuda.Stream(device=cuda)
    a = torch.randn(4096, 4096, device=cuda)
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        for _ in range(8):
            a = a @ a
            a = a / a.norm()
    return st, a


def _repeat_runs(cuda, mod, b, gout):
    sd = copy.deepcopy(mod.state_dict())
    runs = {}
    was_cache, was_overlap = pt_utils.cache_enabled, pt_utils.overlap_enabled
    try:
        for i in range(3):
            pt_utils.clear_neighbor_cache()
            runs[f"eager{i}"] = _eager(mod, sd, b, gout)
        pt_utils.clear_neighbor_cache()
        pt_utils.overlap_enabled = False
        runs["overlap off"] = _eager(mod, sd, b, gout)
        pt_utils.overlap_enabled = was_overlap
        pt_utils.cache_enabled = False
        runs["cache off"] = _eager(mod, sd, b, gout)
        pt_utils.cache_enabled = was_cache
        pt_utils.clear_neighbor_cache()
        st, _ = _busy_matmul(cuda)
        runs["beside a matmul"] = _eager(mod, sd, b, gout)
        torch.cuda.current_stream().wait_stream(st)
    finally:
        pt_utils.cache_enabled, pt_utils.overlap_enabled = was_cache, was_overlap
    return runs, sd


def _assert_equal_runs(runs):
    ref = runs["eager0"]
    for name, r in runs.items():
        assert len(r) == len(ref), name
        for i, (a, e) in enumerate(zip(r, ref)):
            assert torch.equal(a, e), f"{name}: tensor {i} differs (max {float((a.float() - e.float()).abs().max())})"


def _graph_run(mod, sd, b, gout):
    from closerlook3d_b200.graphed import GraphedStep
    mod.load_state_dict(sd)
    was = pt_utils.cache_enabled
    pt_utils.cache_enabled = False
    try:
        gs = GraphedStep(mod, b["xyz"], b["mask"], b["features"], gout)
        # the warm-up steps moved the running statistics: start the replay from the eager runs' state, in place
        with torch.no_grad():
            for buf, v in zip(mod.buffers(), [sd[k] for k, _ in mod.named_buffers()]):
                buf.copy_(v)
        gs.load(b["xyz"], b["mask"], b["features"])
        gs.replay()
        torch.cuda.synchronize()
        return [gs.out.clone(), gs.features.grad.clone()] + [g.clone() for g in gs.grads()] + _state(mod)
    finally:
        pt_utils.cache_enabled = was


def _run_family(cuda, la, over, C, B, N, K, graph=True, train=True):
    mod = _module(cuda, la, over, C, N, K).train(train)
    b = {k: v.to(cuda) for k, v in synth.make_cloud_batch(B, N, C, 11).items()}
    gout = torch.randn(B, C, N, device=cuda, generator=torch.Generator(device=cuda).manual_seed(1))
    runs, sd = _repeat_runs(cuda, mod, b, gout)
    if graph:
        runs["graph"] = _graph_run(mod, sd, b, gout)
    _assert_equal_runs(runs)
    return mod, sd, b, gout, runs["eager0"]


@pytest.mark.parametrize("la,over,C", FAMILIES, ids=lambda v: str(v))
def test_local_aggregation_is_repeatable(cuda, det, la, over, C):
    _run_family(cuda, la, over, C, 2, 2304, 16)


def test_pointwisemlp_eval_mode_is_repeatable(cuda, det):
    """frozen BatchNorm: the backward has no dense term, and gathers over the canonical lists all the same"""
    _run_family(cuda, *PWMLP, 2, 2304, 16, graph=False, train=False)


@pytest.mark.parametrize("i", [2, 3, 4, 5])
def test_local_aggregation_is_repeatable_at_baseline_shape(cuda, det, i):
    t = baseline_config(i)
    B = {2: 8, 3: 2, 4: 2, 5: 1}[i]
    _run_family(cuda, t["la"], t["over"], t["C"], B, t["N"], t["K"])


@pytest.mark.parametrize("la,over,C", [FAMILIES[0], FAMILIES[5], FAMILIES[7], FAMILIES[9], FAMILIES[10], PWMLP],
                         ids=lambda v: str(v))
def test_backward_is_the_one_of_the_canonical_lists(cuda, det, la, over, C, monkeypatch):
    """the deterministic step equals the default step fed with numpy-built canonical lists, bit for bit"""
    mod, sd, b, gout, ref = _run_family(cuda, la, over, C, 2, 2304, 16, graph=False)
    torch.use_deterministic_algorithms(False)

    def numpy_lists(self, all_slots):
        self.wait()
        off, ent = canonical_lists(self.idx.cpu().numpy(), None if all_slots else self.ncount.cpu().numpy(), self.N)
        return torch.from_numpy(off).to(cuda), torch.from_numpy(ent).to(cuda)

    monkeypatch.setattr(pt_utils.NeighborList, "_lists", numpy_lists)
    monkeypatch.setattr(ops, "deterministic_mode", lambda d=None: True if d is None else bool(d))
    pt_utils.clear_neighbor_cache()
    got = _eager(mod, sd, b, gout)
    pt_utils.clear_neighbor_cache()
    for i, (a, e) in enumerate(zip(got, ref)):
        assert torch.equal(a, e), f"tensor {i}"


def _sibling(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(os.path.dirname(__file__), name + ".py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.mark.parametrize("la,over,C", [FAMILIES[0], FAMILIES[9], PWMLP], ids=lambda v: str(v))
def test_lists_built_with_the_flag_off_are_rebuilt_when_it_is_on(cuda, la, over, C):
    """forward with the flag off (lists in arrival order, cached in the NeighborList), backward with it on: the
    backward rebuilds canonical lists and equals a step run wholly under the flag"""
    mod, sd, b, gout, ref = _run_family_det(cuda, la, over, C)
    pt_utils.clear_neighbor_cache()
    mod.load_state_dict(sd)
    for p in mod.parameters():
        p.grad = None
    f = b["features"].clone().requires_grad_(True)
    out = mod(b["xyz"], b["xyz"], b["mask"], b["mask"], f)
    torch.use_deterministic_algorithms(True)
    try:
        out.backward(gout)
        torch.cuda.synchronize()
    finally:
        torch.use_deterministic_algorithms(False)
    got = [out.detach(), f.grad] + [p.grad for p in mod.parameters()] + _state(mod)
    for i, (a, e) in enumerate(zip(got, ref)):
        assert torch.equal(a, e), f"tensor {i}"


def _run_family_det(cuda, la, over, C):
    torch.use_deterministic_algorithms(True)
    try:
        return _run_family(cuda, la, over, C, 2, 2304, 16, graph=False)
    finally:
        torch.use_deterministic_algorithms(False)


@pytest.mark.parametrize("la,over,C", FAMILIES, ids=lambda v: str(v))
def test_still_matches_the_oracle(cuda, oracle_ext, det, la, over, C):
    _sibling("test_local_aggregation_gpu").run_case(cuda, oracle_ext, la, over, 2, 1024, 16, C, seed=21)


# ---------------------------------------------------------------------------------------------------------------
# max-pool, upsample, grouping: the gather forms
# ---------------------------------------------------------------------------------------------------------------
def _pool_runs(cuda, fn, inputs, grad):
    """fn(*inputs) -> out; returns (out, d/dfeatures) for three runs, overlap off, cache off, beside a matmul"""
    res = []
    was_cache, was_overlap = pt_utils.cache_enabled, pt_utils.overlap_enabled
    try:
        for arm in ("a", "b", "c", "overlap", "cache", "busy"):
            pt_utils.clear_neighbor_cache()
            pt_utils.overlap_enabled = arm != "overlap"
            pt_utils.cache_enabled = arm != "cache"
            st = _busy_matmul(cuda)[0] if arm == "busy" else None
            f = inputs[-1].clone().requires_grad_(True)
            out = fn(*inputs[:-1], f)
            out.backward(grad(out))
            if st is not None:
                torch.cuda.current_stream().wait_stream(st)
            torch.cuda.synchronize()
            res.append((out.detach().clone(), f.grad.clone()))
    finally:
        pt_utils.cache_enabled, pt_utils.overlap_enabled = was_cache, was_overlap
    return res


@pytest.mark.parametrize("what", ["maxpool", "upsample_nearest", "upsample_max", "grouping"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_pool_and_grouping_are_repeatable_and_correct(cuda, what, dtype):
    B, N, C, K = 2, 4000, 40, 26
    d = {k: v.to(cuda) for k, v in synth.make_cloud_batch(B, N, C, 17).items()}
    xyz, mask, feats = d["xyz"], d["mask"], d["features"].to(dtype)
    r = synth.ball_radius(N, K)
    g = torch.Generator(device=cuda).manual_seed(2)
    grad = lambda out: torch.randn(out.shape, device=cuda, generator=g.manual_seed(2)).to(out.dtype)
    if what == "maxpool":
        pool = pt_utils.MaskedMaxPool(N // 4, r, K, 2 * r)
        fn = lambda x, m, f: pool(x, m, f)[2]
        inputs = (xyz, mask, feats)
    elif what == "grouping":
        idx = pt_utils.neighbors(xyz, xyz, mask, mask, r, K).wait().idx
        fn = lambda i, f: pt_utils.grouping_operation(f, i)
        inputs = (idx, feats)
    else:
        sub_xyz, sub_mask = pt_utils.masked_grid_subsampling(xyz, mask, N // 4, 2 * r)
        sub_f = feats[:, :, :N // 4].contiguous()
        up = pt_utils.MaskedUpsample(2 * r, K, mode=what.split("_")[1])
        fn = lambda ux, x, um, m, f: up(ux, x, um, m, f)
        inputs = (xyz, sub_xyz.contiguous(), mask, sub_mask.contiguous(), sub_f)
    torch.use_deterministic_algorithms(True)
    try:
        runs = _pool_runs(cuda, fn, inputs, grad)
    finally:
        torch.use_deterministic_algorithms(False)
    for out, gf in runs[1:]:
        assert torch.equal(out, runs[0][0]) and torch.equal(gf, runs[0][1])
    # the default (atomic) path computes the same sums in another order
    out, gf = _pool_runs(cuda, fn, inputs, grad)[0]
    assert torch.equal(out, runs[0][0])
    scale = max(1.0, float(gf.float().abs().max()))
    tol = 1e-5 if dtype == torch.float32 else 1e-2
    assert float((gf.float() - runs[0][1].float()).abs().max()) <= tol * scale


# ---------------------------------------------------------------------------------------------------------------
# whole networks: tools/train_synth.py --deterministic in child processes
# ---------------------------------------------------------------------------------------------------------------
NETWORKS = [
    ("classification", "pseudo_grid", []),
    ("scene_segmentation", "pointwisemlp", []),
    ("multi_part_segmentation", "adaptive_weight", ["--dataset", "shapenetpart"]),
]


def _train(task, la, extra, amp):
    import json
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable, os.path.join(root, "tools", "train_synth.py"), "--task", task, "--la", la, "--batch", "2",
           "--points", "3000", "--steps", "3", "--warmup", "0", "--deterministic", "--no-dropout", "--amp", amp] + extra
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=root)
    assert r.returncode == 0, f"{task} {la} {amp}: exit {r.returncode}\n{r.stderr[-3000:]}"
    return json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("{")][-1])


@pytest.mark.parametrize("amp", ["off", "bf16"])
@pytest.mark.parametrize("task,la,extra", NETWORKS, ids=lambda v: str(v))
def test_whole_network_steps_are_repeatable(cuda, task, la, extra, amp):
    """two runs of three SGD steps from the same state: identical losses, parameters and running statistics"""
    a, b = _train(task, la, extra, amp), _train(task, la, extra, amp)
    assert a["deterministic"] and len(a["losses"]) == 3
    assert a["losses"] == b["losses"]
    assert a["state_sha256"] == b["state_sha256"]
