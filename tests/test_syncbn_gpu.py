"""GPU: fused operators under nn.SyncBatchNorm (ops.bn_sync_group).

Ranks are spawned processes with a file:// rendezvous: NCCL, one GPU per rank, when the machine has two GPUs, else two
processes on one GPU over gloo.  Every process is joined with a deadline and killed past it.  Each rank runs its own
reference (the whole batch through plain BatchNorm, in one process), so only small results travel back.

  1. world size 1 (no process group, and a 1-rank group): a converted model is bit for bit the unconverted one;
  2. two ranks holding shards (even, uneven, the per-GPU c4 shape) against one process with the whole batch, every
     fused family, fp32 and bf16 autocast: outputs and d/dfeatures within 1e-5 of their largest value (plus one unit in
     the last place of a 16-bit output), the rank sum of every parameter gradient within 1e-4, running statistics within
     1e-6 relative, num_batches_tracked equal;
  3. channels whose mean is 1e2..1e4 times their spread, split over the ranks: statistics against float64;
  4. deterministic mode: two runs agree bit for bit and both ranks hold the same statistics;
  5. a scene-segmentation network on two ranks against one rank with the whole batch, per stage;
  6. GraphedStep over a SyncBatchNorm LocalAggregation with NCCL: the replay equals the eager step.
"""
import copy
import os
import time

import numpy as np
import pytest
import torch

from closerlook3d_b200 import dist as cdist, ops, synth
from closerlook3d_b200.config import la_config

pytestmark = pytest.mark.gpu

XYZ = dict(pospool=dict(position_embedding="xyz", reduction="avg"))
SINCOS = dict(pospool=dict(position_embedding="sin_cos", reduction="avg"))
AW = dict(adaptive_weight=dict(weight_type="dp", num_mlps=1, shared_channels=1, reduction="avg"))
PW = dict(pointwisemlp=dict(feature_type="dp_fi_df", num_mlps=1, reduction="max"))
FAMILIES = {"pospool-xyz": ("pospool", XYZ), "pospool-sincos": ("pospool", SINCOS),
            "adaptive_weight": ("adaptive_weight", AW), "pseudo_grid": ("pseudo_grid", {}), "pointwisemlp": ("pointwisemlp", PW)}
# (clouds in the whole batch, N, K, C): small layers, a deep-stage layer (88 queries per cloud) and the per-GPU
# BASELINE c4 shape (32 clouds over 8 GPUs: 4 per rank)
SHAPES = {"small": (3, 1024, 16, 24), "deep": (4, 88, 16, 72), "c4": (8, 10000, 32, 72)}
DEADLINE_S = 900


# ---- process plumbing ---------------------------------------------------------------------------------------------
def _worker(job, rank, world, init, backend, out_dir, kw):
    import torch.distributed as dist
    dev = torch.device("cuda", rank if backend == "nccl" else 0)
    torch.cuda.set_device(dev)
    extra = {"device_id": dev} if backend == "nccl" else {}
    dist.init_process_group(backend, init_method=init, rank=rank, world_size=world, **extra)
    try:
        res = globals()[job](rank, world, dev, **kw)
        torch.save(res, os.path.join(out_dir, f"{job}_{rank}.pt"))
        dist.barrier()
    finally:
        dist.destroy_process_group()


def _backend(world=2):
    return "nccl" if torch.cuda.device_count() >= world else "gloo"


def _spawn(job, tmp_path, world=2, backend=None, **kw):
    """run globals()[job](rank, world, device, **kw) on `world` spawned ranks -> their results in rank order"""
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    init = "file://" + str(tmp_path / f"rdv_{job}_{time.monotonic_ns()}")
    procs = [ctx.Process(target=_worker, args=(job, r, world, init, backend or _backend(world), str(tmp_path), kw))
             for r in range(world)]
    for p in procs:
        p.start()
    t_end = time.monotonic() + DEADLINE_S
    try:
        for p in procs:
            p.join(timeout=max(1.0, t_end - time.monotonic()))
    finally:
        for p in procs:
            if p.is_alive():
                p.kill()
                p.join(30)
    codes = [p.exitcode for p in procs]
    assert codes == [0] * world, f"{job}: rank exit codes {codes}"
    return [torch.load(tmp_path / f"{job}_{r}.pt") for r in range(world)]


# ---- one layer ----------------------------------------------------------------------------------------------------
def _layer(fam, C, N, K, seed):
    from closerlook3d_b200.local_aggregation_operators import LocalAggregation
    la, over = FAMILIES[fam]
    torch.manual_seed(seed)
    np.random.seed(seed)
    mod = LocalAggregation(C, C, synth.ball_radius(N, K), K, la_config(la, **over))
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for name, p in mod.named_parameters():     # BatchNorm affine parameters away from (1, 0)
            if "out_transform" in name or ".1." in name:
                p.copy_((1.0 + 0.5 * torch.randn(p.shape, generator=g)) if name.endswith("weight")
                        else 0.5 * torch.randn(p.shape, generator=g))
        for name, b in mod.named_buffers():
            if name.endswith("running_var"):
                b.copy_(0.5 + torch.rand(b.shape, generator=g))
            elif name.endswith("running_mean"):
                b.copy_(torch.randn(b.shape, generator=g))
    return mod


def _batch(B, N, C, seed, dev):
    d = {k: v.to(dev) for k, v in synth.make_cloud_batch(B, N, C, seed).items()}
    d["gout"] = torch.randn(B, C, N, generator=torch.Generator().manual_seed(seed + 2)).to(dev)
    return d


def _step(mod, d, lo, hi, dtype, steps=1):
    """`steps` training steps of mod on clouds [lo, hi) -> (out, d/dfeatures, {name: grad}) of the last; 16-bit
    features under autocast for dtype=bfloat16"""
    from closerlook3d_b200 import pt_utils
    xyz, mask = d["xyz"][lo:hi].contiguous(), d["mask"][lo:hi].contiguous()
    for _ in range(steps):
        pt_utils.clear_neighbor_cache()
        for p in mod.parameters():
            p.grad = None
        f = d["features"][lo:hi].to(dtype, copy=True).requires_grad_(True)
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=dtype == torch.bfloat16):
            out = mod(xyz, xyz, mask, mask, f)
        out.backward(d["gout"][lo:hi].to(out.dtype))
    return out.detach(), f.grad.detach(), {n: p.grad.detach().clone() for n, p in mod.named_parameters()}


def _stats(mod):
    return {n: b.detach().clone() for n, b in mod.named_buffers() if "running" in n or "num_batches" in n}


def _ulp16(x):
    _, e = torch.frexp(x.float())
    return torch.ldexp(torch.ones_like(x, dtype=torch.float32), (e - 1).clamp(min=-126) - 7)


def _err(a, b):
    """max |a - b| over max(1, max |b|), less one bf16 ulp of b where a is bf16"""
    d = (a.float() - b.float()).abs()
    if a.dtype == torch.bfloat16:
        d = (d - _ulp16(b)).clamp(min=0)
    return float(d.max()) / max(1.0, float(b.float().abs().max()))


def shards_job(rank, world, dev, cases):
    """check 2 on this rank: per case its errors against the whole-batch plain-BatchNorm run, its local parameter
    gradients and the reference's, and the running statistics of both"""
    out = {}
    for fam, shape, sizes, dtype in cases:
        B, N, K, C = SHAPES[shape]
        B = sum(sizes)
        lo = sum(sizes[:rank])
        hi = lo + sizes[rank]
        seed = 100 + len(fam) + C + B
        mod = _layer(fam, C, N, K, seed).to(dev).train()
        sync = torch.nn.SyncBatchNorm.convert_sync_batchnorm(copy.deepcopy(mod))
        d = _batch(B, N, C, seed, dev)
        o_r, gf_r, gp_r = _step(mod, d, 0, B, dtype, steps=2)
        o, gf, gp = _step(sync, d, lo, hi, dtype, steps=2)
        out[(fam, shape, tuple(sizes), str(dtype))] = dict(
            out=_err(o, o_r[lo:hi]), dfeat=_err(gf, gf_r[lo:hi]), dtypes=(str(o.dtype), str(gf.dtype)),
            grads={n: g.cpu() for n, g in gp.items()}, grads_ref={n: g.cpu() for n, g in gp_r.items()},
            stats={n: b.cpu() for n, b in _stats(sync).items()}, stats_ref={n: b.cpu() for n, b in _stats(mod).items()})
        del mod, sync, d
        torch.cuda.empty_cache()
    return out


def _check_shards(results):
    for key in results[0]:
        per = [r[key] for r in results]
        for r in per:
            assert r["dtypes"] == (key[3], key[3]), key
            assert r["out"] <= 1e-5 and r["dfeat"] <= 1e-5, (key, r["out"], r["dfeat"])
        ref = per[0]["grads_ref"]
        for n, g_ref in ref.items():
            g = sum(r["grads"][n] for r in per)
            err = float((g - g_ref).abs().max()) / max(1.0, float(g_ref.abs().max()))
            assert err <= 1e-4, (key, n, err)
        for r in per:
            for n, b_ref in r["stats_ref"].items():
                b = r["stats"][n]
                if "num_batches" in n:
                    assert torch.equal(b, b_ref), (key, n)
                else:
                    err = float((b - b_ref).abs().max()) / float(b_ref.abs().max())
                    assert err <= 1e-6, (key, n, err)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
def test_two_ranks_match_one_process_with_the_whole_batch(cuda, tmp_path, dtype):
    cases = []
    for fam in FAMILIES:
        cases += [(fam, "small", (2, 1), dtype), (fam, "small", (2, 2), dtype), (fam, "deep", (2, 2), dtype),
                  (fam, "c4", (4, 4), dtype)]
    _check_shards(_spawn("shards_job", tmp_path, cases=cases))


# ---- world size 1 -------------------------------------------------------------------------------------------------
def _bit_identical_to_plain(cuda):
    """check 1 in this process: every family, converted against unconverted, deterministic mode (no atomics)"""
    B, N, K, C = SHAPES["small"]
    torch.use_deterministic_algorithms(True)
    try:
        for fam in FAMILIES:
            mod = _layer(fam, C, N, K, 7).to(cuda).train()
            sync = torch.nn.SyncBatchNorm.convert_sync_batchnorm(copy.deepcopy(mod))
            assert any(isinstance(m, torch.nn.SyncBatchNorm) for m in sync.modules())
            d = _batch(B, N, C, 7, cuda)
            a, b = _step(mod, d, 0, B, torch.float32, steps=2), _step(sync, d, 0, B, torch.float32, steps=2)
            assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]), fam
            for n in a[2]:
                assert torch.equal(a[2][n], b[2][n]), (fam, n)
            for (n, x), y in zip(_stats(mod).items(), _stats(sync).values()):
                assert torch.equal(x, y), (fam, n)
    finally:
        torch.use_deterministic_algorithms(False)


def test_world_size_one_is_bit_identical_to_plain_batchnorm(cuda, tmp_path):
    import torch.distributed as dist
    assert not dist.is_initialized()
    _bit_identical_to_plain(cuda)                  # no process group
    dist.init_process_group("gloo", init_method="file://" + str(tmp_path / "rdv1"), rank=0, world_size=1)
    try:
        assert cdist.world_size() == 1
        _bit_identical_to_plain(cuda)              # a 1-rank group: torch's rule does not synchronise
    finally:
        dist.destroy_process_group()


def test_fused_head_eligibility_follows_the_sync_rule(cuda, tmp_path):
    """the fused multi-shape head keeps per-GPU statistics: it stands aside only when the BatchNorm would synchronise"""
    _spawn("head_job", tmp_path)


def head_job(rank, world, dev):
    from closerlook3d_b200 import partseg
    import torch.nn as nn
    C = 32
    heads = nn.ModuleList([nn.Sequential(nn.Conv1d(C, C, 1, bias=False), nn.BatchNorm1d(C), nn.ReLU(),
                                         nn.Conv1d(C, n, 1)) for n in (3, 5)]).to(dev)
    x = torch.randn(2, C, 100, device=dev)
    assert partseg.fused_eligible(heads, x)
    sync = nn.SyncBatchNorm.convert_sync_batchnorm(copy.deepcopy(heads))
    assert not partseg.fused_eligible(sync.train(), x)
    assert partseg.fused_eligible(sync.eval(), x)
    return {}


# ---- large-mean channels ------------------------------------------------------------------------------------------
def _tile_partials(x):
    """(ntiles, n, C) float64 values -> this library's (ntiles, 4, C) fp32 BatchNorm partials of their fp32 values,
    formed as the forward kernels form them (centre = the tile's fp32 mean)"""
    v = x.float()
    c = v.mean(1)
    e = v - c[:, None]
    n = torch.full_like(c, x.shape[1])
    return torch.stack([n, c, e.sum(1), (e * e).sum(1)], 1).contiguous()


def large_mean_job(rank, world, dev):
    C, n = 12, 128
    ratios = torch.tensor([1e2, 1e3, 1e4] * 4, dtype=torch.float64)
    g = torch.Generator().manual_seed(11)
    mean = (1.0 + torch.rand(C, generator=g, dtype=torch.float64)) * 1e3
    ntiles = [37, 12][:world]
    full = mean + mean / ratios * torch.randn(sum(ntiles), n, C, generator=g, dtype=torch.float64)
    full = full.float().double()                   # the values the kernels would see
    lo = sum(ntiles[:rank])
    part = _tile_partials(full[lo:lo + ntiles[rank]]).to(dev)
    rm = torch.zeros(C, device=dev)
    rv = torch.ones(C, device=dev)
    stats, count = ops.bn_finalize_ranks(part, C, ntiles[rank] * n, 1e-30, 1.0, rm, rv, torch.distributed.group.WORLD)
    return dict(stats=stats.cpu(), rm=rm.cpu(), rv=rv.cpu(), count=count.cpu(), values=full if rank == 0 else None)


def test_large_mean_channels_split_over_ranks(cuda, tmp_path):
    res = _spawn("large_mean_job", tmp_path)
    full = res[0]["values"].reshape(-1, res[0]["values"].shape[-1])
    m64, v64 = full.mean(0), full.var(0, unbiased=False)
    cnt = full.shape[0]
    for r in res:
        assert float(r["count"]) == cnt
        assert float(((r["stats"][0].double() - m64).abs() - 1e-6 * m64.abs()).max()) <= 1e-5 * float(v64.sqrt().min())
        var = 1.0 / r["stats"][1].double() ** 2
        assert float(((var - v64) / v64).abs().max()) <= 1e-5
        assert float(((r["rv"].double() - v64 * cnt / (cnt - 1)) / v64).abs().max()) <= 1e-5
        assert torch.equal(r["stats"], res[0]["stats"]) and torch.equal(r["rv"], res[0]["rv"])


# ---- deterministic mode -------------------------------------------------------------------------------------------
def det_job(rank, world, dev):
    B, N, K, C = SHAPES["small"]
    sizes = (2, 1)
    lo = sum(sizes[:rank])
    saved = []
    fin = ops.bn_finalize_ranks

    def record(*a, **k):
        s, c = fin(*a, **k)
        saved.append(s.clone())
        return s, c

    ops.bn_finalize_ranks = record
    torch.use_deterministic_algorithms(True)
    out = {}
    try:
        for fam in FAMILIES:
            runs = []
            for _ in range(2):
                saved.clear()
                mod = torch.nn.SyncBatchNorm.convert_sync_batchnorm(_layer(fam, C, N, K, 3)).to(dev).train()
                d = _batch(3, N, C, 3, dev)
                o, gf, gp = _step(mod, d, lo, lo + sizes[rank], torch.float32, steps=2)
                runs.append((o, gf, gp, _stats(mod), [s.cpu() for s in saved]))
            (o1, g1, p1, s1, st1), (o2, g2, p2, s2, st2) = runs
            assert torch.equal(o1, o2) and torch.equal(g1, g2), fam
            assert all(torch.equal(p1[n], p2[n]) for n in p1), fam
            assert all(torch.equal(s1[n], s2[n]) for n in s1), fam
            assert len(st1) == 2 and all(torch.equal(a, b) for a, b in zip(st1, st2)), fam
            out[fam] = dict(save_stats=st1, stats={n: b.cpu() for n, b in s1.items()})
    finally:
        torch.use_deterministic_algorithms(False)
        ops.bn_finalize_ranks = fin
    return out


def test_deterministic_two_rank_step(cuda, tmp_path):
    res = _spawn("det_job", tmp_path)
    for fam in FAMILIES:
        a, b = res[0][fam], res[1][fam]
        assert all(torch.equal(x, y) for x, y in zip(a["save_stats"], b["save_stats"])), fam
        assert all(torch.equal(a["stats"][n], b["stats"][n]) for n in a["stats"]), fam


# ---- whole network ------------------------------------------------------------------------------------------------
def network_job(rank, world, dev):
    from closerlook3d_b200 import backbone as bb, pt_utils
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    c = bb.model_config("scene_segmentation", "pseudo_grid")
    c.width, c.radius, c.sampleDl = 24, 0.06, 0.03
    c.npoints, c.nsamples, c.num_classes = [1024, 320, 96, 32], [16, 18, 20, 18, 16], 9
    torch.manual_seed(3)
    np.random.seed(3)
    model = bb.build_scene_segmentation(c)[0]
    model.init_weights()
    for m in model.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    model = model.to(dev).train()
    sync = torch.nn.SyncBatchNorm.convert_sync_batchnorm(copy.deepcopy(model))
    B, N = 4, 3000
    d = {k: v.to(dev) for k, v in synth.make_cloud_batch(B, N, c.input_features_dim, 21).items()}
    lo, hi = cdist.shard_range(B, world, rank)

    def run(m, a, b):
        pt_utils.clear_neighbor_cache()
        ep = {}
        h = m.backbone.register_forward_hook(lambda mod, args, res: ep.update(res))
        with torch.no_grad():
            m(d["xyz"][a:b].contiguous(), d["mask"][a:b].contiguous(), d["features"][a:b].contiguous())
        h.remove()
        return {k: v.cpu() for k, v in ep.items() if k.endswith("_features")}, _stats(m)

    ep_ref, st_ref = run(model, 0, B)
    ep, st = run(sync, lo, hi)
    return dict(res={k: (float((ep[k] - ep_ref[k][lo:hi]).norm()) / max(1e-20, float(ep_ref[k][lo:hi].norm())))
                     for k in ep},
                stats=max(float(((st[n] - st_ref[n]).abs().max()) / max(1e-20, float(st_ref[n].abs().max())))
                          for n in st if "running" in n),
                nbt=all(torch.equal(st[n], st_ref[n]) for n in st if "num_batches" in n))


def test_scene_segmentation_network_on_two_ranks(cuda, tmp_path):
    for r in _spawn("network_job", tmp_path):
        m = r["res"]
        print("SYNCBN-NETWORK", {k: f"{v:.2e}" for k, v in m.items()}, f"running {r['stats']:.2e}")
        # tests/test_model_gpu.py's per-stage bars
        assert m["res1_features"] <= 2e-5 and m["res2_features"] <= 2e-4 and m["res5_features"] <= 2e-4, m
        assert r["stats"] <= 1e-2 and r["nbt"]


# ---- CUDA graph ---------------------------------------------------------------------------------------------------
def graph_job(rank, world, dev):
    from closerlook3d_b200 import pt_utils
    from closerlook3d_b200.graphed import GraphedStep
    B, N, K, C = 2, 2304, 16, 72
    out = {}
    for fam in ("adaptive_weight", "pointwisemlp"):
        mod = torch.nn.SyncBatchNorm.convert_sync_batchnorm(_layer(fam, C, N, K, 5)).to(dev).train()
        d = _batch(B * world, N, C, 5, dev)
        lo, hi = B * rank, B * (rank + 1)
        was = pt_utils.cache_enabled
        pt_utils.cache_enabled = False
        try:
            gs = GraphedStep(mod, d["xyz"][lo:hi], d["mask"][lo:hi], d["features"][lo:hi], d["gout"][lo:hi],
                             allreduce=False)
            state = copy.deepcopy(mod.state_dict())
            gs.replay()
            torch.cuda.synchronize()
            g_out, g_feat, g_par = gs.out.clone(), gs.features.grad.clone(), [g.clone() for g in gs.param_grads]
            g_stats = _stats(mod)
            mod.load_state_dict(state)
            o, gf, gp = _step(mod, d, lo, hi, torch.float32)
        finally:
            pt_utils.cache_enabled = was
        assert float((g_out - o).abs().max()) <= 2e-6 * max(1.0, float(o.abs().max())), fam
        assert float((g_feat - gf).abs().max()) <= 1e-5 * max(1.0, float(gf.abs().max())), fam
        for a, (n, b) in zip(g_par, gp.items()):
            assert float((a - b).abs().max()) <= 5e-5 * max(1.0, float(b.abs().max())), (fam, n)
        for n, b in _stats(mod).items():
            assert torch.allclose(g_stats[n].float(), b.float(), rtol=1e-6, atol=0), (fam, n)
        del gs
        out[fam] = True
    return out


def test_graphed_step_with_sync_batchnorm_nccl(cuda, tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("GraphedStep with a captured NCCL all_gather needs two GPUs (NCCL runs one rank per GPU)")
    _spawn("graph_job", tmp_path, backend="nccl")
