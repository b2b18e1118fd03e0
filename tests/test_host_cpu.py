"""CPU tests (-m "not gpu") of the host side: C-ABI surface, drop-in module surface, error behaviour,
configuration defaults, synthetic generators, data-parallel plumbing (gloo, world_size 2)."""
import ctypes
import os
import re
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_functions():
    hdr = open(os.path.join(ROOT, "include", "cl3d.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    return sorted(set(re.findall(r"\b(cl3d_[a-z0-9_]+)\s*\(", hdr)))


def test_library_exports_every_declared_symbol():
    from closerlook3d_b200 import _lib, build
    so = build.build()
    cdll = ctypes.CDLL(so)
    names = _declared_functions()
    assert len(names) >= 25
    for n in names:
        assert hasattr(cdll, n), f"{n} declared in include/cl3d.h but not exported by libcl3d.so"
        assert n in _lib.SIGNATURES, f"{n} has no ctypes signature in closerlook3d_b200/_lib.py"
    for n in _lib.SIGNATURES:
        assert n in names, f"{n} bound in _lib.py but not declared in include/cl3d.h"
    L = _lib.lib()
    assert L.cl3d_version() >= 100
    assert L.cl3d_padded_channels(66) == 72 and L.cl3d_padded_channels(72) == 72


def test_sass_has_no_legacy_arch():
    """the library is sm_90a only"""
    so = os.path.join(ROOT, "closerlook3d_b200", "libcl3d.so")
    out = subprocess.run(["cuobjdump", "-lelf", so], capture_output=True, text=True).stdout
    archs = set(re.findall(r"sm_(\d+a?)", out))
    assert archs == {"90a"}, archs


def test_state_dict_keys_match_reference_layout():
    from closerlook3d_b200.config import la_config
    from closerlook3d_b200.local_aggregation_operators import LocalAggregation
    P = "local_aggregation_operator."
    bn = lambda p: [p + s for s in ("weight", "bias", "running_mean", "running_var", "num_batches_tracked")]
    want = {
        "pospool": bn(P + "out_transform.0."),
        "adaptive_weight": [P + "mlps.conv0.weight", P + "mlps.conv0.bias"] + bn(P + "out_transform.0."),
        "pointwisemlp": [P + "mlps.conv0.0.weight"] + bn(P + "mlps.conv0.1."),
        "pseudo_grid": [P + "kernel_weights", P + "K_points"] + bn(P + "out_transform.0."),
    }
    for t, keys in want.items():
        m = LocalAggregation(24, 24, 0.1, 8, la_config(t, pointwisemlp=dict(feature_type="dp_fi_df")))
        assert list(m.state_dict().keys()) == keys, t
    m = LocalAggregation(24, 48, 0.1, 8, la_config("pospool"))  # C_in != C_out -> out_conv, as the reference
    assert P + "out_conv.0.weight" in m.state_dict() and P + "out_conv.1.running_var" in m.state_dict()
    sd = m.state_dict()
    assert sd[P + "out_conv.0.weight"].shape == (48, 24, 1)
    pw = LocalAggregation(24, 24, 0.1, 8, la_config("pointwisemlp", pointwisemlp=dict(feature_type="dp_fi_df")))
    assert pw.state_dict()[P + "mlps.conv0.0.weight"].shape == (24, 3 + 48, 1, 1)
    pg = LocalAggregation(24, 24, 0.1, 8, la_config("pseudo_grid"))
    assert pg.state_dict()[P + "K_points"].shape == (15, 3) and float(pg.state_dict()[P + "K_points"][0].abs().max()) == 0


def test_error_behaviour_matches_reference_conventions():
    from closerlook3d_b200 import ops
    from closerlook3d_b200.config import la_config
    from closerlook3d_b200.local_aggregation_operators import LocalAggregation
    x = torch.rand(1, 8, 3)
    m = torch.ones(1, 8, dtype=torch.int32)
    la = LocalAggregation(24, 24, 0.1, 4, la_config("pospool", pospool=dict(reduction="avg")))
    with pytest.raises(RuntimeError, match="CUDA"):           # CPU tensors: "CPU not supported" -> RuntimeError
        la(x, x, m, m, torch.rand(1, 24, 8))
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.ball_query(x, x, m, m, 0.1, 4)
    with pytest.raises(NotImplementedError):                  # same unsupported settings as the reference
        LocalAggregation(24, 24, 0.1, 4, la_config("nope"))
    bad = LocalAggregation(24, 24, 0.1, 4, la_config("pointwisemlp"))  # default feature_type 'dp_fj'
    with pytest.raises(NotImplementedError, match="Feature Type"):
        bad(x, x, m, m, torch.rand(1, 24, 8))
    aw = LocalAggregation(24, 24, 0.1, 4, la_config("adaptive_weight", adaptive_weight=dict(weight_type="df")))
    with pytest.raises(NotImplementedError, match="Weight Type"):
        aw(x, x, m, m, torch.rand(1, 24, 8))


def test_reference_models_import_with_the_drop_in_modules():
    """the reference's models/ build on top of this package's pt_utils / operators (needs a reference checkout)"""
    from oracle.ref_loader import REF_ROOT
    if not os.path.isdir(os.path.join(REF_ROOT, "models")):
        pytest.skip(f"no reference checkout at {REF_ROOT} (set CL3D_REFERENCE)")
    code = r'''
import sys, types
sys.path.insert(0, %r)
from closerlook3d_b200 import shim
shim.install(%r)
from models.backbones.resnet import ResNet
import closerlook3d_b200.local_aggregation_operators as mine
import models.local_aggregation_operators as theirs
assert theirs.LocalAggregation is mine.LocalAggregation
import models.backbones.resnet as rn
assert rn.LocalAggregation is mine.LocalAggregation, "resnet bound the reference's unfused LocalAggregation"
import pt_utils as ptu, closerlook3d_b200.pt_utils as mine_ptu
assert ptu is mine_ptu and rn.MaskedMaxPool is mine_ptu.MaskedMaxPool
cfg = shim.reference_config(%r + "/cfgs/s3dis/pospool_xyz_avg.yaml")
net = ResNet(cfg, cfg.input_features_dim, cfg.radius, cfg.sampleDl, cfg.nsamples, cfg.npoints, width=cfg.width, depth=cfg.depth, bottleneck_ratio=cfg.bottleneck_ratio)
n = sum(p.numel() for p in net.parameters())
assert n > 1e6, n
las = [m for m in net.modules() if type(m).__name__ == "LocalAggregation"]
assert las and all(type(m) is mine.LocalAggregation for m in las), "backbone holds foreign LocalAggregation modules"
print("params", n)
''' % (ROOT, REF_ROOT, REF_ROOT)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]


def test_config_defaults_and_baseline_table():
    from closerlook3d_b200.config import baseline_config, la_config
    c = la_config()
    assert c.bn_momentum == 0.1 and c.density_parameter == 5.0 and c.pospool.reduction == "sum"
    assert c.pseudo_grid.num_kernel_points == 15 and c.adaptive_weight.shared_channels == 1
    shapes = [(2, 1024, 16, 66), (32, 1024, 32, 72), (8, 15000, 26, 72), (32, 10000, 32, 72), (64, 40000, 40, 144)]
    for i, (B, N, K, C) in enumerate(shapes, 1):
        t = baseline_config(i)
        assert (t["B"], t["N"], t["K"], t["C"]) == (B, N, K, C)


def test_synth_is_deterministic_and_prefix_masked():
    from closerlook3d_b200 import synth
    a = synth.make_cloud_batch(5, 200, 6, 3)
    b = synth.make_cloud_batch(5, 200, 6, 3)
    assert all(torch.equal(a[k], b[k]) for k in a)
    for bi in range(5):
        nv = 200 - (bi % 4) * 10
        assert int(a["mask"][bi].sum()) == nv and bool((a["mask"][bi, :nv] == 1).all())
        if nv < 200:  # padded rows duplicate valid rows
            d = (a["xyz"][bi, nv:, None, :] - a["xyz"][bi, None, :nv, :]).abs().sum(-1).min(1)[0]
            assert float(d.max()) == 0.0
    assert abs(synth.ball_radius(15000, 26) - 0.0853) < 1e-3


def _gloo_worker(rank, world, port, q):
    import torch.distributed as dist
    from closerlook3d_b200 import dist as cdist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    lo, hi = cdist.shard_range(10, world, rank)
    torch.manual_seed(0)
    w = torch.nn.Linear(4, 3)
    x = torch.arange(40, dtype=torch.float32).view(10, 4)[lo:hi]
    w(x).sum().backward()
    cdist.allreduce_gradients(list(w.parameters()), average=False)
    g_copy = (w.weight.grad.tolist(), w.bias.grad.tolist())
    # the same exchange through the persistent flat buffer (p.grad are views: one collective, nothing copied)
    w2 = torch.nn.Linear(4, 3)
    w2.load_state_dict(w.state_dict())
    fg = cdist.FlatGradients(list(w2.parameters())).attach()
    fg.zero()
    w2(x).sum().backward()
    assert w2.weight.grad.data_ptr() == fg.flat.data_ptr()          # autograd accumulated in place
    cdist.allreduce_gradients(list(w2.parameters()), average=False)  # takes the no-copy path
    assert w2.weight.grad.tolist() == g_copy[0] and w2.bias.grad.tolist() == g_copy[1]
    fg.zero()
    w2(x).sum().backward()
    fg.allreduce(average=True)
    assert torch.allclose(w2.weight.grad * world, torch.tensor(g_copy[0]))
    # plain lists: a tensor would travel as a shared-memory handle that dies with this process
    q.put((rank, lo, hi, g_copy[0], g_copy[1]))
    dist.barrier()
    dist.destroy_process_group()


def test_data_parallel_plumbing_gloo_world2():
    """batch sharding + gradient all-reduce (the only exchange on the path) with gloo, world_size 2"""
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + (os.getpid() % 400)
    procs = [ctx.Process(target=_gloo_worker, args=(r, 2, port, q)) for r in range(2)]
    [p.start() for p in procs]
    res = sorted([q.get(timeout=120) for _ in procs], key=lambda t: t[0])
    [p.join(timeout=60) for p in procs]
    assert (res[0][1], res[0][2], res[1][1], res[1][2]) == (0, 5, 5, 10)
    torch.manual_seed(0)
    w = torch.nn.Linear(4, 3)
    w(torch.arange(40, dtype=torch.float32).view(10, 4)).sum().backward()
    for r in res:
        assert torch.allclose(torch.tensor(r[3]), w.weight.grad) and torch.allclose(torch.tensor(r[4]), w.bias.grad)
