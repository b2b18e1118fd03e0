"""Turn the light ncu CSV logs of tools/capture_traffic.sh into profiles/traffic.json:
   python tools/ncu_traffic.py gpurun_out/r2r_traffic_c{1,2,3,4,5}.csv > profiles/traffic.json
Per config: DRAM bytes and device time per step of every C-ABI entry point (kernels mapped to entry points), the
step total against the SURVEY 8(d) algorithmic bytes, and the kernel list with times (the launch list)."""
import collections, csv, json, os, re, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from closerlook3d_b200.config import baseline_config

MAP = [("gemm_tf32x3", "cl3d_sgemm_algo"), ("sgemm", "cl3d_sgemm_algo"), ("splitk_reduce", "cl3d_sgemm_algo"),
       ("ball_query", "cl3d_ball_query_csr"), ("grid_build_fused", "cl3d_ball_query_csr"), ("csr_", "cl3d_ball_query_csr"),
       ("pg2_kernel<(bool)0", "cl3d_agg_fwd"), ("pg2_kernel<(bool)1", "cl3d_agg_bwd"), ("pg2_kernel<0", "cl3d_agg_fwd"),
       ("pg2_kernel<1", "cl3d_agg_bwd"), ("pg3_bwd_kernel", "cl3d_agg_bwd"), ("pg3_fwd_kernel", "cl3d_agg_fwd"),
       ("aggmax_fwd", "cl3d_agg_fwd"), ("aggmax_bwd", "cl3d_agg_bwd"), ("nearest_query", "cl3d_nearest_query"),
       ("pwmlp_fwd_kernel", "cl3d_pwmlp_fwd_stats"), ("pwmlp_bwd", "cl3d_pwmlp_bwd"),
       ("agg_fwd", "cl3d_agg_fwd"), ("sincos_fwd", "cl3d_agg_fwd"), ("agg_bwd", "cl3d_agg_bwd"), ("sincos_bwd", "cl3d_agg_bwd"),
       ("bn_relu_fwd", "cl3d_bn_relu_fwd"), ("bn_relu_bwd", "cl3d_bn_relu_bwd"),
       ("bn_finalize", "cl3d_bn_finalize"), ("to_point_major_aug", "cl3d_to_point_major_aug"),
       ("to_point_major", "cl3d_to_point_major"), ("pwmlp_prep", "cl3d_pwmlp_prep_weights"),
       ("pwmlp_wgrad", "cl3d_pwmlp_weight_grad"), ("reduce_partials", "cl3d_reduce_partials"),
       ("to_channel_major", "cl3d_to_channel_major")]
SCALE = {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "nsecond": 1e-3, "ns": 1e-3, "usecond": 1, "us": 1,
         "msecond": 1e3, "ms": 1e3}
out = {}
for path in sys.argv[1:]:
    cfg = re.search(r"_c(\d)\.csv", path).group(1)
    spec = baseline_config(int(cfg))
    Bl = spec["B"] if spec["gpus"] == 1 else max(1, spec["B"] // spec["gpus"])
    rows = [r for r in csv.reader(open(path, errors="replace")) if len(r) > 8]
    h = next(r for r in rows if r[0] == "ID")
    ki, mn, mu, mv = h.index("Kernel Name"), h.index("Metric Name"), h.index("Metric Unit"), h.index("Metric Value")
    launches = collections.OrderedDict()   # id -> [name, bytes, us]
    # a capture restricted to this library's kernels (capture_traffic.sh: -k regex:cl3d on mangled names) prints the
    # names without the namespace; an unrestricted one is filtered here
    namespaced = any("cl3d::" in r[ki] for r in rows if r[0] != "ID")
    for r in rows:
        if r[0] == "ID" or (namespaced and "cl3d::" not in r[ki]):
            continue
        e = launches.setdefault(r[0], [r[ki], 0.0, 0.0])
        v = float(r[mv].replace(",", "")) * SCALE.get(r[mu], 1)
        if r[mn].startswith("dram__bytes"):
            e[1] += v
        elif r[mn].startswith("gpu__time"):
            e[2] += v
    # every family runs cl3d_bn_finalize exactly once per step: its launch count is the number of captured steps
    steps = float(max(1, sum(1 for name, _, _ in launches.values() if "bn_finalize_kernel" in name)))
    per = collections.defaultdict(lambda: [0.0, 0, 0.0])
    kern = collections.OrderedDict()
    for name, b, us in launches.values():
        ent = next((e for k, e in MAP if k in name), "other")
        per[ent][0] += b; per[ent][1] += 1; per[ent][2] += us
        short = re.sub(r"\(.*", "", name.replace("cl3d::", "").replace("void ", ""))
        k = kern.setdefault(short, [0, 0.0, 0.0])
        k[0] += 1; k[1] += us; k[2] += b
    d = {e: {"dram_bytes_per_step": v[0] / steps, "kernels": v[1] / steps, "time_us_under_ncu": v[2] / steps}
         for e, v in per.items()}
    algo = (16 * spec["C"] + 8 * spec["K"] + 32) * Bl * spec["N"]
    tot = sum(v[0] for v in per.values()) / steps
    d["_clouds_per_gpu"] = Bl
    d["_report"] = os.path.basename(path) + " (ncu --metrics dram__bytes_read.sum,dram__bytes_write.sum,gpu__time_duration.sum)"
    d["_total_dram_bytes_per_step"] = tot
    d["_algorithmic_bytes_per_step"] = algo
    d["_dram_over_algorithmic"] = tot / algo
    d["_launches_per_step"] = len(launches) / steps
    d["_steps_captured"] = steps
    d["_kernels"] = {k: {"launches_per_step": v[0] / steps, "us_per_step": v[1] / steps, "dram_mb_per_step": v[2] / steps / 1e6}
                     for k, v in kern.items()}
    out["c" + cfg] = d
print(json.dumps(out, indent=1))
