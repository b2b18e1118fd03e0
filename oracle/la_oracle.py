"""oracle/la_oracle.py -- torch restatement of the reference's python hot path (unfused, like the reference).

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).  This is the travelling checker for the GPU box, where
/root/reference does not exist: the same unfused algorithm as the reference's python layer, written
functionally on top of a pluggable `ext` (oracle.ext = C restatement on CPU tensors; or the reference's
own compiled CUDA extension from oracle/_ref on CUDA tensors, which gives the "reference GPU path").

Follows (reference, /root/reference/pytorch):
  ops/pt_custom_ops/pt_utils.py:16-61    GroupingOperation fwd/bwd
  ops/pt_custom_ops/pt_utils.py:114-144  MaskedQueryAndGroup.forward
  ops/pt_custom_ops/pt_utils.py:147-176  MaskedNearestQueryAndGroup.forward
  ops/pt_custom_ops/pt_utils.py:179-202  MaskedMaxPool.forward
  ops/pt_custom_ops/pt_utils.py:205-227  MaskedUpsample.forward
  models/local_aggregation_operators.py:47-112   PosPool.forward
  models/local_aggregation_operators.py:170-224  AdaptiveWeight.forward
  models/local_aggregation_operators.py:274-316  PointWiseMLP.forward
  models/local_aggregation_operators.py:368-426  PseudoGrid.forward

Pinned against the unmodified reference modules by tests/test_oracle_vs_reference.py (container) and through
tests/golden/*.pt (everywhere).
"""
import torch
import torch.nn.functional as F


# --------------------------------------------------------------------------------------------------
# grouping (pt_utils.py)
# --------------------------------------------------------------------------------------------------
def make_grouping(ext):
    class _Group(torch.autograd.Function):  # pt_utils.py:16-61
        @staticmethod
        def forward(ctx, features, idx):
            ctx.idx = idx
            ctx.n = features.shape[2]
            return ext.group_points(features, idx)

        @staticmethod
        def backward(ctx, grad_out):
            return ext.group_points_grad(grad_out.contiguous(), ctx.idx, ctx.n), None

    return _Group.apply


# torch's CUDA kernel for `tensor / python_scalar` multiplies by the fp32 reciprocal of the scalar
# (aten/src/ATen/native/cuda/BinaryDivTrueKernel.cu: "compute a * reciprocal(b)"), the CPU kernel divides.  The
# reference's `grouped_xyz /= self.radius` (pt_utils.py:129) therefore differs by up to 1 ulp between its GPU path
# and a CPU run -- harmless, except that PosPool sin_cos evaluates sin(100 * dp / dim): one ulp of dp is ~1e-5 rad
# there.  GPU parity tests set this flag so that the oracle follows the reference's GPU arithmetic; the pins
# against the unmodified reference modules on CPU (tests/test_oracle_cpu.py, tests/golden) keep it False.
GPU_SCALAR_DIVISION = False

# Same reason, second constant: the reference builds the sin_cos wave lengths with torch.pow ON THE DEVICE of the
# inputs (local_aggregation_operators.py:72-75).  CPU torch.pow is vectorised differently on different hosts
# (AVX2 body + scalar tail vs AVX-512), so its last bit is host dependent, and one ulp of a wave length moves
# sin(100*dp/dim) by up to ~3e-6 coherently over a channel.  GPU parity tests install a function here that
# evaluates the reference's expression on the GPU (fd -> (fd,) float32 CPU tensor); None = evaluate on the CPU.
DIM_MAT_FN = None

# Checker-side diagnostics: when this is a dict, pointwise_mlp() leaves its pre-max activations (B,C,M,K) and the
# neighbour indices (B,M,K) in it, so that a parity test can find the (query, channel) positions whose two best
# DISTINCT neighbours are closer than the comparison tolerance -- there the arg-max, and with it the gradient
# routing, is decided by rounding (see argmax_is_decided()).  The max reductions of the other families leave their
# pre-max products ("premax"), and every family its output before the final ReLU ("pre_relu").
KEEP = None


def argmax_is_decided(premax, idx, rel=2e-5, relu=True):
    """(B,C,M) bool: the largest activation over K beats the best activation of any OTHER neighbour by more than
    rel * max(1, |value|).  Duplicated slots of the same neighbour (cyclic padding) do not count as competitors:
    routing the gradient to either copy is the same gradient; neither does a maximum of 0 (ReLU output)."""
    xs, order = premax.sort(dim=-1, descending=True)
    ig = idx[:, None, :, :].expand(-1, premax.shape[1], -1, -1).gather(-1, order)
    other = ig != ig[..., :1]
    second = torch.where(other, xs, torch.full_like(xs, float("-inf"))).max(-1)[0]
    v1 = xs[..., 0]
    clear = (v1 - second) > rel * v1.abs().clamp(min=1.0)
    # post-ReLU activations (PointWiseMLP): a maximum of exactly 0 passes no gradient whichever slot holds it
    return (clear | (v1 <= 0)) if relu else clear


def query_and_group(ext, query_xyz, support_xyz, query_mask, support_mask, features, radius, nsample,
                    normalize_xyz):
    """pt_utils.py:121-144 with use_xyz=False, ret_grouped_xyz=True (the only way LA uses it).
    Returns (grouped_features (B,C,M,K), grouped_xyz (B,3,M,K), idx_mask (B,M,K), idx (B,M,K))."""
    group = make_grouping(ext)
    with torch.no_grad():
        idx, idx_mask = ext.masked_ordered_ball_query(query_xyz, support_xyz, query_mask, support_mask,
                                                      radius, nsample)
    xyz_t = support_xyz.transpose(1, 2).contiguous()
    grouped_xyz = group(xyz_t, idx)
    grouped_xyz = grouped_xyz - query_xyz.transpose(1, 2).unsqueeze(-1)      # :127
    if normalize_xyz:
        if GPU_SCALAR_DIVISION:
            inv = (torch.ones((), dtype=torch.float32) / torch.tensor(radius, dtype=torch.float32)).item()
            grouped_xyz = grouped_xyz * inv                                   # what the CUDA kernel computes
        else:
            grouped_xyz = grouped_xyz / radius                                # :128-129 true division by float(radius)
    if features is not None:   # float64 run: dp is formed in fp32 like the reference, then joins the features' dtype
        grouped_xyz = grouped_xyz.to(features.dtype)
    grouped_features = group(features, idx) if features is not None else None
    if KEEP is not None:
        KEEP["idx"] = idx.long()
    return grouped_features, grouped_xyz, idx_mask, idx


def nearest_and_group(ext, query_xyz, support_xyz, query_mask, support_mask, features):
    """pt_utils.py:154-176 with use_xyz=False."""
    group = make_grouping(ext)
    with torch.no_grad():
        idx, idx_mask = ext.masked_nearest_query(query_xyz, support_xyz, query_mask, support_mask)
    return group(features, idx), idx_mask, idx


def masked_max_pool(ext, xyz, mask, features, npoint, radius, nsample, sampleDl):
    """pt_utils.py:188-202 -> (sub_xyz, sub_mask, sub_features)."""
    with torch.no_grad():
        sub_xyz, sub_mask = ext.masked_grid_subsampling(xyz, mask, npoint, sampleDl)
    sub_xyz = sub_xyz.contiguous()
    sub_mask = sub_mask.contiguous()
    gf, _, _, _ = query_and_group(ext, sub_xyz, xyz, sub_mask, mask, features, radius, nsample, False)
    return sub_xyz, sub_mask, gf.max(dim=-1)[0]


def masked_upsample_nearest(ext, up_xyz, xyz, up_mask, mask, features):
    """pt_utils.py:216-227 mode='nearest'."""
    gf, _, _ = nearest_and_group(ext, up_xyz, xyz, up_mask, mask, features)
    return gf[..., 0].contiguous()


# --------------------------------------------------------------------------------------------------
# shared pieces of the four operators
# --------------------------------------------------------------------------------------------------
def _feature_mask(idx_mask, query_mask):
    # local_aggregation_operators.py:92-93: padded queries (query_mask==0) count every slot
    return idx_mask + (1 - query_mask[:, :, None])


def _reduce(agg, idx_mask, query_mask, reduction):
    """local_aggregation_operators.py:87-105 (identical in all families). agg (B,C,M,K) -> (B,C,M)"""
    if reduction == "max":
        if KEEP is not None:
            KEEP["premax"] = agg.detach()
        return agg.max(dim=-1)[0]
    fm = _feature_mask(idx_mask, query_mask)[:, None, :, :]
    agg = agg * fm
    out = agg.sum(-1)
    if reduction in ("avg", "mean"):
        out = out / fm.sum(-1)
    elif reduction != "sum":
        raise NotImplementedError(reduction)
    return out


def _bn(x, st, prefix, momentum, training):
    """nn.BatchNorm{1,2}d semantics; updates running stats in `st` in place when training."""
    w, b = st[prefix + ".weight"], st[prefix + ".bias"]
    rm, rv = st[prefix + ".running_mean"], st[prefix + ".running_var"]
    y = F.batch_norm(x, rm, rv, w, b, training, momentum, 1e-5)
    if training and (prefix + ".num_batches_tracked") in st:
        st[prefix + ".num_batches_tracked"] += 1
    return y


def _out_block(out, st, cfg_out_conv, cin, cout, momentum, training):
    """out_conv (Conv1d 1x1 no bias + BN1d + ReLU) or out_transform (BN1d + ReLU): :37-45,107-110"""
    if cfg_out_conv or cin != cout:
        out = F.conv1d(out, st["out_conv.0.weight"])
        y = _bn(out, st, "out_conv.1", momentum, training)
    else:
        y = _bn(out, st, "out_transform.0", momentum, training)
    if KEEP is not None:
        KEEP["pre_relu"] = y.detach()
    return F.relu(y)


# --------------------------------------------------------------------------------------------------
# the four families.  `st` maps the reference's state-dict key (without the
# 'local_aggregation_operator.' prefix) -> tensor; cfg is the reference config (attribute access).
# --------------------------------------------------------------------------------------------------
def pospool(ext, st, cfg, cin, cout, radius, nsample, q_xyz, s_xyz, q_mask, s_mask, feats, training=True):
    B, C, M = feats.shape[0], feats.shape[1], q_xyz.shape[1]
    gf, dp, idx_mask, _ = query_and_group(ext, q_xyz, s_xyz, q_mask, s_mask, feats, radius, nsample, True)
    pe = cfg.pospool.position_embedding
    if pe == "xyz":                                                           # :65-69
        agg = (dp.unsqueeze(1) * gf.view(B, C // 3, 3, M, nsample)).view(B, C, M, nsample)
    elif pe == "sin_cos":                                                     # :70-83
        fd = C // 6
        rng = torch.arange(fd, dtype=torch.float32, device=q_xyz.device)
        dim_mat = torch.pow(1.0 * 1000, (1.0 / fd) * rng) if DIM_MAT_FN is None else DIM_MAT_FN(fd).to(rng.device)
        # the argument fl32(fl32(100 dp) / dim) is part of the reference's function: it is formed in fp32 even in a
        # float64 run (one ulp of it moves sin by ~1e-5), only sin / cos are then taken in the features' dtype
        div = torch.div((100 * dp.float()).unsqueeze(-1), dim_mat).to(gf.dtype)   # (B,3,M,K,fd)
        emb = torch.cat([torch.sin(div), torch.cos(div)], -1)                # (B,3,M,K,2fd)
        emb = emb.permute(0, 1, 4, 2, 3).contiguous().view(B, C, M, nsample)
        agg = gf * emb
    else:
        raise NotImplementedError(pe)
    out = _reduce(agg, idx_mask, q_mask, cfg.pospool.reduction)
    return _out_block(out, st, cfg.pospool.output_conv, cin, cout, cfg.bn_momentum, training)


def adaptive_weight(ext, st, cfg, cin, cout, radius, nsample, q_xyz, s_xyz, q_mask, s_mask, feats,
                    training=True):
    B, C, M = feats.shape[0], feats.shape[1], q_xyz.shape[1]
    aw = cfg.adaptive_weight
    if aw.weight_type != "dp":                                                # :188-192
        raise NotImplementedError(aw.weight_type)
    gf, dp, idx_mask, _ = query_and_group(ext, q_xyz, s_xyz, q_mask, s_mask, feats, radius, nsample, True)
    w = F.conv2d(dp, st["mlps.conv0.weight"], st["mlps.conv0.bias"])          # :148-151
    for i in range(aw.num_mlps - 1):                                          # :152-158
        w = F.conv2d(F.relu(w), st[f"mlps.conv{i + 1}.weight"], st[f"mlps.conv{i + 1}.bias"])
    S = aw.shared_channels
    agg = (gf.view(B, C // S, S, M, nsample) * w.unsqueeze(2)).view(B, C, M, nsample)   # :194-197
    out = _reduce(agg, idx_mask, q_mask, aw.reduction)
    return _out_block(out, st, aw.output_conv, cin, cout, cfg.bn_momentum, training)


def pointwise_mlp(ext, st, cfg, cin, cout, radius, nsample, q_xyz, s_xyz, q_mask, s_mask, feats,
                  training=True):
    pw = cfg.pointwisemlp
    if pw.feature_type != "dp_fi_df":                                         # :288-295
        raise NotImplementedError(pw.feature_type)
    gf, dp, idx_mask, idx = query_and_group(ext, q_xyz, s_xyz, q_mask, s_mask, feats, radius, nsample, True)
    center = gf[..., 0:1].expand(-1, -1, -1, nsample)                         # slot 0 = nearest neighbour
    x = torch.cat([dp, center, gf - center], 1)
    for i in range(pw.num_mlps):                                              # :252-272 conv + BN2d + ReLU
        x = F.conv2d(x, st[f"mlps.conv{i}.0.weight"])
        y = _bn(x, st, f"mlps.conv{i}.1", cfg.bn_momentum, training)
        x = F.relu(y)
    if KEEP is not None:
        KEEP["pwmlp_premax"], KEEP["idx"] = x.detach(), idx.long()
        if pw.reduction == "max":   # max_k relu(y) = relu(max_k y): the output's value before the ReLU
            KEEP["pre_relu"] = y.detach().max(dim=-1)[0]
    return _reduce(x, idx_mask, q_mask, pw.reduction)                         # no out_transform (:297-316)


def pseudo_grid(ext, st, cfg, cin, cout, radius, nsample, q_xyz, s_xyz, q_mask, s_mask, feats,
                training=True):
    B, C, M = feats.shape[0], feats.shape[1], q_xyz.shape[1]
    pg = cfg.pseudo_grid
    extent = 2 * pg.KP_extent * radius / cfg.density_parameter               # :344
    gf, dp, idx_mask, _ = query_and_group(ext, q_xyz, s_xyz, q_mask, s_mask, feats, radius, nsample, False)
    kp = st["K_points"]                                                       # (15,3)
    diff = dp.permute(0, 2, 3, 1).unsqueeze(3) - kp                           # (B,M,K,15,3)  :385-389
    sq = torch.sum(diff ** 2, -1)                                             # (B,M,K,15)
    if pg.KP_influence == "constant":
        h = torch.ones_like(sq)
    elif pg.KP_influence == "linear":
        h = torch.clamp(1 - torch.sqrt(sq) / extent, min=0.0)                 # :395-398
    else:
        raise ValueError("Unknown influence function type (config.KP_influence)")
    h = h.permute(0, 1, 3, 2)                                                 # (B,M,15,K)
    fm = _feature_mask(idx_mask, q_mask)                                      # :407-409
    h = h * fm[:, :, None, :]
    if pg.convolution_mode != "sum":
        raise NotImplementedError(pg.convolution_mode)
    nk = kp.shape[0]
    wf = torch.bmm(h.reshape(-1, nk, nsample),
                   gf.permute(0, 2, 3, 1).contiguous().view(-1, nsample, C))  # (BM,15,C)  :415-417
    out = torch.sum(wf * st["kernel_weights"], 1).view(B, M, C).transpose(1, 2)  # :418-419
    return _out_block(out, st, pg.output_conv, cin, cout, cfg.bn_momentum, training)


FAMILIES = {"pospool": pospool, "adaptive_weight": adaptive_weight, "pointwisemlp": pointwise_mlp,
            "pseudo_grid": pseudo_grid}


class OracleLocalAggregation:
    """Functional stand-in for the reference's LocalAggregation (:429-464) holding a reference state dict.

    state: dict key -> tensor, keys as in the reference module's state_dict() (with or without the
    'local_aggregation_operator.' prefix).  Float tensors that the reference registers as Parameters get
    requires_grad=True so .grads() mirrors the reference's parameter gradients.
    dtype: cast every floating state tensor (parameters, BatchNorm state, kernel points) to it, e.g. torch.float64
    with oracle.f64_ext as `ext` for a high-precision reference; None keeps the state's own dtype."""

    PREFIX = "local_aggregation_operator."
    _BUFFERS = ("running_mean", "running_var", "num_batches_tracked", "K_points")

    def __init__(self, ext, la_type, in_channels, out_channels, radius, nsample, cfg, state, device="cpu",
                 dtype=None):
        self.ext, self.la_type = ext, la_type
        self.cin, self.cout, self.radius, self.nsample, self.cfg = in_channels, out_channels, radius, nsample, cfg
        self.st = {}
        for k, v in state.items():
            k = k[len(self.PREFIX):] if k.startswith(self.PREFIX) else k
            v = v.detach().clone().to(device)
            if dtype is not None and v.is_floating_point():
                v = v.to(dtype)
            if v.is_floating_point() and not k.endswith(self._BUFFERS):
                v.requires_grad_(True)
            self.st[k] = v
        self.training = True

    def __call__(self, q_xyz, s_xyz, q_mask, s_mask, feats):
        return FAMILIES[self.la_type](self.ext, self.st, self.cfg, self.cin, self.cout, self.radius,
                                      self.nsample, q_xyz, s_xyz, q_mask, s_mask, feats, self.training)

    def params(self):
        return {k: v for k, v in self.st.items() if v.requires_grad}

    def grads(self):
        return {k: v.grad for k, v in self.st.items() if v.requires_grad and v.grad is not None}
