"""CPU: which BatchNorms the fused operators synchronise (ops.bn_sync_group), against torch's own SyncBatchNorm rule,
and that converting a model leaves its checkpoint keys alone.

Over a process group of more than one rank, torch's SyncBatchNorm refuses a CPU input exactly when it decides to
synchronise, so on CPU its forward is the oracle there: it raises ValueError iff it would synchronise."""
import copy

import pytest
import torch
import torch.nn as nn

from closerlook3d_b200 import ops


def _torch_syncs(bn):
    """whether torch's SyncBatchNorm forward would synchronise `bn` over a group of >1 rank (a CPU input makes that
    path raise; it checks the device before the group size)"""
    x = torch.randn(4, bn.num_features, 5)
    try:
        bn(x)
    except ValueError:
        return True
    return False


def _variants():
    """(name, module) over plain / Sync, train / eval, with and without running statistics"""
    out = []
    for sync in (False, True):
        for track in (True, False):
            for train in (True, False):
                bn = nn.BatchNorm1d(6, track_running_stats=track)
                if sync:
                    bn = nn.SyncBatchNorm.convert_sync_batchnorm(bn)
                out.append((f"{'sync' if sync else 'plain'}-{'track' if track else 'notrack'}-"
                            f"{'train' if train else 'eval'}", bn.train(train)))
    return out


def test_no_sync_without_a_process_group():
    import torch.distributed as dist
    assert not dist.is_initialized()
    for name, bn in _variants():
        assert ops.bn_sync_group(bn) is None, name
        assert not _torch_syncs(bn), name


def test_one_rank_group_does_not_sync(tmp_path):
    import torch.distributed as dist
    dist.init_process_group("gloo", init_method="file://" + str(tmp_path / "rdv"), rank=0, world_size=1)
    try:
        for name, bn in _variants():
            assert ops.bn_sync_group(bn) is None, name
    finally:
        dist.destroy_process_group()


def _two_rank_worker(rank, init, q):
    import torch.distributed as dist
    dist.init_process_group("gloo", init_method=init, rank=rank, world_size=2)
    try:
        seen = []
        for name, bn in _variants():
            group = ops.bn_sync_group(bn)
            seen.append((name, group is not None, _torch_syncs(bn)))
            if group is not None:
                assert group == dist.group.WORLD
        # a process group of one rank (every rank creates both, as torch requires)
        solo = [dist.new_group([0]), dist.new_group([1])]
        pair = dist.new_group([0, 1])
        for pg, tag in ((solo[rank], "solo"), (pair, "pair")):
            bn = nn.SyncBatchNorm(6, process_group=pg).train()
            group = ops.bn_sync_group(bn)
            assert group is None or group is pg
            seen.append((tag, group is not None, None))
        q.put((rank, seen))
        dist.barrier()
    finally:
        dist.destroy_process_group()


def test_sync_decision_matches_torch_on_two_ranks(tmp_path):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    init = "file://" + str(tmp_path / "rdv2")
    procs = [ctx.Process(target=_two_rank_worker, args=(r, init, q)) for r in range(2)]
    for p in procs:
        p.start()
    try:
        res = dict(q.get(timeout=180) for _ in procs)
    finally:
        for p in procs:
            p.join(timeout=60)
            if p.is_alive():
                p.kill()
                p.join(10)
    assert [p.exitcode for p in procs] == [0, 0]
    for rank, seen in res.items():
        for name, ours, theirs in seen:
            assert theirs is None or ours == theirs, (rank, name, ours, theirs)
        got = {name: ours for name, ours, _ in seen}
        # torch's rule: a SyncBatchNorm in training mode, with or without running statistics, over >1 rank
        assert got == {"plain-track-train": False, "plain-track-eval": False, "plain-notrack-train": False,
                       "plain-notrack-eval": False, "sync-track-train": True, "sync-track-eval": False,
                       "sync-notrack-train": True, "sync-notrack-eval": False, "solo": False, "pair": True}


@pytest.mark.parametrize("la,over", [
    ("pospool", dict(pospool=dict(position_embedding="sin_cos"))),
    ("adaptive_weight", dict()),
    ("pseudo_grid", dict()),
    ("pointwisemlp", dict(pointwisemlp=dict(feature_type="dp_fi_df"))),
])
def test_converted_model_keeps_its_checkpoint_keys(la, over):
    from closerlook3d_b200.config import la_config
    from closerlook3d_b200.local_aggregation_operators import LocalAggregation
    m = LocalAggregation(24, 24, 0.1, 8, la_config(la, **over))
    sd = m.state_dict()
    conv = nn.SyncBatchNorm.convert_sync_batchnorm(copy.deepcopy(m))
    assert any(isinstance(x, nn.SyncBatchNorm) for x in conv.modules())
    csd = conv.state_dict()
    assert list(csd.keys()) == list(sd.keys())
    assert all(csd[k].shape == sd[k].shape and torch.equal(csd[k], sd[k]) for k in sd)
    conv.load_state_dict(sd, strict=True)                 # a plain checkpoint loads into the converted model
    m.load_state_dict(csd, strict=True)                   # and back


def test_converted_scene_network_keeps_its_checkpoint_keys():
    from closerlook3d_b200 import backbone as bb
    c = bb.model_config("scene_segmentation", "pospool")
    c.width = 24
    model = bb.build_scene_segmentation(c)[0]
    keys = list(model.state_dict().keys())
    conv = nn.SyncBatchNorm.convert_sync_batchnorm(copy.deepcopy(model))
    assert sum(isinstance(x, nn.SyncBatchNorm) for x in conv.modules()) > 10
    assert list(conv.state_dict().keys()) == keys
    conv.load_state_dict(model.state_dict(), strict=True)

