"""CPU: the numpy construction of the canonical transposed lists, and which wrappers ask the library for the
deterministic forms (a stub library records the arguments; no GPU needed)."""
import numpy as np
import pytest
import torch

from closerlook3d_b200 import _lib, ops


def canonical_lists(idx, ncount, N):
    """numpy: (off (B,N+1), ent (B,M*K)) with every list in ascending q*K + k.  ncount None = all K slots; entries
    past off[N] are -1"""
    B, M, K = idx.shape
    off = np.zeros((B, N + 1), np.int32)
    ent = np.full((B, M * K), -1, np.int32)
    for b in range(B):
        e = np.arange(M * K)
        keep = np.ones(M * K, bool) if ncount is None else (e % K) < np.repeat(ncount[b], K)
        e, j = e[keep], idx[b].reshape(-1)[keep]
        order = np.argsort(j, kind="stable")
        ent[b, :len(e)] = e[order]
        off[b, 1:] = np.cumsum(np.bincount(j, minlength=N))
    return off, ent


def _brute_lists(idx, ncount, N):
    B, M, K = idx.shape
    lists = []
    for b in range(B):
        per = [[] for _ in range(N)]
        for q in range(M):
            for k in range(K if ncount is None else int(ncount[b, q])):
                per[int(idx[b, q, k])].append(q * K + k)
        lists.append(per)
    return lists


@pytest.mark.parametrize("counted", [False, True])
def test_canonical_lists_match_their_definition(counted):
    rng = np.random.default_rng(7)
    B, M, K, N = 2, 37, 5, 11
    idx = rng.integers(0, N, (B, M, K)).astype(np.int32)
    idx[0, 3] = 4                                   # a query that fills every slot with one point
    ncount = rng.integers(0, K + 1, (B, M)).astype(np.int32) if counted else None
    off, ent = canonical_lists(idx, ncount, N)
    want = _brute_lists(idx, ncount, N)
    for b in range(B):
        for j in range(N):
            assert list(ent[b, off[b, j]:off[b, j + 1]]) == want[b][j]   # ascending q*K + k by construction


class _Stub:
    """stands in for libcl3d: records every call's arguments, returns success / a small workspace size"""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def fn(*args):
            self.calls.append((name, args))
            return 64 if name.endswith("workspace_bytes") else 0
        return fn

    def args(self, name):
        return [a for n, a in self.calls if n == name]


@pytest.fixture
def stub(monkeypatch):
    s = _Stub()
    monkeypatch.setattr(_lib, "lib", lambda: s)
    monkeypatch.setattr(ops, "stream_ptr", lambda: None)
    monkeypatch.setattr(ops, "require_cuda", lambda *a: None)
    monkeypatch.setattr(ops, "require_features", lambda t, n: ops.DTYPE_CODE[t.dtype])
    yield s
    torch.use_deterministic_algorithms(False)


MODES = [(False, None, 0), (True, None, 1), (False, True, 1), (True, False, 0)]   # (torch flag, argument, expected)


@pytest.mark.parametrize("flag,arg,want", MODES)
def test_build_csr_passes_the_mode(stub, flag, arg, want):
    torch.use_deterministic_algorithms(flag)
    idx = torch.zeros(2, 5, 3, dtype=torch.int32)
    ops.build_csr(idx, None, 7, deterministic=arg)
    (ws,), (call,) = stub.args("cl3d_csr_workspace_bytes"), stub.args("cl3d_build_csr")
    assert ws[-1] == want and call[-2] == want


@pytest.mark.parametrize("flag,arg,want", MODES)
def test_ball_query_passes_the_mode_to_both_phases(stub, flag, arg, want):
    torch.use_deterministic_algorithms(flag)
    xyz = torch.zeros(1, 6, 3)
    m = torch.ones(1, 6, dtype=torch.int32)
    ops.ball_query(xyz, xyz, m, m, 0.1, 4, csr="all", after_search=lambda: None, deterministic=arg)
    (ws,) = stub.args("cl3d_ball_query_csr_workspace_bytes")
    calls = stub.args("cl3d_ball_query_csr")
    assert ws[-1] == want
    assert [c[-3] for c in calls] == [1, 2] and all(c[-2] == want for c in calls)


@pytest.mark.parametrize("flag,arg,want", MODES)
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_group_points_grad_passes_lists_exactly_when_asked(stub, flag, arg, want, dtype):
    torch.use_deterministic_algorithms(flag)
    g = torch.zeros(1, 3, 5, 2, dtype=dtype)
    ops.group_points_grad(g, torch.zeros(1, 5, 2, dtype=torch.int32), 9, deterministic=arg)
    (call,) = stub.args("cl3d_group_points_grad")
    off, ent, acc = call[8], call[9], call[11]
    assert (off is not None) == bool(want) and (ent is not None) == bool(want)
    assert len(stub.args("cl3d_build_csr")) == want
    if want:
        assert stub.args("cl3d_build_csr")[0][-2] == 1 and acc is None   # canonical lists; no fp32 scratch
    else:
        assert (acc is not None) == (dtype != torch.float32)


@pytest.mark.parametrize("flag,arg,want", MODES)
def test_gather_max_grad_passes_lists_exactly_when_asked(stub, flag, arg, want):
    torch.use_deterministic_algorithms(flag)
    g = torch.zeros(1, 3, 5)
    idx = torch.zeros(1, 5, 2, dtype=torch.int32)
    arg_ = torch.zeros(1, 5, 8, dtype=torch.uint8)
    ops.gather_max_grad(g, idx, arg_, 9, deterministic=arg)
    (call,) = stub.args("cl3d_gather_max_bwd")
    assert (call[9] is not None) == bool(want) and (call[10] is not None) == bool(want)
    assert len(stub.args("cl3d_build_csr")) == want
    # lists the caller already has are used as they are
    stub.calls.clear()
    given = (torch.zeros(1, 10, dtype=torch.int32), torch.zeros(1, 10, dtype=torch.int32))
    ops.gather_max_grad(g, idx, arg_, 9, csr=given, deterministic=arg)
    (call,) = stub.args("cl3d_gather_max_bwd")
    assert stub.args("cl3d_build_csr") == []
    assert (call[9] is not None) == bool(want)


@pytest.mark.parametrize("flag,arg,want", MODES)
@pytest.mark.parametrize("training", [True, False])
def test_pwmlp_bwd_passes_the_mode(stub, flag, arg, want, training):
    torch.use_deterministic_algorithms(flag)
    B, N, M, K, Cout = 1, 6, 4, 2, 8
    ab = torch.zeros(B, N, 16)
    ysel = torch.zeros(B, Cout, M)
    idx = torch.zeros(B, M, K, dtype=torch.int32)
    g = torch.zeros(B, Cout, M)
    ops.pwmlp_bwd(g, None, ab, None, None, None, None, idx, None, None, ysel, None, None, None, None, None, 0.1,
                  training=training, deterministic=arg)
    (sc,), (call,) = stub.args("cl3d_pwmlp_bwd_scratch_floats"), stub.args("cl3d_pwmlp_bwd")
    assert sc[-1] == want
    assert call[23] == int(training) and call[24] == want
