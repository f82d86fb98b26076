"""DP-FedAvg on the H100: the clip kernel and the DP instantiations of the fused aggregation kernel (with and without a
server optimizer) against the ATen oracle (``TorchCollective``) on one process and on loopback ranks (one-shot and
two-shot), the device noise against the numpy oracle, graph replay, the launch count, the NaN guard and a graphed
ResNet18 ``federated_multi`` run against the ATen collective."""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("CUDA device required", allow_module_level=True)

from federated_pytorch_test_b200.algo import privacy  # noqa: E402
from federated_pytorch_test_b200.parallel import Topology, TorchCollective  # noqa: E402
from federated_pytorch_test_b200.parallel.collective import DPRound  # noqa: E402
from federated_pytorch_test_b200.parallel.fused import FusedCollective  # noqa: E402
from federated_pytorch_test_b200.parallel.loopback import LoopbackWorld  # noqa: E402

DEV = torch.device("cuda", 0)
SIZES = [850, 5130, 73984, 295424, 4720640]
KEY = privacy.noise_key(69)


def _round_inputs(xs, z, C, g):
    """Workers 0, 2, 4 ... move well inside the bound, 1, 3, 5 ... well outside it."""
    N = z.numel()
    for k, x in enumerate(xs):
        x.copy_(z + torch.randn(N, device=DEV, generator=g) * ((3.0 if k % 2 else 0.2) * C / math.sqrt(N)))


@pytest.mark.parametrize("kind", [None, "adam"])
@pytest.mark.parametrize("K", [1, 2, 4, 8, 10])
@pytest.mark.parametrize("N", SIZES)
def test_fused_matches_oracle_single_process(N, K, kind):
    topo = Topology.single_process(K, DEV)
    coll, oracle = FusedCollective(topo), TorchCollective(topo)
    stride = -(-N // 32) * 32
    arena = coll.heap.alloc(K * stride)
    xs = [arena[k * stride: k * stride + N] for k in range(K)]
    g = torch.Generator(device=DEV).manual_seed(N + K)
    z = coll.zeros_like_block(xs[0], "z")
    z.copy_(torch.randn(N, device=DEV, generator=g))
    zr = z.clone()
    C, sigma = 1e-3 * math.sqrt(N), 1.5
    t, tr = torch.zeros(1, dtype=torch.int64, device=DEV), torch.zeros(1, dtype=torch.int64, device=DEV)
    if kind:
        m, v = coll.zeros_like_block(xs[0], "m"), coll.zeros_like_block(xs[0], "v").fill_(1e-6)
        mr, vr = m.clone(), v.clone()
    for r in range(2):
        _round_inputs(xs, z, C, g)
        xr = [x.clone() for x in xs]
        before = [x.clone() for x in xs]
        coll.dp_clip_(xs, z, C)
        oracle.dp_clip_(xr, zr, C)
        for k in range(0, K, 2):                         # inside the bound: not written at all
            assert torch.equal(xs[k], before[k])
        for x, y in zip(xs, xr):
            torch.testing.assert_close(x, y, rtol=1e-5, atol=1e-6)
        dp, dpr = DPRound(sigma * C / K, KEY, t), DPRound(sigma * C / K, KEY, tr)
        if kind:
            got = coll.fedopt_(xs, z, m, v, kind, 1e-2, 0.9, 0.99, 1e-3, dp=dp)
            want = float(oracle.fedopt_(xr, zr, mr, vr, kind, 1e-2, 0.9, 0.99, 1e-3, dp=dpr))
            torch.testing.assert_close(m, mr, rtol=1e-4, atol=2e-6)   # m = 0.1 (mean - z): float32 cancellation
        else:
            got = coll.fedavg_(xs, z, dp=dp)
            want = float(oracle.fedavg_(xr, zr, dp=dpr))
        assert got == pytest.approx(want, rel=1e-3)
        torch.testing.assert_close(z, zr, rtol=1e-5, atol=2e-5)
        assert all(torch.equal(x, z) for x in xs)
        clipped, norms = coll.last_dp
        assert clipped == oracle.last_dp[0] == K // 2
        assert norms == pytest.approx(oracle.last_dp[1], rel=1e-4)
        zr.copy_(z)                                      # next round from the same server model
        if kind:
            mr.copy_(m)
            vr.copy_(v)
    assert int(t) == int(tr) == 2
    assert coll.last_nonfinite == 0.0


def test_device_noise_matches_numpy_oracle():
    """One worker at z = 0: z' = std * xi exactly, for an odd length (scalar tail) and two rounds."""
    N = 1_000_003
    topo = Topology.single_process(1, DEV)
    coll = FusedCollective(topo)
    x = coll.heap.alloc(N + 32)[:N]
    z = coll.zeros_like_block(x, "z")
    t = torch.full((1,), 41, dtype=torch.int64, device=DEV)
    for r in (41, 42):
        x.zero_()
        z.zero_()
        coll.dp_clip_([x], z, 1.0)
        coll.fedavg_([x], z, dp=DPRound(1.0, KEY, t))
        want = privacy.dp_noise(KEY, r, N)
        got = z.double().cpu().numpy()
        np.testing.assert_allclose(got, want, rtol=2e-5, atol=2e-5)
    assert int(t) == 43


@pytest.mark.parametrize("kind", [None, "adam"])
@pytest.mark.parametrize("two_shot", ["0", "1"])
@pytest.mark.parametrize("W,per_rank", [(2, 1), (4, 1), (2, 2)])
@pytest.mark.parametrize("N", [5130, 295424, 4720640])
def test_loopback_ranks_agree_bitwise_and_match_oracle(N, W, per_rank, two_shot, kind):
    K = W * per_rank
    world = LoopbackWorld(W, DEV, max_blocks=8, timeout_s=10.0, K=K)
    for c in world.colls:
        c.two_shot_mode = two_shot
    stride = -(-N // 32) * 32
    xs_rank = [[] for _ in range(W)]
    for _ in range(per_rank):
        for r, buf in enumerate(world.alloc(stride)):
            xs_rank[r].append(buf[:N])
    by_worker = [xs_rank[ck % W][ck // W] for ck in range(K)]
    g = torch.Generator(device=DEV).manual_seed(N + K)
    z0 = torch.randn(N, device=DEV, generator=g)
    zs = [c.zeros_like_block(x[0], "z") for c, x in zip(world.colls, xs_rank)]
    for zz in zs:
        zz.copy_(z0)
    ts = [torch.zeros(1, dtype=torch.int64, device=DEV) for _ in range(W)]
    if kind:                                  # symmetric slices: two-shot ranks broadcast their slice of m and v
        ms = [c.zeros_like_block(x[0], "m") for c, x in zip(world.colls, xs_rank)]
        vs = [c.zeros_like_block(x[0], "v").fill_(1e-6) for c, x in zip(world.colls, xs_rank)]
        mr, vr = ms[0].clone(), vs[0].clone()
    oracle = TorchCollective(Topology.single_process(K, DEV))
    zr, tr = z0.clone(), torch.zeros(1, dtype=torch.int64, device=DEV)
    C = 1e-3 * math.sqrt(N)
    for r in range(2):
        _round_inputs(by_worker, zr, C, g)
        xr = [x.clone() for x in by_worker]
        torch.cuda.synchronize()

        def one(rank, c):
            c.dp_clip_(xs_rank[rank], zs[rank], C)
            dp = DPRound(C / K, KEY, ts[rank])
            if kind:
                c.launch_fedopt_(xs_rank[rank], zs[rank], ms[rank], vs[rank], kind, 1e-2, 0.9, 0.99, 1e-3, dp=dp)
            else:
                c.launch_fedavg_(xs_rank[rank], zs[rank], True, dp=dp)
        world.run(one)
        oracle.dp_clip_(xr, zr, C)
        if kind:
            want = float(oracle.fedopt_(xr, zr, mr, vr, kind, 1e-2, 0.9, 0.99, 1e-3, dp=DPRound(C / K, KEY, tr)))
        else:
            want = float(oracle.fedavg_(xr, zr, dp=DPRound(C / K, KEY, tr)))
        for rank, c in enumerate(world.colls):
            rec = c.read_record()
            assert rec[0] == pytest.approx(want, rel=1e-3)
            assert c.last_dp[0] == oracle.last_dp[0] == K // 2
            assert c.last_dp[1] == pytest.approx(oracle.last_dp[1], rel=1e-4)
            assert c.last_two_shot == (two_shot == "1" and per_rank == 1)     # two-shot needs one replica per rank
        for zz in zs[1:]:
            assert torch.equal(zz, zs[0])
        torch.testing.assert_close(zs[0], zr, rtol=1e-5, atol=2e-5)
        zr.copy_(zs[0])
        if kind:
            for mm, vv in zip(ms[1:], vs[1:]):
                assert torch.equal(mm, ms[0]) and torch.equal(vv, vs[0])
            torch.testing.assert_close(ms[0], mr, rtol=1e-4, atol=2e-6)
            mr.copy_(ms[0])
            vr.copy_(vs[0])
    assert all(int(t) == 2 for t in ts)


def test_huge_finite_attacker_is_clipped_like_the_oracle():
    """An update whose float32 sum of squares overflows is clipped to the bound, as the ATen path does."""
    K, N = 4, 295424
    topo = Topology.single_process(K, DEV)
    coll, oracle = FusedCollective(topo), TorchCollective(topo)
    arena = coll.heap.alloc(K * N)
    xs = [arena[k * N:(k + 1) * N] for k in range(K)]
    g = torch.Generator(device=DEV).manual_seed(3)
    z = coll.zeros_like_block(xs[0], "z")
    z.copy_(torch.randn(N, device=DEV, generator=g))
    C = 1e-3 * math.sqrt(N)
    _round_inputs(xs, z, C, g)
    xs[3].copy_(z + 1e30 * torch.randn(N, device=DEV, generator=g))
    zr, xr = z.clone(), [x.clone() for x in xs]
    coll.dp_clip_(xs, z, C)
    oracle.dp_clip_(xr, zr, C)
    assert float(torch.linalg.vector_norm(xs[3].double() - z.double())) == pytest.approx(C, rel=1e-5)
    for x, y in zip(xs, xr):
        torch.testing.assert_close(x, y, rtol=1e-5, atol=1e-6)
    t = torch.zeros(1, dtype=torch.int64, device=DEV)
    coll.fedavg_(xs, z, dp=DPRound(C / K, KEY, t))
    assert coll.last_dp[0] == 2 and math.isfinite(coll.last_dp[1]) and coll.last_nonfinite == 0.0   # workers 1 and 3
    assert torch.isfinite(z).all()


def test_parameter_layout_keeps_padding_noise_free():
    """Per 32-float chunk only the leading dp_valid floats get noise: the alignment padding of the arena stays 0."""
    N = 5000
    counts = [32] * (N // 32) + [N % 32]
    counts[3], counts[40], counts[100] = 7, 0, 31
    valid = torch.tensor(counts, dtype=torch.uint8, device=DEV)
    topo = Topology.single_process(2, DEV)
    coll, oracle = FusedCollective(topo), TorchCollective(topo)
    arena = coll.heap.alloc(2 * 5024)
    xs = [arena[:N], arena[5024:5024 + N]]
    z = coll.zeros_like_block(xs[0], "z")
    for x in xs:
        x.zero_()
    zr, xr = z.clone(), [x.clone() for x in xs]
    t, tr = torch.zeros(1, dtype=torch.int64, device=DEV), torch.zeros(1, dtype=torch.int64, device=DEV)
    coll.dp_clip_(xs, z, 1.0)
    coll.fedavg_(xs, z, dp=DPRound(1.0, KEY, t, valid))
    oracle.dp_clip_(xr, zr, 1.0)
    oracle.fedavg_(xr, zr, dp=DPRound(1.0, KEY, tr, valid))
    mask = DPRound(1.0, KEY, t, valid).mask(N)
    assert torch.equal(z[~mask], torch.zeros(int((~mask).sum()), device=DEV)) and int((~mask).sum()) == 25 + 32 + 1
    assert bool((z[mask] != 0).all())
    torch.testing.assert_close(z, zr, rtol=1e-5, atol=1e-6)


def test_graph_replay_draws_fresh_noise_and_two_launches_per_round():
    K, N = 4, 73984
    topo = Topology.single_process(K, DEV)
    coll = FusedCollective(topo)
    stride = N
    arena = coll.heap.alloc(K * stride)
    xs = [arena[k * stride:(k + 1) * stride] for k in range(K)]
    z = coll.zeros_like_block(xs[0], "z")
    t = torch.zeros(1, dtype=torch.int64, device=DEV)
    dp = DPRound(0.5, KEY, t)
    n0 = coll.launches
    coll.dp_clip_(xs, z, 1.0)
    coll.launch_fedavg_(xs, z, True, dp=dp)
    assert coll.launches - n0 == 2
    coll.read_record()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            coll.dp_clip_(xs, z, 1.0)
            coll.launch_fedavg_(xs, z, True, dp=dp)
    torch.cuda.current_stream().wait_stream(s)
    for r in (1, 2):                               # capture did not run the kernels; each replay is round t, then t + 1
        for x in xs:
            x.zero_()
        z.zero_()
        graph.replay()
        torch.cuda.synchronize()
        np.testing.assert_allclose(z.double().cpu().numpy(), 0.5 * privacy.dp_noise(KEY, r, N), rtol=2e-5, atol=2e-5)
        assert int(t) == r + 1


def _run(**kw):
    from federated_pytorch_test_b200.api import federated_multi

    base = dict(K=4, use_resnet=True, Nloop=1, Nadmm=2, max_minibatches=3, train_size=2048, test_size=256,
                check_results=False, save_model=False, graphs=True)
    lines = []
    eng = federated_multi.run(federated_multi.Config(**{**base, **kw}), log=lines.append)
    return eng, lines


def test_nan_attacker_trips_the_guard():
    with pytest.raises(FloatingPointError, match="non-finite"):
        _run(K=4, dp_clip=1e-3, byzantine=1, attack="nan", Nadmm=1, max_minibatches=1)


def test_graphed_resnet18_run_matches_aten_and_reports_epsilon():
    kw = dict(dp_clip=1e-3, dp_noise=1.0)
    eng, fused = _run(**kw)
    _, aten = _run(**kw, collective="torch")
    df = [l for l in fused if l.startswith("dual (")]
    da = [l for l in aten if l.startswith("dual (")]
    assert len(df) == len(da) > 0
    for a, b in zip(df, da):
        assert a.split("=")[:-1] == b.split("=")[:-1]
        assert float(a.rsplit("=", 1)[1]) == pytest.approx(float(b.rsplit("=", 1)[1]), rel=2e-2)
    dp = [l for l in fused if l.startswith("dp:")]
    T = len(df)
    assert dp[-1] == privacy.dp_line(1.0, 1e-3, 1e-5, T, planned=False)
    assert dp[-1].endswith("epsilon=%.4f" % privacy.gaussian_epsilon(1.0, T, 1e-5))
    assert eng.strategy.dp_rounds == T and int(eng.strategy.dp_t) == T
