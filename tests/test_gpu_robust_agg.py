"""Byzantine-robust aggregation on the H100: the robust instantiations of the fused aggregation kernel (coordinate-wise
median and trimmed mean, with and without a server optimizer) against the ATen oracle (``TorchCollective``) on one
process, on loopback ranks (one-shot, two-shot, two replicas per rank), inside a CUDA graph and across real ranks; the
non-finite count, the launch count and ``federated_multi`` ResNet18 runs, with and without a sign-flipping attacker."""
import math
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("CUDA device required", allow_module_level=True)

from federated_pytorch_test_b200.algo.strategies import FedAvg  # noqa: E402
from federated_pytorch_test_b200.ops import cuda_ops  # noqa: E402
from federated_pytorch_test_b200.parallel import Topology, TorchCollective  # noqa: E402
from federated_pytorch_test_b200.parallel.fused import FusedCollective  # noqa: E402
from federated_pytorch_test_b200.parallel.loopback import LoopbackWorld  # noqa: E402

DEV = torch.device("cuda", 0)
SIZES = [850, 5130, 73984, 295424, 4720640]
RULES = [("median", 0), ("trimmed_mean", 1), ("trimmed_mean", 2)]


def _check(agg, z, zr):
    """median: the order statistic and (lo + hi) * 0.5 are exact, so bit for bit; trimmed mean: rtol 1e-6."""
    if agg == "median":
        assert torch.equal(z, zr)
    else:
        torch.testing.assert_close(z, zr, rtol=1e-6, atol=1e-6)


def _perturb(xs, g, scale=0.05):
    return [scale * torch.randn(x.numel(), device=DEV, generator=g) * (1 + k) for k, x in enumerate(xs)]


@pytest.mark.parametrize("agg,b", RULES)
@pytest.mark.parametrize("K", [2, 3, 4, 5, 8, 10, 16])
@pytest.mark.parametrize("N", SIZES)
def test_fused_matches_oracle_single_process(N, K, agg, b):
    if 2 * b >= K:
        pytest.skip("trimmed mean needs 2 trim_b < K")
    topo = Topology.single_process(K, DEV)
    coll, oracle = FusedCollective(topo), TorchCollective(topo)
    stride = -(-N // 32) * 32
    arena = coll.heap.alloc(K * stride)
    xs = [arena[k * stride: k * stride + N] for k in range(K)]
    g = torch.Generator(device=DEV).manual_seed(N + K + b)
    for k, x in enumerate(xs):
        x.copy_(torch.randn(N, device=DEV, generator=g) * (1 + k))
    z = coll.zeros_like_block(xs[0], "z")
    xr, zr = [x.clone() for x in xs], z.clone()
    for _ in range(2):
        got = coll.robust_(xs, z, agg, b)
        want = float(oracle.robust_(xr, zr, agg, b))
        assert got == pytest.approx(want, rel=1e-4)
        _check(agg, z, zr)
        for x in xs:
            assert torch.equal(x, z)
        for x, y, d in zip(xs, xr, _perturb(xs, g)):
            x.add_(d)
            y.add_(d)
    assert coll.last_nonfinite == 0.0 and not coll.last_two_shot


def _with_nonfinite(xs, nbad, g):
    """Puts NaN / +inf / -inf into up to ``nbad`` workers at every coordinate (different workers per coordinate)."""
    K, N = len(xs), xs[0].numel()
    full = torch.stack(xs)
    rank = torch.rand(K, N, device=DEV, generator=g).argsort(0).argsort(0)         # a random permutation per column
    cnt = torch.randint(0, nbad + 1, (N,), device=DEV, generator=g)
    kind = torch.randint(0, 3, (K, N), device=DEV, generator=g)
    vals = torch.tensor([float("nan"), float("inf"), float("-inf")], device=DEV)[kind]
    full = torch.where(rank < cnt, vals, full)
    for x, row in zip(xs, full):
        x.copy_(row)


@pytest.mark.parametrize("agg,b", [("median", 0), ("trimmed_mean", 1), ("trimmed_mean", 2)])
@pytest.mark.parametrize("N", [850, 5130, 295424])
def test_nonfinite_in_at_most_b_workers_is_harmless_and_more_is_counted(agg, b, N):
    K = 5
    nbad = 2 if agg == "median" else b                  # median of five: two of them may be anything
    topo = Topology.single_process(K, DEV)
    coll, oracle = FusedCollective(topo), TorchCollective(topo)
    stride = -(-N // 32) * 32
    arena = coll.heap.alloc(K * stride)
    xs = [arena[k * stride: k * stride + N] for k in range(K)]
    g = torch.Generator(device=DEV).manual_seed(7 * N + b)
    for x in xs:
        x.copy_(torch.randn(N, device=DEV, generator=g))
    _with_nonfinite(xs, nbad, g)
    assert not all(torch.isfinite(x).all() for x in xs)
    z = coll.zeros_like_block(xs[0], "z")
    xr, zr = [x.clone() for x in xs], z.clone()
    dual = coll.robust_(xs, z, agg, b)
    oracle.robust_(xr, zr, agg, b)
    assert math.isfinite(dual) and coll.last_nonfinite == 0.0 and torch.isfinite(z).all()
    _check(agg, z, zr)
    for x in xs:                                         # one more worker goes bad at coordinates 0 and N - 1 (the tail)
        x.copy_(torch.randn(N, device=DEV, generator=g))
    for k in range(nbad + 1):
        xs[k][0] = float("nan")
        xs[k][N - 1] = float("inf")
    coll.robust_(xs, z, agg, b)
    assert coll.last_nonfinite == 2.0


def _loopback_slices(world, K, N, seed):
    """Per rank the list of its replicas' slices, and all K slices ordered by worker id (worker r + j W)."""
    W = world.world
    stride = -(-N // 32) * 32
    per_rank = [[] for _ in range(W)]
    for _ in range(K // W):
        for r, t in enumerate(world.alloc(stride)):
            per_rank[r].append(t[:N])
    g = torch.Generator(device=DEV).manual_seed(seed)
    by_worker = [per_rank[ck % W][ck // W] for ck in range(K)]
    for k, x in enumerate(by_worker):
        x.copy_(torch.randn(N, device=DEV, generator=g) * (1 + k % 3))
    return per_rank, by_worker, g


@pytest.mark.parametrize("agg,b", [("median", 0), ("trimmed_mean", 1)])
@pytest.mark.parametrize("N", [850, 5130, 295424, 4720640])
@pytest.mark.parametrize("W,per_rank", [(2, 1), (4, 1), (2, 2), (4, 2)])
@pytest.mark.parametrize("two_shot", ["0", "1"])
def test_loopback_ranks_agree_bitwise_and_match_oracle(agg, b, N, W, per_rank, two_shot):
    K = W * per_rank
    if 2 * b >= K:
        pytest.skip("trimmed mean needs 2 trim_b < K")
    world = LoopbackWorld(W, DEV, max_blocks=8, timeout_s=10.0, K=K)
    for c in world.colls:
        c.two_shot_mode = two_shot
    xs_rank, xs, g = _loopback_slices(world, K, N, 11 * N + K)
    zs = [c.zeros_like_block(x[0], "z") for c, x in zip(world.colls, xs_rank)]
    oracle = TorchCollective(Topology.single_process(K, DEV))
    xr = [x.clone() for x in xs]
    zr = torch.zeros(N, device=DEV)
    for _ in range(2):
        world.run(lambda r, c: c.launch_robust_(xs_rank[r], zs[r], agg, b))
        want = float(oracle.robust_(xr, zr, agg, b))
        for r, c in enumerate(world.colls):
            rec = c.read_record()
            assert rec[0] == pytest.approx(want, rel=1e-4) and rec[2] == 0.0
            assert bool(rec[6]) == (two_shot == "1" and per_rank == 1)
            _check(agg, zs[r], zr)
            assert torch.equal(zs[r], zs[0])
            for x in xs_rank[r]:
                assert torch.equal(x, zs[r])
        for x, y, d in zip(xs, xr, _perturb(xs, g)):
            x.add_(d)
            y.add_(d)


def _fedopt_state(make, x, tau):
    z, m, v = make(x, "z"), make(x, "srv_m"), make(x, "srv_v")
    v.fill_(tau * tau)
    return z, m, v


HP = (0.02, 0.9, 0.95, 1e-3)          # FedAdam: lr, beta1, beta2, tau


@pytest.mark.parametrize("agg,b", [("median", 0), ("trimmed_mean", 1)])
@pytest.mark.parametrize("N", [5130, 295424])
def test_fedadam_on_the_robust_aggregate_matches_oracle(agg, b, N):
    K = 5
    topo = Topology.single_process(K, DEV)
    coll, oracle = FusedCollective(topo), TorchCollective(topo)
    stride = -(-N // 32) * 32
    arena = coll.heap.alloc(K * stride)
    xs = [arena[k * stride: k * stride + N] for k in range(K)]
    g = torch.Generator(device=DEV).manual_seed(N)
    for x in xs:
        x.copy_(torch.randn(N, device=DEV, generator=g))
    z, m, v = _fedopt_state(coll.zeros_like_block, xs[0], HP[3])
    z.copy_(torch.stack(xs).mean(0))
    xr = [x.clone() for x in xs]
    zr, mr, vr = z.clone(), m.clone(), v.clone()
    for _ in range(3):
        for x, y, d in zip(xs, xr, _perturb(xs, g)):
            x.add_(d)
            y.add_(d)
        got = coll.fedopt_(xs, z, m, v, "adam", *HP, agg=agg, trim_b=b)
        want = float(oracle.fedopt_(xr, zr, mr, vr, "adam", *HP, agg=agg, trim_b=b))
        assert got == pytest.approx(want, rel=1e-4)
        for p, q in ((z, zr), (m, mr)):
            torch.testing.assert_close(p, q, rtol=1e-5, atol=1e-6)
        torch.testing.assert_close(v, vr, rtol=1e-4, atol=1e-9)
        for x in xs:
            assert torch.equal(x, z)


@pytest.mark.parametrize("two_shot", ["0", "1"])
def test_loopback_robust_fedadam_ranks_agree_bitwise(two_shot):
    W, N = 4, 295424
    world = LoopbackWorld(W, DEV, max_blocks=8, timeout_s=10.0)
    for c in world.colls:
        c.two_shot_mode = two_shot
    xs_rank, xs, g = _loopback_slices(world, W, N, 5)
    st = [_fedopt_state(c.zeros_like_block, x[0], HP[3]) for c, x in zip(world.colls, xs_rank)]
    z0 = torch.stack(xs).mean(0)
    for z, _, _ in st:
        z.copy_(z0)
    oracle = TorchCollective(Topology.single_process(W, DEV))
    xr = [x.clone() for x in xs]
    zr, mr, vr = z0.clone(), torch.zeros_like(z0), torch.full_like(z0, HP[3] ** 2)
    for _ in range(3):
        for x, y, d in zip(xs, xr, _perturb(xs, g)):
            x.add_(d)
            y.add_(d)
        world.run(lambda r, c: c.launch_fedopt_(xs_rank[r], *st[r], "adam", *HP, agg="median"))
        want = float(oracle.fedopt_(xr, zr, mr, vr, "adam", *HP, agg="median"))
        for r, c in enumerate(world.colls):
            rec = c.read_record()
            assert rec[0] == pytest.approx(want, rel=1e-4) and bool(rec[6]) == (two_shot == "1")
            z, m, v = st[r]
            torch.testing.assert_close(z, zr, rtol=1e-5, atol=1e-6)
            torch.testing.assert_close(m, mr, rtol=1e-5, atol=1e-6)
            for a, bb in zip(st[r], st[0]):
                assert torch.equal(a, bb)
            assert torch.equal(xs_rank[r][0], z)


def test_median_round_is_graph_capturable():
    K, N = 5, 73984
    topo = Topology.single_process(K, DEV)
    coll = FusedCollective(topo)
    stride = -(-N // 32) * 32
    arena = coll.heap.alloc(K * stride)
    xs = [arena[k * stride: k * stride + N] for k in range(K)]
    g = torch.Generator(device=DEV).manual_seed(9)
    z = coll.zeros_like_block(xs[0], "z")
    coll._launch(0, xs, None, z, 0.0, agg="median")                        # warm-up (lazy init) outside the capture
    torch.cuda.synchronize()
    for x in xs:
        x.copy_(torch.randn(N, device=DEV, generator=g))
    z.zero_()
    xr, zr = [x.clone() for x in xs], z.clone()
    st = torch.cuda.Stream()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=st):
        coll._launch(0, xs, None, z, 0.0, agg="median")
    e0 = int(coll.sync[0])
    oracle = TorchCollective(topo)
    for _ in range(3):
        for x, y, d in zip(xs, xr, _perturb(xs, g)):
            x.add_(d)
            y.add_(d)
        graph.replay()
        want = float(oracle.robust_(xr, zr, "median", 0))
        assert coll.read_record()[0] == pytest.approx(want, rel=1e-4)
        assert torch.equal(z, zr)
        for x in xs:
            assert torch.equal(x, zr)
    assert int(coll.sync[0]) == e0 + 3


@pytest.mark.parametrize("deferred", [False, True])
@pytest.mark.parametrize("agg", ["median", "trimmed_mean"])
def test_one_launch_per_round(deferred, agg):
    K, N = 5, 5130
    topo = Topology.single_process(K, DEV)
    coll = FusedCollective(topo)
    strat = FedAvg(coll, topo, aggregator=agg, trim_fraction=0.2)
    assert coll.warm_robust
    arena = coll.heap.alloc(K * 5152)
    xs = [arena[k * 5152: k * 5152 + N] for k in range(K)]
    for x in xs:
        x.normal_()
    coll.warmup()
    torch.cuda.synchronize()
    strat.begin_block(0, N, xs)
    for r in range(3):
        for k, x in enumerate(xs):
            x.add_(0.01 * (k + 1))
        before = cuda_ops.launch_count()
        res = strat.aggregate_end(strat.aggregate_begin(r)) if deferred else strat.aggregate(r)
        assert cuda_ops.launch_count() - before == 1
        assert math.isfinite(res["dual"]) and res["dual"] > 0.0


def test_robust_limits_are_rejected():
    topo = Topology.single_process(17, DEV)
    coll = FusedCollective(topo)
    xs = [coll.heap.alloc(256) for _ in range(17)]
    z = coll.zeros_like_block(xs[0], "z")
    with pytest.raises(ValueError, match="16"):
        coll.robust_(xs, z, "median")
    with pytest.raises(ValueError, match="trim"):
        FusedCollective(Topology.single_process(4, DEV)).robust_(xs[:4], z, "trimmed_mean", 2)


# ------------------------------------------------------------------------------------------ engine
def _run_fed(**kw):
    from federated_pytorch_test_b200.api import federated_multi
    lines = []
    base = dict(K=2, model="ResNet18", Nloop=1, Nadmm=2, max_minibatches=4, check_results=False, save_model=False,
                train_size=4096, test_size=256, aggregator="median")
    eng = federated_multi.run(federated_multi.Config(**{**base, **kw}), log=lines.append)
    return eng, lines


def test_resnet18_median_graphed_equals_aten():
    e1, l_fast = _run_fed(graphs=True)
    e2, l_aten = _run_fed(graphs=False, fast=False)
    assert e1.coll.name == "fused" and e2.coll.name == "torch" and e1.strategy.aggregator == "median"
    d_fast = [float(l.rsplit("=", 1)[1]) for l in l_fast if l.startswith("dual (")]
    d_aten = [float(l.rsplit("=", 1)[1]) for l in l_aten if l.startswith("dual (")]
    print("fused + graphed:", d_fast[:6], "\nATen:", d_aten[:6])
    assert len(d_fast) == len(d_aten) == 20
    for a, b in zip(d_fast, d_aten):                                     # TF32 convolutions against fp32 ATen
        assert a == pytest.approx(b, rel=5e-2)
    assert getattr(e1, "graph_replays", 0) > 0


def test_resnet18_signflip_attacker_median_beats_mean():
    """K = 4 co-resident replicas, worker 3 sends z - 4 (x - z) before every aggregation.  Final test accuracy of the honest
    worker 0 (chance: 10 %).  The first H100 run ended at 100 % with the median and 0 % with the mean; the thresholds
    leave 20 points of margin on the median and 30 on the gap."""
    acc = {}
    for agg in ("mean", "median"):
        _, lines = _run_fed(K=4, aggregator=agg, byzantine=1, attack="signflip", attack_scale=4.0, Nadmm=3,
                            max_minibatches=8, check_results=True, test_size=1000, train_size=8192, graphs=True)
        accs = [float(l.rsplit("%", 1)[1]) for l in lines if l.startswith("Accuracy of the network 0 ")]
        assert len(accs) == 10 * 3
        acc[agg] = accs[-1]
    print("final test accuracy of worker 0 with one sign-flipping attacker of four (%):", acc)
    assert acc["median"] >= 80.0 and acc["median"] >= acc["mean"] + 70.0


# ------------------------------------------------------------------------------------------ real ranks
def _worker(rank, world, port, out_dir):
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch.distributed as dist

    topo = Topology.from_env(world)
    dev = topo.device
    fused, base = FusedCollective(topo), TorchCollective(topo)
    report = {"transport": fused.heap.transport, "multicast": bool(fused.heap.allocs[-1]["mc_ptr"]), "cases": []}
    for use_mc in (True, False):
        fused.use_multimem = use_mc
        for two_shot in ("0", "1"):
            fused.two_shot_mode = two_shot
            for agg, b in (("median", 0), ("trimmed_mean", 0)):
                for N in (456, 73984, 1180672, 4720640):
                    g = torch.Generator(device=dev).manual_seed(1000 * rank + N)
                    x = fused.heap.alloc(-(-N // 32) * 32)[:N]
                    x.copy_(torch.randn(N, device=dev, generator=g))
                    xr = x.clone()
                    z = fused.zeros_like_block(x, "z")
                    zr = z.clone()
                    ok = True
                    for _ in range(2):
                        a = float(fused.robust_([x], z, agg, b))
                        bb = float(base.robust_([xr], zr, agg, b))
                        ok = ok and abs(a - bb) <= 1e-4 * abs(bb) + 1e-6
                        ok = ok and (torch.equal(z, zr) if agg == "median" else torch.allclose(z, zr, rtol=1e-6, atol=1e-6))
                        ok = ok and torch.equal(x, z)
                        d = 0.05 * torch.randn(N, device=dev, generator=g)
                        x.add_(d)
                        xr.add_(d)
                    report["cases"].append((use_mc, two_shot, agg, N, bool(ok), bool(fused.last_two_shot)))
    torch.cuda.synchronize()
    if rank == 0:
        torch.save(report, os.path.join(out_dir, "report.pt"))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.multigpu
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason=">= 2 CUDA devices required")
def test_fused_robust_across_ranks_matches_nccl(tmp_path):
    import torch.multiprocessing as mp
    port = 30900 + (os.getpid() % 1000)
    mp.spawn(_worker, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    rep = torch.load(str(tmp_path / "report.pt"), weights_only=False)
    print(rep["transport"], "multicast:", rep["multicast"])
    bad = [c for c in rep["cases"] if not c[4]]
    assert not bad, bad
