"""Server optimizers of federated averaging on the H100: the FedOpt instantiation of the fused aggregation kernel against
the ATen oracle (``TorchCollective.fedopt_``) on one process, on loopback ranks (one-shot and two-shot), inside a CUDA
graph and across real ranks; the non-finite guard, the launch count and ``federated_multi`` ResNet18 runs."""
import math
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("CUDA device required", allow_module_level=True)

from federated_pytorch_test_b200.algo.strategies import FedOpt  # noqa: E402
from federated_pytorch_test_b200.ops import cuda_ops  # noqa: E402
from federated_pytorch_test_b200.parallel import Topology, TorchCollective  # noqa: E402
from federated_pytorch_test_b200.parallel.fused import FusedCollective  # noqa: E402
from federated_pytorch_test_b200.parallel.loopback import LoopbackWorld  # noqa: E402

DEV = torch.device("cuda", 0)
KINDS = ["avgm", "adagrad", "adam", "yogi"]
SIZES = [850, 5130, 73984, 295424, 4720640]
HP = {"avgm": (0.9, 0.8, 0.99, 1e-3), "adagrad": (0.05, 0.9, 0.99, 1e-3), "adam": (0.02, 0.9, 0.95, 1e-3),
      "yogi": (0.03, 0.85, 0.99, 1e-3)}       # lr, beta1 (avgm: momentum), beta2, tau


def _state(make, x, tau):
    z, m, v = make(x, "z"), make(x, "srv_m"), make(x, "srv_v")
    v.fill_(tau * tau)
    return z, m, v


def _close(a, b, rtol=1e-5, atol=1e-6, keep=None):
    if keep is not None:
        a, b = a[keep], b[keep]
    torch.testing.assert_close(a, b, rtol=rtol, atol=atol)


def _yogi_ties(kind, mean, z, v, ties):
    """Yogi's v - (1 - beta2) d^2 sign(v - d^2) jumps where v = d^2: where the oracle's v and d^2 agree to 1e-4, rounding
    differences of d between the kernel and ATen may pick the other branch, and that element's state differs from then
    on.  Marks such elements (they are excluded from the comparison and must stay rare)."""
    if kind == "yogi":
        d2 = (mean - z) ** 2
        ties |= (v - d2).abs() <= 1e-4 * (v + d2)
        assert int(ties.sum()) <= max(2, ties.numel() // 1000)
    return ~ties


def _perturb(xs, g):
    """Local training moves every replica differently (same draws for the fused run and the oracle)."""
    return [0.05 * torch.randn(x.numel(), device=DEV, generator=g) + 0.01 for x in xs]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("N", SIZES)
@pytest.mark.parametrize("K", [1, 4])
def test_fused_matches_oracle_single_process(kind, N, K):
    lr, b1, b2, tau = HP[kind]
    topo = Topology.single_process(K, DEV)
    coll, oracle = FusedCollective(topo), TorchCollective(topo)
    stride = -(-N // 32) * 32
    arena = coll.heap.alloc(K * stride)
    xs = [arena[k * stride: k * stride + N] for k in range(K)]
    g = torch.Generator(device=DEV).manual_seed(N + K)
    for x in xs:
        x.copy_(torch.randn(N, device=DEV, generator=g))
    z, m, v = _state(coll.zeros_like_block, xs[0], tau)
    z.copy_(torch.stack(xs).mean(0))
    xr = [x.clone() for x in xs]
    zr, mr, vr = z.clone(), m.clone(), v.clone()
    ties = torch.zeros(N, dtype=torch.bool, device=DEV)
    for _ in range(3):
        for x, y, d in zip(xs, xr, _perturb(xs, g)):
            x.add_(d)
            y.add_(d)
        keep = _yogi_ties(kind, torch.stack(xr).mean(0), zr, vr, ties)
        got = coll.fedopt_(xs, z, m, v, kind, lr, b1, b2, tau)
        want = float(oracle.fedopt_(xr, zr, mr, vr, kind, lr, b1, b2, tau))
        assert got == pytest.approx(want, rel=1e-4)
        _close(z, zr, keep=keep)
        _close(m, mr, keep=keep)
        if kind != "avgm":
            _close(v, vr, rtol=1e-4, atol=1e-9, keep=keep)
        for x, y in zip(xs, xr):
            _close(x, y, keep=keep)
            assert torch.equal(x, z)
    assert coll.last_nonfinite == 0.0 and not coll.last_two_shot


def _slices(world, N, seed):
    stride = -(-N // 32) * 32
    xs = [t[:N] for t in world.alloc(stride)]
    g = torch.Generator(device=DEV).manual_seed(seed)
    for x in xs:
        x.copy_(torch.randn(N, device=DEV, generator=g))
    return xs, g


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("N", SIZES)
@pytest.mark.parametrize("W", [2, 4])
@pytest.mark.parametrize("two_shot", ["0", "1"])
def test_loopback_matches_oracle_and_ranks_agree_bitwise(kind, N, W, two_shot):
    lr, b1, b2, tau = HP[kind]
    world = LoopbackWorld(W, DEV, max_blocks=8, timeout_s=10.0)
    for c in world.colls:
        c.two_shot_mode = two_shot
    xs, g = _slices(world, N, 3 * N + W)
    st = [_state(c.zeros_like_block, x, tau) for c, x in zip(world.colls, xs)]
    z0 = torch.stack(xs).mean(0)
    for z, _, _ in st:
        z.copy_(z0)
    oracle = TorchCollective(Topology.single_process(W, DEV))
    xr = [x.clone() for x in xs]
    zr, mr, vr = z0.clone(), torch.zeros_like(z0), torch.full_like(z0, tau * tau)
    ties = torch.zeros(N, dtype=torch.bool, device=DEV)
    for _ in range(3):
        for x, y, d in zip(xs, xr, _perturb(xs, g)):
            x.add_(d)
            y.add_(d)
        keep = _yogi_ties(kind, torch.stack(xr).mean(0), zr, vr, ties)
        world.run(lambda r, c: c._launch_fedopt([xs[r]], st[r][0], st[r][1], st[r][2], kind, lr, b1, b2, tau))
        want = float(oracle.fedopt_(xr, zr, mr, vr, kind, lr, b1, b2, tau))
        for r, c in enumerate(world.colls):
            rec = c.read_record()
            assert rec[0] == pytest.approx(want, rel=1e-4)
            assert bool(rec[6]) == (two_shot == "1") and rec[2] == 0.0
            z, m, v = st[r]
            _close(z, zr, keep=keep)
            _close(m, mr, keep=keep)
            if kind != "avgm":
                _close(v, vr, rtol=1e-4, atol=1e-9, keep=keep)
            _close(xs[r], xr[r], keep=keep)
            assert torch.equal(xs[r], z)
            for a, b in zip(st[r], st[0]):              # every rank holds the same server state, bit for bit
                assert torch.equal(a, b)


def test_nonfinite_replica_is_counted_and_raised_by_the_guard():
    topo = Topology.single_process(4, DEV)
    coll = FusedCollective(topo)
    arena = coll.heap.alloc(4 * 4096)
    xs = [arena[k * 4096:(k + 1) * 4096] for k in range(4)]
    for x in xs:
        x.normal_()
    z, m, v = _state(coll.zeros_like_block, xs[0], 1e-3)
    xs[2][77] = float("nan")
    dual = coll.fedopt_(xs, z, m, v, "adam", 1e-2, 0.9, 0.99, 1e-3)
    assert coll.last_nonfinite >= 1.0 and not math.isfinite(dual)

    from federated_pytorch_test_b200.algo.engine import Engine
    from federated_pytorch_test_b200.api import federated_multi

    orig_init = Engine.__init__

    def patched(self, *a, **k):
        orig_init(self, *a, **k)

        def hook(e):
            if e.steps_done == 2:                        # one replica diverges inside the first round
                e.replicas[1].arenas["net"].data.fill_(float("nan"))
        self.step_hook = hook
    Engine.__init__ = patched
    try:
        with pytest.raises(FloatingPointError, match="non-finite"):
            federated_multi.run(federated_multi.Config(K=2, model="Net", Nloop=1, Nadmm=2, max_minibatches=2,
                                                       check_results=False, save_model=False, train_size=2048,
                                                       test_size=128, graphs=False, server_opt="adam"), log=lambda s: None)
    finally:
        Engine.__init__ = orig_init


def test_fedopt_round_is_graph_capturable():
    """No memset, clone or host read inside a round: a FedAdam aggregation captured into a CUDA graph, replayed 3 times
    on fresh replica values, against the oracle."""
    K, N, kind = 4, 73984, "adam"
    lr, b1, b2, tau = HP[kind]
    topo = Topology.single_process(K, DEV)
    coll = FusedCollective(topo)
    stride = -(-N // 32) * 32
    arena = coll.heap.alloc(K * stride)
    xs = [arena[k * stride: k * stride + N] for k in range(K)]
    g = torch.Generator(device=DEV).manual_seed(9)
    z, m, v = _state(coll.zeros_like_block, xs[0], tau)
    coll._launch_fedopt(xs, z, m, v, kind, lr, b1, b2, tau)            # warm-up (lazy init) outside the capture
    torch.cuda.synchronize()
    for x in xs:
        x.copy_(torch.randn(N, device=DEV, generator=g))
    z.copy_(torch.stack(xs).mean(0))
    m.zero_()
    v.fill_(tau * tau)
    xr = [x.clone() for x in xs]
    zr, mr, vr = z.clone(), m.clone(), v.clone()
    st = torch.cuda.Stream()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=st):
        coll._launch_fedopt(xs, z, m, v, kind, lr, b1, b2, tau)
    e0 = int(coll.sync[0])
    oracle = TorchCollective(topo)
    for _ in range(3):
        for x, y, d in zip(xs, xr, _perturb(xs, g)):
            x.add_(d)
            y.add_(d)
        graph.replay()
        want = float(oracle.fedopt_(xr, zr, mr, vr, kind, lr, b1, b2, tau))
        assert coll.read_record()[0] == pytest.approx(want, rel=1e-4)
        _close(z, zr)
        _close(m, mr)
        _close(v, vr, rtol=1e-4, atol=1e-9)
        for x, y in zip(xs, xr):
            _close(x, y)
    assert int(coll.sync[0]) == e0 + 3


@pytest.mark.parametrize("deferred", [False, True])
def test_one_launch_per_round_plus_one_per_visit(deferred):
    K, N = 4, 5130
    topo = Topology.single_process(K, DEV)
    coll = FusedCollective(topo)
    strat = FedOpt(coll, topo, "yogi")
    arena = coll.heap.alloc(K * 5152)
    xs = [arena[k * 5152: k * 5152 + N] for k in range(K)]
    for x in xs:
        x.normal_()
    coll.warmup()
    torch.cuda.synchronize()
    before = cuda_ops.launch_count()
    strat.begin_block(0, N, xs)
    assert cuda_ops.launch_count() - before == 1                          # z <- mean of the replicas
    for r in range(3):
        for x in xs:
            x.add_(0.01)
        before = cuda_ops.launch_count()
        if deferred:
            res = strat.aggregate_end(strat.aggregate_begin(r))
        else:
            res = strat.aggregate(r)
        assert cuda_ops.launch_count() - before == 1
        assert math.isfinite(res["dual"]) and res["dual"] > 0.0


# ------------------------------------------------------------------------------------------ engine
def _run_fed(**kw):
    from federated_pytorch_test_b200.api import federated_multi
    lines = []
    base = dict(K=2, model="ResNet18", Nloop=1, Nadmm=2, max_minibatches=4, check_results=False, save_model=False,
                train_size=4096, test_size=256, server_opt="adam")
    eng = federated_multi.run(federated_multi.Config(**{**base, **kw}), log=lines.append)
    return eng, lines


def test_resnet18_fedadam_graphed_equals_aten():
    e1, l_fast = _run_fed(graphs=True)
    e2, l_aten = _run_fed(graphs=False, fast=False)
    assert e1.coll.name == "fused" and e2.coll.name == "torch" and isinstance(e1.strategy, FedOpt)
    d_fast = [float(l.rsplit("=", 1)[1]) for l in l_fast if l.startswith("dual (")]
    d_aten = [float(l.rsplit("=", 1)[1]) for l in l_aten if l.startswith("dual (")]
    print("fused + graphed:", d_fast[:6], "\nATen:", d_aten[:6])
    assert len(d_fast) == len(d_aten) == 20
    for a, b in zip(d_fast, d_aten):                                     # TF32 convolutions against fp32 ATen
        assert a == pytest.approx(b, rel=5e-2)
    assert getattr(e1, "graph_replays", 0) > 0


def test_resnet18_fedadam_default_rate_beats_chance():
    _, lines = _run_fed(Nadmm=3, max_minibatches=8, check_results=True, test_size=1000, graphs=True)
    accs = [float(l.rsplit("%", 1)[1]) for l in lines if l.startswith("Accuracy of the network")]
    print("test accuracy after each round, FedAdam at server_lr 1e-2 (%):", accs)
    assert len(accs) == 2 * 10 * 3                                        # 2 workers, 10 blocks, 3 rounds per visit
    assert accs[-1] >= 50.0                                               # chance is 10 %


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
            for kind in ("avgm", "adam", "yogi"):
                lr, b1, b2, tau = HP[kind]
                for N in (456, 73984, 1180672, 4720640):
                    g = torch.Generator(device=dev).manual_seed(1000 * rank + N)
                    x = fused.heap.alloc(-(-N // 32) * 32)[:N]
                    x.copy_(torch.randn(N, device=dev, generator=g))
                    xr = x.clone()
                    z, m, v = _state(fused.zeros_like_block, x, tau)
                    z0 = base.sum_blocks([x]).div_(world)
                    z.copy_(z0)
                    zr, mr, vr = z0.clone(), m.clone(), v.clone()
                    ok = True
                    ties = torch.zeros(N, dtype=torch.bool, device=dev)
                    for _ in range(3):
                        d = 0.05 * torch.randn(N, device=dev, generator=g)
                        x.add_(d)
                        xr.add_(d)
                        keep = _yogi_ties(kind, base.sum_blocks([xr]).div_(world), zr, vr, ties)
                        a = float(fused.fedopt_([x], z, m, v, kind, lr, b1, b2, tau))
                        b = float(base.fedopt_([xr], zr, mr, vr, kind, lr, b1, b2, tau))
                        ok = ok and abs(a - b) <= 1e-4 * abs(b) + 1e-6
                        ok = ok and all(torch.allclose(p[keep], q[keep], rtol=1e-5, atol=1e-6)
                                        for p, q in ((x, xr), (z, zr), (m, mr)))
                        ok = ok and (kind == "avgm" or torch.allclose(v[keep], vr[keep], rtol=1e-4, atol=1e-9))
                    report["cases"].append((use_mc, two_shot, kind, N, bool(ok), bool(fused.last_two_shot)))
    torch.cuda.synchronize()
    if rank == 0:
        torch.save(report, os.path.join(out_dir, "report.pt"))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.multigpu
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason=">= 2 CUDA devices required")
def test_fused_fedopt_across_ranks_matches_nccl(tmp_path):
    import torch.multiprocessing as mp
    port = 29900 + (os.getpid() % 1000)
    mp.spawn(_worker, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    rep = torch.load(str(tmp_path / "report.pt"), weights_only=False)
    print(rep["transport"], "multicast:", rep["multicast"])
    bad = [c for c in rep["cases"] if not c[4]]
    assert not bad, bad
