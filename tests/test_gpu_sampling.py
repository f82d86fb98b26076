"""Client sampling with sample-count weights on the H100: the sampled instantiations of the fused aggregation kernel select
the oracle's participants, match the ATen oracle (``TorchCollective``) bit for bit for FedAvg and within float32
tolerance for FedAdam, agree across loopback ranks (one-shot, two-shot, two replicas per rank), never read a worker that
sits out, replay from a CUDA graph, take one launch per round, and run a graphed ResNet18 ``federated_multi`` on
Dirichlet shards like the ATen collective does."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("CUDA device required", allow_module_level=True)

from federated_pytorch_test_b200.algo import sampling  # noqa: E402
from federated_pytorch_test_b200.parallel import Topology, TorchCollective  # noqa: E402
from federated_pytorch_test_b200.parallel.collective import SampleRound  # noqa: E402
from federated_pytorch_test_b200.parallel.fused import FusedCollective  # noqa: E402
from federated_pytorch_test_b200.parallel.loopback import LoopbackWorld  # noqa: E402

DEV = torch.device("cuda", 0)
KEY = sampling.sample_key(69)
HYPER = ("adam", 1e-2, 0.9, 0.99, 1e-3)


def _counts(K, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(1, 6000, (K,), generator=g, dtype=torch.int32).to(DEV)


def _blocks(coll, K, N):
    stride = -(-N // 32) * 32
    arena = coll.heap.alloc(K * stride)
    return [arena[k * stride: k * stride + N] for k in range(K)]


def test_selection_matches_the_oracle_for_1000_rounds():
    K, S = 16, 5
    coll = FusedCollective(Topology.single_process(K, DEV))
    xs = _blocks(coll, K, K)
    z = coll.zeros_like_block(xs[0], "z")
    n = torch.ones(K, dtype=torch.int32, device=DEV)
    t = torch.zeros(1, dtype=torch.int64, device=DEV)
    s = SampleRound(S, KEY, t, n)
    got = torch.empty(1000, K, device=DEV)
    for r in range(1000):
        for k, x in enumerate(xs):
            x.zero_()
            x[k] = k + 1.0
        coll.launch_fedavg_(xs, z, True, sample=s)
        got[r] = z
    coll.read_record()
    assert int(t) == 1000
    for r in range(1000):
        assert np.array_equal(np.flatnonzero(got[r].cpu().numpy() != 0), sampling.participants(KEY, r, K, S))


@pytest.mark.parametrize("kind", [None, "adam"])
@pytest.mark.parametrize("N", [7, 5130, 295423, 4720640])
@pytest.mark.parametrize("K", [3, 8, 16])
def test_fused_matches_oracle(K, N, kind):
    topo = Topology.single_process(K, DEV)
    coll, oracle = FusedCollective(topo), TorchCollective(topo)
    n = _counts(K, K + N)
    g = torch.Generator(device=DEV).manual_seed(N + K)
    for S in sorted({1, K // 2, K}):
        xs = _blocks(coll, K, N)
        z = coll.zeros_like_block(xs[0], "z")
        z.copy_(torch.randn(N, device=DEV, generator=g))
        zr = z.clone()
        t, tr = torch.full((1,), 3, dtype=torch.int64, device=DEV), torch.full((1,), 3, dtype=torch.int64, device=DEV)
        if kind:
            m, v = coll.zeros_like_block(xs[0], "m"), coll.zeros_like_block(xs[0], "v").fill_(1e-6)
            mr, vr = m.clone(), v.clone()
        n0 = coll.launches
        for r in range(2):
            for x in xs:
                x.copy_(z + 1e-2 * torch.randn(N, device=DEV, generator=g))
            xr = [x.clone() for x in xs]
            if kind:
                got = coll.fedopt_(xs, z, m, v, *HYPER, sample=SampleRound(S, KEY, t, n))
                want = float(oracle.fedopt_(xr, zr, mr, vr, *HYPER, sample=SampleRound(S, KEY, tr, n)))
                torch.testing.assert_close(z, zr, rtol=1e-5, atol=1e-6)
                torch.testing.assert_close(m, mr, rtol=1e-4, atol=1e-7)
                torch.testing.assert_close(v, vr, rtol=1e-4, atol=1e-12)
                zr.copy_(z)
                mr.copy_(m)
                vr.copy_(v)
            else:
                got = coll.fedavg_(xs, z, sample=SampleRound(S, KEY, t, n))
                want = float(oracle.fedavg_(xr, zr, sample=SampleRound(S, KEY, tr, n)))
                assert torch.equal(z, zr)                          # same terms, same order, each rounded
            assert coll.launches - n0 == r + 1                     # one launch per round
            assert got == pytest.approx(want, rel=1e-3, abs=1e-12)
            assert all(torch.equal(x, z) for x in xs)
        assert int(t) == int(tr) == 5 and coll.last_nonfinite == 0.0


def test_nan_in_a_worker_that_sits_out_is_harmless():
    K, S, N = 8, 3, 5131
    coll = FusedCollective(Topology.single_process(K, DEV))
    xs = _blocks(coll, K, N)
    z = coll.zeros_like_block(xs[0], "z")
    n = _counts(K, 1)
    t = torch.zeros(1, dtype=torch.int64, device=DEV)
    for r in range(4):
        out = [k for k in range(K) if k not in sampling.participants(KEY, r, K, S)]
        for x in xs:
            x.copy_(z + torch.rand(N, device=DEV))
        xs[out[0]].fill_(float("nan"))
        xs[out[1]][N - 1] = float("inf")                              # the scalar tail
        dual = coll.fedavg_(xs, z, sample=SampleRound(S, KEY, t, n))
        assert np.isfinite(dual) and coll.last_nonfinite == 0.0 and torch.isfinite(z).all()
        assert torch.equal(xs[out[0]], z) and torch.equal(xs[out[1]], z)


@pytest.mark.parametrize("kind", [None, "adam"])
@pytest.mark.parametrize("two_shot", ["0", "1"])
@pytest.mark.parametrize("W,per_rank", [(2, 1), (4, 1), (2, 2)])
@pytest.mark.parametrize("N", [5131, 295424, 4720640])
def test_loopback_ranks_agree(N, W, per_rank, two_shot, kind):
    K, S = W * per_rank, max(1, W * per_rank // 2)
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
    zs = [c.zeros_like_block(x[0], "z") for c, x in zip(world.colls, xs_rank)]
    n = _counts(K, N)
    ts = [torch.zeros(1, dtype=torch.int64, device=DEV) for _ in range(W)]
    ms = vs = None
    if kind:
        ms = [c.zeros_like_block(x[0], "m") for c, x in zip(world.colls, xs_rank)]
        vs = [c.zeros_like_block(x[0], "v").fill_(1e-6) for c, x in zip(world.colls, xs_rank)]
    oracle = TorchCollective(Topology.single_process(K, DEV))
    zr = torch.zeros(N, device=DEV)
    tr = torch.zeros(1, dtype=torch.int64, device=DEV)
    if kind:
        mr, vr = torch.zeros(N, device=DEV), torch.full((N,), 1e-6, device=DEV)
    for r in range(3):
        for x in by_worker:
            x.copy_(zs[0] + torch.randn(N, device=DEV, generator=g))
        xr = [x.clone() for x in by_worker]
        torch.cuda.synchronize()

        def one(rank, c):
            s = SampleRound(S, KEY, ts[rank], n)
            if kind:
                c.launch_fedopt_(xs_rank[rank], zs[rank], ms[rank], vs[rank], *HYPER, sample=s)
            else:
                c.launch_fedavg_(xs_rank[rank], zs[rank], True, sample=s)
        world.run(one)
        if kind:
            oracle.fedopt_(xr, zr, mr, vr, *HYPER, sample=SampleRound(S, KEY, tr, n))
        else:
            oracle.fedavg_(xr, zr, sample=SampleRound(S, KEY, tr, n))
        for c in world.colls:
            c.read_record()
            assert c.last_two_shot == (two_shot == "1" and per_rank == 1) and c.last_nonfinite == 0.0
        for zz in zs:
            assert torch.equal(zz, zs[0])
        for x in by_worker:
            assert torch.equal(x, zs[0])
        if kind:
            assert all(torch.equal(mm, ms[0]) and torch.equal(vv, vs[0]) for mm, vv in zip(ms, vs))
            torch.testing.assert_close(zs[0], zr, rtol=1e-5, atol=1e-6)
            zr.copy_(zs[0])
            mr.copy_(ms[0])
            vr.copy_(vs[0])
        else:
            assert torch.equal(zs[0], zr)
    assert all(int(t) == 3 for t in ts)


@pytest.mark.parametrize("kind", [None, "adam"])
def test_graph_replay_samples_fresh_rounds(kind):
    K, N, S = 8, 73984, 3
    n = _counts(K, 5)
    deltas = [torch.randn(K, N, device=DEV, generator=torch.Generator(device=DEV).manual_seed(r)) for r in range(3)]

    def setup():
        coll = FusedCollective(Topology.single_process(K, DEV))
        xs = _blocks(coll, K, N)
        z = coll.zeros_like_block(xs[0], "z")
        s = SampleRound(S, KEY, torch.zeros(1, dtype=torch.int64, device=DEV), n)
        mv = (coll.zeros_like_block(xs[0], "m"), coll.zeros_like_block(xs[0], "v").fill_(1e-6)) if kind else None
        return coll, xs, z, s, mv

    def launch(coll, xs, z, s, mv):
        if kind:
            coll.launch_fedopt_(xs, z, mv[0], mv[1], *HYPER, sample=s)
        else:
            coll.launch_fedavg_(xs, z, True, sample=s)

    coll, xs, z, s, mv = setup()
    eager = []
    for r in range(3):
        for k, x in enumerate(xs):
            x.copy_(z + deltas[r][k])
        launch(coll, xs, z, s, mv)
        coll.read_record()
        eager.append(z.clone())
    coll, xs, z, s, mv = setup()
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(st):
        with torch.cuda.graph(graph, stream=st):
            launch(coll, xs, z, s, mv)
    torch.cuda.current_stream().wait_stream(st)
    assert int(s.t) == 0
    for r in range(3):
        for k, x in enumerate(xs):
            x.copy_(z + deltas[r][k])
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(z, eager[r]) and int(s.t) == r + 1


def test_launcher_rejects_invalid_rounds():
    K, N = 4, 1024
    coll = FusedCollective(Topology.single_process(K, DEV))
    xs = _blocks(coll, K, N)
    z = coll.zeros_like_block(xs[0], "z")
    t = torch.zeros(1, dtype=torch.int64, device=DEV)
    n = torch.ones(K, dtype=torch.int32, device=DEV)
    for S in (K + 1, -1):
        with pytest.raises(RuntimeError, match="1 <= S <= K"):
            coll.fedavg_(xs, z, sample=SampleRound(S, KEY, t, n))
    with pytest.raises(ValueError, match="sampled aggregation"):
        coll.fedavg_(xs, z, write_back=False, sample=SampleRound(2, KEY, t, n))
    with pytest.raises(RuntimeError, match="sample counts"):
        coll.fedavg_(xs, z, sample=SampleRound(2, KEY, t, n[:3]))
    assert int(t) == 0


def test_warmup_runs_the_sampled_instantiations():
    K = 4
    coll = FusedCollective(Topology.single_process(K, DEV))
    coll.warm_sample = coll.warm_fedopt = True
    coll.warmup()
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------ end to end
def _run(**kw):
    from federated_pytorch_test_b200.api import federated_multi

    base = dict(K=8, use_resnet=True, Nloop=1, Nadmm=2, max_minibatches=3, train_size=4096, test_size=256,
                check_results=False, save_model=False, graphs=True, partition="dirichlet", clients_per_round=3,
                dirichlet_alpha=1.0, default_batch=64)
    lines = []
    eng = federated_multi.run(federated_multi.Config(**{**base, **kw}), log=lines.append)
    return eng, lines


def test_graphed_resnet18_dirichlet_sampled_run_matches_aten(monkeypatch):
    from federated_pytorch_test_b200.algo.engine import Engine

    steps = []
    orig = Engine._run_replicas

    def run_replicas(self, visit, nloop, epoch, N):
        ids = self.strategy.round_participants()
        before = [int(o.t_dev) if o.t_dev is not None else o.t for o in self.optimizers]
        orig(self, visit, nloop, epoch, N)
        after = [int(o.t_dev) if o.t_dev is not None else o.t for o in self.optimizers]
        steps.append(all((a > b) == (rep.ck in ids) for a, b, rep in zip(after, before, self.replicas)))

    monkeypatch.setattr(Engine, "_run_replicas", run_replicas)
    eng, fused = _run()
    assert eng.coll.name == "fused" and eng.strategy.sampled and all(steps) and len(steps) == 20
    monkeypatch.setattr(Engine, "_run_replicas", orig)
    _, aten = _run(collective="torch", graphs=False, fast=False)
    df = [float(l.rsplit("=", 1)[1]) for l in fused if l.startswith("dual (")]
    da = [float(l.rsplit("=", 1)[1]) for l in aten if l.startswith("dual (")]
    assert len(df) == len(da) == 20
    for a, b in zip(df, da):                                            # TF32 convolutions against fp32 ATen
        assert a == pytest.approx(b, rel=5e-2)
    assert eng.strategy.samp_rounds == int(eng.strategy.samp_t) == 20


# ------------------------------------------------------------------------------------------ real ranks
def _worker(rank, world, port, out_dir):
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch.distributed as dist

    topo = Topology.from_env(2 * world)
    dev = topo.device
    fused, base = FusedCollective(topo), TorchCollective(topo)
    n = torch.tensor([100, 2000, 350, 4000], dtype=torch.int32, device=dev)
    cases = []
    for two_shot in ("0", "1"):
        fused.two_shot_mode = two_shot
        for N in (456, 1180672):
            g = torch.Generator(device=dev).manual_seed(1000 * rank + N)
            xs = [fused.heap.alloc(-(-N // 32) * 32)[:N] for _ in range(2)]
            for x in xs:
                x.copy_(torch.randn(N, device=dev, generator=g))
            xr = [x.clone() for x in xs]
            z = fused.zeros_like_block(xs[0], "z")
            zr = z.clone()
            t, tr = torch.zeros(1, dtype=torch.int64, device=dev), torch.zeros(1, dtype=torch.int64, device=dev)
            ok = True
            for _ in range(3):
                fused.fedavg_(xs, z, sample=SampleRound(2, KEY, t, n))
                base.fedavg_(xr, zr, sample=SampleRound(2, KEY, tr, n))
                ok = ok and torch.equal(z, zr) and all(torch.equal(x, z) for x in xs)
                for x, y in zip(xs, xr):
                    d = 0.05 * torch.randn(N, device=dev, generator=g)
                    x.add_(d)
                    y.add_(d)
            cases.append((two_shot, N, bool(ok)))
    torch.cuda.synchronize()
    if rank == 0:
        torch.save(cases, os.path.join(out_dir, "report.pt"))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.multigpu
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason=">= 2 CUDA devices required")
def test_fused_sampled_across_ranks_matches_nccl(tmp_path):
    import torch.multiprocessing as mp

    port = 31900 + (os.getpid() % 1000)
    mp.spawn(_worker, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    bad = [c for c in torch.load(str(tmp_path / "report.pt"), weights_only=False) if not c[2]]
    assert not bad, bad
