"""Multi-GPU: the fused NVLink collectives across processes (one rank per GPU) against NCCL all-reduce.
Needs >= 2 GPUs; skipped otherwise."""
import os

import pytest
import torch

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu]

if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
    pytest.skip(">= 2 CUDA devices required", allow_module_level=True)


def _worker(rank, world, port, out_dir):
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch.distributed as dist
    from federated_pytorch_test_b200.parallel import Topology, TorchCollective
    from federated_pytorch_test_b200.parallel.fused import FusedCollective

    topo = Topology.from_env(world)
    dev = topo.device
    fused, base = FusedCollective(topo), TorchCollective(topo)
    report = {"transport": fused.heap.transport, "multicast": bool(fused.heap.allocs[-1]["mc_ptr"]), "cases": []}
    for use_mc in (True, False):
        fused.use_multimem = use_mc
        for N in (456, 5130, 73984, 1180672, 3673088, 4720640):
            g = torch.Generator(device=dev).manual_seed(1000 * rank + N)
            arena = fused.heap.alloc(-(-N // 32) * 32)
            x = arena[:N]
            x.copy_(torch.randn(N, device=dev, generator=g))
            xr = x.clone()
            z, zr = fused.zeros_like_block(x, "z"), torch.zeros(N, device=dev)     # symmetric z: two-shot broadcast target
            d1 = float(fused.fedavg_([x], z, True))
            d2 = float(base.fedavg_([xr], zr, True))
            ok = abs(d1 - d2) <= 1e-4 * abs(d2) + 1e-6 and torch.allclose(x, xr, rtol=1e-5, atol=1e-6) and torch.allclose(z, zr, rtol=1e-5, atol=1e-6)
            x.add_(torch.randn(N, device=dev, generator=g))
            xr.copy_(x)
            y, yr = fused.zeros_like_block(x, "y"), torch.zeros(N, device=dev)
            for _ in range(2):
                a = fused.admm_([x], [y], z, 0.1)
                b = base.admm_([xr], [yr], zr, 0.1)
                ok = ok and abs(float(a[0]) - float(b[0])) <= 1e-3 * abs(float(b[0])) + 1e-6
                ok = ok and abs(float(a[1]) - float(b[1])) <= 1e-3 * abs(float(b[1])) + 1e-6
                ok = ok and torch.allclose(y, yr, rtol=1e-4, atol=1e-5) and torch.allclose(z, zr, rtol=1e-4, atol=1e-5)
            a = fused.fedprox_([x], z, 1.0)
            b = base.fedprox_([xr], zr, 1.0)
            ok = ok and abs(float(a[1]) - float(b[1])) <= 1e-3 * abs(float(b[1])) + 1e-6
            report["cases"].append((use_mc, N, bool(ok), bool(fused.last_two_shot)))
    torch.cuda.synchronize()
    if rank == 0:
        torch.save(report, os.path.join(out_dir, "report.pt"))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("world", sorted({2, min(8, torch.cuda.device_count() if torch.cuda.is_available() else 2)}))
def test_fused_collectives_across_ranks(tmp_path, world):
    import torch.multiprocessing as mp
    port = 29700 + (os.getpid() % 1000)
    mp.spawn(_worker, args=(world, port, str(tmp_path)), nprocs=world, join=True)
    rep = torch.load(str(tmp_path / "report.pt"), weights_only=False)
    print(rep["transport"], "multicast:", rep["multicast"])
    bad = [c for c in rep["cases"] if not c[2]]
    assert not bad, bad


def _engine_worker(rank, world, port, out_dir, K, algo):
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch.distributed as dist
    from federated_pytorch_test_b200.api import consensus_multi, federated_multi

    mod = federated_multi if algo == "fedavg" else consensus_multi
    extra = {} if algo == "fedavg" else dict(bb_update=True)
    lines = []
    cfg = mod.Config(K=K, Nloop=1, Nadmm=3, max_minibatches=2, check_results=False, save_model=False, train_size=4096,
                     test_size=128, model="Net", graphs=False, fast=True, collective="fused", **extra)
    eng = mod.run(cfg, log=lines.append)
    torch.cuda.synchronize()
    if rank == 0:
        torch.save({"lines": lines, "coll": eng.coll.name, "local": [r.ck for r in eng.replicas]}, os.path.join(out_dir, "%s.pt" % algo))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("algo", ["fedavg", "admm"])
def test_co_resident_replicas_across_ranks_match_single_process(tmp_path, algo):
    """K = 4 workers on 2 GPUs (two co-resident replicas per rank, fused NVLink aggregation) must reproduce the
    residual trace of the single-process K = 4 run (the reference's topology)."""
    import torch.multiprocessing as mp
    from federated_pytorch_test_b200.api import consensus_multi, federated_multi
    port = 29800 + (os.getpid() % 1000) + (7 if algo == "admm" else 0)
    mp.spawn(_engine_worker, args=(2, port, str(tmp_path), 4, algo), nprocs=2, join=True)
    got = torch.load(str(tmp_path / ("%s.pt" % algo)), weights_only=False)
    assert got["coll"] == "fused" and got["local"] == [0, 2]
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        os.environ.pop(k, None)
    mod = federated_multi if algo == "fedavg" else consensus_multi
    extra = {} if algo == "fedavg" else dict(bb_update=True)
    lines = []
    mod.run(mod.Config(K=4, Nloop=1, Nadmm=3, max_minibatches=2, check_results=False, save_model=False, train_size=4096,
                       test_size=128, model="Net", graphs=False, fast=True, collective="fused", distributed=False, **extra),
            log=lines.append)
    key = "dual (" if algo == "fedavg" else "block=["
    a = [l for l in got["lines"] if l.startswith(key)]
    b = [l for l in lines if l.startswith(key)]
    assert len(a) == len(b) == 15
    for x, y in zip(a, b):
        vx, vy = float(x.rsplit("=", 1)[1]), float(y.rsplit("=", 1)[1])
        assert vx == pytest.approx(vy, rel=5e-3, abs=1e-9), (x, y)
