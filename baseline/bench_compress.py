"""Cost of compressed client updates in federated averaging (``--compress_bits 8|4 [--compress_ef]``): a compressed round is
one launch of a compressed instantiation of the fused aggregation kernel (encode the local replicas, reduce the K
workers' codes, write back).

  (a) one GPU: device time of one round at each of the ten ResNet18 block sizes, K = 8 co-resident replicas (the one-shot
      path), for six arms: plain FedAvg; 8-bit and 4-bit codes, each without and with error feedback; 8-bit + FedAdam.
      Every round starts by restoring perturbed replicas (untimed) and is timed on its own with CUDA events; median over
      ``--rounds`` rounds.  Byte models (HBM traffic, K replicas of N floats, payload P = N b / 8 + 4 ceil(N / 128)):
      FedAvg 4 N (2 K + 3) (K replicas read, z read / written / read again, K replicas written); compressed
      4 N (2 K + 4) + 2 K P (the same, z once more for the encoder, every payload written and read), + 8 N K for error
      feedback (read and written), + 16 N for FedAdam's m and v.  Event timing of single rounds includes a few
      microseconds of event overhead, which dominates the small blocks;
  (b) several GPUs (one process per GPU, one replica per rank, K = #GPUs): the same arms without FedAdam, one-shot and
      two-shot, with the peer bytes a rank pulls per round (one-shot: (K - 1) 4 N for FedAvg, (K - 1) P compressed;
      two-shot: a 1/K slice of that).  With one visible GPU this prints "not measured".

Prints the device name, power limit and max SM clock beside the numbers, then one JSON line.  Writes nothing to disk.

    python baseline/bench_compress.py [--rounds 30]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from baseline.bench_fedopt import _power_limit, resnet18_block_sizes  # noqa: E402

K_AGG = 8
ARMS = ("fedavg", "q8", "q8_ef", "q4", "q4_ef", "q8_fedadam")
ARM_Q = {"q8": (8, False), "q8_ef": (8, True), "q4": (4, False), "q4_ef": (4, True), "q8_fedadam": (8, False)}


def hbm_bytes(arm: str, N: int, K: int = K_AGG) -> float:
    from federated_pytorch_test_b200.algo.compress import payload_bytes

    if arm == "fedavg":
        return 4.0 * N * (2 * K + 3)
    bits, ef = ARM_Q[arm]
    b = 4.0 * N * (2 * K + 4) + 2.0 * K * payload_bytes(N, bits)
    return b + (8.0 * N * K if ef else 0.0) + (16.0 * N if arm == "q8_fedadam" else 0.0)


def peer_bytes(arm: str, N: int, K: int, two_shot: bool) -> float:
    from federated_pytorch_test_b200.algo.compress import payload_bytes

    per = 4.0 * N if arm == "fedavg" else float(payload_bytes(N, ARM_Q[arm][0]))
    return (K - 1) * per / (K if two_shot else 1)


def _arms(coll, xs, z, m, v, t):
    """One launch per arm (``None`` for FedAvg's compression argument)."""
    from federated_pytorch_test_b200.parallel.collective import QuantRound

    out = {}
    for a in ARMS:
        if a == "fedavg":
            out[a] = lambda: coll._launch(0, xs, None, z, 0.0)
            continue
        bits, ef = ARM_Q[a]
        pay = [coll.payload_like_block(x, bits) for x in xs]
        q = QuantRound(bits, 0, t, [c for c, _ in pay], [s for _, s in pay], [torch.zeros_like(x) for x in xs] if ef else None)
        if a == "q8_fedadam":
            out[a] = (lambda q=q: coll._launch_fedopt(xs, z, m, v, "adam", 1e-2, 0.9, 0.99, 1e-3, compress=q))
        else:
            out[a] = (lambda q=q: coll._launch(0, xs, None, z, 0.0, compress=q))
    return out


def aggregation(args, dev) -> dict:
    from federated_pytorch_test_b200.parallel import Topology
    from federated_pytorch_test_b200.parallel.fused import FusedCollective

    coll = FusedCollective(Topology.single_process(K_AGG, dev))
    coll.warm_fedopt = True
    coll.warm_compress = 8
    coll.warmup()
    res = []
    for N in resnet18_block_sizes(dev):
        stride = -(-N // 32) * 32
        arena = coll.heap.alloc(K_AGG * stride)
        xs = [arena[k * stride: k * stride + N] for k in range(K_AGG)]
        z = coll.zeros_like_block(xs[0], "z")
        m, v = coll.zeros_like_block(xs[0], "m"), coll.zeros_like_block(xs[0], "v").fill_(1e-6)
        g = torch.Generator(device=dev).manual_seed(N)
        z0 = torch.randn(N, device=dev, generator=g)
        saved = [z0 + 1e-2 * torch.randn(N, device=dev, generator=g) for _ in range(K_AGG)]
        t = torch.zeros(1, dtype=torch.int64, device=dev)
        launch = _arms(coll, xs, z, m, v, t)
        times = {a: [] for a in ARMS}
        for rnd in range(args.rounds + 2):
            for a in ARMS:
                z.copy_(z0)
                for x, s in zip(xs, saved):
                    x.copy_(s)
                ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
                ev[0].record()
                launch[a]()
                ev[1].record()
                ev[1].synchronize()
                if rnd >= 2:                                   # two untimed rounds per arm first
                    times[a].append(ev[0].elapsed_time(ev[1]) * 1e3)
        coll.read_record()
        row = {"N": N}
        for a in ARMS:
            us = statistics.median(times[a])
            row[a] = {"us": us, "hbm_bytes": hbm_bytes(a, N), "hbm_GBs": hbm_bytes(a, N) / (us * 1e-6) / 1e9}
        res.append(row)
        del arena, xs, saved
    return {"K": K_AGG, "rounds": args.rounds, "blocks": res}


def _rank_worker(rank, world, port, rounds, sizes, out):
    import torch.distributed as dist

    from federated_pytorch_test_b200.parallel import Topology
    from federated_pytorch_test_b200.parallel.fused import FusedCollective

    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", init_method="tcp://127.0.0.1:%d" % port, rank=rank, world_size=world, device_id=dev)
    topo = Topology(K=world, world_size=world, rank=rank, device=dev, group=dist.group.WORLD)
    coll = FusedCollective(topo)
    coll.warm_compress = 8
    coll.warmup()
    res = []
    for N in sizes:
        stride = -(-N // 32) * 32
        x = coll.heap.alloc(stride)[:N]
        z = coll.zeros_like_block(x, "z")
        g = torch.Generator(device=dev).manual_seed(N + rank)
        z0 = torch.randn(N, device=dev, generator=torch.Generator(device=dev).manual_seed(N))
        saved = z0 + 1e-2 * torch.randn(N, device=dev, generator=g)
        t = torch.zeros(1, dtype=torch.int64, device=dev)
        launch = {a: f for a, f in _arms(coll, [x], z, None, None, t).items() if a != "q8_fedadam"}
        row = {"N": N}
        for mode in ("0", "1"):
            coll.two_shot_mode = mode
            times = {a: [] for a in launch}
            for rnd in range(rounds + 2):
                for a, f in launch.items():
                    z.copy_(z0)
                    x.copy_(saved)
                    topo.barrier()
                    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
                    ev[0].record()
                    f()
                    ev[1].record()
                    ev[1].synchronize()
                    if rnd >= 2:
                        times[a].append(ev[0].elapsed_time(ev[1]) * 1e3)
            coll.read_record()
            two = coll.last_two_shot
            row["two_shot" if mode == "1" else "one_shot"] = {
                a: {"us": statistics.median(v), "peer_bytes": peer_bytes(a, N, world, two), "two_shot": two}
                for a, v in times.items()}
        res.append(row)
    if rank == 0:
        torch.save(res, out)
    dist.destroy_process_group()


def multi_gpu(args, dev) -> dict:
    world = torch.cuda.device_count()
    if world < 2:
        return {"measured": False}
    import tempfile

    import torch.multiprocessing as mp

    sizes = resnet18_block_sizes(dev)
    with tempfile.TemporaryDirectory() as tmp:
        out = os.path.join(tmp, "r0.pt")
        mp.spawn(_rank_worker, args=(world, 29600 + os.getpid() % 2000, args.rounds, sizes, out), nprocs=world, join=True)
        blocks = torch.load(out, weights_only=False)
    return {"measured": True, "world": world, "blocks": blocks}


def main(argv=None) -> dict:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--rounds", type=int, default=30, help="timed rounds per arm and block size")
    ap.add_argument("--skip-multi", action="store_true", help="run (a) only")
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_compress.py measures the GPU path: no CUDA device")
    dev = torch.device("cuda", torch.cuda.current_device())
    res = {"device": torch.cuda.get_device_name(dev), "power_limit,max_sm_clock": _power_limit()}
    res["aggregation"] = aggregation(args, dev)
    res["multi_gpu"] = {"measured": False} if args.skip_multi else multi_gpu(args, dev)
    print("device: %s  (power.limit, clocks.max.sm: %s)" % (res["device"], res["power_limit,max_sm_clock"]))
    for row in res["aggregation"]["blocks"]:
        print("  (a) N=%8d  " % row["N"] + "  ".join(
            "%s %6.1f us (%5.0f GB/s)" % (a, row[a]["us"], row[a]["hbm_GBs"]) for a in ARMS))
    mg = res["multi_gpu"]
    if not mg["measured"]:
        print("  (b) several GPUs: not measured (%d visible)" % torch.cuda.device_count())
    else:
        for row in mg["blocks"]:
            for mode in ("one_shot", "two_shot"):
                print("  (b) W=%d N=%8d %s  " % (mg["world"], row["N"], mode) + "  ".join(
                    "%s %6.1f us (%.2f MB from peers)" % (a, r["us"], r["peer_bytes"] / 1e6) for a, r in row[mode].items()))
    print(json.dumps(res))
    return res


if __name__ == "__main__":
    main()
