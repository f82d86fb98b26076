"""Cost of secure aggregation in federated averaging (``--secagg``): a SecAgg round is one launch of a SecAgg instantiation
of the fused aggregation kernel (encode and mask the local replicas' updates with pairwise ChaCha20 keystreams, sum the K
workers' payloads as integers, decode, write back).

  (a) one GPU: device time of one round at each of the ten ResNet18 block sizes, K = 8 co-resident replicas (the one-shot
      path), for three arms: plain FedAvg, SecAgg and SecAgg + FedAdam.  Every round starts by restoring perturbed
      replicas (untimed) and is timed on its own with CUDA events; median over ``--rounds`` rounds.  Work model beside
      the times: co-resident, every worker masks with K - 1 keystreams, so a round computes K (K - 1) N / 16 ChaCha20
      blocks (about 1 k integer instructions each: 20 rounds of 4 quarter-rounds of 12 operations, plus the additions);
      payload HBM bytes 8 N K (every 4-byte payload word written once and read once);
  (b) several GPUs (one process per GPU, one replica per rank, K = #GPUs): FedAvg and SecAgg, one-shot and two-shot; a
      rank computes only its own worker's (K - 1) N / 16 blocks.  With one visible GPU this prints "not measured".

Prints the device name, power limit and max SM clock beside the numbers, then one JSON line.  Writes nothing to disk.

    python baseline/bench_secagg.py [--rounds 30]
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
ARMS = ("fedavg", "secagg", "secagg_fedadam")
CHACHA_INSNS = 1000                    # integer instructions per ChaCha20 block, approximately


def chacha_blocks(N: int, K: int, per_rank: bool = False) -> int:
    """ChaCha20 blocks of one round: K (K - 1) N / 16 co-resident, (K - 1) N / 16 on each rank of one replica per rank."""
    segs = -(-N // 16)
    return (K - 1) * segs * (1 if per_rank else K)


def payload_bytes(N: int, K: int) -> float:
    """HBM bytes of the payloads in one co-resident round: 4 N bytes per worker, written once and read once."""
    return 8.0 * N * K


def _arms(coll, xs, z, m, v, K):
    """One launch per arm; the SecAgg arms share a throwaway nonce counter and a fixed key table."""
    from federated_pytorch_test_b200.algo import secagg
    from federated_pytorch_test_b200.parallel.collective import SecAggRound

    keys = torch.from_numpy(secagg.pair_keys(0, K).view("int32")).to(z.device)
    sa = SecAggRound(1.0, secagg.frac_bits(1.0, K), keys, torch.zeros(1, dtype=torch.int64, device=z.device),
                     [coll.payload32_like_block(x) for x in xs])
    out = {"fedavg": lambda: coll._launch(0, xs, None, z, 0.0),
           "secagg": lambda: coll._launch(0, xs, None, z, 0.0, secagg=sa)}
    if m is not None:
        out["secagg_fedadam"] = lambda: coll._launch_fedopt(xs, z, m, v, "adam", 1e-2, 0.9, 0.99, 1e-3, secagg=sa)
    return out


def _time(launch, restore, rounds):
    times = {a: [] for a in launch}
    for rnd in range(rounds + 2):
        for a, f in launch.items():
            restore()
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
            ev[0].record()
            f()
            ev[1].record()
            ev[1].synchronize()
            if rnd >= 2:                                       # two untimed rounds per arm first
                times[a].append(ev[0].elapsed_time(ev[1]) * 1e3)
    return {a: statistics.median(v) for a, v in times.items()}


def aggregation(args, dev) -> dict:
    from federated_pytorch_test_b200.parallel import Topology
    from federated_pytorch_test_b200.parallel.fused import FusedCollective

    coll = FusedCollective(Topology.single_process(K_AGG, dev))
    coll.warm_fedopt = True
    coll.warm_secagg = True
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

        def restore():
            z.copy_(z0)
            for x, s in zip(xs, saved):
                x.copy_(s)
        us = _time(_arms(coll, xs, z, m, v, K_AGG), restore, args.rounds)
        coll.read_record()
        nb = chacha_blocks(N, K_AGG)
        row = {"N": N, "chacha_blocks": nb, "payload_hbm_bytes": payload_bytes(N, K_AGG)}
        for a in ARMS:
            row[a] = {"us": us[a]}
            if a != "fedavg":
                row[a]["Gblocks_per_s"] = nb / (us[a] * 1e-6) / 1e9
                row[a]["Tinsn_per_s_model"] = nb * CHACHA_INSNS / (us[a] * 1e-6) / 1e12
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
    coll.warm_secagg = True
    coll.warmup()
    res = []
    for N in sizes:
        stride = -(-N // 32) * 32
        x = coll.heap.alloc(stride)[:N]
        z = coll.zeros_like_block(x, "z")
        g = torch.Generator(device=dev).manual_seed(N + rank)
        z0 = torch.randn(N, device=dev, generator=torch.Generator(device=dev).manual_seed(N))
        saved = z0 + 1e-2 * torch.randn(N, device=dev, generator=g)
        launch = _arms(coll, [x], z, None, None, world)

        def restore():
            z.copy_(z0)
            x.copy_(saved)
            topo.barrier()
        row = {"N": N, "chacha_blocks_per_rank": chacha_blocks(N, world, per_rank=True)}
        for mode in ("0", "1"):
            coll.two_shot_mode = mode
            us = _time(launch, restore, rounds)
            coll.read_record()
            row["two_shot" if mode == "1" else "one_shot"] = {a: {"us": t, "two_shot": coll.last_two_shot}
                                                              for a, t in us.items()}
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
        raise SystemExit("bench_secagg.py measures the GPU path: no CUDA device")
    dev = torch.device("cuda", torch.cuda.current_device())
    res = {"device": torch.cuda.get_device_name(dev), "power_limit,max_sm_clock": _power_limit()}
    res["aggregation"] = aggregation(args, dev)
    res["multi_gpu"] = {"measured": False} if args.skip_multi else multi_gpu(args, dev)
    print("device: %s  (power.limit, clocks.max.sm: %s)" % (res["device"], res["power_limit,max_sm_clock"]))
    for row in res["aggregation"]["blocks"]:
        print("  (a) K=%d N=%8d  %10d ChaCha20 blocks, %6.1f MB payload HBM  " % (
            K_AGG, row["N"], row["chacha_blocks"], row["payload_hbm_bytes"] / 1e6) + "  ".join(
            "%s %7.1f us" % (a, row[a]["us"]) for a in ARMS)
            + "  (%.2f G blocks/s)" % row["secagg"]["Gblocks_per_s"])
    mg = res["multi_gpu"]
    if not mg["measured"]:
        print("  (b) several GPUs: not measured (%d visible)" % torch.cuda.device_count())
    else:
        for row in mg["blocks"]:
            for mode in ("one_shot", "two_shot"):
                print("  (b) W=%d N=%8d %s  " % (mg["world"], row["N"], mode) + "  ".join(
                    "%s %7.1f us" % (a, r["us"]) for a, r in row[mode].items()))
    print(json.dumps(res))
    return res


if __name__ == "__main__":
    main()
