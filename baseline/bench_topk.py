"""Cost of top-k sparsified client updates in federated averaging (``--compress_topk r [--compress_ef]``): a top-k round is
two launches, the cooperative selection kernel on the local replicas and the top-k instantiation of the fused
aggregation kernel.

  (a) one GPU: device time of one round at each of the ten ResNet18 block sizes, K = 8 co-resident replicas (the one-shot
      path), for six arms: plain FedAvg; top-k at r = 0.01 and 0.1, each without and with error feedback; r = 0.01 +
      FedAdam.  The selection and the aggregation are timed separately with CUDA events around each launch; every round
      starts by restoring perturbed replicas (untimed) and queues behind a ~1 ms device sleep, so the events time the
      device and not the host's launch overhead; the arms alternate round by round, and each time is the median over
      ``--rounds`` rounds.  Byte models (HBM traffic, K replicas of N floats, k = ceil(r N), payload
      P = 6 k + 4 (ceil(N / 8192) + 1)):
        FedAvg 4 N (2 K + 3) (K replicas read, z read / written / read again, K replicas written);
        selection K (4 N (8 + ef) + 6 k + 4 k ef): per replica x, z (and e) read and u written once, u read by the three
        further radix passes, the tile count and the entry pass, the entries (and e's zeros) written;
        aggregation 4 N (K + 3) + K P (+ 16 N for FedAdam's m and v): every payload read, z as for FedAvg, K replicas
        written.
  (b) the peer bytes a rank pulls per round with one replica per rank (one-shot: (W - 1) P; two-shot: about a 1/W slice
      of that), from the payload formula, next to FedAvg's (W - 1) 4 N;
  (c) several GPUs: the same rounds one process per GPU, one-shot and two-shot.  With one visible GPU this prints
      "not measured".

Prints the device name, power limit and max SM clock beside the numbers, then one JSON line.  Writes nothing to disk.

    python baseline/bench_topk.py [--rounds 30]
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
ARMS = ("fedavg", "k01", "k01_ef", "k10", "k10_ef", "k01_fedadam")
ARM_K = {"k01": (0.01, False), "k01_ef": (0.01, True), "k10": (0.1, False), "k10_ef": (0.1, True),
         "k01_fedadam": (0.01, False)}


def _payload(N: int, r: float) -> int:
    from federated_pytorch_test_b200.algo.compress import topk_count, topk_payload_bytes

    return topk_payload_bytes(N, topk_count(N, r))


def hbm_bytes(arm: str, N: int, K: int = K_AGG):
    """(selection, aggregation) bytes of one round."""
    from federated_pytorch_test_b200.algo.compress import topk_count

    if arm == "fedavg":
        return 0.0, 4.0 * N * (2 * K + 3)
    r, ef = ARM_K[arm]
    k = topk_count(N, r)
    sel = K * (4.0 * N * (8 + ef) + 6.0 * k + 4.0 * k * ef)
    agg = 4.0 * N * (K + 3) + K * _payload(N, r) + (16.0 * N if arm == "k01_fedadam" else 0.0)
    return sel, agg


def peer_bytes(arm: str, N: int, W: int, two_shot: bool) -> float:
    per = 4.0 * N if arm == "fedavg" else float(_payload(N, ARM_K[arm][0]))
    return (W - 1) * per / (W if two_shot else 1)


def _arms(coll, xs, z, m, v, ev):
    """One round per arm; ev[0..2] are recorded around the selection and the aggregation launch."""
    from federated_pytorch_test_b200.algo.compress import topk_count
    from federated_pytorch_test_b200.parallel.collective import TopKRound

    orig = coll._select_topk

    def timed_select(*a):
        ev[0].record()
        orig(*a)
        ev[1].record()
    coll._select_topk = timed_select

    def fedavg():
        ev[0].record()
        ev[1].record()
        coll._launch(0, xs, None, z, 0.0)

    out = {"fedavg": fedavg}
    N = z.numel()
    for a in ARMS[1:]:
        r, ef = ARM_K[a]
        k = topk_count(N, r)
        tk = TopKRound(k, [coll.sparse_payload_like_block(x, k) for x in xs], [torch.zeros_like(x) for x in xs] if ef else None)
        if a == "k01_fedadam":
            out[a] = (lambda tk=tk: coll._launch_fedopt(xs, z, m, v, "adam", 1e-2, 0.9, 0.99, 1e-3, topk=tk))
        else:
            out[a] = (lambda tk=tk: coll._launch(0, xs, None, z, 0.0, topk=tk))
    return out


def _time(launch, arms, restore, rounds, ev, sync=None):
    times = {a: ([], []) for a in arms}
    for rnd in range(rounds + 2):
        for a in arms:
            restore()
            if sync is not None:
                sync()
            torch.cuda._sleep(2_000_000)                  # the host queues the round while the GPU waits: device time only
            launch[a]()
            ev[2].record()
            ev[2].synchronize()
            if rnd >= 2:                                   # two untimed rounds per arm first
                times[a][0].append(ev[0].elapsed_time(ev[1]) * 1e3)
                times[a][1].append(ev[1].elapsed_time(ev[2]) * 1e3)
    return {a: (statistics.median(s), statistics.median(g)) for a, (s, g) in times.items()}


def aggregation(args, dev) -> dict:
    from federated_pytorch_test_b200.parallel import Topology
    from federated_pytorch_test_b200.parallel.fused import FusedCollective

    coll = FusedCollective(Topology.single_process(K_AGG, dev))
    coll.warm_fedopt = True
    coll.warm_topk = True
    coll.warmup()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
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
        med = _time(_arms(coll, xs, z, m, v, ev), ARMS, restore, args.rounds, ev)
        coll.read_record()
        row = {"N": N}
        for a in ARMS:
            (s_us, g_us), (s_b, g_b) = med[a], hbm_bytes(a, N)
            row[a] = {"select_us": s_us, "aggregate_us": g_us, "select_bytes": s_b, "aggregate_bytes": g_b,
                      "select_GBs": s_b / (s_us * 1e-6) / 1e9 if s_b else 0.0,
                      "aggregate_GBs": g_b / (g_us * 1e-6) / 1e9}
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
    coll.warm_topk = True
    coll.warmup()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    res = []
    for N in sizes:
        stride = -(-N // 32) * 32
        x = coll.heap.alloc(stride)[:N]
        z = coll.zeros_like_block(x, "z")
        g = torch.Generator(device=dev).manual_seed(N + rank)
        z0 = torch.randn(N, device=dev, generator=torch.Generator(device=dev).manual_seed(N))
        saved = z0 + 1e-2 * torch.randn(N, device=dev, generator=g)
        launch = {a: f for a, f in _arms(coll, [x], z, None, None, ev).items() if a != "k01_fedadam"}

        def restore():
            z.copy_(z0)
            x.copy_(saved)
        row = {"N": N}
        for mode in ("0", "1"):
            coll.two_shot_mode = mode
            med = _time(launch, list(launch), restore, rounds, ev, sync=topo.barrier)
            coll.read_record()
            two = coll.last_two_shot
            row["two_shot" if mode == "1" else "one_shot"] = {
                a: {"select_us": s, "aggregate_us": ag, "peer_bytes": peer_bytes(a, N, world, two), "two_shot": two}
                for a, (s, ag) in med.items()}
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
    ap.add_argument("--skip-multi", action="store_true", help="run (a) and (b) only")
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_topk.py measures the GPU path: no CUDA device")
    dev = torch.device("cuda", torch.cuda.current_device())
    res = {"device": torch.cuda.get_device_name(dev), "power_limit,max_sm_clock": _power_limit()}
    res["aggregation"] = aggregation(args, dev)
    sizes = [row["N"] for row in res["aggregation"]["blocks"]]
    res["peer_bytes"] = {str(W): {str(N): {a: {"one_shot": peer_bytes(a, N, W, False), "two_shot": peer_bytes(a, N, W, True)}
                                            for a in ("fedavg", "k01", "k10")} for N in sizes} for W in (2, 4, 8)}
    res["multi_gpu"] = {"measured": False} if args.skip_multi else multi_gpu(args, dev)
    print("device: %s  (power.limit, clocks.max.sm: %s)" % (res["device"], res["power_limit,max_sm_clock"]))
    for row in res["aggregation"]["blocks"]:
        print("  (a) N=%8d  " % row["N"] + "  ".join(
            "%s %6.1f + %6.1f us (%4.0f / %4.0f GB/s)" % (a, row[a]["select_us"], row[a]["aggregate_us"],
                                                         row[a]["select_GBs"], row[a]["aggregate_GBs"]) for a in ARMS))
    for N in sizes:
        pb = res["peer_bytes"]["8"][str(N)]
        print("  (b) W=8 N=%8d  " % N + "  ".join("%s %.3f / %.3f MB" % (a, pb[a]["one_shot"] / 1e6, pb[a]["two_shot"] / 1e6)
                                              for a in pb))
    mg = res["multi_gpu"]
    if not mg["measured"]:
        print("  (c) several GPUs: not measured (%d visible)" % torch.cuda.device_count())
    else:
        for row in mg["blocks"]:
            for mode in ("one_shot", "two_shot"):
                print("  (c) W=%d N=%8d %s  " % (mg["world"], row["N"], mode) + "  ".join(
                    "%s %6.1f + %6.1f us (%.3f MB from peers)" % (a, r["select_us"], r["aggregate_us"], r["peer_bytes"] / 1e6)
                    for a, r in row[mode].items()))
    print(json.dumps(res))
    return res


if __name__ == "__main__":
    main()
