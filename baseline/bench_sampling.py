"""Cost of client sampling with sample-count weights in federated averaging (``--clients_per_round``, ``--partition
dirichlet``), which runs as its own instantiation of the fused aggregation kernel.

Two measurements, each alternating its arms in one process:

  (a) aggregation: device time of one aggregation at each of the ten ResNet18 block sizes, K = 8 co-resident replicas on
      one GPU (the one-shot path), for plain FedAvg (the mean), the sampled weighted mean with S = 8 and equal sample
      counts, the sampled weighted mean with S = 4, and FedAdam from the sampled weighted mean with S = 4.  CUDA events
      around ``--launches`` consecutive aggregations, median over ``--reps`` windows.  Achieved local bandwidth against
      the byte model of the kernel: the S participants are read (4 S N bytes), z is read and written in pass 1 and read
      again in pass 2 (12 N), and the new model is written into the K local replicas (4 K N): 4 N (S + K + 3) bytes
      (FedAdam also reads and writes m and v: 16 N more);
  (b) training: ``federated_multi`` ResNet18, K = 8 co-resident replicas on one GPU, ``--partition dirichlet
      --dirichlet_alpha 0.5`` over 50 000 synthetic samples, batch 128, CUDA-graphed steps, at most 49 minibatches per
      replica and round, with S = 8 and S = 4 participants per round.  Images/s of the steps taken over ``--steps``
      replica steps after ``--warmup`` steps (CUDA events recorded from the engine's step hook), and wall time per round
      over the same window; median over ``--reps`` runs.

The script runs in one process on one GPU, so it cannot measure the two-shot path or the cost across GPUs (one replica per
GPU on several GPUs).  Prints the device name, power limit and max SM clock beside the numbers, then one JSON line.
Writes nothing to disk.

    python baseline/bench_sampling.py [--reps 5] [--launches 50] [--steps 600] [--warmup 40]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from baseline.bench_fedopt import _power_limit, resnet18_block_sizes  # noqa: E402

K = 8
ROUND_STEPS = 49
ARMS = ("mean", "sampled_S8", "sampled_S4", "fedadam_S4")
TRAIN_ARMS = (8, 4)


def agg_bytes(N: int, S: int, fedadam: bool = False) -> int:
    """Bytes one one-shot aggregation of K co-resident replicas with S participants must move (module docstring)."""
    return 4 * N * (S + K + 3) + (16 * N if fedadam else 0)


def aggregation(args, dev) -> dict:
    from federated_pytorch_test_b200.algo.sampling import sample_key
    from federated_pytorch_test_b200.parallel import Topology
    from federated_pytorch_test_b200.parallel.collective import SampleRound
    from federated_pytorch_test_b200.parallel.fused import FusedCollective

    coll = FusedCollective(Topology.single_process(K, dev))
    coll.warm_sample = coll.warm_fedopt = True
    coll.warmup()
    key = sample_key(69)
    n = torch.full((K,), 6250, dtype=torch.int32, device=dev)
    res = []
    for N in resnet18_block_sizes(dev):
        stride = -(-N // 32) * 32
        arena = coll.heap.alloc(K * stride)
        xs = [arena[k * stride: k * stride + N] for k in range(K)]
        for x in xs:
            x.normal_()
        z = coll.zeros_like_block(xs[0], "z")
        m, v = coll.zeros_like_block(xs[0], "m"), coll.zeros_like_block(xs[0], "v").fill_(1e-6)
        s8 = SampleRound(8, key, torch.zeros(1, dtype=torch.int64, device=dev), n)
        s4 = SampleRound(4, key, torch.zeros(1, dtype=torch.int64, device=dev), n)
        fns = {"mean": lambda: coll._launch(0, xs, None, z, 0.0),
               "sampled_S8": lambda: coll._launch(0, xs, None, z, 0.0, sample=s8),
               "sampled_S4": lambda: coll._launch(0, xs, None, z, 0.0, sample=s4),
               "fedadam_S4": lambda: coll._launch_fedopt(xs, z, m, v, "adam", 1e-2, 0.9, 0.99, 1e-3, sample=s4)}
        for f in fns.values():
            f()
        torch.cuda.synchronize()
        times = {a: [] for a in ARMS}
        for _ in range(args.reps):
            for a in ARMS:
                t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                t0.record()
                for _ in range(args.launches):
                    fns[a]()
                t1.record()
                t1.synchronize()
                times[a].append(t0.elapsed_time(t1) * 1e3 / args.launches)        # us per aggregation
        coll.read_record()
        row = {"N": N}
        for a, S in zip(ARMS, (K, 8, 4, 4)):
            us = statistics.median(times[a])
            row[a] = {"us": us, "GBs": agg_bytes(N, S, a == "fedadam_S4") / (us * 1e-6) / 1e9,
                      "min_max_us": [min(times[a]), max(times[a])]}
        res.append(row)
        del arena, xs
    return {"K": K, "launches_per_window": args.launches, "windows": args.reps, "blocks": res}


def training(args, dev) -> dict:
    from federated_pytorch_test_b200.algo.engine import Engine
    from federated_pytorch_test_b200.api import federated_multi

    def one_run(S: int):
        ev = [torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)]
        mark = {}
        first, last = args.warmup, args.warmup + args.steps

        def hook(e: Engine):
            if e.steps_done == first:
                ev[0].record()
                mark["a"] = (e.images_seen, e.aggregations_done, time.perf_counter())
            elif e.steps_done == last:
                ev[1].record()
                ev[1].synchronize()
                mark["b"] = (e.images_seen, e.aggregations_done, time.perf_counter())
                e.stop_requested = True

        orig_init = Engine.__init__

        def patched(self, *a, **k):
            orig_init(self, *a, **k)
            self.step_hook = hook
        Engine.__init__ = patched
        try:
            cfg = federated_multi.Config(K=K, use_resnet=True, Nloop=1, Nadmm=3, Nepoch=1, default_batch=128,
                                         max_minibatches=ROUND_STEPS, check_results=False, save_model=False,
                                         train_size=50000, test_size=128, graphs=True, fast=True, distributed=False,
                                         partition="dirichlet", dirichlet_alpha=0.5, clients_per_round=S)
            eng = federated_multi.run(cfg, log=lambda s: None)
        finally:
            Engine.__init__ = orig_init
        assert eng.steps_done == last and eng.graph_replays > 0 and eng.strategy.sampled
        (i0, a0, h0), (i1, a1, h1) = mark["a"], mark["b"]
        dt = ev[0].elapsed_time(ev[1]) / 1e3
        return (i1 - i0) / dt, 1e3 * (h1 - h0) / max(a1 - a0, 1), a1 - a0

    rates = {S: [] for S in TRAIN_ARMS}
    rounds = {S: [] for S in TRAIN_ARMS}
    one_run(4)                                          # warm-up: module load, first graph capture
    for _ in range(args.reps):
        for S in TRAIN_ARMS:
            ips, ms, na = one_run(S)
            rates[S].append(ips)
            rounds[S].append((ms, na))
    return {"K": K, "steps": args.steps, "warmup_steps": args.warmup, "runs_per_arm": args.reps,
            "images_per_s": {"S%d" % S: statistics.median(v) for S, v in rates.items()},
            "ms_per_round": {"S%d" % S: statistics.median([r[0] for r in v]) for S, v in rounds.items()},
            "images_per_s_all": {"S%d" % S: v for S, v in rates.items()},
            "rounds_in_window": {"S%d" % S: [r[1] for r in v] for S, v in rounds.items()}}


def main(argv=None) -> dict:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--launches", type=int, default=50, help="aggregations per timed window in (a)")
    ap.add_argument("--steps", type=int, default=600, help="timed replica steps per run in (b)")
    ap.add_argument("--warmup", type=int, default=40, help="untimed replica steps before the window in (b)")
    ap.add_argument("--skip-training", action="store_true", help="run (a) only")
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_sampling.py measures the GPU path: no CUDA device")
    dev = torch.device("cuda", torch.cuda.current_device())
    res = {"device": torch.cuda.get_device_name(dev), "power_limit,max_sm_clock": _power_limit()}
    res["aggregation"] = aggregation(args, dev)
    if not args.skip_training:
        res["training"] = training(args, dev)
    print("device: %s  (power.limit, clocks.max.sm: %s)" % (res["device"], res["power_limit,max_sm_clock"]))
    for row in res["aggregation"]["blocks"]:
        print("  (a) N=%8d  " % row["N"] + "  ".join("%s %7.2f us %6.0f GB/s" % (a, row[a]["us"], row[a]["GBs"])
                                                    for a in ARMS))
    print("  (a) two-shot path and multi-GPU cost: not measured by this single-GPU script")
    t = res.get("training")
    if t is not None:
        for k, v in t["images_per_s"].items():
            print("  (b) ResNet18 K=%d co-resident, Dirichlet(0.5), graphed, %s: %9.0f images/s of steps taken, %8.1f ms "
                  "per round  (runs: %s)" % (K, k, v, t["ms_per_round"][k],
                                            ", ".join("%.0f" % r for r in t["images_per_s_all"][k])))
    print(json.dumps(res))
    return res


if __name__ == "__main__":
    main()
