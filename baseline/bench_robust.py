"""Cost of the Byzantine-robust aggregation rules of federated averaging (``--aggregator median|trimmed_mean``), which run
as their own instantiations of the fused aggregation kernel.

Two measurements, each alternating its arms in one process:

  (a) aggregation: device time of one aggregation at each of the ten ResNet18 block sizes, K = 8 co-resident replicas on
      one GPU (the one-shot path), for the mean, the median and the trimmed mean with trim_b = 1 (trim_fraction 0.125).
      CUDA events around ``--launches`` consecutive aggregations, median over ``--reps`` windows.  Achieved local
      bandwidth against the byte model of the kernel, the same for every rule: the K replicas are read (4 K N bytes),
      z is read and written in pass 1 and read again in pass 2 (12 N), and the new model is written into the K local
      replicas (4 K N): 4 N (2 K + 3) bytes;
  (b) training: ``federated_multi`` ResNet18, K = 4 co-resident replicas on one GPU, batch 128, CUDA-graphed steps, 49
      minibatches per replica and round, with the mean and the median.  Images/s over ``--steps`` replica steps after
      ``--warmup`` steps (CUDA events recorded from the engine's step hook; the window spans several aggregations),
      median over ``--reps`` runs.

The script runs in one process on one GPU, so it cannot measure the two-shot path (one replica per GPU on several GPUs).
Prints the device name, power limit and max SM clock beside the numbers, then one JSON line.  Writes nothing to disk.

    python baseline/bench_robust.py [--reps 5] [--launches 50] [--steps 600] [--warmup 40]
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
TRIM_B = 1                      # trim_fraction 0.125 at K = 8
K_TRAIN = 4
ROUND_STEPS = 49
ARMS = ("mean", "median", "trimmed_mean")


def agg_bytes(N: int, K: int = K_AGG) -> int:
    """Bytes one one-shot aggregation of K co-resident replicas must move (see the module docstring)."""
    return 4 * N * (2 * K + 3)


def aggregation(args, dev) -> dict:
    from federated_pytorch_test_b200.parallel import Topology
    from federated_pytorch_test_b200.parallel.fused import FusedCollective

    coll = FusedCollective(Topology.single_process(K_AGG, dev))
    coll.warm_robust = True
    coll.warmup()
    res = []
    for N in resnet18_block_sizes(dev):
        stride = -(-N // 32) * 32
        arena = coll.heap.alloc(K_AGG * stride)
        xs = [arena[k * stride: k * stride + N] for k in range(K_AGG)]
        for x in xs:
            x.normal_()
        z = coll.zeros_like_block(xs[0], "z")
        fns = {"mean": lambda: coll._launch(0, xs, None, z, 0.0),
               "median": lambda: coll._launch(0, xs, None, z, 0.0, agg="median"),
               "trimmed_mean": lambda: coll._launch(0, xs, None, z, 0.0, agg="trimmed_mean", trim_b=TRIM_B)}
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
        for a in ARMS:
            us = statistics.median(times[a])
            row[a] = {"us": us, "GBs": agg_bytes(N) / (us * 1e-6) / 1e9, "min_max_us": [min(times[a]), max(times[a])]}
        res.append(row)
        del arena, xs
    return {"K": K_AGG, "trim_b": TRIM_B, "launches_per_window": args.launches, "windows": args.reps, "blocks": res}


def training(args, dev) -> dict:
    from federated_pytorch_test_b200.algo.engine import Engine
    from federated_pytorch_test_b200.api import federated_multi

    def one_run(aggregator: str) -> float:
        ev = [torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)]
        first, last = args.warmup, args.warmup + args.steps

        def hook(e: Engine):
            if e.steps_done == first:
                ev[0].record()
            elif e.steps_done == last:
                ev[1].record()
                e.stop_requested = True

        orig_init = Engine.__init__

        def patched(self, *a, **k):
            orig_init(self, *a, **k)
            self.step_hook = hook
        Engine.__init__ = patched
        try:
            cfg = federated_multi.Config(K=K_TRAIN, use_resnet=True, Nloop=1, Nadmm=3, Nepoch=1, default_batch=128,
                                         max_minibatches=ROUND_STEPS, check_results=False, save_model=False,
                                         train_size=K_TRAIN * (128 * ROUND_STEPS + 1), test_size=128, graphs=True,
                                         fast=True, distributed=False, aggregator=aggregator)
            eng = federated_multi.run(cfg, log=lambda s: None)
        finally:
            Engine.__init__ = orig_init
        ev[1].synchronize()
        assert eng.steps_done == last and eng.graph_replays > 0
        return 128 * args.steps / (ev[0].elapsed_time(ev[1]) / 1e3)

    rates = {"mean": [], "median": []}
    one_run("median")                                   # warm-up: module load, first graph capture
    for _ in range(args.reps):
        for arm in rates:
            rates[arm].append(one_run(arm))
    return {"K": K_TRAIN, "steps": args.steps, "warmup_steps": args.warmup, "steps_per_round": K_TRAIN * ROUND_STEPS,
            "runs_per_arm": args.reps, "images_per_s": {k: statistics.median(v) for k, v in rates.items()},
            "images_per_s_all": rates}


def main(argv=None) -> dict:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--launches", type=int, default=50, help="aggregations per timed window in (a)")
    ap.add_argument("--steps", type=int, default=600, help="timed replica steps per run in (b)")
    ap.add_argument("--warmup", type=int, default=40, help="untimed replica steps before the window in (b)")
    ap.add_argument("--skip-training", action="store_true", help="run (a) only")
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_robust.py measures the GPU path: no CUDA device")
    if args.warmup + args.steps > 10 * 3 * K_TRAIN * ROUND_STEPS:
        raise SystemExit("--warmup + --steps must fit into one pass over the ten blocks (%d steps)"
                         % (30 * K_TRAIN * ROUND_STEPS))
    dev = torch.device("cuda", torch.cuda.current_device())
    res = {"device": torch.cuda.get_device_name(dev), "power_limit,max_sm_clock": _power_limit()}
    res["aggregation"] = aggregation(args, dev)
    if not args.skip_training:
        res["training"] = training(args, dev)
    print("device: %s  (power.limit, clocks.max.sm: %s)" % (res["device"], res["power_limit,max_sm_clock"]))
    for row in res["aggregation"]["blocks"]:
        print("  (a) N=%8d  " % row["N"] + "  ".join("%s %7.2f us %6.0f GB/s" % (a, row[a]["us"], row[a]["GBs"])
                                                    for a in ARMS))
    print("  (a) two-shot path: not measured by this single-GPU script")
    t = res.get("training")
    if t is not None:
        for k, v in t["images_per_s"].items():
            print("  (b) ResNet18 K=%d co-resident, graphed, aggregator=%-6s %9.0f images/s  (runs: %s)"
                  % (K_TRAIN, k, v, ", ".join("%.0f" % r for r in t["images_per_s_all"][k])))
    print(json.dumps(res))
    return res


if __name__ == "__main__":
    main()
