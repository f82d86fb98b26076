"""Cost of the server optimizers of federated averaging (``--server_opt``), fused into the aggregation kernel.

Two measurements, each alternating its arms in one process:

  (a) aggregation: device time of one aggregation at each of the ten ResNet18 block sizes, K = 8 co-resident replicas on
      one GPU (the one-shot path), for FedAvg, FedAvgM and FedAdam.  CUDA events around ``--launches`` consecutive
      aggregations, median over ``--reps`` windows.  Achieved local bandwidth against the byte model of the kernel:
      FedAvg reads the K replicas and z, writes z, reads z again and writes the K replicas, 4 N (2 K + 3) bytes; the
      server state adds 8 N bytes (m read + written) for avgm and 16 N (m and v) for the adaptive variants;
  (b) training: ``federated_multi`` ResNet18, K = 1, batch 128, CUDA-graphed step, 49 minibatches per round, with
      ``server_opt`` none and adam.  Images/s over ``--steps`` steps after ``--warmup`` steps (CUDA events recorded from
      the engine's step hook; the window spans several aggregations and block visits), median over ``--reps`` runs.

The script runs in one process on one GPU and has no multi-rank mode, so it cannot measure the two-shot path (blocks
>= 256 KB with one replica per GPU on several GPUs, where rank r also broadcasts its slice of m and v); running it under
torchrun does not change that.
Prints the device name, power limit and max SM clock beside the numbers, then one JSON line.  Writes nothing to disk.

    python baseline/bench_fedopt.py [--reps 5] [--launches 50] [--steps 300] [--warmup 20]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

K_AGG = 8
ROUND_STEPS = 49


def _power_limit() -> str:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30)
        return out.stdout.strip().splitlines()[torch.cuda.current_device()] if out.returncode == 0 else "unknown"
    except (OSError, subprocess.SubprocessError, IndexError):
        return "unknown"


def resnet18_block_sizes(dev) -> list:
    from federated_pytorch_test_b200.api import common, federated_multi
    from federated_pytorch_test_b200.parallel import Topology

    cfg = federated_multi.Config(K=1, use_resnet=True, train_size=128, test_size=128, save_model=False, distributed=False)
    task = common.ClassifierTask(cfg, Topology.single_process(1, dev))
    rep = task.build_replica(0, dev, None)
    return [rep.arenas[v.model].count(v.lo, v.hi) for v in task.visits(0)]


def aggregation(args, dev) -> dict:
    from federated_pytorch_test_b200.parallel import Topology
    from federated_pytorch_test_b200.parallel.fused import FusedCollective

    coll = FusedCollective(Topology.single_process(K_AGG, dev))
    coll.warm_fedopt = True
    coll.warmup()
    arms = ("fedavg", "avgm", "adam")
    extra = {"fedavg": 0, "avgm": 8, "adam": 16}
    res = []
    for N in resnet18_block_sizes(dev):
        stride = -(-N // 32) * 32
        arena = coll.heap.alloc(K_AGG * stride)
        xs = [arena[k * stride: k * stride + N] for k in range(K_AGG)]
        for x in xs:
            x.normal_()
        z, m, v = (coll.zeros_like_block(xs[0], t) for t in ("z", "srv_m", "srv_v"))
        v.fill_(1e-6)
        fns = {"fedavg": lambda: coll._launch(0, xs, None, z, 0.0),
               "avgm": lambda: coll._launch_fedopt(xs, z, m, v, "avgm", 1.0, 0.9, 0.99, 1e-3),
               "adam": lambda: coll._launch_fedopt(xs, z, m, v, "adam", 1e-2, 0.9, 0.99, 1e-3)}
        for f in fns.values():
            f()
        torch.cuda.synchronize()
        times = {a: [] for a in arms}
        for _ in range(args.reps):
            for a in arms:
                t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                t0.record()
                for _ in range(args.launches):
                    fns[a]()
                t1.record()
                t1.synchronize()
                times[a].append(t0.elapsed_time(t1) * 1e3 / args.launches)        # us per aggregation
        coll.read_record()
        row = {"N": N}
        for a in arms:
            us = statistics.median(times[a])
            nbytes = 4 * N * (2 * K_AGG + 3) + extra[a] * N
            row[a] = {"us": us, "GBs": nbytes / (us * 1e-6) / 1e9, "min_max_us": [min(times[a]), max(times[a])]}
        res.append(row)
        del arena, xs
    return {"K": K_AGG, "launches_per_window": args.launches, "windows": args.reps, "blocks": res}


def training(args, dev) -> dict:
    from federated_pytorch_test_b200.algo.engine import Engine
    from federated_pytorch_test_b200.api import federated_multi

    def one_run(server_opt: str) -> float:
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
            cfg = federated_multi.Config(K=1, use_resnet=True, Nloop=1, Nadmm=3, Nepoch=1, default_batch=128,
                                         max_minibatches=ROUND_STEPS, check_results=False, save_model=False,
                                         train_size=128 * ROUND_STEPS + 1, test_size=128, graphs=True, fast=True,
                                         distributed=False, server_opt=server_opt)
            eng = federated_multi.run(cfg, log=lambda s: None)
        finally:
            Engine.__init__ = orig_init
        ev[1].synchronize()
        assert eng.steps_done == last and eng.graph_replays > 0
        return 128 * args.steps / (ev[0].elapsed_time(ev[1]) / 1e3)

    rates = {"none": [], "adam": []}
    one_run("adam")                                     # warm-up: module load, first graph capture
    for _ in range(args.reps):
        for arm in rates:
            rates[arm].append(one_run(arm))
    return {"steps": args.steps, "warmup_steps": args.warmup, "steps_per_round": ROUND_STEPS, "runs_per_arm": args.reps,
            "images_per_s": {k: statistics.median(v) for k, v in rates.items()}, "images_per_s_all": rates}


def main(argv=None) -> dict:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--launches", type=int, default=50, help="aggregations per timed window in (a)")
    ap.add_argument("--steps", type=int, default=300, help="timed training steps per run in (b)")
    ap.add_argument("--warmup", type=int, default=20, help="untimed training steps before the window in (b)")
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_fedopt.py measures the GPU path: no CUDA device")
    if args.warmup + args.steps > 10 * 3 * ROUND_STEPS:
        raise SystemExit("--warmup + --steps must fit into one pass over the ten blocks (%d steps)" % (30 * ROUND_STEPS))
    dev = torch.device("cuda", torch.cuda.current_device())
    res = {"device": torch.cuda.get_device_name(dev), "power_limit,max_sm_clock": _power_limit()}
    res["aggregation"] = aggregation(args, dev)
    res["training"] = training(args, dev)
    print("device: %s  (power.limit, clocks.max.sm: %s)" % (res["device"], res["power_limit,max_sm_clock"]))
    for row in res["aggregation"]["blocks"]:
        print("  (a) N=%8d  " % row["N"] + "  ".join("%s %7.2f us %6.0f GB/s" % (a, row[a]["us"], row[a]["GBs"])
                                                    for a in ("fedavg", "avgm", "adam")))
    print("  (a) two-shot path: not measured by this single-GPU script")
    t = res["training"]
    for k, v in t["images_per_s"].items():
        print("  (b) ResNet18 K=1 graphed, server_opt=%-5s %9.0f images/s  (runs: %s)"
              % (k, v, ", ".join("%.0f" % r for r in t["images_per_s_all"][k])))
    print(json.dumps(res))
    return res


if __name__ == "__main__":
    main()
