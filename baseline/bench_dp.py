"""Cost of client-level differential privacy in federated averaging (``--dp_clip c --dp_noise sigma``, DP-FedAvg): a DP
round is the clip kernel followed by a DP instantiation of the fused aggregation kernel.

Two measurements, each alternating its arms in one process:

  (a) aggregation: device time of one round at each of the ten ResNet18 block sizes, K = 8 co-resident replicas on one
      GPU (the one-shot path), for four arms: plain FedAvg; DP with nobody clipped (bound far above every update); DP
      with everybody clipped (bound far below); DP + FedAdam (nobody clipped).  The write-back of a round makes every
      replica equal to z, so each round starts by restoring perturbed replicas (untimed) and is timed on its own with CUDA
      events before the clip, between the two launches and after the aggregation; median over ``--rounds`` rounds.
      Byte models: the clip pass reads z and the K replicas (4 N (K + 1) bytes) and writes the clipped ones (4 N K times
      the clipped fraction; pass 2 also re-reads them and z); the aggregation moves 4 N (2 K + 3) bytes (K replicas read,
      z read / written / read again, K replicas written), plus m and v for FedAdam (read and written: 16 N).
      Event timing of single rounds includes a few microseconds of event overhead, which dominates the small blocks;
  (b) training: ``federated_multi`` ResNet18, K = 4 co-resident replicas on one GPU, batch 128, CUDA-graphed steps, 49
      minibatches per replica and round, without and with DP (``--dp_clip 1e-3 --dp_noise 1``).  Images/s over
      ``--steps`` replica steps after ``--warmup`` steps, median over ``--reps`` runs.

The script runs in one process on one GPU, so it cannot measure the two-shot path.  Prints the device name, power limit
and max SM clock beside the numbers, then one JSON line.  Writes nothing to disk.

    python baseline/bench_dp.py [--reps 3] [--rounds 30] [--steps 600] [--warmup 40]
"""
from __future__ import annotations

import argparse
import json
import math
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from baseline.bench_fedopt import _power_limit, resnet18_block_sizes  # noqa: E402

K_AGG = 8
K_TRAIN = 4
ROUND_STEPS = 49
ARMS = ("fedavg", "dp_none_clipped", "dp_all_clipped", "dp_fedadam")


def clip_bytes(N: int, frac: float, K: int = K_AGG) -> float:
    return 4.0 * N * (K + 1) + 4.0 * N * K * frac


def agg_bytes(N: int, fedadam: bool = False, K: int = K_AGG) -> float:
    return 4.0 * N * (2 * K + 3) + (16.0 * N if fedadam else 0.0)


def aggregation(args, dev) -> dict:
    from federated_pytorch_test_b200.algo.privacy import noise_key
    from federated_pytorch_test_b200.parallel import Topology
    from federated_pytorch_test_b200.parallel.collective import DPRound
    from federated_pytorch_test_b200.parallel.fused import FusedCollective

    coll = FusedCollective(Topology.single_process(K_AGG, dev))
    coll.warm_dp = coll.warm_fedopt = True
    coll.warmup()
    key = noise_key(0)
    res = []
    for N in resnet18_block_sizes(dev):
        stride = -(-N // 32) * 32
        arena = coll.heap.alloc(K_AGG * stride)
        xs = [arena[k * stride: k * stride + N] for k in range(K_AGG)]
        z = coll.zeros_like_block(xs[0], "z")
        m, v = coll.zeros_like_block(xs[0], "m"), coll.zeros_like_block(xs[0], "v").fill_(1e-6)
        g = torch.Generator(device=dev).manual_seed(N)
        z0 = torch.randn(N, device=dev, generator=g)
        saved = [z0 + 1e-2 * torch.randn(N, device=dev, generator=g) for _ in range(K_AGG)]   # ||x - z|| ~ 1e-2 sqrt(N)
        t = torch.zeros(1, dtype=torch.int64, device=dev)
        big, small = 1e3 * math.sqrt(N), 1e-6 * math.sqrt(N)

        def dp(bound):
            return DPRound(bound / K_AGG, key, t)

        def run(arm):
            if arm == "fedavg":
                return None, lambda: coll._launch(0, xs, None, z, 0.0)
            if arm == "dp_fedadam":
                return (lambda: coll.dp_clip_(xs, z, big),
                        lambda: coll._launch_fedopt(xs, z, m, v, "adam", 1e-2, 0.9, 0.99, 1e-3, dp=dp(big)))
            bound = big if arm == "dp_none_clipped" else small
            return lambda: coll.dp_clip_(xs, z, bound), lambda: coll._launch(0, xs, None, z, 0.0, dp=dp(bound))

        times = {a: {"clip": [], "agg": []} for a in ARMS}
        clipped = {}
        for rnd in range(args.rounds + 2):
            for a in ARMS:
                clip, agg = run(a)
                z.copy_(z0)
                for x, s in zip(xs, saved):
                    x.copy_(s)
                ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
                ev[0].record()
                if clip is not None:
                    clip()
                ev[1].record()
                agg()
                ev[2].record()
                ev[2].synchronize()
                if a != "fedavg":
                    clipped[a] = coll.read_record()[8] / K_AGG
                if rnd >= 2:                                   # two untimed rounds per arm first
                    times[a]["clip"].append(ev[0].elapsed_time(ev[1]) * 1e3)
                    times[a]["agg"].append(ev[1].elapsed_time(ev[2]) * 1e3)
        coll.read_record()
        row = {"N": N}
        for a in ARMS:
            cu = statistics.median(times[a]["clip"]) if a != "fedavg" else 0.0
            au = statistics.median(times[a]["agg"])
            frac = clipped.get(a, 0.0)
            r = {"clip_us": cu, "agg_us": au, "round_us": cu + au, "agg_GBs": agg_bytes(N, a == "dp_fedadam") / (au * 1e-6) / 1e9}
            if a != "fedavg":
                r["clipped_fraction"] = frac
                r["clip_GBs"] = clip_bytes(N, frac) / (cu * 1e-6) / 1e9
            row[a] = r
        res.append(row)
        del arena, xs, saved
    return {"K": K_AGG, "rounds": args.rounds, "blocks": res}


def training(args, dev) -> dict:
    from federated_pytorch_test_b200.algo.engine import Engine
    from federated_pytorch_test_b200.api import federated_multi

    def one_run(dp_clip: float) -> float:
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
                                         fast=True, distributed=False, dp_clip=dp_clip, dp_noise=1.0)
            eng = federated_multi.run(cfg, log=lambda s: None)
        finally:
            Engine.__init__ = orig_init
        ev[1].synchronize()
        assert eng.steps_done == last and eng.graph_replays > 0
        return 128 * args.steps / (ev[0].elapsed_time(ev[1]) / 1e3)

    rates = {"fedavg": [], "dp": []}
    one_run(1e-3)                                       # warm-up: module load, first graph capture
    for _ in range(args.reps):
        rates["fedavg"].append(one_run(0.0))
        rates["dp"].append(one_run(1e-3))
    return {"K": K_TRAIN, "steps": args.steps, "warmup_steps": args.warmup, "runs_per_arm": args.reps,
            "images_per_s": {k: statistics.median(v) for k, v in rates.items()}, "images_per_s_all": rates}


def main(argv=None) -> dict:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=30, help="timed rounds per arm and block size in (a)")
    ap.add_argument("--steps", type=int, default=600, help="timed replica steps per run in (b)")
    ap.add_argument("--warmup", type=int, default=40, help="untimed replica steps before the window in (b)")
    ap.add_argument("--skip-training", action="store_true", help="run (a) only")
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_dp.py measures the GPU path: no CUDA device")
    dev = torch.device("cuda", torch.cuda.current_device())
    res = {"device": torch.cuda.get_device_name(dev), "power_limit,max_sm_clock": _power_limit()}
    res["aggregation"] = aggregation(args, dev)
    if not args.skip_training:
        res["training"] = training(args, dev)
    print("device: %s  (power.limit, clocks.max.sm: %s)" % (res["device"], res["power_limit,max_sm_clock"]))
    for row in res["aggregation"]["blocks"]:
        print("  (a) N=%8d  " % row["N"] + "  ".join(
            "%s %6.1f+%6.1f us" % (a, row[a]["clip_us"], row[a]["agg_us"]) for a in ARMS))
    print("  (a) two-shot path: not measured by this single-GPU script")
    t = res.get("training")
    if t is not None:
        for k, v in t["images_per_s"].items():
            print("  (b) ResNet18 K=%d co-resident, graphed, %-6s %9.0f images/s  (runs: %s)"
                  % (K_TRAIN, k, v, ", ".join("%.0f" % r for r in t["images_per_s_all"][k])))
    print(json.dumps(res))
    return res


if __name__ == "__main__":
    main()
