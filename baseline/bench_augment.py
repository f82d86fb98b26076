"""Cost of the opt-in training augmentation (random 4-pixel-padded crop + horizontal flip, ``--augment``).

Two measurements, each alternating its arms in one process:

  (a) input stage: device time of one batch-128 training batch from the HBM-resident dataset (50 000 synthetic CIFAR10
      images), ``index_select`` + ``normalize_u8`` (two launches, no augmentation) against the fused
      ``augment_normalize_u8`` kernel (gather + crop + flip + normalise, one launch), in the ResNet (NHWC) and the
      Net (NCHW) layout.  CUDA events around ``--batches`` consecutive batches, median over ``--reps`` windows;
  (b) training: ``federated_multi`` ResNet18, K = 1, batch 128, CUDA-graphed step, dataset in HBM, with ``augment``
      off and on.  Images/s over ``--steps`` steps after ``--warmup`` steps of the first block visit (CUDA events
      recorded from the engine's step hook), median over ``--reps`` runs per arm.

Prints the device name and power limit beside the numbers, then one JSON line.  Writes nothing to disk.

    python baseline/bench_augment.py [--reps 5] [--batches 1000] [--steps 100] [--warmup 20]
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


def _power_limit() -> str:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30)
        return out.stdout.strip().splitlines()[torch.cuda.current_device()] if out.returncode == 0 else "unknown"
    except (OSError, subprocess.SubprocessError, IndexError):
        return "unknown"


def input_stage(args, dev) -> dict:
    from federated_pytorch_test_b200.data.cifar import augment_key, make_synthetic_cifar, worker_norm
    from federated_pytorch_test_b200.ops import cuda_ops

    imgs, _ = make_synthetic_cifar(True, seed=1234)
    imgs = imgs.to(dev)
    mean, std = worker_norm(0)
    key = augment_key(69, 0)
    g = torch.Generator().manual_seed(0)
    perm = torch.cat([torch.randperm(imgs.shape[0], generator=g) for _ in range(-(-args.batches * 128 // imgs.shape[0]))])
    idx = [t.to(dev) for t in perm[:args.batches * 128].split(128)]

    def plain(cl):
        for i in idx:
            cuda_ops.normalize_u8(imgs.index_select(0, i), mean, std, cl)

    def fused(cl):
        for b, i in enumerate(idx):
            cuda_ops.augment_normalize_u8(imgs, i, key, 128 * b, mean, std, cl)

    arms = {"nhwc_index_select+normalize": lambda: plain(True), "nhwc_fused_augment": lambda: fused(True),
            "nchw_index_select+normalize": lambda: plain(False), "nchw_fused_augment": lambda: fused(False)}
    for fn in arms.values():
        fn()
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for _ in range(args.reps):
        for name, fn in arms.items():
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            fn()
            t1.record()
            t1.synchronize()
            times[name].append(t0.elapsed_time(t1) * 1e3 / len(idx))     # us per batch
    launches = {}
    for name, fn in (("nhwc_index_select+normalize", lambda: cuda_ops.normalize_u8(imgs.index_select(0, idx[0]), mean, std, True)),
                     ("nhwc_fused_augment", lambda: cuda_ops.augment_normalize_u8(imgs, idx[0], key, 0, mean, std, True))):
        before = cuda_ops.launch_count()
        fn()
        launches[name] = cuda_ops.launch_count() - before
    return {"batches_per_window": len(idx),
            "us_per_batch": {k: statistics.median(v) for k, v in times.items()},
            "us_per_batch_min_max": {k: [min(v), max(v)] for k, v in times.items()},
            "handwritten_launches_per_batch": launches}


def training(args, dev) -> dict:
    from federated_pytorch_test_b200.algo.engine import Engine
    from federated_pytorch_test_b200.api import federated_multi

    def one_run(augment: bool) -> float:
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
            cfg = federated_multi.Config(K=1, use_resnet=True, Nloop=1, Nadmm=1, Nepoch=1, default_batch=128,
                                         max_minibatches=last + 1, check_results=False, save_model=False,
                                         train_size=128 * (last + 2) + 1, test_size=128, graphs=True, fast=True,
                                         distributed=False, augment=augment)
            eng = federated_multi.run(cfg, log=lambda s: None)
        finally:
            Engine.__init__ = orig_init
        ev[1].synchronize()
        assert eng.steps_done == last and eng.graph_replays > 0
        return 128 * args.steps / (ev[0].elapsed_time(ev[1]) / 1e3)

    rates = {"augment_off": [], "augment_on": []}
    one_run(False)                                      # warm-up: module load, first graph capture
    for _ in range(args.reps):
        rates["augment_off"].append(one_run(False))
        rates["augment_on"].append(one_run(True))
    return {"steps": args.steps, "warmup_steps": args.warmup, "runs_per_arm": args.reps,
            "images_per_s": {k: statistics.median(v) for k, v in rates.items()},
            "images_per_s_all": rates}


def main(argv=None) -> dict:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--batches", type=int, default=1000, help="batch-128 input stages per timed window in (a)")
    ap.add_argument("--steps", type=int, default=100, help="timed training steps per run in (b)")
    ap.add_argument("--warmup", type=int, default=20, help="untimed training steps before the window in (b)")
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_augment.py measures the GPU path: no CUDA device")
    dev = torch.device("cuda", torch.cuda.current_device())
    res = {"device": torch.cuda.get_device_name(dev), "power_limit,max_sm_clock": _power_limit()}
    res["input_stage"] = input_stage(args, dev)
    res["training"] = training(args, dev)
    print("device: %s  (power.limit, clocks.max.sm: %s)" % (res["device"], res["power_limit,max_sm_clock"]))
    a = res["input_stage"]
    for k, v in a["us_per_batch"].items():
        print("  (a) %-30s %7.2f us per batch-128 input stage (min %.2f, max %.2f)" % (k, v, *a["us_per_batch_min_max"][k]))
    print("  (a) hand-written launches per batch: %s" % a["handwritten_launches_per_batch"])
    t = res["training"]
    for k, v in t["images_per_s"].items():
        print("  (b) ResNet18 K=1 graphed, %-12s %9.0f images/s  (runs: %s)"
              % (k, v, ", ".join("%.0f" % r for r in t["images_per_s_all"][k])))
    print(json.dumps(res))
    return res


if __name__ == "__main__":
    main()
