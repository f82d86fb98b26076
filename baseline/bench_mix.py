"""Cost of label smoothing, mixup and CutMix (``--label_smoothing``, ``--mixup_alpha``, ``--cutmix_alpha``).

Three measurements, each alternating its arms in one process:

  (a) input stage: device time of one batch-128 training batch from the HBM-resident dataset (50 000 synthetic CIFAR10
      images, ResNet NHWC layout): the fused augment kernel (gather + crop + flip + normalise) against the fused mixing
      kernel with augmentation + mixup and augmentation + CutMix (the same plus the partner's pixels, one launch).  The
      host-side draws (``mix_draws``) are made before the window and timed on their own.  CUDA events around ``--batches``
      consecutive batches, median over ``--reps`` windows;
  (b) loss: the hard-label ``cross_entropy`` forward + backward kernels against the ``soft_ce`` ones (label smoothing 0.1,
      mixed targets) at B = 128, C = 10: 100 forward + backward pairs captured in one CUDA graph (so no host launch cost
      is timed), CUDA events around ``--batches`` / 100 replays, median over ``--reps`` windows;
  (c) training: ``federated_multi`` ResNet18, K = 1, batch 128, CUDA-graphed step, dataset in HBM, all with ``--augment``:
      off, label smoothing 0.1, mixup 0.2, CutMix 1.0.  Images/s over ``--steps`` steps after ``--warmup`` steps of the first
      block visit (CUDA events recorded from the engine's step hook), median over ``--reps`` runs per arm.

Prints the device name and power limit beside the numbers, then one JSON line.  Writes nothing to disk.

    python baseline/bench_mix.py [--reps 5] [--batches 1000] [--steps 100] [--warmup 20]
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

from baseline.bench_augment import _power_limit  # noqa: E402


def _timed(arms, reps, per_window):
    for fn in arms.values():
        fn()
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for _ in range(reps):
        for name, fn in arms.items():
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            fn()
            t1.record()
            t1.synchronize()
            times[name].append(t0.elapsed_time(t1) * 1e3 / per_window)     # us per call
    return {"us": {k: statistics.median(v) for k, v in times.items()},
            "us_min_max": {k: [min(v), max(v)] for k, v in times.items()}}


def input_stage(args, dev) -> dict:
    from federated_pytorch_test_b200.data.cifar import augment_key, make_synthetic_cifar, mix_draws, mix_key, worker_norm
    from federated_pytorch_test_b200.ops import cuda_ops

    imgs, _ = make_synthetic_cifar(True, seed=1234)
    imgs = imgs.to(dev)
    mean, std = worker_norm(0)
    akey, key = augment_key(69, 0), mix_key(69, 0)
    g = torch.Generator().manual_seed(0)
    perm = torch.cat([torch.randperm(imgs.shape[0], generator=g) for _ in range(-(-args.batches * 128 // imgs.shape[0]))])
    idx = [t.to(dev) for t in perm[:args.batches * 128].split(128)]

    def augment():
        for b, i in enumerate(idx):
            cuda_ops.augment_normalize_u8(imgs, i, akey, 128 * b, mean, std, True)

    draws, draw_us = {}, {}
    for name, alphas in (("mixup", (0.2, 0.0)), ("cutmix", (0.0, 1.0))):
        t0 = time.perf_counter()
        draws[name] = [mix_draws(key, 128 * b, 128, 32, 32, *alphas) for b in range(len(idx))]
        draw_us[name] = (time.perf_counter() - t0) * 1e6 / len(idx)

    def mixed(name):
        for b, (i, draw) in enumerate(zip(idx, draws[name])):
            cuda_ops.mix_normalize_u8(imgs, i, akey, 128 * b, mean, std, True, draw)

    arms = {"augment": augment, "augment+mixup": lambda: mixed("mixup"), "augment+cutmix": lambda: mixed("cutmix")}
    res = _timed(arms, args.reps, len(idx))
    res["host_draw_us_per_batch"] = draw_us
    before = cuda_ops.launch_count()
    cuda_ops.mix_normalize_u8(imgs, idx[0], akey, 0, mean, std, True, mix_draws(key, 0, 128, 32, 32, 0.0, 1.0))
    res["handwritten_launches_per_mixed_batch"] = cuda_ops.launch_count() - before
    return res


def loss(args, dev) -> dict:
    from federated_pytorch_test_b200.ops import cuda_ops

    g = torch.Generator(device=dev).manual_seed(0)
    z = torch.randn(128, 10, device=dev, generator=g)
    y = torch.randint(0, 10, (128,), device=dev, generator=g)
    lam = torch.full((1,), 0.7, device=dev)

    e = cuda_ops.ext()
    gout = torch.ones(1, device=dev)

    def graphed(step):
        step()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for _ in range(100):
                step()
        replays = max(1, args.batches // 100)

        def run():
            for _ in range(replays):
                g.replay()
        return run

    def hard_step():
        _, p = e.cross_entropy_fwd(z, y)
        e.cross_entropy_bwd(p, y, gout)

    def soft_step():
        _, p = e.soft_ce_fwd(z, y, lam, 0.1)
        e.soft_ce_bwd(p, y, lam, 0.1, gout)

    arms = {"ce_fwd+bwd": graphed(hard_step), "soft_ce_fwd+bwd": graphed(soft_step)}
    return _timed(arms, args.reps, 100 * max(1, args.batches // 100))


def training(args, dev) -> dict:
    from federated_pytorch_test_b200.algo.engine import Engine
    from federated_pytorch_test_b200.api import federated_multi

    def one_run(**kw) -> float:
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
                                         distributed=False, augment=True, **kw)
            eng = federated_multi.run(cfg, log=lambda s: None)
        finally:
            Engine.__init__ = orig_init
        ev[1].synchronize()
        assert eng.steps_done == last and eng.graph_replays > 0
        return 128 * args.steps / (ev[0].elapsed_time(ev[1]) / 1e3)

    arms = {"off": {}, "label_smoothing": dict(label_smoothing=0.1), "mixup": dict(mixup_alpha=0.2),
            "cutmix": dict(cutmix_alpha=1.0)}
    rates = {k: [] for k in arms}
    one_run()                                           # warm-up: module load, first graph capture
    for _ in range(args.reps):
        for name, kw in arms.items():
            rates[name].append(one_run(**kw))
    return {"steps": args.steps, "warmup_steps": args.warmup, "runs_per_arm": args.reps,
            "images_per_s": {k: statistics.median(v) for k, v in rates.items()},
            "images_per_s_all": rates}


def main(argv=None) -> dict:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--batches", type=int, default=1000, help="batch-128 input stages / loss fwd+bwd pairs per timed window")
    ap.add_argument("--steps", type=int, default=100, help="timed training steps per run in (c)")
    ap.add_argument("--warmup", type=int, default=20, help="untimed training steps before the window in (c)")
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_mix.py measures the GPU path: no CUDA device")
    dev = torch.device("cuda", torch.cuda.current_device())
    res = {"device": torch.cuda.get_device_name(dev), "power_limit,max_sm_clock": _power_limit()}
    res["input_stage"] = input_stage(args, dev)
    res["loss"] = loss(args, dev)
    res["training"] = training(args, dev)
    print("device: %s  (power.limit, clocks.max.sm: %s)" % (res["device"], res["power_limit,max_sm_clock"]))
    for part, what in (("input_stage", "per batch-128 input stage"), ("loss", "per B=128, C=10 fwd+bwd")):
        r = res[part]
        for k, v in r["us"].items():
            print("  (%s) %-18s %7.2f us %s (min %.2f, max %.2f)" % ("a" if part == "input_stage" else "b", k, v, what,
                                                                     *r["us_min_max"][k]))
    print("  (a) hand-written launches per mixed batch: %d;  host draw per batch: %s"
          % (res["input_stage"]["handwritten_launches_per_mixed_batch"],
             ", ".join("%s %.1f us" % kv for kv in res["input_stage"]["host_draw_us_per_batch"].items())))
    t = res["training"]
    for k, v in t["images_per_s"].items():
        print("  (c) ResNet18 K=1 graphed, augment + %-16s %9.0f images/s  (runs: %s)"
              % (k, v, ", ".join("%.0f" % r for r in t["images_per_s_all"][k])))
    print(json.dumps(res))
    return res


if __name__ == "__main__":
    main()
