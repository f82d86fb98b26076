"""The ResNet18 stem (conv 3 -> 64, 3 x 3, + training-mode BatchNorm + ELU, batch 128, 32 x 32) on the wgmma pixel-major
convolution it ran on before (3 channels padded to 4) against stem_conv_bn_kernel, alternated in one process:

  fwd_grad     the training forward: old = pad x and w + pixel-major conv (y + statistics) + bn_elu_fwd;
               new = stem STORE_Y + bn_elu_fwd (+ the 4-channel copy of x the weight gradient reads);
  fwd_nograd   the forward without a gradient (diagnostics forward, frozen stem): old = as fwd_grad;
               new = stem STATS_ONLY + stem APPLY, y never stored;
  wgrad        the stem's weight gradient (wgrad_wgmma_kernel on the 4-channel x and dy), this build only: run the script
               with ``--only wgrad`` at another commit to compare.

Each arm is timed with CUDA events around ``--iters`` back-to-back calls, ``--reps`` times, arms alternating; the median is
printed with the HBM bytes the arm must move (modelled from the shapes: every tensor read or written once), the achieved
GB/s and its share of 3.35 TB/s (H100 SXM data sheet), and the card, power limit and max SM clock.  Writes nothing.

    python baseline/bench_stem.py [--batch 128] [--iters 50] [--reps 9] [--only fwd_grad,fwd_nograd,wgrad]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

HBM_BPS = 3.35e12


def _power_limit() -> str:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30)
        return out.stdout.strip().splitlines()[torch.cuda.current_device()] if out.returncode == 0 else "unknown"
    except (OSError, subprocess.SubprocessError, IndexError):
        return "unknown"


def main(argv=None) -> dict:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--reps", type=int, default=9)
    ap.add_argument("--only", default="fwd_grad,fwd_nograd,wgrad")
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_stem.py measures the GPU path: no CUDA device")

    from federated_pytorch_test_b200.ops import cuda_ops

    e = cuda_ops.ext()
    dev = torch.device("cuda", torch.cuda.current_device())
    B, H = args.batch, 32
    g = torch.Generator(device=dev).manual_seed(0)
    xn = torch.randn(B, H, H, 3, device=dev, generator=g)
    wk = torch.randn(64, 3, 3, 3, device=dev, generator=g) * 0.2
    gamma = torch.rand(64, device=dev, generator=g) + 0.5
    beta = torch.rand(64, device=dev, generator=g) - 0.5
    rm, rv = torch.zeros(64, device=dev), torch.ones(64, device=dev)
    dy = torch.randn(B, H, H, 64, device=dev, generator=g)
    dw = torch.zeros(64, 3, 3, 3, device=dev)
    st_old = torch.zeros(129, device=dev)
    st_new = torch.zeros(129, device=dev)
    x4 = F.pad(xn, (0, 1))

    def old_fwd():
        x4_ = F.pad(xn, (0, 1))
        w4 = F.pad(wk, (0, 1))
        y = e.conv2d_nhwc(x4_, w4, st_old, 1, 1, 1)
        e.bn_elu_fwd(y, st_old, gamma, beta, None, rm, rv, 1e-5, 0.1, True, True)

    def new_fwd_grad():
        y = e.stem_conv_bn(xn, wk, st_new, cuda_ops.STEM_STORE_Y)[0]
        e.bn_elu_fwd(y, st_new, gamma, beta, None, rm, rv, 1e-5, 0.1, True, True)
        F.pad(xn, (0, 1))

    def new_fwd_nograd():
        e.stem_conv_bn(xn, wk, st_new, cuda_ops.STEM_STATS_ONLY)
        e.stem_conv_bn(xn, wk, st_new, cuda_ops.STEM_APPLY, gamma, beta, rm, rv, 1e-5, 0.1, True, True)

    def wgrad():
        e.conv_wgrad(x4, dy, dw, 1, 1, 1)

    MB = 1e6
    x3, xp, y = 4 * B * H * H * 3, 4 * B * H * H * 4, 4 * B * H * H * 64
    pad_bytes = x3 + xp
    arms = {
        "fwd_grad": {"old": (old_fwd, pad_bytes + xp + 2 * y + y),          # pad, conv (x4 -> y), bn_elu_fwd (y -> out)
                     "new": (new_fwd_grad, x3 + y + 2 * y + pad_bytes)},
        "fwd_nograd": {"old": (old_fwd, pad_bytes + xp + 2 * y + y),
                       "new": (new_fwd_nograd, x3 + x3 + y)},
        "wgrad": {"new": (wgrad, xp + y)},
    }
    arms = {k: v for k, v in arms.items() if k in args.only.split(",")}

    def timed(fn):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(args.iters):
            fn()
        b.record()
        b.synchronize()
        return a.elapsed_time(b) * 1e3 / args.iters

    for arm in arms.values():                   # warm-up: module load, cudaFuncSetAttribute, allocator
        for fn, _ in arm.values():
            for _ in range(5):
                fn()
    torch.cuda.synchronize()
    times = {k: {v: [] for v in arm} for k, arm in arms.items()}
    for _ in range(args.reps):
        for k, arm in arms.items():
            for v, (fn, _) in arm.items():
                times[k][v].append(timed(fn))

    res = {"device": torch.cuda.get_device_name(dev), "power_limit,max_sm_clock": _power_limit(), "batch": B,
           "iters": args.iters, "reps": args.reps, "arms": {}}
    print("device: %s  (power.limit, clocks.max.sm: %s)" % (res["device"], res["power_limit,max_sm_clock"]))
    for k, arm in arms.items():
        for v, (_, nbytes) in arm.items():
            us = statistics.median(times[k][v])
            gbs = nbytes / (us * 1e-6) / 1e9
            res["arms"]["%s/%s" % (k, v)] = {"us": us, "us_min_max": [min(times[k][v]), max(times[k][v])],
                                             "modelled_MB": nbytes / MB, "GB_s": gbs, "share_of_3.35TBs": gbs * 1e9 / HBM_BPS}
            print("  %-10s %-3s %8.1f us  (min %.1f, max %.1f)  %6.1f MB  %7.0f GB/s  %4.0f %% of 3.35 TB/s"
                  % (k, v, us, min(times[k][v]), max(times[k][v]), nbytes / MB, gbs, 100 * gbs * 1e9 / HBM_BPS))
    print(json.dumps(res))
    return res


if __name__ == "__main__":
    main()
