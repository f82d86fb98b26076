"""Per-kernel time of every ResNet18 convolution shape of the training step at batch 128 (CIFAR10, 32 x 32 input).

Four kinds of launch, each on the wgmma implicit-GEMM convolution (``conv2d_nhwc``):

  fwd       the forward convolution with the BatchNorm sum / sum-of-squares epilogue (3 x 3, stride 1 or 2; the stem has
            its 3 input channels padded to 4 for the 16-byte pixel pitch, and FLOPs count the 4 channels the kernel multiplies)
  dgrad     the stride-1 data gradient: dy [N, H, W, C_out] convolved with the rotated, transposed filter, plain store
  dgrad_s2  the stride-2 data gradient of layers 3 and 4: a 2 x 2 stride-1 convolution of dy with the phase-packed filter
            (4 C_in output columns), stored pixel-shuffled; FLOPs count what that convolution multiplies
  shortcut  the 1 x 1 stride-2 projection of the downsampling blocks, with the statistics epilogue

Each shape is timed with CUDA events around ``--iters`` back-to-back launches (default 200) after ``--warmup`` launches; the
median of ``--reps`` such windows is reported.  FLOPs are 2 * pixels * C_out * kh * kw * C_in from the shape; the share of
peak is against the 495 TFLOP/s dense TF32 figure of the H100 SXM data sheet (a card with a lower power limit or clock
cannot reach it).  ``--orient row,pixel`` times both tile orientations of the kernel per shape (alternated), where the
extension offers the choice; ``auto`` is what the convolution selects by itself.  ``pixel`` runs the window-reuse main loop
where the shape allows it (``conv_window_reuse``: one input box per filter column serves all three filter rows) and the
per-tap loop elsewhere; ``pixel_pertap`` always runs the per-tap loop, so ``--orient pixel,pixel_pertap`` compares the two.

The ``L2->SM MB`` column is the modelled operand traffic of one launch: TMA box bytes x boxes, computed from the shape and
the loop that runs (operand tiles x k-blocks x (activation box + weight boxes)); ``GB/s`` is that over the kernel time.
Prints a table, the device name, power limit and max SM clock, then one JSON line.  Writes nothing to disk.

    python baseline/bench_conv.py [--batch 128] [--orient auto|row|pixel|pixel_pertap|row,pixel] [--iters 200] [--reps 5]
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

PEAK_TF32 = 495e12
ORIENT = {"auto": -1, "row": 0, "pixel": 1, "pixel_pertap": 2}
ROW_M, PIX_M, ROW_BYTES = 128, 256, 128        # output pixels per tile (row-major / pixel-major); bytes per operand row (32 fp32)

# (name, kind, H_in, C_in, C_out, k, stride, pad, sites): the distinct shapes of ResNet18 on 32 x 32 inputs and how often
# one forward (fwd, shortcut) or one backward (dgrad) runs each
SHAPES = [
    ("stem 4->64 3x3 32", "fwd", 32, 4, 64, 3, 1, 1, 1),
    ("l1 64->64 3x3 32", "fwd", 32, 64, 64, 3, 1, 1, 4),
    ("l2 64->128 3x3 s2 ->16", "fwd", 32, 64, 128, 3, 2, 1, 1),
    ("l2 128->128 3x3 16", "fwd", 16, 128, 128, 3, 1, 1, 3),
    ("l3 128->256 3x3 s2 ->8", "fwd", 16, 128, 256, 3, 2, 1, 1),
    ("l3 256->256 3x3 8", "fwd", 8, 256, 256, 3, 1, 1, 3),
    ("l4 256->512 3x3 s2 ->4", "fwd", 8, 256, 512, 3, 2, 1, 1),
    ("l4 512->512 3x3 4", "fwd", 4, 512, 512, 3, 1, 1, 3),
    ("l2 sc 64->128 1x1 s2", "shortcut", 32, 64, 128, 1, 2, 0, 1),
    ("l3 sc 128->256 1x1 s2", "shortcut", 16, 128, 256, 1, 2, 0, 1),
    ("l4 sc 256->512 1x1 s2", "shortcut", 8, 256, 512, 1, 2, 0, 1),
    ("l1 dgrad 64<-64 3x3 32", "dgrad", 32, 64, 64, 3, 1, 1, 4),
    ("l2 dgrad 128<-128 3x3 16", "dgrad", 16, 128, 128, 3, 1, 1, 3),
    ("l3 dgrad 256<-256 3x3 8", "dgrad", 8, 256, 256, 3, 1, 1, 3),
    ("l4 dgrad 512<-512 3x3 4", "dgrad", 4, 512, 512, 3, 1, 1, 3),
    ("l3 dgrad 128<-256 3x3 s2", "dgrad_s2", 16, 128, 256, 3, 2, 1, 1),
    ("l4 dgrad 256<-512 3x3 s2", "dgrad_s2", 8, 256, 512, 3, 2, 1, 1),
]


def _card() -> dict:
    out = {"device": torch.cuda.get_device_name(), "power_limit": "unknown", "max_sm_clock": "unknown"}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        if r.returncode == 0:
            pl, clk = r.stdout.strip().splitlines()[torch.cuda.current_device()].split(",")
            out["power_limit"], out["max_sm_clock"] = pl.strip(), clk.strip()
    except (OSError, subprocess.SubprocessError, IndexError, ValueError):
        pass
    return out


def _k_blocks(cin, k):
    """k-blocks of the per-tap loops: one per (tap, 32-channel block), or 32 / cw taps per k-block when C_in <= 16 is packed."""
    if cin <= 16 and cin % 4 == 0:
        cw = 8 if cin <= 8 else 16
        return -(-k * k // (32 // cw))
    return k * k * -(-cin // 32)


def operand_bytes(e, orient, B, Ho, Wo, cin, cout, k, stride) -> tuple:
    """(loop that runs, modelled L2 -> shared-memory operand bytes of one launch): TMA box bytes x boxes."""
    M = B * Ho * Wo
    if orient < 0:
        orient = e.conv_orientation(B, Ho, Wo, cout, stride)
    if orient == 0:
        bn = 32 if cout <= 32 else (64 if cout <= 64 else 128)
        tiles = -(-M // ROW_M) * -(-cout // bn)
        return "row", tiles * _k_blocks(cin, k) * (ROW_M + bn) * ROW_BYTES
    tiles = -(-M // PIX_M)
    if orient == 1 and e.conv_window_reuse(Ho, Wo, cin, cout, k, stride, 1):
        rows = PIX_M // Wo                 # per (filter column, channel block): one (rows + k - 1)-row window + k weight boxes
        return "window", tiles * k * -(-cin // 32) * ((rows + k - 1) * Wo + k * cout) * ROW_BYTES
    return "pertap", tiles * _k_blocks(cin, k) * (PIX_M + cout) * ROW_BYTES


def _case(e, kind, B, H, Ci, Co, k, s, p, dev):
    """Inputs and a closure launching the convolution once; (closure, FLOPs of one launch, output channels, geometry)."""
    g = torch.Generator(device=dev).manual_seed(B + H + Ci + Co + k)
    Ho = (H + 2 * p - k) // s + 1
    if kind == "dgrad_s2":              # dy [B, Ho, Wo, Co] * phase-packed filter [4 Ci, 2, 2, Co] -> dx [B, H, W, Ci]
        from federated_pytorch_test_b200.ops import conv_math
        dy = torch.randn(B, Ho, Ho, Co, device=dev, generator=g)
        wp = conv_math.pack_dgrad_s2_weight(torch.randn(Co, k, k, Ci, device=dev, generator=g) / (k * k * Ci) ** 0.5)
        flops = 2.0 * B * Ho * Ho * 4 * Ci * 4 * Co
        return (lambda orient: e.conv2d_nhwc_shuffle(dy, wp, 0, Ho, Ho)), flops, 4 * Ci, (B, Ho, Ho, Co, 4 * Ci, 2, 1)
    if kind == "dgrad":                 # dy [B, H, W, Co] * rotated filter [Ci, k, k, Co] -> dx [B, H, W, Ci]
        x = torch.randn(B, Ho, Ho, Co, device=dev, generator=g)
        w = torch.randn(Ci, k, k, Co, device=dev, generator=g) / (k * k * Co) ** 0.5
        stats, cin, cout, pad = None, Co, Ci, k - 1 - p
    else:
        x = torch.randn(B, H, H, Ci, device=dev, generator=g)
        w = torch.randn(Co, k, k, Ci, device=dev, generator=g) / (k * k * Ci) ** 0.5
        stats, cin, cout, pad = torch.zeros(2 * Co, device=dev), Ci, Co, p
    flops = 2.0 * B * Ho * Ho * cout * k * k * cin
    stride = 1 if kind == "dgrad" else s
    geom = (B, Ho, Ho, cin, cout, k, stride)

    def run(orient):
        if orient < 0:
            return e.conv2d_nhwc(x, w, stats, stride, pad, 1)
        return e.conv2d_nhwc(x, w, stats, stride, pad, 1, orient)

    return run, flops, cout, geom


def _time(run, orient, iters) -> float:
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        run(orient)
    t1.record()
    t1.synchronize()
    return t0.elapsed_time(t1) / 1e3 / iters


def main(argv=None) -> dict:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--orient", default="auto", help="comma-separated list of auto, row, pixel")
    ap.add_argument("--iters", type=int, default=200, help="launches per timed window (>= 200)")
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_conv.py measures the GPU path: no CUDA device")
    orients = [o.strip() for o in args.orient.split(",") if o.strip()]
    if any(o not in ORIENT for o in orients):
        raise SystemExit("--orient takes auto, row, pixel, pixel_pertap")

    from federated_pytorch_test_b200.ops import cuda_ops

    e = cuda_ops.ext()
    dev = torch.device("cuda", torch.cuda.current_device())
    card = _card()
    rows = []
    with torch.no_grad():
        for name, kind, H, Ci, Co, k, s, p, sites in SHAPES:
            run, flops, cout, geom = _case(e, kind, args.batch, H, Ci, Co, k, s, p, dev)
            # pixel-major tiles: C_out 64 / 128 only; the shuffled stride-2 data gradient runs row-major tiles only
            avail = [o for o in orients if not o.startswith("pixel") or (cout in (64, 128) and kind != "dgrad_s2")]
            for o in avail:
                for _ in range(args.warmup):
                    run(ORIENT[o])
            torch.cuda.synchronize()
            times = {o: [] for o in avail}
            for _ in range(args.reps):
                for o in avail:
                    times[o].append(_time(run, ORIENT[o], args.iters))
            for o in avail:
                t = statistics.median(times[o])
                loop, nbytes = operand_bytes(e, ORIENT[o], *geom)
                rows.append({"shape": name, "kind": kind, "orient": o, "loop": loop, "sites": sites, "us": t * 1e6,
                             "l2_sm_bytes": nbytes, "l2_sm_GBs": nbytes / t / 1e9,
                             "us_min_max": [min(times[o]) * 1e6, max(times[o]) * 1e6], "gflop": flops / 1e9,
                             "tflops": flops / t / 1e12, "share_of_peak": flops / t / PEAK_TF32})
    print("device: %s  power limit: %s  max SM clock: %s" % (card["device"], card["power_limit"], card["max_sm_clock"]))
    print("%-26s %-8s %-12s %-6s %5s %9s %8s %7s %6s %10s %7s" % ("shape", "kind", "orient", "loop", "sites", "us", "GFLOP",
                                                                  "TFLOP/s", "peak", "L2->SM MB", "GB/s"))
    for r in rows:
        print("%-26s %-8s %-12s %-6s %5d %9.1f %8.2f %7.1f %5.1f%% %10.1f %7.0f" % (
            r["shape"], r["kind"], r["orient"], r["loop"], r["sites"], r["us"], r["gflop"], r["tflops"],
            100 * r["share_of_peak"], r["l2_sm_bytes"] / 1e6, r["l2_sm_GBs"]))
    for o in orients:
        tot = sum(r["us"] * r["sites"] for r in rows if r["orient"] == o)
        print("  %-12s step total over the sites above: %.1f us" % (o, tot))
    res = dict(card, batch=args.batch, iters=args.iters, reps=args.reps, rows=rows)
    print(json.dumps(res))
    return res


if __name__ == "__main__":
    main()
