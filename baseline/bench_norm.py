"""Cost of GroupNorm against BatchNorm in the ResNet18 training step.

BatchNorm gets its batch statistics from the convolution epilogue; GroupNorm needs per-sample statistics and runs its own
statistics pass (``csrc/norm_kernels.cu``).  This script measures what that costs, on one GPU:

1. A CUDA-graphed training step of ResNet18 at batch 128 (forward, backward with every parameter trainable, fused Adam) with
   BatchNorm, GroupNorm G = 32 and GroupNorm G = 2.  The variants alternate window by window; each window replays the graph
   ``--steps`` times between two CUDA events; the median over ``--windows`` windows is reported.
2. Every GroupNorm shape of that network at batch 128, alone on fixed inputs: forward (statistics + merge + apply) and
   backward (reduce + merge + apply), each captured in a CUDA graph (as the training step runs them, without host launch
   cost) and timed with CUDA events over ``--calls`` replays, with the bytes they must move (computed from the shapes) over
   that time against the H100 SXM's 3.35 TB/s.  A second, profiled pass gives each kernel's time and bytes/s.

Prints the device name and its power limit, a table, then one JSON line.  Writes nothing to disk.

    python baseline/bench_norm.py [--windows 9] [--steps 20] [--calls 200]
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

HBM_BYTES_PER_S = 3.35e12          # H100 SXM data sheet
B = 128
# (C, H) of the GroupNorm inputs of ResNet18 at batch 128, with how many layers of the network have that shape
NORM_SHAPES = [(64, 32, 5), (128, 16, 5), (256, 8, 5), (512, 4, 5)]
# kernel: how many [N, HW, C] fp32 tensors it streams (no residual; the backward recomputes ELU' from the input)
KERNELS = {"gn_stats_kernel": 1, "gn_finalize_kernel": 0, "gn_apply_kernel": 2, "gn_bwd_reduce_kernel": 2,
           "gn_bwd_merge_kernel": 0, "gn_bwd_apply_kernel": 3}


def _power_limit() -> str:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30)
        return out.stdout.strip().splitlines()[torch.cuda.current_device()] if out.returncode == 0 else "unknown"
    except (OSError, subprocess.SubprocessError, IndexError):
        return "unknown"


def _graphed_step(norm: str, groups: int, dev):
    """(graph, its loss tensor, the captured step) of one graphed training step of ResNet18 with the given normalisation.
    The step's closure holds the network, its arena, the optimizer and the batch: the graph reads and writes their memory,
    so they must outlive it (the next capture empties the allocator's cache)."""
    from federated_pytorch_test_b200 import models
    from federated_pytorch_test_b200.algo.graphs import capture_graph
    from federated_pytorch_test_b200.ops import cuda_ops
    from federated_pytorch_test_b200.optim.block_adam import BlockAdam
    from federated_pytorch_test_b200.utils import FlatArena, unfreeze_all_layers

    torch.manual_seed(0)
    net = models.ResNet18(norm=norm, groups=groups).to(dev)
    arena = FlatArena(net, channels_last_weights=True)
    unfreeze_all_layers(net)
    opt = BlockAdam(arena, 0, len(arena.params) - 1)
    g = torch.Generator(device=dev).manual_seed(1)
    x = torch.randn(B, 3, 32, 32, device=dev, generator=g).contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 10, (B,), device=dev, generator=g)

    def body():
        arena.zero_grads()
        with cuda_ops.accumulate_into_grad():
            loss = cuda_ops.cross_entropy(net(x), y)
            loss.backward()
        opt.apply_update()
        return loss.detach()

    for _ in range(3):
        body()
    graph, loss = capture_graph(torch.cuda.Stream(), body)
    return graph, loss, body


def _time(fn, n: int) -> float:
    """Seconds per call of ``fn`` over ``n`` calls, between two CUDA events."""
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(n):
        fn()
    t1.record()
    t1.synchronize()
    return t0.elapsed_time(t1) / 1e3 / n


def _norm_calls(C: int, H: int, G: int, dev):
    """(forward, backward, bytes forward, bytes backward) of one GroupNorm call without residual, ELU on (the layout of
    most of the network's groups; the backward recomputes ELU' from the input)."""
    from federated_pytorch_test_b200.ops import cuda_ops

    e = cuda_ops.ext()
    g = torch.Generator(device=dev).manual_seed(C + G)
    y = torch.randn(B, H, H, C, device=dev, generator=g)
    dout = torch.randn_like(y)
    gamma = 1 + 0.1 * torch.randn(C, device=dev, generator=g)
    beta = 0.1 * torch.randn(C, device=dev, generator=g)
    out, mean, rstd = e.gn_elu_fwd(y, gamma, beta, None, G, 1e-5, True)
    nbytes = y.numel() * 4
    fwd = lambda: e.gn_elu_fwd(y, gamma, beta, None, G, 1e-5, True)                                   # noqa: E731
    bwd = lambda: e.gn_elu_bwd(dout, None, y, mean, rstd, gamma, beta, G, False, True, True)          # noqa: E731
    # forward: y read by the statistics and by the apply pass, out written; backward: dout and y read twice, dy written
    return fwd, bwd, 3 * nbytes, 5 * nbytes, nbytes, (y, dout, gamma, beta, mean, rstd)


def main(argv=None) -> dict:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--windows", type=int, default=9)
    ap.add_argument("--steps", type=int, default=20, help="graph replays per timed window")
    ap.add_argument("--calls", type=int, default=200, help="graph replays per GroupNorm timing")
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_norm.py measures the GPU path: no CUDA device")
    from federated_pytorch_test_b200.ops import functional as FX

    FX.set_fast_path(True)
    dev = torch.device("cuda", torch.cuda.current_device())

    variants = {"batch": ("batch", 32), "group32": ("group", 32), "group2": ("group", 2)}
    steps = {k: _graphed_step(n, G, dev) for k, (n, G) in variants.items()}
    for graph, _, _ in steps.values():
        for _ in range(5):
            graph.replay()
    torch.cuda.synchronize()
    times = {k: [] for k in variants}
    for _ in range(args.windows):
        for k, (graph, _, _) in steps.items():
            times[k].append(_time(graph.replay, args.steps))
    step_ms = {k: 1e3 * statistics.median(v) for k, v in times.items()}
    losses = {k: float(loss) for k, (_, loss, _) in steps.items()}

    from federated_pytorch_test_b200.algo.graphs import capture_graph

    rows = []
    for C, H, layers in NORM_SHAPES:
        for G in (32, 2):
            fwd, bwd, bf, bb, nbytes, keep = _norm_calls(C, H, G, dev)
            for _ in range(5):
                fwd(), bwd()
            gf, _ = capture_graph(torch.cuda.Stream(), fwd)
            gb, _ = capture_graph(torch.cuda.Stream(), bwd)
            for _ in range(5):
                gf.replay(), gb.replay()
            tf = statistics.median(_time(gf.replay, args.calls) for _ in range(3))
            tb = statistics.median(_time(gb.replay, args.calls) for _ in range(3))
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(args.calls):
                    gf.replay(), gb.replay()
                torch.cuda.synchronize()
            kernel_us = {}
            for ev in prof.key_averages():
                for k in KERNELS:
                    if k in ev.key and ev.count:
                        kernel_us[k] = kernel_us.get(k, 0.0) + ev.device_time_total / ev.count
            kernel_TBps = {k: KERNELS[k] * nbytes / (us * 1e-6) / 1e12 for k, us in kernel_us.items() if KERNELS[k]}
            rows.append(dict(C=C, HW=H * H, G=G, layers=layers, fwd_us=1e6 * tf, bwd_us=1e6 * tb,
                             fwd_TBps=bf / tf / 1e12, bwd_TBps=bb / tb / 1e12,
                             fwd_of_peak=bf / tf / HBM_BYTES_PER_S, bwd_of_peak=bb / tb / HBM_BYTES_PER_S,
                             kernel_us={k: round(v, 2) for k, v in kernel_us.items()},
                             kernel_TBps={k: round(v, 2) for k, v in kernel_TBps.items()}))
            del gf, gb, keep

    res = {
        "device": torch.cuda.get_device_name(dev),
        "power_limit,max_sm_clock": _power_limit(),
        "batch": B, "windows": args.windows, "steps_per_window": args.steps,
        "step_ms": step_ms,
        "step_ms_min_max": {k: [1e3 * min(v), 1e3 * max(v)] for k, v in times.items()},
        "loss_after_warmup": losses,
        "groupnorm_calls": rows,
    }
    print("device: %s  (power.limit, clocks.max.sm: %s)" % (res["device"], res["power_limit,max_sm_clock"]))
    for k in variants:
        print("  ResNet18 graphed step, batch %d, %-8s %7.3f ms (median of %d windows)" % (B, k, step_ms[k], args.windows))
    print("  GroupNorm calls (no residual, ELU), batch %d:" % B)
    for r in rows:
        print("    C=%4d HW=%4d G=%2d  fwd %7.1f us %5.2f TB/s (%3.0f%%)  bwd %7.1f us %5.2f TB/s (%3.0f%%)"
              % (r["C"], r["HW"], r["G"], r["fwd_us"], r["fwd_TBps"], 100 * r["fwd_of_peak"], r["bwd_us"], r["bwd_TBps"],
                 100 * r["bwd_of_peak"]))
        print("      " + "  ".join("%s %.1f us%s" % (k.replace("_kernel", ""), v, " %.2f TB/s" % r["kernel_TBps"][k]
                                                     if k in r["kernel_TBps"] else "") for k, v in r["kernel_us"].items()))
    print(json.dumps(res))
    return res


if __name__ == "__main__":
    main()
