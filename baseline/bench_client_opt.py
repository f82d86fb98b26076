"""Cost of the client SGD update against the client Adam update, and of the client recipe (AdamW, gradient-norm clipping,
a device learning rate for the schedule), on one GPU.

1. The fused update kernels alone (``adam_prox`` and ``sgd_prox`` with momentum 0.9 and with momentum 0, each without and
   with the consensus vectors ``z`` / ``y``) at the ten ResNet18 block sizes.  Each variant is launched ``--calls`` times
   between two CUDA events, ``--windows`` windows, variants alternating window by window; the median window is reported
   in us per launch and in GB/s of the bytes the update must move per parameter (computed below from what the kernel
   reads and writes: Adam reads x, g, m, v and writes x, m, v = 28 B; SGD with momentum reads x, g, buf and writes x, buf =
   20 B; SGD without momentum reads x, g and writes x = 12 B; z and y add 4 B each).
   The recipe arms run the gradient-norm kernel and the update together, with the learning rate read from the device:
   ``adamw_clip`` (AdamW, weight decay 0.05, clip 1.0) against ``adam``, and ``sgd_m0.9_clip`` against ``sgd_m0.9``.
   Clipping adds one read of g (4 B per parameter), which the byte counts include, and a few KB of per-CTA partials.
2. A CUDA-graphed training step of ResNet18 at batch 128 with every parameter trainable (forward, backward, fused update):
   Adam against SGD (momentum 0.9, Nesterov, weight decay 5e-4) and against AdamW + clipping + a cosine schedule (the
   device learning rate rewritten before every window), alternating window by window, median of ``--windows`` windows
   of ``--steps`` replays.

Prints the device name, its power limit and max SM clock, a table, then one JSON line.  Writes nothing to disk.

    python baseline/bench_client_opt.py [--windows 9] [--calls 200] [--steps 20]
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
from baseline.bench_norm import _time  # noqa: E402

B = 128
# name: (bytes per parameter, momentum, consensus vectors z / y present)
KERNELS = {
    "adam": (28, None, False), "adam_zy": (36, None, True),
    "sgd_m0.9": (20, 0.9, False), "sgd_m0.9_zy": (28, 0.9, True),
    "sgd_m0": (12, 0.0, False), "sgd_m0_zy": (20, 0.0, True),
    "adamw_clip": (32, None, False), "sgd_m0.9_clip": (24, 0.9, False),
}
CLIP = 1.0


def _update_call(name: str, n: int, dev):
    """(call, tensors it keeps alive) of one update launch on a fresh block of ``n`` parameters."""
    from federated_pytorch_test_b200.ops import cuda_ops

    from federated_pytorch_test_b200.ops import flatops

    _, mom, zy = KERNELS[name]
    clip = name.endswith("_clip")
    g = torch.Generator(device=dev).manual_seed(n)
    x = torch.randn(n, device=dev, generator=g)
    gr = 1e-3 * torch.randn(n, device=dev, generator=g)
    z, y = (torch.randn(n, device=dev, generator=g), 1e-3 * torch.randn(n, device=dev, generator=g)) if zy else (None, None)
    rho = 0.1 if zy else 0.0
    if clip:       # the recipe: norm kernel + update, learning rate read from the device
        ws, ticket = flatops.clip_workspace(x)
        lr = torch.full((1,), 1e-3, device=dev)
        if mom is None:
            m, v, step = torch.zeros(n, device=dev), torch.zeros(n, device=dev), torch.ones(1, dtype=torch.int32, device=dev)

            def call():
                cuda_ops.grad_norm(gr, ws, ticket, CLIP)
                cuda_ops.adam_prox_step(x, gr, m, v, step, 0.0, 0.9, 0.999, 1e-8, lr_dev=lr, weight_decay=0.05,
                                        norm_dev=ws[0:1], clip_norm=CLIP)
            return call, (x, gr, m, v, step, ws, ticket, lr)
        buf = torch.zeros(n, device=dev)

        def call():
            cuda_ops.grad_norm(gr, ws, ticket, CLIP)
            cuda_ops.sgd_prox_step(x, gr, buf, 0.0, mom, False, 0.0, lr_dev=lr, norm_dev=ws[0:1], clip_norm=CLIP)
        return call, (x, gr, buf, ws, ticket, lr)
    if mom is None:
        m, v, step = torch.zeros(n, device=dev), torch.zeros(n, device=dev), torch.ones(1, dtype=torch.int32, device=dev)
        return (lambda: cuda_ops.adam_prox_step(x, gr, m, v, step, 1e-3, 0.9, 0.999, 1e-8, z, y, rho, 1e-4, 1e-4)), \
            (x, gr, z, y, m, v, step)
    buf = torch.zeros(n, device=dev) if mom else None
    return (lambda: cuda_ops.sgd_prox_step(x, gr, buf, 1e-3, mom, False, 0.0, z, y, rho, 1e-4, 1e-4)), (x, gr, z, y, buf)


def _graphed_step(kind: str, dev):
    """(graph, the objects its memory belongs to) of one graphed ResNet18 training step with the given block optimizer."""
    from federated_pytorch_test_b200 import models
    from federated_pytorch_test_b200.algo.graphs import capture_graph
    from federated_pytorch_test_b200.ops import cuda_ops
    from federated_pytorch_test_b200.optim import BlockSGD
    from federated_pytorch_test_b200.optim.block_adam import BlockAdam
    from federated_pytorch_test_b200.utils import FlatArena, unfreeze_all_layers

    torch.manual_seed(0)
    net = models.ResNet18().to(dev)
    arena = FlatArena(net, channels_last_weights=True)
    unfreeze_all_layers(net)
    last = len(arena.params) - 1
    if kind == "adam":
        opt = BlockAdam(arena, 0, last)
    elif kind == "adamw_clip_cosine":
        opt = BlockAdam(arena, 0, last, adamw=True, weight_decay=0.05, clip_norm=CLIP, device_lr=True)
    else:
        opt = BlockSGD(arena, 0, last, lr=0.05, momentum=0.9, nesterov=True, weight_decay=5e-4)
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
    return graph, (net, arena, opt, x, y, loss, body)


def main(argv=None) -> dict:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--windows", type=int, default=9)
    ap.add_argument("--calls", type=int, default=200, help="update launches per timed window")
    ap.add_argument("--steps", type=int, default=20, help="graph replays per timed step window")
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_client_opt.py measures the GPU path: no CUDA device")
    from federated_pytorch_test_b200.ops import functional as FX

    FX.set_fast_path(True)
    dev = torch.device("cuda", torch.cuda.current_device())

    rows = []
    for n in resnet18_block_sizes(dev):
        calls = {k: _update_call(k, n, dev) for k in KERNELS}
        for fn, _ in calls.values():
            for _ in range(5):
                fn()
        torch.cuda.synchronize()
        times = {k: [] for k in KERNELS}
        for _ in range(args.windows):
            for k, (fn, _) in calls.items():
                times[k].append(_time(fn, args.calls))
        us = {k: 1e6 * statistics.median(v) for k, v in times.items()}
        rows.append(dict(n=n, us={k: round(v, 2) for k, v in us.items()},
                         GBps={k: round(KERNELS[k][0] * n / (us[k] * 1e-6) / 1e9, 1) for k in KERNELS}))
        del calls

    from federated_pytorch_test_b200.optim.schedule import round_lr

    steps = {k: _graphed_step(k, dev) for k in ("adam", "sgd", "adamw_clip_cosine")}
    for graph, _ in steps.values():
        for _ in range(5):
            graph.replay()
    torch.cuda.synchronize()
    step_times = {k: [] for k in steps}
    sched_opt = steps["adamw_clip_cosine"][1][2]
    for w in range(args.windows):
        sched_opt.set_lr(round_lr(1e-3, w, args.windows, "cosine"))      # a new round's rate, no re-capture
        for k, (graph, _) in steps.items():
            step_times[k].append(_time(graph.replay, args.steps))
    step_ms = {k: 1e3 * statistics.median(v) for k, v in step_times.items()}

    res = {
        "device": torch.cuda.get_device_name(dev),
        "power_limit,max_sm_clock": _power_limit(),
        "windows": args.windows, "calls_per_window": args.calls, "steps_per_window": args.steps,
        "bytes_per_param": {k: v[0] for k, v in KERNELS.items()},
        "update_kernels": rows,
        "resnet18_step_ms": step_ms,
        "resnet18_step_ms_min_max": {k: [1e3 * min(v), 1e3 * max(v)] for k, v in step_times.items()},
    }
    print("device: %s  (power.limit, clocks.max.sm: %s)" % (res["device"], res["power_limit,max_sm_clock"]))
    print("  update kernel, us per launch (GB/s), median of %d windows of %d launches:" % (args.windows, args.calls))
    print("    %9s " % "n" + " ".join("%20s" % k for k in KERNELS))
    for r in rows:
        print("    %9d " % r["n"] + " ".join("%10.2f (%7.1f)" % (r["us"][k], r["GBps"][k]) for k in KERNELS))
    for k, v in step_ms.items():
        print("  ResNet18 graphed step, batch %d, every parameter trainable, %-17s %7.3f ms (median of %d windows)"
              % (B, k, v, args.windows))
    print(json.dumps(res))
    return res


if __name__ == "__main__":
    main()
