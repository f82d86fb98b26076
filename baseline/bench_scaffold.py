"""Cost of SCAFFOLD control variates (``--scaffold``) on one GPU.

(a) The per-round launches SCAFFOLD adds (``algo/scaffold.py``: step 1 ``scaffold_cv``, step 2 the control-variate mean as
    one aggregation launch, step 3 ``scaffold_corr``) against one FedAvg round (the fused aggregation with write-back), at
    the ten ResNet18 block sizes with K = 8 co-resident replicas.  Bytes moved per coordinate, from what the kernels read
    and write: step 1 reads c_i, c, z, x_i and writes c_i (20 B per replica), step 3 reads c, c_i and writes d_i (12 B per
    replica), the mean reads the K c_i and writes c (4 (K + 1) B).
(b) ``sgd_prox`` with and without the correction operand ``y = d_i`` at 4.72 M parameters (the largest block), momentum
    0.9 (20 B -> 24 B per parameter) and 0 (12 B -> 16 B).
(c) A CUDA-graphed ResNet18 training step at batch 128, every parameter trainable, SGD with momentum 0.9: without and with
    the correction operand.

Every arm is timed between two CUDA events over ``--calls`` calls (``--steps`` replays for (c)), ``--windows`` windows
with the arms alternating window by window; the median window is reported.  Prints the device name, its power limit and
max SM clock, a table, then one JSON line.  Writes nothing to disk.

    python baseline/bench_scaffold.py [--windows 9] [--calls 100] [--steps 20]
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

K = 8
B = 128
N_LARGEST = 4720640


def _round_arms(n: int, dev):
    """(FedAvg round, SCAFFOLD steps 1-3, objects kept alive) on K co-resident replicas of an ``n``-parameter block."""
    from federated_pytorch_test_b200.algo.scaffold import ControlVariates
    from federated_pytorch_test_b200.parallel import Topology
    from federated_pytorch_test_b200.parallel.fused import FusedCollective

    topo = Topology.single_process(K, dev)
    coll = FusedCollective(topo)
    stride = -(-n // 32) * 32
    xs = [coll.heap.alloc(stride)[:n] for _ in range(K)]
    g = torch.Generator(device=dev).manual_seed(n)
    for x in xs:
        x.copy_(torch.randn(n, device=dev, generator=g))
    z = coll.zeros_like_block(xs[0], "z")
    cv = ControlVariates(coll, topo)
    cv.begin_block(0, xs)

    def fedavg():
        coll.launch_fedavg_(xs, z, True)

    def scaffold():
        cv.note_local_steps([10] * K, 0.05)
        cv.end_round(xs, z)

    return fedavg, scaffold, (coll, xs, z, cv)


def _sgd_call(momentum: float, with_y: bool, n: int, dev):
    from federated_pytorch_test_b200.ops import cuda_ops

    g = torch.Generator(device=dev).manual_seed(n)
    x = torch.randn(n, device=dev, generator=g)
    gr = 1e-3 * torch.randn(n, device=dev, generator=g)
    y = 1e-3 * torch.randn(n, device=dev, generator=g) if with_y else None
    buf = torch.zeros(n, device=dev) if momentum else None
    return lambda: cuda_ops.sgd_prox_step(x, gr, buf, 1e-3, momentum, False, 0.0, y=y), (x, gr, y, buf)


def _graphed_step(with_y: bool, dev):
    """(graph, the objects its memory belongs to) of one graphed ResNet18 SGD step, with or without the correction."""
    from federated_pytorch_test_b200 import models
    from federated_pytorch_test_b200.algo.graphs import capture_graph
    from federated_pytorch_test_b200.ops import cuda_ops
    from federated_pytorch_test_b200.optim import BlockSGD
    from federated_pytorch_test_b200.utils import FlatArena, unfreeze_all_layers

    torch.manual_seed(0)
    net = models.ResNet18().to(dev)
    arena = FlatArena(net, channels_last_weights=True)
    unfreeze_all_layers(net)
    last = len(arena.params) - 1
    opt = BlockSGD(arena, 0, last, lr=0.05, momentum=0.9)
    d = 1e-4 * torch.randn(opt.x.numel(), device=dev) if with_y else None
    opt.set_penalty(y=d)
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
    return graph, (net, arena, opt, d, x, y, loss, body)


def _alternate(arms: dict, windows: int, calls: int, after=None) -> dict:
    for fn in arms.values():
        for _ in range(3):
            fn()
    if after is not None:
        after()
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for _ in range(windows):
        for k, fn in arms.items():
            times[k].append(_time(fn, calls))
            if after is not None:
                after()
    return times


def main(argv=None) -> dict:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--windows", type=int, default=9)
    ap.add_argument("--calls", type=int, default=100, help="launches (or rounds) per timed window")
    ap.add_argument("--steps", type=int, default=20, help="graph replays per timed step window")
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_scaffold.py measures the GPU path: no CUDA device")
    from federated_pytorch_test_b200.ops import functional as FX

    FX.set_fast_path(True)
    dev = torch.device("cuda", torch.cuda.current_device())

    rounds = []                                                   # (a)
    for n in resnet18_block_sizes(dev):
        fedavg, scaffold, keep = _round_arms(n, dev)
        t = _alternate({"fedavg_round": fedavg, "scaffold_steps": scaffold}, args.windows, args.calls,
                       after=keep[0].read_record)
        us = {k: 1e6 * statistics.median(v) for k, v in t.items()}
        nbytes = (20 * K + 12 * K + 4 * (K + 1)) * n
        rounds.append(dict(n=n, us={k: round(v, 2) for k, v in us.items()},
                           scaffold_GBps=round(nbytes / (us["scaffold_steps"] * 1e-6) / 1e9, 1)))
        del keep, fedavg, scaffold

    sgd_arms, keep = {}, []                                       # (b)
    for mom, base in ((0.9, 20), (0.0, 12)):
        for with_y in (False, True):
            fn, k = _sgd_call(mom, with_y, N_LARGEST, dev)
            sgd_arms["sgd_m%g%s" % (mom, "_y" if with_y else "")] = fn
            keep.append(k)
    sgd_bytes = {"sgd_m0.9": 20, "sgd_m0.9_y": 24, "sgd_m0": 12, "sgd_m0_y": 16}
    t = _alternate(sgd_arms, args.windows, args.calls)
    sgd_us = {k: 1e6 * statistics.median(v) for k, v in t.items()}
    del keep

    steps = {k: _graphed_step(k == "sgd_m0.9_scaffold", dev) for k in ("sgd_m0.9", "sgd_m0.9_scaffold")}   # (c)
    t = _alternate({k: g.replay for k, (g, _) in steps.items()}, args.windows, args.steps)
    step_ms = {k: 1e3 * statistics.median(v) for k, v in t.items()}

    res = {
        "device": torch.cuda.get_device_name(dev),
        "power_limit,max_sm_clock": _power_limit(),
        "K": K, "windows": args.windows, "calls_per_window": args.calls, "steps_per_window": args.steps,
        "round_us": rounds,
        "sgd_prox_us": {k: round(v, 2) for k, v in sgd_us.items()},
        "sgd_prox_GBps": {k: round(sgd_bytes[k] * N_LARGEST / (v * 1e-6) / 1e9, 1) for k, v in sgd_us.items()},
        "resnet18_step_ms": step_ms,
        "resnet18_step_ms_min_max": {k: [1e3 * min(v), 1e3 * max(v)] for k, v in t.items()},
    }
    print("device: %s  (power.limit, clocks.max.sm: %s)" % (res["device"], res["power_limit,max_sm_clock"]))
    print("  (a) per round, K = %d co-resident replicas, us (median of %d windows of %d rounds):" % (K, args.windows,
                                                                                                   args.calls))
    print("    %9s %14s %16s %12s" % ("n", "fedavg_round", "scaffold_steps", "GB/s"))
    for r in rounds:
        print("    %9d %14.2f %16.2f %12.1f" % (r["n"], r["us"]["fedavg_round"], r["us"]["scaffold_steps"],
                                               r["scaffold_GBps"]))
    print("  (b) sgd_prox at n = %d, us per launch (GB/s):" % N_LARGEST)
    for k, v in sgd_us.items():
        print("    %-12s %8.2f (%7.1f)" % (k, v, res["sgd_prox_GBps"][k]))
    for k, v in step_ms.items():
        print("  (c) ResNet18 graphed step, batch %d, %-18s %7.3f ms" % (B, k, v))
    print(json.dumps(res))
    return res


if __name__ == "__main__":
    main()
