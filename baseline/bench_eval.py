"""Test-set evaluation throughput of ResNet18 with train-mode and eval-mode BatchNorm.

One replica evaluates 10 000 synthetic CIFAR10 test images at batch 128 (78 full batches + one of 16), with weights after a
few Adam steps so that the running statistics are not trivial.  Three arms, alternated in one process, each warmed up and
CUDA-graphed where the engine graphs it (``ClassifierTask.evaluate``):

  (a) batch    train-mode BatchNorm on the hand-written kernels (the default, ``eval_bn='batch'``, SURVEY Q4), graphed;
  (b) running  eval-mode BatchNorm on the hand-written kernels (``eval_bn='running'``): conv + BN + residual + ELU per launch, graphed;
  (c) aten     eval-mode BatchNorm on the ATen / cuDNN composition (``net.eval()`` without the fast path), eager.

Prints images/s per arm (median over the repetitions, CUDA events around each full pass), the hand-written kernel launches
per batch-128 forward, the agreement of (b) with (c) on the whole test set, the device name and its power limit, then one
JSON line.  Writes nothing to disk.

    python baseline/bench_eval.py [--reps 7] [--adam-steps 20]
"""
from __future__ import annotations

import argparse
import copy
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


def main(argv=None) -> dict:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--reps", type=int, default=7, help="timed passes over the test set per arm")
    ap.add_argument("--adam-steps", type=int, default=20)
    ap.add_argument("--test-size", type=int, default=10000)
    ap.add_argument("--batch", type=int, default=128)
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_eval.py measures the GPU path: no CUDA device")

    from federated_pytorch_test_b200 import models
    from federated_pytorch_test_b200.algo.graphs import GraphedEval
    from federated_pytorch_test_b200.data.cifar import ShardLoader, make_synthetic_cifar, worker_norm
    from federated_pytorch_test_b200.ops import cuda_ops, losses
    from federated_pytorch_test_b200.ops import functional as FX

    dev = torch.device("cuda", torch.cuda.current_device())
    torch.manual_seed(69)
    mean, std = worker_norm(0, True)
    tr_x, tr_y = make_synthetic_cifar(True, seed=1234, size=args.adam_steps * args.batch)
    te_x, te_y = make_synthetic_cifar(False, seed=1235, size=args.test_size)
    train = list(ShardLoader(tr_x.to(dev), tr_y.to(dev), range(tr_x.shape[0]), args.batch, dev, mean, std, seed=1, channels_last=True))
    test = [(x.clone(), y.clone()) for x, y in ShardLoader(te_x.to(dev), te_y.to(dev), range(te_x.shape[0]), args.batch, dev,
                                                           mean, std, shuffle=False, channels_last=True)]

    # weights and running statistics after a few Adam steps on the fast path (train mode, as the drivers train)
    FX.set_fast_path(True)
    net = models.ResNet18().to(dev).to(memory_format=torch.channels_last)
    opt = torch.optim.Adam(net.parameters(), lr=1e-3)
    for x, y in train:
        opt.zero_grad()
        losses.cross_entropy(net(x), y).backward()
        opt.step()
    torch.cuda.synchronize()
    net_batch = copy.deepcopy(net)          # arm (a) moves its running statistics (train-mode BN on test data): its own copy
    net.eval()

    counter = torch.zeros(2, dtype=torch.int64, device=dev)
    graphs = {}

    def pass_fast(model, arm):
        FX.set_fast_path(True)
        with torch.no_grad():
            for x, y in test:
                key = (arm, tuple(x.shape))
                ge = graphs.get(key)
                if ge is None:
                    ge = graphs[key] = GraphedEval(model, (x, y), counter, dev)
                ge.run((x, y))

    def pass_aten(model):
        FX.set_fast_path(False)
        with torch.no_grad():
            for x, y in test:
                logits = model(x)
                counter[0] += (logits.argmax(dim=1) == y).sum()
                counter[1] += y.shape[0]
        FX.set_fast_path(True)

    arms = {"batch": lambda: pass_fast(net_batch, "batch"), "running": lambda: pass_fast(net, "running"),
            "aten": lambda: pass_aten(net)}
    for fn in arms.values():                # warm-up: eager passes, graph capture, cuDNN algorithm choice
        for _ in range(GraphedEval.WARMUP + 2):
            fn()
    torch.cuda.synchronize()

    times = {k: [] for k in arms}
    correct = {}
    for _ in range(args.reps):
        for name, fn in arms.items():
            counter.zero_()
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            fn()
            t1.record()
            t1.synchronize()
            times[name].append(t0.elapsed_time(t1) / 1e3)
            correct[name] = int(counter[0])

    # hand-written kernel launches of one eager batch-128 forward
    launches = {}
    x0 = test[0][0]
    with torch.no_grad():
        for name, model in (("batch", net_batch), ("running", net)):
            before = cuda_ops.launch_count()
            model(x0)
            launches[name] = cuda_ops.launch_count() - before
        FX.set_fast_path(False)
        before = cuda_ops.launch_count()
        net(x0)
        launches["aten"] = cuda_ops.launch_count() - before
        FX.set_fast_path(True)

        # agreement of (b) with (c) on the whole test set (eager forwards, same weights and running statistics)
        same = total = 0
        worst = 0.0
        for x, _ in test:
            b = net(x)
            FX.set_fast_path(False)
            c = net(x)
            FX.set_fast_path(True)
            same += int((b.argmax(1) == c.argmax(1)).sum())
            total += x.shape[0]
            worst = max(worst, float((b - c).abs().max() / c.abs().max().clamp_min(1e-12)))

    n = sum(x.shape[0] for x, _ in test)
    res = {
        "device": torch.cuda.get_device_name(dev),
        "power_limit,max_sm_clock": _power_limit(),
        "images": n, "batch": args.batch, "reps": args.reps,
        "images_per_s": {k: n / statistics.median(v) for k, v in times.items()},
        "ms_per_pass": {k: 1e3 * statistics.median(v) for k, v in times.items()},
        "ms_per_pass_min_max": {k: [1e3 * min(v), 1e3 * max(v)] for k, v in times.items()},
        "handwritten_launches_per_batch": launches,
        "correct": correct,
        "running_vs_aten_argmax_agreement": same / total,
        "running_vs_aten_max_rel_logit_err": worst,
    }
    print("device: %s  (power.limit, clocks.max.sm: %s)" % (res["device"], res["power_limit,max_sm_clock"]))
    for k in arms:
        print("  %-8s %9.0f images/s  %7.2f ms per %d images  %3d hand-written launches per batch  %d correct"
              % (k, res["images_per_s"][k], res["ms_per_pass"][k], n, launches[k], correct[k]))
    print("  running vs aten: argmax agreement %.4f, max relative logit error %.2e" % (same / total, worst))
    print(json.dumps(res))
    return res


if __name__ == "__main__":
    main()
