"""Per-kernel device time of the headline training step, and the ResNet stem's share of it.

Builds the engine ``bench.py --gpus 1`` builds (``federated_multi``, K = 1, ResNet18, batch 128, block 0 active, CUDA
graphs on, post-step diagnostics forward), runs it past graph capture, then replays ``--steps`` graphed steps under
``torch.profiler`` with CUDA activities.  The window ends before the round's first aggregation, so it holds minibatch steps
only.  Prints, per step:

  * device time and launches of every kernel, grouped by kernel name (template arguments kept, parameter list dropped);
  * the stem's kernels, found by their place in the step: the forward convolution of a 3-channel input (twice: training
    and diagnostics forward) and the ``bn_elu_fwd`` that follows each; the last ``bn_elu_bwd_reduce`` / ``bn_elu_bwd_apply``
    before the weight gradient; the weight gradient itself (block 0 is the stem, so it is the step's only one);

with the card name, its power limit and max SM clock, then one JSON line.  Profiling slows the host, not the device
kernels; end-to-end step times come from ``bench.py``.  The trace is written to a temporary directory.

    python baseline/profile_step.py [--steps 20] [--top 25]
"""
from __future__ import annotations

import argparse
import collections
import json
import os
import re
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

STEPS_PER_ROUND = 49          # bench.py: ceil(6249 / 128)
FIRST_STEP = 12               # past eager warm-up and graph capture


def _power_limit() -> str:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30)
        return out.stdout.strip().splitlines()[torch.cuda.current_device()] if out.returncode == 0 else "unknown"
    except (OSError, subprocess.SubprocessError, IndexError):
        return "unknown"


def short_name(name: str) -> str:
    """``void f<64, 4, 0>(CUtensorMap_st, ...)`` -> ``f<64, 4, 0>``."""
    name = re.sub(r"^void ", "", name)
    depth = 0
    for i, ch in enumerate(name):
        if ch == "<":
            depth += 1
        elif ch == ">":
            depth -= 1
        elif ch == "(" and depth == 0:
            return name[:i]
    return name


def stem_kernels(kernels, steps: int) -> dict:
    """Stem kernels of the trace (``kernels``: (short name, duration us) in issue order), in microseconds per step."""
    out = collections.defaultdict(float)
    after_stem_conv = False
    def base(name):
        return name.split("<")[0].split("::")[-1]

    for i, (name, dur) in enumerate(kernels):
        b = base(name)
        if b == "stem_conv_bn_kernel" or b + name[len(name.split("<")[0]):] == "igemm_wgmma_pix_kernel<64, 4, 0>":
            out["conv (" + name + ")"] += dur
            # y goes through bn_elu_fwd after the wgmma convolution and after stem_conv_bn_kernel<0> (STORE_Y) only
            after_stem_conv = b != "stem_conv_bn_kernel" or name.endswith("<0>")
        elif b == "bn_elu_fwd_kernel" and after_stem_conv:
            out["bn_elu_fwd"] += dur
            after_stem_conv = False
        elif b == "wgrad_wgmma_kernel":
            out["wgrad (" + name + ")"] += dur
            for want in ("bn_elu_bwd_apply_kernel", "bn_elu_bwd_reduce_kernel"):
                for j in range(i - 1, -1, -1):
                    if base(kernels[j][0]) == want:
                        out[want.replace("_kernel", "")] += kernels[j][1]
                        break
    res = {k: v / steps for k, v in out.items()}
    res["total"] = sum(res.values())
    return res


def main(argv=None) -> dict:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=20, help="profiled steps (ends before step %d)" % STEPS_PER_ROUND)
    ap.add_argument("--top", type=int, default=25, help="kernel groups printed")
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("profile_step.py profiles the GPU step: no CUDA device")
    if not 1 <= args.steps <= STEPS_PER_ROUND - FIRST_STEP - 1:
        ap.error("--steps must leave the window inside the first round")

    from torch.profiler import ProfilerActivity, profile

    from federated_pytorch_test_b200.algo.engine import Engine
    from federated_pytorch_test_b200.algo.strategies import FedAvg
    from federated_pytorch_test_b200.api import common, federated_multi

    cfg = federated_multi.Config(K=1, use_resnet=True, Nloop=1000, Nadmm=3, Nepoch=1, check_results=False, save_model=False,
                                 be_verbose=False, biased_input=True, data_on_device=True, graphs=True, fast=True,
                                 collective="auto", diagnostics="post", max_minibatches=STEPS_PER_ROUND, seed=69,
                                 optimizer="adam")
    topo, coll = common.setup_runtime(cfg)
    task = common.ClassifierTask(cfg, topo, cfg.lambda1, cfg.lambda2)
    eng = Engine(task, topo, FedAvg(coll, topo), coll, common.engine_config(cfg), log=lambda m: None)
    dev = topo.device
    last = FIRST_STEP + args.steps
    prof = profile(activities=[ProfilerActivity.CUDA])

    def hook(e):
        n = e.steps_done
        if n == FIRST_STEP:
            torch.cuda.synchronize(dev)
            prof.__enter__()
        elif n == last:
            torch.cuda.synchronize(dev)
            prof.__exit__(None, None, None)
            e.stop_requested = True

    eng.step_hook = hook
    eng.run()

    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            trace = json.load(f)
    evs = sorted((e for e in trace["traceEvents"] if e.get("cat") == "kernel"), key=lambda e: e["ts"])
    kernels = [(short_name(e["name"]), float(e["dur"])) for e in evs]
    groups = collections.defaultdict(lambda: [0.0, 0])
    for name, dur in kernels:
        groups[name][0] += dur
        groups[name][1] += 1
    S = args.steps
    total = sum(d for _, d in kernels) / S
    table = sorted(((v[0] / S, v[1] / S, k) for k, v in groups.items()), reverse=True)
    stem = stem_kernels(kernels, S)

    res = {"device": torch.cuda.get_device_name(dev), "power_limit,max_sm_clock": _power_limit(), "steps": S,
           "kernel_us_per_step": total, "launches_per_step": len(kernels) / S,
           "kernels": [{"name": k, "us_per_step": t, "launches_per_step": c} for t, c, k in table],
           "stem_us_per_step": stem}
    print("device: %s  (power.limit, clocks.max.sm: %s)" % (res["device"], res["power_limit,max_sm_clock"]))
    print("%d profiled steps: %.1f us of kernel time and %.1f launches per step" % (S, total, len(kernels) / S))
    for t, c, k in table[:args.top]:
        print("  %9.1f us  %5.1f x  %s" % (t, c, k[:110]))
    print("stem, per step:")
    for k, v in stem.items():
        print("  %9.1f us  %s" % (v, k))
    print(json.dumps(res))
    return res


if __name__ == "__main__":
    main()
