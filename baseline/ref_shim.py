"""Run the UNMODIFIED reference scripts offline and time them (SURVEY Appendix A).

The reference (``oracle/_ref/src/*.py``, a verbatim copy of the original project made by
``oracle/install_reference.sh``) cannot run without a network: it downloads CIFAR10 through
torchvision and has no timers.  This shim

1. replaces ``torchvision.datasets.CIFAR10`` *in memory* by a synthetic dataset with the same
   constructor signature and item contract (uint8 HWC image -> PIL -> the script's own transform),
2. overrides module-level constants of the script by regex on the source text (the reference's own
   "config system": constants edited by hand), nothing else is touched,
3. ``exec``s the script and observes it from outside: ``torch.optim.Adam.step`` is wrapped to count
   optimizer steps, record CUDA events at the warm-up / end boundaries and stop the run.

Everything on the timed path — the models, the DataLoader with its worker process, ``.to(device)``,
closures, Adam, the diagnostics forward and ``.item()`` — is the reference's own code.
"""
from __future__ import annotations

import json
import os
import re
import sys
import time
from typing import Dict, Optional

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REF_SRC = os.path.join(os.path.dirname(HERE), "oracle", "_ref", "src")


class _StopBench(Exception):
    pass


def _install_synthetic_cifar(seed: int = 1234) -> None:
    import numpy as np
    import torchvision
    from PIL import Image

    sys.path.insert(0, os.path.dirname(HERE))
    from federated_pytorch_test_b200.data.cifar import make_synthetic_cifar

    cache: Dict[bool, tuple] = {}

    class SyntheticCIFAR10(torch.utils.data.Dataset):
        def __init__(self, root=None, train=True, transform=None, target_transform=None, download=False):
            if train not in cache:
                imgs, labs = make_synthetic_cifar(train, seed)
                cache[train] = (imgs.numpy(), labs.tolist())
            self.data, self.targets = cache[train]
            self.transform, self.target_transform = transform, target_transform

        def __len__(self):
            return len(self.targets)

        def __getitem__(self, i):
            img, target = Image.fromarray(self.data[i]), self.targets[i]
            if self.transform is not None:
                img = self.transform(img)
            if self.target_transform is not None:
                target = self.target_transform(target)
            return img, target

    torchvision.datasets.CIFAR10 = SyntheticCIFAR10


def _override(src: str, consts: Dict[str, object]) -> str:
    for name, val in consts.items():
        src, n = re.subn(r"(?m)^%s\s*=.*$" % re.escape(name), "%s=%r" % (name, val), src, count=1)
        if n != 1:
            raise RuntimeError("constant %s not found in the reference script" % name)
    return src


def _use_lbfgs(src: str) -> str:
    """The reference's own commented-out alternative (e.g. fedprox_multi.py:162-163): swap which optimizer line is
    commented.  Nothing else in the script changes."""
    lines = src.split("\n")
    done = 0
    for i, ln in enumerate(lines):
        st = ln.lstrip()
        ind = ln[: len(ln) - len(st)]
        if st.startswith("#opt_dict[ck]=LBFGSNew("):
            lines[i] = ind + st[1:]
            done += 1
        elif st.startswith("opt_dict[ck]=optim.Adam("):
            lines[i] = ind + "#" + st
            done += 1
    if done < 2:
        raise RuntimeError("optimizer lines not found in the reference script")
    return "\n".join(lines)


def run_reference_script(script: str, consts: Dict[str, object], steps: Optional[int] = None, warmup: int = 0,
                         workdir: Optional[str] = None, on_timed_start=None, optimizer: str = "adam") -> Dict:
    """Execute ``oracle/_ref/src/<script>``; if ``steps`` is given stop after ``warmup+steps`` optimizer steps."""
    path = os.path.join(REF_SRC, script)
    if not os.path.exists(path):
        raise FileNotFoundError(path)
    _install_synthetic_cifar()
    src = _override(open(path).read(), consts)
    sys.path.insert(0, REF_SRC)
    if optimizer == "lbfgs":
        src = _use_lbfgs(src)
        import lbfgsnew as _ref_lbfgs       # the reference's module (REF_SRC is first on sys.path)

        opt_cls = _ref_lbfgs.LBFGSNew
    else:
        opt_cls = torch.optim.Adam
    cuda = torch.cuda.is_available()
    state = {"n": 0, "ev0": None, "ev1": None, "t0": 0.0, "t1": 0.0}
    orig_step = opt_cls.step

    def counted_step(self, closure=None):
        if steps is not None and state["n"] == warmup:
            if cuda:
                torch.cuda.synchronize()
                state["ev0"] = torch.cuda.Event(enable_timing=True)
                if on_timed_start is not None:
                    on_timed_start()
                state["ev0"].record()
            state["t0"] = time.perf_counter()
        out = orig_step(self, closure)
        state["n"] += 1
        return out

    # the diagnostics forward + .item() follow each step inside the script; stop at the START of step warmup+steps
    def stopping_step(self, closure=None):
        if steps is not None and state["n"] == warmup + steps:
            if cuda:
                state["ev1"] = torch.cuda.Event(enable_timing=True)
                state["ev1"].record()
                torch.cuda.synchronize()
            state["t1"] = time.perf_counter()
            raise _StopBench()
        return counted_step(self, closure)

    opt_cls.step = stopping_step
    cwd = os.getcwd()
    if workdir:
        os.makedirs(workdir, exist_ok=True)
        os.chdir(workdir)
    try:
        exec(compile(src, script, "exec"), {"__name__": "__main__"})
    except _StopBench:
        pass
    finally:
        opt_cls.step = orig_step
        os.chdir(cwd)
    res = {"optimizer_steps": state["n"]}
    if steps is not None and state["ev0"] is not None and state["ev1"] is not None:
        res["device_ms"] = state["ev0"].elapsed_time(state["ev1"])
    if steps is not None:
        res["wall_ms"] = (state["t1"] - state["t0"]) * 1e3
    return res


_SCRIPTS = {"federated": "federated_multi.py", "consensus": "consensus_multi.py", "fedprox": "fedprox_multi.py",
            "vae": "federated_vae.py"}
MIN_TIMED_OPT_STEPS = 100      # >= 1 s of reference time: a 0.2-0.3 s window moved 46 % between two boxes (VERDICT r1)


def run_reference_bench(gpus: int, steps: int, warmup: int, driver: str = "federated", bb: bool = False,
                        optimizer: str = "adam") -> Dict:
    """``bench.py --impl reference``: the matching unmodified script, ResNet18 (or the VAE), K = gpus workers — all on
    ONE device, visited sequentially, which is what the reference does on any box (SURVEY §0).  One benchmark *step* =
    one minibatch on every worker = ``gpus`` optimizer steps of 128 images.

    The reference visits its workers one after the other, a whole shard each (49 minibatches), and aggregates after
    the last one.  The timed window is placed like the product arm's: it straddles the first aggregation when the
    requested number of steps allows, and it is at least MIN_TIMED_OPT_STEPS optimizer steps long (``timed_steps`` in
    the record) so that DataLoader jitter averages out; ``ms_per_step`` and ``value`` are per benchmark step."""
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return {}
    if driver not in _SCRIPTS:
        return {"impl": "reference", "unavailable": "federated_cpc.py cannot run as shipped (TypeError at :219, needs h5py + LOFAR files; SURVEY Q12)"
                if driver == "cpc" else "no reference arm for driver %r" % driver}
    script = _SCRIPTS[driver]
    if not os.path.exists(os.path.join(REF_SRC, script)):
        return {"impl": "reference", "unavailable": "oracle/_ref missing: run oracle/install_reference.sh /path/to/federated-pytorch-test"}
    if not torch.cuda.is_available():
        return {"impl": "reference", "unavailable": "no CUDA device"}
    per_round = max(1, -(-(50000 // gpus - 1) // 128))          # minibatches per worker per round (49 for K = 8... 391 for K = 1)
    timed = max(steps, -(-MIN_TIMED_OPT_STEPS // gpus))          # benchmark steps actually timed
    opt_per_round = per_round * gpus                            # sequential optimizer steps before the first aggregation
    first = opt_per_round - (timed * gpus) // 2                 # straddle the first aggregation ...
    if first < warmup * gpus or timed * gpus >= 2 * opt_per_round:
        first = warmup * gpus                                   # ... unless the window is long enough to reach it anyway
    nadmm = max(3, -(-(first + timed * gpus) // opt_per_round) + 1)     # same rule as the product arm: block 0 stays active
    consts = dict(K=gpus, Nloop=1000, Nadmm=nadmm, Nepoch=1, check_results=False, save_model=False, load_model=False)
    if driver != "vae":
        consts.update(use_resnet=True, be_verbose=False)
    if driver == "consensus":
        consts["bb_update"] = bool(bb)
    from bench import ClockSampler  # same clock sampling as the product arm

    sampler = ClockSampler(0)
    sampler.start()      # early (NVML start-up must not fall into the timed region); the window is marked by sample index
    marks = {}
    res = run_reference_script(script, consts, steps=timed * gpus, warmup=first, workdir="/tmp/fedref_run",
                               on_timed_start=lambda: marks.setdefault("i0", sampler.mark()), optimizer=optimizer)
    clocks = sampler.window(marks.get("i0", 0), sampler.mark())
    sampler.stop()
    ms = max(res.get("device_ms", 0.0), res.get("wall_ms", 0.0))
    images = 128 * gpus * timed
    value = images / (ms / 1e3)
    aggs = sum(1 for b in range(opt_per_round, first + timed * gpus + 1, opt_per_round) if first < b <= first + timed * gpus)
    return {
        "metric": "train_images_per_sec", "value": value, "unit": "images/s", "n_gpus": gpus, "steps": steps, "warmup": warmup,
        "ms_per_step": ms / timed, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
        "dtype": "fp32 storage, tf32 conv (PyTorch defaults)", "data": "synthetic", "impl": "reference",
        "config": {"model": "AutoEncoderCNN" if driver == "vae" else "ResNet18",
                   "algo": {"federated": "fedavg", "consensus": "admm" + ("+bb" if bb else ""), "fedprox": "fedprox", "vae": "fedavg"}[driver],
                   "optimizer": optimizer, "global_batch": 128 * gpus, "K": gpus,
                   "parallelism": "reference: K=%d replicas sequential on ONE GPU (no distributed runtime)" % gpus,
                   "script": "oracle/_ref/src/%s (unmodified; constants overridden by regex; synthetic CIFAR10 class)" % script,
                   "timed_steps": timed, "timed_optimizer_steps": [first, first + timed * gpus], "aggregations_in_window": aggs,
                   "timing": "CUDA events around optimizer steps %d..%d, observed via a wrapper on the optimizer's step()" % (first, first + timed * gpus),
                   "device_ms": res.get("device_ms"), "wall_ms": res.get("wall_ms")},
        "clocks": clocks,
        "e2e": {"value": value, "unit": "images/s", "h2d_bytes_per_step": gpus * (128 * 3 * 32 * 32 * 4 + 128 * 8),
                "d2h_bytes_per_step": gpus * 4, "note": "the reference's only path is end to end (DataLoader -> .to(device) -> step -> .item())"},
        "gpu_launches": 0,
    }


if __name__ == "__main__":
    print(json.dumps(run_reference_bench(int(sys.argv[1]) if len(sys.argv) > 1 else 1, 5, 3)))
