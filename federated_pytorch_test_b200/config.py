"""Configuration: one dataclass per entry point, with the reference's knob names.

The reference has no flag system — its knobs are module-level constants edited
by hand (SURVEY §5.6; e.g. /root/reference/src/consensus_multi.py:8-59).  Every
constant is a dataclass field here with the same name and default, settable
from the command line as ``--K 8 --use_resnet --Nloop 2`` (booleans accept
``--flag`` / ``--no-flag`` / ``--flag=false``).  Fields that do not exist in the
reference (runtime placement, parity switches, synthetic-data options) are
grouped at the end of :class:`CommonConfig`.
"""
from __future__ import annotations

import argparse
import dataclasses
from dataclasses import dataclass, field
from typing import Optional, Sequence, Type, TypeVar

T = TypeVar("T")


@dataclass
class CommonConfig:
    K: int = 10
    default_batch: int = 128
    Nloop: int = 12
    Nepoch: int = 1
    Nadmm: int = 3
    load_model: bool = False
    init_model: bool = True
    save_model: bool = True
    check_results: bool = True
    biased_input: bool = True
    be_verbose: bool = False
    use_resnet: bool = False
    use_cuda: bool = True
    # ---- new in this framework -------------------------------------------------
    model: str = ""                 # '', 'Net', 'Net1', 'Net2', 'ResNet18', 'ResNet9' ('' = follow use_resnet)
    optimizer: str = "adam"         # 'adam' | 'lbfgs' (the reference's commented-out alternative)
    seed: int = 69                  # torch.manual_seed(69) at the top of every reference script
    data: str = "synthetic"         # 'synthetic' | 'torchvision' (needs local files, never downloads)
    data_seed: int = 1234
    data_noise: float = 0.6         # synthetic data: noise std relative to the class-template amplitude (harder when larger)
    train_size: int = 50000
    test_size: int = 10000
    data_on_device: bool = True     # dataset resident in HBM; False = pinned host + native batch assembler
    fix_shard_off_by_one: bool = False   # Q1
    intended_elastic_net_gate: bool = False  # Q2: regularise whenever the block holds dense-layer weights
    diagnostics: str = "post"       # Q17: 'post' (extra forward after the step) | 'pre'
    nan_guard: str = "raise"        # non-finite aggregation residual: 'raise' | 'warn' | 'off'
    collective: str = "auto"        # 'auto' | 'fused' | 'torch'
    fast: bool = True               # use the hand-written sm_90a kernels on CUDA devices
    graphs: bool = True             # CUDA-graph the per-minibatch step when possible
    distributed: bool = True        # honour torchrun env (one process per GPU); False = all K replicas here
    ckpt_dir: str = "."
    metrics_path: str = ""
    max_minibatches: int = 0        # >0 caps minibatches per round (smoke tests / benchmarks)
    resume: str = ""                # path of a true-resume record written by this framework: re-enter the schedule there
    resume_out: str = ""            # write the true-resume record here after every aggregation round ('' = never)
    streams: bool = True            # co-resident replicas (K > #GPUs) step concurrently on their own CUDA streams


@dataclass
class NoConsensusConfig(CommonConfig):
    Nepoch: int = 20
    Nloop: int = 1
    Nadmm: int = 1


@dataclass
class FederatedConfig(CommonConfig):
    lambda1: float = 0.0001
    lambda2: float = 0.0001


@dataclass
class FedProxConfig(CommonConfig):
    Nadmm: int = 5
    lambda1: float = 0.0001
    lambda2: float = 0.0001
    admm_rho0: float = 1.0


@dataclass
class ConsensusConfig(CommonConfig):
    Nadmm: int = 5
    lambda1: float = 0.0001
    lambda2: float = 0.0001
    admm_rho0: float = 0.1
    bb_update: bool = False
    bb_period_T: int = 2
    bb_alphacorrmin: float = 0.2
    bb_epsilon: float = 1e-3
    bb_rhomax: float = 0.1
    bb_seed_yhat0_zero: bool = False    # Q9


@dataclass
class VAEConfig(CommonConfig):
    Nadmm: int = 3
    be_verbose: bool = True             # the VAE driver prints every minibatch unconditionally
    check_results: bool = False


@dataclass
class VAECLConfig(CommonConfig):
    K: int = 1
    Kc: int = 10
    Lc: int = 32
    Nloop: int = 1
    Nadmm: int = 1
    lambda2: float = 0.001
    be_verbose: bool = True
    check_results: bool = False
    batched_clusters: bool = True


@dataclass
class CPCConfig(CommonConfig):
    K: int = 4
    Lc: int = 256
    Rc: int = 32
    batch_size: int = 128
    Nloop: int = 1
    Niter: int = 10
    Nadmm: int = 1
    load_model: bool = True
    init_model: bool = False
    be_verbose: bool = True
    check_results: bool = False
    # synthetic LOFAR source (the reference reads HDF5 files from a Colab drive)
    file_list: str = ""                 # comma separated .h5 paths ('' = synthetic)
    sap_list: str = ""                  # comma separated SAP ids
    nbase: int = 64
    ntime: int = 64
    nfreq: int = 64
    patch_layout: str = "batch_major"   # Q13: 'batch_major' | 'reference'


# ----------------------------------------------------------------------------
def _str2bool(v: str) -> bool:
    if v.lower() in ("1", "true", "yes", "y", "on"):
        return True
    if v.lower() in ("0", "false", "no", "n", "off"):
        return False
    raise argparse.ArgumentTypeError("expected a boolean, got %r" % v)


def build_parser(cls: Type[T], prog: Optional[str] = None) -> argparse.ArgumentParser:
    p = argparse.ArgumentParser(prog=prog, description=(cls.__doc__ or "").strip() or None)
    for f in dataclasses.fields(cls):
        name = "--" + f.name
        if f.type in (bool, "bool"):
            p.add_argument(name, nargs="?", const=True, default=f.default, type=_str2bool)
            p.add_argument("--no-" + f.name, dest=f.name, action="store_false")
        else:
            typ = {"int": int, "float": float, "str": str}.get(f.type if isinstance(f.type, str) else f.type.__name__, str)
            p.add_argument(name, type=typ, default=f.default)
    return p


def parse_config(cls: Type[T], argv: Optional[Sequence[str]] = None, prog: Optional[str] = None) -> T:
    ns = build_parser(cls, prog).parse_args(argv)
    return cls(**vars(ns))


def override(cfg: T, **kw) -> T:
    return dataclasses.replace(cfg, **kw)
