"""In-tree build + load of the native extensions.

Two extensions, both built with ``torch.utils.cpp_extension`` into
``federated_pytorch_test_b200/_build/<name>/`` so that the resulting ``.so``
travels with the source tree (a JIT cache under ``~/.cache`` would not):

* ``fedb200_runtime`` — C++ host runtime (batch assembler), no CUDA needed;
* ``fedb200_cuda``    — the sm_90a kernels (``csrc/*.cu``), compiled with
  ``-gencode arch=compute_90a,code=sm_90a -lineinfo`` and nothing else: there
  is no fallback architecture and no second backend.

``load(name)`` imports the prebuilt ``.so`` when it is newer than its sources and
otherwise rebuilds (nvcc cross-compiles without a GPU).  On a CUDA box a missing
or unbuildable ``fedb200_cuda`` is a hard error — the fast path never silently
degrades to ATen there.
"""
from __future__ import annotations

import importlib.util
import os
import sys
import threading
from typing import Dict, List

_HERE = os.path.dirname(os.path.abspath(__file__))
_CSRC = os.path.join(_HERE, "csrc")
_BUILD = os.path.join(_HERE, "_build")

CUDA_ARCH_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ["-O3", "-lineinfo", "--use_fast_math", "-std=c++17", "--expt-relaxed-constexpr",
              "-Xptxas", "-v"] + CUDA_ARCH_FLAGS
CXX_FLAGS = ["-O3", "-std=c++17", "-fPIC"]

_SPECS: Dict[str, Dict] = {
    "fedb200_runtime": {"sources": ["batch_loader.cpp"], "cuda": False},
    "fedb200_cuda": {
        "sources": ["bindings.cpp", "flat_kernels.cu", "elementwise_kernels.cu", "loss_kernels.cu",
                    "comm_kernels.cu", "gemm_wgmma.cu", "aux_kernels.cu"],
        "cuda": True,
    },
}

_loaded: Dict[str, object] = {}
_lock = threading.Lock()


def _sources(name: str) -> List[str]:
    return [os.path.join(_CSRC, s) for s in _SPECS[name]["sources"] if os.path.exists(os.path.join(_CSRC, s))]


def _so_path(name: str) -> str:
    return os.path.join(_BUILD, name, name + ".so")


def _stale(name: str) -> bool:
    so = _so_path(name)
    if not os.path.exists(so):
        return True
    t = os.path.getmtime(so)
    deps = _sources(name) + [os.path.join(_CSRC, f) for f in os.listdir(_CSRC) if f.endswith((".cuh", ".h", ".hpp"))]
    return any(os.path.getmtime(s) > t for s in deps)


def _import_so(name: str):
    spec = importlib.util.spec_from_file_location(name, _so_path(name))
    mod = importlib.util.module_from_spec(spec)
    import torch  # noqa: F401  (libtorch symbols must be loaded first)

    spec.loader.exec_module(mod)
    sys.modules[name] = mod
    return mod


def build(name: str, verbose: bool = False):
    """(Re)build extension ``name`` in-tree and import it."""
    os.environ.setdefault("TORCH_CUDA_ARCH_LIST", "9.0a")  # silence arch autodetect; real flags are explicit
    os.environ.setdefault("MAX_JOBS", str(min(8, os.cpu_count() or 4)))
    from torch.utils import cpp_extension

    spec = _SPECS[name]
    out_dir = os.path.join(_BUILD, name)
    os.makedirs(out_dir, exist_ok=True)
    kw = dict(name=name, sources=_sources(name), build_directory=out_dir, verbose=verbose,
              extra_cflags=CXX_FLAGS, extra_include_paths=[_CSRC])
    if spec["cuda"]:
        kw.update(extra_cuda_cflags=NVCC_FLAGS, with_cuda=True, extra_ldflags=["-lcuda"] if _has_libcuda() else [])
    mod = cpp_extension.load(**kw)
    _loaded[name] = mod
    return mod


def _has_libcuda() -> bool:
    # The driver library is absent in the (GPU-less) build container; kernels that need
    # driver entry points (tensor maps) resolve them at run time via cudaGetDriverEntryPoint.
    return False


def load(name: str, required: bool = True):
    """Return the extension module, building it if the in-tree ``.so`` is missing or stale."""
    with _lock:
        if name in _loaded:
            return _loaded[name]
        try:
            if not _stale(name):
                mod = _import_so(name)
            else:
                mod = build(name)
            _loaded[name] = mod
            return mod
        except Exception as exc:  # pragma: no cover - depends on toolchain
            if required:
                raise RuntimeError("native extension %s unavailable: %s" % (name, exc)) from exc
            _loaded[name] = None
            return None


def available(name: str) -> bool:
    return load(name, required=False) is not None


def build_all(verbose: bool = False) -> None:
    for name in _SPECS:
        build(name, verbose=verbose)
