"""GroupNorm ResNets on the sm_90a kernels (``csrc/norm_kernels.cu``), against float64 ATen.

1. Every distinct conv + GroupNorm (+ residual) (+ ELU) group of ResNet18 through ``cuda_ops.conv_gn_act`` at batch 128 and
   105, for G in {1, 2, 32}, with a trainable weight whose channels-last gradient buffer is pre-filled (``accumulate_into_grad``)
   and with a frozen weight: output, dx, dW, dgamma, dbeta and d(residual).
2. The GroupNorm kernels alone, on fixed convolution outputs: two calls give the same bits, and an input offset by 10^3
   with unit spread keeps the bounds of part 1.
3. The whole ResNet18-GN step (loss and every gradient) with one block trainable and with all, eagerly and from a CUDA graph;
   the kernels it launches (no cuDNN, cuBLAS or CUTLASS kernel, no ATen group norm), profiled in a fresh process.
4. A graphed ``federated_multi`` run of ResNet18-GN with K = 2 co-resident replicas, and ``eval_bn`` on it.

Oracles: ``F.conv2d`` -> ``F.group_norm`` -> ``+ residual`` -> ``F.elu`` in float64, and the model ``.double()`` on the ATen
path.  Errors are max |got - ref| / max |ref| per tensor ("max-normalised"), plus |got - ref|_2 / |ref|_2 for the whole model.
Worst values measured on an H100 80GB HBM3 (SXM, 700 W power limit) over every case, and the bounds (about 3x):

    check                                  worst     bound
    1. output                              3.8e-4    1.2e-3
       dx                                  4.3e-4    1.3e-3
       dW (gradient buffer - pre-fill)     4.8e-4    1.5e-3
       dgamma / dbeta                      4.5e-4    1.4e-3
       d(residual)                         9.7e-4    3e-3
    2. offset 10^3: output / dy            1.0e-4    (part 1 bounds)
       dgamma / dbeta                      4.2e-5    (part 1 bounds)
    3. loss                                1.2e-5    4e-5
       gradients, max-normalised           2.7e-3    8e-3
       gradients, relative L2              2.2e-3    6.5e-3

Run on an H100: ``python -m pytest tests -m gpu``."""
import functools
import json
import os
import subprocess
import sys

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():  # collected (and deselected) on the CPU box
    pytest.skip("CUDA device required", allow_module_level=True)

from federated_pytorch_test_b200 import models  # noqa: E402
from federated_pytorch_test_b200.algo.graphs import capture_graph  # noqa: E402
from federated_pytorch_test_b200.ops import cuda_ops  # noqa: E402
from federated_pytorch_test_b200.ops import functional as FX  # noqa: E402
from federated_pytorch_test_b200.utils import FlatArena, unfreeze_all_layers, unfreeze_one_block  # noqa: E402

DEV = torch.device("cuda", 0)
BATCHES = (128, 105)
GROUP_COUNTS = (1, 2, 32)
EPS = 1e-5

# bounds: about 3x the worst value measured (module docstring)
OUT_TOL = 1.2e-3
DX_TOL = 1.3e-3
DW_TOL = 1.5e-3
DGB_TOL = 1.4e-3               # dgamma and dbeta
DRES_TOL = 3e-3
LOSS_TOL = 4e-5
GRAD_TOL = 8e-3                # whole model, max-normalised per tensor
GRAD_L2_TOL = 6.5e-3           # whole model, relative L2 per tensor


@pytest.fixture(autouse=True)
def _exact_reference_math():
    """The oracle runs in true fp32 / fp64; the fast path is switched on per test."""
    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    FX.set_fast_path(True)
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old
    FX.set_fast_path(True)


def max_err(got, ref):
    return float((got.detach().double() - ref).abs().max() / ref.abs().max().clamp_min(1e-30))


def l2_err(got, ref):
    return float((got.detach().double() - ref).norm() / ref.norm().clamp_min(1e-30))


def _check(kind, got, ref, bound, name=""):
    assert got is not None, "%s %s: no gradient" % (kind, name)
    assert tuple(got.shape) == tuple(ref.shape), "%s %s: shape %s != %s" % (kind, name, tuple(got.shape), tuple(ref.shape))
    e = max_err(got, ref)
    assert e < bound, "%s %s: max-normalised error %.3g >= %.3g" % (kind, name, e, bound)
    return e


# ------------------------------------------------------------------------------------------------ 1. single groups
# name: (C_in, C_out, H_in, k, stride, residual, act) of every distinct group of ResNet18
GROUPS = {
    "stem": (3, 64, 32, 3, 1, False, True),
    "layer1": (64, 64, 32, 3, 1, False, True),
    "layer1-residual": (64, 64, 32, 3, 1, True, True),
}
for _i, (_ci, _co, _h) in enumerate(((64, 128, 32), (128, 256, 16), (256, 512, 8)), start=2):
    GROUPS["layer%d.0.conv1" % _i] = (_ci, _co, _h, 3, 2, False, True)
    GROUPS["layer%d.0.shortcut" % _i] = (_ci, _co, _h, 1, 2, False, False)
    GROUPS["layer%d.0.conv2" % _i] = (_co, _co, _h // 2, 3, 1, True, True)
    GROUPS["layer%d.1.conv1" % _i] = (_co, _co, _h // 2, 3, 1, False, True)


@functools.lru_cache(maxsize=1)
def _group_case(name, B, G):
    """Seeded fp32 inputs of one group and what float64 ATen computes from them."""
    ci, co, h, k, s, res, act = GROUPS[name]
    g = torch.Generator(device=DEV).manual_seed(1000 * B + 7 * G + sum(map(ord, name)))
    x = torch.randn(B, ci, h, h, device=DEV, generator=g)
    if name != "stem":
        x = F.elu(x)
    x = x.contiguous(memory_format=torch.channels_last)
    w = torch.randn(co, ci, k, k, device=DEV, generator=g) / (ci * k * k) ** 0.5
    gamma = 1.0 + 0.2 * torch.randn(co, device=DEV, generator=g)
    beta = 0.2 * torch.randn(co, device=DEV, generator=g)
    ho = (h + 2 * (k // 2) - k) // s + 1
    r = torch.randn(B, co, ho, ho, device=DEV, generator=g).contiguous(memory_format=torch.channels_last) if res else None
    dout = torch.randn(B, co, ho, ho, device=DEV, generator=g).contiguous(memory_format=torch.channels_last)
    inp = dict(x=x, w=w, gamma=gamma, beta=beta, r=r, dout=dout)

    x64, w64 = x.double().requires_grad_(), w.double().requires_grad_()
    g64, b64 = gamma.double().requires_grad_(), beta.double().requires_grad_()
    r64 = r.double().requires_grad_() if res else None
    u = F.group_norm(F.conv2d(x64, w64, None, s, k // 2), G, g64, b64, EPS)
    if res:
        u = u + r64
    out = F.elu(u) if act else u
    out.backward(dout.double())
    ref = dict(out=out.detach(), dx=x64.grad, dw=w64.grad, dgamma=g64.grad, dbeta=b64.grad, dres=r64.grad if res else None)
    return inp, ref


def group_errors(name, B, G, mode):
    """{check: max-normalised error} of one group case (asserting the bounds)."""
    ci, co, h, k, s, res, act = GROUPS[name]
    inp, ref = _group_case(name, B, G)
    trainable = mode == "trainable"
    conv = nn.Conv2d(ci, co, k, s, k // 2, bias=False).to(DEV)
    gn = nn.GroupNorm(G, co, eps=EPS).to(DEV)
    with torch.no_grad():
        # stored channels-last as FlatArena(channels_last_weights=True) stores it: the frozen filter is cached by address
        conv.weight = nn.Parameter(inp["w"].contiguous(memory_format=torch.channels_last), requires_grad=trainable)
        gn.weight.copy_(inp["gamma"])
        gn.bias.copy_(inp["beta"])
    x = inp["x"].detach().requires_grad_()
    r = inp["r"].detach().requires_grad_() if res else None
    assert cuda_ops.conv_gn_act_supported(x, conv, gn) and not cuda_ops.conv_bn_act_supported(x, conv, gn)
    prefill = None
    if trainable:
        gen = torch.Generator(device=DEV).manual_seed(B + co)
        prefill = torch.randn(co, k, k, ci, device=DEV, generator=gen).permute(0, 3, 1, 2) * float(ref["dw"].abs().max())
        conv.weight.grad = prefill.clone()
    with cuda_ops.accumulate_into_grad():
        out = FX.conv_bn_act(x, conv, gn, residual=r, act=act)
        out.backward(inp["dout"])
    torch.cuda.synchronize()
    tag = "%s B=%d G=%d %s" % (name, B, G, mode)
    errs = dict(out=_check("out", out, ref["out"], OUT_TOL, tag), dx=_check("dx", x.grad, ref["dx"], DX_TOL, tag),
                dgamma=_check("dgamma", gn.weight.grad, ref["dgamma"], DGB_TOL, tag),
                dbeta=_check("dbeta", gn.bias.grad, ref["dbeta"], DGB_TOL, tag))
    if res:
        errs["dres"] = _check("dres", r.grad, ref["dres"], DRES_TOL, tag)
    if trainable:
        errs["dw"] = _check("dW", conv.weight.grad.double() - prefill.double(), ref["dw"], DW_TOL, tag)
    else:
        assert conv.weight.grad is None
        if ci % 4 == 0:
            cache = cuda_ops._S2_CACHE if s == 2 else cuda_ops._FLIP_CACHE
            wk = conv.weight.detach().permute(0, 2, 3, 1)
            assert (wk.data_ptr(), tuple(wk.shape)) in cache
    return errs


GROUP_CASES = [(n, B, G, m) for n in GROUPS for B in BATCHES for G in GROUP_COUNTS for m in ("trainable", "frozen")]


@pytest.mark.parametrize("name,B,G,mode", GROUP_CASES)
def test_group_matches_float64(name, B, G, mode):
    group_errors(name, B, G, mode)


# ------------------------------------------------------------------------------------------------ 2. the kernels alone
def _kernel_inputs(B, HW, C, offset, seed, residual):
    g = torch.Generator(device=DEV).manual_seed(seed)
    side = int(HW ** 0.5)
    y = offset + torch.randn(B, side, side, C, device=DEV, generator=g)
    gamma = 1.0 + 0.2 * torch.randn(C, device=DEV, generator=g)
    beta = 0.2 * torch.randn(C, device=DEV, generator=g)
    r = torch.randn(B, side, side, C, device=DEV, generator=g) if residual else None
    dout = torch.randn(B, side, side, C, device=DEV, generator=g)
    return y, gamma, beta, r, dout


def _kernels(y, gamma, beta, r, dout, G, act=True):
    e = cuda_ops.ext()
    out, mean, rstd = e.gn_elu_fwd(y, gamma, beta, r, G, EPS, act)
    dy, dres, dgamma, dbeta = e.gn_elu_bwd(dout, out if r is not None else None, y, mean, rstd, gamma, beta, G, r is not None,
                                           act, True)
    return [t for t in (out, mean, rstd, dy, dres, dgamma, dbeta) if t is not None]


KERNEL_SHAPES = [(128, 1024, 64), (105, 256, 128), (128, 16, 512)]


@pytest.mark.parametrize("B,HW,C", KERNEL_SHAPES)
@pytest.mark.parametrize("G", GROUP_COUNTS)
@pytest.mark.parametrize("residual", [False, True])
def test_kernels_are_bit_identical_run_to_run(B, HW, C, G, residual):
    inp = _kernel_inputs(B, HW, C, 0.0, B + HW + C + G, residual)
    first = _kernels(*inp, G)
    for _ in range(2):
        again = _kernels(*inp, G)
        assert all(torch.equal(a, b) for a, b in zip(first, again))


@pytest.mark.parametrize("B,HW,C", KERNEL_SHAPES)
@pytest.mark.parametrize("G", GROUP_COUNTS)
def test_large_offset_keeps_the_bounds(B, HW, C, G):
    """A convolution output 10^3 above zero with unit spread: the statistics must not cancel (E[y^2] - E[y]^2 would lose
    every digit of the variance in fp32)."""
    y, gamma, beta, r, dout = _kernel_inputs(B, HW, C, 1e3, 5 + G, True)
    out, mean, rstd, dy, dres, dgamma, dbeta = _kernels(y, gamma, beta, r, dout, G)
    torch.cuda.synchronize()
    y64 = y.double().permute(0, 3, 1, 2).requires_grad_()
    g64, b64 = gamma.double().requires_grad_(), beta.double().requires_grad_()
    ref = F.elu(F.group_norm(y64, G, g64, b64, EPS) + r.double().permute(0, 3, 1, 2))
    ref.backward(dout.double().permute(0, 3, 1, 2))
    tag = "offset B=%d HW=%d C=%d G=%d" % (B, HW, C, G)
    _check("out", out.permute(0, 3, 1, 2), ref.detach(), OUT_TOL, tag)
    _check("dy", dy.permute(0, 3, 1, 2), y64.grad, DX_TOL, tag)
    _check("dgamma", dgamma, g64.grad, DGB_TOL, tag)
    _check("dbeta", dbeta, b64.grad, DGB_TOL, tag)
    yg = y.double().view(B, HW, G, C // G)
    _check("mean", mean, yg.mean(dim=(1, 3)), 1e-6, tag)
    _check("rstd", rstd, (yg.var(dim=(1, 3), unbiased=False) + EPS).rsqrt(), 1e-3, tag)


# ------------------------------------------------------------------------------------------------ 3. whole step
def _resnet_pair(seed, G=32):
    torch.manual_seed(seed)
    a = models.ResNet18(norm="group", groups=G).to(DEV)
    with torch.no_grad():
        for m in a.modules():
            if isinstance(m, nn.GroupNorm):
                m.weight.copy_(1.0 + 0.2 * torch.randn_like(m.weight))
                m.bias.copy_(0.2 * torch.randn_like(m.bias))
    b = models.ResNet18(norm="group", groups=G).to(DEV)
    b.load_state_dict(a.state_dict())
    b.double()
    arena = FlatArena(a, channels_last_weights=True)
    return a, b, arena


def _batch(B, seed):
    g = torch.Generator(device=DEV).manual_seed(seed + B)
    x = torch.randn(B, 3, 32, 32, device=DEV, generator=g).contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 10, (B,), device=DEV, generator=g)
    return x, y


def _fast_step(a, arena, x, y):
    arena.zero_grads()
    with cuda_ops.accumulate_into_grad():
        loss = cuda_ops.cross_entropy(a(x), y)
        loss.backward()
    return loss.detach()


def _reference_step(b, x, y):
    for p in b.parameters():
        p.grad = None
    FX.set_fast_path(False)
    try:
        loss = F.cross_entropy(b(x.double()), y)
        loss.backward()
    finally:
        FX.set_fast_path(True)
    return loss.detach(), [p.grad for p in b.parameters()]


def _check_grads(a, ref_grads, tag):
    errs = []
    for (n, p), g in zip(a.named_parameters(), ref_grads):
        if not p.requires_grad:
            assert p.grad is None, n
            continue
        errs.append(_check("grad", p.grad, g, GRAD_TOL, "%s %s" % (n, tag)))
        e = l2_err(p.grad, g)
        assert e < GRAD_L2_TOL, "grad %s %s: relative L2 error %.3g >= %.3g" % (n, tag, e, GRAD_L2_TOL)
    return max(errs)


@functools.lru_cache(maxsize=None)
def _model_case(B):
    a, b, arena = _resnet_pair(5)
    x, y = _batch(B, 5)
    unfreeze_all_layers(b)
    loss, grads = _reference_step(b, x, y)
    return a, arena, x, y, loss, grads


@pytest.mark.parametrize("B", BATCHES)
@pytest.mark.parametrize("block", [0, 3, 7, 9, "all"])
def test_resnet18_gn_step_matches_float64(block, B):
    a, arena, x, y, ref_loss, ref_grads = _model_case(B)
    if block == "all":
        unfreeze_all_layers(a)
    else:
        unfreeze_one_block(a, block)
    loss = _fast_step(a, arena, x, y)
    torch.cuda.synchronize()
    _check("loss", loss, ref_loss, LOSS_TOL)
    _check_grads(a, ref_grads, "block %s B=%d" % (block, B))


@pytest.mark.parametrize("block", [0, "all"])
def test_graphed_step_matches_eager_step(block):
    a, arena, x, y, ref_loss, ref_grads = _model_case(128)
    if block == "all":
        unfreeze_all_layers(a)
    else:
        unfreeze_one_block(a, block)
    eager_loss = _fast_step(a, arena, x, y)
    eager = [p.grad.detach().clone() if p.grad is not None else None for p in a.parameters()]

    def body():
        return _fast_step(a, arena, x, y)

    for _ in range(2):             # the derived-filter caches exist before the capture
        body()
    graph, loss_out = capture_graph(torch.cuda.Stream(), body)
    arena.grad.fill_(float("nan"))
    graph.replay()
    torch.cuda.synchronize()
    _check("loss", loss_out, eager_loss.double(), LOSS_TOL, "graph vs eager")
    _check("loss", loss_out, ref_loss, LOSS_TOL, "graph")
    for (n, p), g in zip(a.named_parameters(), eager):
        if g is None:
            assert p.grad is None, n
            continue
        _check("grad", p.grad, g.double(), GRAD_TOL, "%s graph vs eager" % n)
    _check_grads(a, ref_grads, "graph block %s" % block)


GN_KERNELS = ("gn_stats_kernel", "gn_finalize_kernel", "gn_apply_kernel", "gn_bwd_reduce_kernel", "gn_bwd_merge_kernel",
              "gn_bwd_apply_kernel")


def _step_launches():
    """{kernel name: launches} of one forward + backward of ResNet18-GN at batch 128, every parameter trainable, after a
    warm-up step."""
    a, _, arena = _resnet_pair(5)
    unfreeze_all_layers(a)
    x, y = _batch(128, 5)
    _fast_step(a, arena, x, y)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        _fast_step(a, arena, x, y)
        torch.cuda.synchronize()
    counts = {}
    for e in prof.key_averages():
        counts[e.key] = counts.get(e.key, 0) + e.count
    return counts


def _launches_in_fresh_process():
    """``_step_launches()`` in a new Python process: late in a long test session the profiler has been seen to return fewer
    kernel records than the step launched (tests/test_gpu_resnet_step.py), which would make exact counts depend on what ran
    before."""
    here = os.path.dirname(os.path.abspath(__file__))
    code = ("import json, sys; sys.path[:0] = [%r, %r]; import test_gpu_groupnorm as t; print(json.dumps(t._step_launches()))"
            % (here, os.path.dirname(here)))
    flags = ["-s"] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable] + flags + ["-c", code], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


def test_step_runs_no_library_kernel():
    launches = _launches_in_fresh_process()
    names = list(launches)
    low = [n.lower() for n in names]
    banned = ("cudnn", "cublas", "cutlass", "xmma", "sgemm", "group_norm", "groupnorm", "rowwisemoments")
    assert not [n for n, l in zip(names, low) if any(b in l for b in banned)], names
    n_norm = sum(isinstance(m, nn.GroupNorm) for m in models.ResNet18(norm="group").modules())
    count = {k: sum(c for n, c in launches.items() if k in n) for k in GN_KERNELS}
    # one launch of each GroupNorm kernel per GroupNorm layer, forward and backward
    assert all(c == n_norm for c in count.values()), (n_norm, count)


# ------------------------------------------------------------------------------------------------ 4. federated run
def test_graphed_federated_run_with_co_resident_replicas():
    from federated_pytorch_test_b200.api import federated_multi

    cfg = federated_multi.Config(K=2, model="ResNet18", norm="group", Nloop=1, Nadmm=1, max_minibatches=3,
                                 train_size=2048, test_size=384, save_model=False, graphs=True, fast=True,
                                 collective="fused", distributed=False, check_results=False)
    eng = federated_multi.run(cfg, log=lambda m: None)
    torch.cuda.synchronize()
    r0, r1 = eng.replicas
    assert isinstance(r0.nets["net"].bn1, nn.GroupNorm)
    assert torch.equal(r0.arenas["net"].data, r1.arenas["net"].data)
    assert all(rep.running_loss == rep.running_loss and abs(rep.running_loss) < float("inf") for rep in eng.replicas)
    # eval_bn has no effect on GroupNorm: train-mode and eval-mode evaluation give the same accuracies
    task = eng.task
    batch = task.evaluate(eng.replicas, eng)
    task.cfg.eval_bn = "running"
    running = task.evaluate(eng.replicas, eng)
    assert batch == running and all(0.0 <= a <= 100.0 for a in batch)
