"""The batch-128 ResNet18 training step as training runs it, against float64 ATen.

1. Every distinct conv + BatchNorm (+ residual) (+ ELU) group of ResNet18 through ``cuda_ops.conv_bn_act`` at batch 128 and
   at batch 105 (the partial last batch of a 6249-sample shard), with a trainable weight whose channels-last gradient buffer is
   pre-filled (``accumulate_into_grad``) and with a frozen weight whose data gradient runs on the cached derived filter.  Each
   case runs three times on the same inputs: the self-cleaning BatchNorm scratch buffers must leave every call exact.
2. The kernels those steps launch: the window-reuse pixel-major kernel for layer 1, the per-tap 128-channel pixel-major kernel
   for layer 2, the wgmma weight gradient, as ``conv_orientation`` / ``conv_window_reuse`` predict for this GPU.
3. The whole step (loss and every parameter gradient) with one block trainable at a time, and with all parameters.
4. The rotated / phase-packed filters of frozen layers, cached at stable addresses, after the weights of those layers change
   in place and ``refresh_caches`` runs (the start of a block visit), eagerly and through a captured CUDA graph.

Oracles: ``F.conv2d`` -> ``F.batch_norm(training=True)`` -> ``+ residual`` -> ``F.elu`` in float64, and the model ``.double()``
on the ATen path.  Errors are max |got - ref| / max |ref| per tensor ("max-normalised"), plus |got - ref|_2 / |ref|_2 for the
whole model.  Worst values over two runs on an H100 80GB HBM3 (SXM, 132 SMs, 700 W power limit), and the bounds (about 3x):

    check                                  worst     bound
    1. output                              3.9e-4    1e-3
       running_mean / running_var          1.1e-3    3e-3  /  8.4e-5   2.5e-4
       dx                                  3.9e-4    1e-3
       dW (gradient buffer - pre-fill)     4.4e-4    1.2e-3
       dgamma / dbeta                      4.2e-4    1.2e-3
       d(residual)                         7.8e-4    2e-3
    3. loss                                1.3e-5    4e-5
       gradients, max-normalised           3.5e-3    1e-2
       gradients, relative L2              2.9e-3    8e-3
    4. loss                                1.2e-5    4e-5
       stem gradients, max-normalised      3.7e-3    1e-2

The file takes about 50 s on that GPU, 33 s of it the two fresh processes of part 2.  Run on an H100: ``python -m pytest tests -m gpu``."""
import functools
import json
import os
import re
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
PIXEL = 1                      # ext().conv_orientation: pixel-major tiles
BATCHES = (128, 105)

# bounds: about 3x the worst value measured (module docstring)
OUT_TOL = 1e-3
DW_TOL = 1.2e-3
DX_TOL = 1e-3
DGB_TOL = 1.2e-3               # dgamma and dbeta
DRES_TOL = 2e-3
RUNNING_MEAN_TOL = 3e-3
RUNNING_VAR_TOL = 2.5e-4
LOSS_TOL = 4e-5
GRAD_TOL = 1e-2                # whole model, max-normalised per tensor
GRAD_L2_TOL = 8e-3             # whole model, relative L2 per tensor


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


def _check_l2(kind, got, ref, bound, name=""):
    e = l2_err(got, ref)
    assert e < bound, "%s %s: relative L2 error %.3g >= %.3g" % (kind, name, e, bound)


def _krsc_key(weight):
    """Key of a filter in the derived-filter caches: address and shape of its [C_out, kh, kw, C_in] view."""
    wk = weight.detach().permute(0, 2, 3, 1)
    return wk.data_ptr(), tuple(wk.shape)


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

MOMENTUM, EPS = 0.1, 1e-5
CALLS = 3


@functools.lru_cache(maxsize=1)
def _group_case(name, B):
    """Seeded fp32 inputs of one group and what float64 ATen computes from them (one and ``CALLS`` running-stat updates)."""
    ci, co, h, k, s, res, act = GROUPS[name]
    g = torch.Generator(device=DEV).manual_seed(1000 * B + sum(map(ord, name)))
    x = torch.randn(B, ci, h, h, device=DEV, generator=g)
    if name != "stem":       # block inputs are ELU outputs: a per-channel mean the running statistics can see
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
    rm, rv = torch.zeros(co, dtype=torch.float64, device=DEV), torch.ones(co, dtype=torch.float64, device=DEV)
    y = F.conv2d(x64, w64, None, s, k // 2)
    u = F.batch_norm(y, rm, rv, g64, b64, True, MOMENTUM, EPS)
    if res:
        u = u + r64
    out = F.elu(u) if act else u
    out.backward(dout.double())
    running = [(rm.clone(), rv.clone())]
    with torch.no_grad():
        for _ in range(CALLS - 1):
            F.batch_norm(y, rm, rv, None, None, True, MOMENTUM, EPS)
            running.append((rm.clone(), rv.clone()))
    ref = dict(out=out.detach(), dx=x64.grad, dw=w64.grad, dgamma=g64.grad, dbeta=b64.grad, dres=r64.grad if res else None,
               running=running)
    return inp, ref


def _group_modules(inp, k, s, trainable):
    """The conv / BatchNorm pair of one group, the filter stored channels-last as FlatArena(channels_last_weights=True) stores
    it (so the glue's [C_out, kh, kw, C_in] view aliases the parameter and a frozen filter is cached by address)."""
    co, ci = inp["w"].shape[:2]
    conv = nn.Conv2d(ci, co, k, s, k // 2, bias=False).to(DEV)
    bn = nn.BatchNorm2d(co, momentum=MOMENTUM, eps=EPS).to(DEV)
    with torch.no_grad():
        conv.weight = nn.Parameter(inp["w"].contiguous(memory_format=torch.channels_last), requires_grad=trainable)
        bn.weight.copy_(inp["gamma"])
        bn.bias.copy_(inp["beta"])
    return conv, bn


GROUP_CASES = [(n, B, m) for n in GROUPS for B in BATCHES for m in ("trainable", "frozen")]


@pytest.mark.parametrize("name,B,mode", GROUP_CASES)
def test_group_matches_float64_and_repeats(name, B, mode):
    ci, co, h, k, s, res, act = GROUPS[name]
    inp, ref = _group_case(name, B)
    trainable = mode == "trainable"
    conv, bn = _group_modules(inp, k, s, trainable)
    x = inp["x"].detach().requires_grad_()
    r = inp["r"].detach().requires_grad_() if res else None
    assert cuda_ops.conv_bn_act_supported(x, conv, bn)
    prefill = None
    if trainable:
        # the gradient arena's layout: a contiguous [C_out, kh, kw, C_in] buffer seen as the logical [C_out, C_in, kh, kw] .grad,
        # holding what earlier backward calls accumulated (of the size of one gradient, so an overwrite cannot pass)
        gen = torch.Generator(device=DEV).manual_seed(B + co)
        prefill = torch.randn(co, k, k, ci, device=DEV, generator=gen).permute(0, 3, 1, 2) * float(ref["dw"].abs().max())
        conv.weight.grad = prefill.clone()
        assert conv.weight.grad.permute(0, 2, 3, 1).is_contiguous()
    for call in range(CALLS):
        x.grad = None
        if r is not None:
            r.grad = None
        bn.weight.grad = bn.bias.grad = None
        if trainable:
            conv.weight.grad.copy_(prefill)            # in place: the buffer the kernel accumulates into stays the same
        with cuda_ops.accumulate_into_grad():
            out = cuda_ops.conv_bn_act(x, conv, bn, residual=r, act=act)
            out.backward(inp["dout"])
        torch.cuda.synchronize()
        tag = "call %d" % call
        _check("out", out, ref["out"], OUT_TOL, tag)
        rm, rv = ref["running"][call]
        _check("running_mean", bn.running_mean, rm, RUNNING_MEAN_TOL, tag)
        _check("running_var", bn.running_var, rv, RUNNING_VAR_TOL, tag)
        _check("dx", x.grad, ref["dx"], DX_TOL, tag)
        _check("dgamma", bn.weight.grad, ref["dgamma"], DGB_TOL, tag)
        _check("dbeta", bn.bias.grad, ref["dbeta"], DGB_TOL, tag)
        if res:
            _check("dres", r.grad, ref["dres"], DRES_TOL, tag)
        if trainable:
            _check("dW", conv.weight.grad.double() - prefill.double(), ref["dw"], DW_TOL, tag)
        else:
            assert conv.weight.grad is None
    if not trainable and ci % 4 == 0:
        # the data gradient really ran on the cached filter (the stem's is channel-padded, a transient, never cached)
        cache = cuda_ops._S2_CACHE if s == 2 else cuda_ops._FLIP_CACHE
        assert _krsc_key(conv.weight) in cache


# ------------------------------------------------------------------------------------------------ shared model set-up
def _resnet_pair(seed):
    """(fast ResNet18 on a channels-last FlatArena, the same network in float64 for the ATen path).  BatchNorm affine
    parameters are drawn away from 1 / 0 so that a gamma / beta mix-up cannot hide."""
    torch.manual_seed(seed)
    a = models.ResNet18().to(DEV)
    with torch.no_grad():
        for m in a.modules():
            if isinstance(m, nn.BatchNorm2d):
                m.weight.copy_(1.0 + 0.2 * torch.randn_like(m.weight))
                m.bias.copy_(0.2 * torch.randn_like(m.bias))
    b = models.ResNet18().to(DEV)
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
    """Loss and gradients of the float64 model on the ATen path (only the parameters that require a gradient get one)."""
    for p in b.parameters():
        p.grad = None
    FX.set_fast_path(False)
    try:
        loss = F.cross_entropy(b(x.double()), y)
        loss.backward()
    finally:
        FX.set_fast_path(True)
    return loss.detach(), [p.grad for p in b.parameters()]


# ------------------------------------------------------------------------------------------------ 2. routes
_PIX = re.compile(r"igemm_wgmma_pix_kernel<(\d+), *(\d+), *(\d+)>")


def _step_launches(B):
    """{kernel name: launches} of one forward + backward of ResNet18 at batch ``B``, every parameter trainable, after a
    warm-up step."""
    a, _, arena = _resnet_pair(3)
    unfreeze_all_layers(a)
    x, y = _batch(B, 3)
    _fast_step(a, arena, x, y)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        _fast_step(a, arena, x, y)
        torch.cuda.synchronize()
    counts = {}
    for e in prof.key_averages():
        name = e.key.split("(")[0]
        counts[name] = counts.get(name, 0) + e.count
    return counts


def _launches_in_fresh_process(B):
    """``_step_launches(B)`` in a new Python process.  Late in a long test session the profiler has been seen to return fewer
    kernel records than the step launched (same launch calls, the data gradients of a few layers missing), which makes
    exact counts depend on what ran before; a fresh process profiles exactly."""
    here = os.path.dirname(os.path.abspath(__file__))
    code = ("import json, sys; sys.path[:0] = [%r, %r]; import test_gpu_resnet_step as t; print(json.dumps(t._step_launches(%d)))"
            % (here, os.path.dirname(here), B))
    flags = ["-s"] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable] + flags + ["-c", code], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


def _pix_launches(launches, c_out, window):
    """Launches of the pixel-major kernel with ``c_out`` output channels, window-reuse loop or per-tap loop."""
    n = 0
    for key, count in launches.items():
        m = _PIX.search(key)
        if m and int(m.group(1)) == c_out and (int(m.group(3)) > 0) == window:
            n += count
    return n


@pytest.mark.parametrize("B", BATCHES)
def test_training_step_runs_the_pixel_major_and_weight_gradient_kernels(B):
    """Forward + backward of ResNet18, every parameter trainable.  Layer 1 (64 channels, 32 x 32): four convolutions forward
    and four data gradients (rotated filter, stride 1).  Layer 2 (128 channels, 16 x 16): conv1 (stride 2), the 1 x 1 shortcut,
    three stride-1 convolutions forward, and the data gradients of those three (the stride-2 ones run the phase-packed
    row-major convolution).  Every convolution's weight gradient runs on the wgmma kernel."""
    e = cuda_ops.ext()
    launches = _launches_in_fresh_process(B)
    fedb = {k: c for k, c in launches.items() if "igemm" in k or "wgrad" in k}
    assert any(_PIX.search(k) for k in launches), "no pixel-major kernel among %s" % fedb

    l1 = e.conv_orientation(B, 32, 32, 64, 1) == PIXEL
    window = l1 and e.conv_window_reuse(32, 32, 64, 64, 3, 1, 1)
    l2_fwd = sum(e.conv_orientation(B, 16, 16, 128, s) == PIXEL for s in (2, 2, 1, 1, 1))
    l2_dgrad = 3 * int(e.conv_orientation(B, 16, 16, 128, 1) == PIXEL)
    assert _pix_launches(launches, 64, True) == (8 if window else 0), fedb
    assert _pix_launches(launches, 128, False) == l2_fwd + l2_dgrad, fedb
    n_conv = sum(isinstance(m, nn.Conv2d) for m in models.ResNet18().modules())
    assert sum(c for k, c in launches.items() if "wgrad_wgmma_kernel" in k) == n_conv, fedb
    if B == 128:
        # the routes parts 1 and 3 exist to cover: a heuristic change that leaves them must show up here
        assert window and l2_fwd == 5 and l2_dgrad == 3


# ------------------------------------------------------------------------------------------------ 3. whole step
@functools.lru_cache(maxsize=None)
def _model_case(B):
    a, b, arena = _resnet_pair(5)
    x, y = _batch(B, 5)
    unfreeze_all_layers(b)
    loss, grads = _reference_step(b, x, y)      # a parameter's gradient does not depend on which others are frozen
    return a, arena, x, y, loss, grads


@pytest.mark.parametrize("B", BATCHES)
@pytest.mark.parametrize("block", [0, 3, 7, 9, "all"])
def test_resnet18_step_matches_float64(block, B):
    a, arena, x, y, ref_loss, ref_grads = _model_case(B)
    if block == "all":
        unfreeze_all_layers(a)
    else:
        unfreeze_one_block(a, block)
    loss = _fast_step(a, arena, x, y)
    torch.cuda.synchronize()
    _check("loss", loss, ref_loss, LOSS_TOL)
    names = [n for n, _ in a.named_parameters()]
    for n, p, g in zip(names, a.parameters(), ref_grads):
        if not p.requires_grad:
            assert p.grad is None, n
            continue
        _check("grad", p.grad, g, GRAD_TOL, n)
        _check_l2("grad", p.grad, g, GRAD_L2_TOL, n)


# ------------------------------------------------------------------------------------------------ 4. derived-filter caches
def _overwrite(arena, p, gen):
    """New values for parameter ``p``, written in place into its slot of the arena's flat buffer (where the FedAvg write-back
    puts them); returns them as a logical tensor."""
    i = next(j for j, q in enumerate(arena.params) if q is p)
    new = torch.randn(p.shape, device=DEV, generator=gen) * float(p.detach().std())
    with torch.no_grad():
        arena.data[arena.offsets[i]: arena.offsets[i] + p.numel()].copy_(new.permute(0, 2, 3, 1).reshape(-1))
    return new


@pytest.mark.parametrize("graphed", [False, True], ids=["eager", "graph"])
def test_frozen_filter_caches_follow_weights_across_visits(graphed):
    a, b, arena = _resnet_pair(7)
    unfreeze_one_block(a, 0)           # the bench configuration: the stem trains, the data gradient crosses every frozen layer
    unfreeze_one_block(b, 0)
    x, y = _batch(128, 7)
    mods_a, mods_b = dict(a.named_modules()), dict(b.named_modules())
    stem = [n for n, p in a.named_parameters() if p.requires_grad]
    assert stem == ["conv1.weight", "bn1.weight", "bn1.bias"]

    if graphed:
        def body():
            return _fast_step(a, arena, x, y)

        for _ in range(2):             # eager warm-up: the caches and the per-layer scratch exist before the capture
            body()
        graph, loss_out = capture_graph(torch.cuda.Stream(), body)

        def step():
            graph.replay()
            return loss_out
    else:
        def step():
            return _fast_step(a, arena, x, y)

    def check(stage):
        loss = step()
        torch.cuda.synchronize()
        ref_loss, ref_grads = _reference_step(b, x, y)
        _check("loss", loss, ref_loss, LOSS_TOL, "after " + stage)
        got = dict(a.named_parameters())
        for n, g in zip([n for n, _ in b.named_parameters()], ref_grads):
            if n in stem:
                _check("stem grad", got[n].grad, g, GRAD_TOL, "%s after %s" % (n, stage))
            else:
                assert got[n].grad is None, n

    check("the first step")
    # every frozen convolution keeps its derived filter at a stable address: rotated (stride 1) or phase-packed (stride 2)
    convs = [n for n, m in mods_a.items() if isinstance(m, nn.Conv2d) and n != "conv1"]
    for n in convs:
        cache = cuda_ops._S2_CACHE if mods_a[n].stride[0] == 2 else cuda_ops._FLIP_CACHE
        assert _krsc_key(mods_a[n].weight) in cache, n

    gen = torch.Generator(device=DEV).manual_seed(11)
    stages = [("layer 1", [n for n in convs if n.startswith("layer1.")]),
              ("layer2.0.conv1", ["layer2.0.conv1"]),
              ("layer 3", [n for n in convs if n.startswith("layer3.")])]
    for stage, names in stages:
        for n in names:
            new = _overwrite(arena, mods_a[n].weight, gen)
            with torch.no_grad():
                mods_b[n].weight.copy_(new.double())
        cuda_ops.refresh_caches()      # what Engine._refresh_derived runs at the start of every block visit
        check("new %s weights" % stage)
