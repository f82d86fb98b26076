"""Eval-mode BatchNorm on the hand-written kernels: conv + BatchNorm(running statistics) + residual + ELU in the wgmma
epilogue (one launch), or split-K convolution + the running-statistics mode of bn_elu_fwd.  Run on an H100."""
import math

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():  # collected (and deselected) on the CPU box
    pytest.skip("CUDA device required", allow_module_level=True)

from federated_pytorch_test_b200 import models  # noqa: E402
from federated_pytorch_test_b200.ops import cuda_ops  # noqa: E402
from federated_pytorch_test_b200.ops import functional as FX  # noqa: E402

DEV = torch.device("cuda", 0)
_LIB = ("cudnn", "cutlass", "cublas", "sgemm", "xmma", "implicit_gemm", "gemv", "gemmk1")


@pytest.fixture(autouse=True)
def _exact_reference_math(monkeypatch):
    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    monkeypatch.delenv("FEDB200_SPLITK", raising=False)
    FX.set_fast_path(True)
    yield
    FX.set_fast_path(True)
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def rel_err(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-12))


def _group(cin, cout, k, stride, seed):
    """conv + eval-mode BatchNorm with running statistics far from (0, 1)."""
    g = torch.Generator().manual_seed(seed)
    conv = nn.Conv2d(cin, cout, k, stride=stride, padding=k // 2, bias=False)
    bn = nn.BatchNorm2d(cout)
    with torch.no_grad():
        conv.weight.copy_(torch.randn(conv.weight.shape, generator=g) / math.sqrt(cin * k * k))
        bn.weight.copy_(1.0 + 0.3 * torch.randn(cout, generator=g))
        bn.bias.copy_(0.5 * torch.randn(cout, generator=g))
        bn.running_mean.copy_(1.5 * torch.randn(cout, generator=g) + 0.7)
        bn.running_var.copy_(0.05 + 4.0 * torch.rand(cout, generator=g))
    return conv.to(DEV), bn.to(DEV).eval()


def _oracle(x, conv, bn, res, act):
    y = F.conv2d(x.double(), conv.weight.double(), None, conv.stride, conv.padding)
    y = F.batch_norm(y, bn.running_mean.double(), bn.running_var.double(), bn.weight.double(), bn.bias.double(), False, 0.0, bn.eps)
    if res is not None:
        y = y + res.double()
    return F.elu(y) if act else y


# (cin, cout, k, stride, H, act): stem, layer-1 3x3, layer-2 entry, 1x1 stride-2 shortcut (no ELU), layer-4 entry and 3x3
SHAPES = [(3, 64, 3, 1, 32, True), (64, 64, 3, 1, 32, True), (64, 128, 3, 2, 32, True), (64, 128, 1, 2, 32, False),
          (256, 512, 3, 2, 8, True), (512, 512, 3, 1, 4, True)]


def _check_group(cin, cout, k, stride, H, act, B, with_res):
    conv, bn = _group(cin, cout, k, stride, seed=cin + cout + k + stride + H)
    g = torch.Generator(device=DEV).manual_seed(B + cin)
    x = torch.randn(B, cin, H, H, device=DEV, generator=g).contiguous(memory_format=torch.channels_last)
    Ho = (H + 2 * (k // 2) - k) // stride + 1
    res = torch.randn(B, cout, Ho, Ho, device=DEV, generator=g).contiguous(memory_format=torch.channels_last) if with_res else None
    state = [t.clone() for t in (bn.running_mean, bn.running_var, bn.num_batches_tracked)]
    with torch.no_grad():
        assert cuda_ops.conv_bn_act_eval_supported(x, conv, bn, res)
        before = cuda_ops.launch_count()
        out = FX.conv_bn_act(x, conv, bn, res, act)
        launches = cuda_ops.launch_count() - before
        ref = _oracle(x, conv, bn, res, act)
    err = rel_err(out, ref)
    assert err < 5e-3, err
    for a, b in zip(state, (bn.running_mean, bn.running_var, bn.num_batches_tracked)):
        assert torch.equal(a, b)
    return launches


@pytest.mark.parametrize("with_res", [False, True], ids=["plain", "residual"])
@pytest.mark.parametrize("B", [128, 16])
@pytest.mark.parametrize("cin,cout,k,stride,H,act", SHAPES)
def test_conv_bn_eval_matches_fp64_oracle(cin, cout, k, stride, H, act, B, with_res):
    launches = _check_group(cin, cout, k, stride, H, act, B, with_res)
    assert launches in (1, 2)
    if H // stride == 4 and B == 128:
        assert launches == 2, "layer-4 shapes at batch 128 run as split-K convolution + running-statistics pass"


@pytest.mark.parametrize("with_res", [False, True], ids=["plain", "residual"])
@pytest.mark.parametrize("B", [128, 16])
@pytest.mark.parametrize("cin,cout,k,stride,H,act", [s for s in SHAPES if s[4] // s[3] == 4])
def test_conv_bn_eval_single_launch_branch(monkeypatch, cin, cout, k, stride, H, act, B, with_res):
    monkeypatch.setenv("FEDB200_SPLITK", "1")
    assert _check_group(cin, cout, k, stride, H, act, B, with_res) == 1


def test_bn_elu_fwd_running_mode_matches_oracle():
    e = cuda_ops.ext()
    g = torch.Generator(device=DEV).manual_seed(3)
    M, C = 1000, 96
    y, r = torch.randn(M, C, device=DEV, generator=g), torch.randn(M, C, device=DEV, generator=g)
    gamma, beta = torch.randn(C, device=DEV, generator=g), torch.randn(C, device=DEV, generator=g)
    rm, rv = torch.randn(C, device=DEV, generator=g), torch.rand(C, device=DEV, generator=g) + 0.1
    rm0, rv0 = rm.clone(), rv.clone()
    out, sm, si = e.bn_elu_fwd(y, None, gamma, beta, r, rm, rv, 1e-5, 0.1, True, False, True)
    assert sm is None and si is None
    ref = F.elu((y - rm) / torch.sqrt(rv + 1e-5) * gamma + beta + r)
    torch.testing.assert_close(out, ref, rtol=1e-5, atol=1e-5)
    assert torch.equal(rm, rm0) and torch.equal(rv, rv0)


# ------------------------------------------------------------------------------------------ whole models
@pytest.mark.parametrize("name", ["ResNet18", "ResNet9"])
def test_eval_forward_matches_golden_and_aten(golden, fill, name):
    net = fill(getattr(models, name)()).to(DEV).eval()
    x = torch.randn(4, 3, 32, 32, generator=torch.Generator().manual_seed(1)).to(DEV)
    with torch.no_grad():
        before = cuda_ops.launch_count()
        y = net(x)
        assert cuda_ops.launch_count() > before
        assert rel_err(y.cpu(), golden["forward"][name]["y"]) < 1e-2
        xb = torch.randn(128, 3, 32, 32, device=DEV, generator=torch.Generator(device=DEV).manual_seed(2))
        xb = xb.contiguous(memory_format=torch.channels_last)
        fast = net(xb)
        FX.set_fast_path(False)
        aten = net(xb)
        FX.set_fast_path(True)
    assert rel_err(fast, aten) < 1e-2


def test_eval_forward_leaves_state_and_training_path_intact():
    torch.manual_seed(0)
    a, b = models.ResNet9().to(DEV), models.ResNet9().to(DEV)
    b.load_state_dict(a.state_dict())
    x = torch.randn(16, 3, 32, 32, device=DEV).contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 10, (16,), device=DEV)
    # one training step first, so that the fast path's cached statistics buffers exist
    for net, fast in ((a, True), (b, False)):
        FX.set_fast_path(fast)
        F.cross_entropy(net(x), y).backward()
    FX.set_fast_path(True)
    bufs = {k: v.clone() for k, v in a.named_buffers()}
    a.eval()
    with torch.no_grad():
        a(x)
    a.train()
    for k, v in a.named_buffers():
        assert torch.equal(v, bufs[k]), k
    for net in (a, b):
        net.zero_grad()
    b.load_state_dict(a.state_dict())
    la = F.cross_entropy(a(x), y)
    la.backward()
    FX.set_fast_path(False)
    lb = F.cross_entropy(b(x), y)
    lb.backward()
    FX.set_fast_path(True)
    assert float(la) == pytest.approx(float(lb), rel=1e-3)
    for (n, pa), (_, pb) in zip(a.named_parameters(), b.named_parameters()):
        assert rel_err(pa.grad, pb.grad) < 1e-2, n
    for (n, ba), (_, bb) in zip(a.named_buffers(), b.named_buffers()):
        if "num_batches" not in n:
            torch.testing.assert_close(ba, bb, rtol=5e-3, atol=5e-4, msg=n)


def test_resnet18_eval_forward_uses_no_library_kernels_and_one_launch_per_group(monkeypatch):
    torch.manual_seed(0)
    net = models.ResNet18().to(DEV).eval()
    x = torch.rand(128, 3, 32, 32, device=DEV).contiguous(memory_format=torch.channels_last)
    with torch.no_grad():
        net(x)
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            net(x)
            torch.cuda.synchronize()
        names = [e.key for e in prof.key_averages()]
        lib = [n for n in names if any(t in n.lower() for t in _LIB)]
        assert not lib, lib
        assert any("igemm_wgmma" in n for n in names)
        monkeypatch.setenv("FEDB200_SPLITK", "1")
        before = cuda_ops.launch_count()
        net(x)
        assert cuda_ops.launch_count() - before == 21      # 20 conv + BatchNorm (+ residual) (+ ELU) groups + the fused head


def test_engine_running_eval_graphed_eager_and_aten_agree(monkeypatch):
    """federated_multi with ``eval_bn='running'``: at every evaluation the same networks are also evaluated eagerly on the
    fast path and on the ATen path; graphed and eager counts are identical, ATen agrees within 1 % of the test images, and the
    BatchNorm buffers do not move."""
    from federated_pytorch_test_b200.api import common, federated_multi
    from federated_pytorch_test_b200.config import override

    seen = []
    original = common.ClassifierTask.evaluate

    def watched(self, reps, engine):
        bufs = [{k: v.clone() for k, v in r.nets["net"].named_buffers()} for r in reps]
        graphed = original(self, reps, engine)
        cfg = self.cfg
        try:
            self.cfg = override(cfg, graphs=False)
            eager = original(self, reps, engine)
            FX.set_fast_path(False)
            aten = original(self, reps, engine)
        finally:
            FX.set_fast_path(True)
            self.cfg = cfg
        for r, b in zip(reps, bufs):
            for k, v in r.nets["net"].named_buffers():
                assert torch.equal(v, b[k]), k
        seen.append((graphed, eager, aten))
        return graphed

    monkeypatch.setattr(common.ClassifierTask, "evaluate", watched)
    test_size = 512
    cfg = federated_multi.Config(K=2, model="ResNet9", Nloop=1, Nadmm=1, max_minibatches=3, check_results=True, save_model=False,
                                 train_size=4096, test_size=test_size, default_batch=128, eval_bn="running", graphs=True)
    eng = federated_multi.run(cfg, log=lambda s: None)
    assert len(seen) == len(eng.task.blocks)                   # one evaluation per aggregation round
    assert any(key[2] is False for key in eng.task._eval_graphs), "no eval-mode graph was captured"
    for graphed, eager, aten in seen:
        assert graphed == eager
        for a, b in zip(eager, aten):
            assert abs(a - b) * test_size / 100.0 <= 0.01 * test_size
