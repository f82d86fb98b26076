"""Numerics of every hand-written sm_90a kernel against a plain PyTorch fp32 reference of the same op.
Run on an H100: ``python -m pytest tests -m gpu``."""
import math

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():  # collected (and deselected) on the CPU box
    pytest.skip("CUDA device required", allow_module_level=True)

from federated_pytorch_test_b200 import models  # noqa: E402
from federated_pytorch_test_b200.ops import cuda_ops, flatops  # noqa: E402
from federated_pytorch_test_b200.ops import functional as FX  # noqa: E402

DEV = torch.device("cuda", 0)


@pytest.fixture(autouse=True)
def _exact_reference_math():
    """The oracle runs in true fp32; the fast path is switched on per test."""
    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    FX.set_fast_path(True)
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def rel_err(a, b):
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-12))


def test_extension_is_native_and_loaded():
    e = cuda_ops.ext()
    assert e.__file__.endswith(".so") and "federated_pytorch_test_b200/_build" in e.__file__
    assert torch.cuda.get_device_capability(0) == (9, 0), "these kernels are sm_90a only"


# ------------------------------------------------------------------------------------------ flat ops
@pytest.mark.parametrize("n", [850, 5130, 73984, 1180672])
def test_adam_prox_matches_oracle(n):
    g = torch.Generator(device=DEV).manual_seed(n)
    x = torch.randn(n, device=DEV, generator=g)
    z, y = torch.randn(n, device=DEV, generator=g), torch.randn(n, device=DEV, generator=g)
    xr, m, v = x.clone(), torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
    mr, vr = m.clone(), v.clone()
    for t in range(1, 4):
        gr = torch.randn(n, device=DEV, generator=g)
        cuda_ops.adam_prox_step(x, gr, m, v, t, 1e-3, 0.9, 0.999, 1e-8, z, y, 0.3, 1e-4, 1e-4)
        FX.set_fast_path(False)
        flatops.adam_prox_step(xr, gr, mr, vr, t, 1e-3, 0.9, 0.999, 1e-8, z, y, 0.3, 1e-4, 1e-4)
        FX.set_fast_path(True)
    torch.testing.assert_close(x, xr, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(m, mr, rtol=1e-5, atol=1e-7)
    torch.testing.assert_close(v, vr, rtol=1e-4, atol=1e-8)


def test_adam_device_step_counter_and_plain_adam():
    n = 4096
    x = torch.randn(n, device=DEV)
    p = nn.Parameter(x.clone())
    opt = torch.optim.Adam([p], lr=1e-3)
    m, v, step = torch.zeros(n, device=DEV), torch.zeros(n, device=DEV), torch.zeros(1, dtype=torch.int32, device=DEV)
    for _ in range(5):
        g = torch.randn(n, device=DEV)
        p.grad = g.clone()
        opt.step()
        cuda_ops.bump_step(step)
        cuda_ops.adam_prox_step(x, g, m, v, step, 1e-3, 0.9, 0.999, 1e-8)
    assert int(step) == 5
    torch.testing.assert_close(x, p.detach(), rtol=1e-5, atol=1e-6)


def test_lbfgs_on_cuda_arena_runs_and_descends():
    from federated_pytorch_test_b200.optim import LBFGSNew
    from federated_pytorch_test_b200.utils import FlatArena
    torch.manual_seed(0)
    net = nn.Sequential(nn.Flatten(), nn.Linear(3 * 32 * 32, 64), nn.ELU(), nn.Linear(64, 10)).to(DEV)
    FlatArena(net).attach_grads()
    opt = LBFGSNew(net.parameters(), history_size=7, max_iter=4, line_search_fn=True, batch_mode=True)
    x, y = torch.randn(64, 3, 32, 32, device=DEV), torch.randint(0, 10, (64,), device=DEV)
    losses = []
    for _ in range(6):
        def closure():
            if torch.is_grad_enabled():
                opt.zero_grad()
            loss = F.cross_entropy(net(x), y)
            if loss.requires_grad:
                loss.backward()
            return loss
        losses.append(float(opt.step(closure)))
    assert opt._v().fused and losses[-1] < losses[0]


# ------------------------------------------------------------------------------------------ input
def test_normalize_u8():
    u8 = torch.randint(0, 256, (16, 32, 32, 3), dtype=torch.uint8, device=DEV)
    mean, std = (0.53, 0.47, 0.5), (0.53, 0.47, 0.5)
    ref = (u8.float() / 255 - torch.tensor(mean, device=DEV)) / torch.tensor(std, device=DEV)
    a = cuda_ops.normalize_u8(u8, mean, std, channels_last=False)
    torch.testing.assert_close(a, ref.permute(0, 3, 1, 2).contiguous(), rtol=1e-5, atol=1e-5)
    b = cuda_ops.normalize_u8(u8, mean, std, channels_last=True)
    assert b.shape == (16, 3, 32, 32) and b.is_contiguous(memory_format=torch.channels_last)
    torch.testing.assert_close(b.contiguous(), ref.permute(0, 3, 1, 2).contiguous(), rtol=1e-5, atol=1e-5)


# ------------------------------------------------------------------------------------------ tensor cores
@pytest.mark.parametrize("M,N,K", [(128, 10, 512), (128, 120, 400), (1280, 128, 384), (300, 64, 100), (4096, 256, 1024)])
@pytest.mark.parametrize("act", [False, True])
def test_linear_tf32_tcgen05(M, N, K, act):
    g = torch.Generator(device=DEV).manual_seed(M + N + K)
    x = torch.randn(M, K, device=DEV, generator=g)
    w = torch.randn(N, K, device=DEV, generator=g) / math.sqrt(K)
    b = torch.randn(N, device=DEV, generator=g)
    out = cuda_ops.linear_tf32(x, w, b, act)
    ref = F.linear(x.double(), w.double(), b.double())
    ref = (F.elu(ref) if act else ref).float()
    assert out.shape == ref.shape
    assert rel_err(out, ref) < 3e-3, "tf32 tensor-core GEMM deviates from the fp64 oracle"


CONVS = [  # (B, H, Cin, Cout, k, stride, pad)   -- every distinct ResNet18 site of SURVEY §2.10(a), small batch
    (4, 32, 4, 64, 3, 1, 1), (4, 32, 64, 64, 3, 1, 1), (4, 32, 64, 128, 3, 2, 1), (4, 16, 128, 128, 3, 1, 1),
    (4, 32, 64, 128, 1, 2, 0), (8, 16, 128, 256, 3, 2, 1), (8, 8, 256, 256, 3, 1, 1), (8, 16, 128, 256, 1, 2, 0),
    (16, 8, 256, 512, 3, 2, 1), (16, 4, 512, 512, 3, 1, 1), (16, 8, 256, 512, 1, 2, 0), (13, 4, 512, 512, 3, 1, 1),
]


@pytest.mark.parametrize("B,H,Ci,Co,k,s,p", CONVS)
def test_conv2d_nhwc_tcgen05(B, H, Ci, Co, k, s, p):
    g = torch.Generator(device=DEV).manual_seed(B * H + Ci + Co + k + s)
    x = torch.randn(B, H, H, Ci, device=DEV, generator=g)
    w = torch.randn(Co, k, k, Ci, device=DEV, generator=g) / math.sqrt(k * k * Ci)
    stats = torch.zeros(2 * Co, device=DEV)
    y = cuda_ops.conv2d_nhwc(x, w, stats, s, p)
    ref = F.conv2d(x.permute(0, 3, 1, 2).double(), w.permute(0, 3, 1, 2).double(), None, s, p).permute(0, 2, 3, 1).float()
    assert y.shape == ref.shape
    assert rel_err(y, ref) < 3e-3
    flat = ref.reshape(-1, Co)
    torch.testing.assert_close(stats[:Co], flat.sum(0), rtol=2e-3, atol=2e-2 * math.sqrt(flat.shape[0]))
    torch.testing.assert_close(stats[Co:], (flat * flat).sum(0), rtol=5e-3, atol=1e-2)


@pytest.mark.parametrize("B,H,Ci,Co,k,p", [(4, 32, 64, 128, 3, 1), (8, 16, 128, 256, 3, 1), (16, 8, 256, 512, 3, 1),
                                         (4, 32, 64, 128, 1, 0), (16, 8, 256, 512, 1, 0)])
def test_stride2_data_gradient_as_one_stride1_conv(B, H, Ci, Co, k, p):
    """dgrad of the stride-2 sites = 2x2 stride-1 implicit GEMM over dy with the phase-packed filter + pixel shuffle."""
    e = cuda_ops.ext()
    g = torch.Generator(device=DEV).manual_seed(H + Ci + k)
    x = torch.randn(B, H, H, Ci, device=DEV, generator=g)
    w = torch.randn(Co, k, k, Ci, device=DEV, generator=g) / math.sqrt(k * k * Ci)
    dy = torch.randn(B, H // 2, H // 2, Co, device=DEV, generator=g)
    assert cuda_ops._s2_dgrad_supported(e, x, dy, k, k, p)
    dx = cuda_ops._s2_dgrad(e, dy, w, True)
    ref = torch.ops.aten.convolution_backward(
        dy.permute(0, 3, 1, 2).double(), x.permute(0, 3, 1, 2).double(), w.permute(0, 3, 1, 2).double(), None,
        [2, 2], [p, p], [1, 1], False, [0, 0], 1, [True, False, False])[0].permute(0, 2, 3, 1).float()
    assert dx.shape == ref.shape
    assert rel_err(dx, ref) < 3e-3


# ------------------------------------------------------------------------------------------ BN + ELU
@pytest.mark.parametrize("C,M,res,act", [(64, 4096, False, True), (128, 2048, True, True), (512, 256, True, False), (12, 777, False, True),
                                          (256, 8192, False, True), (64, 131072, True, True)])
def test_bn_elu_forward_backward(C, M, res, act):
    e = cuda_ops.ext()
    g = torch.Generator(device=DEV).manual_seed(C + M)
    y = torch.randn(M, C, device=DEV, generator=g) * 2 + 0.5
    gamma, beta = torch.rand(C, device=DEV, generator=g) + 0.5, torch.randn(C, device=DEV, generator=g)
    r = torch.randn(M, C, device=DEV, generator=g) if res else None
    dout = torch.randn(M, C, device=DEV, generator=g)
    rm, rv = torch.zeros(C, device=DEV), torch.ones(C, device=DEV)
    stats = torch.zeros(2 * C, device=DEV)
    e.col_stats(y, stats)
    torch.testing.assert_close(stats[:C], y.sum(0), rtol=1e-4, atol=1e-2)
    stats = torch.cat([stats, torch.zeros(1, device=DEV)])      # [sum | sumsq | block counter]
    out, mean, invstd = e.bn_elu_fwd(y, stats, gamma, beta, r, rm, rv, 1e-5, 0.1, act, True)
    assert float(stats.abs().sum()) == 0.0, "the kernel must leave its accumulator clean for the next use"
    # oracle
    yr, gr, br = y.clone().requires_grad_(), gamma.clone().requires_grad_(), beta.clone().requires_grad_()
    rr = r.clone().requires_grad_() if res else None
    rm2, rv2 = torch.zeros(C, device=DEV), torch.ones(C, device=DEV)
    u = F.batch_norm(yr, rm2, rv2, gr, br, True, 0.1, 1e-5)
    if res:
        u = u + rr
    o = F.elu(u) if act else u
    torch.testing.assert_close(out, o.detach(), rtol=1e-4, atol=1e-4)
    torch.testing.assert_close(rm, rm2, rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(rv, rv2, rtol=1e-4, atol=1e-5)
    o.backward(dout)
    dg, db = torch.zeros(C, device=DEV), torch.zeros(C, device=DEV)
    dy, dres = e.bn_elu_bwd(dout, out, y, mean, invstd, gamma, beta, dg, db, res, act, None)
    torch.testing.assert_close(dy, yr.grad, rtol=2e-3, atol=2e-4)
    if not res and act:   # ELU' recomputed from y instead of read from the layer output
        dy2, _ = e.bn_elu_bwd(dout, None, y, mean, invstd, gamma, beta, None, None, False, act, None)
        torch.testing.assert_close(dy2, yr.grad, rtol=2e-3, atol=2e-4)
    torch.testing.assert_close(dg, gr.grad, rtol=2e-3, atol=2e-2)
    torch.testing.assert_close(db, br.grad, rtol=2e-3, atol=2e-2)
    if res:
        torch.testing.assert_close(dres, rr.grad, rtol=1e-4, atol=1e-5)
    # self-cleaning per-layer scratch [sum du | sum du*xhat | counter]: three calls on the same buffer, no memset between them
    sb = torch.zeros(2 * C + 1, device=DEV)
    for _ in range(3):
        dy3, _ = e.bn_elu_bwd(dout, out, y, mean, invstd, gamma, beta, None, None, False, act, sb)
        torch.testing.assert_close(dy3, dy, rtol=1e-5, atol=1e-6)
    assert float(sb.abs().max()) == 0.0


def _block_pair(cin, planes, stride):
    torch.manual_seed(1)
    a = models.BasicBlock(cin, planes, stride).to(DEV)
    b = models.BasicBlock(cin, planes, stride).to(DEV)
    b.load_state_dict(a.state_dict())
    return a, b


@pytest.mark.parametrize("cin,planes,stride,H", [(64, 64, 1, 32), (64, 128, 2, 32), (256, 512, 2, 8)])
def test_basic_block_fast_path_matches_aten(cin, planes, stride, H):
    a, b = _block_pair(cin, planes, stride)
    x = torch.randn(8, cin, H, H, device=DEV).contiguous(memory_format=torch.channels_last)
    xa, xb = x.clone().requires_grad_(), x.clone().requires_grad_()
    FX.set_fast_path(True)
    oa = a(xa)
    FX.set_fast_path(False)
    ob = b(xb)
    FX.set_fast_path(True)
    assert rel_err(oa, ob) < 5e-3
    go = torch.randn_like(ob)
    oa.backward(go)
    ob.backward(go)
    assert rel_err(xa.grad, xb.grad) < 2e-2
    for (n, pa), (_, pb) in zip(a.named_parameters(), b.named_parameters()):
        assert rel_err(pa.grad, pb.grad) < 2e-2, n
    for (n, ba), (_, bb) in zip(a.named_buffers(), b.named_buffers()):
        if "num_batches" not in n:
            torch.testing.assert_close(ba, bb, rtol=5e-3, atol=5e-4, msg=n)


def test_resnet18_fast_path_matches_aten_and_respects_freezing():
    from federated_pytorch_test_b200.utils import FlatArena, unfreeze_one_block
    torch.manual_seed(0)
    a, b = models.ResNet18().to(DEV), models.ResNet18().to(DEV)
    b.load_state_dict(a.state_dict())
    FlatArena(a, channels_last_weights=True)
    x = torch.randn(16, 3, 32, 32, device=DEV).contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 10, (16,), device=DEV)
    for blk in (0, 4, 9):
        unfreeze_one_block(a, blk)
        unfreeze_one_block(b, blk)
        a._flat_arena.zero_grads()
        for p in b.parameters():
            p.grad = None
        FX.set_fast_path(True)
        la = cuda_ops.cross_entropy(a(x), y)
        la.backward()
        FX.set_fast_path(False)
        lb = F.cross_entropy(b(x), y)
        lb.backward()
        FX.set_fast_path(True)
        # error budget: whole-network gradients of the tf32 fast path vs an fp64 oracle are ~1e-3 ... 3e-3, like cuDNN with
        # TF32 on; the loss agrees to ~5e-5
        assert float(la) == pytest.approx(float(lb), rel=1e-3)
        for (n, pa), (_, pb) in zip(a.named_parameters(), b.named_parameters()):
            assert (pa.grad is None) == (pb.grad is None), n
            if pb.grad is not None:
                assert rel_err(pa.grad.contiguous(), pb.grad) < 1e-2, n


# ------------------------------------------------------------------------------------------ losses
def test_cross_entropy_and_vae_loss():
    lg = torch.randn(128, 10, device=DEV, requires_grad=True)
    lb = torch.randint(0, 10, (128,), device=DEV)
    a = cuda_ops.cross_entropy(lg, lb)
    (ga,) = torch.autograd.grad(a, lg)
    lr = lg.detach().clone().requires_grad_()
    b = F.cross_entropy(lr, lb)
    (gb,) = torch.autograd.grad(b, lr)
    torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(ga, gb, rtol=1e-4, atol=1e-7)
    r, x = torch.rand(8, 3, 32, 32, device=DEV, requires_grad=True), torch.rand(8, 3, 32, 32, device=DEV)
    mu, lv = torch.randn(8, 10, device=DEV, requires_grad=True), torch.randn(8, 10, device=DEV, requires_grad=True)
    la = cuda_ops.vae_loss(r, x, mu, lv)
    ga = torch.autograd.grad(la, (r, mu, lv))
    lbv = torch.sum((r - x) ** 2) - 0.5 * torch.sum(1 + lv - mu.pow(2) - lv.exp())
    gb = torch.autograd.grad(lbv, (r, mu, lv))
    torch.testing.assert_close(la, lbv, rtol=1e-4, atol=1e-3)
    for u, v in zip(ga, gb):
        torch.testing.assert_close(u, v, rtol=1e-4, atol=1e-6)


# ------------------------------------------------------------------------------------------ collectives (one process)
@pytest.mark.parametrize("N", [456, 850, 1856, 5130, 73984, 919040])
def test_fused_collective_single_process_matches_torch(N):
    from federated_pytorch_test_b200.parallel import Topology, TorchCollective
    from federated_pytorch_test_b200.parallel.fused import FusedCollective
    K = 4
    topo = Topology.single_process(K, DEV)
    fused, base = FusedCollective(topo), TorchCollective(topo)
    g = torch.Generator(device=DEV).manual_seed(N)
    stride = -(-N // 32) * 32                                # block slices start 128-B aligned (FlatArena contract);
    arena = fused.heap.alloc(K * stride)                     # their LENGTH may be odd (scalar tail in the kernel)
    xs = [arena[k * stride: k * stride + N] for k in range(K)]
    for x in xs:
        x.copy_(torch.randn(N, device=DEV, generator=g))
    xr = [x.clone() for x in xs]
    z, zr = torch.randn(N, device=DEV, generator=g), None
    zr = z.clone()
    d1 = fused.fedavg_(xs, z, True)
    d2 = base.fedavg_(xr, zr, True)
    assert float(d1) == pytest.approx(float(d2), rel=1e-4)
    torch.testing.assert_close(z, zr, rtol=1e-5, atol=1e-6)
    for a, b in zip(xs, xr):
        torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-6)
    for x, r in zip(xs, xr):
        x.add_(torch.randn(N, device=DEV, generator=g))
        r.copy_(x)
    d1, p1 = fused.fedprox_(xs, z, 1.5)
    d2, p2 = base.fedprox_(xr, zr, 1.5)
    assert float(d1) == pytest.approx(float(d2), rel=1e-4) and float(p1) == pytest.approx(float(p2), rel=1e-4)
    ys = [fused.zeros_like_block(x, "y") for x in xs]
    yr = [torch.zeros_like(x) for x in xr]
    for rnd in range(2):
        d1, p1 = fused.admm_(xs, ys, z, 0.1)
        d2, p2 = base.admm_(xr, yr, zr, 0.1)
        assert float(d1) == pytest.approx(float(d2), rel=1e-3, abs=1e-6) and float(p1) == pytest.approx(float(p2), rel=1e-4)
        torch.testing.assert_close(z, zr, rtol=1e-4, atol=1e-5)
        for a, b in zip(ys, yr):
            torch.testing.assert_close(a, b, rtol=1e-4, atol=1e-5)


# ------------------------------------------------------------------------------------------ engine on the GPU
def _run_fed(**kw):
    from federated_pytorch_test_b200.api import federated_multi
    lines = []
    cfg = federated_multi.Config(K=2, Nloop=1, Nadmm=2, max_minibatches=5, check_results=False, save_model=False,
                                 train_size=4096, test_size=256, default_batch=64, **kw)
    eng = federated_multi.run(cfg, log=lines.append)
    return eng, [float(l.rsplit("=", 1)[1]) for l in lines if l.startswith("dual (")]


def test_engine_resnet_graphs_equal_eager_and_fast_close_to_aten():
    e1, d_graph = _run_fed(model="ResNet9", graphs=True, fast=True)
    e2, d_eager = _run_fed(model="ResNet9", graphs=False, fast=True)
    e3, d_aten = _run_fed(model="ResNet9", graphs=False, fast=False, collective="torch")
    assert len(d_graph) == len(d_eager) == len(d_aten) == 16
    for a, b in zip(d_graph, d_eager):
        assert a == pytest.approx(b, rel=2e-2)
    worst = max(abs(a - b) / abs(b) for a, b in zip(d_eager, d_aten))
    print("fast-vs-ATen residual trace, worst relative deviation: %.3e" % worst)
    for a, b in zip(d_eager, d_aten):
        assert a == pytest.approx(b, rel=0.25)          # tf32 kernels vs fp32 ATen after a few Adam steps
    assert getattr(e1, "graph_replays", 0) > 0 and cuda_ops.launch_count() > 0


def test_host_resident_loader_matches_device_resident():
    from federated_pytorch_test_b200.data import ShardLoader, make_synthetic_cifar, worker_norm
    imgs, labs = make_synthetic_cifar(True, seed=3, size=1000)
    mean, std = worker_norm(1)
    a = ShardLoader(imgs.to(DEV), labs.to(DEV), range(0, 900), 128, DEV, mean, std, seed=5)
    b = ShardLoader(imgs.pin_memory(), labs.pin_memory(), range(0, 900), 128, DEV, mean, std, seed=5)
    assert b.host_resident and b._assembler.native
    for (xa, ya), (xb, yb) in zip(a, b):
        torch.testing.assert_close(xa, xb)
        assert torch.equal(ya, yb)


# ------------------------------------------------------------------------------------------ conv kernel variants
VARIANT_ENVS = [
    dict(FEDB200_SPLITK="1"),                                                         # one K slice: statistics fused in the epilogue
    dict(FEDB200_SPLITK="1", FEDB200_PERSIST="0"),                                    # one tile per CTA (non-persistent)
    dict(FEDB200_SPLITK="2", FEDB200_BLOCK_N="64"),                                   # persistent, several tiles per CTA, split-K
    dict(FEDB200_SPLITK="1", FEDB200_BLOCK_N="64"),
    dict(FEDB200_SPLITK="2"),                                                         # split-K on the widest tile (128)
    dict(FEDB200_SPLITK="4"),                                                         # split-K with bulk reduce-adds
    dict(),                                                                           # defaults
    dict(FEDB200_SPLITK="8", FEDB200_BLOCK_N="32"),
    dict(FEDB200_SPLITK="1", FEDB200_BLOCK_N="32"),                                   # 64 x 32 wgmma tiles
    dict(FEDB200_SPLITK="2", FEDB200_BLOCK_N="128"),
    dict(FEDB200_SPLITK="2", FEDB200_PERSIST="0"),
    dict(FEDB200_SPLITK="1", FEDB200_TMA_STORE="0"),                                  # direct stores from the accumulator fragments
    dict(FEDB200_SPLITK="2", FEDB200_TMA_STORE="0"),                                  # split-K through atomics
    dict(FEDB200_TAP_PACK="0"),                                                       # one tap per k-block at C_in = 4
    dict(FEDB200_TAP_PACK="0", FEDB200_BLOCK_N="32"),
]


@pytest.mark.parametrize("env", VARIANT_ENVS, ids=lambda e: ",".join("%s=%s" % (k[8:], v) for k, v in e.items()) or "defaults")
@pytest.mark.parametrize("B,H,Ci,Co", [(5, 32, 64, 64), (3, 32, 4, 64), (6, 16, 128, 128), (16, 8, 256, 256), (20, 32, 64, 64)])
def test_conv_kernel_variants(monkeypatch, env, B, H, Ci, Co):
    import os
    for k in ("FEDB200_SPLITK", "FEDB200_BLOCK_N", "FEDB200_PERSIST", "FEDB200_TMA_STORE", "FEDB200_TAP_PACK"):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    g = torch.Generator(device=DEV).manual_seed(B + H + Ci)
    x = torch.randn(B, H, H, Ci, device=DEV, generator=g)
    w = torch.randn(Co, 3, 3, Ci, device=DEV, generator=g) / math.sqrt(9 * Ci)
    stats = torch.zeros(2 * Co, device=DEV)
    y = cuda_ops.conv2d_nhwc(x, w, stats, 1, 1)
    ref = F.conv2d(x.permute(0, 3, 1, 2).double(), w.permute(0, 3, 1, 2).double(), None, 1, 1).permute(0, 2, 3, 1).float()
    assert rel_err(y, ref) < 3e-3
    flat = ref.reshape(-1, Co)
    torch.testing.assert_close(stats[:Co], flat.sum(0), rtol=2e-3, atol=2e-2 * math.sqrt(flat.shape[0]))
    torch.testing.assert_close(stats[Co:], (flat * flat).sum(0), rtol=5e-3, atol=1e-2)
