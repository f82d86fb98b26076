"""Client SGD on the H100: the fused ``sgd_prox`` kernel against the ATen composition and ``torch.optim.SGD``, the graphed
step against the eager step, the classifier drivers on the fused path against the ATen path, and co-resident replicas."""
import pytest
import torch
import torch.nn as nn

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():  # collected (and deselected) on the CPU box
    pytest.skip("CUDA device required", allow_module_level=True)

from federated_pytorch_test_b200 import models  # noqa: E402
from federated_pytorch_test_b200.api import consensus_multi, federated_multi, fedprox_multi  # noqa: E402
from federated_pytorch_test_b200.ops import cuda_ops, flatops, losses  # noqa: E402
from federated_pytorch_test_b200.ops import functional as FX  # noqa: E402
from federated_pytorch_test_b200.optim import BlockSGD  # noqa: E402
from federated_pytorch_test_b200.utils.flat import FlatArena  # noqa: E402

DEV = torch.device("cuda", 0)
SGD = dict(optimizer="sgd", lr=0.05, momentum=0.9)
OPTIONS = [dict(momentum=m, nesterov=n, weight_decay=wd, pen=pen)
           for m, n in ((0.0, False), (0.9, False), (0.9, True)) for wd in (0.0, 5e-4) for pen in (False, True)]


@pytest.fixture(autouse=True)
def _fast_path():
    FX.set_fast_path(True)
    yield
    FX.set_fast_path(True)


# ------------------------------------------------------------------------------------------ kernel
@pytest.mark.parametrize("n", [1856, 73984 + 3, 4720640])
@pytest.mark.parametrize("rho_dev", [False, True])
def test_sgd_prox_matches_oracle(n, rho_dev):
    g = torch.Generator(device=DEV).manual_seed(n)
    for o in OPTIONS:
        x = torch.randn(n, device=DEV, generator=g)
        z, y = (torch.randn(n, device=DEV, generator=g), torch.randn(n, device=DEV, generator=g)) if o["pen"] else (None, None)
        rho, l1, l2 = (0.3, 1e-4, 1e-4) if o["pen"] else (0.0, 0.0, 0.0)
        rd = torch.full((1,), rho, device=DEV) if rho_dev else None
        xr = x.clone()
        buf = torch.zeros(n, device=DEV) if o["momentum"] else None
        bufr = buf.clone() if buf is not None else None
        for _ in range(3):
            gr = torch.randn(n, device=DEV, generator=g)
            args = (0.05, o["momentum"], o["nesterov"], o["weight_decay"], z, y, 0.0 if rho_dev else rho, l1, l2, rd)
            cuda_ops.sgd_prox_step(x, gr, buf, *args)
            FX.set_fast_path(False)
            flatops.sgd_prox_step(xr, gr, bufr, *args)
            FX.set_fast_path(True)
        torch.testing.assert_close(x, xr, rtol=1e-5, atol=1e-6, msg=lambda m: "%s: %s" % (o, m))
        if buf is not None:
            torch.testing.assert_close(buf, bufr, rtol=1e-5, atol=1e-6, msg=lambda m: "%s: %s" % (o, m))


def test_no_momentum_allocates_and_passes_no_buffer():
    net = models.Net().to(DEV)
    arena = FlatArena(net, device=DEV)
    for p in net.parameters():
        p.requires_grad = True
    arena.attach_grads()
    before = torch.cuda.memory_allocated(DEV)
    opt = BlockSGD(arena, 0, len(arena.params) - 1, lr=0.1)
    assert opt.buf is None and torch.cuda.memory_allocated(DEV) == before
    x0 = opt.x.clone()
    arena.grad.normal_()
    opt.apply_update()
    torch.testing.assert_close(opt.x, x0 - 0.1 * opt.g)
    x = torch.zeros(64, device=DEV)
    with pytest.raises(RuntimeError, match="momentum"):          # the binding refuses a buffer without momentum ...
        cuda_ops.sgd_prox_step(x, x.clone(), torch.zeros(64, device=DEV), 0.1, 0.0, False, 0.0)
    with pytest.raises(RuntimeError, match="momentum"):          # ... and momentum without a buffer
        cuda_ops.sgd_prox_step(x, x.clone(), None, 0.1, 0.9, False, 0.0)


def test_plain_kernel_matches_torch_sgd_over_20_steps():
    n = 73984 + 3
    x = torch.randn(n, device=DEV)
    p = nn.Parameter(x.clone())
    opt = torch.optim.SGD([p], lr=0.05, momentum=0.9, nesterov=True, weight_decay=5e-4)
    buf = torch.zeros(n, device=DEV)
    for _ in range(20):
        g = torch.randn(n, device=DEV)
        p.grad = g.clone()
        opt.step()
        cuda_ops.sgd_prox_step(x, g, buf, 0.05, 0.9, True, 5e-4)
    torch.testing.assert_close(x, p.detach(), rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(buf, opt.state[p]["momentum_buffer"], rtol=1e-5, atol=1e-5)


# ------------------------------------------------------------------------------------------ graphed step
def _run(mod, **kw):
    lines = []
    base = dict(K=2, model="ResNet18", Nloop=1, Nadmm=2, max_minibatches=4, check_results=False, save_model=False,
                train_size=4096, test_size=256, default_batch=64, distributed=False)
    eng = mod.run(mod.Config(**{**base, **kw}), log=lines.append)
    torch.cuda.synchronize()
    return eng, lines


def _duals(lines):
    return [float(l.rsplit("=", 1)[1]) for l in lines if l.startswith("dual (")]


def _residuals(lines):
    return [tuple(float(v) for v in l.split("primal=")[1].split(" dual=")) for l in lines if l.startswith("block=[")]


def test_graphed_step_equals_eager_step():
    """(a) On identical state, one replay and one eager step of an SGD ResNet18 block visit give the same loss, block and
    momentum buffer, within the spread between two eager steps from that state; (b) over a whole run the graphed residuals
    stay within a tolerance derived from the spread between two eager runs (the weight-gradient kernels sum in a
    float-atomic order, so neither path is bit-reproducible)."""
    kw = dict(**SGD, nesterov=True, weight_decay=5e-4)
    ea, a = _run(federated_multi, **kw, graphs=False)
    ea2, a2 = _run(federated_multi, **kw, graphs=False)
    eb, b = _run(federated_multi, **kw, graphs=True)
    assert eb.graph_replays > 0 and ea.graph_replays == 0
    da, da2, db = _duals(a), _duals(a2), _duals(b)
    assert len(da) == len(db) == 20
    spread = max(abs(u - v) / max(abs(u), 1e-12) for u, v in zip(da, da2))
    print("eager-vs-eager relative spread of the duals: %.2e" % spread)
    for u, v in zip(da, db):
        assert v == pytest.approx(u, rel=max(5e-2, 5 * spread), abs=1e-7)

    # (a): the last block visit's graph of replica 0
    from federated_pytorch_test_b200.algo.graphs import GraphedAdamStep

    steps = [gs for gs in eb._graphs.values() if isinstance(gs, GraphedAdamStep) and gs.graph is not None
             and gs.rep is eb.replicas[0] and gs.opt is eb.optimizers[0]]
    assert len(steps) == 1
    gs = steps[0]
    opt, pen = gs.opt, eb.strategy.penalty(0)
    assert isinstance(opt, BlockSGD) and opt.buf is not None
    batch = [t.clone() if torch.is_tensor(t) else t for t in gs.static]
    x0, b0 = opt.x.clone(), opt.buf.clone()

    def restore():
        opt.x.copy_(x0)
        opt.buf.copy_(b0)

    def eager():
        restore()
        opt.set_penalty(pen.z, pen.y, pen.rho, gs.visit.lambda1, gs.visit.lambda2, pen.rho_dev)
        loss = gs._body().clone()
        torch.cuda.synchronize()
        return loss, opt.x.clone(), opt.buf.clone()

    restore()
    n_replays = eb.graph_replays
    loss_g = gs.run(batch, pen)
    assert eb.graph_replays == n_replays + 1                        # it replayed, no re-capture
    got = (loss_g, opt.x.clone(), opt.buf.clone())
    e1, e2 = eager(), eager()
    for name, g_, u, v in zip(("loss", "block", "momentum buffer"), got, e1, e2):
        spread = float((u - v).abs().max())
        diff = float((g_ - u).abs().max())
        print("%s: replay-vs-eager %.3e, eager-vs-eager %.3e" % (name, diff, spread))
        assert diff <= 4 * spread + 1e-6 * max(float(u.abs().max()), 1.0), name
    assert not torch.equal(got[1], x0)                            # the step moved the block


@pytest.mark.parametrize("mod,extra", [(federated_multi, {}), (fedprox_multi, {}), (consensus_multi, dict(bb_update=True))],
                         ids=["fedavg", "fedprox", "admm_bb"])
def test_resnet18_sgd_graphed_equals_aten(mod, extra):
    e1, l_fast = _run(mod, **SGD, **extra, graphs=True)
    e2, l_aten = _run(mod, **SGD, **extra, graphs=False, fast=False)
    assert e1.coll.name == "fused" and e2.coll.name == "torch" and e1.graph_replays > 0
    assert all(isinstance(o, BlockSGD) for o in e1.optimizers)
    if mod is federated_multi:
        d_fast, d_aten = _duals(l_fast), _duals(l_aten)
    else:
        d_fast = [d for _, d in _residuals(l_fast)]
        d_aten = [d for _, d in _residuals(l_aten)]
    print("fused + graphed:", d_fast[:6], "\nATen:", d_aten[:6])
    assert len(d_fast) == len(d_aten) == 20
    for a, b in zip(d_fast, d_aten):                                     # TF32 convolutions against fp32 ATen
        assert a == pytest.approx(b, rel=5e-2)


# ------------------------------------------------------------------------------------------ co-resident replicas
def test_four_coresident_replicas_lower_the_loss(monkeypatch):
    """K = 4 replicas on one GPU, each on its own stream: the diagnostics loss of the last minibatches of the run is below
    that of the first ones."""
    from federated_pytorch_test_b200.algo.engine import Engine

    step_losses = []
    orig_init = Engine.__init__

    def patched(self, *a, **k):
        orig_init(self, *a, **k)
        self.step_hook = lambda e: step_losses.append(e.last_loss1)
    monkeypatch.setattr(Engine, "__init__", patched)
    eng, lines = _run(federated_multi, K=4, **SGD, Nadmm=3, max_minibatches=8, graphs=True)
    assert len(eng.replicas) == 4 and all(isinstance(o, BlockSGD) for o in eng.optimizers) and eng.graph_replays > 0
    assert eng.cfg.streams and len(eng._streams) == 4
    vals = [float(v) for v in step_losses]
    assert len(vals) == 10 * 3 * 4 * 8
    first, last = sum(vals[:16]) / 16, sum(vals[-16:]) / 16
    print("mean diagnostics loss of the first / last 16 minibatches: %.4f -> %.4f" % (first, last))
    assert all(v == v for v in vals) and last < first


_LIB = ("cudnn", "cutlass", "cublas", "sgemm", "xmma", "implicit_gemm", "gemv", "gemmk1")


def test_training_step_launches_no_library_kernel():
    """The profiler's kernel list of one SGD training step (forward, backward, fused SGD update) of ResNet18 with every
    parameter trainable and momentum on."""
    torch.manual_seed(0)
    net = models.ResNet18().to(DEV)
    arena = FlatArena(net, device=DEV, channels_last_weights=True)
    for p in net.parameters():
        p.requires_grad = True
    arena.attach_grads()
    opt = BlockSGD(arena, 0, len(arena.params) - 1, lr=0.05, momentum=0.9, nesterov=True, weight_decay=5e-4)
    x = torch.rand(64, 3, 32, 32, device=DEV).contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 10, (64,), device=DEV)

    def step():
        opt.zero_grad()
        with cuda_ops.accumulate_into_grad():
            losses.cross_entropy(net(x), y).backward()
        opt.apply_update()

    step()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        step()
        torch.cuda.synchronize()
    names = [e.key for e in prof.key_averages()]
    lib = [n for n in names if any(t in n.lower() for t in _LIB)]
    assert not lib, lib
    assert any("sgd_prox" in n for n in names), names
