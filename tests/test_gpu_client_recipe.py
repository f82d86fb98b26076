"""Client training recipe on the H100: the ``adam_prox`` / ``sgd_prox`` kernels with a device learning rate, AdamW decay and
gradient-norm clipping (``grad_norm_kernel``) against the ``flatops`` oracle, reproducibility of the clipped update, the
graphed step across learning-rate changes, the classifier drivers on the fused path against the ATen path, co-resident
replicas and the kernels a training step launches."""
import pytest
import torch

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():  # collected (and deselected) on the CPU box
    pytest.skip("CUDA device required", allow_module_level=True)

from federated_pytorch_test_b200 import models  # noqa: E402
from federated_pytorch_test_b200.algo.graphs import GraphedAdamStep, capture_graph  # noqa: E402
from federated_pytorch_test_b200.api import consensus_multi, federated_multi, fedprox_multi, no_consensus_multi  # noqa: E402
from federated_pytorch_test_b200.ops import cuda_ops, flatops, losses  # noqa: E402
from federated_pytorch_test_b200.ops import functional as FX  # noqa: E402
from federated_pytorch_test_b200.optim import BlockSGD  # noqa: E402
from federated_pytorch_test_b200.optim.block_adam import BlockAdam  # noqa: E402
from federated_pytorch_test_b200.optim.schedule import round_lr  # noqa: E402
from federated_pytorch_test_b200.utils.flat import FlatArena  # noqa: E402

DEV = torch.device("cuda", 0)
RECIPE = dict(optimizer="adamw", weight_decay=0.05, lr_schedule="cosine", lr_warmup=2, lr_min=0.1, clip_norm=1.0)
SIZES = [1856, 73984 + 3, 4720640]          # the smallest and largest ResNet18 blocks, and an odd length


@pytest.fixture(autouse=True)
def _fast_path():
    FX.set_fast_path(True)
    yield
    FX.set_fast_path(True)


# ------------------------------------------------------------------------------------------ kernels
def _assert_close_but_for_discontinuities(got, want, what):
    """Elementwise agreement except at a few elements where the update is discontinuous or ill-conditioned: x crossing 0
    flips the elastic-net term l1 sign(x), and where the total gradient cancels to rounding level Adam's m / sqrt(v) takes
    its sign from the rounding.  The fused kernel (FMA) and the ATen oracle round differently there."""
    bad = ~torch.isclose(got, want, rtol=1e-5, atol=1e-6)
    assert int(bad.sum()) <= max(2, got.numel() // 200000), "%s: %d elements differ, max %g" % (
        what, int(bad.sum()), float((got - want).abs().max()))
    assert float((got - want).abs().max()) <= 1e-3 * max(float(want.abs().max()), 1.0), what


def _oracle(fn):
    FX.set_fast_path(False)
    try:
        fn()
    finally:
        FX.set_fast_path(True)


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("kind", ["adam", "adamw", "sgd"])
def test_update_kernels_match_oracle(n, kind):
    g = torch.Generator(device=DEV).manual_seed(n)
    for clip in (0.0, n ** 0.5, 1e9):                       # off, clipping the last two of three steps, never clipping
        for pen in (False, True):
            for rho_dev in ((False, True) if pen else (False,)):
                x = torch.randn(n, device=DEV, generator=g)
                z, y = (torch.randn(n, device=DEV, generator=g), 1e-2 * torch.randn(n, device=DEV, generator=g)) \
                    if pen else (None, None)
                rho, l1, l2 = (0.3, 1e-4, 1e-4) if pen else (0.0, 0.0, 0.0)
                rd = torch.full((1,), rho, device=DEV) if rho_dev else None
                xr = x.clone()
                st = [torch.zeros(n, device=DEV) for _ in range(2)]
                sr = [t.clone() for t in st]
                lr = torch.zeros(1, device=DEV)
                ws = flatops.clip_workspace(x)
                FX.set_fast_path(False)
                wsr = flatops.clip_workspace(xr)
                FX.set_fast_path(True)
                for k in range(3):
                    lr.fill_(round_lr(1e-2 if kind != "sgd" else 0.05, k, 3, "cosine", 1))
                    gr = (0.5 + k) * torch.randn(n, device=DEV, generator=g)
                    args = (z, y, 0.0 if rho_dev else rho, l1, l2, rd)
                    if kind == "sgd":
                        def step(xx, s, w):
                            flatops.sgd_prox_step(xx, gr, s[0], lr, 0.9, True, 5e-4, *args, clip_norm=clip, clip_ws=w)
                    else:
                        def step(xx, s, w):
                            flatops.adam_prox_step(xx, gr, s[0], s[1], k + 1, lr, 0.9, 0.999, 1e-8, *args,
                                                   weight_decay=0.05 if kind == "adamw" else 0.0, clip_norm=clip,
                                                   clip_ws=w)
                    step(x, st, ws)
                    _oracle(lambda: step(xr, sr, wsr))
                what = "%s n=%d clip=%g pen=%s rho_dev=%s" % (kind, n, clip, pen, rho_dev)
                _assert_close_but_for_discontinuities(x, xr, what)
                _assert_close_but_for_discontinuities(st[0], sr[0], what)
                if clip:
                    torch.testing.assert_close(ws[0][:4], wsr[0][:4], rtol=1e-5, atol=0, msg=lambda m: "%s: %s" % (what, m))
                    assert float(ws[0][3]) == 3 and int(ws[1]) == 0                # three steps; the ticket reset itself


def test_default_arguments_launch_the_kernels_of_before():
    """No device lr, no decay, no clipping: the new arguments change no bit of the Adam and SGD updates."""
    n = 73984 + 3
    x, gr = torch.randn(n, device=DEV), torch.randn(n, device=DEV)
    m, v, buf = torch.zeros(n, device=DEV), torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
    xs = [x.clone() for _ in range(4)]
    ms = [t.clone() for t in (m, m, buf, buf)]
    vs = [v.clone(), v.clone()]
    cuda_ops.adam_prox_step(xs[0], gr, ms[0], vs[0], 1, 1e-3, 0.9, 0.999, 1e-8)
    lr = torch.full((1,), 1e-3, device=DEV)
    cuda_ops.adam_prox_step(xs[1], gr, ms[1], vs[1], 1, 0.0, 0.9, 0.999, 1e-8, lr_dev=lr)
    cuda_ops.sgd_prox_step(xs[2], gr, ms[2], 0.05, 0.9, True, 5e-4)
    lr.fill_(0.05)
    cuda_ops.sgd_prox_step(xs[3], gr, ms[3], 0.0, 0.9, True, 5e-4, lr_dev=lr)
    assert torch.equal(xs[0], xs[1]) and torch.equal(ms[0], ms[1]) and torch.equal(vs[0], vs[1])
    assert torch.equal(xs[2], xs[3]) and torch.equal(ms[2], ms[3])


@pytest.mark.parametrize("n", SIZES)
def test_clipped_update_is_bit_reproducible_and_its_norm_is_float64s(n):
    gen = torch.Generator(device=DEV).manual_seed(7)
    x0, gr = torch.randn(n, device=DEV, generator=gen), 1e-2 * torch.randn(n, device=DEV, generator=gen)
    outs = []
    for _ in range(2):
        x, m, v = x0.clone(), torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
        ws = flatops.clip_workspace(x)
        for k in range(3):
            flatops.adam_prox_step(x, gr, m, v, k + 1, 1e-3, 0.9, 0.999, 1e-8, weight_decay=0.01, clip_norm=0.1,
                                   clip_ws=ws)
        outs.append((x, m, ws[0][:4].clone()))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    assert torch.equal(outs[0][2], outs[1][2])
    want = float(gr.double().norm())
    assert float(outs[0][2][0]) == pytest.approx(want, rel=2e-6)
    assert float(outs[0][2][1]) == pytest.approx(3 * want, rel=2e-6) and float(outs[0][2][2]) == 3


@pytest.mark.parametrize("bad", [float("nan"), float("inf")])
def test_non_finite_gradient_gives_non_finite_parameters(bad):
    n = 73984 + 3
    x, gr = torch.randn(n, device=DEV), torch.randn(n, device=DEV)
    gr[1234] = bad
    flatops.adam_prox_step(x, gr, torch.zeros(n, device=DEV), torch.zeros(n, device=DEV), 1, 1e-3, 0.9, 0.999, 1e-8,
                           clip_norm=1.0)
    assert not torch.isfinite(x).all()
    x = torch.randn(n, device=DEV)
    flatops.sgd_prox_step(x, gr, None, 0.1, clip_norm=1.0)
    assert not torch.isfinite(x).all()


# ------------------------------------------------------------------------------------------ graphed update
def _resnet18_block_opt(make):
    torch.manual_seed(0)
    net = models.ResNet18().to(DEV)
    arena = FlatArena(net, device=DEV, channels_last_weights=True)
    for p in net.parameters():
        p.requires_grad = True
    arena.attach_grads()
    return net, arena, make(arena, 0, len(arena.params) - 1)


@pytest.mark.parametrize("kind", ["adamw", "sgd"])
def test_graphed_update_follows_the_learning_rate_without_recapture(kind):
    """One captured update, replayed across three rounds whose learning rate changes, gives the same bits as the eager
    update from the same state."""
    def make(arena, lo, hi):
        if kind == "sgd":
            return BlockSGD(arena, lo, hi, lr=0.05, momentum=0.9, clip_norm=1.0, device_lr=True)
        return BlockAdam(arena, lo, hi, lr=1e-3, adamw=True, weight_decay=0.05, clip_norm=1.0, device_lr=True)

    _, arena, opt = _resnet18_block_opt(make)
    arena.grad.normal_()
    x0 = opt.x.clone()
    state = [t for t in (getattr(opt, "m", None), getattr(opt, "v", None), getattr(opt, "buf", None)) if t is not None]
    opt.apply_update()                      # warm-up (eager), then back to the start
    opt.x.copy_(x0)
    for t in state:
        t.zero_()
    opt.clip_stats.zero_()
    if kind == "adamw":
        opt.t_dev.zero_()
    graph, _ = capture_graph(torch.cuda.Stream(), lambda: opt.apply_update())
    # the eager twin: the same optimizer on a copy of the arena
    _, arena2, opt2 = _resnet18_block_opt(make)
    arena2.data.copy_(arena.data)
    opt2.x.copy_(x0)
    arena2.grad.copy_(arena.grad)
    for r in range(3):
        lr = round_lr(1e-3 if kind == "adamw" else 0.05, r, 3, "cosine", 1)
        opt.set_lr(lr)
        opt2.set_lr(lr)
        graph.replay()
        opt2.apply_update()
        torch.cuda.synchronize()
        assert torch.equal(opt.x, opt2.x), r
    assert not torch.equal(opt.x, x0)
    assert torch.equal(opt.clip_stats, opt2.clip_stats) and float(opt.clip_stats[2]) == 3


# ------------------------------------------------------------------------------------------ drivers
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


def test_graphed_run_equals_eager_run_and_captures_once(monkeypatch):
    captures = []
    orig = GraphedAdamStep._capture

    def counting(self):
        captures.append(self)
        orig(self)
    monkeypatch.setattr(GraphedAdamStep, "_capture", counting)
    ea, a = _run(federated_multi, **RECIPE, graphs=False)
    eb, b = _run(federated_multi, **RECIPE, graphs=True)
    graphs = [gs for gs in eb._graphs.values() if isinstance(gs, GraphedAdamStep)]
    assert eb.graph_replays > 0 and len(captures) == len(graphs) == 2 * 10      # once per (replica, block)
    da, db = _duals(a), _duals(b)
    assert len(da) == len(db) == 20
    for u, v in zip(da, db):
        assert v == pytest.approx(u, rel=5e-2, abs=1e-7)
    last = round_lr(1e-3, 19, 20, "cosine", 2, lr_min=0.1)
    assert all(float(o.lr_dev) == last for o in eb.optimizers)


@pytest.mark.parametrize("mod,extra", [(federated_multi, {}), (fedprox_multi, {}), (consensus_multi, dict(bb_update=True)),
                                       (no_consensus_multi, dict(Nepoch=3))],
                         ids=["fedavg", "fedprox", "admm_bb", "no_consensus"])
def test_resnet18_recipe_fused_equals_aten(mod, extra):
    e1, l_fast = _run(mod, **RECIPE, **extra, graphs=True)
    e2, l_aten = _run(mod, **RECIPE, **extra, graphs=False, fast=False)
    assert e1.graph_replays > 0
    assert all(isinstance(o, BlockAdam) and o.adamw and o.clip_ws is not None for o in e1.optimizers)
    if mod is no_consensus_multi:
        a, b = e1.replicas[0].running_loss, e2.replicas[0].running_loss
        print("fused + graphed: %.5f  ATen: %.5f" % (a, b))
        assert a == pytest.approx(b, rel=5e-2)
        return
    assert e1.coll.name == "fused" and e2.coll.name == "torch"
    if mod is federated_multi:
        d_fast, d_aten = _duals(l_fast), _duals(l_aten)
    else:
        d_fast = [d for _, d in _residuals(l_fast)]
        d_aten = [d for _, d in _residuals(l_aten)]
    print("fused + graphed:", d_fast[:6], "\nATen:", d_aten[:6])
    assert len(d_fast) == len(d_aten) == 20
    for a, b in zip(d_fast, d_aten):                                     # TF32 convolutions against fp32 ATen
        assert a == pytest.approx(b, rel=5e-2)


def test_four_coresident_replicas_lower_the_loss(monkeypatch):
    from federated_pytorch_test_b200.algo.engine import Engine

    step_losses = []
    orig_init = Engine.__init__

    def patched(self, *a, **k):
        orig_init(self, *a, **k)
        self.step_hook = lambda e: step_losses.append(e.last_loss1)
    monkeypatch.setattr(Engine, "__init__", patched)
    eng, lines = _run(federated_multi, K=4, **RECIPE, Nadmm=3, max_minibatches=8, graphs=True)
    assert len(eng.replicas) == 4 and eng.graph_replays > 0 and len(eng._streams) == 4
    vals = [float(v) for v in step_losses]
    assert len(vals) == 10 * 3 * 4 * 8
    first, last = sum(vals[:16]) / 16, sum(vals[-16:]) / 16
    print("mean diagnostics loss of the first / last 16 minibatches: %.4f -> %.4f" % (first, last))
    assert all(v == v for v in vals) and last < first
    lrs = {float(o.lr_dev) for o in eng.optimizers}
    assert len(lrs) == 1


def test_kernels_per_replay():
    """The default configuration captures the kernels it always did; a schedule adds none; clipping adds the norm."""
    counts = {}
    for name, kw in (("default", {}), ("schedule", dict(lr_schedule="cosine")), ("clip", dict(clip_norm=1.0))):
        eng, _ = _run(federated_multi, K=1, Nadmm=1, max_minibatches=5, graphs=True, **kw)
        counts[name] = sorted({gs.kernels_per_replay for gs in eng._graphs.values() if isinstance(gs, GraphedAdamStep)})
    print(counts)
    assert counts["schedule"] == counts["default"]
    assert counts["clip"] == [c + 1 for c in counts["default"]]


_LIB = ("cudnn", "cutlass", "cublas", "sgemm", "xmma", "implicit_gemm", "gemv", "gemmk1")


def test_graphed_step_launches_no_library_kernel_and_shows_the_recipe_kernels():
    net, arena, opt = _resnet18_block_opt(
        lambda a, lo, hi: BlockAdam(a, lo, hi, lr=1e-3, adamw=True, weight_decay=0.05, clip_norm=1.0, device_lr=True))
    x = torch.rand(128, 3, 32, 32, device=DEV).contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 10, (128,), device=DEV)

    def body():
        arena.zero_grads()
        with cuda_ops.accumulate_into_grad():
            losses.cross_entropy(net(x), y).backward()
        opt.apply_update()

    for _ in range(3):
        body()
    graph, _ = capture_graph(torch.cuda.Stream(), body)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        opt.set_lr(5e-4)
        graph.replay()
        torch.cuda.synchronize()
    names = [e.key for e in prof.key_averages()]
    lib = [n for n in names if any(t in n.lower() for t in _LIB)]
    assert not lib, lib
    assert any("grad_norm_kernel" in n for n in names), names
    assert any("adam_prox_kernel" in n for n in names), names
