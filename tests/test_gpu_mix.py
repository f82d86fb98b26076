"""Label smoothing, mixup and CutMix on the H100: the fused mixing input kernel bit for bit against the ATen composition of
the oracle draws, its launch count, the deterministic soft-target cross-entropy kernels against float64, the kernels a
graphed step launches, and the classifier drivers (graphed against eager, fused against ATen, L-BFGS, accuracy)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():  # collected (and deselected) on the CPU box
    pytest.skip("CUDA device required", allow_module_level=True)

from federated_pytorch_test_b200 import models  # noqa: E402
from federated_pytorch_test_b200.algo.graphs import GraphedAdamStep, capture_graph  # noqa: E402
from federated_pytorch_test_b200.api import consensus_multi, federated_multi, fedprox_multi, no_consensus_multi  # noqa: E402
from federated_pytorch_test_b200.data import (ShardLoader, augment_key, augment_u8, make_synthetic_cifar,  # noqa: E402
                                              mix_draws, mix_images, mix_key, worker_norm)
from federated_pytorch_test_b200.ops import cuda_ops, losses  # noqa: E402
from federated_pytorch_test_b200.ops import functional as FX  # noqa: E402

DEV = torch.device("cuda", 0)
COUNTERS = [0, 6249, (1 << 32) - 3, (1 << 32) + 11, 3 << 40]
ALPHAS = {"mixup": (0.4, 0.0), "cutmix": (0.0, 1.0)}
FLAGS = dict(augment=True, cutmix_alpha=1.0, mixup_alpha=0.2, label_smoothing=0.1)


@pytest.fixture(autouse=True)
def _fast_path():
    FX.set_fast_path(True)
    yield
    FX.set_fast_path(True)


@pytest.fixture(scope="module")
def data():
    imgs, labs = make_synthetic_cifar(True, seed=11, size=2000)
    return imgs.to(DEV), labs.to(DEV)


# ------------------------------------------------------------------------------------------ input kernel
@pytest.mark.parametrize("mode", ["mixup", "cutmix"])
@pytest.mark.parametrize("augment", [False, True])
@pytest.mark.parametrize("channels_last", [False, True])
@pytest.mark.parametrize("n", [128, 105])
def test_kernel_is_bit_identical_to_aten_mixing_of_the_oracle_draw(data, mode, augment, channels_last, n):
    imgs, _ = data
    mean, std = worker_norm(3)
    g = torch.Generator().manual_seed(n)
    for ck, counter in enumerate(COUNTERS):
        akey, key = augment_key(69, ck), mix_key(69, ck)
        idx = torch.randperm(imgs.shape[0], generator=g)[:n].to(DEV)
        u8 = imgs.index_select(0, idx)
        draw = mix_draws(key, counter, n, 32, 32, *ALPHAS[mode])
        base = cuda_ops.normalize_u8(augment_u8(u8, akey, counter) if augment else u8, mean, std, channels_last)
        want = mix_images(base, draw[0], draw[1], draw[2])
        aug = akey if augment else None
        gathered = cuda_ops.mix_normalize_u8(imgs, idx, aug, counter, mean, std, channels_last, draw)   # index-gather mode
        batch = cuda_ops.mix_normalize_u8(u8, None, aug, counter, mean, std, channels_last, draw)
        for got, lam in (gathered, batch):
            assert got.shape == (n, 3, 32, 32) and got.stride() == want.stride()
            assert torch.equal(got, want), (mode, augment, n, channels_last, counter)
            assert lam.shape == (1,) and lam.dtype == torch.float32 and float(lam) == float(np.float32(draw[3]))


@pytest.mark.parametrize("channels_last", [False, True])
def test_host_resident_mixing_loader_matches_device_resident(channels_last):
    imgs, labs = make_synthetic_cifar(True, seed=3, size=1000)
    mean, std = worker_norm(1)
    kw = dict(seed=5, channels_last=channels_last, augment=True, aug_key=augment_key(69, 1), mixup_alpha=0.2,
              cutmix_alpha=1.0, mix_key=mix_key(69, 1))
    a = ShardLoader(imgs.to(DEV), labs.to(DEV), range(0, 900), 128, DEV, mean, std, **kw)
    b = ShardLoader(imgs.pin_memory(), labs.pin_memory(), range(0, 900), 128, DEV, mean, std, **kw)
    assert b.host_resident and b._assembler.native
    n = 0
    for epoch in range(2):
        for (xa, ya, la), (xb, yb, lb) in zip(a, b):
            assert torch.equal(xa, xb) and torch.equal(ya, yb) and torch.equal(la, lb) and la.is_cuda
            n += ya.numel()
    assert n == 1800 and a.aug_counter == b.aug_counter == 1800


@pytest.mark.parametrize("augment", [False, True])
def test_mixed_device_batch_is_one_handwritten_launch(data, augment):
    imgs, labs = data
    ld = ShardLoader(imgs, labs, range(0, 1500), 128, DEV, *worker_norm(0), seed=1, channels_last=True, augment=augment,
                     aug_key=augment_key(69, 0), mixup_alpha=0.2, cutmix_alpha=1.0, mix_key=mix_key(69, 0))
    it = iter(ld)
    next(it)
    before = cuda_ops.launch_count()
    x, y, lam = next(it)
    assert cuda_ops.launch_count() - before == 1
    assert x.shape == (128, 3, 32, 32) and x.is_contiguous(memory_format=torch.channels_last)


# ------------------------------------------------------------------------------------------ loss kernels
def _soft_targets(y, lam, eps, C):
    s = (1.0 - eps) * F.one_hot(y, C).double() + eps / C
    return lam * s + (1.0 - lam) * s.flip(0)


@pytest.mark.parametrize("C", [10, 100])
@pytest.mark.parametrize("B", [1, 105, 128, 4096])
def test_soft_ce_matches_float64_and_repeats_bit_for_bit(B, C):
    g = torch.Generator(device=DEV).manual_seed(B + C)
    z = 3.0 * torch.randn(B, C, device=DEV, generator=g)
    y = torch.randint(0, C, (B,), device=DEV, generator=g)
    for eps, lam in ((0.1, None), (0.0, 0.3), (0.1, 0.7), (0.2, 1.0)):
        lam_t = None if lam is None else torch.tensor([lam], dtype=torch.float32, device=DEV)
        zz = z.clone().requires_grad_()
        loss = cuda_ops.soft_cross_entropy(zz, y, lam_t, eps)
        (gz,) = torch.autograd.grad(loss, zz)
        z64 = z.double().requires_grad_()
        ref = F.cross_entropy(z64, _soft_targets(y, 1.0 if lam is None else float(np.float32(lam)), eps, C))
        (gref,) = torch.autograd.grad(ref, z64)
        assert float(loss.detach()) == pytest.approx(float(ref.detach()), rel=1e-5), (eps, lam)
        torch.testing.assert_close(gz.double(), gref, rtol=1e-5, atol=1e-6 / B)
        again = [cuda_ops.ext().soft_ce_fwd(z, y, lam_t, eps)[0] for _ in range(3)]
        assert all(torch.equal(a, loss.detach()) for a in again)


def test_soft_ce_without_smoothing_or_mixing_agrees_with_the_hard_label_kernel():
    g = torch.Generator(device=DEV).manual_seed(0)
    z = (3.0 * torch.randn(128, 10, device=DEV, generator=g)).requires_grad_()
    y = torch.randint(0, 10, (128,), device=DEV, generator=g)
    one = torch.ones(1, device=DEV)
    for lam in (None, one):
        a = cuda_ops.soft_cross_entropy(z, y, lam, 0.0)
        b = cuda_ops.cross_entropy(z, y)
        assert float(a) == pytest.approx(float(b), rel=1e-6)
        ga, = torch.autograd.grad(a, z)
        gb, = torch.autograd.grad(b, z)
        torch.testing.assert_close(ga, gb, rtol=1e-5, atol=1e-6)
    before = cuda_ops.launch_count()
    losses.cross_entropy(z, y).backward()                      # the default dispatch: the hard-label kernels
    assert cuda_ops.launch_count() - before == 2


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


def test_kernels_per_replay():
    """Smoothing or mixing swaps the two cross-entropy kernels for the soft-target ones: the count stays."""
    counts = {}
    for name, kw in (("default", {}), ("smoothing", dict(label_smoothing=0.1)), ("mixup", dict(mixup_alpha=0.2)),
                     ("cutmix", dict(cutmix_alpha=1.0))):
        eng, _ = _run(federated_multi, K=1, Nadmm=1, max_minibatches=5, graphs=True, **kw)
        counts[name] = sorted({gs.kernels_per_replay for gs in eng._graphs.values() if isinstance(gs, GraphedAdamStep)})
    print(counts)
    assert counts["default"] and all(c == counts["default"] for c in counts.values())


_LIB = ("cudnn", "cutlass", "cublas", "sgemm", "xmma", "implicit_gemm", "gemv", "gemmk1")


@pytest.mark.parametrize("lam", [False, True])
def test_graphed_step_launches_no_library_kernel_and_shows_the_soft_ce_kernels(lam):
    from federated_pytorch_test_b200.optim.block_adam import BlockAdam
    from federated_pytorch_test_b200.utils.flat import FlatArena

    torch.manual_seed(0)
    net = models.ResNet18().to(DEV)
    arena = FlatArena(net, device=DEV, channels_last_weights=True)
    for p in net.parameters():
        p.requires_grad = True
    arena.attach_grads()
    opt = BlockAdam(arena, 0, len(arena.params) - 1, lr=1e-3)
    x = torch.rand(128, 3, 32, 32, device=DEV).contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 10, (128,), device=DEV)
    lam_t = torch.full((1,), 0.75, device=DEV) if lam else None

    def body():
        arena.zero_grads()
        with cuda_ops.accumulate_into_grad():
            losses.cross_entropy(net(x), y, 0.1, lam_t).backward()
        opt.apply_update()

    for _ in range(3):
        body()
    graph, _ = capture_graph(torch.cuda.Stream(), body)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        if lam:
            lam_t.fill_(0.5)
        graph.replay()
        torch.cuda.synchronize()
    names = [e.key for e in prof.key_averages()]
    lib = [n for n in names if any(t in n.lower() for t in _LIB)]
    assert not lib, lib
    assert any("soft_ce_fwd_kernel" in n for n in names) and any("soft_ce_bwd_kernel" in n for n in names), names
    assert not any("ce_fwd_kernel" in n and "soft" not in n for n in names), names


def test_graphed_run_equals_eager_run_and_captures_once(monkeypatch):
    captures = []
    orig = GraphedAdamStep._capture

    def counting(self):
        captures.append(self)
        orig(self)
    monkeypatch.setattr(GraphedAdamStep, "_capture", counting)
    ea, a = _run(federated_multi, **FLAGS, graphs=False)
    eb, b = _run(federated_multi, **FLAGS, graphs=True)
    graphs = [gs for gs in eb._graphs.values() if isinstance(gs, GraphedAdamStep)]
    assert eb.graph_replays > 0 and len(captures) == len(graphs) == 2 * 10      # once per (replica, block)
    assert all(len(gs.static) == 3 for gs in graphs)
    da, db = _duals(a), _duals(b)
    assert len(da) == len(db) == 20
    for u, v in zip(da, db):
        assert v == pytest.approx(u, rel=5e-2, abs=1e-7)
    assert all(ld.aug_counter > 0 for ld in eb.task._loaders.values())


@pytest.mark.parametrize("mod,extra", [(federated_multi, {}), (fedprox_multi, {}), (consensus_multi, dict(bb_update=True)),
                                       (no_consensus_multi, dict(Nepoch=3))],
                         ids=["fedavg", "fedprox", "admm_bb", "no_consensus"])
def test_resnet18_mixing_fused_equals_aten(mod, extra):
    e1, l_fast = _run(mod, **FLAGS, **extra, graphs=True)
    e2, l_aten = _run(mod, **FLAGS, **extra, graphs=False, fast=False)
    assert e1.graph_replays > 0
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


def test_lbfgs_graphed_closure_with_mixing_equals_eager():
    kw = dict(K=2, Nloop=1, Nadmm=2, max_minibatches=4, model="Net", default_batch=32, optimizer="lbfgs", mixup_alpha=0.2,
              label_smoothing=0.1)
    ea, a = _run(fedprox_multi, **kw, graphs=False)
    ea2, a2 = _run(fedprox_multi, **kw, graphs=False)
    eb, b = _run(fedprox_multi, **kw, graphs=True)
    assert eb.graph_replays > 0 and ea.graph_replays == 0
    ra, ra2, rb = _residuals(a), _residuals(a2), _residuals(b)
    assert len(ra) == len(rb) == 5 * 2
    spread = max(abs(u - v) / max(abs(u), 1e-12) for x, y in zip(ra, ra2) for u, v in zip(x, y))     # eager vs eager
    print("eager-vs-eager relative spread of the residuals: %.2e" % spread)
    for (pa, da), (pb, db) in zip(ra, rb):
        assert pa == pytest.approx(pb, rel=max(5e-2, 5 * spread), abs=1e-7)
        assert da == pytest.approx(db, rel=max(5e-2, 5 * spread), abs=1e-7)
    ident, gc_ = eb._graphs[("lbfgs", eb.replicas[0].ck)]
    assert len(gc_.static) == 3 and gc_.graph[True] is not None


def test_resnet18_cutmix_smoothing_training_beats_chance():
    lines = []
    cfg = federated_multi.Config(K=2, model="ResNet18", Nloop=1, Nadmm=1, max_minibatches=12, check_results=True,
                                 save_model=False, train_size=4096, test_size=1000, augment=True, cutmix_alpha=1.0,
                                 label_smoothing=0.1)
    federated_multi.run(cfg, log=lines.append)
    accs = [float(l.rsplit("%", 1)[1]) for l in lines if l.startswith("Accuracy of the network")]
    print("test accuracy after each block visit (%):", accs)
    assert len(accs) == 20
    # chance is 10 %; an H100 run of this configuration ended at 100 % (rising from 6 % after the first block visit)
    assert accs[-1] >= 50.0
