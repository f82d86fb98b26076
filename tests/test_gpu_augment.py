"""Training augmentation on the H100: the fused gather + crop + flip + normalise kernel against the ATen composition
(bit for bit on the normalisation of the oracle's augmented uint8 batch), device- vs host-resident loaders, its launch
count, and ResNet18 federated_multi runs with ``augment=True``."""
import pytest
import torch

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():  # collected (and deselected) on the CPU box
    pytest.skip("CUDA device required", allow_module_level=True)

from federated_pytorch_test_b200.data import (ShardLoader, augment_batch, augment_key, augment_u8,  # noqa: E402
                                              make_synthetic_cifar, worker_norm)
from federated_pytorch_test_b200.ops import cuda_ops  # noqa: E402
from federated_pytorch_test_b200.ops import functional as FX  # noqa: E402

DEV = torch.device("cuda", 0)
COUNTERS = [0, 6249, (1 << 32) - 3, (1 << 32) + 11, 3 << 40]


@pytest.fixture(autouse=True)
def _fast_path():
    FX.set_fast_path(True)
    yield
    FX.set_fast_path(True)


@pytest.fixture(scope="module")
def data():
    imgs, labs = make_synthetic_cifar(True, seed=11, size=2000)
    return imgs.to(DEV), labs.to(DEV)


@pytest.mark.parametrize("channels_last", [False, True])
@pytest.mark.parametrize("n", [128, 105])
def test_kernel_is_bit_identical_to_normalize_of_oracle_crop(data, n, channels_last):
    imgs, _ = data
    mean, std = worker_norm(3)
    g = torch.Generator().manual_seed(n)
    for ck, counter in enumerate(COUNTERS):
        key = augment_key(69, ck)
        idx = torch.randperm(imgs.shape[0], generator=g)[:n].to(DEV)
        want = cuda_ops.normalize_u8(augment_u8(imgs.index_select(0, idx), key, counter), mean, std, channels_last)
        gathered = cuda_ops.augment_normalize_u8(imgs, idx, key, counter, mean, std, channels_last)   # index-gather mode
        batch = cuda_ops.augment_normalize_u8(imgs.index_select(0, idx), None, key, counter, mean, std, channels_last)
        for got in (gathered, batch):
            assert got.shape == (n, 3, 32, 32) and got.stride() == want.stride()
            assert torch.equal(got, want), (n, channels_last, counter)


def test_crop_at_centre_without_flip_reproduces_normalize_u8(data):
    """A draw of (dx, dy) = (4, 4) without a flip is the identity crop: the kernel's arithmetic is normalize_u8's."""
    from federated_pytorch_test_b200.data import augment_draws

    imgs, _ = data
    key = augment_key(5, 0)
    dx, dy, flip = augment_draws(key, 0, imgs.shape[0])
    ident = torch.nonzero((dx == 4) & (dy == 4) & ~flip).flatten()
    assert ident.numel() > 5
    out = cuda_ops.augment_normalize_u8(imgs, torch.arange(imgs.shape[0], device=DEV), key, 0, *worker_norm(2), False)
    ref = cuda_ops.normalize_u8(imgs, *worker_norm(2), False)
    assert torch.equal(out[ident.to(DEV)], ref[ident.to(DEV)])


@pytest.mark.parametrize("channels_last", [False, True])
def test_kernel_matches_aten_composition(data, channels_last):
    imgs, _ = data
    mean, std = worker_norm(7)
    idx = torch.randperm(imgs.shape[0], generator=torch.Generator().manual_seed(1))[:105].to(DEV)
    for counter in (0, (1 << 32) + 11):
        key = augment_key(69, 7)
        got = cuda_ops.augment_normalize_u8(imgs, idx, key, counter, mean, std, channels_last)
        FX.set_fast_path(False)
        ref = augment_batch(imgs.index_select(0, idx), mean, std, channels_last, key, counter)
        FX.set_fast_path(True)
        torch.testing.assert_close(got, ref, rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("channels_last", [False, True])
def test_host_resident_loader_with_augmentation_matches_device_resident(channels_last):
    imgs, labs = make_synthetic_cifar(True, seed=3, size=1000)
    mean, std = worker_norm(1)
    kw = dict(seed=5, channels_last=channels_last, augment=True, aug_key=augment_key(69, 1))
    a = ShardLoader(imgs.to(DEV), labs.to(DEV), range(0, 900), 128, DEV, mean, std, **kw)
    b = ShardLoader(imgs.pin_memory(), labs.pin_memory(), range(0, 900), 128, DEV, mean, std, **kw)
    assert b.host_resident and b._assembler.native
    n = 0
    for epoch in range(2):
        for (xa, ya), (xb, yb) in zip(a, b):
            assert torch.equal(xa, xb) and torch.equal(ya, yb)
            n += ya.numel()
    assert n == 1800 and a.aug_counter == b.aug_counter == 1800


def test_augmented_device_batch_is_one_handwritten_launch(data):
    imgs, labs = data
    ld = ShardLoader(imgs, labs, range(0, 1500), 128, DEV, *worker_norm(0), seed=1, channels_last=True, augment=True,
                     aug_key=augment_key(69, 0))
    it = iter(ld)
    next(it)
    before = cuda_ops.launch_count()
    x, y = next(it)
    assert cuda_ops.launch_count() - before == 1
    assert x.shape == (128, 3, 32, 32) and x.is_contiguous(memory_format=torch.channels_last)


# ------------------------------------------------------------------------------------------ engine
def _run_fed(**kw):
    from federated_pytorch_test_b200.api import federated_multi
    lines = []
    base = dict(K=2, model="ResNet18", Nloop=1, Nadmm=2, max_minibatches=5, check_results=False, save_model=False,
                train_size=4096, test_size=256, augment=True)
    eng = federated_multi.run(federated_multi.Config(**{**base, **kw}), log=lines.append)
    return eng, lines


def test_resnet18_augmented_graphed_equals_eager():
    e1, l_graph = _run_fed(graphs=True)
    _, l_eager = _run_fed(graphs=False)
    d_graph = [float(l.rsplit("=", 1)[1]) for l in l_graph if l.startswith("dual (")]
    d_eager = [float(l.rsplit("=", 1)[1]) for l in l_eager if l.startswith("dual (")]
    assert len(d_graph) == len(d_eager) == 20
    for a, b in zip(d_graph, d_eager):
        assert a == pytest.approx(b, rel=2e-2)
    assert getattr(e1, "graph_replays", 0) > 0
    assert all(ld.aug_counter > 0 for ld in e1.task._loaders.values())


def test_resnet18_augmented_training_beats_chance():
    _, lines = _run_fed(Nadmm=1, max_minibatches=12, check_results=True, test_size=1000)
    accs = [float(l.rsplit("%", 1)[1]) for l in lines if l.startswith("Accuracy of the network")]
    print("test accuracy after each block visit (%):", accs)
    assert len(accs) == 20
    # chance is 10 %; an H100 run of this configuration ended at 99 % (rising from 6 % after the first block visit)
    assert accs[-1] >= 80.0
