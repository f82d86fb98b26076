"""Training augmentation (random 4-pixel-padded crop + horizontal flip) on CPU: the counter-based draws, the ATen
composition against a literal per-sample loop, the loader, the configuration and end-to-end runs (determinism,
true resume, two gloo processes == one process)."""
import os

import numpy as np
import pytest
import torch

from federated_pytorch_test_b200.api import (federated_cpc, federated_multi, federated_vae, federated_vae_cl)
from federated_pytorch_test_b200.config import FederatedConfig, parse_config
from federated_pytorch_test_b200.data import (ShardLoader, augment_batch, augment_draws, augment_key, make_synthetic_cifar,
                                              normalize_batch, worker_norm)

TINY = dict(train_size=1024, test_size=128, save_model=False, graphs=False, fast=False)
M64 = (1 << 64) - 1


def _splitmix_word(key, c):
    """Output c of splitmix64 seeded with key, in plain Python integers."""
    z = (key + (c + 1) * 0x9E3779B97F4A7C15) & M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


@pytest.mark.parametrize("key,counter", [(0, 0), (augment_key(69, 3), 6249), (M64, (1 << 32) - 5), (0x123456789ABCDEF0, 3 << 40)])
def test_draws_match_the_documented_hash(key, counter):
    dx, dy, flip = augment_draws(key, counter, 64)
    for i in range(64):
        z = _splitmix_word(key, counter + i)
        assert int(dx[i]) == ((z & 0xFFFFFFFF) * 9) >> 32
        assert int(dy[i]) == (((z >> 32) & 0x7FFFFFFF) * 9) >> 31
        assert bool(flip[i]) == bool(z >> 63)


def test_draws_are_deterministic_in_range_and_uniform():
    key = augment_key(69, 0)
    n = 100_000
    dx, dy, flip = augment_draws(key, 12345, n)
    a = augment_draws(key, 12345, n)
    assert torch.equal(dx, a[0]) and torch.equal(dy, a[1]) and torch.equal(flip, a[2])
    assert dx.dtype == dy.dtype == torch.int64 and flip.dtype == torch.bool
    assert int(dx.min()) == 0 and int(dx.max()) == 8 and int(dy.min()) == 0 and int(dy.max()) == 8
    for d in (dx, dy):
        rate = torch.bincount(d, minlength=9).double() / n
        assert ((rate - 1 / 9).abs() < 0.1 / 9).all(), rate
    assert 0.49 <= float(flip.double().mean()) <= 0.51
    # a window of the sequence is the sequence from a later counter
    tail = augment_draws(key, 12345 + 1000, 10)
    assert torch.equal(tail[0], dx[1000:1010]) and torch.equal(tail[2], flip[1000:1010])
    assert augment_key(69, 0) != augment_key(69, 1) != augment_key(70, 1)


def _literal(u8, mean, std, key, counter):
    """Per-sample numpy loop: zero-pad by 4, crop at (dy, dx), flip, normalise; returns NCHW float32."""
    dx, dy, flip = augment_draws(key, counter, u8.shape[0])
    x = u8.numpy()
    out = np.empty((x.shape[0], 3, 32, 32), dtype=np.float32)
    m = np.asarray(mean, dtype=np.float32)
    s = np.asarray(std, dtype=np.float32)
    for i in range(x.shape[0]):
        pad = np.zeros((40, 40, 3), dtype=np.uint8)
        pad[4:36, 4:36] = x[i]
        crop = pad[int(dy[i]):int(dy[i]) + 32, int(dx[i]):int(dx[i]) + 32]
        if flip[i]:
            crop = crop[:, ::-1]
        img = (crop.astype(np.float32) / np.float32(255.0) - m) / s
        out[i] = img.transpose(2, 0, 1)
    return torch.from_numpy(out)


@pytest.mark.parametrize("channels_last", [False, True])
def test_augment_batch_equals_literal_loop(channels_last):
    u8, _ = make_synthetic_cifar(True, seed=5, size=37)
    mean, std = worker_norm(2)
    key = augment_key(69, 2)
    for counter in (0, 37, (1 << 33) + 7):
        got = augment_batch(u8, mean, std, channels_last, key, counter)
        assert got.shape == (37, 3, 32, 32) and got.dtype == torch.float32
        assert got.is_contiguous(memory_format=torch.channels_last if channels_last else torch.contiguous_format)
        assert torch.equal(got.contiguous(), _literal(u8, mean, std, key, counter))


def test_padding_normalises_to_minus_mean_over_std():
    u8 = torch.full((64, 32, 32, 3), 200, dtype=torch.uint8)
    mean, std = worker_norm(4)
    x = augment_batch(u8, mean, std, False, augment_key(1, 0), 0)
    dx, dy, _ = augment_draws(augment_key(1, 0), 0, 64)
    i = int(torch.nonzero((dy == 0) & (dx == 0))[0])       # shifted down and right by 4: top rows come from the padding
    for c in range(3):
        assert float(x[i, c, 0, 10]) == pytest.approx(-mean[c] / std[c], rel=1e-6)
        assert float(x[i, c, 20, 20]) == pytest.approx((200 / 255 - mean[c]) / std[c], rel=1e-6)


def test_loader_same_labels_different_images_and_keys():
    imgs, labs = make_synthetic_cifar(True, seed=1, size=1000)
    mean, std = worker_norm(0)

    def loader(augment, key=augment_key(69, 0)):
        return ShardLoader(imgs, labs, range(100, 400), 128, torch.device("cpu"), mean, std, seed=3, augment=augment,
                           aug_key=key)

    plain, aug, aug2, other = loader(False), loader(True), loader(True), loader(True, augment_key(69, 1))
    for epoch in range(2):
        for (x0, y0), (x1, y1), (x2, y2), (x3, y3) in zip(plain, aug, aug2, other):
            assert torch.equal(y0, y1) and torch.equal(y1, y2) and torch.equal(y1, y3)
            assert x1.shape == x0.shape and not torch.equal(x0, x1)
            assert torch.equal(x1, x2) and not torch.equal(x1, x3)
    assert plain.aug_counter == 0 and aug.aug_counter == 2 * 300
    # batch b of an epoch is the augmentation of exactly its samples at the loader's counter
    ld = loader(True)
    order = ShardLoader(imgs, labs, range(100, 400), 128, torch.device("cpu"), mean, std, seed=3)._order()
    for b, (x, _) in enumerate(ld):
        idx = order[b * 128:(b + 1) * 128]
        assert torch.equal(x, augment_batch(imgs[idx], mean, std, False, augment_key(69, 0), b * 128))


def test_task_augments_training_loaders_only():
    from federated_pytorch_test_b200.api import common
    from federated_pytorch_test_b200.parallel.topology import Topology

    cfg = federated_multi.Config(K=2, use_cuda=False, augment=True, **TINY)
    task = common.ClassifierTask(cfg, Topology.single_process(2, torch.device("cpu")))
    assert task.loader(0).augment and task.loader(1).augment and task.loader(0).aug_key != task.loader(1).aug_key
    assert task.loader(1).aug_key == augment_key(cfg.seed, 1)
    te = task.test_loader(1)
    assert not te.augment
    mean, std = worker_norm(1)
    x, _ = next(iter(te))
    assert torch.equal(x, normalize_batch(task.data.test_images[:128], mean, std))


def test_augment_flag_parses_and_non_classifier_drivers_refuse_it():
    assert parse_config(FederatedConfig, ["--augment"]).augment is True
    assert parse_config(FederatedConfig, []).augment is False
    assert parse_config(FederatedConfig, ["--augment=false"]).augment is False
    for mod in (federated_vae, federated_vae_cl, federated_cpc):
        with pytest.raises(ValueError, match="augment"):
            mod.run(mod.Config(**{**TINY, "use_cuda": False, "augment": True, "max_minibatches": 1}), log=lambda s: None)


# ------------------------------------------------------------------------------------------ end to end
def _run(**kw):
    lines = []
    eng = federated_multi.run(federated_multi.Config(**{**TINY, **kw}), log=lines.append)
    return eng, [l for l in lines if l.startswith("dual (")]


KW = dict(K=2, Nloop=1, Nadmm=2, max_minibatches=2, check_results=False, use_cuda=False)


def test_federated_multi_with_augmentation_is_deterministic_and_differs():
    e1, a = _run(augment=True, **KW)
    _, b = _run(augment=True, **KW)
    _, c = _run(augment=False, **KW)
    assert len(a) == 10 and a == b
    assert a != c
    assert all(float(l.rsplit("=", 1)[1]) == float(l.rsplit("=", 1)[1]) for l in a)
    assert all(ld.aug_counter > 0 for ld in e1.task._loaders.values())


class _Killed(Exception):
    pass


def test_kill_and_resume_with_augmentation_reproduces_the_trace(tmp_path):
    from federated_pytorch_test_b200.algo.engine import Engine

    kw = dict(KW, Nadmm=3, augment=True)
    _, full = _run(**kw)
    assert len(full) == 15
    rec = str(tmp_path / "resume.pt")
    kill_at = 2 * 2 * (3 + 2) - 1
    orig_init = Engine.__init__

    def patched(self, *a, **k):
        orig_init(self, *a, **k)

        def hook(e):
            if e.steps_done == kill_at:
                raise _Killed()
        self.step_hook = hook
    Engine.__init__ = patched
    first = []
    try:
        with pytest.raises(_Killed):
            federated_multi.run(federated_multi.Config(**{**TINY, **kw, "resume_out": rec}), log=first.append)
    finally:
        Engine.__init__ = orig_init
    first = [l for l in first if l.startswith("dual (")]
    assert 0 < len(first) < 15 and os.path.exists(rec)
    assert all(st["aug_counter"] > 0 for st in torch.load(rec, weights_only=False)["loader_rng"].values())
    _, second = _run(**kw, resume=rec)
    assert first + second == full


def test_resume_record_without_counter_restores_zero(tmp_path):
    from federated_pytorch_test_b200.utils import ckpt

    rec = str(tmp_path / "resume.pt")
    _run(**dict(KW, Nadmm=1, augment=True, resume_out=rec))
    r = torch.load(rec, weights_only=False)
    for st in r["loader_rng"].values():
        st.pop("aug_counter")
    torch.save(r, rec)

    class _Probe(Exception):
        pass

    orig = ckpt.load_resume

    def load_and_stop(path, engine):
        orig(path, engine)
        raise _Probe([engine.task.loader(ck).aug_counter for ck in (0, 1)])
    ckpt.load_resume = load_and_stop
    try:
        with pytest.raises(_Probe) as got:
            _run(**dict(KW, Nadmm=1, augment=True, resume=rec))
    finally:
        ckpt.load_resume = orig
    assert got.value.args[0] == [0, 0]


def _dist_worker(rank, world, port, out):
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch.distributed as dist
    lines = []
    cfg = federated_multi.Config(K=2, Nloop=1, Nadmm=2, max_minibatches=2, check_results=False, use_cuda=False,
                                 augment=True, **TINY)
    eng = federated_multi.run(cfg, log=lines.append)
    if rank == 0:
        torch.save({"lines": lines, "flat": eng.replicas[0].arenas["net"].data.clone()}, out)
    dist.destroy_process_group()


def test_two_process_gloo_with_augmentation_equals_single_process(tmp_path):
    import torch.multiprocessing as mp
    out = str(tmp_path / "r0.pt")
    port = 33500 + (os.getpid() % 2000)
    mp.spawn(_dist_worker, args=(2, port, out), nprocs=2, join=True)
    got = torch.load(out, weights_only=False)
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        os.environ.pop(k, None)
    eng, single = _run(augment=True, **KW)
    multi = [l for l in got["lines"] if l.startswith("dual (")]
    assert len(single) == len(multi) == 10
    for a, b in zip(single, multi):
        assert a.split("=")[:-1] == b.split("=")[:-1]
        assert float(a.rsplit("=", 1)[1]) == pytest.approx(float(b.rsplit("=", 1)[1]), rel=1e-4)
    torch.testing.assert_close(got["flat"], eng.replicas[0].arenas["net"].data, rtol=1e-4, atol=1e-6)
