"""Label smoothing, mixup and CutMix (``--label_smoothing``, ``--mixup_alpha``, ``--cutmix_alpha``) on CPU: configuration,
the counter-based per-batch draws and their distributions, the ATen mixing against a per-pixel transcription, the soft-target
loss against float64, the loaders, and true resume."""
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from federated_pytorch_test_b200.api import common, federated_cpc, federated_multi, federated_vae, federated_vae_cl
from federated_pytorch_test_b200.config import FederatedConfig, check_mix, parse_config
from federated_pytorch_test_b200.data import (ShardLoader, augment_batch, augment_key, make_synthetic_cifar, mix_batch,
                                              mix_draws, mix_key, normalize_batch, worker_norm)
from federated_pytorch_test_b200.ops import losses
from federated_pytorch_test_b200.parallel import Topology

CPU = torch.device("cpu")
TINY = dict(train_size=1024, test_size=128, save_model=False, graphs=False, fast=False)
KW = dict(K=2, Nloop=1, Nadmm=2, max_minibatches=2, check_results=False, use_cuda=False)
MIX = dict(mixup_alpha=0.2, label_smoothing=0.1)
M64 = (1 << 64) - 1


# ------------------------------------------------------------------------------------------ configuration
@pytest.mark.parametrize("kw,field", [(dict(label_smoothing=-0.1), "label_smoothing"), (dict(label_smoothing=1.0), "label_smoothing"),
                                      (dict(label_smoothing=float("nan")), "label_smoothing"),
                                      (dict(mixup_alpha=-1.0), "mixup_alpha"), (dict(mixup_alpha=float("inf")), "mixup_alpha"),
                                      (dict(cutmix_alpha=-0.5), "cutmix_alpha"), (dict(cutmix_alpha=float("nan")), "cutmix_alpha")])
def test_check_mix_rejects_bad_values(kw, field):
    args = {**dict(label_smoothing=0.0, mixup_alpha=0.0, cutmix_alpha=0.0), **kw}
    with pytest.raises(ValueError, match=field):
        check_mix(**args)
    with pytest.raises(ValueError, match=field):
        common.ClassifierTask(federated_multi.Config(K=2, use_cuda=False, **TINY, **kw), Topology.single_process(2, CPU))
    check_mix(0.0, 0.0, 0.0)
    check_mix(0.999, 1e-3, 1e3)


def test_flags_parse_and_default_off():
    cfg = parse_config(FederatedConfig, [])
    assert (cfg.label_smoothing, cfg.mixup_alpha, cfg.cutmix_alpha) == (0.0, 0.0, 0.0)
    cfg = parse_config(FederatedConfig, ["--label_smoothing", "0.1", "--mixup_alpha", "0.2", "--cutmix_alpha", "1"])
    assert (cfg.label_smoothing, cfg.mixup_alpha, cfg.cutmix_alpha) == (0.1, 0.2, 1.0)


@pytest.mark.parametrize("field,val", [("label_smoothing", 0.1), ("mixup_alpha", 0.2), ("cutmix_alpha", 1.0)])
@pytest.mark.parametrize("mod,task", [(federated_vae, "VAETask"), (federated_vae_cl, "VAECLTask"), (federated_cpc, "CPCTask")])
def test_unsupervised_drivers_reject_the_flags(mod, task, field, val):
    with pytest.raises(ValueError, match="%s is supported by the classifier drivers only, not by %s" % (field, task)):
        mod.run(mod.Config(**{**TINY, "use_cuda": False, "max_minibatches": 1, field: val}), log=lambda s: None)


# ------------------------------------------------------------------------------------------ draws
def _splitmix_word(key, i):
    z = (key + (i + 1) * 0x9E3779B97F4A7C15) & M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


@pytest.mark.parametrize("counter", [0, 6249, (1 << 32) - 5, (1 << 32) + 128, 3 << 40, M64])
def test_draws_are_reproducible_and_follow_the_documented_words(counter):
    key = mix_key(69, 3)
    a = mix_draws(key, counter, 128, 32, 32, 0.2, 1.0)
    assert a == mix_draws(key, counter, 128, 32, 32, 0.2, 1.0)
    w0 = _splitmix_word(key, (counter * 256) & M64)
    assert a[0] == ("cutmix" if w0 >> 63 else "mixup")
    if a[0] == "cutmix":                          # the box is centred on (cy, cx) of words 1 and 2 unless it was clipped
        cy = ((_splitmix_word(key, (counter * 256 + 1) & M64) >> 32) * 32) >> 32
        y0, y1, _, _ = a[2]
        assert y0 <= cy <= y1
    assert mix_draws(key, counter + 1, 128, 32, 32, 0.2, 1.0) != a
    assert mix_draws(mix_key(69, 4), counter, 128, 32, 32, 0.2, 1.0) != a


def test_mix_key_is_not_the_augment_key():
    keys = {mix_key(s, k) for s in (0, 69) for k in range(8)} | {augment_key(s, k) for s in (0, 69) for k in range(8)}
    assert len(keys) == 32


@pytest.mark.parametrize("alpha", [0.2, 1.0])
@pytest.mark.parametrize("mode", ["mixup", "cutmix"])
def test_lambda_is_beta_distributed(alpha, mode):
    import scipy.stats

    key = mix_key(69, 0)
    kw = dict(mixup_alpha=alpha, cutmix_alpha=0.0) if mode == "mixup" else dict(mixup_alpha=0.0, cutmix_alpha=alpha)
    draws = [mix_draws(key, 128 * c, 128, 32, 32, **kw) for c in range(20000)]
    assert {d[0] for d in draws} == {mode}
    lams = np.array([d[1] for d in draws])
    assert ((lams >= 0.0) & (lams <= 1.0)).all()
    p = scipy.stats.kstest(lams, scipy.stats.beta(alpha, alpha).cdf).pvalue
    assert p > 1e-3, p


def test_mode_split_box_and_effective_lambda():
    key = mix_key(7, 1)
    H, W = 32, 24
    draws = [mix_draws(key, c, 105, H, W, 0.2, 1.0) for c in range(0, 20000 * 105, 105)]
    share = sum(d[0] == "cutmix" for d in draws) / len(draws)
    assert 0.48 < share < 0.52, share
    for mode, lam, (y0, y1, x0, x1), lam_eff in draws:
        if mode == "mixup":
            assert lam_eff == lam and (y0, y1, x0, x1) == (0, 0, 0, 0)
            continue
        assert 0 <= y0 <= y1 <= H and 0 <= x0 <= x1 <= W
        assert lam_eff == 1.0 - (y1 - y0) * (x1 - x0) / (H * W)
        r = math.sqrt(1.0 - lam)
        assert y1 - y0 <= 2 * (int(H * r) // 2) and x1 - x0 <= 2 * (int(W * r) // 2)
    assert mix_draws(key, 0, 8, H, W, 0.0, 1.0)[0] == "cutmix" and mix_draws(key, 0, 8, H, W, 0.3, 0.0)[0] == "mixup"
    with pytest.raises(ValueError):
        mix_draws(key, 0, 8, H, W, 0.0, 0.0)


def test_tiny_alpha_gives_a_defined_lambda():
    lams = [mix_draws(mix_key(1, 0), c, 16, 32, 32, 1e-3, 0.0)[1] for c in range(200)]
    assert all(0.0 <= v <= 1.0 for v in lams) and {round(v) for v in lams} == {0, 1}


# ------------------------------------------------------------------------------------------ ATen mixing
def _literal(x, mode, lam, box):
    """Per-pixel transcription of the mixing formulas on a normalised NCHW float32 batch."""
    x = x.contiguous().numpy()
    n = x.shape[0]
    out = np.empty_like(x)
    lam_f, mlam_f = np.float32(lam), np.float32(1.0 - lam)
    y0, y1, x0, x1 = box
    for i in range(n):
        j = n - 1 - i
        for h in range(x.shape[2]):
            for w in range(x.shape[3]):
                if mode == "mixup":
                    out[i, :, h, w] = (lam_f * x[i, :, h, w]).astype(np.float32) + (mlam_f * x[j, :, h, w]).astype(np.float32)
                else:
                    out[i, :, h, w] = x[j, :, h, w] if (y0 <= h < y1 and x0 <= w < x1) else x[i, :, h, w]
    return torch.from_numpy(out)


@pytest.mark.parametrize("augment", [False, True])
@pytest.mark.parametrize("channels_last", [False, True])
@pytest.mark.parametrize("alphas", [(0.4, 0.0), (0.0, 1.0)], ids=["mixup", "cutmix"])
def test_mix_batch_equals_per_pixel_transcription(augment, channels_last, alphas):
    u8, _ = make_synthetic_cifar(True, seed=5, size=9)
    mean, std = worker_norm(2)
    akey, key = augment_key(69, 2), mix_key(69, 2)
    for counter in (0, 9, (1 << 33) + 7):
        got, lam_t = mix_batch(u8, mean, std, channels_last, akey if augment else None, key, counter, *alphas)
        mode, lam, box, lam_eff = mix_draws(key, counter, 9, 32, 32, *alphas)
        base = augment_batch(u8, mean, std, False, akey, counter) if augment else normalize_batch(u8, mean, std)
        assert got.shape == (9, 3, 32, 32) and got.dtype == torch.float32
        assert got.is_contiguous(memory_format=torch.channels_last if channels_last else torch.contiguous_format)
        assert torch.equal(got.contiguous(), _literal(base, mode, lam, box))
        assert lam_t.dtype == torch.float32 and lam_t.shape == (1,) and float(lam_t) == float(np.float32(lam_eff))
        assert mode != "cutmix" or box[1] > box[0]     # alpha = 1: a box this small would be rare at these counters


# ------------------------------------------------------------------------------------------ loss
def _soft_targets(y, lam, eps, C):
    s = (1.0 - eps) * F.one_hot(y, C).double() + eps / C
    return lam * s + (1.0 - lam) * s.flip(0)


@pytest.mark.parametrize("B,C", [(1, 10), (105, 10), (128, 100)])
@pytest.mark.parametrize("eps,lam", [(0.1, None), (0.0, 0.3), (0.1, 0.7), (0.2, 1.0)])
def test_cpu_loss_and_gradient_equal_float64_soft_targets(B, C, eps, lam):
    g = torch.Generator().manual_seed(B * C)
    z = (3.0 * torch.randn(B, C, generator=g)).requires_grad_()
    y = torch.randint(0, C, (B,), generator=g)
    lam_t = None if lam is None else torch.tensor([lam], dtype=torch.float32)
    loss = losses.cross_entropy(z, y, eps, lam_t)
    (gz,) = torch.autograd.grad(loss, z)
    z64 = z.detach().double().requires_grad_()
    q = _soft_targets(y, 1.0 if lam is None else float(np.float32(lam)), eps, C)
    ref = F.cross_entropy(z64, q)
    (gref,) = torch.autograd.grad(ref, z64)
    assert float(loss.detach()) == pytest.approx(float(ref.detach()), rel=1e-5)
    torch.testing.assert_close(gz.double(), gref, rtol=1e-5, atol=1e-7)


def test_cpu_loss_without_smoothing_or_mixing_is_plain_cross_entropy():
    z = torch.randn(64, 10)
    y = torch.randint(0, 10, (64,))
    assert torch.equal(losses.cross_entropy(z, y), F.cross_entropy(z, y))
    assert torch.equal(losses.cross_entropy(z, y, 0.0, None), F.cross_entropy(z, y))


# ------------------------------------------------------------------------------------------ loaders
def test_default_loader_is_unchanged():
    cfg = federated_multi.Config(K=2, use_cuda=False, **TINY)
    task = common.ClassifierTask(cfg, Topology.single_process(2, CPU))
    ld = task.loader(0)
    assert not ld.mixing
    batches = list(ld)
    assert all(len(b) == 2 for b in batches) and ld.aug_counter == 0


def test_mixing_loader_yields_lam_and_advances_the_counter():
    imgs, labs = make_synthetic_cifar(True, seed=1, size=1000)
    mean, std = worker_norm(0)
    kw = dict(seed=3, mixup_alpha=0.2, cutmix_alpha=1.0, mix_key=mix_key(69, 0))
    plain = ShardLoader(imgs, labs, range(100, 400), 128, CPU, mean, std, seed=3)
    mixed = ShardLoader(imgs, labs, range(100, 400), 128, CPU, mean, std, **kw)
    order = ShardLoader(imgs, labs, range(100, 400), 128, CPU, mean, std, seed=3)._order()
    for epoch in range(2):
        for b, ((x0, y0), (x, y, lam)) in enumerate(zip(plain, mixed)):
            assert torch.equal(y0, y) and x.shape == x0.shape
            counter = epoch * 300 + b * 128
            if epoch == 0:
                idx = order[b * 128:(b + 1) * 128]
                want, wlam = mix_batch(imgs[idx], mean, std, False, None, mix_key(69, 0), counter, 0.2, 1.0)
                assert torch.equal(x, want) and torch.equal(lam, wlam)
    assert plain.aug_counter == 0 and mixed.aug_counter == 600


def test_task_mixes_training_loaders_only():
    cfg = federated_multi.Config(K=2, use_cuda=False, cutmix_alpha=1.0, **TINY)
    task = common.ClassifierTask(cfg, Topology.single_process(2, CPU))
    assert task.loader(1).mixing and task.loader(1).mix_key == mix_key(cfg.seed, 1)
    assert not task.test_loader(1).mixing
    assert len(next(iter(task.loader(0)))) == 3 and len(next(iter(task.test_loader(0)))) == 2


# ------------------------------------------------------------------------------------------ end to end
def _run(**kw):
    lines = []
    eng = federated_multi.run(federated_multi.Config(**{**TINY, **kw}), log=lines.append)
    return eng, [l for l in lines if l.startswith("dual (")]


def test_federated_multi_with_mixing_is_deterministic_and_differs():
    e1, a = _run(**KW, **MIX, augment=True)
    _, b = _run(**KW, **MIX, augment=True)
    _, c = _run(**KW, augment=True)
    _, d = _run(**KW, label_smoothing=0.1)
    assert len(a) == 10 and a == b and a != c and d != c
    assert all(ld.aug_counter > 0 for ld in e1.task._loaders.values())


class _Killed(Exception):
    pass


def _killed_run(kw, kill_at):
    from federated_pytorch_test_b200.algo.engine import Engine

    orig_init = Engine.__init__

    def patched(self, *a, **k):
        orig_init(self, *a, **k)

        def hook(e):
            if e.steps_done == kill_at:
                raise _Killed()
        self.step_hook = hook
    Engine.__init__ = patched
    lines = []
    try:
        with pytest.raises(_Killed):
            federated_multi.run(federated_multi.Config(**{**TINY, **kw}), log=lines.append)
    finally:
        Engine.__init__ = orig_init
    return [l for l in lines if l.startswith("dual (")]


def test_kill_and_resume_with_mixing_reproduces_the_run(tmp_path):
    kw = dict(KW, Nadmm=3, **MIX)
    eng, full = _run(**kw)
    assert len(full) == 15
    rec = str(tmp_path / "resume.pt")
    first = _killed_run({**kw, "resume_out": rec}, 2 * 2 * (3 + 2) - 1)
    assert 0 < len(first) < 15 and os.path.exists(rec)
    st = torch.load(rec, weights_only=False)
    assert st["position"]["recipe"]["mixup_alpha"] == 0.2 and st["position"]["recipe"]["label_smoothing"] == 0.1
    assert all(s["aug_counter"] > 0 for s in st["loader_rng"].values())
    eng2, second = _run(**kw, resume=rec)
    assert first + second == full
    assert torch.equal(eng.replicas[0].arenas["net"].data, eng2.replicas[0].arenas["net"].data)


def test_resume_record_without_mixing_keys_resumes_and_other_settings_raise(tmp_path):
    rec = str(tmp_path / "r.pt")
    _killed_run({**KW, **MIX, "resume_out": rec}, 6)
    with pytest.raises(ValueError, match="mixup_alpha"):
        _run(**KW, **dict(MIX, mixup_alpha=0.4), resume=rec)
    with pytest.raises(ValueError, match="cutmix_alpha"):
        _run(**KW, **MIX, cutmix_alpha=1.0, resume=rec)
    plain = str(tmp_path / "plain.pt")              # as written before mixing existed: no mixing keys in the recipe
    _killed_run({**KW, "resume_out": plain}, 6)
    st = torch.load(plain, weights_only=False)
    for name in ("label_smoothing", "mixup_alpha", "cutmix_alpha"):
        del st["position"]["recipe"][name]
    torch.save(st, plain)
    _, lines = _run(**KW, resume=plain)
    assert len(lines) > 0
    with pytest.raises(ValueError, match="label_smoothing"):
        _run(**KW, label_smoothing=0.1, resume=plain)
