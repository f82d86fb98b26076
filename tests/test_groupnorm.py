"""GroupNorm ResNets (``--norm group``) on CPU: the model keeps the BatchNorm model's parameter layout, the ATen composition
of a conv + GroupNorm (+ residual) (+ ELU) group against float64, configuration errors, an end-to-end federated run,
legacy checkpoints of the other norm, and the resume record."""
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from federated_pytorch_test_b200 import models
from federated_pytorch_test_b200.api import common, federated_multi
from federated_pytorch_test_b200.config import CPCConfig, FederatedConfig, VAECLConfig, VAEConfig, parse_config
from federated_pytorch_test_b200.ops import functional as FX
from federated_pytorch_test_b200.parallel import Topology
from federated_pytorch_test_b200.utils import ckpt

CPU = torch.device("cpu")
E2E = ["--K", "2", "--no-use_cuda", "--model", "ResNet9", "--norm", "group", "--Nloop", "1", "--Nadmm", "1",
       "--max_minibatches", "2", "--train_size", "512", "--test_size", "256"]


# ------------------------------------------------------------------------------------------ model
@pytest.mark.parametrize("factory", [models.ResNet18, models.ResNet9])
@pytest.mark.parametrize("groups", [1, 2, 32])
def test_group_model_has_the_batch_models_parameter_layout(factory, groups):
    bn, gn = factory(), factory(norm="group", groups=groups)
    pb, pg = list(bn.named_parameters()), list(gn.named_parameters())
    assert [(n, tuple(p.shape)) for n, p in pb] == [(n, tuple(p.shape)) for n, p in pg]
    assert bn.train_order_block_ids() == gn.train_order_block_ids()
    for lo, hi in bn.train_order_block_ids():       # block message sizes
        assert sum(p.numel() for _, p in pb[lo:hi + 1]) == sum(p.numel() for _, p in pg[lo:hi + 1])
    norms = [m for m in gn.modules() if isinstance(m, (nn.BatchNorm2d, nn.GroupNorm))]
    assert norms and all(type(m) is nn.GroupNorm and m.num_groups == groups and m.affine for m in norms)
    assert len(norms) == sum(isinstance(m, nn.BatchNorm2d) for m in bn.modules())
    assert {"bn1", "layer2.0.shortcut.1"} <= {n for n, m in gn.named_modules() if isinstance(m, nn.GroupNorm)}
    # the affine keys are the BatchNorm model's; only the running buffers are gone
    assert list(gn.state_dict()) == [k for k in bn.state_dict()
                                     if not k.endswith(("running_mean", "running_var", "num_batches_tracked"))]
    assert not list(gn.buffers())


def test_defaults_build_the_batch_model():
    for factory in (models.ResNet18, models.ResNet9):
        torch.manual_seed(3)
        a = factory()
        torch.manual_seed(3)
        b = factory(norm="batch", groups=4)
        assert repr(a) == repr(b)
        sa, sb = a.state_dict(), b.state_dict()
        assert list(sa) == list(sb) and all(torch.equal(sa[k], sb[k]) for k in sa)
    with pytest.raises(ValueError, match="norm"):
        models.ResNet9(norm="layer")


# ------------------------------------------------------------------------------------------ ATen group vs float64
@pytest.mark.parametrize("groups", [1, 2, 32])
@pytest.mark.parametrize("stride,k,residual,act", [(1, 3, False, True), (1, 3, True, True), (2, 3, False, True),
                                                   (2, 1, False, False)])
def test_conv_gn_group_matches_float64(groups, stride, k, residual, act):
    g = torch.Generator().manual_seed(groups * 100 + stride * 10 + k)
    ci, co, h, B = 16, 64, 8, 3
    x = torch.randn(B, ci, h, h, generator=g)
    conv = nn.Conv2d(ci, co, k, stride, k // 2, bias=False)
    gn = nn.GroupNorm(groups, co)
    with torch.no_grad():
        conv.weight.copy_(torch.randn(conv.weight.shape, generator=g) / (ci * k * k) ** 0.5)
        gn.weight.copy_(1 + 0.2 * torch.randn(co, generator=g))
        gn.bias.copy_(0.2 * torch.randn(co, generator=g))
    ho = (h + 2 * (k // 2) - k) // stride + 1
    r = torch.randn(B, co, ho, ho, generator=g) if residual else None
    dout = torch.randn(B, co, ho, ho, generator=g)

    xs = x.clone().requires_grad_()
    rs = r.clone().requires_grad_() if residual else None
    out = FX.conv_bn_act(xs, conv, gn, residual=rs, act=act)
    out.backward(dout)

    x64 = x.double().requires_grad_()
    w64 = conv.weight.detach().double().requires_grad_()
    g64 = gn.weight.detach().double().requires_grad_()
    b64 = gn.bias.detach().double().requires_grad_()
    r64 = r.double().requires_grad_() if residual else None
    u = F.group_norm(F.conv2d(x64, w64, None, stride, k // 2), groups, g64, b64, gn.eps)
    if residual:
        u = u + r64
    ref = F.elu(u) if act else u
    ref.backward(dout.double())

    def close(got, want):
        assert float((got.double() - want).abs().max() / want.abs().max()) < 1e-5

    close(out.detach(), ref.detach())
    close(xs.grad, x64.grad)
    close(conv.weight.grad, w64.grad)
    close(gn.weight.grad, g64.grad)
    close(gn.bias.grad, b64.grad)
    if residual:
        close(rs.grad, r64.grad)


def test_skip_group_falls_back_to_the_plain_group():
    torch.manual_seed(0)
    blk = models.BasicBlock(16, 16, 1, lambda c: nn.GroupNorm(4, c))
    x = torch.randn(2, 16, 8, 8)
    h = FX.conv_bn_act(x, blk.conv1, blk.bn1)
    assert torch.equal(h, F.elu(F.group_norm(F.conv2d(x, blk.conv1.weight, None, 1, 1), 4, blk.bn1.weight, blk.bn1.bias)))


# ------------------------------------------------------------------------------------------ configuration
def test_defaults_and_flags():
    cfg = parse_config(FederatedConfig, [])
    assert (cfg.norm, cfg.norm_groups) == ("batch", 32)
    cfg = parse_config(FederatedConfig, ["--norm", "group", "--norm_groups", "8"])
    assert (cfg.norm, cfg.norm_groups) == ("group", 8)


@pytest.mark.parametrize("flag,kw", [
    ("norm", dict(norm="layer", model="ResNet9")),
    ("norm_groups", dict(norm="group", norm_groups=3, model="ResNet9")),
    ("norm_groups", dict(norm="group", norm_groups=128, model="ResNet18")),
    ("norm_groups", dict(norm="group", norm_groups=0, model="ResNet18")),
    ("model", dict(norm="group", model="Net")),
    ("model", dict(norm="group", model="Net1")),
    ("model", dict(norm="group", model="Net2")),
    ("model", dict(norm="group", use_resnet=False)),
])
def test_invalid_norm_settings_raise(flag, kw):
    cfg = FederatedConfig(K=2, use_cuda=False, train_size=256, test_size=128, **kw)
    with pytest.raises(ValueError, match=flag):
        common.ClassifierTask(cfg, Topology.single_process(2, CPU))


@pytest.mark.parametrize("driver,cls", [("federated_vae", VAEConfig), ("federated_vae_cl", VAECLConfig),
                                        ("federated_cpc", CPCConfig)])
def test_unsupervised_drivers_accept_only_batch_norm(driver, cls):
    import importlib

    mod = importlib.import_module("federated_pytorch_test_b200.api." + driver)
    with pytest.raises(ValueError, match="norm 'batch'"):
        mod.run(cls(norm="group", use_cuda=False))


def test_eval_bn_running_is_accepted_for_group_norm():
    cfg = FederatedConfig(K=2, use_cuda=False, model="ResNet9", norm="group", eval_bn="running", train_size=256, test_size=128)
    task = common.ClassifierTask(cfg, Topology.single_process(2, CPU))
    net = task.factory()
    assert isinstance(net.bn1, nn.GroupNorm) and net.bn1.num_groups == 32


# ------------------------------------------------------------------------------------------ end to end, checkpoints, resume
@pytest.fixture(scope="module")
def e2e(tmp_path_factory):
    d = tmp_path_factory.mktemp("gn")
    rec = str(d / "resume.pt")
    lines = []
    cfg = parse_config(FederatedConfig, E2E + ["--ckpt_dir", str(d), "--resume_out", rec])
    eng = federated_multi.run(cfg, log=lines.append)
    return eng, lines, d, rec


def test_federated_multi_trains_a_group_norm_resnet9(e2e):
    eng, lines, d, _ = e2e
    net = eng.replicas[0].nets["net"]
    assert isinstance(net.bn1, nn.GroupNorm) and isinstance(net.layer4[0].shortcut[1], nn.GroupNorm)
    duals = [l for l in lines if l.startswith("dual (")]
    assert len(duals) == len(net.train_order_block_ids())
    assert all(float(l.rsplit("=", 1)[1]) == float(l.rsplit("=", 1)[1]) for l in duals)
    assert eng.images_seen > 0
    # FedAvg left every replica with the same model
    a, b = (r.nets["net"].state_dict() for r in eng.replicas)
    assert all(torch.equal(a[k], b[k]) for k in a)


def test_legacy_checkpoint_of_the_other_norm_is_rejected(e2e):
    _, _, d, _ = e2e
    bn = models.ResNet9()
    before = {k: v.clone() for k, v in bn.state_dict().items()}
    with pytest.raises(KeyError, match="state_dict mismatch"):
        ckpt.load_worker(str(d), 0, bn, CPU)
    assert all(torch.equal(before[k], v) for k, v in bn.state_dict().items())      # nothing partially loaded
    gn = models.ResNet9(norm="group")
    ckpt.load_worker(str(d), 0, gn, CPU)
    ckpt.save_worker(str(d), 7, bn, 0, None, 0.0)
    with pytest.raises(KeyError, match="running_mean"):
        ckpt.load_worker(str(d), 7, gn, CPU)
    with pytest.raises(KeyError, match="state_dict mismatch"):
        federated_multi.run(parse_config(FederatedConfig, E2E[:-4] + ["--train_size", "256", "--test_size", "128", "--norm",
                                                                     "batch", "--load_model", "--ckpt_dir", str(d)]),
                            log=lambda m: None)


def test_resume_record_round_trips(e2e):
    eng, _, _, rec = e2e
    state = torch.load(rec, map_location="cpu", weights_only=False)
    for rep in eng.replicas:
        saved = state["replicas"][rep.ck]["net"]
        net = models.ResNet9(norm="group")
        ckpt.load_into(net, saved)
        own = rep.nets["net"].state_dict()
        assert list(saved) == list(own)
        assert all(torch.equal(net.state_dict()[k], own[k]) for k in own)
        with pytest.raises(KeyError, match="state_dict mismatch"):
            ckpt.load_into(models.ResNet9(), saved)
    # a run resumed from the record re-enters the schedule with the group-norm replicas
    eng2 = federated_multi.run(parse_config(FederatedConfig, E2E + ["--save_model=false", "--resume", rec]),
                               log=lambda m: None)
    for r1, r2 in zip(eng.replicas, eng2.replicas):
        assert torch.equal(r1.arenas["net"].data, r2.arenas["net"].data)
