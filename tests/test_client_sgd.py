"""Client SGD (``--optimizer sgd --lr --momentum --nesterov --weight_decay``) on CPU: configuration, the ATen composition
against ``torch.optim.SGD``, ``BlockSGD``'s stock-SGD state, and the classifier drivers end to end (determinism, true
resume, two gloo processes == one process)."""
import os

import pytest
import torch
import torch.nn.functional as F

from federated_pytorch_test_b200 import models
from federated_pytorch_test_b200.api import common, consensus_multi, federated_multi, fedprox_multi, no_consensus_multi
from federated_pytorch_test_b200.config import (CPCConfig, FederatedConfig, NoConsensusConfig, VAECLConfig, VAEConfig,
                                                parse_config)
from federated_pytorch_test_b200.ops import flatops
from federated_pytorch_test_b200.optim import BlockSGD
from federated_pytorch_test_b200.parallel import Topology
from federated_pytorch_test_b200.utils.flat import FlatArena

CPU = torch.device("cpu")
TINY = dict(train_size=1024, test_size=128, save_model=False, graphs=False, fast=False)
KW = dict(K=2, Nloop=1, Nadmm=2, max_minibatches=2, check_results=False, use_cuda=False, model="Net")
SGD = dict(optimizer="sgd", lr=0.05, momentum=0.9, nesterov=True, weight_decay=5e-4)


# ------------------------------------------------------------------------------------------ configuration
def test_defaults_parse_as_today_and_flags_parse():
    cfg = parse_config(FederatedConfig, [])
    assert (cfg.optimizer, cfg.lr, cfg.momentum, cfg.nesterov, cfg.weight_decay) == ("adam", 0.0, 0.0, False, 0.0)
    task = common.ClassifierTask(FederatedConfig(K=2, use_cuda=False, train_size=256, test_size=128),
                                 Topology.single_process(2, CPU))
    assert {v.optimizer for v in task.visits(0)} == {"adam"} and all(v.opt_kwargs == dict(lr=1e-3) for v in task.visits(0))
    cfg = parse_config(FederatedConfig, ["--optimizer", "sgd", "--lr", "0.05", "--momentum", "0.9", "--nesterov",
                                         "--weight_decay", "5e-4"])
    assert (cfg.optimizer, cfg.lr, cfg.momentum, cfg.nesterov, cfg.weight_decay) == ("sgd", 0.05, 0.9, True, 5e-4)
    task = common.ClassifierTask(FederatedConfig(K=2, use_cuda=False, train_size=256, test_size=128, **SGD),
                                 Topology.single_process(2, CPU))
    assert all(v.opt_kwargs == dict(lr=0.05, momentum=0.9, nesterov=True, weight_decay=5e-4) for v in task.visits(0))


INVALID = [
    ("optimizer", dict(optimizer="rmsprop")),
    ("lr", dict(optimizer="sgd")),                                   # SGD has no default learning rate
    ("lr", dict(optimizer="sgd", lr=-0.1)),
    ("lr", dict(optimizer="lbfgs", lr=0.1)),
    ("momentum", dict(optimizer="sgd", lr=0.1, momentum=1.0)),
    ("momentum", dict(optimizer="sgd", lr=0.1, momentum=-0.5)),
    ("momentum", dict(momentum=0.9)),                                # adam
    ("momentum", dict(optimizer="lbfgs", momentum=0.9)),
    ("nesterov", dict(nesterov=True)),
    ("nesterov", dict(optimizer="sgd", lr=0.1, nesterov=True)),     # needs momentum > 0
    ("weight_decay", dict(weight_decay=1e-4)),
    ("weight_decay", dict(optimizer="sgd", lr=0.1, weight_decay=-1e-4)),
]


def _argv(kw):
    out = []
    for k, v in kw.items():
        out += ["--" + k, str(v)]
    return out


@pytest.mark.parametrize("field,kw", INVALID)
def test_invalid_client_opt_settings_raise(field, kw):
    topo = Topology.single_process(2, CPU)
    base = dict(K=2, use_cuda=False, train_size=256, test_size=128)
    with pytest.raises(ValueError, match=field):
        common.ClassifierTask(FederatedConfig(**base, **kw), topo)
    cfg = parse_config(FederatedConfig, _argv({**base, **kw}))
    with pytest.raises(ValueError, match=field):
        common.ClassifierTask(cfg, topo)
    with pytest.raises(ValueError, match=field):
        no_consensus_multi.run(parse_config(NoConsensusConfig, _argv({**base, **kw})))


@pytest.mark.parametrize("driver,cls", [("federated_vae", VAEConfig), ("federated_vae_cl", VAECLConfig),
                                        ("federated_cpc", CPCConfig)])
@pytest.mark.parametrize("field,val", [("lr", 0.05), ("momentum", 0.9), ("nesterov", True), ("weight_decay", 5e-4)])
def test_unsupervised_drivers_reject_client_opt_flags(driver, cls, field, val):
    import importlib

    mod = importlib.import_module("federated_pytorch_test_b200.api." + driver)
    with pytest.raises(ValueError, match="%s fixes its own optimizer.*%s" % (driver, field)):
        mod.run(cls(use_cuda=False, **{field: val}))


def _run(mod, **kw):
    lines = []
    eng = mod.run(mod.Config(**{**TINY, **kw}), log=lines.append)
    return eng, [l for l in lines if l.startswith(("dual (", "block=["))]


def test_explicit_adam_lr_is_the_default_run():
    e0, a = _run(federated_multi, **KW)
    e1, b = _run(federated_multi, **KW, lr=1e-3)
    assert len(a) == 10 and a == b
    assert torch.equal(e0.replicas[0].arenas["net"].data, e1.replicas[0].arenas["net"].data)
    assert type(e1.optimizers[0]).__name__ == "BlockAdam"


# ------------------------------------------------------------------------------------------ the update
@pytest.mark.parametrize("momentum,nesterov", [(0.0, False), (0.9, False), (0.9, True)])
@pytest.mark.parametrize("weight_decay", [0.0, 5e-4])
@pytest.mark.parametrize("rho_dev", [False, True])
def test_sgd_prox_step_matches_torch_sgd(momentum, nesterov, weight_decay, rho_dev):
    torch.manual_seed(0)
    N, lr, rho, l1, l2 = 301, 0.05, 0.5, 1e-3, 2e-3
    x = torch.randn(N)
    p = torch.nn.Parameter(x.clone())
    opt = torch.optim.SGD([p], lr=lr, momentum=momentum, nesterov=nesterov, weight_decay=weight_decay)
    buf = torch.zeros(N) if momentum else None
    z, y = torch.randn(N), torch.randn(N)
    rd = torch.tensor([rho]) if rho_dev else None
    for _ in range(6):
        g = torch.randn(N)
        opt.zero_grad()
        loss = (p * g).sum() + torch.dot(y, p - z) + 0.5 * rho * torch.norm(p - z) ** 2 + l1 * torch.norm(p, 1) \
            + l2 * torch.norm(p, 2) ** 2
        loss.backward()
        opt.step()
        flatops.sgd_prox_step(x, g, buf, lr, momentum, nesterov, weight_decay, z, y, 0.0 if rho_dev else rho, l1, l2, rd)
        torch.testing.assert_close(x, p.detach(), rtol=1e-5, atol=1e-6)
        if momentum:
            torch.testing.assert_close(buf, opt.state[p]["momentum_buffer"], rtol=1e-5, atol=1e-6)


def test_sgd_prox_step_needs_a_buffer_exactly_with_momentum():
    x, g = torch.zeros(8), torch.ones(8)
    with pytest.raises(ValueError, match="momentum"):
        flatops.sgd_prox_step(x, g, None, 0.1, 0.9)
    with pytest.raises(ValueError, match="momentum"):
        flatops.sgd_prox_step(x, g, torch.zeros(8), 0.1, 0.0)


@pytest.mark.parametrize("channels_last", [False, True])
def test_block_sgd_state_dict_is_torch_sgds(channels_last):
    """BlockSGD over a block of a flat arena == torch.optim.SGD over the block's parameters; its state_dict loads into
    torch.optim.SGD with the same momentum buffers (in the parameters' memory layout)."""
    torch.manual_seed(1)
    net_a, net_b = models.Net(), models.Net()
    net_b.load_state_dict(net_a.state_dict())
    arena = FlatArena(net_a, channels_last_weights=channels_last)
    lo, hi = 0, 3                                            # conv1 + conv2 (4-D weights) and their biases
    pa = list(net_a.parameters())
    for i, p in enumerate(pa):
        p.requires_grad = lo <= i <= hi
    arena.attach_grads()
    pb = list(net_b.parameters())[lo:hi + 1]
    opt_a = BlockSGD(arena, lo, hi, lr=0.05, momentum=0.9, nesterov=True, weight_decay=5e-4)
    opt_b = torch.optim.SGD(pb, lr=0.05, momentum=0.9, nesterov=True, weight_decay=5e-4)
    for _ in range(4):
        xb, yb = torch.randn(8, 3, 32, 32), torch.randint(0, 10, (8,))
        opt_a.step(lambda: (opt_a.zero_grad(), F.cross_entropy(net_a(xb), yb).backward()))
        opt_b.zero_grad()
        F.cross_entropy(net_b(xb), yb).backward()
        opt_b.step()
    for a, b in zip(pa[lo:hi + 1], pb):
        torch.testing.assert_close(a.detach(), b.detach(), rtol=1e-5, atol=1e-6)
    sd = opt_a.state_dict()
    assert set(sd["param_groups"][0]) == set(opt_b.state_dict()["param_groups"][0])
    opt_c = torch.optim.SGD(pa[lo:hi + 1], lr=1.0)
    opt_c.load_state_dict(sd)
    assert opt_c.param_groups[0]["momentum"] == 0.9 and opt_c.param_groups[0]["nesterov"]
    for a, b in zip(pa[lo:hi + 1], pb):
        got, want = opt_c.state[a]["momentum_buffer"], opt_b.state[b]["momentum_buffer"]
        assert got.stride() == a.stride()
        torch.testing.assert_close(got, want, rtol=1e-5, atol=1e-6)


def test_block_sgd_without_momentum_has_no_buffer():
    arena = FlatArena(models.Net())
    opt = BlockSGD(arena, 0, 1, lr=0.1)
    assert opt.buf is None
    assert all(s["momentum_buffer"] is None for s in opt.state_dict()["state"].values())


# ------------------------------------------------------------------------------------------ end to end
E2E = [
    (federated_multi, {}),
    (federated_multi, dict(server_opt="adam")),
    (federated_multi, dict(K=4, clients_per_round=2)),
    (fedprox_multi, {}),
    (consensus_multi, dict(bb_update=True)),
    (no_consensus_multi, dict(Nepoch=2, Nadmm=1)),
]


@pytest.mark.parametrize("mod,extra", E2E, ids=["fedavg", "fedadam", "sampled", "fedprox", "admm_bb", "no_consensus"])
def test_drivers_train_with_sgd_deterministically(mod, extra):
    e0, a = _run(mod, **{**KW, **SGD, **extra})
    e1, b = _run(mod, **{**KW, **SGD, **extra})
    assert a == b and (mod is no_consensus_multi or len(a) == 10)
    assert all(type(o) is BlockSGD for o in e0.optimizers)
    x0, x1 = e0.replicas[0].arenas["net"].data, e1.replicas[0].arenas["net"].data
    assert torch.equal(x0, x1) and torch.isfinite(x0).all()
    init = models.Net()
    torch.manual_seed(0)
    from federated_pytorch_test_b200.utils.simple_utils import init_weights
    init.apply(init_weights)
    assert not torch.equal(x0, FlatArena(init).data)                  # it trained


def test_legacy_checkpoint_loads_into_torch_sgd(tmp_path):
    eng, _ = _run(federated_multi, **KW, **SGD, save_model=True, ckpt_dir=str(tmp_path))
    rec = torch.load(str(tmp_path / "s0.model"), weights_only=False)
    opt = eng.optimizers[0]
    net = models.Net()
    params = list(net.parameters())[opt.lo: opt.hi + 1]
    sgd = torch.optim.SGD(params, lr=1.0)
    sgd.load_state_dict(rec["optimizer_state_dict"])
    assert (sgd.param_groups[0]["lr"], sgd.param_groups[0]["momentum"]) == (0.05, 0.9)
    arena = eng.replicas[0].arenas["net"]
    full = torch.zeros(arena.total)
    a, b = arena.span(opt.lo, opt.hi)
    full[a:b] = opt.buf
    bufs = torch.cat([sgd.state[p]["momentum_buffer"].reshape(-1) for p in params])
    assert bufs.abs().sum() > 0
    torch.testing.assert_close(bufs, arena.compact(opt.lo, opt.hi, src=full), rtol=0, atol=0)


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


def test_kill_and_resume_reproduces_the_trace_and_weights(tmp_path):
    kw = dict(KW, K=3, Nadmm=3, **SGD)
    eng, full = _run(federated_multi, **kw)
    assert len(full) == 15
    rec = str(tmp_path / "resume.pt")
    first = _killed_run({**kw, "resume_out": rec}, 27)           # 6 steps per round: round 1 of the second block's visit
    assert 0 < len(first) < 15 and os.path.exists(rec)
    st = torch.load(rec, weights_only=False)
    assert st["position"]["optimizer"] == "sgd"
    assert all(o["optimizer"] == "sgd" and o["buf"].abs().sum() > 0 for o in st["optimizers"].values())
    eng2, second = _run(federated_multi, **kw, resume=rec)
    assert first + second == full
    assert torch.equal(eng.replicas[0].arenas["net"].data, eng2.replicas[0].arenas["net"].data)


def test_resume_with_the_other_optimizer_raises(tmp_path):
    sgd_rec, adam_rec = str(tmp_path / "sgd.pt"), str(tmp_path / "adam.pt")
    _killed_run({**KW, **SGD, "resume_out": sgd_rec}, 6)
    _killed_run({**KW, "resume_out": adam_rec}, 6)
    with pytest.raises(ValueError, match="optimizer"):
        _run(federated_multi, **KW, resume=sgd_rec)
    with pytest.raises(ValueError, match="optimizer"):
        _run(federated_multi, **KW, **SGD, resume=adam_rec)
    rec = torch.load(adam_rec, weights_only=False)          # as written before SGD: no optimizer name in the position
    del rec["position"]["optimizer"]
    torch.save(rec, adam_rec)
    with pytest.raises(ValueError, match="optimizer"):
        _run(federated_multi, **KW, **SGD, resume=adam_rec)


DIST_KW = dict(KW, K=4, **SGD)


def _dist_worker(rank, world, port, out):
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch.distributed as dist
    lines = []
    eng = federated_multi.run(federated_multi.Config(**DIST_KW, **TINY), log=lines.append)
    if rank == 0:
        torch.save({"lines": lines, "flat": eng.replicas[0].arenas["net"].data.clone()}, out)
    dist.destroy_process_group()


def test_two_process_gloo_equals_single_process(tmp_path):
    import torch.multiprocessing as mp
    out = str(tmp_path / "r0.pt")
    port = 39500 + (os.getpid() % 2000)
    mp.spawn(_dist_worker, args=(2, port, out), nprocs=2, join=True)
    got = torch.load(out, weights_only=False)
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        os.environ.pop(k, None)
    eng, single = _run(federated_multi, **DIST_KW)
    multi = [l for l in got["lines"] if l.startswith("dual (")]
    assert len(single) == len(multi) == 10
    for a, b in zip(single, multi):
        assert a.split("=")[:-1] == b.split("=")[:-1]
        assert float(a.rsplit("=", 1)[1]) == pytest.approx(float(b.rsplit("=", 1)[1]), rel=1e-4)
    torch.testing.assert_close(got["flat"], eng.replicas[0].arenas["net"].data, rtol=1e-4, atol=1e-6)
