"""Client training recipe (``--optimizer adamw``, ``--lr_schedule const|step|cosine``, ``--lr_warmup``, ``--clip_norm``) on
CPU: configuration, the schedule against torch's schedulers, the ATen updates against ``torch.optim.AdamW`` / ``SGD`` with
``clip_grad_norm_``, ``BlockAdam``'s AdamW state, and the classifier drivers end to end (determinism, metrics rows, true
resume, two gloo processes == one process)."""
import json
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
from federated_pytorch_test_b200.optim.block_adam import BlockAdam
from federated_pytorch_test_b200.optim.schedule import round_lr
from federated_pytorch_test_b200.parallel import Topology
from federated_pytorch_test_b200.utils.flat import FlatArena

CPU = torch.device("cpu")
TINY = dict(train_size=1024, test_size=128, save_model=False, graphs=False, fast=False)
KW = dict(K=2, Nloop=1, Nadmm=2, max_minibatches=2, check_results=False, use_cuda=False, model="Net")
RECIPE = dict(optimizer="adamw", weight_decay=0.05, lr_schedule="cosine", lr_warmup=2, lr_min=0.1, clip_norm=0.5)


# ------------------------------------------------------------------------------------------ configuration
def test_defaults_parse_as_today_and_flags_parse():
    cfg = parse_config(FederatedConfig, [])
    assert (cfg.lr_schedule, cfg.lr_warmup, cfg.lr_gamma, cfg.lr_step_rounds, cfg.lr_min, cfg.clip_norm) == \
        ("const", 0, 0.1, 0, 0.0, 0.0)
    cfg = parse_config(FederatedConfig, ["--optimizer", "adamw", "--weight_decay", "0.01", "--lr_schedule", "step",
                                         "--lr_warmup", "3", "--lr_gamma", "0.5", "--lr_step_rounds", "4",
                                         "--clip_norm", "1.5"])
    assert (cfg.optimizer, cfg.weight_decay, cfg.lr_schedule, cfg.lr_warmup, cfg.lr_gamma, cfg.lr_step_rounds,
            cfg.clip_norm) == ("adamw", 0.01, "step", 3, 0.5, 4, 1.5)
    topo = Topology.single_process(2, CPU)
    base = dict(K=2, use_cuda=False, train_size=256, test_size=128)
    task = common.ClassifierTask(FederatedConfig(**base, optimizer="adamw", weight_decay=0.01, clip_norm=1.5), topo)
    assert all(v.optimizer == "adamw" and v.opt_kwargs == dict(lr=1e-3, weight_decay=0.01, clip_norm=1.5)
               for v in task.visits(0))
    task = common.ClassifierTask(FederatedConfig(**base, optimizer="adamw"), topo)     # wd 0: AdamW is Adam
    assert all(v.opt_kwargs == dict(lr=1e-3, weight_decay=0.0) for v in task.visits(0))
    task = common.ClassifierTask(FederatedConfig(**base, lr_schedule="cosine", lr_min=0.1), topo)
    assert all(v.opt_kwargs == dict(lr=1e-3) for v in task.visits(0))


INVALID = [
    ("lr_schedule", dict(lr_schedule="exp")),
    ("lr_warmup", dict(lr_warmup=-1)),
    ("lr_gamma", dict(lr_schedule="step", lr_step_rounds=1, lr_gamma=0.0)),
    ("lr_gamma", dict(lr_schedule="step", lr_step_rounds=1, lr_gamma=1.5)),
    ("lr_gamma", dict(lr_gamma=0.5)),                                   # belongs to step
    ("lr_gamma", dict(lr_schedule="cosine", lr_gamma=0.5)),
    ("lr_step_rounds", dict(lr_schedule="step")),                       # step needs S >= 1
    ("lr_step_rounds", dict(lr_step_rounds=-1)),
    ("lr_step_rounds", dict(lr_schedule="cosine", lr_step_rounds=2)),
    ("lr_min", dict(lr_schedule="cosine", lr_min=1.0)),
    ("lr_min", dict(lr_schedule="cosine", lr_min=-0.1)),
    ("lr_min", dict(lr_schedule="step", lr_step_rounds=1, lr_min=0.1)),
    ("clip_norm", dict(clip_norm=-1.0)),
    ("clip_norm", dict(clip_norm=float("inf"))),
    ("clip_norm", dict(clip_norm=float("nan"))),
    ("lr_schedule", dict(optimizer="lbfgs", lr_schedule="cosine")),
    ("lr_warmup", dict(optimizer="lbfgs", lr_warmup=2)),
    ("clip_norm", dict(optimizer="lbfgs", clip_norm=1.0)),
    ("momentum", dict(optimizer="adamw", momentum=0.9)),
    ("nesterov", dict(optimizer="adamw", nesterov=True)),
    ("weight_decay", dict(weight_decay=1e-4)),                          # adam: no coupled L2 decay
    ("weight_decay", dict(optimizer="adamw", weight_decay=-1e-4)),
]


def _argv(kw):
    out = []
    for k, v in kw.items():
        out += ["--" + k, str(v)]
    return out


@pytest.mark.parametrize("field,kw", INVALID)
def test_invalid_recipe_settings_raise(field, kw):
    topo = Topology.single_process(2, CPU)
    base = dict(K=2, use_cuda=False, train_size=256, test_size=128)
    with pytest.raises(ValueError, match=field):
        common.ClassifierTask(FederatedConfig(**base, **kw), topo)
    cfg = parse_config(FederatedConfig, _argv({**base, **kw}))
    with pytest.raises(ValueError, match=field):
        common.ClassifierTask(cfg, topo)
    with pytest.raises(ValueError, match=field):
        no_consensus_multi.run(parse_config(NoConsensusConfig, _argv({**base, **kw})))


def test_warmup_as_long_as_the_run_raises():
    # Net: 5 block visits x Nadmm 2 = 10 rounds
    with pytest.raises(ValueError, match="lr_warmup"):
        _run(federated_multi, **KW, lr_warmup=10)
    eng, _ = _run(federated_multi, **KW, lr_warmup=9)
    assert eng.total_rounds == 10
    with pytest.raises(ValueError, match="lr_warmup"):
        _run(no_consensus_multi, **dict(KW, Nepoch=3, Nadmm=1), lr_warmup=3)
    with pytest.raises(ValueError, match="lr_warmup"):
        round_lr(1e-3, 0, 5, "const", 5)


@pytest.mark.parametrize("driver,cls", [("federated_vae", VAEConfig), ("federated_vae_cl", VAECLConfig),
                                        ("federated_cpc", CPCConfig)])
@pytest.mark.parametrize("field,val", [("lr_schedule", "cosine"), ("lr_warmup", 2), ("lr_gamma", 0.5),
                                       ("lr_step_rounds", 2), ("lr_min", 0.1), ("clip_norm", 1.0),
                                       ("optimizer", "adamw")])
def test_unsupervised_drivers_reject_recipe_flags(driver, cls, field, val):
    import importlib

    mod = importlib.import_module("federated_pytorch_test_b200.api." + driver)
    with pytest.raises(ValueError, match="%s fixes its own optimizer.*%s" % (driver, field)):
        mod.run(cls(use_cuda=False, **{field: val}))


# ------------------------------------------------------------------------------------------ the schedule
def _torch_lrs(make, T, lr=0.1):
    p = torch.nn.Parameter(torch.zeros(1))
    opt = torch.optim.SGD([p], lr=lr)
    sched = make(opt)
    out = []
    for _ in range(T):
        out.append(opt.param_groups[0]["lr"])
        opt.step()
        sched.step()
    return out


@pytest.mark.parametrize("W,T", [(1, 5), (4, 9), (7, 8)])
def test_warmup_is_linear_lr(W, T):
    from torch.optim.lr_scheduler import LinearLR

    want = _torch_lrs(lambda o: LinearLR(o, start_factor=1.0 / (W + 1), total_iters=W), T)
    got = [round_lr(0.1, r, T, "const", W) for r in range(T)]
    assert got == pytest.approx(want, rel=1e-6)


@pytest.mark.parametrize("S,gamma,W", [(1, 0.998, 0), (3, 0.1, 0), (2, 0.5, 3)])
def test_step_is_step_lr(S, gamma, W):
    from torch.optim.lr_scheduler import StepLR

    T = 12
    decay = _torch_lrs(lambda o: StepLR(o, step_size=S, gamma=gamma), T - W)
    got = [round_lr(0.1, r, T, "step", W, gamma, S) for r in range(T)]
    for r in range(T):
        want = 0.1 * (r + 1) / (W + 1) if r < W else decay[r - W]
        assert got[r] == pytest.approx(want, rel=1e-6), r


@pytest.mark.parametrize("m,W", [(0.0, 0), (0.1, 0), (0.05, 4)])
def test_cosine_is_cosine_annealing_lr(m, W):
    from torch.optim.lr_scheduler import CosineAnnealingLR

    T = 15
    decay = _torch_lrs(lambda o: CosineAnnealingLR(o, T_max=T - W, eta_min=m * 0.1), T - W)
    got = [round_lr(0.1, r, T, "cosine", W, lr_min=m) for r in range(T)]
    for r in range(T):
        want = 0.1 * (r + 1) / (W + 1) if r < W else decay[r - W]
        assert got[r] == pytest.approx(want, rel=1e-6, abs=1e-9), r


def test_round_lr_is_float32():
    v = round_lr(1e-3, 3, 10, "cosine")
    assert torch.tensor(v, dtype=torch.float32).item() == v


# ------------------------------------------------------------------------------------------ the updates
def _pen_loss(p, z, y, rho, l1, l2):
    if z is None:
        return l1 * torch.norm(p, 1) + l2 * torch.norm(p, 2) ** 2
    return torch.dot(y, p - z) + 0.5 * rho * torch.norm(p - z) ** 2 + l1 * torch.norm(p, 1) + l2 * torch.norm(p, 2) ** 2


def _clipped_data_grad(p, g, clip):
    """torch: clip the data-loss gradient alone, then add the penalty gradient."""
    p.grad = g.clone()
    if clip:
        torch.nn.utils.clip_grad_norm_([p], clip)
    return p.grad.clone()


@pytest.mark.parametrize("weight_decay", [0.0, 0.05])
@pytest.mark.parametrize("clip", [0.0, 5.0])
@pytest.mark.parametrize("pen,rho_dev", [(False, False), (True, False), (True, True)])
def test_adam_prox_step_matches_torch_adamw(weight_decay, clip, pen, rho_dev):
    torch.manual_seed(0)
    N, rho, l1, l2 = 301, 0.5, 1e-3, 2e-3
    x = torch.randn(N)
    p = torch.nn.Parameter(x.clone())
    opt = torch.optim.AdamW([p], lr=1.0, weight_decay=weight_decay)
    m, v = torch.zeros(N), torch.zeros(N)
    z, y = (torch.randn(N), torch.randn(N)) if pen else (None, None)
    rd = torch.tensor([rho]) if rho_dev else None
    ws = flatops.clip_workspace(x)
    lr_t = torch.zeros(1)
    norms = []
    for k in range(6):
        lr_t.fill_(1e-2 * (0.7 ** k))                                  # a new rate every step
        opt.param_groups[0]["lr"] = float(lr_t)
        g = torch.randn(N) * (k + 1) * 0.1                             # norms from ~1.7 to ~10: some steps clip
        norms.append(float(g.norm()))
        gc = _clipped_data_grad(p, g, clip)
        opt.zero_grad()
        pl = _pen_loss(p, z, y, rho, l1, l2)
        if pl.requires_grad:
            pl.backward()
        p.grad = p.grad + gc if p.grad is not None else gc
        opt.step()
        flatops.adam_prox_step(x, g, m, v, k + 1, lr_t, 0.9, 0.999, 1e-8, z, y, 0.0 if rho_dev else rho, l1, l2, rd,
                               weight_decay=weight_decay, clip_norm=clip, clip_ws=ws)
        torch.testing.assert_close(x, p.detach(), rtol=1e-5, atol=1e-6)
        torch.testing.assert_close(m, opt.state[p]["exp_avg"], rtol=1e-5, atol=1e-6)
    if clip:
        norm_sum, clipped, steps = ws[0][1:4].tolist()
        assert steps == 6 and clipped == sum(n > clip for n in norms) and 0 < clipped < 6
        assert norm_sum == pytest.approx(sum(norms), rel=1e-5)


@pytest.mark.parametrize("momentum,nesterov", [(0.0, False), (0.9, True)])
@pytest.mark.parametrize("clip", [0.0, 5.0])
@pytest.mark.parametrize("pen,rho_dev", [(False, False), (True, True)])
def test_sgd_prox_step_matches_torch_sgd_with_clipping(momentum, nesterov, clip, pen, rho_dev):
    torch.manual_seed(1)
    N, rho, l1, l2 = 301, 0.5, 1e-3, 2e-3
    x = torch.randn(N)
    p = torch.nn.Parameter(x.clone())
    opt = torch.optim.SGD([p], lr=1.0, momentum=momentum, nesterov=nesterov, weight_decay=5e-4)
    buf = torch.zeros(N) if momentum else None
    z, y = (torch.randn(N), torch.randn(N)) if pen else (None, None)
    rd = torch.tensor([rho]) if rho_dev else None
    ws = flatops.clip_workspace(x)
    lr_t = torch.zeros(1)
    for k in range(6):
        lr_t.fill_(0.05 * (0.8 ** k))
        opt.param_groups[0]["lr"] = float(lr_t)
        g = torch.randn(N) * (k + 1) * 0.1
        gc = _clipped_data_grad(p, g, clip)
        opt.zero_grad()
        pl = _pen_loss(p, z, y, rho, l1, l2)
        pl.backward()
        p.grad = p.grad + gc
        opt.step()
        flatops.sgd_prox_step(x, g, buf, lr_t, momentum, nesterov, 5e-4, z, y, 0.0 if rho_dev else rho, l1, l2, rd,
                              clip_norm=clip, clip_ws=ws)
        torch.testing.assert_close(x, p.detach(), rtol=1e-5, atol=1e-6)


def test_clip_statistics_count_norms_and_clipped_steps():
    ws = flatops.clip_workspace(torch.zeros(4))
    norms = []
    for s in (0.5, 2.0, 3.0):
        g = torch.full((4,), s)
        norms.append(float(g.norm()))
        flatops.sgd_prox_step(torch.zeros(4), g, None, 0.1, clip_norm=4.0, clip_ws=ws)
    norm_sum, clipped, steps = ws[0][1:4].tolist()
    assert steps == 3 and clipped == 1 and norm_sum == pytest.approx(sum(norms))


@pytest.mark.parametrize("bad", [float("nan"), float("inf")])
@pytest.mark.parametrize("kind", ["adamw", "sgd"])
def test_non_finite_gradient_gives_non_finite_parameters(bad, kind):
    x, g = torch.randn(64), torch.randn(64)
    g[7] = bad
    if kind == "adamw":
        flatops.adam_prox_step(x, g, torch.zeros(64), torch.zeros(64), 1, 1e-3, 0.9, 0.999, 1e-8, weight_decay=0.01,
                               clip_norm=1.0)
    else:
        flatops.sgd_prox_step(x, g, None, 0.1, clip_norm=1.0)
    assert not torch.isfinite(x).all()


def test_block_adamw_follows_torch_and_its_state_dict_loads():
    """BlockAdam(adamw) with clipping and a device learning rate that changes every step == torch.optim.AdamW with
    clip_grad_norm_ over the block's parameters; its state_dict loads into torch.optim.AdamW."""
    torch.manual_seed(1)
    net_a, net_b = models.Net(), models.Net()
    net_b.load_state_dict(net_a.state_dict())
    arena = FlatArena(net_a)
    lo, hi = 0, 3
    pa = list(net_a.parameters())
    for i, p in enumerate(pa):
        p.requires_grad = lo <= i <= hi
    arena.attach_grads()
    pb = list(net_b.parameters())[lo:hi + 1]
    opt_a = BlockAdam(arena, lo, hi, lr=1e-2, adamw=True, weight_decay=0.05, clip_norm=0.5, device_lr=True)
    opt_b = torch.optim.AdamW(pb, lr=1e-2, weight_decay=0.05)
    for k in range(4):
        lr = round_lr(1e-2, k, 4, "cosine", 1)
        opt_a.set_lr(lr)
        opt_b.param_groups[0]["lr"] = lr
        xb, yb = torch.randn(8, 3, 32, 32), torch.randint(0, 10, (8,))
        opt_a.step(lambda: (opt_a.zero_grad(), F.cross_entropy(net_a(xb), yb).backward()))
        opt_b.zero_grad()
        F.cross_entropy(net_b(xb), yb).backward()
        torch.nn.utils.clip_grad_norm_(pb, 0.5)
        opt_b.step()
    for a, b in zip(pa[lo:hi + 1], pb):
        torch.testing.assert_close(a.detach(), b.detach(), rtol=1e-5, atol=1e-6)
    assert float(opt_a.lr_dev) == opt_a.param_groups[0]["lr"]
    sd = opt_a.state_dict()
    assert set(sd["param_groups"][0]) == set(opt_b.state_dict()["param_groups"][0])
    opt_c = torch.optim.AdamW(pa[lo:hi + 1], lr=1.0)
    opt_c.load_state_dict(sd)
    assert opt_c.param_groups[0]["weight_decay"] == 0.05 and opt_c.param_groups[0]["decoupled_weight_decay"]
    for a, b in zip(pa[lo:hi + 1], pb):
        torch.testing.assert_close(opt_c.state[a]["exp_avg_sq"], opt_b.state[b]["exp_avg_sq"], rtol=1e-5, atol=1e-9)


def test_legacy_adamw_checkpoint_loads_into_torch_adamw(tmp_path):
    eng, _ = _run(federated_multi, **KW, **RECIPE, save_model=True, ckpt_dir=str(tmp_path))
    rec = torch.load(str(tmp_path / "s0.model"), weights_only=False)
    opt = eng.optimizers[0]
    net = models.Net()
    params = list(net.parameters())[opt.lo: opt.hi + 1]
    adamw = torch.optim.AdamW(params, lr=1.0)
    adamw.load_state_dict(rec["optimizer_state_dict"])
    grp = adamw.param_groups[0]
    assert grp["weight_decay"] == 0.05 and grp["decoupled_weight_decay"]
    assert grp["lr"] == round_lr(1e-3, 9, 10, "cosine", 2, lr_min=0.1)            # the last round's rate
    arena = eng.replicas[0].arenas["net"]
    full = torch.zeros(arena.total)
    a, b = arena.span(opt.lo, opt.hi)
    full[a:b] = opt.m
    m = torch.cat([adamw.state[p]["exp_avg"].reshape(-1) for p in params])
    assert m.abs().sum() > 0
    torch.testing.assert_close(m, arena.compact(opt.lo, opt.hi, src=full), rtol=0, atol=0)


# ------------------------------------------------------------------------------------------ end to end
def _run(mod, **kw):
    lines = []
    eng = mod.run(mod.Config(**{**TINY, **kw}), log=lines.append)
    return eng, [l for l in lines if l.startswith(("dual (", "block=["))]


def _rows(path):
    with open(path) as f:
        return [r for r in map(json.loads, f) if r.get("kind") == "round"]


def test_explicit_defaults_are_the_default_run(tmp_path):
    e0, a = _run(federated_multi, **KW, metrics_path=str(tmp_path / "a.jsonl"))
    e1, b = _run(federated_multi, **KW, lr_schedule="const", lr_warmup=0, clip_norm=0.0,
                 metrics_path=str(tmp_path / "b.jsonl"))
    assert len(a) == 10 and a == b
    assert torch.equal(e0.replicas[0].arenas["net"].data, e1.replicas[0].arenas["net"].data)
    assert all(o.lr_dev is None and o.clip_ws is None for o in e1.optimizers)
    for r in _rows(str(tmp_path / "b.jsonl")):
        assert not {"lr", "grad_norm", "clip_frac"} & set(r)


@pytest.mark.parametrize("sched", [dict(lr_schedule="cosine", lr_warmup=3, lr_min=0.2),
                                   dict(lr_schedule="step", lr_step_rounds=3, lr_gamma=0.5),
                                   dict(lr_warmup=5)], ids=["cosine", "step", "warmup"])
def test_metrics_rows_carry_the_schedule(tmp_path, sched):
    path = str(tmp_path / "m.jsonl")
    eng, _ = _run(federated_multi, **KW, **sched, clip_norm=0.5, metrics_path=path)
    rows = _rows(path)
    assert eng.total_rounds == len(rows) == 10
    sched = dict(sched)
    kind, warmup = sched.pop("lr_schedule", "const"), sched.pop("lr_warmup", 0)
    want = [round_lr(1e-3, r, 10, kind, warmup, **sched) for r in range(10)]
    assert [r["lr"] for r in rows] == want
    assert all(r["grad_norm"] > 0 and 0.0 <= r["clip_frac"] <= 1.0 for r in rows)
    assert any(r["clip_frac"] > 0 for r in rows)


E2E = [
    (federated_multi, {}),
    (fedprox_multi, {}),
    (consensus_multi, dict(bb_update=True)),
    (no_consensus_multi, dict(Nepoch=3, Nadmm=1)),
]


@pytest.mark.parametrize("mod,extra", E2E, ids=["fedavg", "fedprox", "admm_bb", "no_consensus"])
def test_drivers_train_with_the_recipe_deterministically(mod, extra):
    e0, a = _run(mod, **{**KW, **RECIPE, **extra})
    e1, b = _run(mod, **{**KW, **RECIPE, **extra})
    assert a == b and (mod is no_consensus_multi or len(a) == 10)
    assert all(type(o) is BlockAdam and o.adamw and o.lr_dev is not None and o.clip_ws is not None
               for o in e0.optimizers)
    x0, x1 = e0.replicas[0].arenas["net"].data, e1.replicas[0].arenas["net"].data
    assert torch.equal(x0, x1) and torch.isfinite(x0).all()
    last = round_lr(1e-3, e0.total_rounds - 1, e0.total_rounds, "cosine", 2, lr_min=0.1)
    assert all(float(o.lr_dev) == last for o in e0.optimizers)
    e2, c = _run(mod, **{**KW, **extra, "optimizer": "adamw", "weight_decay": 0.05})     # the schedule and clip change it
    assert not torch.equal(x0, e2.replicas[0].arenas["net"].data)


def test_sgd_with_schedule_and_clipping():
    e0, a = _run(federated_multi, **KW, optimizer="sgd", lr=0.05, momentum=0.9, lr_schedule="step", lr_step_rounds=5,
                 lr_gamma=0.5, clip_norm=0.5)
    assert all(type(o) is BlockSGD and o.lr_dev is not None for o in e0.optimizers)
    assert float(e0.optimizers[0].lr_dev) == pytest.approx(0.05 * 0.5 ** 1)          # round 9 of 10
    assert torch.isfinite(e0.replicas[0].arenas["net"].data).all()


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


def test_kill_and_resume_across_a_learning_rate_change(tmp_path):
    kw = dict(KW, K=3, Nadmm=3, **RECIPE)
    eng, full = _run(federated_multi, **kw)
    assert len(full) == 15
    rec = str(tmp_path / "resume.pt")
    first = _killed_run({**kw, "resume_out": rec}, 27)           # 6 steps per round: round 1 of the second block's visit
    assert 0 < len(first) < 15 and os.path.exists(rec)
    st = torch.load(rec, weights_only=False)
    assert st["position"]["optimizer"] == "adamw"
    assert st["position"]["recipe"]["lr_schedule"] == "cosine" and st["position"]["recipe"]["clip_norm"] == 0.5
    eng2, second = _run(federated_multi, **kw, resume=rec)
    assert first + second == full
    assert torch.equal(eng.replicas[0].arenas["net"].data, eng2.replicas[0].arenas["net"].data)


@pytest.mark.parametrize("field,val", [("lr_schedule", "const"), ("lr_warmup", 1), ("lr_min", 0.2), ("clip_norm", 1.0)])
def test_resume_with_other_recipe_settings_raises(tmp_path, field, val):
    rec = str(tmp_path / "r.pt")
    _killed_run({**KW, **RECIPE, "resume_out": rec}, 6)
    with pytest.raises(ValueError, match=field):
        _run(federated_multi, **{**KW, **RECIPE, field: val, "resume": rec})


def test_resume_adamw_against_adam_or_other_decay_raises(tmp_path):
    rec = str(tmp_path / "r.pt")
    _killed_run({**KW, **RECIPE, "resume_out": rec}, 6)
    with pytest.raises(ValueError, match="optimizer"):
        _run(federated_multi, **{**KW, **RECIPE, "optimizer": "adam", "weight_decay": 0.0, "resume": rec})
    with pytest.raises(ValueError, match="weight_decay"):
        _run(federated_multi, **{**KW, **RECIPE, "weight_decay": 0.01, "resume": rec})
    plain = str(tmp_path / "plain.pt")                            # a record without schedule settings resumes as const
    _killed_run({**KW, "resume_out": plain}, 6)
    st = torch.load(plain, weights_only=False)
    del st["position"]["recipe"]
    torch.save(st, plain)
    _run(federated_multi, **KW, resume=plain)
    with pytest.raises(ValueError, match="lr_schedule"):
        _run(federated_multi, **KW, lr_schedule="cosine", resume=plain)


DIST_KW = dict(KW, K=4, **RECIPE)


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
    port = 41500 + (os.getpid() % 2000)
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
