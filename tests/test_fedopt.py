"""Server optimizers of federated averaging (FedAvgM, FedAdagrad, FedAdam, FedYogi) on CPU: configuration, the ATen
operator against a literal float64 transcription of the update table, and ``federated_multi`` end to end (FedAvg
equivalence, determinism, true resume, two gloo processes == one process)."""
import os
import re

import numpy as np
import pytest
import torch

from federated_pytorch_test_b200.algo.strategies import FedAvg, FedOpt
from federated_pytorch_test_b200.api import federated_multi, fedprox_multi
from federated_pytorch_test_b200.config import FederatedConfig, FedProxConfig, parse_config
from federated_pytorch_test_b200.parallel import Topology, TorchCollective

TINY = dict(train_size=1024, test_size=128, save_model=False, graphs=False, fast=False)
KW = dict(K=2, Nloop=1, Nadmm=2, max_minibatches=2, check_results=False, use_cuda=False)
KINDS = ["avgm", "adagrad", "adam", "yogi"]


# ------------------------------------------------------------------------------------------ configuration
def test_flags_parse_and_defaults_keep_fedavg():
    cfg = parse_config(FederatedConfig, [])
    assert (cfg.server_opt, cfg.server_lr, cfg.server_momentum, cfg.server_beta1, cfg.server_beta2, cfg.server_tau) == \
        ("none", 0.0, 0.9, 0.9, 0.99, 1e-3)
    cfg = parse_config(FederatedConfig, ["--server_opt", "yogi", "--server_lr", "0.03", "--server_beta1", "0.5",
                                         "--server_beta2", "0.9", "--server_tau", "1e-4", "--server_momentum", "0"])
    assert (cfg.server_opt, cfg.server_lr, cfg.server_beta1, cfg.server_beta2, cfg.server_tau, cfg.server_momentum) == \
        ("yogi", 0.03, 0.5, 0.9, 1e-4, 0.0)


@pytest.mark.parametrize("bad", [dict(server_opt="sgd"), dict(server_lr=-1e-3), dict(server_momentum=1.0),
                                 dict(server_momentum=-0.1), dict(server_beta1=1.0), dict(server_beta2=1.5),
                                 dict(server_beta2=-1e-9), dict(server_tau=0.0), dict(server_tau=-1.0)])
def test_invalid_settings_raise(bad):
    key = next(iter(bad))
    with pytest.raises(ValueError, match=key):
        FederatedConfig(**bad)
    with pytest.raises(ValueError, match=key):
        parse_config(FederatedConfig, ["--%s=%s" % (key, bad[key])])


def test_other_drivers_have_no_server_optimizer():
    with pytest.raises(SystemExit):
        parse_config(FedProxConfig, ["--server_opt", "adam"])
    assert not hasattr(FedProxConfig(), "server_opt")


def test_none_constructs_fedavg_itself():
    topo = Topology.single_process(2, torch.device("cpu"))
    coll = TorchCollective(topo)
    assert type(federated_multi.make_strategy(FederatedConfig(), coll, topo)) is FedAvg
    s = federated_multi.make_strategy(FederatedConfig(server_opt="adam"), coll, topo)
    assert type(s) is FedOpt and s.name != FedAvg.name and (s.lr, s.beta1, s.beta2, s.tau) == (1e-2, 0.9, 0.99, 1e-3)
    s = federated_multi.make_strategy(FederatedConfig(server_opt="avgm", server_momentum=0.5), coll, topo)
    assert (s.lr, s.beta1) == (1.0, 0.5)
    with pytest.raises(ValueError):
        FedOpt(coll, topo, "none")


# ------------------------------------------------------------------------------------------ the operator
def _literal_round(kind, hp, x64, st):
    """One round of the update table in float64, on numpy arrays; returns ||z_old - z_new|| / N."""
    lr, b1, b2, tau = hp
    d = np.mean(x64, axis=0) - st["z"]
    if kind == "avgm":
        st["m"] = b1 * st["m"] + d
        znew = st["z"] + lr * st["m"]
    else:
        st["m"] = b1 * st["m"] + (1 - b1) * d
        if kind == "adagrad":
            st["v"] = st["v"] + d * d
        elif kind == "adam":
            st["v"] = b2 * st["v"] + (1 - b2) * d * d
        else:
            st["v"] = st["v"] - (1 - b2) * d * d * np.sign(st["v"] - d * d)
        znew = st["z"] + lr * st["m"] / (np.sqrt(st["v"]) + tau)
    dual = np.linalg.norm(st["z"] - znew) / st["z"].size
    st["z"] = znew
    return dual


@pytest.mark.parametrize("kind", KINDS)
def test_operator_matches_float64_table_over_rounds_and_visits(kind):
    K, N = 4, 257
    topo = Topology.single_process(K, torch.device("cpu"))
    lr = {"avgm": 0.7, "adagrad": 0.05, "adam": 0.02, "yogi": 0.03}[kind]
    strat = FedOpt(TorchCollective(topo), topo, kind, lr=lr, momentum=0.8, beta1=0.85, beta2=0.95, tau=1e-2)
    hp = (lr, 0.8 if kind == "avgm" else 0.85, 0.95, 1e-2)
    g = torch.Generator().manual_seed(5)
    blocks = {0: [torch.randn(N, generator=g) for _ in range(K)], 1: [torch.randn(N + 6, generator=g) for _ in range(K)]}
    ref = {ci: {"m": np.zeros(len(xs[0])), "v": np.full(len(xs[0]), 1e-4)} for ci, xs in blocks.items()}
    for ci, rounds in ((0, 3), (1, 1), (0, 3)):          # block 0 is visited twice: its m / v carry over
        xs = blocks[ci]
        for x in xs:                                     # replicas differ at the visit start: z is their mean
            x.add_(0.1 * torch.randn(x.shape, generator=g))
        strat.begin_block(ci, xs[0].numel(), xs)
        st = ref[ci]
        st["z"] = np.mean([x.double().numpy() for x in xs], axis=0)
        np.testing.assert_allclose(strat.z.numpy(), st["z"], rtol=1e-6, atol=1e-7)
        for _ in range(rounds):
            for x in xs:                                 # local training moves every replica differently
                x.add_(0.05 * torch.randn(x.shape, generator=g) + 0.02)
            want = _literal_round(kind, hp[:4], np.stack([x.double().numpy() for x in xs]), st)
            got = strat.aggregate(0)["dual"]
            assert got == pytest.approx(want, rel=1e-5)
            np.testing.assert_allclose(strat.z.numpy(), st["z"], rtol=1e-5, atol=1e-6)
            np.testing.assert_allclose(strat.m.numpy(), st["m"], rtol=1e-5, atol=1e-7)
            if kind != "avgm":                           # d^2 doubles the relative fp32 error of d = mean - z (cancellation)
                np.testing.assert_allclose(strat.v.numpy(), st["v"], rtol=1e-4, atol=1e-9)
            for x in xs:
                assert torch.equal(x, strat.z)
    assert strat.ms[0] is not strat.ms[1] and (kind == "avgm") == (strat.v is None)


# ------------------------------------------------------------------------------------------ end to end
def _run(**kw):
    lines = []
    eng = federated_multi.run(federated_multi.Config(**{**TINY, **kw}), log=lines.append)
    return eng, [l for l in lines if l.startswith("dual (")]


def _val(line):
    return float(line.rsplit("=", 1)[1])


def test_avgm_without_momentum_at_unit_rate_is_fedavg():
    """beta = 0, lr = 1: z + (mean - z) = mean.  The first round of a visit differs by design (FedAvg's dual is measured
    from z = 0, the server model starts at the replicas' mean), every later round and the weights agree.  (The step is
    evaluated as mean + (lr m - d), so the agreement is exact.)"""
    kw = dict(KW, Nadmm=3, model="Net")
    e0, a = _run(**kw)
    e1, b = _run(server_opt="avgm", server_momentum=0.0, server_lr=1.0, **kw)
    assert len(a) == len(b) == 15
    later = [(x, y) for x, y in zip(a, b) if not re.search(r"avg=0\)", x)]
    assert len(later) == 10
    for x, y in later:
        assert x.split("=")[:-1] == y.split("=")[:-1]
        assert _val(y) == pytest.approx(_val(x), rel=1e-6)
    for x, y in zip(a, b):
        if "avg=0)" in x:
            assert _val(y) < _val(x)                     # a step from the replicas' mean, not from the origin
    assert torch.equal(e1.replicas[0].arenas["net"].data, e0.replicas[0].arenas["net"].data)


@pytest.mark.parametrize("kind", ["avgm", "adam"])
def test_runs_are_deterministic_and_differ_from_fedavg(kind):
    _, a = _run(server_opt=kind, **KW)
    _, b = _run(server_opt=kind, **KW)
    _, c = _run(**KW)
    assert len(a) == 10 and a == b and a != c
    assert all(np.isfinite(_val(l)) for l in a)


class _Killed(Exception):
    pass


def _killed_run(kw, kill_at, **extra):
    """A run that dies once ``kill_at`` minibatch steps are done (counted over the whole run, resumes included); returns
    its residual lines."""
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
            federated_multi.run(federated_multi.Config(**{**TINY, **kw, **extra}), log=lines.append)
    finally:
        Engine.__init__ = orig_init
    return [l for l in lines if l.startswith("dual (")]


RESUME_KW = dict(KW, Nadmm=3, Nloop=2, server_opt="adam")     # 4 steps per round, 12 per block visit


def test_kill_and_resume_reproduces_the_trace(tmp_path):
    """Killed inside a visit of the first loop; the resumed run reaches the second visit of every block (Nloop = 2), so
    it needs the restored state of blocks it never visited itself."""
    _, full = _run(**RESUME_KW)
    assert len(full) == 30
    rec = str(tmp_path / "resume.pt")
    first = _killed_run(RESUME_KW, 19, resume_out=rec)          # inside round 1 of the second visit of loop 0
    assert 0 < len(first) < 15 and os.path.exists(rec)
    st = torch.load(rec, weights_only=False)["strategy_state"]
    assert st["server_opt"] == "adam" and sorted(st["m"]) == sorted(st["v"]) == [0, 1]
    _, second = _run(**RESUME_KW, resume=rec)
    assert first + second == full
    with pytest.raises(ValueError, match="server optimizer"):
        _run(**{**RESUME_KW, "server_opt": "yogi"}, resume=rec)
    with pytest.raises(ValueError, match="strategy 'fedopt'"):     # nor can plain FedAvg continue a FedOpt record
        _run(**{**RESUME_KW, "server_opt": "none"}, resume=rec)


def test_chained_kill_and_resume_keeps_every_block(tmp_path):
    """Kill, resume with a new record, kill again before the resumed run has revisited block 0, resume again: the second
    record must still carry block 0's state (restored from the first record, not yet revisited)."""
    _, full = _run(**RESUME_KW)
    rec1, rec2 = str(tmp_path / "r1.pt"), str(tmp_path / "r2.pt")
    first = _killed_run(RESUME_KW, 19, resume_out=rec1)         # record after round 0 of visit 1: blocks 0, 1
    second = _killed_run(RESUME_KW, 22, resume=rec1, resume_out=rec2)   # record after round 1 of visit 1
    assert len(second) == 1
    st = torch.load(rec2, weights_only=False)["strategy_state"]
    assert sorted(st["m"]) == sorted(st["v"]) == [0, 1]
    st1 = torch.load(rec1, weights_only=False)["strategy_state"]
    assert torch.equal(st["m"][0], st1["m"][0]) and torch.equal(st["v"][0], st1["v"][0])
    _, third = _run(**RESUME_KW, resume=rec2)
    assert first + second + third == full


def _dist_worker(rank, world, port, out):
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch.distributed as dist
    lines = []
    eng = federated_multi.run(federated_multi.Config(server_opt="yogi", **KW, **TINY), log=lines.append)
    if rank == 0:
        torch.save({"lines": lines, "flat": eng.replicas[0].arenas["net"].data.clone()}, out)
    dist.destroy_process_group()


def test_two_process_gloo_equals_single_process(tmp_path):
    import torch.multiprocessing as mp
    out = str(tmp_path / "r0.pt")
    port = 34500 + (os.getpid() % 2000)
    mp.spawn(_dist_worker, args=(2, port, out), nprocs=2, join=True)
    got = torch.load(out, weights_only=False)
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        os.environ.pop(k, None)
    eng, single = _run(server_opt="yogi", **KW)
    multi = [l for l in got["lines"] if l.startswith("dual (")]
    assert len(single) == len(multi) == 10
    for a, b in zip(single, multi):
        assert a.split("=")[:-1] == b.split("=")[:-1]
        assert _val(a) == pytest.approx(_val(b), rel=1e-4)
    torch.testing.assert_close(got["flat"], eng.replicas[0].arenas["net"].data, rtol=1e-4, atol=1e-6)
