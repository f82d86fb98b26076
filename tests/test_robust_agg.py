"""Byzantine-robust aggregation (coordinate-wise median / trimmed mean) and simulated attackers on CPU: configuration,
the ATen operators against float64 numpy / scipy, the FedOpt composition, and ``federated_multi`` end to end (median of
two is the mean, robustness to a sign-flipping and a NaN attacker, determinism, true resume, two gloo processes == one
process)."""
import os

import numpy as np
import pytest
import scipy.stats
import torch

from federated_pytorch_test_b200.algo.byzantine import ByzantineAttack
from federated_pytorch_test_b200.algo.strategies import FedAvg, FedOpt
from federated_pytorch_test_b200.api import federated_multi
from federated_pytorch_test_b200.config import FederatedConfig, FedProxConfig, parse_config
from federated_pytorch_test_b200.parallel import Topology, TorchCollective

TINY = dict(train_size=1024, test_size=128, save_model=False, graphs=False, fast=False)
KW = dict(K=2, Nloop=1, Nadmm=2, max_minibatches=2, check_results=False, use_cuda=False, model="Net")
INF = float("inf")


# ------------------------------------------------------------------------------------------ configuration
def test_defaults_parse_to_the_mean_and_build_todays_strategies():
    cfg = parse_config(FederatedConfig, [])
    assert (cfg.aggregator, cfg.trim_fraction, cfg.byzantine, cfg.attack, cfg.attack_scale) == \
        ("mean", 0.1, 0, "signflip", 4.0)
    cfg = parse_config(FederatedConfig, ["--K", "5", "--aggregator", "trimmed_mean", "--trim_fraction", "0.2",
                                         "--byzantine", "2", "--attack", "gaussian", "--attack_scale", "0.5"])
    assert (cfg.aggregator, cfg.trim_fraction, cfg.byzantine, cfg.attack, cfg.attack_scale) == \
        ("trimmed_mean", 0.2, 2, "gaussian", 0.5)
    topo = Topology.single_process(10, torch.device("cpu"))
    coll = TorchCollective(topo)
    s = federated_multi.make_strategy(FederatedConfig(), coll, topo)
    assert type(s) is FedAvg and s.aggregator == "mean" and s.trim_b == 0
    s = federated_multi.make_strategy(FederatedConfig(server_opt="adam"), coll, topo)
    assert type(s) is FedOpt and s.aggregator == "mean"
    assert federated_multi.make_attack(FederatedConfig()) is None
    s = federated_multi.make_strategy(FederatedConfig(aggregator="trimmed_mean", trim_fraction=0.25), coll, topo)
    assert (s.aggregator, s.trim_b) == ("trimmed_mean", 2)
    s = federated_multi.make_strategy(FederatedConfig(aggregator="median", server_opt="yogi"), coll, topo)
    assert type(s) is FedOpt and (s.aggregator, s.kind) == ("median", "yogi")
    a = federated_multi.make_attack(FederatedConfig(byzantine=3, attack="nan"))
    assert a.attackers == {7, 8, 9} and a.kind == "nan"


@pytest.mark.parametrize("field,bad", [
    ("aggregator", dict(aggregator="krum")),
    ("trim_fraction", dict(trim_fraction=0.5)),
    ("trim_fraction", dict(trim_fraction=-0.01)),
    ("trim_fraction", dict(aggregator="trimmed_mean", trim_fraction=0.05)),          # floor(0.05 * 10) = 0
    ("trim_fraction", dict(aggregator="trimmed_mean", trim_fraction=0.0)),
    ("aggregator", dict(aggregator="median", K=17)),
    ("aggregator", dict(aggregator="trimmed_mean", K=32)),
    ("byzantine", dict(byzantine=-1)),
    ("byzantine", dict(byzantine=10)),
    ("byzantine", dict(K=2, byzantine=2)),
    ("attack", dict(byzantine=1, attack="labelflip")),
    ("attack_scale", dict(attack_scale=0.0)),
    ("attack_scale", dict(attack_scale=-4.0)),
])
def test_invalid_settings_raise(field, bad):
    with pytest.raises(ValueError, match=field):
        FederatedConfig(**bad)
    with pytest.raises(ValueError, match=field):
        parse_config(FederatedConfig, ["--%s=%s" % kv for kv in bad.items()])


def test_mean_accepts_any_K_and_other_drivers_have_no_robust_flags():
    FederatedConfig(K=64)
    FederatedConfig(K=16, aggregator="median")
    for flag in ("--aggregator", "--trim_fraction", "--byzantine", "--attack", "--attack_scale"):
        with pytest.raises(SystemExit):
            parse_config(FedProxConfig, [flag, "median" if flag in ("--aggregator", "--attack") else "1"])
    assert not hasattr(FedProxConfig(), "aggregator")


# ------------------------------------------------------------------------------------------ the operators
def _np_reference(x64, agg, b):
    """float64 ground truth: NaN ordered as +inf (nan_to_num keeping the infinities), then np.median / trim_mean."""
    x64 = np.nan_to_num(x64, nan=np.inf, posinf=np.inf, neginf=-np.inf)
    if agg == "median":
        return np.median(x64, axis=0)
    return scipy.stats.trim_mean(x64, b / x64.shape[0], axis=0)


def _inputs(K, N, nbad, seed):
    """K float32 blocks of odd length N; every coordinate has non-finite values (NaN, +inf, -inf) in up to ``nbad``
    workers, different ones per coordinate."""
    g = torch.Generator().manual_seed(seed)
    xs = [torch.randn(N, generator=g) * (1 + k) for k in range(K)]
    if nbad:
        full = torch.stack(xs)
        for i in range(N):
            cnt = int(torch.randint(0, nbad + 1, (1,), generator=g))
            who = torch.randperm(K, generator=g)[:cnt]
            for w in who.tolist():
                full[w, i] = (float("nan"), INF, -INF)[int(torch.randint(0, 3, (1,), generator=g))]
        xs = list(full.unbind(0))
        xs = [x.clone() for x in xs]
    return xs


def _cases():
    for K in (1, 2, 3, 4, 5, 8, 10, 16):
        yield K, "median", 0, (K - 1) // 2
        for b in sorted({1, (K - 1) // 2}):
            if 2 * b < K:
                yield K, "trimmed_mean", b, b


@pytest.mark.parametrize("K,agg,b,nbad", list(_cases()))
@pytest.mark.parametrize("with_bad", [False, True])
def test_operator_matches_numpy_and_scipy(K, agg, b, nbad, with_bad):
    N = 301
    xs = _inputs(K, N, nbad if with_bad else 0, 100 * K + b)
    topo = Topology.single_process(K, torch.device("cpu"))
    coll = TorchCollective(topo)
    want = _np_reference(np.stack([x.double().numpy() for x in xs]), agg, b)
    got = coll.robust_aggregate(xs, agg, b)
    assert torch.isfinite(got).all()
    np.testing.assert_allclose(got.double().numpy(), want, rtol=2e-6, atol=1e-6)
    if agg == "median" and K % 2:                        # the middle value itself
        assert np.array_equal(got.double().numpy(), want)
    z = torch.full((N,), 0.5)
    xr = [x.clone() for x in xs]
    dual_sq = coll.robust_(xr, z, agg, b)
    assert torch.equal(z, got) and all(torch.equal(x, got) for x in xr)
    assert float(dual_sq) == pytest.approx(float(((0.5 - got.double()) ** 2).sum()), rel=1e-5)
    z2 = torch.zeros(N)
    xr = [x.clone() for x in xs]
    coll.robust_(xr, z2, agg, b, write_back=False)
    assert torch.equal(z2, got)
    for x, y in zip(xr, xs):                             # no write-back: the replicas are untouched
        torch.testing.assert_close(x, y, rtol=0, atol=0, equal_nan=True)


def test_extreme_values_do_not_cancel_and_more_bad_workers_than_b_reach_the_aggregate():
    K = 5
    coll = TorchCollective(Topology.single_process(K, torch.device("cpu")))
    xs = [torch.tensor([1.0, 2.0, 3.0]) for _ in range(K)]
    xs[4] = torch.tensor([1e30, -1e30, float("nan")])
    assert torch.equal(coll.robust_aggregate(xs, "trimmed_mean", 1), torch.tensor([1.0, 2.0, 3.0]))
    assert torch.equal(coll.robust_aggregate(xs, "median", 0), torch.tensor([1.0, 2.0, 3.0]))
    xs[3] = torch.tensor([float("nan")] * 3)                    # two large values where b = 1: one is kept
    out = coll.robust_aggregate(xs, "trimmed_mean", 1)
    assert out[0] > 1e29 and out[1] == 2.0 and out[2] == INF
    xs[2] = torch.tensor([INF] * 3)                             # three of five: the median is one of them
    assert torch.equal(coll.robust_aggregate(xs, "median", 0), torch.tensor([1e30, 2.0, INF]))   # NaN orders as +inf
    with pytest.raises(ValueError, match="trim"):
        coll.robust_aggregate(xs, "trimmed_mean", 3)
    with pytest.raises(ValueError, match="robust"):
        coll.robust_aggregate(xs, "krum", 0)


def test_even_median_is_the_halved_sum_of_the_middle_pair():
    coll = TorchCollective(Topology.single_process(4, torch.device("cpu")))
    xs = [torch.tensor([v], dtype=torch.float32) for v in (3e38, 3e38, 3e38, -1.0)]
    assert torch.equal(coll.robust_aggregate(xs, "median", 0), torch.tensor([INF]))    # (lo + hi) * 0.5 in float32
    xs = [torch.tensor([v], dtype=torch.float32) for v in (0.1, 0.7, -1.0, 5.0)]
    lo, hi = torch.tensor(0.1), torch.tensor(0.7)
    assert torch.equal(coll.robust_aggregate(xs, "median", 0), ((lo + hi) * 0.5).reshape(1))


@pytest.mark.parametrize("kind,agg", [("adam", "median"), ("avgm", "trimmed_mean"), ("yogi", "median")])
def test_fedopt_composition_over_rounds(kind, agg):
    """Robust FedOpt: the pseudo-gradient is aggregate - z; the server model at the start of a visit is the mean."""
    K, N = 5, 257
    topo = Topology.single_process(K, torch.device("cpu"))
    lr = {"avgm": 0.7, "adam": 0.02, "yogi": 0.03}[kind]
    strat = FedOpt(TorchCollective(topo), topo, kind, lr=lr, momentum=0.8, beta1=0.85, beta2=0.95, tau=1e-2,
                   aggregator=agg, trim_fraction=0.2)
    assert strat.trim_b == (1 if agg == "trimmed_mean" else 0)
    b1 = 0.8 if kind == "avgm" else 0.85
    g = torch.Generator().manual_seed(7)
    xs = [torch.randn(N, generator=g) for _ in range(K)]
    strat.begin_block(0, N, xs)
    z = np.mean([x.double().numpy() for x in xs], axis=0)
    np.testing.assert_allclose(strat.z.numpy(), z, rtol=1e-6, atol=1e-7)
    m, v = np.zeros(N), np.full(N, 1e-4)
    for r in range(4):
        for k, x in enumerate(xs):
            x.add_(0.05 * torch.randn(N, generator=g) + 0.02 * k)
        xs[4].add_(10.0)                                             # an outlier the robust rule ignores
        a = _np_reference(np.stack([x.double().numpy() for x in xs]), agg, strat.trim_b)
        d = a - z
        if kind == "avgm":
            m = b1 * m + d
            znew = z + lr * m
        else:
            m = b1 * m + (1 - b1) * d
            if kind == "adam":
                v = 0.95 * v + 0.05 * d * d
            else:
                v = v - 0.05 * d * d * np.sign(v - d * d)
            znew = z + lr * m / (np.sqrt(v) + 1e-2)
        want = np.linalg.norm(z - znew) / N
        z = znew
        got = strat.aggregate(r)["dual"]
        assert got == pytest.approx(want, rel=1e-4)
        np.testing.assert_allclose(strat.z.numpy(), z, rtol=1e-4, atol=1e-6)
        np.testing.assert_allclose(strat.m.numpy(), m, rtol=1e-4, atol=1e-6)
        assert all(torch.equal(x, strat.z) for x in xs)


def test_gaussian_draws_depend_on_seed_worker_and_round_only():
    a = ByzantineAttack(4, 2, "gaussian", 2.0, seed=3)
    like = torch.zeros(1000)
    assert torch.equal(a.noise(3, 5, like), a.noise(3, 5, like))
    assert not torch.equal(a.noise(3, 5, like), a.noise(2, 5, like))
    assert not torch.equal(a.noise(3, 5, like), a.noise(3, 6, like))
    assert not torch.equal(a.noise(3, 5, like), ByzantineAttack(4, 2, "gaussian", 2.0, seed=4).noise(3, 5, like))
    xs = [torch.ones(1000) for _ in range(4)]
    z = torch.full((1000,), 0.5)
    a.apply(xs, [0, 1, 2, 3], z, 5)
    assert torch.equal(xs[0], torch.ones(1000)) and torch.equal(xs[1], torch.ones(1000))
    assert torch.allclose(xs[3], z + 2.0 * a.noise(3, 5, like))
    s = ByzantineAttack(4, 1, "signflip", 4.0)
    xs = [torch.full((1000,), 2.0) for _ in range(4)]
    s.apply(xs, [0, 1, 2, 3], z, 0)
    assert torch.equal(xs[3], torch.full((1000,), 0.5 - 4.0 * 1.5)) and torch.equal(xs[2], torch.full((1000,), 2.0))


# ------------------------------------------------------------------------------------------ end to end
def _run(**kw):
    lines = []
    eng = federated_multi.run(federated_multi.Config(**{**TINY, **kw}), log=lines.append)
    return eng, [l for l in lines if l.startswith("dual (")]


def _val(line):
    return float(line.rsplit("=", 1)[1])


def test_median_of_two_is_the_mean():
    e0, a = _run(**KW)
    e1, b = _run(**KW, aggregator="median")
    assert len(a) == 10 and a == b
    assert torch.equal(e0.replicas[0].arenas["net"].data, e1.replicas[0].arenas["net"].data)


ATTACK_KW = dict(KW, K=5, trim_fraction=0.2)


def _deviation(trace, clean):
    """Largest factor (as |log|) between a dual trace and the attack-free one."""
    return max(abs(np.log(_val(x) / _val(y))) for x, y in zip(trace, clean))


def test_signflip_attacker_moves_the_mean_but_not_the_robust_rules():
    devs = {}
    for agg in ("mean", "median", "trimmed_mean"):
        _, clean = _run(**ATTACK_KW, aggregator=agg)
        _, hit = _run(**ATTACK_KW, aggregator=agg, byzantine=1, attack="signflip")
        _, again = _run(**ATTACK_KW, aggregator=agg, byzantine=1, attack="signflip")
        assert hit == again and len(hit) == len(clean) == 10                 # deterministic
        devs[agg] = _deviation(hit, clean)
    print("largest |log| ratio of the dual trace to the attack-free run:", devs)
    assert devs["mean"] > 1.0
    assert devs["median"] < 0.1 * devs["mean"] and devs["trimmed_mean"] < 0.1 * devs["mean"]


def test_nan_attacker_trips_the_guard_for_the_mean_only():
    with pytest.raises(FloatingPointError, match="non-finite"):
        _run(**ATTACK_KW, byzantine=1, attack="nan")
    for agg in ("median", "trimmed_mean"):
        eng, trace = _run(**ATTACK_KW, aggregator=agg, byzantine=1, attack="nan")
        assert len(trace) == 10 and all(np.isfinite(_val(l)) for l in trace)
        assert torch.isfinite(eng.replicas[0].arenas["net"].data).all()


class _Killed(Exception):
    pass


def _killed_run(kw, kill_at, **extra):
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


def test_kill_and_resume_with_a_gaussian_attacker_reproduces_the_trace(tmp_path):
    kw = dict(KW, K=3, Nadmm=3, aggregator="median", byzantine=1, attack="gaussian", attack_scale=0.5)
    _, full = _run(**kw)
    assert len(full) == 15
    rec = str(tmp_path / "resume.pt")
    first = _killed_run(kw, 27, resume_out=rec)                  # 6 steps per round: round 1 of the second block's visit
    assert 0 < len(first) < 15 and os.path.exists(rec)
    st = torch.load(rec, weights_only=False)["strategy_state"]
    assert st["aggregator"] == "median"
    _, second = _run(**kw, resume=rec)
    assert first + second == full
    with pytest.raises(ValueError, match="aggregator"):
        _run(**{**kw, "aggregator": "mean"}, resume=rec)


def _dist_worker(rank, world, port, out, agg):
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch.distributed as dist
    lines = []
    eng = federated_multi.run(federated_multi.Config(**{**DIST_KW, "aggregator": agg}, **TINY), log=lines.append)
    if rank == 0:
        torch.save({"lines": lines, "flat": eng.replicas[0].arenas["net"].data.clone()}, out)
    dist.destroy_process_group()


DIST_KW = dict(KW, K=4, trim_fraction=0.25, byzantine=1, attack="gaussian", attack_scale=0.5)


@pytest.mark.parametrize("agg", ["median", "trimmed_mean"])
def test_two_process_gloo_equals_single_process(tmp_path, agg):
    import torch.multiprocessing as mp
    out = str(tmp_path / "r0.pt")
    port = 35500 + (os.getpid() % 2000) + (agg == "median")
    mp.spawn(_dist_worker, args=(2, port, out, agg), nprocs=2, join=True)
    got = torch.load(out, weights_only=False)
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        os.environ.pop(k, None)
    eng, single = _run(**DIST_KW, aggregator=agg)
    multi = [l for l in got["lines"] if l.startswith("dual (")]
    assert len(single) == len(multi) == 10
    for a, b in zip(single, multi):
        assert a.split("=")[:-1] == b.split("=")[:-1]
        assert _val(a) == pytest.approx(_val(b), rel=1e-4)
    torch.testing.assert_close(got["flat"], eng.replicas[0].arenas["net"].data, rtol=1e-4, atol=1e-6)
