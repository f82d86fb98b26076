"""Client-level differential privacy (DP-FedAvg) on CPU: configuration, the accountant against scipy, the noise draw,
the ATen operators against a float64 transcription, and ``federated_multi`` end to end (bitwise FedAvg without noise,
a bounded sign-flipping attacker, true resume, two gloo processes == one process)."""
import math
import os

import numpy as np
import pytest
import scipy.optimize
import scipy.stats
import torch

from federated_pytorch_test_b200.algo import privacy
from federated_pytorch_test_b200.algo.strategies import FedAvg, FedOpt
from federated_pytorch_test_b200.api import federated_multi
from federated_pytorch_test_b200.config import FederatedConfig, FedProxConfig, parse_config
from federated_pytorch_test_b200.parallel import Topology, TorchCollective

TINY = dict(train_size=1024, test_size=128, save_model=False, graphs=False, fast=False)
KW = dict(K=2, Nloop=1, Nadmm=2, max_minibatches=2, check_results=False, use_cuda=False, model="Net")


# ------------------------------------------------------------------------------------------ configuration
def test_defaults_are_off_and_build_todays_strategies():
    cfg = parse_config(FederatedConfig, [])
    assert (cfg.dp_clip, cfg.dp_noise, cfg.dp_delta) == (0.0, 1.0, 1e-5)
    topo = Topology.single_process(4, torch.device("cpu"))
    s = federated_multi.make_strategy(cfg, TorchCollective(topo), topo)
    assert type(s) is FedAvg and not s.dp and s.state().keys() == {"z"}
    cfg = parse_config(FederatedConfig, ["--dp_clip", "1e-3", "--dp_noise", "0.5", "--dp_delta", "1e-6",
                                         "--server_opt", "adam"])
    s = federated_multi.make_strategy(cfg, TorchCollective(topo), topo)
    assert type(s) is FedOpt and s.dp and (s.dp_clip, s.dp_noise, s.dp_delta) == (1e-3, 0.5, 1e-6)


@pytest.mark.parametrize("field,bad", [
    ("dp_clip", dict(dp_clip=-1e-3)),
    ("dp_clip", dict(dp_clip=float("inf"))),
    ("dp_clip", dict(dp_clip=float("nan"))),
    ("dp_noise", dict(dp_noise=-0.1)),
    ("dp_delta", dict(dp_delta=0.0)),
    ("dp_delta", dict(dp_delta=1.0)),
    ("aggregator", dict(dp_clip=1e-3, aggregator="median")),
])
def test_invalid_settings_raise(field, bad):
    with pytest.raises(ValueError, match=field):
        FederatedConfig(**bad)
    with pytest.raises(ValueError, match=field):
        parse_config(FederatedConfig, ["--%s=%s" % kv for kv in bad.items()])


def test_other_drivers_have_no_dp_flags():
    for flag in ("--dp_clip", "--dp_noise", "--dp_delta"):
        with pytest.raises(SystemExit):
            parse_config(FedProxConfig, [flag, "0.1"])


# ------------------------------------------------------------------------------------------ accountant
def _scipy_epsilon(sigma, T, delta):
    mu = math.sqrt(T) / sigma
    f = lambda e: scipy.stats.norm.cdf(-e / mu + mu / 2) - math.exp(e) * scipy.stats.norm.cdf(-e / mu - mu / 2) - delta
    return scipy.optimize.brentq(f, 0.0, 500.0, xtol=1e-12)


def _rdp_epsilon(sigma, T, delta):
    alphas = np.concatenate([np.linspace(1.01, 10, 2000), np.linspace(10, 2000, 20000)])
    return float(np.min(T * alphas / (2 * sigma ** 2) + np.log(1 / delta) / (alphas - 1)))


@pytest.mark.parametrize("sigma,T,want", [(1.0, 1, 4.377), (10.0, 360, 9.371), (20.0, 360, 4.119)])
def test_accountant_reference_values(sigma, T, want):
    assert privacy.gaussian_epsilon(sigma, T, 1e-5) == pytest.approx(want, abs=1e-3)


@pytest.mark.parametrize("sigma,T,delta", [(0.7, 1, 1e-5), (1.0, 50, 1e-5), (3.0, 1000, 1e-6), (10.0, 360, 1e-3),
                                           (40.0, 5, 1e-5)])
def test_accountant_against_scipy_and_rdp(sigma, T, delta):
    eps = privacy.gaussian_epsilon(sigma, T, delta)
    assert eps == pytest.approx(_scipy_epsilon(sigma, T, delta), rel=1e-7, abs=1e-9)
    assert eps <= _rdp_epsilon(sigma, T, delta)
    assert privacy.noise_for_epsilon(eps, delta, T) == pytest.approx(sigma, rel=1e-6)


def test_accountant_edges():
    assert _rdp_epsilon(10.0, 360, 1e-5) == pytest.approx(10.905, abs=2e-3)
    assert privacy.gaussian_epsilon(0.0, 10, 1e-5) == math.inf
    assert privacy.gaussian_epsilon(1.0, 0, 1e-5) == 0.0
    assert privacy.gaussian_epsilon(1e4, 1, 0.5) == 0.0
    e = [privacy.gaussian_epsilon(2.0, T, 1e-5) for T in (1, 10, 100)]
    assert e[0] < e[1] < e[2]
    assert "planned_rounds=360 epsilon=9.3709" in privacy.dp_line(10.0, 1e-3, 1e-5, 360, planned=True)


# ------------------------------------------------------------------------------------------ noise draw
def test_noise_moments_and_ks():
    x = privacy.dp_noise(privacy.noise_key(69), 3, 1_000_001)
    assert x.shape == (1_000_001,)
    assert abs(x.mean()) < 5e-3 and abs(x.std() - 1.0) < 3e-3
    assert abs(scipy.stats.skew(x)) < 1e-2 and abs(scipy.stats.kurtosis(x)) < 2e-2
    assert scipy.stats.kstest(x, "norm").pvalue > 1e-3
    assert np.abs(x).max() <= math.sqrt(48 * math.log(2)) + 1e-12


def test_noise_rounds_are_uncorrelated_and_keyed():
    k = privacy.noise_key(5)
    a, b = privacy.dp_noise(k, 0, 200_000), privacy.dp_noise(k, 1, 200_000)
    assert abs(np.corrcoef(a, b)[0, 1]) < 1e-2
    assert abs(np.corrcoef(a[0::2], a[1::2])[0, 1]) < 1e-2                 # the two halves of a Box-Muller pair
    assert not np.array_equal(a, privacy.dp_noise(privacy.noise_key(6), 0, 200_000))
    assert np.array_equal(a, privacy.dp_noise(k, 0, 200_000))


def _xi_scalar(key, t, i):
    """xi_i of round t from the documented formula, one coordinate at a time with Python integers."""
    M = (1 << 64) - 1

    def F(z):
        z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M
        z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M
        return z ^ (z >> 31)
    G = 0x9E3779B97F4A7C15
    w = F((F((key + (t + 1) * G) & M) + (i // 2 + 1) * G) & M)
    u1, u2 = ((w >> 40) + 1) * 2.0 ** -24, (w & 0xFFFFFF) * 2.0 ** -24
    r = math.sqrt(-2.0 * math.log(u1))
    return r * (math.sin if i % 2 else math.cos)(2.0 * math.pi * u2)


def test_noise_is_a_function_of_key_round_and_coordinate_only():
    """Each coordinate's draw, evaluated on its own (as a rank or a two-shot slice starting anywhere would), equals the
    block's draw at that coordinate, and a shorter block draws a prefix of it."""
    k = privacy.noise_key(1)
    full = privacy.dp_noise(k, 7, 100_001)
    for i in (0, 1, 2, 3, 31, 32, 455, 456, 4097, 50_000, 100_000):
        assert full[i] == pytest.approx(_xi_scalar(k, 7, i), rel=1e-12, abs=1e-12)
    assert np.array_equal(privacy.dp_noise(k, 7, 333), full[:333])
    assert privacy.dp_noise(k, 8, 1)[0] == pytest.approx(_xi_scalar(k, 8, 0), rel=1e-12)


# ------------------------------------------------------------------------------------------ the operator
def _dp_reference(xs64, z64, C, std, xi):
    """float64 transcription of one DP round: clipped workers, mean + std xi, #clipped and the norm sum."""
    out, clipped, norms = [], 0, 0.0
    for x in xs64:
        d = x - z64
        n = np.linalg.norm(d)
        norms += n
        if n > C:
            clipped += 1
            x = z64 + (C / n) * d
        out.append(x)
    return out, np.mean(out, axis=0) + std * xi, clipped, norms


@pytest.mark.parametrize("K", [1, 2, 3, 5, 8])
@pytest.mark.parametrize("kind", [None, "avgm", "adagrad", "adam", "yogi"])
def test_dp_round_matches_float64(K, kind):
    N, sigma, clip = 301, 0.8, 0.05
    C = clip * math.sqrt(N)
    topo = Topology.single_process(K, torch.device("cpu"))
    coll = TorchCollective(topo)
    kw = dict(dp_clip=clip, dp_noise=sigma, dp_delta=1e-5, seed=11)
    strat = FedAvg(coll, topo, **kw) if kind is None else FedOpt(coll, topo, kind, lr=0.05, momentum=0.5, beta1=0.8,
                                                                 beta2=0.9, tau=1e-2, **kw)
    g = torch.Generator().manual_seed(K)
    z0 = torch.randn(N, generator=g)
    xs = [z0.clone() for _ in range(K)]
    strat.begin_block(0, N, xs)
    assert torch.equal(strat.z, z0)
    z = z0.double().numpy()
    m, v = np.zeros(N), np.full(N, 1e-4)
    for r in range(3):
        for k, x in enumerate(xs):                          # even workers stay inside the bound, odd ones leave it
            x.add_(torch.randn(N, generator=g) * (3.0 * C if k % 2 else 0.2 * C) / math.sqrt(N))
        xs64 = [x.double().numpy() for x in xs]
        xi = privacy.dp_noise(strat.dp_key, r, N)
        before = [x.clone() for x in xs]
        ref, mean, clipped, norms = _dp_reference(xs64, z, C, sigma * C / K, xi)
        if kind is None:
            znew = mean
        else:
            d = mean - z
            if kind == "avgm":
                m = 0.5 * m + d
                znew = z + 0.05 * m
            else:
                m = 0.8 * m + 0.2 * d
                v = {"adagrad": v + d * d, "adam": 0.9 * v + 0.1 * d * d,
                     "yogi": v - 0.1 * d * d * np.sign(v - d * d)}[kind]
                znew = z + 0.05 * m / (np.sqrt(v) + 1e-2)
        if kind is None:
            # the clip writes only the workers over the bound
            strat.coll.dp_clip_(xs, strat.z, C)
            for k in range(K):
                if np.linalg.norm(xs64[k] - z) <= C:
                    assert torch.equal(xs[k], before[k])
                else:
                    np.testing.assert_allclose(xs[k].double().numpy(), ref[k], rtol=1e-5, atol=1e-6)
            for x, b in zip(xs, before):
                x.copy_(b)
        met = strat.aggregate(r)
        assert met["dp_clipped"] == clipped == (K // 2)
        assert met["dp_update_norm"] == pytest.approx(norms / K, rel=1e-5)
        assert met["dp_clip_norm"] == pytest.approx(C)
        assert met["dp_epsilon"] == pytest.approx(privacy.gaussian_epsilon(sigma, r + 1, 1e-5))
        assert met["dual"] == pytest.approx(np.linalg.norm(z - znew) / N, rel=1e-4)
        np.testing.assert_allclose(strat.z.double().numpy(), znew, rtol=1e-5, atol=1e-6)
        assert all(torch.equal(x, strat.z) for x in xs)
        z = znew
    assert int(strat.dp_t) == strat.dp_rounds == 3


def test_huge_finite_update_is_clipped():
    """An update whose float32 sum of squares would overflow is still clipped to the bound (norms in double)."""
    K, N, C = 3, 1001, 0.5
    coll = TorchCollective(Topology.single_process(K, torch.device("cpu")))
    z = torch.randn(N, generator=torch.Generator().manual_seed(0))
    xs = [z + 0.001, z - 0.001, z + 1e30]
    coll.dp_clip_(xs, z, C)
    assert coll.last_dp[0] == 1 and coll.last_dp[1] == pytest.approx(1e30 * math.sqrt(N), rel=1e-6)
    assert float(torch.linalg.vector_norm(xs[2].double() - z.double())) == pytest.approx(C, rel=1e-5)
    xs = [z + 0.001, z - 0.001, torch.full((N,), 3e38)]
    xs[2][::2] = -3e38
    coll.dp_clip_(xs, z, C)
    assert torch.isfinite(xs[2]).all() and float(torch.linalg.vector_norm(xs[2].double() - z.double())) <= C * 1.0001


def test_large_signflip_attacker_stays_finite():
    _, trace, _ = _run(**{**KW, "K": 5}, dp_clip=1e-3, dp_noise=1.0, byzantine=1, attack="signflip", attack_scale=1e30)
    _, clean, _ = _run(**{**KW, "K": 5}, dp_clip=1e-3, dp_noise=1.0)
    assert len(trace) == 10 and all(math.isfinite(_val(l)) for l in trace)
    assert max(_val(a) / _val(b) for a, b in zip(trace, clean)) < 10.0


def test_alignment_padding_gets_no_noise():
    eng, _, _ = _run(**KW, dp_clip=1e-3, dp_noise=5.0)
    arena = eng.replicas[0].arenas["net"]
    pad = torch.ones(arena.total, dtype=torch.bool)
    for off, n in zip(arena.offsets, arena.numels):
        pad[off:off + n] = False
    assert pad.any() and torch.equal(arena.data[pad], torch.zeros(int(pad.sum())))


def test_nonfinite_update_is_not_clipped_and_reaches_the_mean():
    K, N = 3, 17
    coll = TorchCollective(Topology.single_process(K, torch.device("cpu")))
    z = torch.zeros(N)
    xs = [torch.ones(N) for _ in range(K)]
    xs[2][3] = float("nan")
    coll.dp_clip_(xs, z, 1.0)
    assert coll.last_dp[0] == 2 and math.isnan(coll.last_dp[1])
    assert math.isnan(float(xs[2][3])) and float(xs[2][0]) == 1.0
    assert math.isnan(float(coll.fedavg_(xs, z)))


# ------------------------------------------------------------------------------------------ end to end
def _run(**kw):
    lines = []
    eng = federated_multi.run(federated_multi.Config(**{**TINY, **kw}), log=lines.append)
    return eng, [l for l in lines if l.startswith("dual (")], [l for l in lines if l.startswith("dp:")]


def _val(line):
    return float(line.rsplit("=", 1)[1])


def test_large_clip_without_noise_is_bitwise_fedavg():
    e0, a, _ = _run(**KW)
    e1, b, dp = _run(**KW, dp_clip=1e6, dp_noise=0.0)
    assert len(a) == len(b) == 10
    assert torch.equal(e0.replicas[0].arenas["net"].data, e1.replicas[0].arenas["net"].data)
    assert torch.equal(e0.replicas[1].arenas["net"].data, e1.replicas[1].arenas["net"].data)
    assert a[1::2] == b[1::2]                     # only the first round of a visit (z = server model, not 0) differs
    assert dp == ["dp: sigma=0 clip=1e+06*sqrt(N) delta=1e-05 planned_rounds=10 epsilon=inf",
                  "dp: sigma=0 clip=1e+06*sqrt(N) delta=1e-05 rounds=10 epsilon=inf"]


def test_replicas_are_equal_when_a_visit_starts():
    orig = FedAvg.begin_block
    seen = []

    def check(self, ci, N, xs):
        seen.append(all(torch.equal(x, xs[0]) for x in xs))
        orig(self, ci, N, xs)
    FedAvg.begin_block = check
    try:
        _run(**{**KW, "K": 3}, dp_clip=1e-3, dp_noise=1.0)
    finally:
        FedAvg.begin_block = orig
    assert len(seen) == 5 and all(seen)


def test_signflip_attacker_is_bounded_by_clipping():
    """With sigma = 0 one clipped attacker moves the aggregate by at most 2 b C / K from the attack-free one."""
    K, b, clip = 5, 1, 2e-3
    topo = Topology.single_process(K, torch.device("cpu"))
    from federated_pytorch_test_b200.algo.byzantine import ByzantineAttack
    g = torch.Generator().manual_seed(3)
    N = 1001
    C = clip * math.sqrt(N)
    z = torch.randn(N, generator=g)
    xs = [z + torch.randn(N, generator=g) * 0.01 for _ in range(K)]
    ratios = []
    for scale in (1.0, 4.0, 100.0):
        clean = FedAvg(TorchCollective(topo), topo, dp_clip=clip, dp_noise=0.0)
        hit = FedAvg(TorchCollective(topo), topo, dp_clip=clip, dp_noise=0.0)
        xc, xh = [x.clone() for x in xs], [x.clone() for x in xs]
        clean.begin_block(0, N, [z.clone() for _ in range(K)])
        hit.begin_block(0, N, [z.clone() for _ in range(K)])
        clean.xs, hit.xs = xc, xh
        ByzantineAttack(K, b, "signflip", scale).apply(xh, list(range(K)), z, 0)
        clean.aggregate(0)
        hit.aggregate(0)
        ratios.append(float(torch.linalg.vector_norm(hit.z - clean.z)) / (2 * b * C / K))
    print("attacked / attack-free distance over 2bC/K:", ratios)
    assert max(ratios) <= 1.0 + 1e-5


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


@pytest.mark.parametrize("server_opt", ["none", "adam"])
def test_kill_and_resume_reproduces_the_noisy_trace(tmp_path, server_opt):
    kw = dict(KW, K=3, Nadmm=3, dp_clip=1e-3, dp_noise=2.0, server_opt=server_opt)
    _, full, dp_full = _run(**kw)
    assert len(full) == 15
    rec = str(tmp_path / "resume.pt")
    first = _killed_run(dict(kw, resume_out=rec), 27)
    assert 0 < len(first) < 15 and os.path.exists(rec)
    st = torch.load(rec, weights_only=False)["strategy_state"]
    assert st["dp_t"] == len(first) and st["dp"][:3] == (1e-3, 2.0, 1e-5)
    _, second, dp = _run(**kw, resume=rec)
    assert first + second == full
    assert dp[-1] == dp_full[-1]
    with pytest.raises(ValueError, match="DP settings"):
        _run(**{**kw, "dp_noise": 1.0}, resume=rec)
    with pytest.raises(ValueError, match="DP settings"):
        _run(**{**kw, "dp_clip": 0.0}, resume=rec)


def _dist_worker(rank, world, port, out):
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch.distributed as dist
    lines = []
    eng = federated_multi.run(federated_multi.Config(**DIST_KW, **TINY), log=lines.append)
    if rank == 0:
        torch.save({"lines": lines, "flat": eng.replicas[0].arenas["net"].data.clone()}, out)
    dist.destroy_process_group()


DIST_KW = dict(KW, K=4, dp_clip=1e-3, dp_noise=1.0, byzantine=1, attack="signflip")


def test_two_process_gloo_equals_single_process(tmp_path):
    import torch.multiprocessing as mp
    out = str(tmp_path / "r0.pt")
    port = 37600 + (os.getpid() % 2000)
    mp.spawn(_dist_worker, args=(2, port, out), nprocs=2, join=True)
    got = torch.load(out, weights_only=False)
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        os.environ.pop(k, None)
    eng, single, dp = _run(**DIST_KW)
    multi = [l for l in got["lines"] if l.startswith("dual (")]
    assert len(single) == len(multi) == 10
    for a, b in zip(single, multi):
        assert a.split("=")[:-1] == b.split("=")[:-1]
        assert _val(a) == pytest.approx(_val(b), rel=1e-4)
    assert [l for l in got["lines"] if l.startswith("dp:")] == dp
    # the all-reduce sums in another order; the attacker and the noise amplify that in a few weights
    torch.testing.assert_close(got["flat"], eng.replicas[0].arenas["net"].data, rtol=1e-4, atol=1e-3)

