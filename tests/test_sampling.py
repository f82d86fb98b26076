"""Client sampling and sample-weighted federated averaging over Dirichlet shards, on CPU: the partition, the numpy oracle
of the participant draw and the weights, the ATen operators against float64 references, the engine's treatment of
workers that sit out, true resume, and configuration."""
import os

import numpy as np
import pytest
import torch
from scipy import stats

from federated_pytorch_test_b200.algo import sampling
from federated_pytorch_test_b200.algo.engine import Engine
from federated_pytorch_test_b200.algo.strategies import FedAvg, FedOpt
from federated_pytorch_test_b200.api import federated_multi
from federated_pytorch_test_b200.config import FederatedConfig, FedProxConfig, VAEConfig, CPCConfig, parse_config
from federated_pytorch_test_b200.data.cifar import class_histogram, dirichlet_shards, make_synthetic_cifar
from federated_pytorch_test_b200.parallel import Topology, TorchCollective
from federated_pytorch_test_b200.parallel.collective import SampleRound

TINY = dict(train_size=1024, test_size=128, save_model=False, graphs=False, fast=False)
KW = dict(K=4, Nloop=1, Nadmm=2, max_minibatches=2, check_results=False, use_cuda=False, model="Net")
KEY = sampling.sample_key(69)
CPU = torch.device("cpu")


# ------------------------------------------------------------------------------------------ Dirichlet partition
def _labels(n=5000):
    return make_synthetic_cifar(True, 1234, n)[1]


@pytest.mark.parametrize("K,alpha", [(4, 0.5), (8, 0.3), (10, 5.0)])
def test_dirichlet_shards_are_disjoint_cover_everything_and_respect_min_size(K, alpha):
    lab = _labels()
    shards = dirichlet_shards(lab, K, alpha, 7, 64)
    assert len(shards) == K
    allidx = np.concatenate(shards)
    assert allidx.size == lab.numel() and np.array_equal(np.sort(allidx), np.arange(lab.numel()))
    assert min(s.size for s in shards) >= 64
    assert all(np.all(np.diff(s) > 0) for s in shards)
    again = dirichlet_shards(lab, K, alpha, 7, 64)
    assert all(np.array_equal(a, b) for a, b in zip(shards, again))
    other = dirichlet_shards(lab, K, alpha, 8, 64)
    assert not all(np.array_equal(a, b) for a, b in zip(shards, other))


def test_dirichlet_shards_follow_the_drawn_proportions():
    lab = _labels()
    K, alpha, seed = 6, 0.4, 3
    hist = np.array(class_histogram(lab, dirichlet_shards(lab, K, alpha, seed, 0)))
    rng = np.random.Generator(np.random.PCG64(seed))                 # min_size 0: the first draw is kept
    labn = lab.numpy()
    for c in range(10):
        idx = np.flatnonzero(labn == c)
        rng.shuffle(idx)
        p = rng.dirichlet(np.full(K, alpha))
        cuts = np.floor(np.cumsum(p) * idx.size).astype(np.int64)
        cuts[-1] = idx.size
        want = np.diff(np.concatenate([[0], cuts]))
        assert np.array_equal(hist[:, c], want)
        assert np.abs(want / idx.size - p).max() <= 2.0 / idx.size + 1e-12


def test_dirichlet_redraw_cap_raises():
    with pytest.raises(ValueError, match=r"alpha = 0.01.*K = 10"):
        dirichlet_shards(_labels(2000), 10, 0.01, 0, 200)


# ------------------------------------------------------------------------------------------ participants and weights
def test_participants_are_the_smallest_words():
    for K, S in ((1, 1), (5, 2), (8, 3), (16, 16), (64, 7)):
        for t in range(50):
            p = sampling.participants(KEY, t, K, S)
            h = sampling.words(KEY, t, K)
            brute = sorted(sorted(range(K), key=lambda k: (int(h[k]), k))[:S])
            assert p.tolist() == brute and len(set(p.tolist())) == S
            assert np.array_equal(p, sampling.participants(KEY, t, K, S))
            assert np.array_equal(np.flatnonzero(sampling.mask(KEY, t, K, S)), p)
    assert not all(np.array_equal(sampling.participants(KEY, t, 8, 3), sampling.participants(KEY + 1, t, 8, 3))
                   for t in range(10))
    for bad in (0, 9):
        with pytest.raises(ValueError, match="1..K"):
            sampling.participants(KEY, 0, 8, bad)


def test_participant_frequencies_are_uniform():
    K, S, T = 8, 3, 20000
    counts = np.zeros(K)
    pairs = np.zeros((K, K))
    for t in range(T):
        p = sampling.participants(KEY, t, K, S)
        counts[p] += 1
        pairs[np.ix_(p, p)] += 1
    assert stats.chisquare(counts, np.full(K, T * S / K)).pvalue > 1e-3
    off = pairs[~np.eye(K, dtype=bool)]                   # every pair equally often: E = T S (S - 1) / (K (K - 1))
    assert stats.chisquare(off, np.full(off.size, off.sum() / off.size)).pvalue > 1e-3


def test_weights_are_correctly_rounded_quotients():
    n = np.array([6249, 100, 33333, 7, 12345, 1])
    m = np.array([True, False, True, True, False, True])
    w = sampling.weights(n, m)
    assert w.dtype == np.float32 and np.all(w[~m] == 0)
    tot = int(n[m].sum())
    for k in np.flatnonzero(m):
        assert w[k] == np.float32(np.float32(n[k]) / np.float32(tot))
        assert abs(float(w[k]) - n[k] / tot) <= np.spacing(np.float32(n[k] / tot))
    assert abs(float(w.sum()) - 1.0) < 1e-6


# ------------------------------------------------------------------------------------------ ATen operators
def _round(K, S, N, seed, nan_outsider=False):
    g = torch.Generator().manual_seed(seed)
    xs = [torch.randn(N, generator=g) for _ in range(K)]
    n = torch.randint(1, 5000, (K,), generator=g, dtype=torch.int32)
    t = torch.tensor([seed % 5], dtype=torch.int64)
    m = sampling.mask(KEY, int(t), K, S)
    if nan_outsider and not m.all():
        xs[int(np.flatnonzero(~m)[0])][N // 2] = float("nan")
    return xs, n, t, m


@pytest.mark.parametrize("K,S,N", [(3, 1, 7), (5, 3, 1001), (8, 8, 513), (16, 5, 64)])
def test_torch_weighted_fedavg_matches_float64(K, S, N):
    xs, n, t, m = _round(K, S, N, K + S, nan_outsider=True)
    w64 = np.where(m, n.numpy() / n.numpy()[m].sum(), 0.0)
    want = sum(w64[k] * xs[k].double().numpy() for k in range(K) if m[k])
    coll = TorchCollective(Topology.single_process(K, CPU))
    z = torch.randn(N)
    z0 = z.clone()
    dual = coll.fedavg_(xs, z, sample=SampleRound(S, KEY, t, n))
    np.testing.assert_allclose(z.numpy(), want, rtol=1e-5, atol=1e-6)
    assert torch.isfinite(z).all() and all(torch.equal(x, z) for x in xs)        # the NaN outsider was not read
    assert float(dual) == pytest.approx(float(((z0 - z).double() ** 2).sum()), rel=1e-5)
    assert int(t) == (K + S) % 5 + 1


@pytest.mark.parametrize("kind", ["avgm", "adam"])
def test_torch_weighted_fedopt_matches_float64(kind):
    K, S, N = 6, 4, 777
    xs, n, t, m = _round(K, S, N, 11, nan_outsider=True)
    w64 = np.where(m, n.numpy() / n.numpy()[m].sum(), 0.0)
    mean = sum(w64[k] * xs[k].double().numpy() for k in range(K) if m[k])
    coll = TorchCollective(Topology.single_process(K, CPU))
    z = torch.randn(N)
    mm, vv = torch.randn(N) * 1e-2, torch.rand(N) * 1e-3
    z64, m64, v64 = z.double().numpy(), mm.double().numpy(), vv.double().numpy()
    lr, b1, b2, tau = (1.0, 0.9, 0.99, 1e-3) if kind == "avgm" else (1e-2, 0.9, 0.99, 1e-3)
    d = mean - z64
    if kind == "avgm":
        m64 = b1 * m64 + d
        want = z64 + lr * m64
    else:
        m64 = b1 * m64 + (1 - b1) * d
        v64 = b2 * v64 + (1 - b2) * d * d
        want = z64 + lr * m64 / (np.sqrt(v64) + tau)
    coll.fedopt_(xs, z, mm, vv, kind, lr, b1, b2, tau, sample=SampleRound(S, KEY, t, n))
    np.testing.assert_allclose(z.numpy(), want, rtol=1e-4, atol=1e-6)
    np.testing.assert_allclose(mm.numpy(), m64, rtol=1e-4, atol=1e-7)
    if kind == "adam":
        np.testing.assert_allclose(vv.numpy(), v64, rtol=1e-4, atol=1e-10)
    assert all(torch.equal(x, z) for x in xs)


# ------------------------------------------------------------------------------------------ engine
def _run(**kw):
    lines = []
    eng = federated_multi.run(federated_multi.Config(**{**TINY, **kw}), log=lines.append)
    return eng, [l for l in lines if l.startswith("dual (")]


def test_engine_trains_only_participants(monkeypatch):
    checked = []
    orig_run, orig_agg = Engine._run_replicas, Engine._aggregate

    def run_replicas(self, visit, nloop, epoch, N):
        ids = self.strategy.round_participants()
        before = {}
        for rep, opt in zip(self.replicas, self.optimizers):
            ld = self.task.loader(rep.ck)
            before[rep.ck] = (rep.block(visit).clone(), ld.gen.get_state().clone(), ld.aug_counter, opt.t, opt.m.clone())
        imgs = self.images_seen
        orig_run(self, visit, nloop, epoch, N)
        for rep, opt in zip(self.replicas, self.optimizers):
            x, gen, aug, t, m = before[rep.ck]
            ld = self.task.loader(rep.ck)
            same = (torch.equal(rep.block(visit), x) and torch.equal(ld.gen.get_state(), gen) and ld.aug_counter == aug
                    and opt.t == t and torch.equal(opt.m, m))
            assert same == (rep.ck not in ids), (rep.ck, ids)
        assert self.images_seen - imgs == sum(min(len(self.task.shards[k]), 2 * 128) for k in ids)   # 2 minibatches each
        checked.append(list(ids))

    def aggregate(self, visit, nloop, nadmm, epoch, N):
        orig_agg(self, visit, nloop, nadmm, epoch, N)
        assert all(torch.equal(rep.block(visit), self.strategy.z) for rep in self.replicas)

    monkeypatch.setattr(Engine, "_run_replicas", run_replicas)
    monkeypatch.setattr(Engine, "_aggregate", aggregate)
    eng, trace = _run(**KW, clients_per_round=2, augment=True)
    assert len(trace) == len(checked) == 10 and all(len(ids) == 2 for ids in checked)
    assert eng.strategy.samp_rounds == int(eng.strategy.samp_t) == 10
    assert checked == [sampling.participants(eng.strategy.samp_key, t, 4, 2).tolist() for t in range(10)]


def test_metrics_rows_carry_participants_and_the_partition(tmp_path):
    path = str(tmp_path / "m.jsonl")
    eng, _ = _run(**KW, clients_per_round=3, partition="dirichlet", dirichlet_alpha=2.0, metrics_path=path)
    import json

    rows = [json.loads(l) for l in open(path)]
    part = [r for r in rows if r["kind"] == "partition"]
    assert len(part) == 1 and sum(part[0]["shard_sizes"]) == 1024
    assert [sum(h) for h in part[0]["class_histogram"]] == part[0]["shard_sizes"] == eng.task.shard_sizes()
    rounds = [r for r in rows if r["kind"] == "round"]
    assert len(rounds) == 10
    for t, r in enumerate(rounds):
        ids = sampling.participants(eng.strategy.samp_key, t, 4, 3).tolist()
        assert r["participants"] == ids
        assert r["participant_samples"] == sum(part[0]["shard_sizes"][k] for k in ids)


def test_defaults_build_todays_strategies():
    cfg = parse_config(FederatedConfig, [])
    assert (cfg.clients_per_round, cfg.partition) == (0, "iid")
    topo = Topology.single_process(4, CPU)
    for argv, typ in (([], FedAvg), (["--server_opt", "adam"], FedOpt), (["--clients_per_round", "4"], FedAvg)):
        s = federated_multi.make_strategy(parse_config(FederatedConfig, ["--K", "4"] + argv), TorchCollective(topo), topo)
        assert type(s) is typ and not s.sampled and "sample" not in s.state()
    s = federated_multi.make_strategy(parse_config(FederatedConfig, ["--K", "4", "--partition", "dirichlet"]),
                                      TorchCollective(topo), topo, [5, 6, 7, 8])
    assert s.sampled and s.samp_S == 4 and s.client_n == [5, 6, 7, 8]


# ------------------------------------------------------------------------------------------ resume
class _Killed(Exception):
    pass


def _killed_run(kw, kill_at):
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
def test_kill_and_resume_reproduces_the_run(tmp_path, server_opt):
    kw = dict(KW, K=4, Nadmm=3, clients_per_round=2, partition="dirichlet", dirichlet_alpha=2.0, server_opt=server_opt)
    eng, full = _run(**kw)
    assert len(full) == 15
    rec = str(tmp_path / "resume.pt")
    first = _killed_run(dict(kw, resume_out=rec), 30)
    assert 0 < len(first) < 15 and os.path.exists(rec)
    st = torch.load(rec, weights_only=False)["strategy_state"]
    assert st["samp_t"] == len(first) and st["sample"][0] == 2 and list(st["sample"][2]) == eng.task.shard_sizes()
    eng2, second = _run(**kw, resume=rec)
    assert first + second == full
    for r1, r2 in zip(eng.replicas, eng2.replicas):
        assert torch.equal(r1.arenas["net"].data, r2.arenas["net"].data)
    assert eng2.strategy.samp_rounds == eng.strategy.samp_rounds == 15
    assert eng2.images_seen == eng.images_seen
    with pytest.raises(ValueError, match="client-sampling settings"):
        _run(**{**kw, "clients_per_round": 3}, resume=rec)


# ------------------------------------------------------------------------------------------ configuration
@pytest.mark.parametrize("field,bad", [
    ("clients_per_round", dict(clients_per_round=-1)),
    ("clients_per_round", dict(K=4, clients_per_round=5)),
    ("aggregator", dict(K=8, clients_per_round=4, aggregator="median")),
    ("dp_clip", dict(K=8, clients_per_round=4, dp_clip=1e-3)),
    ("compress_bits", dict(K=8, clients_per_round=4, compress_bits=8)),
    ("aggregator", dict(K=8, partition="dirichlet", aggregator="trimmed_mean", trim_fraction=0.25)),
    ("dp_clip", dict(K=8, partition="dirichlet", dp_clip=1e-3)),
    ("compress_bits", dict(K=8, partition="dirichlet", compress_bits=4)),
    ("partition", dict(partition="shards")),
    ("dirichlet_alpha", dict(partition="dirichlet", dirichlet_alpha=0.0)),
])
def test_invalid_settings_raise(field, bad):
    with pytest.raises(ValueError, match=field):
        FederatedConfig(**bad)
    with pytest.raises(ValueError, match=field):
        parse_config(FederatedConfig, ["--%s=%s" % kv for kv in bad.items()])


def test_byzantine_workers_stay_allowed_with_sampling():
    cfg = FederatedConfig(K=8, clients_per_round=3, byzantine=2)
    assert cfg.byzantine == 2


def test_other_drivers_have_no_sampling_flag_and_unsupervised_ones_reject_dirichlet():
    with pytest.raises(SystemExit):
        parse_config(FedProxConfig, ["--clients_per_round", "2"])
    from federated_pytorch_test_b200.api import federated_cpc, federated_vae

    with pytest.raises(ValueError, match="partition"):
        federated_vae.run(VAEConfig(partition="dirichlet", use_cuda=False))
    with pytest.raises(ValueError, match="partition"):
        federated_cpc.run(CPCConfig(partition="dirichlet", use_cuda=False))


def test_fedprox_runs_on_dirichlet_shards():
    from federated_pytorch_test_b200.api import fedprox_multi

    eng = fedprox_multi.run(fedprox_multi.Config(**{**TINY, **KW, "Nadmm": 1}, partition="dirichlet", dirichlet_alpha=2.0),
                            log=lambda m: None)
    assert sum(eng.task.shard_sizes()) == 1024 and len(set(eng.task.shard_sizes())) > 1
