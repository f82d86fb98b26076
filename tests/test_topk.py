"""Top-k sparsified client updates (optional error feedback) on CPU: configuration, the numpy oracle of the selection and
its payload, error feedback, the ATen operators, and ``federated_multi`` end to end (finite runs, the NaN guard, true
resume, two gloo processes == one process)."""
import math
import os

import numpy as np
import pytest
import torch

from federated_pytorch_test_b200.algo import compress
from federated_pytorch_test_b200.algo.strategies import FedAvg, FedOpt
from federated_pytorch_test_b200.api import federated_multi
from federated_pytorch_test_b200.config import (ConsensusConfig, FederatedConfig, FedProxConfig, VAEConfig,
                                                parse_config)
from federated_pytorch_test_b200.parallel import Topology, TorchCollective

TINY = dict(train_size=1024, test_size=128, save_model=False, graphs=False, fast=False)
KW = dict(K=4, Nloop=1, Nadmm=2, max_minibatches=2, check_results=False, use_cuda=False, model="Net")


# ------------------------------------------------------------------------------------------ configuration
def test_defaults_are_off_and_build_todays_strategies():
    cfg = parse_config(FederatedConfig, [])
    assert cfg.compress_topk == 0.0
    topo = Topology.single_process(4, torch.device("cpu"))
    s = federated_multi.make_strategy(cfg, TorchCollective(topo), topo)
    assert type(s) is FedAvg and not s.topk_r and s.state().keys() == {"z"}
    cfg = parse_config(FederatedConfig, ["--compress_topk", "0.01", "--compress_ef", "--server_opt", "adam"])
    s = federated_multi.make_strategy(cfg, TorchCollective(topo), topo)
    assert type(s) is FedOpt and (s.topk_r, s.q_ef_on, s.q_bits) == (0.01, True, 0)


@pytest.mark.parametrize("field,bad", [
    ("compress_topk", dict(compress_topk=1.0)),
    ("compress_topk", dict(compress_topk=-0.1)),
    ("compress_topk", dict(compress_topk=2.5)),
    ("compress_topk", dict(compress_topk=float("nan"))),
    ("compress_bits", dict(compress_topk=0.1, compress_bits=8)),
    ("compress_ef", dict(compress_ef=True)),
    ("dp_clip", dict(compress_topk=0.1, dp_clip=1e-3)),
    ("aggregator", dict(compress_topk=0.1, aggregator="median")),
    ("compress_topk", dict(compress_topk=0.1, K=8, clients_per_round=4)),
    ("compress_topk", dict(compress_topk=0.1, partition="dirichlet")),
    ("compress_topk", dict(compress_topk=0.1, secagg=True)),
    ("compress_topk", dict(compress_topk=0.1, scaffold=True, optimizer="sgd")),
])
def test_invalid_settings_raise(field, bad):
    with pytest.raises(ValueError, match=field):
        FederatedConfig(**bad)
    with pytest.raises(ValueError, match=field):
        parse_config(FederatedConfig, ["--%s=%s" % kv for kv in bad.items()])


def test_strategy_rejects_combinations():
    topo = Topology.single_process(4, torch.device("cpu"))
    coll = TorchCollective(topo)
    with pytest.raises(ValueError, match="compress_topk"):
        FedAvg(coll, topo, compress_topk=0.1, secagg=True)
    with pytest.raises(ValueError, match="compress_topk"):
        FedOpt(coll, topo, "adam", compress_topk=0.1, scaffold=True)
    with pytest.raises(ValueError, match="compress_topk"):
        FedAvg(coll, topo, compress_topk=0.1, client_n=[1, 2, 3, 4])


def test_other_drivers_have_no_topk_flag():
    for cls in (FedProxConfig, ConsensusConfig, VAEConfig):
        with pytest.raises(SystemExit):
            parse_config(cls, ["--compress_topk", "0.01"])


# ------------------------------------------------------------------------------------------ the oracle
def _update(n, seed, scale=1.0):
    g = np.random.default_rng(seed)
    return (g.standard_normal(n) * scale * np.exp(g.standard_normal(n))).astype(np.float32)


def _brute(u, k):
    key = compress.topk_keys(u).astype(np.int64)
    return np.sort(np.lexsort((np.arange(u.size), -key))[:k])


def _check_payload(pay, u, k):
    offsets, idx, vals = pay
    n = u.size
    T = -(-n // 8192)
    assert offsets.dtype == np.uint32 and idx.dtype == np.uint16 and vals.dtype == np.float32
    assert offsets.shape == (T + 1,) and idx.shape == vals.shape == (k,)
    assert offsets[0] == 0 and offsets[-1] == k and np.all(np.diff(offsets.astype(np.int64)) >= 0)
    sel = compress.topk_indices(offsets, idx)
    assert np.all(np.diff(sel) > 0) and sel.max() < n                # ascending, inside their tiles
    counts = np.bincount(sel // 8192, minlength=T)
    np.testing.assert_array_equal(np.diff(offsets.astype(np.int64)), counts)   # the offsets are a prefix sum
    assert np.array_equal(vals.view(np.uint32), u[sel].view(np.uint32))
    assert compress.topk_payload_bytes(n, k) == 4 * offsets.size + 2 * idx.size + 4 * vals.size
    return sel


@pytest.mark.parametrize("n", [1, 8191, 8192, 8193, 100_003])
@pytest.mark.parametrize("r", [0.001, 0.01, 0.3])
def test_selection_equals_brute_force(n, r):
    u = _update(n, n)
    k = compress.topk_count(n, r)
    assert k == max(1, math.ceil(r * n))
    sel = _check_payload(compress.topk_select(u, k), u, k)
    np.testing.assert_array_equal(sel, _brute(u, k))
    assert np.abs(u[sel]).min() >= np.abs(np.delete(u, sel)).max(initial=0.0)
    pay = compress.topk_select(u, k)
    unpacked = compress.topk_unpack(compress.topk_pack(pay, n), n, k)
    assert all(np.array_equal(a.view(np.uint8), b.view(np.uint8)) for a, b in zip(pay, unpacked))
    assert compress.topk_pack(pay, n).size == compress.topk_layout(n, k)[3] <= 2 * (-(-n // 32) * 32)


def test_ties_and_zero_updates_select_the_lowest_indices():
    n = 20_000
    for u in (np.zeros(n, dtype=np.float32), np.full(n, -0.5, dtype=np.float32),
              np.where(np.arange(n) % 2 == 0, 0.25, -0.25).astype(np.float32)):
        for k in (1, 7, 8192, 9000):
            sel = _check_payload(compress.topk_select(u, k), u, k)
            np.testing.assert_array_equal(sel, np.arange(k))
    u = np.zeros(n, dtype=np.float32)
    u[[5, 17000, 9000]] = [1.0, -1.0, 1.0]
    u[3] = -0.0
    sel = _check_payload(compress.topk_select(u, 5), u, 5)
    np.testing.assert_array_equal(sel, [0, 1, 5, 9000, 17000])


@pytest.mark.parametrize("bad", [float("nan"), float("inf"), -float("inf")])
def test_nonfinite_values_are_always_selected(bad):
    u = _update(30_000, 3, scale=1e30)
    u[[7, 12_345, 29_999]] = bad
    sel = _check_payload(compress.topk_select(u, 3), u, 3)
    np.testing.assert_array_equal(sel, [7, 12_345, 29_999])
    u[100] = float("nan")
    sel = compress.topk_indices(*compress.topk_select(u, 1)[:2])
    assert list(sel) == [100 if not math.isnan(bad) else 7]


def test_error_feedback_telescopes():
    """For a fixed update sequence, sum_t s_t + e_T == sum_t g_t (float32 tolerance), and e is 0 where selected."""
    n, T, k = 3000, 50, 30
    e = np.zeros(n, dtype=np.float32)
    sent = np.zeros(n, dtype=np.float64)
    total = np.zeros(n, dtype=np.float64)
    for t in range(T):
        g = _update(n, 100 + t, 0.01)
        total += g
        u = g + e
        pay = compress.topk_select(u, k)
        sel = compress.topk_indices(*pay[:2])
        s = np.zeros(n, dtype=np.float32)
        s[sel] = pay[2]
        e = u - s
        assert np.all(e[sel] == 0.0)
        sent += s
    np.testing.assert_allclose(sent + e, total, rtol=0, atol=1e-6 * T)


# ------------------------------------------------------------------------------------------ the ATen operators
@pytest.mark.parametrize("K", [1, 3, 4])
@pytest.mark.parametrize("kind", [None, "avgm", "adam"])
@pytest.mark.parametrize("ef", [False, True])
def test_round_matches_numpy_transcription(K, kind, ef):
    N, r = 9000, 0.05
    topo = Topology.single_process(K, torch.device("cpu"))
    coll = TorchCollective(topo)
    kw = dict(compress_topk=r, compress_ef=ef)
    strat = FedAvg(coll, topo, **kw) if kind is None else FedOpt(coll, topo, kind, lr=0.05, momentum=0.5, beta1=0.8,
                                                                 beta2=0.9, tau=1e-2, **kw)
    g = torch.Generator().manual_seed(K)
    z0 = torch.randn(N, generator=g)
    xs = [z0.clone() for _ in range(K)]
    strat.begin_block(0, N, xs)
    assert torch.equal(strat.z, z0) and strat.topk_k == math.ceil(r * N)
    k_sel = strat.topk_k
    z = z0.numpy().copy()
    e = [np.zeros(N, dtype=np.float32) for _ in range(K)]
    m, v = np.zeros(N, dtype=np.float32), np.full(N, 1e-4, dtype=np.float32)
    for rnd in range(3):
        for x in xs:
            x.add_(torch.randn(N, generator=g) * 0.01)
        acc = np.zeros(N, dtype=np.float32)
        err = nrm = 0.0
        pays = []
        for k, x in enumerate(xs):
            u = x.numpy() - z + (e[k] if ef else np.float32(0))
            pay = compress.topk_select(u, k_sel)
            pays.append(pay)
            s = np.zeros(N, dtype=np.float32)
            s[compress.topk_indices(*pay[:2])] = pay[2]
            if ef:
                e[k] = u - s
            err += float(np.sum((u - s).astype(np.float64) ** 2))
            nrm += float(np.sum(u.astype(np.float64) ** 2))
            acc = acc + s
        d = acc * np.float32(1.0 / K)
        if kind is None:
            znew = z + d
        elif kind == "avgm":
            m = np.float32(0.5) * m + d
            znew = z + np.float32(0.05) * m
        else:
            m = np.float32(0.8) * m + np.float32(0.2) * d
            v = np.float32(0.9) * v + np.float32(0.1) * d * d
            znew = z + np.float32(0.05) * m / (np.sqrt(v) + np.float32(1e-2))
        met = strat.aggregate(rnd)
        assert met["topk_k"] == k_sel and met["q_bytes"] == compress.topk_payload_bytes(N, k_sel)
        assert met["q_rel_err"] == pytest.approx(math.sqrt(err / nrm), rel=1e-6)
        np.testing.assert_allclose(strat.z.numpy(), znew, rtol=1e-6, atol=1e-7)
        if kind is not None:
            np.testing.assert_allclose(strat.m.numpy(), m, rtol=1e-6, atol=1e-8)
            if kind == "adam":
                np.testing.assert_allclose(strat.v.numpy(), v, rtol=1e-6, atol=1e-10)
        assert all(torch.equal(x, strat.z) for x in xs)
        for k in range(K):
            got = compress.topk_unpack(strat.topk_payload[k].numpy(), N, k_sel)
            assert all(np.array_equal(a.view(np.uint8), b.view(np.uint8)) for a, b in zip(got, pays[k]))
            if ef:
                np.testing.assert_array_equal(strat.q_ef[0][k].numpy(), e[k])
        z = strat.z.numpy().copy()


# ------------------------------------------------------------------------------------------ end to end
def _run(**kw):
    lines = []
    eng = federated_multi.run(federated_multi.Config(**{**TINY, **kw}), log=lines.append)
    return eng, [l for l in lines if l.startswith("dual (")]


def _val(line):
    return float(line.rsplit("=", 1)[1])


@pytest.mark.parametrize("r,ef,server_opt", [(0.01, False, "none"), (0.1, True, "none"), (0.05, True, "adam")])
def test_cpu_runs_finish_with_finite_metrics(r, ef, server_opt):
    eng, trace = _run(**KW, compress_topk=r, compress_ef=ef, server_opt=server_opt)
    assert len(trace) == 10 and all(math.isfinite(_val(l)) for l in trace)
    arena = eng.replicas[0].arenas["net"]
    assert torch.isfinite(arena.data).all()
    for rep in eng.replicas[1:]:
        assert torch.equal(rep.arenas["net"].data, arena.data)
    if ef:
        for efs in eng.strategy.q_ef.values():
            for e in efs:
                assert torch.isfinite(e).all()


def test_nan_attacker_trips_the_guard():
    with pytest.raises(FloatingPointError, match="non-finite"):
        _run(**{**KW, "Nadmm": 1, "max_minibatches": 1}, compress_topk=0.01, byzantine=1, attack="nan")


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
def test_kill_and_resume_with_error_feedback_reproduces_the_run(tmp_path, server_opt):
    kw = dict(KW, K=3, Nadmm=3, compress_topk=0.02, compress_ef=True, server_opt=server_opt)
    eng, full = _run(**kw)
    assert len(full) == 15
    rec = str(tmp_path / "resume.pt")
    first = _killed_run(dict(kw, resume_out=rec), 27)
    assert 0 < len(first) < 15 and os.path.exists(rec)
    st = torch.load(rec, weights_only=False)["strategy_state"]
    assert st["topk"] == (0.02, True) and len(st["q_ef"]) >= 1 and "compress" not in st
    eng2, second = _run(**kw, resume=rec)
    assert first + second == full
    assert torch.equal(eng.replicas[0].arenas["net"].data, eng2.replicas[0].arenas["net"].data)
    ef1, ef2 = eng.strategy.state()["q_ef"], eng2.strategy.state()["q_ef"]
    assert ef1.keys() == ef2.keys() and all(torch.equal(ef1[ci].cpu(), ef2[ci].cpu()) for ci in ef1)
    for other in ({"compress_topk": 0.05}, {"compress_ef": False}, {"compress_topk": 0.0, "compress_ef": False},
                  {"compress_topk": 0.0, "compress_bits": 8}):
        with pytest.raises(ValueError, match="(top-k|compression) settings"):
            _run(**{**kw, **other}, resume=rec)


def test_records_without_topk_resume_with_topk_off(tmp_path):
    kw = dict(KW, K=2, Nadmm=2)
    rec = str(tmp_path / "plain.pt")
    _killed_run(dict(kw, resume_out=rec), 5)
    assert "topk" not in torch.load(rec, weights_only=False)["strategy_state"]
    _run(**kw, resume=rec)
    with pytest.raises(ValueError, match="top-k settings"):
        _run(**kw, compress_topk=0.1, resume=rec)


def _dist_worker(rank, world, port, out):
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch.distributed as dist
    lines = []
    eng = federated_multi.run(federated_multi.Config(**DIST_KW, **TINY), log=lines.append)
    if rank == 0:
        torch.save({"lines": lines, "flat": eng.replicas[0].arenas["net"].data.clone()}, out)
    dist.destroy_process_group()


DIST_KW = dict(KW, K=4, compress_topk=0.03, compress_ef=True)


def test_two_process_gloo_equals_single_process(tmp_path):
    """The selection depends on each worker's update only and the sparse updates are summed in worker order, so the
    process layout does not change the result at all."""
    import torch.multiprocessing as mp
    out = str(tmp_path / "r0.pt")
    port = 40600 + (os.getpid() % 2000)
    mp.spawn(_dist_worker, args=(2, port, out), nprocs=2, join=True)
    got = torch.load(out, weights_only=False)
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        os.environ.pop(k, None)
    eng, single = _run(**DIST_KW)
    multi = [l for l in got["lines"] if l.startswith("dual (")]
    assert len(single) == len(multi) == 10
    assert single == multi
    assert torch.equal(got["flat"], eng.replicas[0].arenas["net"].data)
