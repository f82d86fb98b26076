"""Compressed client updates (stochastic 8- / 4-bit codes, optional error feedback) on CPU: configuration, the numpy
oracle of the encoder, error feedback, the ATen operators, and ``federated_multi`` end to end (finite runs, the NaN guard,
true resume, two gloo processes == one process)."""
import math
import os

import numpy as np
import pytest
import torch

from federated_pytorch_test_b200.algo import compress
from federated_pytorch_test_b200.algo.strategies import FedAvg, FedOpt
from federated_pytorch_test_b200.api import federated_multi
from federated_pytorch_test_b200.config import FederatedConfig, FedProxConfig, parse_config
from federated_pytorch_test_b200.parallel import Topology, TorchCollective

TINY = dict(train_size=1024, test_size=128, save_model=False, graphs=False, fast=False)
KW = dict(K=4, Nloop=1, Nadmm=2, max_minibatches=2, check_results=False, use_cuda=False, model="Net")
KEY = compress.compress_key(69)


# ------------------------------------------------------------------------------------------ configuration
def test_defaults_are_off_and_build_todays_strategies():
    cfg = parse_config(FederatedConfig, [])
    assert (cfg.compress_bits, cfg.compress_ef) == (0, False)
    topo = Topology.single_process(4, torch.device("cpu"))
    s = federated_multi.make_strategy(cfg, TorchCollective(topo), topo)
    assert type(s) is FedAvg and not s.q_bits and s.state().keys() == {"z"}
    cfg = parse_config(FederatedConfig, ["--server_opt", "adam", "--compress_bits", "0"])
    s = federated_multi.make_strategy(cfg, TorchCollective(topo), topo)
    assert type(s) is FedOpt and not s.q_bits and "compress" not in s.state()
    cfg = parse_config(FederatedConfig, ["--compress_bits", "4", "--compress_ef", "--server_opt", "adam"])
    s = federated_multi.make_strategy(cfg, TorchCollective(topo), topo)
    assert type(s) is FedOpt and (s.q_bits, s.q_ef_on) == (4, True)


@pytest.mark.parametrize("field,bad", [
    ("compress_bits", dict(compress_bits=2)),
    ("compress_bits", dict(compress_bits=16)),
    ("compress_bits", dict(compress_bits=-8)),
    ("compress_ef", dict(compress_ef=True)),
    ("dp_clip", dict(compress_bits=8, dp_clip=1e-3)),
    ("aggregator", dict(compress_bits=8, aggregator="median")),
    ("aggregator", dict(compress_bits=4, aggregator="trimmed_mean", trim_fraction=0.25)),
])
def test_invalid_settings_raise(field, bad):
    with pytest.raises(ValueError, match=field):
        FederatedConfig(**bad)
    with pytest.raises(ValueError, match=field):
        parse_config(FederatedConfig, ["--%s=%s" % kv for kv in bad.items()])


def test_other_drivers_have_no_compression_flags():
    for flag in ("--compress_bits", "--compress_ef"):
        with pytest.raises(SystemExit):
            parse_config(FedProxConfig, [flag, "8"])


# ------------------------------------------------------------------------------------------ the oracle
def _update(n, seed, scale=1.0):
    g = np.random.default_rng(seed)
    return (g.standard_normal(n) * scale * np.exp(g.standard_normal(n))).astype(np.float32)


@pytest.mark.parametrize("bits", [8, 4])
@pytest.mark.parametrize("n", [1, 127, 128, 129, 1000, 5130])
def test_codes_are_in_range_and_within_one_step(bits, n):
    L = compress.levels(bits)
    u = _update(n, n + bits)
    codes, scales = compress.quantize(u, bits, KEY, 3, 7)
    assert codes.dtype == np.int8 and codes.shape == (n,) and scales.shape == (-(-n // 128),)
    assert codes.min() >= -L and codes.max() <= L
    s = np.repeat(scales, 128)[:n]
    for g in range(scales.size):                          # s = max|u| / L, correctly rounded in float32
        grp = u[128 * g: 128 * (g + 1)]
        assert scales[g] == np.float32(np.abs(grp).max()) / np.float32(L)
    deq = compress.dequantize(codes, scales)
    assert np.all(np.abs(deq.astype(np.float64) - u) <= s.astype(np.float64) * (1 + 1e-6))
    assert compress.payload_bytes(n, bits) == -(-n * bits // 8) + 4 * scales.size


def test_zero_update_gives_zero_codes():
    for bits in (8, 4):
        u = np.zeros(1000, dtype=np.float32)
        u[300:400] = _update(100, 1)                       # groups 2 and 3 partly non-zero, the rest exactly zero
        codes, scales = compress.quantize(u, bits, KEY, 0, 0)
        assert scales[0] == scales[1] == scales[4] == 0.0 and np.all(codes[:256] == 0) and np.all(codes[512:] == 0)
        assert np.all(codes[u == 0] == 0)                  # a zero coordinate codes to 0 in a non-zero group too


@pytest.mark.parametrize("bad", [float("nan"), float("inf"), -float("inf")])
def test_nonfinite_value_makes_its_group_scale_nonfinite(bad):
    for bits in (8, 4):
        u = _update(700, 5)
        u[130] = bad
        codes, scales = compress.quantize(u, bits, KEY, 2, 1)
        assert not math.isfinite(scales[1]) and np.all(np.isfinite(np.delete(scales, 1)))
        assert np.all(codes[128:256] == 0)
        deq = compress.dequantize(codes, scales)
        assert np.all(np.isnan(deq[128:256])) and np.all(np.isfinite(deq[:128])) and np.all(np.isfinite(deq[256:]))


@pytest.mark.parametrize("bits", [8, 4])
def test_rounding_is_unbiased(bits):
    """Averaged over T rounds, q s converges to u.  Per coordinate q s - u has mean 0 and |q s - u| <= s, so the mean
    over T independent rounds has standard deviation at most s / (2 sqrt(T)); 6 of those bound every coordinate's mean
    error (a false failure has probability below 1e-8 per coordinate)."""
    n, T = 4096, 2000
    u = _update(n, 11)
    acc = np.zeros(n)
    for t in range(T):
        codes, scales = compress.quantize(u, bits, KEY, 1, t)
        acc += compress.dequantize(codes, scales)
    s = np.repeat(compress.quantize(u, bits, KEY, 1, 0)[1], 128)[:n].astype(np.float64)
    assert np.all(np.abs(acc / T - u) <= 6 * s / (2 * math.sqrt(T)))
    assert np.abs(acc / T - u).mean() < 0.02 * s.mean()


def _u_scalar(key, k, t, i):
    """U_i of worker k in round t from the documented formula, one coordinate at a time with Python integers."""
    M = (1 << 64) - 1

    def F(z):
        z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M
        z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M
        return z ^ (z >> 31)
    G = 0x9E3779B97F4A7C15
    w = F((F((F((key + (t + 1) * G) & M) + (k + 1) * G) & M) + (i // 2 + 1) * G) & M)
    return ((w & 0xFFFFFF) if i % 2 else (w >> 40)) * 2.0 ** -24


def test_draw_is_a_function_of_key_worker_round_and_coordinate_only():
    full = compress.uniforms(KEY, 5, 9, 100_001)
    assert full.dtype == np.float32 and full.min() >= 0.0 and full.max() < 1.0
    for i in (0, 1, 2, 127, 128, 4097, 50_000, 100_000):
        assert full[i] == _u_scalar(KEY, 5, 9, i)
    assert np.array_equal(compress.uniforms(KEY, 5, 9, 333), full[:333])
    assert not np.array_equal(compress.uniforms(KEY, 6, 9, 1000), full[:1000])
    assert not np.array_equal(compress.uniforms(KEY, 5, 10, 1000), full[:1000])
    assert not np.array_equal(compress.uniforms(compress.compress_key(70), 5, 9, 1000), full[:1000])
    assert abs(full.mean() - 0.5) < 3e-3
    u = _update(1000, 3)
    a = compress.quantize(u, 8, KEY, 5, 9)
    b = compress.quantize(u, 8, KEY, 5, 9)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


def test_pack4_roundtrip():
    codes = np.arange(-7, 8, dtype=np.int8).repeat(3)
    packed = compress.pack4(codes)
    assert packed.size == -(-codes.size // 2) and packed[0] == (np.uint8(-7 & 0xF) | np.uint8((-7 & 0xF) << 4))
    assert np.array_equal(compress.unpack4(packed, codes.size), codes)


@pytest.mark.parametrize("bits", [8, 4])
def test_error_feedback_telescopes(bits):
    """For a fixed update sequence, sum_t q_t s_t + e_T == sum_t u_t (float32 tolerance)."""
    n, T = 3000, 50
    e = np.zeros(n, dtype=np.float32)
    sent = np.zeros(n, dtype=np.float64)
    total = np.zeros(n, dtype=np.float64)
    for t in range(T):
        g = _update(n, 100 + t, 0.01)
        total += g
        u = g + e
        codes, scales = compress.quantize(u, bits, KEY, 0, t)
        deq = compress.dequantize(codes, scales)
        e = u - deq
        sent += deq
    np.testing.assert_allclose(sent + e, total, rtol=0, atol=1e-6 * T)
    assert np.abs(e).max() < np.abs(total).max()


# ------------------------------------------------------------------------------------------ the ATen operators
@pytest.mark.parametrize("K", [1, 3, 4])
@pytest.mark.parametrize("kind", [None, "avgm", "adam"])
@pytest.mark.parametrize("bits,ef", [(8, False), (4, True)])
def test_round_matches_numpy_transcription(K, kind, bits, ef):
    N = 517
    topo = Topology.single_process(K, torch.device("cpu"))
    coll = TorchCollective(topo)
    kw = dict(compress_bits=bits, compress_ef=ef, seed=4)
    strat = FedAvg(coll, topo, **kw) if kind is None else FedOpt(coll, topo, kind, lr=0.05, momentum=0.5, beta1=0.8,
                                                                 beta2=0.9, tau=1e-2, **kw)
    g = torch.Generator().manual_seed(K)
    z0 = torch.randn(N, generator=g)
    xs = [z0.clone() for _ in range(K)]
    strat.begin_block(0, N, xs)
    assert torch.equal(strat.z, z0)
    z = z0.numpy().copy()
    e = [np.zeros(N, dtype=np.float32) for _ in range(K)]
    m, v = np.zeros(N, dtype=np.float32), np.full(N, 1e-4, dtype=np.float32)
    for r in range(3):
        for x in xs:
            x.add_(torch.randn(N, generator=g) * 0.01)
        acc = np.zeros(N, dtype=np.float32)
        err = nrm = 0.0
        for k, x in enumerate(xs):
            u = x.numpy() - z + (e[k] if ef else np.float32(0))
            codes, scales = compress.quantize(u, bits, strat.q_key, k, r)
            deq = compress.dequantize(codes, scales)
            e[k] = u - deq
            err += float(np.sum(e[k].astype(np.float64) ** 2))
            nrm += float(np.sum(u.astype(np.float64) ** 2))
            acc = acc + deq
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
        met = strat.aggregate(r)
        assert met["q_bits"] == bits and met["q_bytes"] == compress.payload_bytes(N, bits)
        assert met["q_rel_err"] == pytest.approx(math.sqrt(err / nrm), rel=1e-6)
        np.testing.assert_allclose(strat.z.numpy(), znew, rtol=1e-6, atol=1e-7)
        assert all(torch.equal(x, strat.z) for x in xs)
        if ef:
            for k in range(K):
                np.testing.assert_array_equal(strat.q_ef[0][k].numpy(), e[k])
        z = strat.z.numpy().copy()
    assert int(strat.q_t) == strat.q_rounds == 3


def test_payload_buffers_hold_the_codes():
    K, N = 2, 300
    topo = Topology.single_process(K, torch.device("cpu"))
    for bits in (8, 4):
        strat = FedAvg(TorchCollective(topo), topo, compress_bits=bits, seed=1)
        z0 = torch.zeros(N)
        xs = [z0.clone() for _ in range(K)]
        strat.begin_block(0, N, xs)
        us = [torch.randn(N) for _ in range(K)]
        for x, u in zip(xs, us):
            x.copy_(u)
        strat.aggregate(0)
        for k in range(K):
            codes, scales = compress.quantize(us[k].numpy(), bits, strat.q_key, k, 0)
            raw = strat.q_payload[k][0].numpy()
            got = raw[:N].view(np.int8) if bits == 8 else compress.unpack4(raw, N)
            assert np.array_equal(got, codes) and np.array_equal(strat.q_payload[k][1].numpy(), scales)


# ------------------------------------------------------------------------------------------ end to end
def _run(**kw):
    lines = []
    eng = federated_multi.run(federated_multi.Config(**{**TINY, **kw}), log=lines.append)
    return eng, [l for l in lines if l.startswith("dual (")]


def _val(line):
    return float(line.rsplit("=", 1)[1])


@pytest.mark.parametrize("bits,ef", [(8, False), (4, True)])
def test_cpu_runs_finish_with_finite_metrics(bits, ef):
    eng, trace = _run(**KW, compress_bits=bits, compress_ef=ef)
    assert len(trace) == 10 and all(math.isfinite(_val(l)) and _val(l) > 0 for l in trace)
    assert eng.strategy.q_rounds == int(eng.strategy.q_t) == 10
    arena = eng.replicas[0].arenas["net"]
    assert torch.isfinite(arena.data).all()
    for rep in eng.replicas[1:]:
        assert torch.equal(rep.arenas["net"].data, arena.data)
    pad = torch.ones(arena.total, dtype=torch.bool)      # the alignment padding stays zero: a zero update codes to 0
    for off, n in zip(arena.offsets, arena.numels):
        pad[off:off + n] = False
    assert pad.any() and torch.equal(arena.data[pad], torch.zeros(int(pad.sum())))
    if ef:
        for efs in eng.strategy.q_ef.values():
            for e in efs:
                assert torch.isfinite(e).all()


def test_nan_attacker_trips_the_guard():
    with pytest.raises(FloatingPointError, match="non-finite"):
        _run(**{**KW, "Nadmm": 1, "max_minibatches": 1}, compress_bits=8, byzantine=1, attack="nan")


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
    kw = dict(KW, K=3, Nadmm=3, compress_bits=4, compress_ef=True, server_opt=server_opt)
    eng, full = _run(**kw)
    assert len(full) == 15
    rec = str(tmp_path / "resume.pt")
    first = _killed_run(dict(kw, resume_out=rec), 27)
    assert 0 < len(first) < 15 and os.path.exists(rec)
    st = torch.load(rec, weights_only=False)["strategy_state"]
    assert st["q_t"] == len(first) and st["compress"][:2] == (4, True) and len(st["q_ef"]) >= 1
    eng2, second = _run(**kw, resume=rec)
    assert first + second == full
    assert torch.equal(eng.replicas[0].arenas["net"].data, eng2.replicas[0].arenas["net"].data)
    ef1, ef2 = eng.strategy.state()["q_ef"], eng2.strategy.state()["q_ef"]    # (blocks not revisited keep the record's)
    assert ef1.keys() == ef2.keys() and all(torch.equal(ef1[ci].cpu(), ef2[ci].cpu()) for ci in ef1)
    with pytest.raises(ValueError, match="compression settings"):
        _run(**{**kw, "compress_bits": 8}, resume=rec)
    with pytest.raises(ValueError, match="compression settings"):
        _run(**{**kw, "compress_ef": False}, resume=rec)


def _dist_worker(rank, world, port, out):
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch.distributed as dist
    lines = []
    eng = federated_multi.run(federated_multi.Config(**DIST_KW, **TINY), log=lines.append)
    if rank == 0:
        torch.save({"lines": lines, "flat": eng.replicas[0].arenas["net"].data.clone()}, out)
    dist.destroy_process_group()


DIST_KW = dict(KW, K=4, compress_bits=8, compress_ef=True)


def test_two_process_gloo_equals_single_process(tmp_path):
    """The codes depend on (seed, worker, round, coordinate) only and the dequantized updates are summed in worker order,
    so the process layout does not change the result at all."""
    import torch.multiprocessing as mp
    out = str(tmp_path / "r0.pt")
    port = 38600 + (os.getpid() % 2000)
    mp.spawn(_dist_worker, args=(2, port, out), nprocs=2, join=True)
    got = torch.load(out, weights_only=False)
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        os.environ.pop(k, None)
    eng, single = _run(**DIST_KW)
    multi = [l for l in got["lines"] if l.startswith("dual (")]
    assert len(single) == len(multi) == 10
    assert single == multi
    assert torch.equal(got["flat"], eng.replicas[0].arenas["net"].data)
