"""Secure aggregation (pairwise ChaCha20-masked fixed-point updates) on CPU: configuration, the numpy oracle (RFC 8439
ChaCha20, the fixed-point scale, encoding, mask cancellation, decoding), the ATen operators, and ``federated_multi`` end
to end (finite runs, the NaN guard, true resume of the nonce sequence, two gloo processes == one process bit for bit)."""
import math
import os

import numpy as np
import pytest
import torch

from federated_pytorch_test_b200.algo import secagg
from federated_pytorch_test_b200.algo.strategies import FedAvg, FedOpt
from federated_pytorch_test_b200.api import federated_multi
from federated_pytorch_test_b200.config import ConsensusConfig, FederatedConfig, FedProxConfig, parse_config
from federated_pytorch_test_b200.parallel import Topology, TorchCollective

TINY = dict(train_size=1024, test_size=128, save_model=False, graphs=False, fast=False)
KW = dict(K=4, Nloop=1, Nadmm=2, max_minibatches=2, check_results=False, use_cuda=False, model="Net")
RFC_KEY = np.frombuffer(bytes(range(32)), dtype="<u4")
RFC_T = 0x4A00000009000000                 # nonce bytes 00 00 00 09 00 00 00 4a 00 00 00 00 as (t mod 2^32, t div 2^32, 0)
RFC_BLOCK1 = [0xE4E7F110, 0x15593BD1, 0x1FDD0F50, 0xC47120A3, 0xC7F4D1C7, 0x0368C033, 0x9AAA2204, 0x4E6CD4C3,
              0x466482D2, 0x09AA9F07, 0x05D7C214, 0xA2028BD9, 0xD19C12B5, 0xB94E16DE, 0xE883D0CB, 0x4E3C50A2]


# ------------------------------------------------------------------------------------------ configuration
def test_defaults_are_off_and_build_todays_strategies():
    cfg = parse_config(FederatedConfig, [])
    assert (cfg.secagg, cfg.secagg_clip) == (False, 1.0)
    topo = Topology.single_process(4, torch.device("cpu"))
    s = federated_multi.make_strategy(cfg, TorchCollective(topo), topo)
    assert type(s) is FedAvg and not s.sa and s.state().keys() == {"z"}
    cfg = parse_config(FederatedConfig, ["--server_opt", "adam"])
    s = federated_multi.make_strategy(cfg, TorchCollective(topo), topo)
    assert type(s) is FedOpt and not s.sa and "secagg" not in s.state()
    cfg = parse_config(FederatedConfig, ["--secagg", "--secagg_clip", "0.5", "--server_opt", "adam"])
    s = federated_multi.make_strategy(cfg, TorchCollective(topo), topo)
    assert type(s) is FedOpt and s.sa and (s.sa_clip, s.sa_f) == (0.5, secagg.frac_bits(0.5, 4))


@pytest.mark.parametrize("field,bad", [
    ("secagg_clip", dict(secagg_clip=0.0)),
    ("secagg_clip", dict(secagg_clip=-1.0)),
    ("secagg_clip", dict(secagg_clip=float("nan"))),
    ("secagg_clip", dict(secagg_clip=float("inf"))),
    ("secagg_clip", dict(secagg_clip=1e9)),            # f < 0: K rint(R) > 2^31 - 1
    ("secagg_clip", dict(secagg_clip=1e-38)),          # f > 126
    ("K", dict(K=1)),
    ("aggregator", dict(aggregator="median")),
    ("dp_clip", dict(dp_clip=1e-3)),
    ("compress_bits", dict(compress_bits=8)),
    ("clients_per_round", dict(clients_per_round=2)),
    ("dirichlet", dict(partition="dirichlet")),
])
def test_invalid_settings_raise(field, bad):
    kw = {"K": 4, "secagg": True, **bad}
    with pytest.raises(ValueError, match=field):
        FederatedConfig(**kw)
    with pytest.raises(ValueError, match=field):
        parse_config(FederatedConfig, ["--%s=%s" % kv for kv in kw.items()])


def test_other_drivers_have_no_secagg_flags():
    for cls in (FedProxConfig, ConsensusConfig):
        for argv in (["--secagg"], ["--secagg_clip", "1.0"]):
            with pytest.raises(SystemExit):
                parse_config(cls, argv)


# ------------------------------------------------------------------------------------------ the oracle
def test_chacha20_reproduces_rfc8439_block_vector():
    out = secagg.chacha20_blocks(RFC_KEY, [1], secagg.nonce(RFC_T))
    assert out.dtype == np.uint32 and out.tolist() == RFC_BLOCK1


def test_chacha20_matches_cryptography_over_many_blocks():
    algorithms = pytest.importorskip("cryptography.hazmat.primitives.ciphers.algorithms")
    from cryptography.hazmat.primitives.ciphers import Cipher

    key = secagg.pair_keys(3, 5)[7]
    for t in (0, 1, 2 ** 32 + 5):
        n0, n1, _ = secagg.nonce(t)
        nonce16 = np.array([0, n0, n1, 0], dtype="<u4").tobytes()        # 4-byte counter 0, then the 12-byte nonce
        ks = Cipher(algorithms.ChaCha20(key.astype("<u4").tobytes(), nonce16), mode=None).encryptor().update(bytes(64 * 1500))
        assert secagg.chacha20_blocks(key, np.arange(1500), secagg.nonce(t)).astype("<u4").tobytes() == ks


@pytest.mark.parametrize("K", [2, 3, 4, 8, 16, 64])
@pytest.mark.parametrize("clip", [1.0, 0.1, 3.7, 1e-3])
def test_scale_rule(K, clip):
    f = secagg.frac_bits(clip, K)
    R = float(np.float32(clip))
    assert K * round(R * 2.0 ** f) <= 2 ** 31 - 1 < K * round(R * 2.0 ** (f + 1))
    assert 0 <= f <= 126


def test_scale_rule_documented_values():
    assert secagg.frac_bits(1.0, 8) == 27 and secagg.frac_bits(1.0, 64) == 24


def test_encode_rounds_half_to_even_and_counts_exactly():
    f = 2                                                     # codes in quarters
    u = np.array([0.125, 0.375, -0.125, -0.375, 0.6, 2.0, -3.0, 1.0, np.nan, np.inf, -np.inf, 0.0], dtype=np.float32)
    q, clipped, nonfinite = secagg.encode(u, 1.0, f)
    assert q.dtype == np.int32
    assert q.tolist() == [0, 2, 0, -2, 2, 4, -4, 4, 0, 0, 0, 0]
    assert (clipped, nonfinite) == (2, 3)                     # |u| > R: 2.0, -3.0 (1.0 is not clipped)
    g = np.random.default_rng(0)
    u = (g.standard_normal(100_003) * 0.7).astype(np.float32)
    u[::97] = np.nan
    q, clipped, nonfinite = secagg.encode(u, 1.0, 27)
    fin = np.isfinite(u)
    assert nonfinite == int((~fin).sum()) and clipped == int((np.abs(u[fin]) > 1.0).sum())
    assert np.all(q[~fin] == 0) and np.abs(q).max() <= 2 ** 27


def _codes(K, n, f, seed):
    g = np.random.default_rng(seed)
    lim = round(2.0 ** f)
    return [g.integers(-lim, lim + 1, n).astype(np.int32) for _ in range(K)]


@pytest.mark.parametrize("K", [2, 3, 4, 8])
@pytest.mark.parametrize("n", [1, 17, 1001])
def test_masks_cancel(K, n):
    keys = secagg.pair_keys(11, K)
    f = secagg.frac_bits(1.0, K)
    q = _codes(K, n, f, K * n)
    for t in (0, 7, 2 ** 33 + 1):
        y = np.stack([secagg.payload(q[k], keys, K, k, t) for k in range(K)])
        assert np.array_equal(secagg.unmask_sum(y), np.sum(np.stack(q).astype(np.int64), axis=0).astype(np.int32))
        for k in range(K):                                    # a payload is not its codes
            assert not np.array_equal(y[k].view(np.int32), q[k]) or n == 0


def test_single_payload_top_byte_is_uniform():
    from scipy.stats import chisquare

    K, n = 4, 1 << 16
    keys = secagg.pair_keys(5, K)
    q = np.zeros(n, dtype=np.int32)                           # the most structured update there is
    y = secagg.payload(q, keys, K, 1, 3)
    counts = np.bincount((y >> np.uint32(24)).astype(np.int64), minlength=256)
    assert chisquare(counts).pvalue > 1e-4


def test_key_table_layout():
    K = 6
    keys = secagg.pair_keys(9, K)
    assert keys.shape == (15, 8) and keys.dtype == np.uint32 and len({r.tobytes() for r in keys}) == 15
    rows = [(i, j) for i in range(K) for j in range(i + 1, K)]
    assert [secagg.pair_row(i, j, K) for i, j in rows] == list(range(15))
    assert not np.array_equal(secagg.pair_keys(10, K), keys)


@pytest.mark.parametrize("K", [2, 3, 8])
def test_decoded_update_is_the_clamped_mean_within_half_a_step(K):
    n = 5000
    f = secagg.frac_bits(1.0, K)
    g = np.random.default_rng(K)
    us = [(g.standard_normal(n) * 0.5).astype(np.float32) for _ in range(K)]
    keys = secagg.pair_keys(1, K)
    y = np.stack([secagg.payload(secagg.encode(u, 1.0, f)[0], keys, K, k, 0) for k, u in enumerate(us)])
    d = secagg.decode(secagg.unmask_sum(y), f, K).astype(np.float64)
    want = np.mean([np.clip(u, -1.0, 1.0).astype(np.float64) for u in us], axis=0)
    assert np.all(np.abs(d - want) <= 2.0 ** -f / 2 + np.abs(want) * 2.0 ** -23 + 1e-30)


# ------------------------------------------------------------------------------------------ the ATen operators
@pytest.mark.parametrize("K", [2, 3])
@pytest.mark.parametrize("kind", [None, "adam"])
def test_round_matches_numpy_transcription(K, kind):
    N = 517
    topo = Topology.single_process(K, torch.device("cpu"))
    coll = TorchCollective(topo)
    kw = dict(secagg=True, secagg_clip=0.05, seed=4)
    strat = FedAvg(coll, topo, **kw) if kind is None else FedOpt(coll, topo, kind, lr=0.05, beta1=0.8, beta2=0.9, tau=1e-2,
                                                                 **kw)
    g = torch.Generator().manual_seed(K)
    z0 = torch.randn(N, generator=g)
    xs = [z0.clone() for _ in range(K)]
    strat.begin_block(0, N, xs)
    assert torch.equal(strat.z, z0)
    f, keys = strat.sa_f, secagg.pair_keys(4, K)
    z = z0.numpy().copy()
    m, v = np.zeros(N, dtype=np.float32), np.full(N, 1e-4, dtype=np.float32)
    for r in range(3):
        for x in xs:
            x.add_(torch.randn(N, generator=g) * 0.03)
        pays, clipped = [], 0
        for k, x in enumerate(xs):
            q, c, _ = secagg.encode(x.numpy() - z, 0.05, f)
            clipped += c
            pays.append(secagg.payload(q, keys, K, k, r))
        d = secagg.decode(secagg.unmask_sum(np.stack(pays)), f, K)
        if kind is None:
            znew = z + d
        else:
            m = np.float32(0.8) * m + np.float32(0.2) * d
            v = np.float32(0.9) * v + np.float32(0.1) * d * d
            znew = z + np.float32(0.05) * m / (np.sqrt(v) + np.float32(1e-2))
        met = strat.aggregate(r)
        assert met["sa_frac_bits"] == f and met["sa_clipped"] == clipped and clipped > 0
        for k in range(K):
            assert np.array_equal(strat.sa_payload[k][:N].numpy().view(np.uint32), pays[k])
        if kind is None:
            assert np.array_equal(strat.z.numpy(), znew)
        else:
            np.testing.assert_allclose(strat.z.numpy(), znew, rtol=1e-6, atol=1e-7)
        assert all(torch.equal(x, strat.z) for x in xs)
        z = strat.z.numpy().copy()
    assert int(strat.sa_t) == strat.sa_rounds == 3


def test_explicit_key_table():
    K = 3
    topo = Topology.single_process(K, torch.device("cpu"))
    keys = np.arange(24, dtype=np.uint32).reshape(3, 8)
    s = FedAvg(TorchCollective(topo), topo, secagg=True, secagg_keys=keys)
    assert np.array_equal(s.sa_keys.numpy().view(np.uint32), keys)
    assert s.state()["secagg"][2] == secagg.key_digest(keys)
    with pytest.raises(ValueError, match="secagg_keys"):
        FedAvg(TorchCollective(topo), topo, secagg=True, secagg_keys=keys[:2])


# ------------------------------------------------------------------------------------------ end to end
def _run(**kw):
    lines = []
    eng = federated_multi.run(federated_multi.Config(**{**TINY, **kw}), log=lines.append)
    return eng, [l for l in lines if l.startswith("dual (")]


def _val(line):
    return float(line.rsplit("=", 1)[1])


@pytest.mark.parametrize("server_opt", ["none", "adam"])
def test_cpu_runs_finish_with_finite_metrics(server_opt):
    eng, trace = _run(**KW, secagg=True, server_opt=server_opt)
    assert len(trace) == 10 and all(math.isfinite(_val(l)) and _val(l) > 0 for l in trace)
    assert eng.strategy.sa_rounds == int(eng.strategy.sa_t) == 10
    arena = eng.replicas[0].arenas["net"]
    assert torch.isfinite(arena.data).all()
    for rep in eng.replicas[1:]:
        assert torch.equal(rep.arenas["net"].data, arena.data)


def test_nan_attacker_trips_the_guard():
    with pytest.raises(FloatingPointError, match="non-finite"):
        _run(**{**KW, "Nadmm": 1, "max_minibatches": 1}, secagg=True, byzantine=1, attack="nan")


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


def test_kill_and_resume_continues_the_nonce_sequence(tmp_path):
    kw = dict(KW, K=3, Nadmm=3, secagg=True)
    eng, full = _run(**kw)
    assert len(full) == 15
    rec = str(tmp_path / "resume.pt")
    first = _killed_run(dict(kw, resume_out=rec), 27)
    assert 0 < len(first) < 15 and os.path.exists(rec)
    st = torch.load(rec, weights_only=False)["strategy_state"]
    assert st["sa_t"] == len(first) and st["secagg"][:2] == (1.0, secagg.frac_bits(1.0, 3))
    assert st["secagg"][2] == secagg.key_digest(secagg.pair_keys(kw.get("seed", 69), 3))
    eng2, second = _run(**kw, resume=rec)
    assert first + second == full
    assert eng2.strategy.sa_rounds == eng.strategy.sa_rounds == 15
    assert torch.equal(eng.replicas[0].arenas["net"].data, eng2.replicas[0].arenas["net"].data)
    # the last round's payloads (nonce t = 14) are those of the uninterrupted run
    for a, b in zip(eng.strategy.sa_payload, eng2.strategy.sa_payload):
        assert torch.equal(a, b)
    with pytest.raises(ValueError, match="secure-aggregation settings"):
        _run(**{**kw, "secagg_clip": 0.5}, resume=rec)
    with pytest.raises(ValueError, match="secure-aggregation settings"):
        _run(**{**kw, "seed": 70}, resume=rec)


def _dist_worker(rank, world, port, out):
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch.distributed as dist
    lines = []
    eng = federated_multi.run(federated_multi.Config(**DIST_KW, **TINY), log=lines.append)
    if rank == 0:
        torch.save({"lines": lines, "flat": eng.replicas[0].arenas["net"].data.clone(),
                    "pay": [p.clone() for p in eng.strategy.sa_payload]}, out)
    dist.destroy_process_group()


DIST_KW = dict(KW, K=4, secagg=True)


def test_two_process_gloo_equals_single_process_bit_for_bit(tmp_path):
    """Masked codes are summed as integers mod 2^32, which is exact and order-free, so the process layout does not change
    the result at all."""
    import torch.multiprocessing as mp
    out = str(tmp_path / "r0.pt")
    port = 39600 + (os.getpid() % 2000)
    mp.spawn(_dist_worker, args=(2, port, out), nprocs=2, join=True)
    got = torch.load(out, weights_only=False)
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        os.environ.pop(k, None)
    eng, single = _run(**DIST_KW)
    multi = [l for l in got["lines"] if l.startswith("dual (")]
    assert len(single) == len(multi) == 10
    assert single == multi
    assert torch.equal(got["flat"], eng.replicas[0].arenas["net"].data)
    # rank 0 hosts workers 0 and 2
    assert torch.equal(got["pay"][0], eng.strategy.sa_payload[0]) and torch.equal(got["pay"][1], eng.strategy.sa_payload[2])
