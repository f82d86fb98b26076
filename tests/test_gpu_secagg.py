"""Secure aggregation on the H100: the SecAgg instantiations of the fused aggregation kernel (with and without a server
optimizer) against the numpy oracle (``algo/secagg.py``): the FedAvg model and the payloads bit for bit, the FedAdam state
within float32 tolerance; the RFC 8439 block vector through the device; loopback ranks (one-shot and two-shot) equal to
one process bit for bit; one launch per round; graph replay advancing the nonce; the NaN guard; and a graphed ResNet18
``federated_multi`` run against the ATen collective."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("CUDA device required", allow_module_level=True)

from federated_pytorch_test_b200.algo import secagg  # noqa: E402
from federated_pytorch_test_b200.ops import cuda_ops  # noqa: E402
from federated_pytorch_test_b200.parallel import Topology  # noqa: E402
from federated_pytorch_test_b200.parallel.collective import SecAggRound  # noqa: E402
from federated_pytorch_test_b200.parallel.fused import FusedCollective  # noqa: E402
from federated_pytorch_test_b200.parallel.loopback import LoopbackWorld  # noqa: E402

DEV = torch.device("cuda", 0)
SIZES = [850, 5130, 73984, 295424, 4720640]
HYPER = ("adam", 1e-2, 0.9, 0.99, 1e-3)
CLIP = 0.01


def _keys_dev(keys):
    return torch.from_numpy(np.array(keys, dtype=np.uint32).view(np.int32)).to(DEV)


def _round(coll, xs, K, t, clip=CLIP, keys=None):
    keys = secagg.pair_keys(69, K) if keys is None else keys
    return SecAggRound(float(np.float32(clip)), secagg.frac_bits(clip, K), _keys_dev(keys), t,
                       [coll.payload32_like_block(x) for x in xs]), keys


def _step(xs, z, g):
    """Local updates of a round: every worker moves from the server model, worker k by (k + 1) times as much; some
    coordinates land beyond the clip."""
    N = z.numel()
    for k, x in enumerate(xs):
        x.copy_(z + torch.randn(N, device=DEV, generator=g) * (2e-3 * (k + 1)))


def _codes(xs, z, sa):
    zn = z.cpu().numpy()
    return [secagg.encode(x.cpu().numpy() - zn, sa.clip, sa.f) for x in xs]


@pytest.mark.parametrize("kind", [None, "adam"])
@pytest.mark.parametrize("K", [2, 3, 4, 8, 16])
@pytest.mark.parametrize("N", SIZES)
def test_fused_matches_oracle_single_process(N, K, kind):
    topo = Topology.single_process(K, DEV)
    coll = FusedCollective(topo)
    stride = -(-N // 32) * 32
    arena = coll.heap.alloc(K * stride)
    xs = [arena[k * stride: k * stride + N] for k in range(K)]
    g = torch.Generator(device=DEV).manual_seed(N + K)
    z = coll.zeros_like_block(xs[0], "z")
    z.copy_(torch.randn(N, device=DEV, generator=g) * 0.1)
    t = torch.zeros(1, dtype=torch.int64, device=DEV)
    sa, keys = _round(coll, xs, K, t)
    if kind:
        m, v = coll.zeros_like_block(xs[0], "m"), coll.zeros_like_block(xs[0], "v").fill_(1e-6)
        mr, vr = m.clone(), v.clone()
    check_payload = K <= 4 or N <= 295424
    n0, l0 = coll.launches, cuda_ops.launch_count()
    for r in range(2):
        _step(xs, z, g)
        enc = _codes(xs, z, sa)
        S = np.sum(np.stack([q.astype(np.int64) for q, _, _ in enc]), axis=0).astype(np.int32)
        d = torch.from_numpy(secagg.decode(S, sa.f, K)).to(DEV)
        zo = z.clone()
        if kind:
            got = coll.fedopt_(xs, z, m, v, *HYPER, secagg=sa)
            mr.mul_(0.9).add_(d, alpha=0.1)
            vr.mul_(0.99).add_(d * d, alpha=0.01)
            torch.testing.assert_close(m, mr, rtol=1e-4, atol=1e-7)
            torch.testing.assert_close(v, vr, rtol=1e-4, atol=1e-12)
            torch.testing.assert_close(z, zo + 1e-2 * mr / (vr.sqrt() + 1e-3), rtol=1e-5, atol=1e-6)
            mr.copy_(m)
            vr.copy_(v)
        else:
            got = coll.fedavg_(xs, z, secagg=sa)
            assert torch.equal(z, zo + d)                          # bit for bit
            assert got == pytest.approx(float(torch.dot(zo - z, zo - z)), rel=1e-3, abs=1e-30)
        assert coll.launches - n0 == r + 1 and cuda_ops.launch_count() - l0 == r + 1      # one launch per round
        assert all(torch.equal(x, z) for x in xs)
        assert coll.last_sa == (sum(c for _, c, _ in enc), 0) and coll.last_nonfinite == 0.0
        pays = [p[:N].cpu().numpy().view(np.uint32) for p in sa.payload]
        if check_payload and r == 0:
            for k in range(K):
                assert np.array_equal(pays[k], secagg.payload(enc[k][0], keys, K, k, r)), k
        else:                                                      # the masks cancel in the device's payloads
            assert np.array_equal(secagg.unmask_sum(np.stack(pays)), S)
    assert int(t) == 2


def test_rfc8439_block_vector_through_the_device():
    K, N = 2, 64
    topo = Topology.single_process(K, DEV)
    coll = FusedCollective(topo)
    arena = coll.heap.alloc(K * N)
    xs = [arena[k * N:(k + 1) * N] for k in range(K)]
    z = coll.zeros_like_block(xs[0], "z")
    z.copy_(torch.randn(N, device=DEV))
    for x in xs:
        x.copy_(z)                                                 # u = 0: the payloads are the masks
    t = torch.full((1,), 0x4A00000009000000, dtype=torch.int64, device=DEV)
    sa, _ = _round(coll, xs, K, t, keys=np.frombuffer(bytes(range(32)), dtype="<u4").reshape(1, 8))
    zo = z.clone()
    coll.fedavg_(xs, z, secagg=sa)
    want = np.array([0xE4E7F110, 0x15593BD1, 0x1FDD0F50, 0xC47120A3, 0xC7F4D1C7, 0x0368C033, 0x9AAA2204, 0x4E6CD4C3,
                     0x466482D2, 0x09AA9F07, 0x05D7C214, 0xA2028BD9, 0xD19C12B5, 0xB94E16DE, 0xE883D0CB, 0x4E3C50A2],
                    dtype=np.uint32)
    y0 = sa.payload[0].cpu().numpy().view(np.uint32)
    y1 = sa.payload[1].cpu().numpy().view(np.uint32)
    assert np.array_equal(y0[16:32], want)
    assert np.array_equal(y1[16:32], np.uint32(0) - want)
    assert torch.equal(z, zo)


def _loopback_setup(N, W, per_rank, two_shot, kind):
    """W loopback ranks of per_rank replicas each; returns the world, the replicas by rank and by worker, z, the SecAgg
    rounds, m and v (or None) of every rank."""
    K = W * per_rank
    world = LoopbackWorld(W, DEV, max_blocks=8, timeout_s=30.0, K=K)
    for c in world.colls:
        c.two_shot_mode = two_shot
    stride = -(-N // 32) * 32
    xs_rank = [[] for _ in range(W)]
    for _ in range(per_rank):
        for r, buf in enumerate(world.alloc(stride)):
            xs_rank[r].append(buf[:N])
    by_worker = [xs_rank[ck % W][ck // W] for ck in range(K)]
    z0 = torch.randn(N, device=DEV, generator=torch.Generator(device=DEV).manual_seed(N + K)) * 0.1
    zs = [c.zeros_like_block(x[0], "z") for c, x in zip(world.colls, xs_rank)]
    for zz in zs:
        zz.copy_(z0)
    ts = [torch.zeros(1, dtype=torch.int64, device=DEV) for _ in range(W)]
    sas = [_round(c, xs_rank[r], K, ts[r])[0] for r, c in enumerate(world.colls)]
    ms = vs = None
    if kind:                                  # symmetric slices: two-shot ranks broadcast their slice of m and v
        ms = [c.zeros_like_block(x[0], "m") for c, x in zip(world.colls, xs_rank)]
        vs = [c.zeros_like_block(x[0], "v").fill_(1e-6) for c, x in zip(world.colls, xs_rank)]
    return world, xs_rank, by_worker, zs, sas, ms, vs


@pytest.mark.parametrize("kind", [None, "adam"])
@pytest.mark.parametrize("N", SIZES)
def test_64_workers_match_oracle(N, kind):
    """64 workers exceed the 16 replicas one process hosts: 4 loopback ranks of 16 replicas each, against the oracle."""
    W, K = 4, 64
    world, xs_rank, by_worker, zs, sas, ms, vs = _loopback_setup(N, W, K // W, "0", kind)
    keys = secagg.pair_keys(69, K)
    g = torch.Generator(device=DEV).manual_seed(N)
    if kind:
        mr, vr = ms[0].clone(), vs[0].clone()
    for r in range(2):
        _step(by_worker, zs[0], g)
        torch.cuda.synchronize()
        enc = _codes(by_worker, zs[0], sas[0])
        S = np.sum(np.stack([q.astype(np.int64) for q, _, _ in enc]), axis=0).astype(np.int32)
        d = torch.from_numpy(secagg.decode(S, sas[0].f, K)).to(DEV)
        zo = zs[0].clone()
        _loopback_round(world, xs_rank, zs, sas, ms, vs)
        for c in world.colls:
            c.read_record()
            assert c.last_sa == (sum(cnt for _, cnt, _ in enc), 0)
        if kind:
            mr.mul_(0.9).add_(d, alpha=0.1)
            vr.mul_(0.99).add_(d * d, alpha=0.01)
            torch.testing.assert_close(ms[0], mr, rtol=1e-4, atol=1e-7)
            torch.testing.assert_close(vs[0], vr, rtol=1e-4, atol=1e-12)
            torch.testing.assert_close(zs[0], zo + 1e-2 * mr / (vr.sqrt() + 1e-3), rtol=1e-5, atol=1e-6)
            mr.copy_(ms[0])
            vr.copy_(vs[0])
        else:
            assert torch.equal(zs[0], zo + d)
        for zz in zs[1:]:
            assert torch.equal(zz, zs[0])
        pays = [sas[ck % W].payload[ck // W][:N].cpu().numpy().view(np.uint32) for ck in range(K)]
        if N <= 295424 and r == 0:
            for k in range(K):
                assert np.array_equal(pays[k], secagg.payload(enc[k][0], keys, K, k, r)), k
        else:
            assert np.array_equal(secagg.unmask_sum(np.stack(pays)), S)


def _loopback_round(world, xs_rank, zs, sas, ms, vs):
    def one(rank, c):
        if ms is not None:
            c.launch_fedopt_(xs_rank[rank], zs[rank], ms[rank], vs[rank], *HYPER, secagg=sas[rank])
        else:
            c.launch_fedavg_(xs_rank[rank], zs[rank], True, secagg=sas[rank])
    world.run(one)


@pytest.mark.parametrize("kind", [None, "adam"])
@pytest.mark.parametrize("two_shot", ["0", "1"])
@pytest.mark.parametrize("W,per_rank", [(2, 1), (4, 1), (2, 2)])
@pytest.mark.parametrize("N", [5130, 295424, 4720640])
def test_loopback_ranks_equal_single_process(N, W, per_rank, two_shot, kind):
    K = W * per_rank
    world, xs_rank, by_worker, zs, sas, ms, vs = _loopback_setup(N, W, per_rank, two_shot, kind)
    ts = [sa.t for sa in sas]
    stride = -(-N // 32) * 32
    g = torch.Generator(device=DEV).manual_seed(N + K)
    z0 = zs[0].clone()
    single = FusedCollective(Topology.single_process(K, DEV))
    arena = single.heap.alloc(K * stride)
    xs1 = [arena[k * stride: k * stride + N] for k in range(K)]
    z1 = single.zeros_like_block(xs1[0], "z")
    z1.copy_(z0)
    t1 = torch.zeros(1, dtype=torch.int64, device=DEV)
    sa1, _ = _round(single, xs1, K, t1)
    if kind:
        m1, v1 = single.zeros_like_block(xs1[0], "m"), single.zeros_like_block(xs1[0], "v").fill_(1e-6)
    for r in range(2):
        _step(by_worker, zs[0], g)
        for x1, x in zip(xs1, by_worker):
            x1.copy_(x)
        torch.cuda.synchronize()
        _loopback_round(world, xs_rank, zs, sas, ms, vs)
        if kind:
            single.fedopt_(xs1, z1, m1, v1, *HYPER, secagg=sa1)
        else:
            single.fedavg_(xs1, z1, secagg=sa1)
        for c in world.colls:
            c.read_record()
            assert c.last_two_shot == (two_shot == "1" and per_rank == 1)
            assert c.last_sa == single.last_sa and single.last_sa[0] > 0
        for zz in zs:
            assert torch.equal(zz, z1)
        for x in by_worker:
            assert torch.equal(x, z1)
        for ck in range(K):
            assert torch.equal(sas[ck % W].payload[ck // W], sa1.payload[ck])
        if kind:
            for mm, vv in zip(ms, vs):
                assert torch.equal(mm, m1) and torch.equal(vv, v1)
    assert all(int(t) == 2 for t in ts) and int(t1) == 2


def test_graph_replay_advances_the_nonce():
    K, N = 4, 73984
    topo = Topology.single_process(K, DEV)
    coll = FusedCollective(topo)
    arena = coll.heap.alloc(K * N)
    xs = [arena[k * N:(k + 1) * N] for k in range(K)]
    z = coll.zeros_like_block(xs[0], "z")
    z.copy_(torch.randn(N, device=DEV, generator=torch.Generator(device=DEV).manual_seed(7)) * 0.1)
    t = torch.zeros(1, dtype=torch.int64, device=DEV)
    sa, keys = _round(coll, xs, K, t)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            coll.launch_fedavg_(xs, z, True, secagg=sa)
    torch.cuda.current_stream().wait_stream(s)
    assert int(t) == 0                                             # capture did not run the kernel
    g = torch.Generator(device=DEV).manual_seed(3)
    prev = None
    for r in range(3):
        _step(xs, z, g)
        enc = _codes(xs, z, sa)
        zo = z.clone()
        graph.replay()
        torch.cuda.synchronize()
        assert int(t) == r + 1
        S = np.sum(np.stack([q.astype(np.int64) for q, _, _ in enc]), axis=0).astype(np.int32)
        assert torch.equal(z, zo + torch.from_numpy(secagg.decode(S, sa.f, K)).to(DEV))
        pays = [p[:N].cpu().numpy().view(np.uint32) for p in sa.payload]
        for k in range(K):
            assert np.array_equal(pays[k], secagg.payload(enc[k][0], keys, K, k, r))
        if prev is not None:
            assert not np.array_equal(pays[0], prev)
        prev = pays[0]


def test_nonfinite_replica_trips_the_guard():
    K, N = 3, 5130
    topo = Topology.single_process(K, DEV)
    coll = FusedCollective(topo)
    stride = -(-N // 32) * 32
    arena = coll.heap.alloc(K * stride)
    xs = [arena[k * stride: k * stride + N] for k in range(K)]
    z = coll.zeros_like_block(xs[0], "z")
    g = torch.Generator(device=DEV).manual_seed(1)
    for bad in (float("nan"), float("inf")):
        z.zero_()
        _step(xs, z, g)
        xs[2][1000] = bad
        xs[1][7] = bad
        sa, _ = _round(coll, xs, K, torch.zeros(1, dtype=torch.int64, device=DEV))
        coll.fedavg_(xs, z, secagg=sa)
        assert coll.last_sa[1] == 2 and coll.last_nonfinite >= 2
        assert torch.isfinite(z).all()                             # non-finite updates code to 0


def _run(**kw):
    from federated_pytorch_test_b200.api import federated_multi

    base = dict(K=4, use_resnet=True, Nloop=1, Nadmm=2, max_minibatches=3, train_size=2048, test_size=256,
                check_results=False, save_model=False, graphs=True)
    lines = []
    eng = federated_multi.run(federated_multi.Config(**{**base, **kw}), log=lines.append)
    return eng, lines


def test_nan_attacker_trips_the_guard():
    with pytest.raises(FloatingPointError, match="non-finite"):
        _run(secagg=True, byzantine=1, attack="nan", Nadmm=1, max_minibatches=1)


def test_graphed_resnet18_run_matches_aten():
    eng, fused = _run(secagg=True)
    _, aten = _run(secagg=True, collective="torch")
    df = [l for l in fused if l.startswith("dual (")]
    da = [l for l in aten if l.startswith("dual (")]
    assert len(df) == len(da) > 0
    # Both collectives form the same new model bit for bit from the same replicas (test_fused_matches_oracle_single_process),
    # but the two runs' training steps differ in the last bits (the weight gradients are accumulated with atomics), and
    # those differences grow over the minibatches of later rounds, as in the DP and compressed comparisons.
    for i, (a, b) in enumerate(zip(df, da)):
        assert a.split("=")[:-1] == b.split("=")[:-1]
        assert float(a.rsplit("=", 1)[1]) == pytest.approx(float(b.rsplit("=", 1)[1]), rel=2e-2 if i == 0 else 0.1), (i, a, b)
    T = len(df)
    assert eng.strategy.sa_rounds == T and int(eng.strategy.sa_t) == T
