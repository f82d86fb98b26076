"""Compressed client updates on the H100: the compressed instantiations of the fused aggregation kernel (8- and 4-bit
codes, with and without error feedback and a server optimizer) against the ATen oracle (``TorchCollective``): payload
codes and scales bit for bit, the model, the server state and the error feedback within float32 tolerance; loopback ranks
(one-shot and two-shot) equal to one process bit for bit; graph replay; one launch per round; the NaN guard; and a
graphed ResNet18 ``federated_multi`` run against the ATen collective."""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("CUDA device required", allow_module_level=True)

from federated_pytorch_test_b200.algo import compress  # noqa: E402
from federated_pytorch_test_b200.parallel import Topology, TorchCollective  # noqa: E402
from federated_pytorch_test_b200.parallel.collective import QuantRound  # noqa: E402
from federated_pytorch_test_b200.parallel.fused import FusedCollective  # noqa: E402
from federated_pytorch_test_b200.parallel.loopback import LoopbackWorld  # noqa: E402

DEV = torch.device("cuda", 0)
SIZES = [850, 5130, 73984, 295424, 4720640]
KEY = compress.compress_key(69)
HYPER = ("adam", 1e-2, 0.9, 0.99, 1e-3)


def _quant(coll, xs, bits, t, ef):
    pay = [coll.payload_like_block(x, bits) for x in xs]
    efs = [torch.zeros_like(x) for x in xs] if ef else None
    return QuantRound(bits, KEY, t, [c for c, _ in pay], [s for _, s in pay], efs)


def _step(xs, z, g):
    """Local updates of a round: every worker moves a little from the server model, worker k by (k + 1) times as much."""
    N = z.numel()
    for k, x in enumerate(xs):
        x.copy_(z + torch.randn(N, device=DEV, generator=g) * (1e-3 * (k + 1)))


def _same_payload(qa, qb, n, bits):
    nb = -(-n * bits // 8)
    for ca, cb, sa, sb in zip(qa.codes, qb.codes, qa.scales, qb.scales):
        assert torch.equal(ca[:nb], cb[:nb])
        assert torch.equal(sa.view(torch.int32), sb.view(torch.int32))


@pytest.mark.parametrize("kind", [None, "adam"])
@pytest.mark.parametrize("ef", [False, True])
@pytest.mark.parametrize("bits", [8, 4])
@pytest.mark.parametrize("K", [1, 2, 3, 4, 8, 10, 16])
@pytest.mark.parametrize("N", SIZES)
def test_fused_matches_oracle_single_process(N, K, bits, ef, kind):
    topo = Topology.single_process(K, DEV)
    coll, oracle = FusedCollective(topo), TorchCollective(topo)
    stride = -(-N // 32) * 32
    arena = coll.heap.alloc(K * stride)
    xs = [arena[k * stride: k * stride + N] for k in range(K)]
    g = torch.Generator(device=DEV).manual_seed(N + K + bits)
    z = coll.zeros_like_block(xs[0], "z")
    z.copy_(torch.randn(N, device=DEV, generator=g))
    zr = z.clone()
    t, tr = torch.zeros(1, dtype=torch.int64, device=DEV), torch.zeros(1, dtype=torch.int64, device=DEV)
    q, qr = _quant(coll, xs, bits, t, ef), _quant(oracle, xs, bits, tr, ef)
    if kind:
        m, v = coll.zeros_like_block(xs[0], "m"), coll.zeros_like_block(xs[0], "v").fill_(1e-6)
        mr, vr = m.clone(), v.clone()
    n0 = coll.launches
    for r in range(2):
        _step(xs, z, g)
        xr = [x.clone() for x in xs]
        if kind:
            got = coll.fedopt_(xs, z, m, v, *HYPER, compress=q)
            want = float(oracle.fedopt_(xr, zr, mr, vr, *HYPER, compress=qr))
            torch.testing.assert_close(m, mr, rtol=1e-4, atol=1e-7)
            torch.testing.assert_close(v, vr, rtol=1e-4, atol=1e-12)
        else:
            got = coll.fedavg_(xs, z, compress=q)
            want = float(oracle.fedavg_(xr, zr, compress=qr))
        assert coll.launches - n0 == r + 1                     # one launch per round
        _same_payload(q, qr, N, bits)
        torch.testing.assert_close(z, zr, rtol=1e-5, atol=1e-6)
        assert got == pytest.approx(want, rel=1e-3, abs=1e-12)
        assert all(torch.equal(x, z) for x in xs)
        if ef:
            for e, er in zip(q.ef, qr.ef):
                torch.testing.assert_close(e, er, rtol=1e-5, atol=1e-9)
        assert coll.last_q[0] == pytest.approx(oracle.last_q[0], rel=1e-4)
        assert coll.last_q[1] == pytest.approx(oracle.last_q[1], rel=1e-4)
        zr.copy_(z)                                            # next round from the same server model
        if kind:
            mr.copy_(m)
            vr.copy_(v)
        if ef:
            for e, er in zip(q.ef, qr.ef):
                er.copy_(e)
    assert int(t) == int(tr) == 2
    assert coll.last_nonfinite == 0.0


def _loopback_round(world, xs_rank, zs, qs, ms, vs):
    def one(rank, c):
        if ms is not None:
            c.launch_fedopt_(xs_rank[rank], zs[rank], ms[rank], vs[rank], *HYPER, compress=qs[rank])
        else:
            c.launch_fedavg_(xs_rank[rank], zs[rank], True, compress=qs[rank])
    world.run(one)


@pytest.mark.parametrize("kind", [None, "adam"])
@pytest.mark.parametrize("bits", [8, 4])
@pytest.mark.parametrize("two_shot", ["0", "1"])
@pytest.mark.parametrize("W,per_rank", [(2, 1), (4, 1), (2, 2)])
@pytest.mark.parametrize("N", [5130, 295424, 4720640])
def test_loopback_ranks_equal_single_process(N, W, per_rank, two_shot, bits, kind):
    K = W * per_rank
    world = LoopbackWorld(W, DEV, max_blocks=8, timeout_s=10.0, K=K)
    for c in world.colls:
        c.two_shot_mode = two_shot
    stride = -(-N // 32) * 32
    xs_rank = [[] for _ in range(W)]
    for _ in range(per_rank):
        for r, buf in enumerate(world.alloc(stride)):
            xs_rank[r].append(buf[:N])
    by_worker = [xs_rank[ck % W][ck // W] for ck in range(K)]
    g = torch.Generator(device=DEV).manual_seed(N + K)
    z0 = torch.randn(N, device=DEV, generator=g)
    zs = [c.zeros_like_block(x[0], "z") for c, x in zip(world.colls, xs_rank)]
    for zz in zs:
        zz.copy_(z0)
    ts = [torch.zeros(1, dtype=torch.int64, device=DEV) for _ in range(W)]
    qs = [_quant(c, xs_rank[r], bits, ts[r], True) for r, c in enumerate(world.colls)]
    ms = vs = None
    if kind:                                  # symmetric slices: two-shot ranks broadcast their slice of m and v
        ms = [c.zeros_like_block(x[0], "m") for c, x in zip(world.colls, xs_rank)]
        vs = [c.zeros_like_block(x[0], "v").fill_(1e-6) for c, x in zip(world.colls, xs_rank)]
    # the same rounds on one process with all K replicas co-resident
    single = FusedCollective(Topology.single_process(K, DEV))
    arena = single.heap.alloc(K * stride)
    xs1 = [arena[k * stride: k * stride + N] for k in range(K)]
    z1 = single.zeros_like_block(xs1[0], "z")
    z1.copy_(z0)
    t1 = torch.zeros(1, dtype=torch.int64, device=DEV)
    q1 = _quant(single, xs1, bits, t1, True)
    if kind:
        m1, v1 = single.zeros_like_block(xs1[0], "m"), single.zeros_like_block(xs1[0], "v").fill_(1e-6)
    for r in range(2):
        _step(by_worker, zs[0], g)
        for x1, x in zip(xs1, by_worker):
            x1.copy_(x)
        torch.cuda.synchronize()
        _loopback_round(world, xs_rank, zs, qs, ms, vs)
        if kind:
            d1 = single.fedopt_(xs1, z1, m1, v1, *HYPER, compress=q1)
        else:
            d1 = single.fedavg_(xs1, z1, compress=q1)
        for rank, c in enumerate(world.colls):
            rec = c.read_record()
            assert c.last_two_shot == (two_shot == "1" and per_rank == 1)     # two-shot needs one replica per rank
            assert rec[0] == pytest.approx(d1, rel=1e-4)
            assert c.last_q[0] == pytest.approx(single.last_q[0], rel=1e-4)
            assert c.last_q[1] == pytest.approx(single.last_q[1], rel=1e-4)
        for zz in zs:
            assert torch.equal(zz, z1)
        for x in by_worker:
            assert torch.equal(x, z1)
        for ck in range(K):
            r, j = ck % W, ck // W
            assert torch.equal(qs[r].ef[j], q1.ef[ck])
            _same_payload(QuantRound(bits, KEY, ts[r], [qs[r].codes[j]], [qs[r].scales[j]]),
                          QuantRound(bits, KEY, t1, [q1.codes[ck]], [q1.scales[ck]]), N, bits)
        if kind:
            for mm, vv in zip(ms, vs):
                assert torch.equal(mm, m1) and torch.equal(vv, v1)
    assert all(int(t) == 2 for t in ts) and int(t1) == 2


@pytest.mark.parametrize("kind", [None, "adam"])
def test_graph_replay_equals_eager_rounds(kind):
    K, N = 4, 73984
    deltas = [torch.randn(K, N, device=DEV, generator=torch.Generator(device=DEV).manual_seed(r)) * 1e-3 for r in range(2)]
    z0 = torch.randn(N, device=DEV, generator=torch.Generator(device=DEV).manual_seed(7))

    def setup():
        topo = Topology.single_process(K, DEV)
        coll = FusedCollective(topo)
        arena = coll.heap.alloc(K * N)
        xs = [arena[k * N:(k + 1) * N] for k in range(K)]
        z = coll.zeros_like_block(xs[0], "z")
        z.copy_(z0)
        t = torch.zeros(1, dtype=torch.int64, device=DEV)
        q = _quant(coll, xs, 8, t, True)
        mv = (coll.zeros_like_block(xs[0], "m"), coll.zeros_like_block(xs[0], "v").fill_(1e-6)) if kind else None
        return coll, xs, z, q, mv

    def launch(coll, xs, z, q, mv):
        if kind:
            coll.launch_fedopt_(xs, z, mv[0], mv[1], *HYPER, compress=q)
        else:
            coll.launch_fedavg_(xs, z, True, compress=q)

    coll, xs, z, q, mv = setup()
    eager = []
    for r in range(2):
        for k, x in enumerate(xs):
            x.copy_(z + deltas[r][k])
        launch(coll, xs, z, q, mv)
        coll.read_record()
        eager.append((z.clone(), [e.clone() for e in q.ef]))
    coll, xs, z, q, mv = setup()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            launch(coll, xs, z, q, mv)
    torch.cuda.current_stream().wait_stream(s)
    assert int(q.t) == 0                           # capture did not run the kernel
    for r in range(2):
        for k, x in enumerate(xs):
            x.copy_(z + deltas[r][k])
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(z, eager[r][0])
        assert all(torch.equal(e, w) for e, w in zip(q.ef, eager[r][1]))
        assert int(q.t) == r + 1


@pytest.mark.parametrize("bits", [8, 4])
def test_nonfinite_worker_sets_nonfinite(bits):
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
        xs[2][1000] = bad                          # group 7: coordinates 896 .. 1023
        q = _quant(coll, xs, bits, torch.zeros(1, dtype=torch.int64, device=DEV), False)
        coll.fedavg_(xs, z, compress=q)
        assert coll.last_nonfinite > 0
        assert math.isnan(float(q.scales[2][7])) and not math.isfinite(coll.last_q[0])
        assert torch.isnan(z[896:1024]).all() and torch.isfinite(z[:896]).all() and torch.isfinite(z[1024:]).all()


def _run(**kw):
    from federated_pytorch_test_b200.api import federated_multi

    base = dict(K=4, use_resnet=True, Nloop=1, Nadmm=2, max_minibatches=3, train_size=2048, test_size=256,
                check_results=False, save_model=False, graphs=True)
    lines = []
    eng = federated_multi.run(federated_multi.Config(**{**base, **kw}), log=lines.append)
    return eng, lines


def test_nan_attacker_trips_the_guard():
    with pytest.raises(FloatingPointError, match="non-finite"):
        _run(K=4, compress_bits=8, byzantine=1, attack="nan", Nadmm=1, max_minibatches=1)


def test_graphed_resnet18_run_matches_aten():
    kw = dict(compress_bits=8, compress_ef=True)
    eng, fused = _run(**kw)
    _, aten = _run(**kw, collective="torch")
    df = [l for l in fused if l.startswith("dual (")]
    da = [l for l in aten if l.startswith("dual (")]
    assert len(df) == len(da) > 0
    # The first round starts both runs from the same model.  Later rounds start from models that differ in the last bits
    # (the kernel scales by a fast reciprocal of K, the ATen path by 1/K): next to the tiny updates of a round that is a
    # good part of a quantization step, so later rounds draw different codes and the trajectories separate by about the
    # quantization noise.
    for i, (a, b) in enumerate(zip(df, da)):
        assert a.split("=")[:-1] == b.split("=")[:-1]
        assert float(a.rsplit("=", 1)[1]) == pytest.approx(float(b.rsplit("=", 1)[1]), rel=2e-2 if i == 0 else 0.25)
    T = len(df)
    assert eng.strategy.q_rounds == T and int(eng.strategy.q_t) == T
