"""SCAFFOLD control variates on the H100: the two per-round kernels against the ATen path, the fused collective against the
ATen collective over several rounds (synchronous and deferred), loopback ranks one- and two-shot, a graphed ResNet18
run on Dirichlet shards with client sampling, and the launches the flag adds."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():  # collected (and deselected) on the CPU box
    pytest.skip("CUDA device required", allow_module_level=True)

from federated_pytorch_test_b200.algo import scaffold as scaf  # noqa: E402
from federated_pytorch_test_b200.algo.scaffold import ControlVariates  # noqa: E402
from federated_pytorch_test_b200.algo.strategies import FedAvg, FedOpt  # noqa: E402
from federated_pytorch_test_b200.ops import cuda_ops, flatops  # noqa: E402
from federated_pytorch_test_b200.ops import functional as FX  # noqa: E402
from federated_pytorch_test_b200.parallel import Topology, TorchCollective  # noqa: E402
from federated_pytorch_test_b200.parallel.fused import FusedCollective  # noqa: E402
from federated_pytorch_test_b200.parallel.loopback import LoopbackWorld  # noqa: E402

DEV = torch.device("cuda", 0)


@pytest.fixture(autouse=True)
def _fast_path():
    FX.set_fast_path(True)
    yield
    FX.set_fast_path(True)


def _aten(fn, *a):
    FX.set_fast_path(False)
    try:
        return fn(*a)
    finally:
        FX.set_fast_path(True)


# ------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("n", [1, 3, 4, 1000003, 4720640])
@pytest.mark.parametrize("R", [1, 5, 16])
def test_kernels_match_the_aten_path(n, R):
    g = torch.Generator(device=DEV).manual_seed(n + R)
    cis = [torch.randn(n, device=DEV, generator=g) for _ in range(R)]
    xs = [torch.randn(n, device=DEV, generator=g) for _ in range(R)]
    c, z = torch.randn(n, device=DEV, generator=g), torch.randn(n, device=DEV, generator=g)
    taus = [0 if j % 3 == 1 else 1 + j for j in range(R)]            # every third replica sat out
    if R > 1:
        xs[1][n // 2] = float("nan")                                  # a sat-out replica's NaN is never read
        xs[0][n - 1] = float("nan")                                   # a participant's NaN propagates (scalar tail too)
    scales = [scaf.step_scale(t, 0.05) for t in taus]
    ref = [t.clone() for t in cis]
    flatops.scaffold_cv_(cis, xs, c, z, scales)
    _aten(flatops.scaffold_cv_, ref, xs, c, z, scales)
    for j in range(R):
        torch.testing.assert_close(cis[j], ref[j], rtol=0, atol=0, equal_nan=True)
    assert R == 1 or torch.isnan(cis[0][n - 1])
    ds = [torch.empty(n, device=DEV) for _ in range(R)]
    dr = [torch.empty(n, device=DEV) for _ in range(R)]
    work = flatops.scaffold_workspace(n, R, DEV)
    assert work[1] is not None                                       # the CUDA workspace
    got = flatops.scaffold_corr_(cis, ds, c, work).clone()
    want = _aten(flatops.scaffold_corr_, ref, dr, c, flatops.scaffold_workspace(n, R, "cpu"))
    for j in range(R):
        torch.testing.assert_close(ds[j], dr[j], rtol=0, atol=0, equal_nan=True)
    torch.testing.assert_close(got.cpu(), want.cpu(), rtol=1e-4, atol=0, equal_nan=True)
    again = flatops.scaffold_corr_(cis, ds, c, work).clone()
    assert torch.equal(got.isnan(), again.isnan()) and torch.equal(got.nan_to_num(), again.nan_to_num())  # fixed order
    assert R == 1 or bool(torch.isnan(got[0]))


# ------------------------------------------------------------------------------------------ fused against ATen
def _blocks(coll, K, N):
    stride = -(-N // 32) * 32
    if hasattr(coll, "heap"):
        arenas = [coll.heap.alloc(stride) for _ in range(K)]    # one arena per replica, as the engine's
    else:
        arenas = [torch.zeros(stride, device=DEV) for _ in range(K)]
    return [a[:N] for a in arenas]


def _strategy(coll, topo, kind, n):
    if kind == "plain":
        return FedAvg(coll, topo, scaffold=True)
    if kind == "dirichlet":
        return FedAvg(coll, topo, clients_per_round=4, client_n=n, seed=5, scaffold=True)
    return FedOpt(coll, topo, "adam", scaffold=True)


def _rounds(coll, topo, kind, N, deferred, rounds=4):
    K = topo.K
    n = [30, 7, 12, 50, 3, 19, 8, 41]
    strat = _strategy(coll, topo, kind, n)
    xs = _blocks(coll, K, N)
    g = torch.Generator(device=DEV).manual_seed(N)
    init = torch.randn(N, device=DEV, generator=g)
    for x in xs:
        x.copy_(init)
    strat.begin_block(0, N, xs)
    out = []
    for r in range(rounds):
        steps = []
        for i, x in enumerate(xs):                       # "local training": the correction and a seeded drift
            part = strat.participates(i)
            steps.append(2 + i if part else 0)
            drift = torch.randn(N, device=DEV, generator=g)
            if part:
                x.add_(0.01 * drift - 0.05 * strat.penalty(i).y)
        strat.note_local_steps(steps, 0.05)
        if deferred:
            m = strat.aggregate_end(strat.aggregate_begin(r))
        else:
            m = strat.aggregate(r)
        out.append(m)
    cv = strat.scaffold
    return out, xs, cv.c[0], cv.cis[0], cv.ds[0]


@pytest.mark.parametrize("kind", ["plain", "dirichlet", "fedadam"])
@pytest.mark.parametrize("N", [5131, 295424])
def test_fused_matches_torch_collective_sync_and_deferred(kind, N):
    K = 8
    topo = Topology.single_process(K, DEV)
    ref = _rounds(TorchCollective(topo), topo, kind, N, deferred=False)
    sync = _rounds(FusedCollective(topo), topo, kind, N, deferred=False)
    dfr = _rounds(FusedCollective(topo), topo, kind, N, deferred=True)
    for got in (sync, dfr):
        for mg, mr in zip(got[0], ref[0]):
            assert mg["dual"] == pytest.approx(mr["dual"], rel=1e-3)        # the model's record, not the c launch's
            assert mg["scaffold_corr"] == pytest.approx(mr["scaffold_corr"], rel=1e-4)
            assert mg.get("participants") == mr.get("participants")
        for a, b in zip(got[1], ref[1]):
            torch.testing.assert_close(a, b, rtol=1e-4, atol=1e-5)
        torch.testing.assert_close(got[2], ref[2], rtol=1e-4, atol=1e-4)
        for part in (3, 4):
            for a, b in zip(got[part], ref[part]):
                torch.testing.assert_close(a, b, rtol=1e-4, atol=1e-4)
    for a, b in zip(sync[1:], dfr[1:]):                   # the two fused paths launch the same kernels
        for u, v in zip(a if isinstance(a, list) else [a], b if isinstance(b, list) else [b]):
            assert torch.equal(u, v)
    for a, b in zip(sync[0], dfr[0]):                     # dual_sq is summed with float atomics: last bits vary
        assert a["dual"] == pytest.approx(b["dual"], rel=1e-5)


# ------------------------------------------------------------------------------------------ loopback ranks
def _loopback(W, per_rank, two_shot, N):
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
    cvs = [ControlVariates(c, c.topo) for c in world.colls]
    for cv, xs in zip(cvs, xs_rank):
        cv.begin_block(0, xs)
    g = torch.Generator(device=DEV).manual_seed(N + K)
    z = torch.randn(N, device=DEV, generator=g)
    zs = [z.clone() for _ in range(W)]
    taus = [0 if k == 1 else 1 + k for k in range(K)]
    cis_ref, c_ref = [np.zeros(N) for _ in range(K)], np.zeros(N)
    for _ in range(3):
        for x in by_worker:
            x.copy_(z + torch.randn(N, device=DEV, generator=g))
        xr = [x.double().cpu().numpy() for x in by_worker]
        for r, cv in enumerate(cvs):
            cv.note_local_steps([taus[ck] for ck in world.colls[r].topo.local_workers], 0.05)
        world.run(lambda r, c: cvs[r].end_round(xs_rank[r], zs[r]))
        for c in world.colls:
            c.read_record()
            assert c.last_two_shot == (two_shot == "1" and per_rank == 1)
        cis_ref, c_ref, _ = scaf.reference_round(cis_ref, xr, c_ref, z.double().cpu().numpy(), taus, 0.05)
    for cv in cvs:
        assert torch.equal(cv.c[0], cvs[0].c[0])
    np.testing.assert_allclose(cvs[0].c[0].double().cpu().numpy(), c_ref, rtol=1e-4, atol=1e-4)
    cis = [cvs[ck % W].cis[0][ck // W] for ck in range(K)]
    ds = [cvs[ck % W].ds[0][ck // W] for ck in range(K)]
    for ci, want in zip(cis, cis_ref):
        np.testing.assert_allclose(ci.double().cpu().numpy(), want, rtol=1e-4, atol=1e-4)
    return cvs[0].c[0].clone(), [t.clone() for t in cis], [t.clone() for t in ds]


@pytest.mark.parametrize("W,per_rank", [(2, 1), (4, 1), (2, 2)])
@pytest.mark.parametrize("N", [5131, 295424])
def test_loopback_ranks_agree_one_and_two_shot(W, per_rank, N):
    one = _loopback(W, per_rank, "0", N)
    two = _loopback(W, per_rank, "1", N)
    assert torch.equal(one[0], two[0])
    for a, b in zip(one[1] + one[2], two[1] + two[2]):
        assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------ end to end
def _run(**kw):
    from federated_pytorch_test_b200.api import federated_multi

    base = dict(K=8, use_resnet=True, Nloop=2, Nadmm=2, max_minibatches=4, train_size=4096, test_size=256,
                check_results=False, save_model=False, graphs=True, partition="dirichlet", clients_per_round=4,
                dirichlet_alpha=1.0, default_batch=64, optimizer="sgd", lr=0.05, momentum=0.9, scaffold=True)
    lines = []
    eng = federated_multi.run(federated_multi.Config(**{**base, **kw}), log=lines.append)
    torch.cuda.synchronize()
    return eng, lines


def test_graphed_resnet18_run_captures_once_and_matches_eager(monkeypatch):
    from federated_pytorch_test_b200.algo.graphs import GraphedAdamStep

    captures = {}
    orig = GraphedAdamStep._capture

    def capture(self):
        key = (self.rep.ck, self.visit.lo, self.visit.hi, tuple(self.static[0].shape))
        captures[key] = captures.get(key, 0) + 1
        orig(self)

    monkeypatch.setattr(GraphedAdamStep, "_capture", capture)
    eng, fused = _run()
    monkeypatch.setattr(GraphedAdamStep, "_capture", orig)
    assert eng.coll.name == "fused" and eng.graph_replays > 0 and captures
    assert set(captures.values()) == {1}              # once per (replica, block, batch shape), over both loops
    eager, plain = _run(graphs=False)
    df = [float(l.rsplit("=", 1)[1]) for l in fused if l.startswith("dual (")]
    de = [float(l.rsplit("=", 1)[1]) for l in plain if l.startswith("dual (")]
    nvis = len(list(eng.task.visits(0)))
    assert len(df) == len(de) == 2 * 2 * nvis
    for a, b in zip(df, de):
        assert a == pytest.approx(b, rel=5e-2)
    for ra, rb in zip(eng.replicas, eager.replicas):
        wa, wb = ra.arenas["net"].data, rb.arenas["net"].data
        assert float((wa - wb).norm()) <= 5e-2 * float(wb.norm())


def test_launches_added_per_round_and_visit(monkeypatch):
    from federated_pytorch_test_b200.algo.engine import Engine

    # the derived-filter refresh at every visit covers the caches of every engine made in this process so far: not
    # counted, so that the two runs compare
    refresh = [0]
    orig = Engine._refresh_derived

    def counted(self):
        before = cuda_ops.launch_count()
        orig(self)
        refresh[0] += cuda_ops.launch_count() - before

    monkeypatch.setattr(Engine, "_refresh_derived", counted)
    kw = dict(K=4, Nloop=1, Nadmm=3, max_minibatches=2, clients_per_round=2)
    counts = []
    for flag in (False, True):
        refresh[0] = 0
        before = cuda_ops.launch_count()
        eng, _ = _run(**kw, scaffold=flag)
        counts.append((eng, cuda_ops.launch_count() - before - refresh[0]))
    (eng_off, off), (eng_on, on) = counts
    visits = len(list(eng_on.task.visits(0)))
    assert eng_on.aggregations_done == eng_off.aggregations_done == 3 * visits
    assert eng_on.graph_kernel_launches == eng_off.graph_kernel_launches
    assert on - off == 3 * eng_on.aggregations_done + visits
