"""SCAFFOLD control variates (algo/scaffold.py) on the CPU: configuration, the ATen path of the two per-round steps
against the float64 reference, drift correction on heterogeneous least squares, the engine against a float64 SCAFFOLD
loop with sampling and unequal local steps, equality with FedAvg while the control variates are 0, resume and gloo."""
import dataclasses
import json
import os

import numpy as np
import pytest
import torch
import torch.nn as nn

from federated_pytorch_test_b200.algo import scaffold as scaf
from federated_pytorch_test_b200.algo.engine import Engine, EngineConfig, Replica, Task, Visit
from federated_pytorch_test_b200.algo.sampling import participants, sample_key
from federated_pytorch_test_b200.algo.strategies import FedAvg, FedOpt
from federated_pytorch_test_b200.api import federated_multi
from federated_pytorch_test_b200.config import FederatedConfig, parse_config
from federated_pytorch_test_b200.ops import flatops
from federated_pytorch_test_b200.parallel import Topology, TorchCollective

TINY = dict(train_size=1024, test_size=128, save_model=False, graphs=False, fast=False)
KW = dict(K=2, Nloop=1, Nadmm=2, max_minibatches=2, check_results=False, use_cuda=False, model="Net")
SGD = dict(optimizer="sgd", lr=0.05, momentum=0.9, nesterov=True, weight_decay=5e-4)


def _run(**kw):
    lines = []
    eng = federated_multi.run(federated_multi.Config(**{**TINY, **kw}), log=lines.append)
    return eng, [l for l in lines if l.startswith("dual (")]


# ------------------------------------------------------------------------------------------------ configuration
def test_flag_parses_and_defaults_are_unchanged():
    cfg = parse_config(FederatedConfig, ["--scaffold", "--optimizer", "sgd", "--lr", "0.1"])
    assert cfg.scaffold and cfg.optimizer == "sgd"
    base = FederatedConfig()
    assert base.scaffold is False
    assert dataclasses.replace(base, scaffold=False) == base
    assert parse_config(FederatedConfig, []) == base


@pytest.mark.parametrize("kw,field", [
    (dict(optimizer="adam"), "optimizer"),
    (dict(optimizer="adamw", lr=1e-3), "optimizer"),
    (dict(optimizer="lbfgs"), "optimizer"),
    (dict(aggregator="median"), "aggregator"),
    (dict(dp_clip=0.1), "dp_clip"),
    (dict(compress_bits=8), "compress_bits"),
    (dict(secagg=True), "secagg"),
])
def test_rejected_combinations_name_the_field(kw, field):
    base = dict(K=4, scaffold=True, optimizer="sgd", lr=0.1)
    with pytest.raises(ValueError, match=field):
        FederatedConfig(**{**base, **kw})


def test_allowed_combinations():
    FederatedConfig(K=4, scaffold=True, optimizer="sgd", lr=0.1, momentum=0.9, nesterov=True, weight_decay=1e-4,
                    server_opt="avgm", server_momentum=0.0, clients_per_round=2, partition="dirichlet", clip_norm=1.0,
                    lr_schedule="cosine", byzantine=1)


def test_strategy_rejects_what_the_config_rejects():
    topo = Topology.single_process(4, "cpu")
    coll = TorchCollective(topo)
    with pytest.raises(ValueError, match="aggregator"):
        FedAvg(coll, topo, aggregator="median", scaffold=True)
    with pytest.raises(ValueError, match="compress_bits"):
        FedOpt(coll, topo, "adam", compress_bits=8, scaffold=True)


# ------------------------------------------------------------------------------------------------ steps 1-3
def test_aten_steps_match_the_float64_reference():
    K, n = 5, 1001
    g = torch.Generator().manual_seed(3)
    cis = [torch.randn(n, generator=g) for _ in range(K)]
    xs = [torch.randn(n, generator=g) for _ in range(K)]
    c, z = torch.randn(n, generator=g), torch.randn(n, generator=g)
    taus, lr = [3, 0, 7, 1, 0], 0.05
    want_cis, want_c, want_ds = scaf.reference_round([t.double().numpy() for t in cis], [t.double().numpy() for t in xs],
                                                     c.double().numpy(), z.double().numpy(), taus, lr)
    before = [t.clone() for t in cis]
    flatops.scaffold_cv_(cis, xs, c, z, [scaf.step_scale(t, lr) for t in taus])
    for j in (1, 4):                                   # sat out: bit for bit untouched
        assert torch.equal(cis[j], before[j])
    for j in (0, 2, 3):                                # the expression, rounded operation by operation
        s = torch.tensor(scaf.step_scale(taus[j], lr))
        assert torch.equal(cis[j], (before[j] - c) + s * (z - xs[j]))
    coll = TorchCollective(Topology.single_process(K, "cpu"))
    coll.average_(cis, c)
    ds = [torch.empty(n) for _ in range(K)]
    norm_sq = flatops.scaffold_corr_(cis, ds, c, flatops.scaffold_workspace(n, K, "cpu"))
    for j in range(K):
        np.testing.assert_allclose(cis[j].numpy(), want_cis[j], rtol=1e-5, atol=1e-4)
        np.testing.assert_allclose(ds[j].numpy(), want_ds[j], rtol=1e-5, atol=1e-4)
        assert torch.equal(ds[j], c - cis[j])
        assert float(norm_sq[j]) == pytest.approx(float(np.square(want_ds[j]).sum()), rel=1e-5)
    np.testing.assert_allclose(c.numpy(), want_c, rtol=1e-5, atol=1e-4)


def test_step_scale_is_float32_of_the_float64_reciprocal():
    assert scaf.step_scale(0, 0.1) == 0.0
    assert scaf.step_scale(7, 0.03) == float(np.float32(1.0 / (7 * 0.03)))


# ------------------------------------------------------------------------------------------------ least squares
D, M = 6, 24


def _clients(K: int, seed: int = 0):
    """Heterogeneous least-squares clients: differently scaled designs (different Hessians) and shifted targets."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for k in range(K):
        A = torch.randn(M, D, generator=g) * (0.5 + 0.5 * k)
        b = torch.randn(M, 1, generator=g) + 2.0 * k
        out.append((A, b))
    return out


def _objective(clients, w: np.ndarray, weights=None):
    """``F(w) = sum_k p_k f_k(w)``, ``f_k = ||A_k w - b_k||^2 / (2M)``: gradient at ``w`` and the minimiser (float64)."""
    weights = weights or [1.0 / len(clients)] * len(clients)
    H = sum(p * A.double().numpy().T @ A.double().numpy() / M for p, (A, _) in zip(weights, clients))
    r = sum(p * A.double().numpy().T @ b.double().numpy()[:, 0] / M for p, (A, b) in zip(weights, clients))
    return H @ w - r, np.linalg.solve(H, r)


class LSTask(Task):
    def __init__(self, clients, taus, lr):
        self.clients, self.taus, self.lr = clients, taus, lr

    def build_replica(self, ck, device, allocator):
        net = nn.Linear(D, 1, bias=False)
        with torch.no_grad():
            net.weight.zero_()
        return Replica(ck, {"net": net}, device, allocator)

    def visits(self, nloop):
        yield Visit("net", 0, 0, 0, (0, 0), "sgd", dict(lr=self.lr))

    def batches(self, rep, visit, epoch):
        return iter([self.clients[rep.ck]] * self.taus[rep.ck])

    def loss(self, rep, batch):
        A, b = batch
        return 0.5 * (rep.nets["net"](A) - b).square().mean()


def _ls_engine(K, taus, lr, rounds, **strat_kw):
    clients = _clients(K)
    topo = Topology.single_process(K, "cpu")
    coll = TorchCollective(topo)
    strat = FedAvg(coll, topo, **strat_kw)
    eng = Engine(LSTask(clients, taus, lr), topo, strat, coll, EngineConfig(Nloop=1, Nadmm=rounds, Nepoch=1),
                 log=lambda m: None)
    return eng, strat, clients


def _weights(eng):
    return eng.replicas[0].nets["net"].weight.detach().double().numpy()[0]


def test_scaffold_removes_client_drift_on_least_squares():
    K, tau, lr, R = 4, 10, 0.02, 150
    eng, _, clients = _ls_engine(K, [tau] * K, lr, R)
    eng.run()
    grad, w_star = _objective(clients, _weights(eng))
    assert np.linalg.norm(grad) > 0.05                       # FedAvg settles away from the global optimum
    eng, strat, _ = _ls_engine(K, [tau] * K, lr, R, scaffold=True)
    eng.run()
    w = _weights(eng)
    grad, _ = _objective(clients, w)
    assert np.linalg.norm(grad) < 1e-4
    np.testing.assert_allclose(w, w_star, rtol=0, atol=1e-4)
    for rep in eng.replicas[1:]:                              # the model was written back into every replica
        assert torch.equal(rep.nets["net"].weight, eng.replicas[0].nets["net"].weight)


def test_engine_matches_a_float64_scaffold_loop_with_sampling_and_unequal_steps():
    K, S, lr, R, seed = 4, 2, 0.02, 6, 11
    taus = [3, 5, 8, 4]
    n = [50, 10, 30, 20]
    eng, strat, clients = _ls_engine(K, taus, lr, R, clients_per_round=S, client_n=n, seed=seed, scaffold=True)
    eng.run()
    Ab = [(A.double().numpy(), b.double().numpy()[:, 0]) for A, b in clients]
    z, c = np.zeros(D), np.zeros(D)
    cis = [np.zeros(D) for _ in range(K)]
    for t in range(R):
        P = [int(k) for k in participants(sample_key(seed), t, K, S)]
        xs = [z.copy() for _ in range(K)]
        for k in P:
            A, b = Ab[k]
            for _ in range(taus[k]):
                xs[k] = xs[k] - lr * (A.T @ (A @ xs[k] - b) / M + (c - cis[k]))
        steps = [taus[k] if k in P else 0 for k in range(K)]
        cis, c, _ = scaf.reference_round(cis, xs, c, z, steps, lr)
        w = np.array([n[k] for k in P], dtype=np.float64)
        z = sum(wk / w.sum() * xs[k] for wk, k in zip(w, P))
    np.testing.assert_allclose(_weights(eng), z, rtol=1e-4, atol=1e-5)
    cv = strat.scaffold
    np.testing.assert_allclose(cv.c[0][:D].double().numpy(), c, rtol=1e-4, atol=1e-5)   # the weight leads the block
    for k in range(K):
        np.testing.assert_allclose(cv.cis[0][k][:D].double().numpy(), cis[k], rtol=1e-4, atol=1e-5)
        np.testing.assert_allclose(cv.ds[0][k][:D].double().numpy(), c - cis[k], rtol=1e-4, atol=1e-5)


# ------------------------------------------------------------------------------------------------ the driver
def test_first_round_with_zero_control_variates_equals_fedavg_bit_for_bit():
    kw = dict(KW, Nadmm=1, **SGD)
    eng_a, _ = _run(**kw)
    eng_b, _ = _run(**kw, scaffold=True)
    for ra, rb in zip(eng_a.replicas, eng_b.replicas):
        assert torch.equal(ra.arenas["net"].data, rb.arenas["net"].data)


def test_round_rows_carry_the_correction_norm(tmp_path):
    path = str(tmp_path / "m.jsonl")
    eng, lines = _run(**KW, **SGD, scaffold=True, metrics_path=path)
    rows = [json.loads(l) for l in open(path) if '"round"' in l]
    rows = [r for r in rows if r.get("kind") == "round"]
    assert len(rows) == len(lines) == 10
    assert all(np.isfinite(r["scaffold_corr"]) and r["scaffold_corr"] >= 0.0 for r in rows)
    assert any(r["scaffold_corr"] > 0.0 for r in rows)
    cv = eng.strategy.scaffold
    ci = rows[-1]["block"]
    want = np.mean([float((cv.c[ci] - t).double().norm()) for t in cv.cis[ci]])
    assert rows[-1]["scaffold_corr"] == pytest.approx(want, rel=1e-5)


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


def test_kill_and_resume_reproduces_the_trace_and_weights(tmp_path):
    kw = dict(KW, K=3, Nadmm=3, Nloop=2, **SGD, scaffold=True)
    eng, full = _run(**kw)
    assert len(full) == 30
    rec = str(tmp_path / "resume.pt")
    first = _killed_run({**kw, "resume_out": rec}, 6 * 3 * 5 + 9)     # round 1 of the second loop's first visit
    assert 0 < len(first) < 30 and os.path.exists(rec)
    st = torch.load(rec, weights_only=False)["strategy_state"]
    assert st["scaffold"] and len(st["scaffold_c"]) == 5            # every block of the first loop
    eng2, second = _run(**kw, resume=rec)
    assert first + second == full
    assert torch.equal(eng.replicas[0].arenas["net"].data, eng2.replicas[0].arenas["net"].data)
    cv, cv2 = eng.strategy.scaffold, eng2.strategy.scaffold
    for ci in cv.c:
        assert torch.equal(cv.c[ci], cv2.c[ci])
        for a, b in zip(cv.cis[ci], cv2.cis[ci]):
            assert torch.equal(a, b)


def test_resume_with_the_other_setting_raises(tmp_path):
    on, off = str(tmp_path / "on.pt"), str(tmp_path / "off.pt")
    _killed_run({**KW, **SGD, "scaffold": True, "resume_out": on}, 6)
    _killed_run({**KW, **SGD, "resume_out": off}, 6)
    with pytest.raises(ValueError, match="scaffold"):
        _run(**KW, **SGD, resume=on)
    with pytest.raises(ValueError, match="scaffold"):
        _run(**KW, **SGD, scaffold=True, resume=off)
    _run(**KW, **SGD, resume=off)                   # records written before the flag carry no key: resumed as off


DIST_KW = dict(KW, K=4, **SGD, scaffold=True, partition="dirichlet", clients_per_round=3)


def _dist_worker(rank, world, port, out):
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch.distributed as dist
    lines = []
    eng = federated_multi.run(federated_multi.Config(**DIST_KW, **TINY), log=lines.append)
    if rank == 0:
        torch.save({"lines": lines, "flat": eng.replicas[0].arenas["net"].data.clone(),
                    "c": {ci: c.clone() for ci, c in eng.strategy.scaffold.c.items()}}, out)
    dist.destroy_process_group()


def test_two_process_gloo_equals_single_process(tmp_path):
    import torch.multiprocessing as mp
    out = str(tmp_path / "r0.pt")
    port = 41500 + (os.getpid() % 2000)
    mp.spawn(_dist_worker, args=(2, port, out), nprocs=2, join=True)
    got = torch.load(out, weights_only=False)
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        os.environ.pop(k, None)
    eng, single = _run(**DIST_KW)
    multi = [l for l in got["lines"] if l.startswith("dual (")]
    assert len(single) == len(multi) == 10
    for a, b in zip(single, multi):
        assert a.split("=")[:-1] == b.split("=")[:-1]
        assert float(a.rsplit("=", 1)[1]) == pytest.approx(float(b.rsplit("=", 1)[1]), rel=1e-4)
    torch.testing.assert_close(got["flat"], eng.replicas[0].arenas["net"].data, rtol=1e-4, atol=1e-6)
    for ci, c in got["c"].items():
        torch.testing.assert_close(c, eng.strategy.scaffold.c[ci], rtol=1e-4, atol=1e-6)
