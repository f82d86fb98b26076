"""Every entry point end to end on the GPU through the fast path (fused collectives, sm_90a kernels, CUDA graphs
where applicable).  Small configurations; the point is coverage of the CUDA code paths of all seven drivers."""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("CUDA device required", allow_module_level=True)

from federated_pytorch_test_b200.api import (consensus_multi, federated_cpc, federated_multi, federated_vae,  # noqa: E402
                                             federated_vae_cl, fedprox_multi, no_consensus_multi)
from federated_pytorch_test_b200.ops import cuda_ops  # noqa: E402

TINY = dict(train_size=2048, test_size=256, save_model=False, fast=True, collective="fused", distributed=False)


def _run(mod, **kw):
    lines = []
    eng = mod.run(mod.Config(**{**TINY, **kw}), log=lines.append)
    torch.cuda.synchronize()
    return eng, lines


def _finite(lines, prefix):
    vals = [float(l.rsplit("=", 1)[1]) for l in lines if l.startswith(prefix)]
    assert vals and all(v == v and abs(v) < 1e30 for v in vals), vals
    return vals


def test_no_consensus_resnet_accuracy_improves():
    eng, lines = _run(no_consensus_multi, K=2, Nepoch=3, max_minibatches=12, check_results=True, model="ResNet9",
                      default_batch=64, graphs=True)
    acc = [float(l.split("%")[-1]) for l in lines if l.startswith("Accuracy of the network 0")]
    assert len(acc) == 3 and acc[-1] > 25.0, acc       # learnable synthetic data: well above the 10 % chance level


def test_consensus_admm_bb_resnet_fused():
    before = cuda_ops.launch_count()
    eng, lines = _run(consensus_multi, K=2, Nloop=1, Nadmm=3, max_minibatches=3, check_results=False, model="ResNet9",
                      default_batch=32, bb_update=True, graphs=True)
    duals = [l for l in lines if l.startswith("block=[")]
    assert len(duals) == 8 * 3 and any(l.startswith("admm 2 deltas=(") for l in lines)
    # 8 warm-up launches at engine construction; per block: x0 seed + 3 aggregations + 1 BB update
    assert eng.coll.name == "fused" and eng.coll.launches - 8 == 8 * 5 and cuda_ops.launch_count() > before


def test_fedprox_lbfgs_resnet():
    """Benchmark configuration 4 (fedprox_multi + LBFGSNew, bench.py) in miniature."""
    eng, lines = _run(fedprox_multi, K=2, Nloop=1, Nadmm=1, max_minibatches=1, check_results=False, model="ResNet9",
                      default_batch=32, optimizer="lbfgs", graphs=False)
    assert len([l for l in lines if l.startswith("block=[")]) == 8
    for l in lines:
        if l.startswith("block=["):
            p, d = l.split("primal=")[1].split(" dual=")
            assert float(p) == float(p) and float(d) == float(d)


def test_lbfgs_graphed_closure_equals_eager():
    """The L-BFGS closure replayed from CUDA graphs (gradient evaluation + line-search probe).  (a) On identical state a replay
    and an eager evaluation give the same loss pair and the same block gradient; (b) a whole run walks the same iterates as
    the eager run up to what L-BFGS makes of float-atomic summation order (two eager runs differ by the same amount)."""
    kw = dict(K=2, Nloop=1, Nadmm=2, max_minibatches=4, check_results=False, model="Net", default_batch=32, optimizer="lbfgs")
    ea, a = _run(fedprox_multi, **kw, graphs=False)
    ea2, a2 = _run(fedprox_multi, **kw, graphs=False)
    eb, b = _run(fedprox_multi, **kw, graphs=True)
    assert eb.graph_replays > 0 and ea.graph_replays == 0

    def residuals(lines):
        return [tuple(float(v) for v in l.split("primal=")[1].split(" dual=")) for l in lines if l.startswith("block=[")]

    ra, ra2, rb = residuals(a), residuals(a2), residuals(b)
    assert len(ra) == len(rb) == 5 * 2
    spread = max(abs(u - v) / max(abs(u), 1e-12) for x, y in zip(ra, ra2) for u, v in zip(x, y))     # eager vs eager
    print("eager-vs-eager relative spread of the residuals: %.2e" % spread)
    for (pa, da), (pb, db) in zip(ra, rb):
        assert pa == pytest.approx(pb, rel=max(5e-2, 5 * spread), abs=1e-7) and da == pytest.approx(db, rel=max(5e-2, 5 * spread), abs=1e-7)
    # (a): same state, replay vs eager body
    ident, gc_ = eb._graphs[("lbfgs", eb.replicas[0].ck)]
    assert gc_.graph[True] is not None and gc_.graph[False] is not None
    g = gc_.rep.block_grad(gc_.visit)
    for with_grad in (True, False):
        out_graph = gc_.evaluate(with_grad).clone()
        g_graph = g.clone()
        with torch.enable_grad() if with_grad else torch.no_grad():
            out_eager = gc_._body(with_grad).clone()
        torch.testing.assert_close(out_graph, out_eager, rtol=1e-5, atol=1e-6)
        if with_grad:
            torch.testing.assert_close(g_graph, g.clone(), rtol=1e-4, atol=1e-6)


def test_federated_vae_and_vae_cl_and_cpc(tmp_path):
    eng, lines = _run(federated_vae, K=2, Nloop=1, Nadmm=1, max_minibatches=2, be_verbose=False, graphs=True)
    _finite(lines, "dual (")
    eng, lines = _run(federated_vae_cl, K=2, Nloop=1, Nadmm=1, max_minibatches=1, be_verbose=False, default_batch=32,
                      Kc=4, Lc=8, graphs=False)
    assert len(_finite(lines, "dual (")) == 3
    eng, lines = _run(federated_vae_cl, K=2, Nloop=1, Nadmm=1, max_minibatches=4, be_verbose=False, default_batch=32,
                      Kc=4, Lc=8, graphs=True)          # L-BFGS closures (encoder / decoder blocks) replayed from CUDA graphs
    assert len(_finite(lines, "dual (")) == 3 and eng.graph_replays > 0
    cfg = federated_cpc.Config(K=2, Lc=64, Rc=16, batch_size=8, Niter=2, load_model=False, init_model=True,
                               save_model=False, be_verbose=False, nbase=16, ckpt_dir=str(tmp_path), fast=True,
                               collective="fused", distributed=False, graphs=False)
    lines = []
    federated_cpc.run(cfg, log=lines.append)
    assert len(_finite(lines, "dual (N=")) == 4
    cfg.graphs, cfg.Niter = True, 4
    lines = []
    eng = federated_cpc.run(cfg, log=lines.append)
    assert len(_finite(lines, "dual (N=")) == 4 and eng.graph_replays > 0


def test_federated_multi_fused_equals_torch_collective():
    """Same run with the fused NVLink-kernel aggregation and with the ATen/NCCL baseline collective."""
    kw = dict(K=3, Nloop=1, Nadmm=2, max_minibatches=2, check_results=False, model="Net", graphs=False)
    _, a = _run(federated_multi, **kw)
    _, b = _run(federated_multi, **{**kw, "collective": "torch"})
    da, db = _finite(a, "dual ("), _finite(b, "dual (")
    assert len(da) == len(db) == 10
    for x, y in zip(da, db):
        assert x == pytest.approx(y, rel=2e-3)


def test_true_resume_record_roundtrip(tmp_path):
    from federated_pytorch_test_b200.utils import ckpt
    eng, _ = _run(consensus_multi, K=2, Nloop=1, Nadmm=1, max_minibatches=1, check_results=False, model="Net", graphs=False)
    path = ckpt.save_resume(str(tmp_path / "resume.pt"), eng, {"nloop": 0, "visit": 4, "round": 1})
    arena = eng.replicas[0].arenas["net"]
    before = arena.data.clone()
    with torch.no_grad():
        for p in eng.replicas[0].nets["net"].parameters():   # perturb parameters only: alignment gaps must stay zero
            p.add_(1.0)
    rec = ckpt.load_resume(str(tmp_path / "resume.pt"), eng)
    assert rec["position"]["visit"] == 4 and rec["strategy"] == "admm" and "rho" in rec["strategy_state"]
    torch.testing.assert_close(arena.data, before)
    assert os.path.exists(path)
