"""LBFGSNew against the original implementation (SURVEY §2.5, §4): its stored trajectories (tests/golden)."""
import warnings

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from federated_pytorch_test_b200.optim import LBFGSNew
from federated_pytorch_test_b200.utils import FlatArena

warnings.filterwarnings("ignore")


def _rosenbrock(cls, device="cpu"):
    x = nn.Parameter(torch.tensor([-1.2, 1.0], device=device))
    opt = cls([x], history_size=7, max_iter=100, line_search_fn=True, batch_mode=False)
    calls = [0]

    def closure():
        calls[0] += 1
        if torch.is_grad_enabled():
            opt.zero_grad()
        f = (1 - x[0]) ** 2 + 100 * (x[1] - x[0] ** 2) ** 2
        if f.requires_grad:
            f.backward()
        return f

    opt.step(closure)
    st = opt.state[opt._params[0]]
    return x.detach().clone(), calls[0], st["n_iter"], st["func_evals"]


def test_rosenbrock_golden():
    x, calls, iters, evals = _rosenbrock(LBFGSNew)
    torch.testing.assert_close(x, torch.tensor([1.0, 1.0]), atol=1e-5, rtol=0)
    assert (calls, iters) == (655, 31)  # the original LBFGSNew on this problem


def test_rosenbrock_identical_to_reference(golden):
    a, b = golden["lbfgs"]["rosenbrock"], _rosenbrock(LBFGSNew)
    assert torch.equal(a[0], b[0]) and tuple(a[1:]) == tuple(b[1:])


def _stochastic(cls, arena=False, steps=5, device="cpu"):
    torch.manual_seed(0)
    net = nn.Sequential(nn.Conv2d(3, 8, 3), nn.ELU(), nn.Flatten(), nn.Linear(8 * 30 * 30, 10)).to(device)
    if arena:
        FlatArena(net).attach_grads()
    opt = cls(net.parameters(), history_size=10, max_iter=4, line_search_fn=True, batch_mode=True)
    g = torch.Generator().manual_seed(1)
    log = []
    for _ in range(steps):
        xb, yb = torch.randn(32, 3, 32, 32, generator=g), torch.randint(0, 10, (32,), generator=g)
        xb, yb = xb.to(device), yb.to(device)
        cnt = [0, 0]

        def closure():
            if torch.is_grad_enabled():
                opt.zero_grad()
            loss = F.cross_entropy(net(xb), yb)
            cnt[0] += 1
            if loss.requires_grad:
                loss.backward()
                cnt[1] += 1
            return loss

        loss = opt.step(closure)
        log.append((float(loss), cnt[0], cnt[1]))
    vec = torch.cat([p.detach().reshape(-1) for p in net.parameters()]).cpu()
    return log, vec, opt


def test_stochastic_identical_to_reference(golden):
    a, b = golden["lbfgs"], _stochastic(LBFGSNew)
    assert [tuple(x) for x in a["stochastic_counts"]] == [x[1:] for x in b[0]]   # forward/backward counts per step
    # the whole iterate: bit-identical on the CPU the golden data was recorded on; on another CPU the float rounding of its
    # convolution kernels (~1e-7) is all that may differ
    torch.testing.assert_close(b[1], a["stochastic_vec"], rtol=1e-5, atol=1e-7)
    assert a["state_keys"] == sorted(b[2].state_dict()["state"][0].keys())


def test_stochastic_on_arena_close_to_reference(golden):
    a, c = golden["lbfgs"], _stochastic(LBFGSNew, arena=True)
    assert [tuple(x) for x in a["stochastic_counts"]] == [x[1:] for x in c[0]]
    torch.testing.assert_close(c[1], a["stochastic_vec"], rtol=1e-4, atol=1e-5)
    assert c[2]._v().fused


def _dense_bfgs_direction(pairs, g, hdiag):
    """``-H g`` with H built densely: ``H = hdiag I``, then for each ``(y, s)``, oldest first,
    ``H <- (I - rho s y^T) H (I - rho y s^T) + rho s s^T`` with ``rho = 1 / y.s``."""
    n = g.numel()
    eye = torch.eye(n, dtype=torch.float64)
    H = hdiag * eye
    for y, s in pairs:
        rho = 1.0 / float(y.dot(s))
        H = (eye - rho * torch.outer(s, y)) @ H @ (eye - rho * torch.outer(y, s)) + rho * torch.outer(s, s)
    return -(H @ g)


@pytest.mark.parametrize("m,pushes", [(4, 7), (4, 4), (1, 1), (1, 3), (6, 2), (5, 11)])
@pytest.mark.parametrize("hdiag", [1.0, 1e-3, 37.5])
def test_two_loop_equals_dense_bfgs(m, pushes, hdiag):
    """The float64 ATen two-loop recursion (the oracle of the CUDA kernel) is the BFGS inverse-Hessian update, also once
    the ring has wrapped and its rows are no longer in storage order."""
    from federated_pytorch_test_b200.ops import flatops

    n = 12
    gen = torch.Generator().manual_seed(m * 100 + pushes)
    hist = flatops.PairHistory(m, torch.zeros(n, dtype=torch.float64))
    pushed = []
    for _ in range(pushes):
        s = torch.randn(n, dtype=torch.float64, generator=gen)
        a = torch.randn(n, n, dtype=torch.float64, generator=gen)
        y = (a @ a.T / n + 0.1 * torch.eye(n, dtype=torch.float64)) @ s          # y = A s, A SPD: y.s > 0
        hist.push(y, s)
        pushed.append((y, s))
    kept = pushed[-m:]
    assert len(hist) == len(kept)
    if pushes > m and m > 1:
        assert hist.order != sorted(hist.order)
    g = torch.randn(n, dtype=torch.float64, generator=gen)
    d = hist.two_loop(g, hdiag)
    ref = _dense_bfgs_direction(kept, g, hdiag)
    assert float((d - ref).abs().max() / ref.abs().max()) < 1e-12
    # the pairs in storage order instead of age order give another matrix: the comparison sees the order
    if pushes > m and m > 1:
        wrong = _dense_bfgs_direction([(hist.Y[r], hist.S[r]) for r in range(m)], g, hdiag)
        assert float((wrong - ref).abs().max() / ref.abs().max()) > 1e-6


def test_state_dict_roundtrip():
    _, _, opt = _stochastic(LBFGSNew, steps=3)
    sd = opt.state_dict()
    assert "_hist" not in sd["state"][0]
    assert len(sd["state"][0]["old_dirs"]) > 0
    assert "_hist" in opt.state[opt._params[0]]  # live state untouched
