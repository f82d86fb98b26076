"""``LBFGSNew`` — stochastic / full-batch L-BFGS with line searches.

Behavioural spec: /root/reference/src/lbfgsnew.py:9-765 (SURVEY §2.5): same
constructor signature, closure contract, termination tests, curvature-pair
rule, inter-batch (Welford) step bound, Armijo backtracking with the
negative-step probe (stochastic mode), Fletcher bracketing + zoom with
finite-difference directional derivatives (full-batch mode), and the same
``state_dict`` keys.

Implementation is new and flat-vector based:

* the parameter list is addressed as ONE vector.  When the parameters live in a
  :class:`~..utils.flat.FlatArena` and form a contiguous index range (always
  the case for the block-coordinate trainers) the vector *is* the arena slice:
  the flat gradient is a zero-copy view, ``x += t*d`` is one axpy, and line
  searches snapshot/restore one buffer (the reference loops over tensors and
  ``torch.cat``s, lbfgsnew.py:81-121);
* curvature pairs live in two ``[history, n]`` ring buffers; the two-loop
  recursion, the pair update and the Welford update go through
  :mod:`..ops.flatops`, which on an H100 are fused sm_90a kernels with
  device-resident scalars (SURVEY G16) and otherwise ATen;
* every host decision of one inner iteration reads its scalars in one batch.

Scalar arithmetic that the reference performs on fp32 0-dim tensors is done in
``numpy.float32`` so branch decisions match it exactly.
"""
from __future__ import annotations

import math
from typing import Callable, List, Optional

import numpy as np
import torch
from torch.optim.optimizer import Optimizer

from ..ops import flatops
from ..utils.flat import arena_of

be_verbose = False
_f32 = np.float32


class _FlatVars:
    """The optimizer's parameters seen as one vector ``x`` with gradient ``g``."""

    def __init__(self, params: List[torch.Tensor]):
        self.params = params
        self.numel = sum(p.numel() for p in params)
        self.arena = None
        self.lo = self.hi = -1
        self._bind_arena()

    def _bind_arena(self) -> None:
        arena = None
        owner = getattr(self.params[0], "_arena_owner", None)
        if owner is not None:
            arena = owner
        if arena is None:
            return
        ids = {id(p): i for i, p in enumerate(arena.params)}
        idx = [ids.get(id(p), -1) for p in self.params]
        if -1 in idx or idx != list(range(idx[0], idx[0] + len(idx))):
            return
        if not arena.check_views():
            return
        self.arena, self.lo, self.hi = arena, idx[0], idx[-1]

    @property
    def fused(self) -> bool:
        return self.arena is not None

    # -- vector access ---------------------------------------------------
    def x(self) -> torch.Tensor:
        if self.fused:
            return self.arena.block(self.lo, self.hi)
        return torch.cat([p.data.reshape(-1) for p in self.params])

    def grad(self) -> torch.Tensor:
        """Flat gradient.  Arena: a fresh copy of the slice (the slice itself is
        overwritten by the next backward); otherwise gathered (zeros for None)."""
        if self.fused:
            self._ensure_attached()
            return self.arena.block_grad(self.lo, self.hi).clone()
        views = []
        for p in self.params:
            if p.grad is None:
                views.append(p.data.new_zeros(p.numel()))
            elif p.grad.is_sparse:
                views.append(p.grad.to_dense().reshape(-1))
            else:
                views.append(p.grad.reshape(-1))
        return torch.cat(views)

    def _ensure_attached(self) -> None:
        for i in range(self.lo, self.hi + 1):
            p = self.arena.params[i]
            if p.requires_grad and (p.grad is None or p.grad.data_ptr() != self.arena.grad_view(i).data_ptr()):
                g = self.arena.grad_view(i)
                if p.grad is not None:
                    g.copy_(p.grad)
                else:
                    g.zero_()
                p.grad = g

    def zero_grad(self) -> None:
        if self.fused:
            self._ensure_attached()
            self.arena.zero_grads(self.lo, self.hi)
        else:
            for p in self.params:
                if p.grad is not None:
                    p.grad.detach_()
                    p.grad.zero_()

    def axpy(self, alpha: float, d: torch.Tensor) -> None:
        """``x += alpha * d``"""
        alpha = float(alpha)
        if self.fused:
            self.arena.block(self.lo, self.hi).add_(d, alpha=alpha)
            return
        pos = 0
        for p in self.params:
            k = p.numel()
            p.data.add_(d[pos: pos + k].view_as(p.data), alpha=alpha)
            pos += k

    def snapshot(self) -> torch.Tensor:
        return self.x().clone()

    def restore(self, snap: torch.Tensor) -> None:
        if self.fused:
            self.arena.block(self.lo, self.hi).copy_(snap)
            return
        pos = 0
        for p in self.params:
            k = p.numel()
            p.data.copy_(snap[pos: pos + k].view_as(p.data))
            pos += k


class LBFGSNew(Optimizer):
    """L-BFGS (see module docstring).

    Arguments (identical to the reference, lbfgsnew.py:58-60):
        lr, max_iter, max_eval (default ``max_iter*5//4``), tolerance_grad,
        tolerance_change, history_size, line_search_fn (bool), batch_mode (bool).

    The closure must only call ``backward()`` when ``loss.requires_grad`` and
    guard ``zero_grad()`` with ``torch.is_grad_enabled()`` — line searches run
    it under ``no_grad``.
    """

    def __init__(self, params, lr=1, max_iter=10, max_eval=None,
                 tolerance_grad=1e-5, tolerance_change=1e-9, history_size=7,
                 line_search_fn=False, batch_mode=False):
        if max_eval is None:
            max_eval = max_iter * 5 // 4
        defaults = dict(lr=lr, max_iter=max_iter, max_eval=max_eval,
                        tolerance_grad=tolerance_grad, tolerance_change=tolerance_change,
                        history_size=history_size, line_search_fn=line_search_fn,
                        batch_mode=batch_mode)
        super().__init__(params, defaults)
        if len(self.param_groups) != 1:
            raise ValueError("LBFGSNew doesn't support per-parameter options (parameter groups)")
        self._params = self.param_groups[0]["params"]
        self._vars: Optional[_FlatVars] = None
        self._numel_cache = None

    # -- flat helpers (names kept from the reference for API familiarity) --
    def _v(self) -> _FlatVars:
        if self._vars is None:
            self._vars = _FlatVars(self._params)
        return self._vars

    def _numel(self) -> int:
        if self._numel_cache is None:
            self._numel_cache = sum(p.numel() for p in self._params)
        return self._numel_cache

    def _gather_flat_grad(self) -> torch.Tensor:
        return self._v().grad()

    def _add_grad(self, step_size, update) -> None:
        self._v().axpy(step_size, update)

    def _copy_params_out(self) -> torch.Tensor:
        return self._v().snapshot()

    def _copy_params_in(self, new_params: torch.Tensor) -> None:
        self._v().restore(new_params)

    def zero_grad(self, set_to_none: bool = False) -> None:  # keep arena views alive
        v = self._v()
        if v.fused or not set_to_none:
            v.zero_grad()
        else:
            super().zero_grad(set_to_none=True)

    # ------------------------------------------------------------------
    # stochastic mode: Armijo backtracking (+ negative step probe)
    # ------------------------------------------------------------------
    def _linesearch_backtrack(self, closure: Callable, pk: torch.Tensor, gk: torch.Tensor, alphabar) -> float:
        c1, max_halvings = 1e-4, 35
        state = self.state[self._params[0]]
        v = self._v()
        x0 = v.snapshot()
        alphabar = float(alphabar)

        f0 = float(closure())
        v.axpy(alphabar, pk)
        f_try = float(closure())
        # fp32 scalar pipeline of the reference: prodterm = c1*(g.p) is an fp32 tensor there
        slope = _f32(c1) * _f32(float(torch.dot(gk, pk)))

        def armijo_fails(f: float, a: float) -> bool:
            bound = _f32(f0) + _f32(a) * slope
            return math.isnan(f) or _f32(f) > bound

        halvings = 0
        a_pos = alphabar
        while halvings < max_halvings and armijo_fails(f_try, a_pos):
            a_pos *= 0.5
            v.restore(x0)
            v.axpy(a_pos, pk)
            f_try = float(closure())
            halvings += 1
        chosen = a_pos

        if _f32(f0 - f_try) < abs(slope):
            # insufficient decrease: probe the opposite direction with the same budget
            a_neg = -alphabar
            v.restore(x0)
            v.axpy(a_neg, pk)
            f_neg = float(closure())
            while halvings < max_halvings and armijo_fails(f_neg, a_neg):
                a_neg *= 0.5
                v.restore(x0)
                v.axpy(a_neg, pk)
                f_neg = float(closure())
                halvings += 1
            if f_neg < f_try:
                chosen = a_neg

        v.restore(x0)
        state["func_evals"] += halvings
        return chosen

    # ------------------------------------------------------------------
    # full-batch mode: Fletcher bracketing / zoom with central differences
    # ------------------------------------------------------------------
    class _Probe:
        """Evaluates phi(a)=f(x0+a*p) while tracking the current offset along ``p``."""

        def __init__(self, opt: "LBFGSNew", closure: Callable, x0: torch.Tensor, p: torch.Tensor, h: float):
            self.v, self.closure, self.x0, self.p, self.h = opt._v(), closure, x0, p, h

        def reset_to(self, a: float) -> None:
            self.v.restore(self.x0)
            self.v.axpy(a, self.p)

        def shift(self, da: float) -> None:
            self.v.axpy(da, self.p)

        def value(self) -> float:
            return float(self.closure())

        def slope_here(self, pre: float = 0.0) -> float:
            """Move by ``pre`` (folded into the first axpy, as the reference does), then take a
            central difference around that point; leaves the point at (a - h)."""
            self.shift(pre + self.h)
            up = self.value()
            self.shift(-2.0 * self.h)
            dn = self.value()
            return (up - dn) / (2.0 * self.h)

    def _linesearch_cubic(self, closure: Callable, pk: torch.Tensor, step: float) -> float:
        lr = self.param_groups[0]["lr"]
        a_first = 10 * lr
        sigma, rho_ls = 0.1, 0.01
        t1, t2, t3 = 9, 0.1, 0.5
        result = lr
        state = self.state[self._params[0]]
        x0 = self._v().snapshot()
        pr = LBFGSNew._Probe(self, closure, x0, pk, step)

        phi0 = pr.value()
        tol = min(phi0 * 0.01, 1e-6)
        dphi0 = pr.slope_here()
        if abs(dphi0) < 1e-12:
            return 1.0
        mu = (tol - phi0) / (rho_ls * dphi0)
        if math.isnan(mu):
            return 1.0

        evals = 3
        a_prev, a_cur = 0.0, a_first
        phi_prev = phi0
        for rnd in range(1, 4):
            pr.reset_to(a_cur)
            phi_cur = pr.value()
            if phi_cur < tol:
                result = a_cur
                break
            if phi_cur > phi0 + a_cur * dphi0 or (rnd > 1 and phi_cur >= phi_prev):
                result = self._linesearch_zoom(closure, x0, pk, a_prev, a_cur, phi0, dphi0, sigma, rho_ls, t1, t2, t3, step)
                break
            dphi_cur = pr.slope_here()
            if abs(dphi_cur) <= -sigma * dphi0:
                result = a_cur
                break
            if dphi_cur >= 0.0:
                result = self._linesearch_zoom(closure, x0, pk, a_cur, a_prev, phi0, dphi0, sigma, rho_ls, t1, t2, t3, step)
                break
            if mu <= 2.0 * a_cur - a_prev:
                a_prev, a_cur = a_cur, mu
            else:
                lo_pt = 2.0 * a_cur - a_prev
                hi_pt = min(mu, a_cur + t1 * (a_cur - a_prev))
                # NB: like the reference, a_prev is *not* advanced on this path
                a_cur = self._cubic_interpolate(closure, x0, pk, lo_pt, hi_pt, step)
            phi_prev = phi_cur
            evals += 3

        self._v().restore(x0)
        state["func_evals"] += evals
        return result

    def _cubic_interpolate(self, closure: Callable, xk: torch.Tensor, pk: torch.Tensor, a: float, b: float, step: float) -> float:
        """Minimiser of the cubic through (a, f, f') and (b, f, f'), clipped to the interval."""
        state = self.state[self._params[0]]
        pr = LBFGSNew._Probe(self, closure, xk, pk, step)
        pr.reset_to(a)
        fa = pr.value()
        dfa = pr.slope_here()              # now at a - step
        pr.shift(-a + step + b)            # -> b
        fb = pr.value()
        dfb = pr.slope_here()              # now at b - step
        evals = 6

        w = 3.0 * (fa - fb) / (b - a) + dfb - dfa
        disc = w * w - dfa * dfb
        if disc > 0.0:
            root = math.sqrt(disc)
            denom = dfb - dfa + 2.0 * root
            if denom == 0.0:
                return (a + b) * 0.5
            z0 = b - (dfb + root - w) * (b - a) / denom
            hi_end, lo_end = max(a, b), min(a, b)
            if z0 > hi_end or z0 < lo_end:
                fz = fa + fb
            else:
                # the reference moves to a + z0*(b-a) (not to z0) before evaluating; kept
                pr.shift(-b + step + a + z0 * (b - a))
                fz = pr.value()
                evals += 1
            state["func_evals"] += evals
            if fa < fb and fa < fz:
                return a
            if fb < fz:
                return b
            return z0
        state["func_evals"] += evals
        return a if fa < fb else b

    def _linesearch_zoom(self, closure, xk, pk, a, b, phi_0, gphi_0, sigma, rho, t1, t2, t3, step) -> float:
        state = self.state[self._params[0]]
        pr = LBFGSNew._Probe(self, closure, xk, pk, step)
        lo, hi = a, b
        evals = 0
        cand = None
        for _ in range(4):
            cand = self._cubic_interpolate(closure, xk, pk, lo + t2 * (hi - lo), hi - t3 * (hi - lo), step)
            pr.reset_to(cand)
            phi_c = pr.value()
            pr.shift(-cand + lo)
            phi_lo = pr.value()
            evals += 2
            if phi_c > phi_0 + rho * cand * gphi_0 or phi_c >= phi_lo:
                hi = cand
                continue
            dphi_c = pr.slope_here(pre=-lo + cand)
            evals += 2
            if (lo - cand) * dphi_c <= step or abs(dphi_c) <= -sigma * gphi_0:
                break
            if dphi_c * (hi - lo) >= 0.0:
                hi = lo
            lo = cand
        state["func_evals"] += evals
        return cand

    # ------------------------------------------------------------------
    def step(self, closure: Callable):
        assert len(self.param_groups) == 1
        group = self.param_groups[0]
        lr, max_iter, max_eval = group["lr"], group["max_iter"], group["max_eval"]
        tol_g, tol_x = group["tolerance_grad"], group["tolerance_change"]
        use_ls, m, batch_mode = group["line_search_fn"], group["history_size"], group["batch_mode"]
        v = self._v()

        state = self.state[self._params[0]]
        state.setdefault("func_evals", 0)
        state.setdefault("n_iter", 0)

        orig_loss = closure()
        loss = float(orig_loss.detach()) if torch.is_tensor(orig_loss) else float(orig_loss)
        evals_here = 1
        state["func_evals"] += 1

        g = v.grad()
        g_l1, g_l2 = flatops.l1_l2(g)          # one batched D2H read
        if g_l1 <= tol_g:
            return orig_loss

        d = state.get("d")
        t = state.get("t")
        hist: Optional[flatops.PairHistory] = state.get("_hist")
        H_diag = state.get("H_diag")
        g_prev = state.get("prev_flat_grad")
        prev_loss = state.get("prev_loss")
        run_mean = run_m2 = None
        alphabar = lr
        trust = 1e-6
        grad_nrm = g_l2                        # intentionally never refreshed (SURVEY Q16)

        inner = 0
        while inner < max_iter and not math.isnan(grad_nrm):
            inner += 1
            state["n_iter"] += 1
            first_ever = state["n_iter"] == 1

            if first_ever:
                d = g.neg()
                hist = flatops.PairHistory(m, g)
                H_diag = 1
                if batch_mode:
                    run_mean, run_m2 = torch.zeros_like(g), torch.zeros_like(g)
            else:
                if batch_mode:
                    run_mean, run_m2 = state.get("running_avg"), state.get("running_avg_sq")
                    if run_mean is None:
                        run_mean, run_m2 = torch.zeros_like(g), torch.zeros_like(g)
                if hist is None:  # e.g. after load_state_dict: rebuild the ring from the lists
                    hist = flatops.PairHistory(m, g)
                    for y_old, s_old in zip(state.get("old_dirs") or [], state.get("old_stps") or []):
                        hist.push(y_old, s_old)
                y, s, ys, sn, yy = flatops.make_pair(g, g_prev, d, float(t), trust if batch_mode else 0.0)
                new_batch = batch_mode and inner == 1 and state["n_iter"] > 1
                if new_batch:
                    m2_sum = flatops.welford_update(g, run_mean, run_m2, state["n_iter"])
                    alphabar = float(_f32(1) / (_f32(1) + _f32(m2_sum) / _f32((state["n_iter"] - 1) * grad_nrm)))
                    if be_verbose:
                        print("iter %d ||grad|| %f y^Ts %f alphabar=%f" % (state["n_iter"], grad_nrm, ys, alphabar))
                if _f32(ys) > _f32(1e-10 * sn * sn) and not new_batch:
                    hist.push(y, s)
                    H_diag = float(_f32(ys) / _f32(yy))
                if isinstance(H_diag, float) and math.isnan(H_diag):
                    print("Warning H_diag nan")
                d = hist.two_loop(g, H_diag)

            if g_prev is None:
                g_prev = g.clone()
            else:
                g_prev.copy_(g)
            prev_loss = loss

            if first_ever:
                t = min(1.0, float(_f32(1) / _f32(g_l1))) * lr
            else:
                t = lr

            gtd, d_l1 = flatops.dir_stats(g, d)      # one batched read; also feeds the step-size termination test below
            if math.isnan(gtd):
                print("Warning grad norm infinite")
                print("iter %d" % state["n_iter"])
                print("||grad||=%f" % grad_nrm)
                print("||d||=%f" % float(d.norm()))

            fresh = 0
            if use_ls:
                with torch.no_grad():
                    if batch_mode:
                        t = self._linesearch_backtrack(closure, d, g, alphabar)
                    else:
                        t = self._linesearch_cubic(closure, d, 1e-6)
                if math.isnan(t):
                    print("Warning: stepsize nan")
                    t = lr
                if be_verbose:
                    print("step size=%f" % t)
            v.axpy(t, d)

            if inner != max_iter:
                # re-evaluate (with gradient) unless this was the last inner iteration
                loss_t = closure()
                g = v.grad()
                loss, g_l1 = flatops.loss_and_l1(loss_t, g)      # one batched read
                if math.isnan(g_l1):
                    print("Warning: gradient nan")
                    break
                fresh = 1
            evals_here += fresh
            state["func_evals"] += fresh

            if inner == max_iter or evals_here >= max_eval:
                break
            if g_l1 <= tol_g or gtd > -tol_x:
                break
            if d_l1 * abs(t) <= tol_x:
                break
            if abs(loss - prev_loss) < tol_x:
                break

        state["d"], state["t"] = d, t
        state["_hist"] = hist
        state["old_dirs"] = hist.dirs() if hist is not None else []
        state["old_stps"] = hist.steps() if hist is not None else []
        state["H_diag"] = H_diag
        state["prev_flat_grad"] = g_prev
        state["prev_loss"] = prev_loss
        if hist is not None:
            state["ro"], state["al"] = hist.ro_list(), hist.al_list()
        if batch_mode:
            if run_mean is None:
                run_mean, run_m2 = torch.zeros_like(g), torch.zeros_like(g)
            state["running_avg"], state["running_avg_sq"] = run_mean, run_m2
        return orig_loss

    # -- true resume (utils/ckpt.py): everything step() carries between calls, as plain CPU tensors ----------------
    def flat_state(self) -> dict:
        st = self.state[self._params[0]]
        hist = st.get("_hist")
        out = {k: st.get(k) for k in ("func_evals", "n_iter", "t", "H_diag", "prev_loss")}
        for k in ("d", "prev_flat_grad", "running_avg", "running_avg_sq"):
            v = st.get(k)
            out[k] = v.detach().cpu().clone() if torch.is_tensor(v) else None
        if hist is not None:
            out["hist_Y"] = torch.stack([y.detach().cpu() for y in hist.dirs()]) if len(hist) else None
            out["hist_S"] = torch.stack([x.detach().cpu() for x in hist.steps()]) if len(hist) else None
            out["hist_m"] = hist.m
        return out

    def load_flat_state(self, rec: dict) -> None:
        st = self.state[self._params[0]]
        dev = self._params[0].device
        for k in ("func_evals", "n_iter", "t", "H_diag", "prev_loss"):
            if rec.get(k) is not None:
                st[k] = rec[k]
        for k in ("d", "prev_flat_grad", "running_avg", "running_avg_sq"):
            if rec.get(k) is not None:
                st[k] = rec[k].to(dev)
        if rec.get("hist_m") is not None and st.get("d") is not None:
            hist = flatops.PairHistory(int(rec["hist_m"]), st["d"])
            if rec.get("hist_Y") is not None:
                for y, x in zip(rec["hist_Y"], rec["hist_S"]):
                    hist.push(y.to(dev), x.to(dev))
            st["_hist"] = hist

    def state_dict(self):
        sd = super().state_dict()
        # the ring-buffer object is an implementation detail; ``old_dirs``/``old_stps`` carry the data
        sd["state"] = {k: {kk: vv for kk, vv in st.items() if kk != "_hist"} for k, st in sd["state"].items()}
        return sd
