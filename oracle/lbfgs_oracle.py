"""TEST INFRASTRUCTURE -- CPU restatement of the reference optimiser loop for ONE
frame: L-BFGS with strong-Wolfe cubic line search (code/optimizers/lbfgs_ls.py)
driven by FittingMonitor.run_fitting (code/utils/fitting.py:71-142).

The restatement works on a flat parameter vector and a callable
`fg(x) -> (loss: float, grad: tensor)` instead of nn.Parameters + closure, but it
keeps the reference's arithmetic types (fp32 0-dim tensors for dot products,
Python floats for losses) and every branch, so that iterates match the reference
when both are given the same closure.  Pinned by tests/test_oracle_vs_reference.py.

Counters follow BASELINE.md section 3: an *iteration* is one pass of the
`while n_iter < max_iter` body (lbfgs_ls.py:304-434), an *eval* is one closure call.
"""
from __future__ import annotations

import numpy as np
import torch


def _margin(a, b):
    """relative distance of the two sides of a comparison (how far a decision lies from its threshold); None when a side
    is not finite (a comparison with Inf or NaN is not decided by rounding)"""
    a, b = float(a), float(b)
    if not (np.isfinite(a) and np.isfinite(b)):
        return None
    den = max(abs(a), abs(b))
    return abs(a - b) / den if den > 0 else 0.0


def _sign_margin(v, scale):
    """distance of a sign test on v (v >= 0) from its threshold, relative to the scale of the operands v came from"""
    v, scale = float(v), float(scale)
    if not (np.isfinite(v) and np.isfinite(scale)):
        return None
    return abs(v) / scale if scale > 0 else 0.0


def _mn(*ms):
    """the smallest of the margins that are not None (None if all are)"""
    ms = [m for m in ms if m is not None]
    return min(ms) if ms else None


def cubic_min(x1, f1, g1, x2, f2, g2, bounds=None, log=None):
    """lbfgs_ls.py:11-36.  log: optional list; with bounds (the bracket phase) the branch taken is appended as
    (name, margin): 'cubic_mid' (d2^2 < 0), 'clamp_lo' / 'clamp_hi' (the minimiser clamped to a bound) or 'cubic_free'."""
    if bounds is not None:
        lo, hi = bounds
    else:
        lo, hi = (x1, x2) if x1 <= x2 else (x2, x1)
    d1 = g1 + g2 - 3 * (f1 - f2) / (x1 - x2)
    sq = d1 ** 2 - g1 * g2
    if sq >= 0:
        d2 = sq.sqrt() if torch.is_tensor(sq) else sq ** 0.5
        if x1 <= x2:
            pos = x2 - (x2 - x1) * ((g2 + d2 - d1) / (g2 - g1 + 2 * d2))
        else:
            pos = x1 - (x1 - x2) * ((g1 + d2 - d1) / (g1 - g2 + 2 * d2))
        if log is not None and bounds is not None:
            m_sq = _margin(d1 ** 2, g1 * g2)
            if float(pos) < float(lo):
                log.append(("clamp_lo", _mn(m_sq, _margin(pos, lo))))
            elif float(pos) > float(hi):
                log.append(("clamp_hi", _mn(m_sq, _margin(pos, hi))))
            else:
                log.append(("cubic_free", _mn(m_sq, _margin(pos, lo), _margin(pos, hi))))
        return min(max(pos, lo), hi)
    if log is not None and bounds is not None:
        log.append(("cubic_mid", _margin(d1 ** 2, g1 * g2)))
    return (lo + hi) / 2.


def strong_wolfe(phi, t, d, f, g, gtd, c1=1e-4, c2=0.9, tol_change=1e-9, max_iter=20, max_ls=25, log=None):
    """lbfgs_ls.py:39-167.  `phi(t) -> (f_new: float, g_new: tensor)` evaluates the
    closure at x + t*d (lbfgs_ls.py:249-254).

    log: optional list.  Every branch taken is appended as (name, margin), margin being the relative distance of the
    comparisons that decided it from their thresholds (sign tests: relative to the scale of their operands; None for
    decisions on integers or on non-finite values); the arithmetic is unchanged."""
    rec = log.append if log is not None else (lambda e: None)
    d_norm = d.abs().max()
    g = g.clone()
    f_new, g_new = phi(t)
    evals = 1
    gtd_new = g_new.dot(d)
    t_prev, f_prev, g_prev, gtd_prev = 0, f, g, gtd
    done = False
    it = 0
    br = None
    while it < max_ls:
        arm = f + c1 * t * gtd
        m_arm = _margin(f_new, arm)
        if f_new > arm or (it > 1 and f_new >= f_prev):
            rec(("armijo_fail", m_arm) if f_new > arm else ("ls_f_prev", _mn(m_arm, _margin(f_new, f_prev))))
            br = ([t_prev, t], [f_prev, f_new], [g_prev, g_new.clone()], [gtd_prev, gtd_new])
            break
        m_arm = _mn(m_arm, _margin(f_new, f_prev)) if it > 1 else m_arm
        m_curv = _mn(m_arm, _margin(abs(gtd_new), -c2 * gtd))
        if abs(gtd_new) <= -c2 * gtd:
            rec(("wolfe_first" if it == 0 else "wolfe_bracket", m_curv))
            br = ([t], [f_new], [g_new], [gtd_new])
            done = True
            break
        m_pos = _mn(m_curv, _sign_margin(gtd_new, g_new.abs().max() * d_norm * d.numel()))
        if gtd_new >= 0:
            rec(("gtd_new_pos", m_pos))
            br = ([t_prev, t], [f_prev, f_new], [g_prev, g_new.clone()], [gtd_prev, gtd_new])
            break
        rec(("extrapolate", m_pos))
        lo_step = t + 0.01 * (t - t_prev)
        hi_step = t * 10
        keep = t
        t = cubic_min(t_prev, f_prev, gtd_prev, t, f_new, gtd_new, bounds=(lo_step, hi_step), log=log)
        t_prev, f_prev, g_prev, gtd_prev = keep, f_new, g_new.clone(), gtd_new
        f_new, g_new = phi(t)
        evals += 1
        gtd_new = g_new.dot(d)
        it += 1
    if it == max_ls:
        rec(("max_ls", None))
        br = ([0, t], [f, f_new], [g, g_new], [gtd, gtd_new])
    bt, bf, bg, bgtd = br
    stalled = False
    lo, hi = (0, 1) if bf[0] <= bf[-1] else (1, 0)
    while not done and it < max_iter:
        t = cubic_min(bt[0], bf[0], bgtd[0], bt[1], bf[1], bgtd[1])
        eps = 0.1 * (max(bt) - min(bt))
        m_eps = _margin(min(max(bt) - t, t - min(bt)), eps)
        if min(max(bt) - t, t - min(bt)) < eps:
            m_in = _mn(m_eps, _margin(t, max(bt)), _margin(t, min(bt)))
            if stalled or t >= max(bt) or t <= min(bt):
                rec(("insuf_move", _mn(m_in, _margin(abs(t - max(bt)), abs(t - min(bt))))))
                if abs(t - max(bt)) < abs(t - min(bt)):
                    t = max(bt) - eps
                else:
                    t = min(bt) + eps
                stalled = False
            else:
                rec(("insuf_set", m_in))
                stalled = True
        else:
            rec(("zoom_interp", m_eps))
            stalled = False
        f_new, g_new = phi(t)
        evals += 1
        gtd_new = g_new.dot(d)
        it += 1
        arm = f + c1 * t * gtd
        m_arm = _mn(_margin(f_new, arm), _margin(f_new, bf[lo]))
        if f_new > arm or f_new >= bf[lo]:
            bt[hi], bf[hi], bg[hi], bgtd[hi] = t, f_new, g_new.clone(), gtd_new
            lo0 = lo
            lo, hi = (0, 1) if bf[0] <= bf[1] else (1, 0)
            rec(("zoom_armijo_fail", m_arm))
            if lo != lo0:
                rec(("zoom_swap", _margin(bf[0], bf[1])))
        else:
            m_curv = _mn(m_arm, _margin(abs(gtd_new), -c2 * gtd))
            if abs(gtd_new) <= -c2 * gtd:
                rec(("zoom_done_curv", m_curv))
                done = True
            elif gtd_new * (bt[hi] - bt[lo]) >= 0:
                rec(("zoom_flip", _mn(m_curv, _sign_margin(gtd_new, g_new.abs().max() * d_norm * d.numel()))))
                bt[hi], bf[hi], bg[hi], bgtd[hi] = bt[lo], bf[lo], bg[lo], bgtd[lo]
            else:
                rec(("zoom_keep", _mn(m_curv, _sign_margin(gtd_new, g_new.abs().max() * d_norm * d.numel()))))
            bt[lo], bf[lo], bg[lo], bgtd[lo] = t, f_new, g_new.clone(), gtd_new
        if abs(bt[1] - bt[0]) * d_norm < tol_change:
            rec(("zoom_tol_change", _margin(abs(bt[1] - bt[0]) * d_norm, tol_change)))
            break
    if not done and it >= max_iter and abs(bt[1] - bt[0]) * d_norm >= tol_change:
        rec(("zoom_max_iter", None))
    return bf[lo], bg[lo], bt[lo], evals


class LBFGSOracle:
    """lbfgs_ls.py:172-445 with line_search_fn='strong_Wolfe' (optim_factory.py:50-52)."""

    def __init__(self, x0: torch.Tensor, fg, lr=1.0, max_iter=30, max_eval=None,
                 tolerance_grad=1e-5, tolerance_change=1e-9, history_size=100, log=None):
        """log: optional list that step(), strong_wolfe and run_fitting append every branch they take to, as
        (name, margin) (see strong_wolfe), and ("eval", kind) before every closure call (kind: 'entry', 'ls');
        the arithmetic is unchanged."""
        self.x = x0.clone()
        self.log = log
        self.fg = fg
        self.lr, self.max_iter = lr, max_iter
        self.max_eval = max_eval if max_eval is not None else max_iter * 5 // 4
        self.tol_g, self.tol_c, self.hist = tolerance_grad, tolerance_change, history_size
        self.st = dict(func_evals=0, n_iter=0)
        self.last_grad = None            # what p.grad holds after step() (the last closure call)
        self.iters = 0
        self.evals = 0
        self.trial_t = []                # the step length of every line-search evaluation

    def _rec(self, e):
        if self.log is not None:
            self.log.append(e)

    def _eval(self, x, kind="ls"):
        self._rec(("eval", kind))
        f, g = self.fg(x)
        self.evals += 1
        self.last_grad = g.clone()
        return float(f), g

    def step(self):
        st = self.st
        loss, flat_grad = self._eval(self.x, "entry")
        orig_loss = loss
        current_evals = 1
        st["func_evals"] += 1
        m_g = _margin(flat_grad.abs().max(), self.tol_g)
        if flat_grad.abs().max() <= self.tol_g:
            self._rec(("exit_entry", m_g))
            return orig_loss
        d, t = st.get("d"), st.get("t")
        old_dirs, old_stps, ro = st.get("old_dirs"), st.get("old_stps"), st.get("ro")
        H_diag, prev_flat_grad, prev_loss = st.get("H_diag"), st.get("prev_flat_grad"), st.get("prev_loss")
        n_iter = 0
        while n_iter < self.max_iter:
            n_iter += 1
            st["n_iter"] += 1
            self.iters += 1
            if st["n_iter"] == 1:
                d = flat_grad.neg()
                old_dirs, old_stps, ro = [], [], []
                H_diag = 1
            else:
                y = flat_grad.sub(prev_flat_grad)
                s = d.mul(t)
                ys = y.dot(s)
                self._rec(("push" if ys > 1e-10 else "skip", _margin(ys, 1e-10)))
                if ys > 1e-10:
                    if len(old_dirs) == self.hist:
                        self._rec(("drop_oldest", None))
                        old_dirs.pop(0); old_stps.pop(0); ro.pop(0)
                    old_dirs.append(y); old_stps.append(s); ro.append(1. / ys)
                    H_diag = (ys / y.dot(y)) * 1.
                k = len(old_dirs)
                al = [None] * k
                q = flat_grad.neg()
                for i in range(k - 1, -1, -1):
                    al[i] = old_stps[i].dot(q) * ro[i]
                    q.add_(old_dirs[i], alpha=-float(al[i]))
                d = r = torch.mul(q, H_diag)
                for i in range(k):
                    be = old_dirs[i].dot(r) * ro[i]
                    r.add_(old_stps[i], alpha=float(al[i] - be))
            prev_flat_grad = flat_grad.clone() if prev_flat_grad is None else prev_flat_grad.copy_(flat_grad)
            prev_loss = loss
            if st["n_iter"] == 1:
                inv = 1. / flat_grad.abs().sum()
                self._rec(("t_first_inv" if inv < 1. else "t_first_one", _margin(inv, 1.)))
                t = min(1., inv) * self.lr
            else:
                t = self.lr
            gtd = flat_grad.dot(d)
            m_gtd = _margin(gtd, -self.tol_c)
            if gtd > -self.tol_c:
                self._rec(("gtd_stop", m_gtd))
                break
            x0 = self.x.clone()

            def phi(tt, x0=x0, d=d):
                self.trial_t.append(float(tt))
                return self._eval(torch.add(x0, d, alpha=float(tt)))
            loss, flat_grad, t, ls_evals = strong_wolfe(phi, t, d, loss, flat_grad, gtd, max_iter=self.max_iter,
                                                        log=self.log)
            self.x = torch.add(x0, d, alpha=float(t))
            opt_cond = flat_grad.abs().max() <= self.tol_g
            current_evals += ls_evals
            st["func_evals"] += ls_evals
            if n_iter == self.max_iter:
                self._rec(("end_max_iter", None))
                break
            if current_evals >= self.max_eval:
                self._rec(("end_max_eval", None))
                break
            m_end = _margin(flat_grad.abs().max(), self.tol_g)
            if opt_cond:
                self._rec(("end_opt", m_end))
                break
            m_end = _mn(m_end, _margin(d.mul(t).abs().max(), self.tol_c))
            if d.mul(t).abs().max() <= self.tol_c:
                self._rec(("end_step_max", m_end))
                break
            m_end = _mn(m_end, _margin(abs(loss - prev_loss), self.tol_c))
            if abs(loss - prev_loss) < self.tol_c:
                self._rec(("end_dloss", m_end))
                break
            self._rec(("next_iter", m_end))
        st.update(d=d, t=t, old_dirs=old_dirs, old_stps=old_stps, ro=ro, H_diag=H_diag,
                  prev_flat_grad=prev_flat_grad, prev_loss=prev_loss)
        return orig_loss


PARAM_SEGMENTS = ((0, 10), (10, 13), (13, 82), (82, 85), (85, 86))


def run_fitting(opt: LBFGSOracle, maxiters=30, ftol=1e-9, gtol=1e-9, segments=PARAM_SEGMENTS):
    """fitting.py:71-142 (visualisation branch removed).  Returns (final prev_loss, outer steps).
    Note the gtol test is abs(max(grad)) per parameter tensor on the grads left by
    the LAST closure call (fitting.py:115-117)."""
    rec = opt.log.append if getattr(opt, "log", None) is not None else (lambda e: None)
    prev_loss = None
    n_done = 0
    for n in range(maxiters):
        loss = opt.step()
        n_done = n + 1
        if np.isnan(loss) or np.isinf(loss):
            rec(("mon_nan", None))
            break
        if n > 0 and prev_loss is not None and ftol > 0:
            rel = (prev_loss - loss) / max([abs(prev_loss), abs(loss), 1])      # utils/utils.py:348-349
            if rel <= ftol:
                rec(("mon_ftol", _margin(rel, ftol)))
                break
        g = opt.last_grad
        gm = [abs(float(g[a:b].max())) for a, b in segments]
        if all(v < gtol for v in gm):
            rec(("mon_gtol", _mn(*[_margin(v, gtol) for v in gm])))
            break
        prev_loss = loss
    else:
        rec(("mon_max_outer", None))
    return prev_loss, n_done
