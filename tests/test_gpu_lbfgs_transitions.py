"""The device L-BFGS state machine (lbfgs_advance_core, mvs_lbfgs_core.cuh) transition by transition against float64.

The host drives the production lbfgs_advance_kernel through the testing aids mvs_debug_lbfgs_state / _advance: it evaluates
an analytic objective in float64 at the device's fp32 trial point, rounds f and g to fp32, hands them to the kernel and reads
the whole optimiser state back after every transition.  Every tight check is either

* stateless: one transition from a known state against float64 (ring bookkeeping bit for bit, ro and the block Gram within
  the dot-product error bound, the search direction within 4x the error of the textbook fp32 two-loop recursion), or
* bit-identical by construction: frames in a batch against the same frames alone, the frame-resident optimiser (regime A)
  against one LBFGS.step per call (regime C);

and the free-running comparison with the oracle L-BFGS (oracle/lbfgs_oracle.py, which restates lbfgs_ls.py) only uses short
runs on objectives whose branch decisions all lie at least 1e-4 (relative) from their thresholds; the test asserts that
margin from the oracle's branch log.  Run with -s to see the worst errors and the branches reached."""
import ctypes
import math

import numpy as np
import pytest
import torch

from mvsmplfitting_b200 import _lib
from mvsmplfitting_b200 import synthetic as S

NP = 86
PH_STEP_ENTRY, PH_LS_BRACKET, PH_LS_ZOOM, PH_DONE = 0, 1, 2, 3
U32 = 2.0 ** -24


def gamma(n):
    return n * U32 / (1 - n * U32)


_INTS = ("phase", "outer_n", "state_n_iter", "n_iter", "current_evals", "ls_iter", "ls_evals", "ls_first", "low", "high",
         "done", "insuf", "have_prev", "hist_len", "hist_head", "nan_flag", "pushed_slot", "stage", "stage_end", "nan_acc")
_FLOATS1 = ("t", "H_diag", "gtd0", "t_prev", "gtd_prev", "d_norm")
_FLOATS2 = ("loss", "prev_loss", "orig_loss", "f_prev", "mon_prev_loss", "final_loss")


class FrameScalars(ctypes.Structure):
    """host mirror of mvs::FrameScalars (mvs_lbfgs_core.cuh), checked against mvs_debug_lbfgs_layout"""
    _fields_ = ([(n, ctypes.c_int) for n in _INTS] + [(n, ctypes.c_float) for n in _FLOATS1] +
                [("bt", ctypes.c_float * 2), ("bgtd", ctypes.c_float * 2), ("bf", ctypes.c_float * 2)] +
                [(n, ctypes.c_float) for n in _FLOATS2] + [("iters", ctypes.c_longlong), ("evals", ctypes.c_longlong)])


def debug_lib():
    lib = _lib.load()
    vp, ci = ctypes.c_void_p, ctypes.c_int
    lib.mvs_debug_lbfgs_layout.argtypes = [vp]
    lib.mvs_debug_lbfgs_layout.restype = ci
    lib.mvs_debug_lbfgs_state.argtypes = [vp, ci, ci] + [vp] * 15
    lib.mvs_debug_lbfgs_state.restype = ci
    lib.mvs_debug_lbfgs_advance.argtypes = [vp, ctypes.POINTER(_lib.LbfgsConfig), ci, ci]
    lib.mvs_debug_lbfgs_advance.restype = ci
    return lib


def test_frame_scalars_mirror_matches_the_library():
    """CPU: sizeof(FrameScalars) and the offset of every field, as the library was compiled"""
    lib = debug_lib()
    n = lib.mvs_debug_lbfgs_layout(None)
    out = (ctypes.c_int * n)()
    assert lib.mvs_debug_lbfgs_layout(ctypes.cast(out, ctypes.c_void_p)) == n
    names = [f for f, _ in FrameScalars._fields_]
    assert n == 1 + len(names)
    assert out[0] == ctypes.sizeof(FrameScalars)
    assert [getattr(FrameScalars, f).offset for f in names] == list(out[1:])


# ------------------------------------------------------------------------------------------------ host-driven state machine
_ARRS = ("x", "g", "d", "prev_g", "x_init", "g_prev", "bg", "hist_s", "hist_y", "ro", "gram", "x_eval", "g_eval", "loss_eval")


class Machine:
    """the optimiser state of a context's B frames, read and written through mvs_debug_lbfgs_state"""

    def __init__(self, ctx, H):
        self.ctx, self.lib, self.B, self.H = ctx, debug_lib(), ctx.B, H
        B = self.B
        self.shapes = dict(x=(B, NP), g=(B, NP), d=(B, NP), prev_g=(B, NP), x_init=(B, NP), g_prev=(B, NP), bg=(B, 2, NP),
                           hist_s=(B, H, NP), hist_y=(B, H, NP), ro=(B, H), gram=(B, 16, 8, 8), x_eval=(B, NP),
                           g_eval=(B, NP), loss_eval=(B,))

    def _call(self, write, sc, arrs):
        p = lambda a: None if a is None else a.ctypes.data_as(ctypes.c_void_p)
        scp = None if sc is None else ctypes.cast(sc, ctypes.c_void_p)
        rc = self.lib.mvs_debug_lbfgs_state(self.ctx.h, write, self.H, scp, *[p(arrs.get(k)) for k in _ARRS])
        _lib.check(self.ctx.h, rc, "mvs_debug_lbfgs_state")

    def read(self):
        sc = (FrameScalars * self.B)()
        arrs = {k: np.zeros(self.shapes[k], np.float32) for k in _ARRS}
        self._call(0, sc, arrs)
        return sc, arrs

    def write(self, sc=None, **arrs):
        arrs = {k: np.ascontiguousarray(v, np.float32) for k, v in arrs.items()}
        for k, v in arrs.items():
            assert v.shape == self.shapes[k], k
        self._call(1, sc, arrs)

    def advance(self, cfg, step_mode=0, pose_len=69):
        _lib.check(self.ctx.h, self.lib.mvs_debug_lbfgs_advance(self.ctx.h, ctypes.byref(cfg), step_mode, pose_len),
                   "mvs_debug_lbfgs_advance")

    def start(self, x0, poison=True):
        """every frame a fresh optimiser at x0 [B][86] (lbfgs_init_kernel with reset); ring, ro and Gram poisoned with NaN"""
        sc = (FrameScalars * self.B)()
        for s in sc:
            s.phase, s.H_diag, s.final_loss, s.stage, s.stage_end = PH_STEP_ENTRY, 1.0, float("nan"), 0, 1
        z = lambda k: np.zeros(self.shapes[k], np.float32)
        fill = (lambda k: np.full(self.shapes[k], np.nan, np.float32)) if poison else z
        self.write(sc, x=x0, x_eval=x0, g=z("g"), d=z("d"), prev_g=z("prev_g"), x_init=z("x_init"), g_prev=z("g_prev"),
                   bg=z("bg"), hist_s=fill("hist_s"), hist_y=fill("hist_y"), ro=fill("ro"), gram=fill("gram"))


def lbfgs_cfg(H, max_outer=100000, max_iter=30, max_eval=None, lr=1.0, tol_grad=1e-5, tol_change=1e-9, ftol=0.0, gtol=0.0):
    return _lib.LbfgsConfig(int(max_outer), int(max_iter), int(max_eval if max_eval is not None else max_iter * 5 // 4),
                            int(H), float(lr), float(tol_grad), float(tol_change), float(ftol), float(gtol))


def f32(a):
    return np.asarray(a, np.float64).astype(np.float32)


# ------------------------------------------------------------------------------------------------ float64 references
def live_slots(hl, head, H):
    """ring slots of the stored pairs, oldest -> newest"""
    return [(head + k) % H for k in range(hl)]


def two_loop64(g, S_, Y_, H_diag):
    q = -np.asarray(g, np.float64)
    ro = [1.0 / np.dot(y, s) for s, y in zip(S_, Y_)]
    al = [0.0] * len(S_)
    for i in range(len(S_) - 1, -1, -1):
        al[i] = ro[i] * np.dot(S_[i], q)
        q -= al[i] * Y_[i]
    r = q * H_diag
    for i in range(len(S_)):
        be = ro[i] * np.dot(Y_[i], r)
        r += (al[i] - be) * S_[i]
    return r


def two_loop_textbook32(g, S_, Y_):
    """lbfgs_ls.py's sequential fp32 recursion (what the reference computes) on the same pairs"""
    q = -torch.tensor(g, dtype=torch.float32)
    Ss = [torch.tensor(s) for s in S_]
    Ys = [torch.tensor(y) for y in Y_]
    ro = [1.0 / y.dot(s) for s, y in zip(Ss, Ys)]
    H_diag = (Ys[-1].dot(Ss[-1]) / Ys[-1].dot(Ys[-1])) if Ss else 1.0
    al = [None] * len(Ss)
    for i in range(len(Ss) - 1, -1, -1):
        al[i] = Ss[i].dot(q) * ro[i]
        q.add_(Ys[i], alpha=-float(al[i]))
    r = torch.mul(q, H_diag)
    for i in range(len(Ss)):
        be = Ys[i].dot(r) * ro[i]
        r.add_(Ss[i], alpha=float(al[i] - be))
    return r.numpy().astype(np.float64)


class Worst:
    """largest error / bar ratio of each check (printed with -s)"""

    def __init__(self):
        self.v = {}

    def add(self, name, ratio):
        self.v[name] = max(self.v.get(name, 0.0), float(ratio))

    def report(self, tag):
        print("\n[%s] worst error / bar: %s" % (tag, ", ".join("%s %.3g" % kv for kv in sorted(self.v.items()))))


# Search direction bar: 4 x max(the error of the textbook fp32 recursion, D_FLOOR x |d64|_inf).  The floor is needed: the
# two recursions round differently, and on a given direction the textbook order's error is now and then far below its
# typical size (its rounding errors happen to cancel), so it alone is no yardstick there.  On the H100 the blocked
# recursion's error exceeded 4x the textbook error (by up to 8.7x) only on directions where it stayed below
# 5.1e-5 |d64|_inf, i.e. where the floor applies; a slot, Gram entry or coefficient read wrongly costs O(1) of |d64|_inf.
D_FACTOR = 4.0
D_FLOOR = 1e-4
GRAM_FACTOR = 2.0       # x gamma_86 sum |s_i| |y_j|
RO_FACTOR = 2.0


class RingChecker:
    """2(a) of the design: after every transition that began an iteration, the device's ring bookkeeping (exact), ro and the
    live block-Gram entries (float64 within the dot-product error bound) and the search direction (float64 two-loop
    recursion of the device's own stored pairs, bar: 4x the error of the textbook fp32 recursion)"""

    def __init__(self, H, B, worst):
        self.H, self.worst = H, worst
        self.pushes = [0] * B
        self.skips = [0] * B
        self.heads = [set() for _ in range(B)]

    def check(self, b, began, pre, post_s, post, t_used, pushed=None):
        """began: the transition pre -> post began an iteration (ITER_BEGIN ran).  pushed: None when the device's
        pushed_slot of this very transition says whether the pair was stored; "predict" when the transition spans several
        advances (one LBFGS.step per call): then the sign of y.s, which must lie clearly off the threshold, says so"""
        H = self.H
        s_new = post_s
        if not began or s_new.state_n_iter <= 1:
            assert pushed is not None or s_new.pushed_slot == -1
            return
        y = f32(post["g"][b].astype(np.float32) - pre["prev_g"][b])
        s = f32(pre["d"][b] * np.float32(t_used))
        ys = float(np.dot(y.astype(np.float64), s.astype(np.float64)))
        bound = gamma(NP) * float(np.dot(np.abs(y), np.abs(s)))
        clear = abs(ys - 1e-10) > 4 * bound + 1e-12             # the device's fp32 ys is on the same side of the threshold
        if pushed is None:
            pushed = s_new.pushed_slot >= 0
            if clear:
                assert pushed == (ys > 1e-10), (b, ys, bound)
        else:
            assert clear, (b, ys, bound)
            pushed = ys > 1e-10
        if pushed:
            self.pushes[b] += 1
        else:
            self.skips[b] += 1
        n = self.pushes[b]
        hl, head = min(n, H), ((n - H) % H if n > H else 0)
        assert (s_new.hist_len, s_new.hist_head) == (hl, head), (b, n, s_new.hist_len, s_new.hist_head)
        self.heads[b].add(head)
        slots = live_slots(hl, head, H)
        if pushed:
            assert s_new.pushed_slot in (-1, slots[-1])
            assert np.array_equal(post["hist_s"][b, slots[-1]].view(np.uint32), s.view(np.uint32))
            assert np.array_equal(post["hist_y"][b, slots[-1]].view(np.uint32), y.view(np.uint32))
        Sv = [post["hist_s"][b, w].astype(np.float64) for w in slots]
        Yv = [post["hist_y"][b, w].astype(np.float64) for w in slots]
        for k, w in enumerate(slots):
            ys_k = float(np.dot(Sv[k], Yv[k]))
            rb = RO_FACTOR * (gamma(NP) * float(np.dot(np.abs(Sv[k]), np.abs(Yv[k]))) / abs(ys_k) + 2 * U32) / abs(ys_k)
            err = abs(float(post["ro"][b, w]) - 1.0 / ys_k)
            self.worst.add("ro", err / rb)
            assert err <= rb, (b, w, err, rb)
        live = set(slots)
        gram = post["gram"][b]
        for i in slots:
            for j in slots:
                if i >> 3 != j >> 3:
                    continue
                ref = float(np.dot(post["hist_s"][b, i].astype(np.float64), post["hist_y"][b, j].astype(np.float64)))
                bar = GRAM_FACTOR * gamma(NP) * float(np.dot(np.abs(post["hist_s"][b, i]).astype(np.float64),
                                                             np.abs(post["hist_y"][b, j]).astype(np.float64))) + 1e-30
                err = abs(float(gram[i >> 3, i & 7, j & 7]) - ref)
                self.worst.add("gram", err / bar)
                assert err <= bar, (b, i, j, err, bar)
        assert live
        d = post["d"][b].astype(np.float64)
        g = post["prev_g"][b]                                   # the gradient the recursion started from
        assert np.isfinite(d).all(), b
        H_diag = float(np.dot(Sv[-1], Yv[-1]) / np.dot(Yv[-1], Yv[-1])) if slots else float(post_s.H_diag)
        d64 = two_loop64(g, Sv, Yv, H_diag)
        dtb = two_loop_textbook32(g, [post["hist_s"][b, w] for w in slots], [post["hist_y"][b, w] for w in slots])
        scale = float(np.abs(d64).max())
        bar = D_FACTOR * max(float(np.abs(dtb - d64).max()), D_FLOOR * scale)
        err = float(np.abs(d - d64).max())
        self.worst.add("d", err / bar)
        assert err <= bar, (b, len(slots), err, bar, scale)


# ------------------------------------------------------------------------------------------------ objectives
class QuadObjective:
    """0.5 (x-c)^T A (x-c) + beta sum log cosh x: A with 86 distinct curvatures 1 .. cond in a random basis.  At every
    step() boundary the target c moves (the curvature does not), every second time so that the next pair has y.s < 0
    (the pair is skipped)."""

    def __init__(self, seed, cond=1e4, beta=0.5):
        rng = np.random.default_rng(seed)
        Q, _ = np.linalg.qr(rng.standard_normal((NP, NP)))
        lam = np.geomspace(1.0, cond, NP)
        self.A = (Q * lam) @ Q.T
        self.c = rng.standard_normal(NP)
        self.beta = beta
        self.rng = rng
        self.k = 0

    def __call__(self, x):
        x = np.asarray(x, np.float64)
        r = x - self.c
        Ar = self.A @ r
        f = 0.5 * float(r @ Ar) + self.beta * float(np.sum(np.logaddexp(x, -x) - math.log(2.0)))
        return f, Ar + self.beta * np.tanh(x)

    def boundary(self, g, prev_g, d, t):
        """a new step() is about to evaluate its entry point"""
        self.k += 1
        s = f32(d * np.float32(t)).astype(np.float64)
        ss = float(s @ s)
        if self.k % 2 == 0 and ss > 0:
            ys0 = float((g.astype(np.float64) - prev_g) @ s)
            delta = -(2 * abs(ys0) + 1e-3 * math.sqrt(ss) * float(np.abs(g).max())) * s / ss
            self.c = self.c - np.linalg.solve(self.A, delta)
        else:
            self.c = self.c + 0.5 * self.rng.standard_normal(NP)


def drive(ctx, H, objs, x0, cfg, target_pushes, checker=None, trace=None, max_rounds=20000):
    """host loop: evaluate -> advance -> check, until every frame pushed target_pushes pairs (then it is parked as PH_DONE)"""
    m = Machine(ctx, H)
    B = ctx.B
    m.start(x0)
    pre_s, pre = m.read()
    done = [False] * B
    for _ in range(max_rounds):
        if all(done):
            break
        loss, ge = pre["loss_eval"].copy(), pre["g_eval"].copy()
        for b in range(B):
            if done[b]:
                continue
            s = pre_s[b]
            if s.phase == PH_STEP_ENTRY and s.state_n_iter > 0 and hasattr(objs[b], "boundary"):
                objs[b].boundary(pre["g"][b], pre["prev_g"][b], pre["d"][b], s.t)
            f, g = objs[b](pre["x_eval"][b])
            loss[b], ge[b] = np.float32(f), f32(g)
            if trace is not None:
                trace[b].append(pre["x_eval"][b].copy())
        m.write(loss_eval=loss, g_eval=ge)
        m.advance(cfg)
        post_s, post = m.read()
        park = False
        for b in range(B):
            if done[b]:
                continue
            t_used = post_s[b].bt[post_s[b].low] if pre_s[b].phase in (PH_LS_BRACKET, PH_LS_ZOOM) else pre_s[b].t
            if checker is not None:
                checker.check(b, post_s[b].iters != pre_s[b].iters, pre, post_s[b], post, t_used)
                if checker.pushes[b] >= target_pushes:
                    done[b] = park = True
                    post_s[b].phase = PH_DONE
            assert post_s[b].phase != PH_DONE or done[b], (b, "the frame finished before its ring wrapped")
        if park:
            m.write(post_s)
        pre_s, pre = post_s, post
    assert all(done)
    return pre_s, pre


HISTORIES = [1, 2, 7, 8, 9, 15, 16, 17, 63, 64, 65, 100, 101, 127, 128]


def _ctx(model, B):
    from mvsmplfitting_b200.context import FittingContext
    ctx = FittingContext(0)
    ctx.set_model(model)
    ctx.set_batch(B)
    return ctx


def _x0(B, seed):
    return f32(np.random.default_rng(seed).standard_normal((B, NP)) * 0.5)


@pytest.mark.gpu
@pytest.mark.parametrize("H", HISTORIES)
def test_two_loop_recursion_through_ring_wrap_against_float64(H, syn_model):
    """five frames with their own objectives (so their rings wrap at different times), NaN in every dead ring slot, ro and
    Gram entry, at least 2H + 16 pushes (the ring wraps twice, the head visits every position mod 8), skipped pairs
    included"""
    B = 5
    ctx = _ctx(syn_model, B)
    worst = Worst()
    chk = RingChecker(H, B, worst)
    objs = [QuadObjective(100 * H + b) for b in range(B)]
    drive(ctx, H, objs, _x0(B, H), lbfgs_cfg(H, max_iter=7, max_eval=10000), 2 * H + 16, chk)
    for b in range(B):
        assert chk.pushes[b] >= 2 * H + 16 and chk.skips[b] >= 1, (b, chk.pushes[b], chk.skips[b])
        assert len(chk.heads[b]) == min(H, 8) if H < 8 else {h % 8 for h in chk.heads[b]} == set(range(8)), (b, chk.heads[b])
    worst.report("H=%d pushes %s skips %s" % (H, chk.pushes, chk.skips))
    ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("H", [9, 100])
def test_frames_of_a_batch_follow_their_own_transitions(H, syn_model):
    """2(c): each of five frames gives, in a batch, the bits (every trial point, the final state) it gives alone"""
    B = 5
    x0 = _x0(B, 7 + H)
    cfg = lbfgs_cfg(H, max_iter=7, max_eval=10000)
    ctx = _ctx(syn_model, B)
    trace = [[] for _ in range(B)]
    sb, ab = drive(ctx, H, [QuadObjective(500 + b) for b in range(B)], x0, cfg, 2 * H + 16, RingChecker(H, B, Worst()), trace)
    ctx.close()
    for b in range(B):
        c1 = _ctx(syn_model, 1)
        tr1 = [[]]
        s1, a1 = drive(c1, H, [QuadObjective(500 + b)], x0[b:b + 1], cfg, 2 * H + 16, RingChecker(H, 1, Worst()), tr1)
        c1.close()
        assert len(tr1[0]) == len(trace[b]), b
        assert np.array_equal(np.array(tr1[0]).view(np.uint32), np.array(trace[b]).view(np.uint32)), b
        for k in ("x", "d", "g", "hist_s", "hist_y", "ro"):
            assert np.array_equal(a1[k][0].view(np.uint32), ab[k][b].view(np.uint32)), (b, k)
        assert bytes(s1[0]) == bytes(sb[b]), b


# ------------------------------------------------------------------------------------------------ regimes A and B
def _real_ctx(model, gmm, B, seed, H=None):
    from mvsmplfitting_b200.context import FittingContext
    cams = S.make_cameras(4)
    fr = S.make_frames(model, cams, B, seed=seed)
    ctx = FittingContext(0)
    ctx.set_model(model)
    ctx.set_gmm_from_dict(gmm)
    ctx.set_cameras(cams["R"], cams["t"], cams["f"], cams["c"])
    ctx.set_batch(B)
    ctx.set_keypoints(fr["gt_uv"], fr["conf"], fr["joint_weights"])
    ctx.set_loss(body_prior="gmm", data_weight=500.0 / 1536, body_pose_weight=4.78, shape_weight=5.0,
                 bending_prior_weight=3.17 * 4.78)
    return ctx, S.pack_params(fr["init"])


@pytest.mark.gpu
@pytest.mark.parametrize("H", [1, 7, 8, 9, 16, 17, 100])
def test_frame_resident_optimiser_equals_one_step_per_call(H, syn_model, syn_gmm):
    """regime A (lbfgs_resident_kernel: ring and Gram in shared memory only) against regime C (frame-resident closure +
    lbfgs_advance_kernel, one LBFGS.step per call): K outer steps of M iterations, ftol = gtol = 0, give the same bits"""
    B, M = 3, 6
    K = 2 * H + 16                      # every step runs at least one iteration
    ca, X0 = _real_ctx(syn_model, syn_gmm, B, 40 + H)
    cc, _ = _real_ctx(syn_model, syn_gmm, B, 40 + H)
    xa = torch.tensor(X0, device="cuda")
    e_a, _ = ca.lbfgs_run(xa.clone(), ca.make_lbfgs_config(max_outer=1, max_iter=M, history_size=H, ftol=0.0, gtol=0.0))
    fa, sta = ca.lbfgs_run(xa, ca.make_lbfgs_config(max_outer=K, max_iter=M, history_size=H, ftol=0.0, gtol=0.0))
    xc = torch.tensor(X0, device="cuda")
    cfg = cc.make_lbfgs_config(max_outer=1, max_iter=M, history_size=H, ftol=0.0, gtol=0.0)
    iters = evals = 0
    for k in range(K):
        lc, _, st = cc.lbfgs_step(xc, cfg, reset=(k == 0))
        if k == 0:
            assert torch.equal(lc, e_a), "entry losses of the two closures differ"
        iters += st["frame_iterations"]
        evals += st["frame_evals"]
    print("\n[H=%d] K=%d M=%d: %d iterations, %d evaluations" % (H, K, M, iters, evals))
    assert iters >= B * (2 * H + 16)
    sc, _ = Machine(cc, H).read()
    # regime C's rings are full.  With H = 100 the real closure converges first: its later pairs have y.s <= 1e-10 and are
    # skipped, and the rings hold 42 .. 48 pairs (measured on the H100)
    if H <= 17:
        assert all(s.hist_len == H for s in sc), [s.hist_len for s in sc]
    assert torch.equal(xa, xc)
    assert torch.equal(fa, lc)
    assert (sta["frame_iterations"], sta["frame_evals"]) == (iters, evals)
    ca.close()
    cc.close()


@pytest.mark.gpu
@pytest.mark.parametrize("H", [1, 7, 8, 9, 17, 100, 128])
def test_frame_step_ring_against_float64(H, syn_model):
    """regime B: frame_step stages ring, ro and Gram into shared memory and writes back only the pushed slot.  One
    LBFGS.step of one iteration per call through the dense rounds (SDF term on, use_vposer = 2); after every call the state
    passes the checks of the host-driven test, starting from NaN in every dead entry"""
    import os
    c = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "vposer_s11.npz"))
    from mvsmplfitting_b200.context import FittingContext
    B = 2
    ctx = FittingContext(0)
    ctx.set_model(syn_model)
    ctx.set_vposer(S.make_vposer(11))
    ctx.set_cameras(c["cam_R"], c["cam_t"], c["cam_f"], c["cam_c"])
    ctx.set_batch(B)
    ctx.set_keypoints(c["gt_uv"], c["conf"], c["joint_weights"])
    dw, bpw, sw, bend = [float(v) for v in c["w3"]]
    ctx.set_loss(body_prior="l2", use_vposer=2, interpenetration=True, coll_loss_weight=1000.0, sdf_grid=32, data_weight=dw,
                 body_pose_weight=bpw, shape_weight=sw, bending_prior_weight=bend)
    X = c["X"].copy()
    X[:, 13:82] = 0.0
    X[:, 13:45] = c["closure_Z"]
    x = torch.tensor(X, device="cuda")
    m = Machine(ctx, H)
    nan = lambda k: np.full(m.shapes[k], np.nan, np.float32)
    m.write(hist_s=nan("hist_s"), hist_y=nan("hist_y"), ro=nan("ro"), gram=nan("gram"))
    cfg = ctx.make_lbfgs_config(max_outer=1, max_iter=1, history_size=H)
    worst = Worst()
    chk = RingChecker(H, B, worst)
    calls = max(2 * H + 16, 24) if H <= 17 else 24
    pre_s, pre = None, None
    n0 = ctx.launch_count()
    for k in range(calls):
        ctx.lbfgs_step(x, cfg, reset=(k == 0))
        post_s, post = m.read()
        if k == 0:
            assert ctx.launch_count() - n0 > 8                   # dense rounds
        for b in range(B):
            if pre_s is not None:
                # one call: entry evaluation -> ITER_BEGIN (the pair of the previous call's accepted step) -> line search
                ps = post_s[b]
                assert ps.state_n_iter == pre_s[b].state_n_iter + 1
                y = f32(post["prev_g"][b].astype(np.float32) - pre["prev_g"][b])
                post_iter = dict(post)
                post_iter["g"] = post["prev_g"]                  # the gradient the iteration began from
                chk.check(b, True, pre, ps, post_iter, pre_s[b].t, pushed="predict")
                if ps.pushed_slot >= 0:
                    assert np.array_equal(post["hist_y"][b, ps.pushed_slot].view(np.uint32), y.view(np.uint32))
        pre_s, pre = post_s, post
    worst.report("frame_step H=%d calls %d pushes %s skips %s" % (H, calls, chk.pushes, chk.skips))
    if H <= 17:
        assert min(chk.pushes) >= 2 * H, chk.pushes
    ctx.close()


# ------------------------------------------------------------------------------------------------ branches against the oracle
class BranchObjective:
    """scale x [0.5 sum_i lam_i (x_i - c_i)^2 + phi(U x)]: lam log-spaced over 1 .. lam_hi (lam_hi = 0: no quadratic) on the
    coordinates of mask (all by default), U three random directions.  phi: 'quad' none, 'cos' ripples amp cos(3 u.x)
    (non-convex stretches), 'lin' a steady descent -amp (z + z^1.5) along u_0, 'abs' a rounded kink amp |u_0.x - 1|.
    radius: f = g = NaN outside the box |x|_inf <= radius (a closure that overflows); nan: the loss is NaN everywhere"""

    def __init__(self, seed, kind="quad", lam_hi=30.0, amp=1.0, scale=1.0, mask=None, radius=None, nan=False):
        rng = np.random.default_rng(seed)
        self.lam = np.geomspace(1.0, lam_hi, NP) if lam_hi > 0 else np.zeros(NP)
        if mask is not None:
            self.lam[[i for i in range(NP) if not (mask[0] <= i < mask[1])]] = 0.0
        self.c = f32(rng.standard_normal(NP)).astype(np.float64)
        self.U = rng.standard_normal((3, NP)) / math.sqrt(NP)
        self.kind, self.amp, self.scale, self.radius, self.nan = kind, amp, scale, radius, nan

    def __call__(self, x):
        x = np.asarray(x, np.float64)
        nan_loss = self.nan
        if self.radius is not None and not np.abs(x).max() <= self.radius:
            return float("nan"), np.full(NP, np.nan)
        r = x - self.c
        f, g = 0.5 * float(np.sum(self.lam * r * r)), self.lam * r
        z = self.U @ x
        if self.kind == "cos":
            f += self.amp * float(np.sum(np.cos(3 * z)))
            g = g + self.U.T @ (-3 * self.amp * np.sin(3 * z))
        elif self.kind == "lin":
            zp = max(float(z[0]), 0.0)
            f += -self.amp * float(z[0]) - self.amp * zp ** 1.5
            g = g + self.U[0] * (-self.amp - 1.5 * self.amp * math.sqrt(zp))
        elif self.kind == "abs":             # a rounded kink at u_0.x = 1
            w = math.sqrt(1e-6 + (float(z[0]) - 1.0) ** 2)
            f += self.amp * w
            g = g + self.U[0] * (self.amp * (float(z[0]) - 1.0) / w)
        return (float("nan") if nan_loss else self.scale * f), self.scale * g

    def x0(self, kind, eps=0.0):
        """'zero'; 'min': the minimiser of the quadratic (exact in fp32); 'near': eps / lam off it"""
        if kind == "zero":
            return np.zeros(NP, np.float32)
        lam = np.where(self.lam > 0, self.lam, 1.0)
        return f32(self.c + (eps / lam if kind == "near" else 0.0))


class Run:
    """one frame's run: objective, starting point and the optimiser configuration (cfg: lbfgs_cfg arguments)"""

    def __init__(self, obj, x0="zero", eps=0.0, step_mode=0, pose_len=69, **cfg):
        self.obj_kw, self.x0_kw = obj, (x0, eps)
        self.step_mode, self.pose_len = step_mode, pose_len
        self.cfg = dict(dict(H=5, max_outer=3, max_iter=8), **cfg)

    def objective(self):
        return BranchObjective(**self.obj_kw)

    def start(self):
        return self.objective().x0(*self.x0_kw)

    def key(self):
        return (self.step_mode, self.pose_len, tuple(sorted(self.cfg.items())))

    def __repr__(self):
        return "Run(%r, %r, step_mode=%d, pose_len=%d, %r)" % (self.obj_kw, self.x0_kw, self.step_mode, self.pose_len, self.cfg)


SEG32 = ((0, 10), (10, 13), (13, 45), (82, 85), (85, 86))
# Every branch decision of these runs lies >= 1e-4 from its threshold (asserted from the oracle's log below)
BRANCH_RUNS = [
    Run(dict(seed=0)),
    Run(dict(seed=1, lam_hi=1e3)),
    Run(dict(seed=0), lr=6.0),
    Run(dict(seed=2, kind="cos", amp=20.0)),
    Run(dict(seed=0, kind="lin", amp=20.0), lr=6.0),
    Run(dict(seed=0), "min", 0.0),                          # exit at entry
    Run(dict(seed=0), "near", 1e-4, gtol=1e-3),             # gtol with pose_len 69
    # tolerance_change 1e-3: the zoom still tests the bracket width against the reference's 1e-9 (lbfgs_ls.py:393-397); a
    # zoom that tested it against tolerance_change would stop one evaluation early here
    Run(dict(seed=0, kind="abs", lam_hi=0.0), "near", 0.1, max_outer=1, max_iter=8, lr=6.0, tol_change=1e-3),
    Run({'seed': 1, 'kind': 'abs', 'lam_hi': 1000.0, 'amp': 1.0, 'scale': 1.0}, 'min', 0.1, max_outer=1, max_iter=1, lr=6.0, tol_change=1e-09, tol_grad=1e-05, ftol=0.0, gtol=0.0),            # armijo_fail insuf_set zoom_done_curv
    Run({'seed': 4, 'kind': 'cos', 'lam_hi': 30.0, 'amp': 1.0, 'scale': 1.0}, max_outer=1, max_iter=1, lr=1.0, tol_change=1e-05, tol_grad=1e-05, ftol=0.01, gtol=0.001),            # clamp_hi extrapolate wolfe_bracket
    Run({'seed': 4, 'kind': 'abs', 'lam_hi': 0.0, 'amp': 20.0, 'scale': 1.0, 'nan': True, 'mask': (45, 82)}, 'near', 0.0001, pose_len=32, max_outer=6, max_iter=1, lr=6.0, tol_change=0.01, tol_grad=1e-05, ftol=0.0, gtol=0.0),            # cubic_mid
    Run({'seed': 0, 'kind': 'cos', 'lam_hi': 30.0, 'amp': 1.0, 'scale': 1.0}, 'near', 0.1, pose_len=32, max_outer=1, max_iter=25, lr=1.0, tol_change=0.01, tol_grad=1e-05, ftol=0.0, gtol=0.0),            # drop_oldest
    Run({'seed': 1, 'kind': 'quad', 'lam_hi': 1000.0, 'amp': 1.0, 'scale': 1.0}, 'near', 0.0001, pose_len=32, max_outer=6, max_iter=25, lr=0.001, tol_change=1e-09, tol_grad=1e-05, ftol=0.0, gtol=0.001),            # end_dloss
    Run({'seed': 4, 'kind': 'cos', 'lam_hi': 1000.0, 'amp': 1.0, 'scale': 1.0}, pose_len=32, max_outer=1, max_iter=2, lr=6.0, tol_change=1e-05, tol_grad=1e-05, ftol=0.01, gtol=0.0),            # end_max_eval t_first_inv wolfe_first
    Run({'seed': 2, 'kind': 'cos', 'lam_hi': 30.0, 'amp': 20.0, 'scale': 1.0, 'mask': (45, 82)}, 'min', 0.0001, pose_len=32, max_outer=1, max_iter=1, lr=6.0, tol_change=1e-09, tol_grad=1e-05, ftol=0.0, gtol=0.0),            # end_max_iter
    Run({'seed': 5, 'kind': 'quad', 'lam_hi': 1000.0, 'amp': 20.0, 'scale': 0.0001, 'mask': (45, 82)}, 'near', 0.1, max_outer=3, max_iter=25, lr=6.0, tol_change=1e-09, tol_grad=1e-05, ftol=0.0, gtol=0.001),            # end_opt
    Run({'seed': 1, 'kind': 'quad', 'lam_hi': 1000.0, 'amp': 1.0, 'scale': 1.0}, 'near', 0.005, step_mode=1, max_outer=1, max_iter=25, lr=0.001, tol_change=1e-05, tol_grad=1e-05, ftol=0.01, gtol=0.0),            # end_step_max
    Run({'seed': 0, 'kind': 'lin', 'lam_hi': 30.0, 'amp': 1.0, 'scale': 0.0001, 'nan': True, 'mask': (45, 82)}, pose_len=32, max_outer=6, max_iter=25, lr=0.3, tol_change=0.01, tol_grad=0.5, ftol=0.0, gtol=0.001),            # exit_entry mon_nan
    Run({'seed': 1, 'kind': 'lin', 'lam_hi': 1000.0, 'amp': 1.0, 'scale': 1.0, 'radius': 5.0}, 'near', 0.1, max_outer=1, max_iter=8, lr=0.3, tol_change=0.01, tol_grad=1e-05, ftol=0.01, gtol=0.001),            # gtd_new_pos
    Run({'seed': 5, 'kind': 'abs', 'lam_hi': 0.0, 'amp': 20.0, 'scale': 0.0001, 'radius': 5.0}, pose_len=32, max_outer=1, max_iter=25, lr=0.001, tol_change=1e-05, tol_grad=1e-05, ftol=0.01, gtol=0.0),            # gtd_stop t_first_one
    Run({'seed': 0, 'kind': 'abs', 'lam_hi': 1000.0, 'amp': 20.0, 'scale': 1.0}, 'near', 0.0001, pose_len=32, max_outer=1, max_iter=8, lr=1.0, tol_change=1e-09, tol_grad=0.5, ftol=0.01, gtol=0.001),            # insuf_move
    Run({'seed': 0, 'kind': 'abs', 'lam_hi': 30.0, 'amp': 1.0, 'scale': 0.0001, 'radius': 2.0}, 'near', 0.1, step_mode=1, pose_len=32, max_outer=6, max_iter=2, lr=1.0, tol_change=1e-09, tol_grad=1e-05, ftol=0.0, gtol=0.0),            # max_ls
    Run({'seed': 3, 'kind': 'quad', 'lam_hi': 30.0, 'amp': 20.0, 'scale': 0.0001}, 'min', 0.0001, pose_len=32, max_outer=6, max_iter=25, lr=0.001, tol_change=0.01, tol_grad=1e-05, ftol=0.01, gtol=0.0),            # mon_ftol
    Run({'seed': 0, 'kind': 'quad', 'lam_hi': 1000.0, 'amp': 20.0, 'scale': 0.0001, 'mask': (45, 82)}, 'near', 0.1, pose_len=32, max_outer=3, max_iter=1, lr=6.0, tol_change=1e-09, tol_grad=0.5, ftol=0.01, gtol=0.001),            # mon_gtol
    Run({'seed': 0, 'kind': 'cos', 'lam_hi': 30.0, 'amp': 1.0, 'scale': 0.0001}, pose_len=32, max_outer=1, max_iter=8, lr=0.3, tol_change=1e-09, tol_grad=0.5, ftol=0.01, gtol=0.0),            # mon_max_outer
    Run({'seed': 1, 'kind': 'cos', 'lam_hi': 1000.0, 'amp': 1.0, 'scale': 1.0, 'mask': (45, 82)}, 'min', 0.0001, pose_len=32, max_outer=1, max_iter=8, lr=0.3, tol_change=0.01, tol_grad=1e-05, ftol=0.0, gtol=0.0),            # next_iter push
    Run({'seed': 0, 'kind': 'cos', 'lam_hi': 1000.0, 'amp': 1.0, 'scale': 0.0001}, 'min', 0.0001, max_outer=3, max_iter=1, lr=6.0, tol_change=1e-05, tol_grad=1e-05, ftol=0.01, gtol=0.0),            # skip
    Run({'seed': 1, 'kind': 'abs', 'lam_hi': 0.0, 'amp': 20.0, 'scale': 1.0}, 'near', 0.005, pose_len=32, max_outer=1, max_iter=2, lr=1.0, tol_change=1e-09, tol_grad=0.5, ftol=0.0, gtol=0.0),            # zoom_armijo_fail
    Run({'seed': 0, 'kind': 'abs', 'lam_hi': 0.0, 'amp': 20.0, 'scale': 1.0, 'mask': (45, 82)}, 'min', 0.1, pose_len=32, max_outer=1, max_iter=1, lr=6.0, tol_change=0.01, tol_grad=1e-05, ftol=0.0, gtol=0.001),            # zoom_flip
    Run({'seed': 5, 'kind': 'cos', 'lam_hi': 1000.0, 'amp': 1.0, 'scale': 1.0}, 'min', 0.005, step_mode=1, pose_len=32, max_outer=3, max_iter=2, lr=1.0, tol_change=1e-09, tol_grad=0.5, ftol=0.01, gtol=0.001),            # zoom_interp
    Run({'seed': 0, 'kind': 'cos', 'lam_hi': 1000.0, 'amp': 1.0, 'scale': 1.0, 'nan': True}, 'min', 0.005, step_mode=1, max_outer=3, max_iter=1, lr=6.0, tol_change=1e-09, tol_grad=1e-05, ftol=0.01, gtol=0.001),            # zoom_keep
    Run({'seed': 1, 'kind': 'abs', 'lam_hi': 30.0, 'amp': 20.0, 'scale': 1.0}, 'near', 0.0001, pose_len=32, max_outer=1, max_iter=1, lr=1.0, tol_change=1e-05, tol_grad=1e-05, ftol=0.0, gtol=0.0),            # zoom_max_iter
]
# trial points, relative to max(|x|_inf, 1).  The directions differ in the last bits and the drift compounds over a run on
# a non-convex objective: 'cos' at lr 6 drifted to 5e-3 within three steps, so such runs are not used.  Worst on the
# H100: 1.43e-5.
X_BAR = 6e-5
# trial step lengths, relative: t comes out of the cubic interpolation, which magnifies the last-bit differences of the
# directions (5.9e-4 measured on the H100 where the trial points agreed within 6e-5)
T_BAR = 1e-2
# every branch of lbfgs_ls.py / run_fitting (the oracle's names) the runs must reach
BRANCHES_REQUIRED = {
    "exit_entry", "t_first_inv", "t_first_one",                                             # entry, first step
    "push", "skip", "drop_oldest", "gtd_stop",                                              # pushes, direction test
    "armijo_fail", "wolfe_first", "wolfe_bracket", "gtd_new_pos", "extrapolate",
    "clamp_hi", "cubic_mid", "max_ls",                                          # bracket phase
    "insuf_set", "insuf_move", "zoom_interp", "zoom_armijo_fail", "zoom_flip", "zoom_keep",
    "zoom_done_curv", "zoom_max_iter",                                   # zoom
    "end_max_iter", "end_max_eval", "end_opt", "end_step_max", "end_dloss", "next_iter",    # ends of an iteration
    "mon_nan", "mon_ftol", "mon_gtol", "mon_max_outer",                                     # monitor
    "nonfinite_departure",                                                                  # DESIGN section 4
}
# Not reached with the 1e-4 margin by any objective tried (a random search over ~50000 runs of the families above):
# "clamp_lo", "ls_f_prev", "zoom_swap", "zoom_tol_change".


def run_oracle(run):
    """the oracle on the run; returns (log, evaluated points, optimiser, final loss of run_fitting or step's return)"""
    from oracle import lbfgs_oracle as L
    obj = run.objective()
    log, xs = [], []

    def fg(x):
        xs.append(x.numpy().copy())
        f, g = obj(x.double().numpy())
        return float(np.float32(f)), torch.tensor(f32(g))
    c = run.cfg
    opt = L.LBFGSOracle(torch.tensor(run.start()), fg, lr=c.get("lr", 1.0), max_iter=c["max_iter"], max_eval=c.get("max_eval"),
                        tolerance_grad=c.get("tol_grad", 1e-5), tolerance_change=c.get("tol_change", 1e-9),
                        history_size=c["H"], log=log)
    if run.step_mode:
        fin = opt.step()
    else:
        fin, _ = L.run_fitting(opt, c["max_outer"], c.get("ftol", 0.0), c.get("gtol", 0.0),
                               SEG32 if run.pose_len == 32 else L.PARAM_SEGMENTS)
    return log, xs, opt, fin


def run_device(ctx, runs):
    """the device state machine on runs (one frame each, same configuration) to PH_DONE; per frame the evaluations as
    (kind, x, t), and the final scalars and state"""
    r0 = runs[0]
    c = dict(r0.cfg)
    H = c.pop("H")
    cfg = lbfgs_cfg(H, **c)
    m = Machine(ctx, H)
    B = ctx.B
    objs = [r.objective() for r in runs]
    m.start(np.stack([r.start() for r in runs]))
    sc, st = m.read()
    evals = [[] for _ in range(B)]
    for _ in range(5000):
        act = [b for b in range(B) if sc[b].phase != PH_DONE]
        if not act:
            break
        loss, ge = st["loss_eval"].copy(), st["g_eval"].copy()
        for b in act:
            f, g = objs[b](st["x_eval"][b])
            loss[b], ge[b] = np.float32(f), f32(g)
            evals[b].append(("entry" if sc[b].phase == PH_STEP_ENTRY else "ls", st["x_eval"][b].copy(), float(sc[b].t)))
        m.write(loss_eval=loss, g_eval=ge)
        m.advance(cfg, r0.step_mode, r0.pose_len)
        sc, st = m.read()
    assert all(s.phase == PH_DONE for s in sc)
    return evals, sc, st


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    both_nan = np.isnan(a) & np.isnan(b)
    err = np.where(both_nan, 0.0, np.abs(a - b))
    return float(np.nan_to_num(err, nan=np.inf).max()) / max(float(np.nan_to_num(np.abs(b), nan=0.0).max()), 1.0)


def check_against_oracle(run, evals, s, st, b, worst, reached):
    log, xs, opt, fin = run_oracle(run)
    for n, mg in log:
        if n != "eval":
            assert mg is None or mg >= 1e-4, (run, n, mg)
            reached.setdefault(n, run)
    kinds = [k for n, k in log if n == "eval"]
    if not np.isfinite(opt.x.numpy()).all():
        # a line search that ends on a non-finite point: the oracle writes NaN into the parameters, the device keeps them at
        # the line search's start and ends the step (DESIGN section 4).  Up to there both evaluate the same points.
        n = len(evals)
        assert n <= len(kinds) and [e[0] for e in evals] == kinds[:n], run
        xs = xs[:n]
        assert np.array_equal(st["x"][b].view(np.uint32), run.start().view(np.uint32)), run
        assert s.t == 0.0, run
        reached.setdefault("nonfinite_departure", run)
        for (kind, xd, td), xo in zip(evals, xs):
            assert _rel(xd, xo) <= X_BAR, run
        return
    assert [e[0] for e in evals] == kinds, run
    for k, ((kind, xd, td), xo) in enumerate(zip(evals, xs)):
        err = _rel(xd, xo)
        worst.add("x_eval", err / X_BAR)
        assert err <= X_BAR, (run, k, err)
    td = [e[2] for e in evals if e[0] == "ls"]
    assert len(td) == len(opt.trial_t), run
    for k, (a, o) in enumerate(zip(td, opt.trial_t)):
        err = 0.0 if (math.isnan(a) and math.isnan(o)) else abs(a - o) / max(abs(o), 1e-30)
        worst.add("t", err / T_BAR)
        assert err <= T_BAR, (run, k, a, o)
    assert (s.iters, s.evals) == (opt.iters, opt.evals), run
    if run.obj_kw.get("nan"):
        return
    if fin is None:                     # run_fitting stopped before any step completed: no previous loss (the device: NaN)
        assert math.isnan(s.final_loss), (run, s.final_loss)
    else:
        assert abs(float(s.final_loss) - fin) <= 1e-5 * max(abs(fin), 1.0), (run, s.final_loss, fin)


@pytest.mark.gpu
def test_line_search_and_monitor_branches_match_the_oracle(syn_model):
    """2(b): short runs, device against the oracle on the same closure values: the same sequence of entry / line-search
    evaluations, every trial point and step length within X_BAR / T_BAR, the same counts and final loss; every branch
    decision of the oracle at least 1e-4 from its threshold, and every branch of BRANCHES_REQUIRED reached.  2(c): the
    frames of each batch give the bits they give alone."""
    reached = {}
    worst = Worst()
    groups = {}
    for r in BRANCH_RUNS:
        groups.setdefault(r.key(), []).append(r)
    for runs in groups.values():
        ctx = _ctx(syn_model, len(runs))
        evals, sc, st = run_device(ctx, runs)
        ctx.close()
        for b, r in enumerate(runs):
            check_against_oracle(r, evals[b], sc[b], st, b, worst, reached)
            if len(runs) > 1:
                c1 = _ctx(syn_model, 1)
                e1, s1, _ = run_device(c1, [r])
                c1.close()
                assert bytes(s1[0]) == bytes(sc[b]), r
                assert len(e1[0]) == len(evals[b]) and all(np.array_equal(u[1].view(np.uint32), v[1].view(np.uint32))
                                                          for u, v in zip(e1[0], evals[b])), r
    worst.report("branches")
    print("[branches] reached: %s" % ", ".join(sorted(reached)))
    missing = BRANCHES_REQUIRED - set(reached)
    assert not missing, sorted(missing)
