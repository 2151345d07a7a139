"""GPU: the causal temporal term of video fits (mvs_fit_seq_temporal, mvs_fit_seq_stream_temporal): every warm frame's stages
2 .. n-1 add sum_i w_i (x_i - x^_i)^2, x^ = the predecessor's fitted row.  Oracles, all exact (np.array_equal; NaN equal to NaN
for losses): seqio.fit_sequences with a batch of S (lock-step), the drivers without the term, and a single-frame mvs_fit with
the warm slice of the stages under mvs_set_anchor(row = predecessor's fitted row, weight = w)."""
import ctypes

import numpy as np
import pytest
import torch

from mvsmplfitting_b200 import _lib, seqio
from mvsmplfitting_b200 import synthetic as S
from tests.test_gpu_seq_stream import GUESS, LENGTHS, OPT, assert_same, cold_after_first, make_ctx, make_seqs, reinit_between, stages

pytestmark = pytest.mark.gpu

LAM = 50.0                                  # a weight that moves every warm frame's result (a scalar: lam x smooth_mask)


def tw_vec(lam=LAM):
    return seqio.temporal_weight_vector(lam)


def kind_args(kind):
    """'gmm': GMM prior, every stage frame-resident (chaining run c = 0, axis-angle pose: the anchor keeps the fitted pose while
    the start point has the hip seed); 'vposer': the shipped configuration (latent pose, L2 prior, c = 0); 'sdf': the benchmark
    configuration (GMM, SDF in stages 2-3: dense chaining, c > 0)"""
    return dict(sdf=kind == "sdf", vposer=kind == "vposer")


def lockstep(model, gmm, cams, seqs, kind, reinit=5000.0, tw=None):
    ctx = make_ctx(model, gmm, cams, len(seqs), vposer=kind == "vposer")
    res, tot = seqio.fit_sequences(ctx, seqs, stages(ctx, **kind_args(kind)), ctx.make_lbfgs_config(**OPT), estimate_scale=True,
                                   pose_format="lsp14", reinit_loss=reinit, temporal_weight=tw)
    ctx.close()
    return np.concatenate([r[0] for r in res]), np.concatenate([r[1] for r in res]), tot


def stream(model, gmm, cams, seqs, B, kind, reinit=5000.0, tw=None):
    """cold start points as fit_sequences computes them, then one mvs_fit_seq_stream(_temporal) call on B slots.  Returns
    (params, final loss, stats, cold start points)"""
    ctx = make_ctx(model, gmm, cams, B, vposer=kind == "vposer")
    cfgs = stages(ctx, **kind_args(kind))
    gt_uv = np.concatenate([q["gt_uv"] for q in seqs], 1)
    conf = np.concatenate([q["conf"] for q in seqs], 1)
    jw = seqio.joint_weights("lsp14")
    x = seqio._cold_guesses(ctx, gt_uv, conf, jw, cfgs, GUESS)
    x0 = x.cpu().numpy()
    kw = {} if tw is None else dict(temporal_weight=tw)
    final, st = ctx.fit_seq_stream(x, gt_uv, conf, jw, [len(q["frames"]) for q in seqs], cfgs, ctx.make_lbfgs_config(**OPT),
                                   reinit_loss=reinit, **kw)
    out = x.cpu().numpy(), final.cpu().numpy(), st, x0
    ctx.close()
    return out


def same_counts(ref, got, what):
    """summed iteration / evaluation counts (a lock-step with sequences of different lengths also counts the idle slots of the
    sequences that ended, so it is compared with equal lengths only)"""
    for k in ("frame_iterations", "frame_evals", "frames_nan"):
        assert ref[2][k] == got[2][k], (what, k, ref[2][k], got[2][k])


@pytest.mark.parametrize("kind", ["vposer", "sdf"])
def test_stream_equals_lockstep(kind, syn_model, syn_gmm):
    cams = S.make_cameras(4)
    seqs = make_seqs(syn_model, cams, LENGTHS, 1100)
    ref = lockstep(syn_model, syn_gmm, cams, seqs, kind, tw=tw_vec())
    off = lockstep(syn_model, syn_gmm, cams, seqs, kind)
    assert not np.array_equal(ref[0], off[0])                     # the term is on
    full = None
    for B in (len(seqs), 2, 1):
        got = stream(syn_model, syn_gmm, cams, seqs, B, kind, tw=tw_vec())
        assert_same(ref, got, "%s B=%d" % (kind, B))
        full = full or got
        same_counts(full, got, "%s B=%d" % (kind, B))


@pytest.mark.parametrize("kind", ["vposer", "sdf"])
def test_stat_sums_equal_the_lockstep(kind, syn_model, syn_gmm):
    cams = S.make_cameras(4)
    seqs = make_seqs(syn_model, cams, (5, 5, 5), 1150)
    ref = lockstep(syn_model, syn_gmm, cams, seqs, kind, tw=tw_vec())
    got = stream(syn_model, syn_gmm, cams, seqs, 2, kind, tw=tw_vec())
    assert_same(ref, got, kind)
    same_counts(ref, got, kind)


@pytest.mark.parametrize("kind", ["gmm", "sdf"])
def test_reinitialised_frames(kind, syn_model, syn_gmm):
    """frames whose predecessor ended above reinit_loss start cold and carry no term (with SDF stages: they park)"""
    cams = S.make_cameras(4)
    seqs = make_seqs(syn_model, cams, LENGTHS, 1200)
    reinit = reinit_between(lockstep(syn_model, syn_gmm, cams, seqs, kind, tw=tw_vec())[1])
    ref = lockstep(syn_model, syn_gmm, cams, seqs, kind, reinit=reinit, tw=tw_vec())
    assert cold_after_first(seqs, ref[1], reinit) >= 1
    got = [stream(syn_model, syn_gmm, cams, seqs, B, kind, reinit=reinit, tw=tw_vec()) for B in (2, 5)]
    for g, B in zip(got, (2, 5)):
        assert_same(ref, g, "%s reinit B=%d" % (kind, B))
    same_counts(got[0], got[1], "%s reinit" % kind)


def test_rigs_and_3d_targets(syn_model, syn_gmm):
    """two rigs and 3-D targets (one frame without an annotation): fit_sequences in lock-step and through the stream"""
    from tests.test_gpu_rigs import RIGS, new_ctx, rig_cams, rig_scales, stage_cfgs
    cams, sc = rig_cams(RIGS[:2]), rig_scales(RIGS[:2])
    seqs = []
    for s_, (r, T) in enumerate(zip((0, 1, 1, 0), (4, 4, 4, 4))):
        fr = S.make_frames(syn_model, cams[r], T, seed=1300 + s_, smooth_walk=True)
        rng = np.random.RandomState(1300 + s_)
        has = np.ones(T, bool)
        if s_ == 1:
            has[2] = False
        seqs.append(dict(gt_uv=fr["gt_uv"], conf=fr["conf"], present=np.ones(fr["conf"].shape[:2], bool),
                         frames=["%05d" % t for t in range(T)], serial="s%02d" % s_, rig=r, has3d=has,
                         joints3d=(fr["gt_joints3d"] + rng.normal(0, 0.02, fr["gt_joints3d"].shape)).astype(np.float32),
                         conf3d=rng.uniform(0.5, 1.0, (T, 17)).astype(np.float32)))
    out = {}
    for B in (len(seqs), 2):
        ctx = new_ctx(syn_model, syn_gmm, B, rigs=cams, scales=sc)
        res, st = seqio.fit_sequences(ctx, seqs, stage_cfgs(ctx, "gmm"), ctx.make_lbfgs_config(**OPT), estimate_scale=True,
                                      pose_format="lsp14", rigs=cams, rig_data_weight_scale=sc, use_3d=True, temporal_weight=LAM)
        ctx.close()
        out[B] = np.concatenate([r[0] for r in res]), np.concatenate([r[1] for r in res]), st
    assert_same(out[len(seqs)], out[2], "rigs + 3-D")
    same_counts(out[len(seqs)], out[2], "rigs + 3-D")


@pytest.mark.parametrize("kind", ["gmm", "sdf"])
def test_off_means_off(kind, syn_model, syn_gmm):
    """weight None and weight all zero: the bits of the drivers without the term, in both drivers"""
    cams = S.make_cameras(4)
    seqs = make_seqs(syn_model, cams, (3, 5, 2), 1400)
    base = lockstep(syn_model, syn_gmm, cams, seqs, kind)
    zero = lockstep(syn_model, syn_gmm, cams, seqs, kind, tw=np.zeros(86, np.float32))
    assert_same(base, zero, "lock-step zero")
    same_counts(base, zero, "lock-step zero")
    sbase = stream(syn_model, syn_gmm, cams, seqs, 2, kind)
    szero = stream(syn_model, syn_gmm, cams, seqs, 2, kind, tw=np.zeros(86, np.float32))
    assert_same(sbase, szero, "stream zero")
    same_counts(sbase, szero, "stream zero")
    assert_same(base, sbase, "stream = lock-step without the term")


def single_frame(model, gmm, cams, seq_gt, seq_conf, f, x_start, cfgs_fn, vposer, anchor=None, tw=None):
    """frame f alone on a one-slot context: mvs_fit from x_start over the stages cfgs_fn(ctx) gives, with
    mvs_set_anchor(anchor, tw) when anchor is given"""
    ctx = make_ctx(model, gmm, cams, 1, vposer=vposer)
    ctx.set_keypoints(seq_gt[:, f:f + 1], seq_conf[:, f:f + 1], seqio.joint_weights("lsp14"))
    if anchor is not None:
        ctx.set_anchor(torch.tensor(anchor[None], device="cuda"), torch.tensor(tw[None], device="cuda"))
    x = torch.tensor(x_start[None], device="cuda").contiguous()
    final, _ = ctx.fit(x, cfgs_fn(ctx), ctx.make_lbfgs_config(**OPT))
    out = x.cpu().numpy()[0], final.cpu().numpy()[0]
    ctx.close()
    return out


@pytest.mark.parametrize("kind", ["gmm", "vposer", "sdf"])
def test_right_rows_right_stages(kind, syn_model, syn_gmm):
    """a warm frame of the stream = mvs_fit on the warm slice of the stages with mvs_set_anchor(predecessor's returned row, w),
    from the warm start the driver builds; a cold frame (first of its sequence, or re-initialised) = mvs_fit of every stage
    from its cold start point, without the term"""
    cams = S.make_cameras(4)
    seqs = make_seqs(syn_model, cams, (4, 3), 1500)
    vp = kind == "vposer"
    first = stream(syn_model, syn_gmm, cams, seqs, 2, kind, tw=tw_vec())
    reinit = reinit_between(first[1])
    x, loss, _, x0 = stream(syn_model, syn_gmm, cams, seqs, 2, kind, reinit=reinit, tw=tw_vec())
    gt = np.concatenate([q["gt_uv"] for q in seqs], 1)
    cf = np.concatenate([q["conf"] for q in seqs], 1)

    def warm_cfgs(ctx):
        c = stages(ctx, **kind_args(kind))
        c[2].body_pose_weight = float(np.float32(c[2].body_pose_weight) * np.float32(0.15))
        return c[2:]

    f, n_warm, n_cold = 0, 0, 0
    for q in seqs:
        for t in range(len(q["frames"])):
            if t > 0 and loss[f - 1] <= np.float32(reinit):
                start = x[f - 1].copy()
                if not vp:                                        # fix_params: the body pose restarts from the hip seed
                    start[13:82] = x0[f, 13:82]
                xr, lr = single_frame(syn_model, syn_gmm, cams, gt, cf, f, start, warm_cfgs, vp, anchor=x[f - 1], tw=tw_vec())
                n_warm += 1
            else:
                xr, lr = single_frame(syn_model, syn_gmm, cams, gt, cf, f, x0[f], lambda c: stages(c, **kind_args(kind)), vp)
                n_cold += 1
            assert np.array_equal(xr, x[f]) and (lr == loss[f] or (np.isnan(lr) and np.isnan(loss[f]))), (kind, f)
            f += 1
    assert n_warm >= 1 and n_cold > len(seqs), (n_warm, n_cold)        # some re-initialised frame among the cold ones


def test_refusals_leave_the_context_usable(syn_model, syn_gmm):
    cams = S.make_cameras(4)
    seqs = make_seqs(syn_model, cams, (2, 3), 1600)
    ctx = make_ctx(syn_model, syn_gmm, cams, 2)
    cfgs = stages(ctx)
    gt_uv = np.concatenate([q["gt_uv"] for q in seqs], 1)
    conf = np.concatenate([q["conf"] for q in seqs], 1)
    jw = seqio.joint_weights("lsp14")
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    opt = ctx.make_lbfgs_config(**OPT)
    arr = (_lib.LossConfig * len(cfgs))(*cfgs)
    x = seqio._cold_guesses(ctx, gt_uv, conf, jw, cfgs, GUESS)
    gtd, cfd, jwd = (torch.tensor(a, device="cuda") for a in (gt_uv, conf, jw))
    fin = torch.empty(5, device="cuda")
    off = np.array([0, 2, 5], np.int32)
    s = _lib.SequenceStream(2, off.ctypes.data_as(ctypes.c_void_p), p(x), p(gtd), p(cfd), p(jwd), p(fin), 5000.0)
    ctx.set_keypoints(gt_uv[:, :2], conf[:, :2], jw)
    xb = x[:2].clone()
    prev = x[:2].clone()
    warm = np.array([1, 0], np.uint8)
    fb = torch.empty(2, device="cuda")

    def calls(w, n=len(cfgs)):
        wa = np.ascontiguousarray(w, np.float32)
        wp = wa.ctypes.data_as(ctypes.c_void_p)
        a = ctx.lib.mvs_fit_seq_temporal(ctx.h, p(xb), n, arr, ctypes.byref(opt), warm.ctypes.data_as(ctypes.c_void_p), p(prev),
                                         wp, p(fb), None, None)
        b = ctx.lib.mvs_fit_seq_stream_temporal(ctx.h, ctypes.byref(s), None, None, None, wp, n, arr, ctypes.byref(opt), None,
                                                None)
        return a, b

    good = tw_vec()
    for bad in (-1.0, np.nan, np.inf):
        w = good.copy()
        w[20] = bad
        assert calls(w) == (-1, -1), bad
    assert calls(good, n=2) == (-1, -1)                                  # n_stages <= 2
    ctx.set_anchor(torch.zeros(2, 86, device="cuda"), torch.ones(2, 86, device="cuda"))
    assert calls(good) == (-4, -4)
    ctx.set_anchor(None)
    ctx.set_exec_mode(1)
    assert calls(good) == (-4, -4)
    ctx.set_exec_mode(0)
    x_before = x.clone()
    assert calls(good) == (0, 0)                                         # usable: both run
    assert torch.isfinite(fb).all() and torch.isfinite(fin).all() and not torch.equal(x, x_before)
    ctx.close()


def test_direction_jitter_goes_down(syn_model, syn_gmm):
    """smooth walks seen with 5 px detection noise: a large weight lowers the mean squared second difference of the fitted 3-D
    keypoints over warm frames"""
    cams = S.make_cameras(4)
    seqs = make_seqs(syn_model, cams, (16, 16), 1700)
    acc = {}
    for lam in (0.0, 1000.0):
        x, loss, _ = lockstep(syn_model, syn_gmm, cams, seqs, "gmm", tw=None if lam == 0 else lam)
        ctx = make_ctx(syn_model, syn_gmm, cams, x.shape[0])
        j = ctx.forward_only(torch.tensor(x, device="cuda"), want_verts=False)["joints"].cpu().numpy().astype(np.float64)
        ctx.close()
        a, f = [], 0
        for q in seqs:
            for t in range(2, len(q["frames"])):              # second differences whose last two frames are warm
                if loss[f + t - 2] <= 5000.0 and loss[f + t - 1] <= 5000.0:
                    a.append(j[f + t] - 2 * j[f + t - 1] + j[f + t - 2])
            f += len(q["frames"])
        assert len(a) >= 20, len(a)
        acc[lam] = float(np.mean(np.stack(a) ** 2))
    assert acc[1000.0] < acc[0.0], acc
