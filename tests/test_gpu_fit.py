"""GPU: mvs_fit, the multi-stage entry point.  Consecutive stages of the same regime run as ONE multi-stage run in
which every frame changes stage on its own; since frames are independent problems with frame-local arithmetic, the
result must be BIT-IDENTICAL to running the stages one after the other with a barrier in between (exec_mode 2 /
mvs_lbfgs_run per stage), and a frame's result must not depend on which other frames share the batch."""
import numpy as np
import pytest
import torch

from mvsmplfitting_b200 import synthetic as S

pytestmark = pytest.mark.gpu


def _ctx(model, cams, gmm, B, mode=0):
    from mvsmplfitting_b200.context import FittingContext
    ctx = FittingContext(0)
    ctx.set_model(model)
    ctx.set_gmm_from_dict(gmm)
    ctx.set_cameras(cams["R"], cams["t"], cams["f"], cams["c"])
    ctx.set_batch(B)
    ctx.set_exec_mode(mode)
    return ctx


def _stages(ctx, sdf_from=None):
    sw = S.STAGE_WEIGHTS
    out = []
    for i in range(4):
        sdf = sdf_from is not None and i >= sdf_from
        bpw = sw["body_pose_prior_weights"][i]
        out.append(ctx.make_loss_config(body_prior="gmm", interpenetration=sdf, sdf_grid=64, data_weight=500.0 / 1536,
                                        body_pose_weight=bpw, shape_weight=sw["shape_weights"][i],
                                        bending_prior_weight=3.17 * bpw,
                                        coll_loss_weight=sw["coll_loss_weights"][i] if sdf else 0.0))
    return out


@pytest.mark.parametrize("sdf_from", [None, 2])
def test_fit_merged_stages_equal_sequential_stages_bitwise(sdf_from, syn_model, syn_gmm):
    cams = S.make_cameras(4)
    B = 24
    fr = S.make_frames(syn_model, cams, B, seed=4242)
    X0 = S.pack_params(fr["init"])
    res = {}
    for name, mode in (("merged", 0), ("barrier", 2), ("per_stage_calls", 0)):
        ctx = _ctx(syn_model, cams, syn_gmm, B, mode)
        ctx.set_keypoints(fr["gt_uv"], fr["conf"], fr["joint_weights"])
        stages = _stages(ctx, sdf_from)
        opt = ctx.make_lbfgs_config(max_outer=4)
        x = torch.tensor(X0, device="cuda")
        n0 = ctx.launch_count()
        if name == "per_stage_calls":
            tot = dict(frame_iterations=0, frame_evals=0)
            for cfg in stages:
                ctx.set_loss(config=cfg)
                final, st = ctx.lbfgs_run(x, opt)
                for k in tot:
                    tot[k] += st[k]
        else:
            final, tot = ctx.fit(x, stages, opt)
        res[name] = (x.cpu().numpy().copy(), final.cpu().numpy().copy(), tot, ctx.launch_count() - n0)
        ctx.close()
    xm, fm, tm, lm = res["merged"]
    for other in ("barrier", "per_stage_calls"):
        xo, fo, to, lo = res[other]
        assert np.array_equal(xm, xo), other
        assert np.array_equal(fm, fo, equal_nan=True), other
        assert tm["frame_iterations"] == to["frame_iterations"] and tm["frame_evals"] == to["frame_evals"], other
    assert tm["frame_iterations"] > 4 * B
    assert lm < res["barrier"][3]                 # fewer launches: no per-stage tails
    if sdf_from is None:
        assert lm <= 4                            # all four stages of all frames: one resident launch + bookkeeping


def test_fit_frame_result_independent_of_batch_mates(syn_model, syn_gmm):
    """the same frame fitted alone and inside a batch of others: identical bits (dense regime included)"""
    cams = S.make_cameras(4)
    B = 9
    fr = S.make_frames(syn_model, cams, B, seed=99)
    X0 = S.pack_params(fr["init"])
    ctx = _ctx(syn_model, cams, syn_gmm, B)
    ctx.set_keypoints(fr["gt_uv"], fr["conf"], fr["joint_weights"])
    opt = ctx.make_lbfgs_config(max_outer=3)
    xb = torch.tensor(X0, device="cuda")
    ctx.fit(xb, _stages(ctx, 2), opt)
    xb = xb.cpu().numpy()
    ctx.close()
    for b in (0, 5):
        c1 = _ctx(syn_model, cams, syn_gmm, 1)
        c1.set_keypoints(fr["gt_uv"][:, b:b + 1], fr["conf"][:, b:b + 1], fr["joint_weights"])
        x1 = torch.tensor(X0[b:b + 1], device="cuda")
        c1.fit(x1, _stages(c1, 2), opt)
        assert np.array_equal(x1.cpu().numpy()[0], xb[b]), b
        c1.close()


def test_fit_host_matches_fit_device(syn_model, syn_gmm):
    cams = S.make_cameras(4)
    B = 6
    fr = S.make_frames(syn_model, cams, B, seed=7)
    X0 = S.pack_params(fr["init"])
    ctx = _ctx(syn_model, cams, syn_gmm, B)
    ctx.set_keypoints(fr["gt_uv"], fr["conf"], fr["joint_weights"])
    stages = _stages(ctx, 2)
    opt = ctx.make_lbfgs_config(max_outer=3)
    xd = torch.tensor(X0, device="cuda")
    fd, sd = ctx.fit(xd, stages, opt)
    xh = X0.copy()
    fh, sh = ctx.fit_host(xh, fr["gt_uv"], fr["conf"], fr["joint_weights"], stages, opt)
    assert np.array_equal(xh, xd.cpu().numpy())
    assert np.array_equal(fh, fd.cpu().numpy(), equal_nan=True)
    assert sh["frame_evals"] == sd["frame_evals"]
    ctx.close()


@pytest.mark.parametrize("sdf_from", [None, 2])
def test_fit_seq_warm_frames_skip_two_stages(sdf_from, syn_model, syn_gmm):
    """mvs_fit_seq (is_seq, non_linear_solver.py:157-162): a warm frame's result is, bit for bit, what mvs_fit gives it with
    the stage list [2 (0.15 x body_pose_weight), 3]; a cold frame in the same batch gets the full schedule; no flags = mvs_fit"""
    cams = S.make_cameras(4)
    B = 6
    fr = S.make_frames(syn_model, cams, B, seed=515)
    X0 = S.pack_params(fr["init"])
    warm = np.array([1, 0, 1, 1, 0, 0], bool)

    def run(stage_fn, warm_flags=None):
        ctx = _ctx(syn_model, cams, syn_gmm, B)
        ctx.set_keypoints(fr["gt_uv"], fr["conf"], fr["joint_weights"])
        x = torch.tensor(X0, device="cuda")
        final, st = ctx.fit(x, stage_fn(ctx), ctx.make_lbfgs_config(max_outer=4), warm=warm_flags)
        out = x.cpu().numpy().copy(), final.cpu().numpy().copy(), st
        ctx.close()
        return out

    def warm_stages(ctx):
        st = _stages(ctx, sdf_from)[2:]
        st[0].body_pose_weight *= 0.15
        st[0].bending_prior_weight = _stages(ctx, sdf_from)[2].bending_prior_weight        # only the pose prior is damped
        return st

    x_seq, f_seq, st_seq = run(lambda c: _stages(c, sdf_from), warm)
    x_cold, f_cold, st_cold = run(lambda c: _stages(c, sdf_from))
    x_warm, f_warm, _ = run(warm_stages)
    assert np.array_equal(x_seq[~warm], x_cold[~warm]) and np.array_equal(f_seq[~warm], f_cold[~warm])
    assert np.array_equal(x_seq[warm], x_warm[warm]) and np.array_equal(f_seq[warm], f_warm[warm])
    assert not np.array_equal(x_seq[warm], x_cold[warm])
    assert st_seq["frame_iterations"] < st_cold["frame_iterations"] and st_seq["frames_nan"] == 0
    x_none, f_none, _ = run(lambda c: _stages(c, sdf_from), np.zeros(B, bool))
    assert np.array_equal(x_none, x_cold) and np.array_equal(f_none, f_cold)


def test_fit_seq_guards(syn_model, syn_gmm):
    """warm frames skip two stages, so a two-stage schedule leaves them nothing (the reference would return an undefined loss);
    the batched reference chain (exec mode 1) has no per-frame stage table"""
    from mvsmplfitting_b200._lib import MvsError
    cams = S.make_cameras(4)
    B = 2
    fr = S.make_frames(syn_model, cams, B, seed=3)
    ctx = _ctx(syn_model, cams, syn_gmm, B)
    ctx.set_keypoints(fr["gt_uv"], fr["conf"], fr["joint_weights"])
    x = torch.tensor(S.pack_params(fr["init"]), device="cuda")
    with pytest.raises(MvsError):
        ctx.fit(x, _stages(ctx)[:2], ctx.make_lbfgs_config(max_outer=1), warm=[True, False])
    ctx.set_exec_mode(1)
    with pytest.raises(MvsError):
        ctx.fit(x, _stages(ctx), ctx.make_lbfgs_config(max_outer=1), warm=[True, False])
    final, st = ctx.fit(x, _stages(ctx), ctx.make_lbfgs_config(max_outer=1), warm=[False, False])      # no warm frame: plain mvs_fit
    assert st["frames_nan"] == 0 and torch.isfinite(final).all()
    ctx.close()


def test_fit_keeps_parameters_finite_when_a_line_search_ends_on_a_non_finite_point(syn_model, syn_gmm):
    """Frame 91 of the benchmark's first batch (8 views, seed 1000, SDF term on a 128 grid in stages 2-3) ends stage 2 on
    the jump of the as-written SDF term, and a stage-3 line search from there reaches only non-finite trial points.  The
    optimiser keeps the line search's start instead of writing NaN into the parameters, so the fit ends finite."""
    cams = S.make_cameras(8)
    fr = S.make_frames(syn_model, cams, 256, seed=1000)
    sl = slice(91, 92)
    ctx = _ctx(syn_model, cams, syn_gmm, 1)
    ctx.set_keypoints(np.ascontiguousarray(fr["gt_uv"][:, sl]), np.ascontiguousarray(fr["conf"][:, sl]), fr["joint_weights"])
    sw = S.STAGE_WEIGHTS
    stages = [ctx.make_loss_config(body_prior="gmm", interpenetration=True, sdf_grid=128, data_weight=500.0 / 1536,
                                   body_pose_weight=sw["body_pose_prior_weights"][i], shape_weight=sw["shape_weights"][i],
                                   bending_prior_weight=3.17 * sw["body_pose_prior_weights"][i],
                                   coll_loss_weight=sw["coll_loss_weights"][i]) for i in range(4)]
    x = torch.tensor(S.pack_params(fr["init"])[sl], device="cuda")
    final, st = ctx.fit(x, stages)
    torch.cuda.synchronize()
    assert st["frames_nan"] == 0 and torch.isfinite(final).all() and torch.isfinite(x).all(), (final, st)
    ctx.close()
