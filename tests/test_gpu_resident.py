"""GPU: the frame-resident kernels (one CTA per frame: fused closure, whole-stage L-BFGS) against the batched
multi-kernel path they replace in the sparse regime (mvs_set_exec_mode(1) forces the batched path)."""
import numpy as np
import pytest
import torch

from mvsmplfitting_b200 import synthetic as S
from tests import golden_util as G

pytestmark = pytest.mark.gpu


def make_ctx(model, cams, B, gmm, mode):
    from mvsmplfitting_b200.context import FittingContext
    ctx = FittingContext(0)
    ctx.set_model(model)
    ctx.set_gmm_from_dict(gmm)
    ctx.set_cameras(cams["R"], cams["t"], cams["f"], cams["c"])
    ctx.set_batch(B)
    ctx.set_exec_mode(mode)
    return ctx


@pytest.mark.parametrize("B,V,prior,bpw", [(1, 8, "gmm", 4.78), (37, 4, "gmm", 57.4), (300, 8, "l2", 4.78), (64, 16, "gmm", 4.78)])
def test_resident_closure_equals_batched_closure(B, V, prior, bpw, syn_model, syn_gmm):
    cams = S.make_cameras(V)
    fr = S.make_frames(syn_model, cams, B, seed=50 + B)
    w = dict(data_weight=500.0 / 1536, body_pose_weight=bpw, shape_weight=5.0, bending_prior_weight=3.17 * bpw)
    outs = []
    for mode in (0, 1):
        ctx = make_ctx(syn_model, cams, B, syn_gmm, mode)
        ctx.set_keypoints(fr["gt_uv"], fr["conf"], fr["joint_weights"])
        ctx.set_loss(body_prior=prior, frozen=("scale",), **w)
        x = torch.tensor(S.pack_params(fr["init"]), device="cuda")
        n0 = ctx.launch_count()
        o = ctx.closure(x, want_joints=True, want_proj=True)
        torch.cuda.synchronize()
        outs.append((o, ctx.launch_count() - n0))
        ctx.close()
    (a, na), (b, nb) = outs
    assert na == 1 and nb >= 5                    # one fused launch instead of the kernel chain
    for k in ("loss", "joints", "proj"):
        assert G.relmax(a[k].cpu().numpy(), b[k].cpu().numpy().astype(np.float64)) < 2e-6, k
    ga, gb = a["grad"].cpu().numpy(), b["grad"].cpu().numpy().astype(np.float64)
    for lo, hi in ((0, 10), (10, 13), (13, 82), (82, 85)):
        assert G.relmax(ga[:, lo:hi], gb[:, lo:hi]) < 2e-5, (lo, hi)
    assert (ga[:, 85] == 0).all()


def test_resident_lbfgs_matches_batched_lbfgs(syn_model, syn_gmm):
    cams = S.make_cameras(8)
    B = 40
    fr = S.make_frames(syn_model, cams, B, seed=77)
    w = dict(data_weight=500.0 / 1536, body_pose_weight=4.78, shape_weight=5.0, bending_prior_weight=3.17 * 4.78)
    res = []
    for mode in (0, 1):
        ctx = make_ctx(syn_model, cams, B, syn_gmm, mode)
        ctx.set_keypoints(fr["gt_uv"], fr["conf"], fr["joint_weights"])
        ctx.set_loss(body_prior="gmm", **w)
        x = torch.tensor(S.pack_params(fr["init"]), device="cuda")
        n0 = ctx.launch_count()
        final, st = ctx.lbfgs_run(x, ctx.make_lbfgs_config(max_outer=6))
        res.append((final.cpu().numpy(), st, x.cpu().numpy(), ctx.launch_count() - n0))
        ctx.close()
    (fa, sa, xa, la), (fb, sb, xb, lb) = res
    assert la <= 3 and lb > 50                    # the whole stage is one kernel launch (+ finalize)
    assert sa["frames_nan"] == 0
    # same optimiser on closures that differ in the last ulps: trajectories agree to tolerance (SURVEY H7)
    assert np.abs(fa - fb).max() / np.abs(fb).max() < 2e-3
    assert abs(sa["frame_evals"] - sb["frame_evals"]) <= sb["frame_evals"] // 10
    assert abs(sa["frame_iterations"] - sb["frame_iterations"]) <= sb["frame_iterations"] // 10
    assert np.median(np.abs(xa - xb).max(axis=1)) < 1e-2


def test_dense_regime_lbfgs_matches_batched_lbfgs(syn_model, syn_gmm):
    """SDF term on: posedirs_gemm_tc -> skin -> sdf_fused -> frame_step rounds against the batched kernel chain"""
    cams = S.make_cameras(4)
    B = 70
    fr = S.make_frames(syn_model, cams, B, seed=2)
    w = dict(data_weight=500.0 / 1536, body_pose_weight=57.4, shape_weight=10.0, bending_prior_weight=3.17 * 57.4)
    X0 = S.pack_params(fr["init"])
    res = []
    for mode in (0, 1):
        ctx = make_ctx(syn_model, cams, B, syn_gmm, mode)
        ctx.set_keypoints(fr["gt_uv"], fr["conf"], fr["joint_weights"])
        ctx.set_loss(body_prior="gmm", interpenetration=True, coll_loss_weight=1000.0, **w)
        x0 = torch.tensor(X0, device="cuda")
        c0 = ctx.closure(x0)                                   # batched chain in both modes (SDF closure)
        # (1) exactly one L-BFGS iteration: entry loss == closure loss, and the step taken is -t*g with the
        #     same gradient (first iteration is steepest descent, lbfgs_ls.py:312-317)
        x1 = x0.clone()
        f1, s1 = ctx.lbfgs_run(x1, ctx.make_lbfgs_config(max_outer=1, max_iter=1))
        # (2) a longer run
        x = x0.clone()
        final, st = ctx.lbfgs_run(x, ctx.make_lbfgs_config(max_outer=3))
        # the optimiser decreases ITS objective: in mode 0 that is the dense-regime kernels' (exec mode 3 evaluates one closure
        # through them).  The as-written SDF objective is discontinuous (parity of ray crossings per voxel), so the fp32 chain can
        # disagree by a voxel's worth of penetration at a point the optimiser parked next to a sign change.
        if mode == 0:
            ctx.set_exec_mode(3)
        l1 = ctx.closure(x, want_grad=False)["loss"].cpu().numpy()
        res.append(dict(l0=c0["loss"].cpu().numpy(), g0=c0["grad"].cpu().numpy(), f1=f1.cpu().numpy(),
                        x1=x1.cpu().numpy(), s1=s1, final=final.cpu().numpy(), st=st, l1=l1))
        ctx.close()
    a, b = res
    assert G.relmax(a["l0"], b["l0"].astype(np.float64)) < 1e-4        # same batched closure in both modes
    for r in (a, b):
        assert G.relmax(r["f1"], r["l0"].astype(np.float64)) < 1e-4        # loss at entry incl. the penetration term (two independent
        #                                                                     fp32-class evaluations: 3xTF32 tensor cores vs fp32 SIMT; measured 1e-5)
        bad = np.where(~(r["l1"] <= r["l0"] * (1 + 1e-4)))[0]
        assert r["st"]["frames_nan"] == 0 and bad.size == 0, (r is a, bad, r["l0"][bad], r["l1"][bad], r["final"][bad], r["f1"][bad])
    step_a, step_b = a["x1"] - X0, b["x1"] - X0
    moved = np.abs(step_b).max(axis=1) > 0
    assert moved.sum() >= B - 8
    # direction of the first step = -gradient in both paths
    cos = (step_a * step_b).sum(1) / (np.linalg.norm(step_a, axis=1) * np.linalg.norm(step_b, axis=1) + 1e-30)
    assert np.median(cos[moved]) > 0.9999
    gdir = -(a["g0"] * step_a).sum(1) / (np.linalg.norm(a["g0"], axis=1) * np.linalg.norm(step_a, axis=1) + 1e-30)
    assert np.median(gdir[moved]) > 0.9999
    # the penetration term is discontinuous: single frames may branch differently, the batch must agree in bulk
    assert abs(a["st"]["frame_evals"] - b["st"]["frame_evals"]) <= b["st"]["frame_evals"] // 4
    # (final losses are NOT compared: with a discontinuous term the two arithmetic paths legitimately end in
    #  different local minima for some frames; every single evaluation is what must agree, checked above)


# the configurations of test_gpu_dense_parity.py that sit inside the frame-resident envelope at one of its limits:
# 8 GMM components, 90 support vertices, kp_on = 0, sj_on = 0, 32 keypoints x 8 views, 16 views x 17 chain-joint keypoints
RESIDENT_LIMITS = ("gmm8", "sup90", "kpe_wide", "skin_dense", "K32_V8", "V16_smpl")


@pytest.mark.parametrize("name", RESIDENT_LIMITS)
def test_resident_lbfgs_first_step_at_the_limits_follows_float64_gradient(name, syn_model, syn_gmm):
    """lbfgs_resident_kernel through the same branches as the closure kernel: one L-BFGS iteration of frames 0-4 in exec
    mode 0.  The loss at entry must equal the frame-resident closure's loss, and the first step is steepest descent, so on
    every frame that moved it must point along the float64 oracle's negative gradient."""
    from tests import test_gpu_dense_parity as P
    case = P.config_case(syn_model, syn_gmm, name)
    assert case["branches"]["resident"], case["branches"]
    ref = P.oracle_case(case)
    B = P.B_SMALL
    ctx = P.case_ctx(case, B)
    ctx.set_keypoints(*P.batch_frames(case["fr"], range(B)), case["fr"]["joint_weights"])
    ctx.set_loss(**case["loss"])
    x0 = torch.tensor(case["X"][:B], device="cuda")
    c0 = ctx.closure(x0)["loss"].cpu().numpy()
    x1 = x0.clone()
    ctx.profile(0xFFFFFFFF)
    f1, st = ctx.lbfgs_run(x1, ctx.make_lbfgs_config(max_outer=1, max_iter=1))
    prof = ctx.profile_read()
    ctx.profile(0)
    f1, step = f1.cpu().numpy(), x1.cpu().numpy() - case["X"][:B]
    ctx.close()
    assert "lbfgs_resident" in prof and "keypoint_loss" not in prof, prof
    assert st["frames_nan"] == 0
    assert G.relmax(f1, c0.astype(np.float64)) < 1e-6, (f1, c0)
    moved = np.abs(step).max(axis=1) > 0
    assert moved.sum() >= B - 1, moved
    cos = []
    for i in np.flatnonzero(moved):
        g = ref[i]["grad"]
        cos.append(-(step[i] * g).sum() / (np.linalg.norm(step[i]) * np.linalg.norm(g)))
    print("[resident lbfgs %s] entry loss vs closure %.1e, cos(step, -grad64) min %.7f over %d frames" % (
        name, G.relmax(f1, c0.astype(np.float64)), min(cos), len(cos)))
    assert min(cos) > 0.9999, cos
