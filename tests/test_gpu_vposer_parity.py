"""GPU: the VPoser latent pose (use_vposer = 2) against the float64 oracle (oracle/closure_oracle.closure_eval_vposer) in
every kernel that decodes it, and the drop-in mode use_vposer = 1 in every closure regime.

The device decodes the latent code in four places: resident_closure (closure_resident_kernel, lbfgs_resident_kernel and
frame_step_kernel; its adjoint is vposer_decode_bwd), next_pose_forward inside frame_step_kernel (the next trial point),
frame_fwd_resident_kernel (every active slot at the start of a dense run and after each compaction) and
vposer_decode_kernel (mvs_vposer_decode).  The frames and latent codes come from tests/vposer_cases.py, whose CPU test
checks that the synthetic decoder's rotations reach all four quaternion branches and both signs of the quaternion's scalar
part, that no rotation lies near a branch surface or an angle of pi, and that the bending term straddles the 1e4 cut-off
the latent pose must not apply.

The oracle gets exactly the float32 constants the context uploads (model, cameras, decoder weights, parameters), widened
to float64.  Each frame is compared on its own: the loss relative to itself, every gradient segment (betas, orient, the 32
latent entries, transl, scale) relative to its own largest entry, joints and projections relative to the frame's largest
coordinate; the 37 pose entries behind the latent code must have an exactly zero gradient.

Each bar is about 4x the worst value measured on an NVIDIA H100 80GB HBM3 (700 W power limit), and never looser than 1e-4
without a written reason; the measured worst case is written next to it.  Every test prints its worst errors next to its
bars (run with -s).
"""
import numpy as np
import pytest
import torch

from oracle import closure_oracle as O
from tests import vposer_cases as VC
from tests.test_gpu_dense_parity import (B_LARGE, B_SMALL, BATCHES, CHECK_FRAMES, CW_SMALL, EDGE_FRAMES, FP32_NOISE,
                                         PARITY_REL, Worst, batch_frames, make_ctx, oracle_model)
from tests.test_gpu_lbfgs_transitions import Machine

pytestmark = pytest.mark.gpu

F64, F32 = torch.float64, torch.float32
SEGS = dict(betas=(0, 10), global_orient=(10, 13), latent=(13, 45), transl=(82, 85), scale=(85, 86))
SEGS_AA = dict(betas=(0, 10), global_orient=(10, 13), body_pose=(13, 82), transl=(82, 85), scale=(85, 86))
WEIGHTS = VC.stage_weights()

# ---- bars (measured worst on the H100 in the comment).  A gradient bar applies to the error relative to the segment's
# largest entry, plus FP32_NOISE times the float32 oracle's own deviation where compare() is given the float32 oracle.
BAR_LOSS = 4e-6            # A, B (SDF weight CW_SMALL), C (worst 8.8e-7)
BAR_GRAD = dict(betas=2e-5, global_orient=1e-4, latent=1.5e-5, transl=6e-5, scale=1e-4)
#                 A and B per segment (worst 4.3e-6, 3.7e-5, 3.6e-6, 1.5e-5, 1.15e-4 inside its float32 allowance)
BAR_JOINTS = 5e-6          # A: keypoints relative to the frame's largest |coordinate| (worst 1.4e-6)
BAR_PROJ = 6e-7            # A: projections relative to the frame's largest |uv| (worst 1.4e-7)
BAR_SDF_LOSS = 2e-5        # B, SDF weight 1000, plus FP32_NOISE x the float32 oracle's own deviation (worst 7.1e-5 with it)
BAR_SDF_ALLOWED = dict(betas=1.0, global_orient=1.0, latent=1.0, transl=1.0, scale=11.0)
#   B, SDF weight 1000: error over BAR_SDF_GRAD x the segment's largest entry + FP32_NOISE x the float32 oracle's deviation
#   (worst 0.29, 0.39, 0.36, 0.31, 2.74).  Scale: the penetration term's scale gradient cancels to rounding noise in exact
#   arithmetic (test_gpu_dense_parity, PARITY_REL / FP32_NOISE), and on frame 192 the float32 oracle lands closer to the
#   float64 value than the kernel's different summation order does; the loss and the other segments of that frame agree.
BAR_SDF_GRAD = 4e-4
# C: gradients at a fitted point are small residuals of cancelling terms, so each segment is far noisier relative to its
# own largest entry than at the starting point (worst 9.0e-5, 5.6e-4, 2.4e-5, 9.6e-4, 8.4e-4, plus the float32 allowance)
BAR_FIT_GRAD = dict(betas=4e-4, global_orient=2.5e-3, latent=1e-4, transl=4e-3, scale=4e-3)
BAR_COS_ALL = 1e-6         # D: 1 - cosine of the first step with the float64 -gradient (worst 1.3e-11)
BAR_COS_LATENT = 1e-5      # D: the same over the 32 latent entries (worst 4.6e-10)
BAR_ROT = 7e-5             # E: decoded rotation matrices, max |entry| (worst 1.6e-5, synthetic frame 203)
BAR_AA = 6e-5              # E: axis-angle / max(1, angle) (worst 1.4e-5)
BAR_V1_LOSS = 1.5e-6       # F (worst 3.3e-7)
BAR_V1_GRAD = dict(betas=3e-6, global_orient=1e-5, body_pose=4e-6, transl=5e-6, scale=2.5e-5)
#                 F per segment, exec modes 0, 1 and 3 (worst 6.9e-7, 2.1e-6, 8.1e-7, 1.0e-6, 6.1e-6)


def vp_ctx(model, gmm, case, B, mode=0):
    ctx = make_ctx(model, gmm, case["cams"], B, mode=mode)
    ctx.set_vposer(case["w"])
    return ctx


def loss_cfg(wname, cw=0.0):
    kw = dict(WEIGHTS[wname])
    if cw:
        kw.update(interpenetration=True, coll_loss_weight=cw, sdf_grid=128)
    return kw


_REF = {}


def oracle_vp(model, case, i, wname, cw=0.0, dtype=F64, body_pose=None):
    """closure_eval_vposer of frame i of a case, with the 86-vector gradient the device returns (latent code in 13:45)"""
    key = (case["decoder"], case["V"], i, wname, cw, dtype, body_pose is not None)
    if key not in _REF:
        om = oracle_model(model, "smpllsp", dtype)
        cfg = O.LossConfig(use_vposer=True, **loss_cfg(wname, cw))
        fr = case["fr"]
        r = O.closure_eval_vposer(om, cfg, O.OraclePriors("l2"), O.cams_to_torch(case["cams"], dtype), case["X"][i],
                                  case["Z"][i], case["w"], fr["gt_uv"][:, i], fr["conf"][:, i], fr["joint_weights"],
                                  body_pose=body_pose)
        g = np.zeros(86)
        g[0:10], g[10:13], g[13:45] = r["g_betas"], r["g_global_orient"], r["g_pose_embedding"]
        g[82:85], g[85:86] = r["g_transl"], r["g_scale"]
        r["grad"] = g
        _REF[key] = r
    return _REF[key]


def closure(ctx, x, mode, want_geom=False):
    ctx.set_exec_mode(mode)
    ctx.profile(0xFFFFFFFF)
    out = ctx.closure(torch.tensor(np.ascontiguousarray(x), device="cuda"), want_joints=want_geom, want_proj=want_geom)
    prof = ctx.profile_read()
    ctx.profile(0)
    res = dict(loss=out["loss"].cpu().numpy(), grad=out["grad"].cpu().numpy(), prof=prof)
    if want_geom:
        res.update(joints=out["joints"].cpu().numpy(), proj=out["proj"].cpu().numpy())
    return res


def compare(worst, tag, ref, loss, grad, where, bar_loss=BAR_LOSS, bar_grad=BAR_GRAD, segs=SEGS, ref32=None):
    """ref32: the float32 oracle of the same frame.  A gradient segment whose terms cancel (scale, whose data term is nearly
    invariant; every segment at a fitted point) is only resolved to the float32 oracle's own deviation: its bar is then
    bar_grad plus FP32_NOISE times that deviation (relative to the segment's largest entry), as in test_gpu_dense_parity"""
    worst.add(tag + " loss", abs(float(loss) - ref["loss"]) / abs(ref["loss"]), bar_loss, where)
    for n, (a, e) in segs.items():
        top = np.abs(ref["grad"][a:e]).max()
        bar = bar_grad[n]
        if ref32 is not None:
            bar += FP32_NOISE * float(np.abs(ref32["grad"][a:e] - ref["grad"][a:e]).max() / top)
        worst.add(tag + " grad " + n, float(np.abs(grad[a:e] - ref["grad"][a:e]).max() / top), bar, where)
    if segs is SEGS:
        assert np.all(grad[45:82] == 0.0), (tag, where, "pose entries behind the latent code must have a zero gradient")


# ----------------------------------------------------------------------------------------------------------------- A
@pytest.mark.parametrize("V", [1, 2, 4, 16])
@pytest.mark.parametrize("decoder", VC.DECODERS)
def test_resident_closure_matches_float64(decoder, V, syn_model, syn_gmm):
    """closure_resident_kernel (exec mode 0, no SDF term): loss, every gradient segment, joints and projections of the
    checked frames at B = 5 and 40, at each stage-weight set (w0, w3 of the VPoser fixtures and body_pose_weight 57.4)"""
    case = VC.make_case(decoder, V=V, n=B_LARGE)
    worst = Worst("A %s V=%d" % (decoder, V))
    for B in (B_SMALL, B_LARGE):
        ctx = vp_ctx(syn_model, syn_gmm, case, B)
        ctx.set_keypoints(*batch_frames(case["fr"], range(B)), case["fr"]["joint_weights"])
        for wname in WEIGHTS:
            ctx.set_loss(body_prior="l2", use_vposer=2, **loss_cfg(wname))
            res = closure(ctx, case["X"][:B], 0, want_geom=True)
            assert "closure_resident" in res["prof"] and "keypoint_loss" not in res["prof"], res["prof"]
            for i in (i for i in CHECK_FRAMES if i < B):
                ref = oracle_vp(syn_model, case, i, wname)
                compare(worst, wname, ref, res["loss"][i], res["grad"][i], (B, i), ref32=oracle_vp(syn_model, case, i, wname, dtype=F32))
                jo, po = ref["joints"], ref["proj"]
                worst.add("joints", float(np.abs(res["joints"][i] - jo).max() / np.abs(jo).max()), BAR_JOINTS, (wname, B, i))
                worst.add("proj", float(np.abs(res["proj"][:, i] - po).max() / np.abs(po).max()), BAR_PROJ, (wname, B, i))
        ctx.close()
    worst.report()


# ----------------------------------------------------------------------------------------------------------------- B
@pytest.mark.parametrize("decoder,sdf", [("synthetic", "small"), ("snapshot", "small"), ("synthetic", "real")])
def test_dense_closure_matches_float64_at_every_batch_size(decoder, sdf, syn_model, syn_gmm):
    """Exec mode 3 (posedirs_gemm_tc -> skin -> sdf_setup -> sdf_fused -> frame_step, the pose decoded by
    frame_fwd_resident_kernel and the adjoint through vposer_decode_bwd) at every kernel-selection batch size, body_pose_weight
    57.4.  Every frame must give the same bits in the batch reversed, every edge frame the same bits alone (B = 1).  With the
    SDF weight CW_SMALL the oracle's penetration stays below 1e-7 of every compared loss (asserted): the data, prior and
    decoder arithmetic alone is compared.  With the real weight (1000, grid 128) a frame is left out only where the oracle's
    own float32 and float64 penetration differ by more than PARITY_REL, and a gradient segment may differ by BAR_SDF_GRAD
    times its largest entry plus FP32_NOISE times the float32 oracle's own deviation (test_gpu_dense_parity)."""
    case = VC.make_case(decoder)
    cw = CW_SMALL if sdf == "small" else 1000.0
    fr, X = case["fr"], case["X"]
    ref, excluded, allow = {}, [], {}
    for i in EDGE_FRAMES:
        r = oracle_vp(syn_model, case, i, "s2", cw)
        p64 = r["terms"]["pen"]
        if sdf == "small":
            assert p64 < 1e-7 * r["loss"], (i, p64, r["loss"])
        else:
            r32 = oracle_vp(syn_model, case, i, "s2", cw, dtype=F32)
            p32 = r32["terms"]["pen"]
            if abs(p32 - p64) > PARITY_REL * abs(p64) and p32 != p64:
                excluded.append(i)
                continue
            r = dict(r, bar_loss=BAR_SDF_LOSS + FP32_NOISE * abs(r32["loss"] - r["loss"]) / abs(r["loss"]))
            allow[i] = {n: BAR_SDF_GRAD * np.abs(r["grad"][a:e]).max() + FP32_NOISE * np.abs(r32["grad"][a:e] - r["grad"][a:e]).max()
                        for n, (a, e) in SEGS.items()}
        ref[i] = dict(r, pen=p64)
    if sdf == "real":
        print("[B %s real] oracle-compared edge frames %d, excluded %d %s" % (decoder, len(ref), len(excluded), excluded))
        assert len(ref) >= 0.9 * len(EDGE_FRAMES), excluded
        assert sum(r["pen"] > 0 for r in ref.values()) >= 3, "the compared frames must penetrate"
    kw = dict(body_prior="l2", use_vposer=2, **loss_cfg("s2", cw))
    alone = {}
    ctx = vp_ctx(syn_model, syn_gmm, case, 1, mode=3)
    ctx.set_loss(**kw)
    for i in EDGE_FRAMES:
        ctx.set_keypoints(*batch_frames(fr, [i]), fr["joint_weights"])
        res = closure(ctx, X[i:i + 1], 3)
        alone[i] = (res["loss"][0], res["grad"][0])
    ctx.close()
    worst = Worst("B %s %s" % (decoder, sdf))
    for B in BATCHES:
        ctx = vp_ctx(syn_model, syn_gmm, case, B, mode=3)
        ctx.set_loss(**kw)
        out = {}
        for name, order in (("id", np.arange(B)), ("rev", np.arange(B)[::-1].copy())):
            ctx.set_keypoints(*batch_frames(fr, order), fr["joint_weights"])
            res = closure(ctx, X[order], 3)
            prof = res["prof"]
            # skin_small_kernel (B <= 8) and skin_kernel share the "skin" id; at B <= 4 skin_small builds the SDF set-up itself
            assert prof.get("frame_step", (0, 0))[1] == 1 and prof.get("skin", (0, 0))[1] == 1, prof
            assert ("sdf_setup" in prof) == (B > 4), (B, prof)
            assert "keypoint_loss" not in prof and "closure_resident" not in prof, prof
            inv = np.argsort(order)
            out[name] = (res["loss"][inv], res["grad"][inv])
        ctx.close()
        loss, grad = out["id"]
        assert np.isfinite(loss).all() and np.isfinite(grad).all(), B
        same = (loss == out["rev"][0]) & (grad == out["rev"][1]).all(1)
        assert same.all(), ("reversed batch", B, np.flatnonzero(~same)[:8])
        for i in (i for i in EDGE_FRAMES if i < B):
            assert loss[i] == alone[i][0] and np.array_equal(grad[i], alone[i][1]), ("alone", B, i)
            if i not in ref:
                continue
            if sdf == "small":
                compare(worst, "mode3", ref[i], loss[i], grad[i], (B, i), ref32=oracle_vp(syn_model, case, i, "s2", cw, dtype=F32))
                continue
            worst.add("loss", abs(float(loss[i]) - ref[i]["loss"]) / abs(ref[i]["loss"]), ref[i]["bar_loss"], (B, i))
            for n, (a, e) in SEGS.items():
                worst.add("grad %s / allowed" % n, float(np.abs(grad[i, a:e] - ref[i]["grad"][a:e]).max() / allow[i][n]),
                      BAR_SDF_ALLOWED[n], (B, i))
            assert np.all(grad[i, 45:82] == 0.0), (B, i)
    worst.report()


# ----------------------------------------------------------------------------------------------------------------- C
def test_dense_run_holds_the_evaluation_at_the_returned_parameters(syn_model, syn_gmm):
    """lbfgs_run in the dense regime (SDF weight CW_SMALL), B = 40, long enough for several compactions, on frames that
    finish at different rounds.  A frame's optimiser state holds the loss and gradient of the point it returned: evaluated
    by frame_step at a trial point decoded by next_pose_forward, or by frame_fwd_resident_kernel after a compaction.  They
    must be bit-identical to a mode-3 closure at the returned parameters (decoded by frame_fwd_resident_kernel at the run's
    start), and both within the bars of test B of float64."""
    case = VC.make_case("synthetic", n=B_LARGE)
    B = B_LARGE
    ctx = vp_ctx(syn_model, syn_gmm, case, B, mode=3)
    ctx.set_keypoints(*batch_frames(case["fr"], range(B)), case["fr"]["joint_weights"])
    ctx.set_loss(body_prior="l2", use_vposer=2, **loss_cfg("s2", CW_SMALL))
    x = torch.tensor(case["X"][:B], device="cuda")
    ctx.profile(0xFFFFFFFF)
    _, st = ctx.lbfgs_run(x, ctx.make_lbfgs_config(max_outer=4, max_iter=10))
    prof = ctx.profile_read()
    ctx.profile(0)
    assert "frame_step" in prof and "lbfgs_resident" not in prof, prof
    sc, arrs = Machine(ctx, 100).read()
    evals = np.array([s.evals for s in sc])
    print("[C] dense rounds %d, evaluations per frame %d .. %d, compactions %d" % (
        st["dense_rounds"], evals.min(), evals.max(), prof["lbfgs_compact"][1]))
    assert evals.max() > 16 and len(set(evals.tolist())) > 3, evals
    assert prof["lbfgs_compact"][1] >= 2, prof
    xr = x.cpu().numpy()
    assert np.array_equal(xr[:, 45:82], case["X"][:B, 45:82]) and not np.array_equal(xr[:, 13:45], case["X"][:B, 13:45])
    held_loss = np.array([s.loss for s in sc], np.float32)
    res = closure(ctx, xr, 3)
    ctx.close()
    same = (held_loss == res["loss"]) & (arrs["g"] == res["grad"]).all(1)
    assert same.all(), ("state differs from the closure at x", np.flatnonzero(~same)[:8],
                        np.abs(held_loss - res["loss"]).max(), np.abs(arrs["g"] - res["grad"]).max())
    worst = Worst("C")
    moved = dict(case, X=xr, Z=xr[:, 13:45].copy())
    for i in CHECK_FRAMES:
        fitted = dict(moved, decoder="synthetic-fitted")
        ref = oracle_vp(syn_model, fitted, i, "s2", CW_SMALL)
        compare(worst, "fitted", ref, res["loss"][i], res["grad"][i], i, bar_grad=BAR_FIT_GRAD,
                ref32=oracle_vp(syn_model, fitted, i, "s2", CW_SMALL, dtype=F32))
    worst.report()


# ----------------------------------------------------------------------------------------------------------------- D
@pytest.mark.parametrize("decoder", VC.DECODERS)
def test_first_resident_step_follows_the_float64_gradient(decoder, syn_model, syn_gmm):
    """one iteration of lbfgs_resident_kernel (max_outer = max_iter = 1) per frame: its first step is t * (-g), so the step
    taken must point along the float64 negative gradient, over the whole 86-vector and over the 32 latent entries alone"""
    case = VC.make_case(decoder, n=B_LARGE)
    B = B_LARGE
    ctx = vp_ctx(syn_model, syn_gmm, case, B)
    ctx.set_keypoints(*batch_frames(case["fr"], range(B)), case["fr"]["joint_weights"])
    worst = Worst("D " + decoder)
    for wname in WEIGHTS:
        ctx.set_loss(body_prior="l2", use_vposer=2, **loss_cfg(wname))
        x = torch.tensor(case["X"][:B], device="cuda")
        ctx.profile(0xFFFFFFFF)
        ctx.lbfgs_run(x, ctx.make_lbfgs_config(max_outer=1, max_iter=1))
        prof = ctx.profile_read()
        ctx.profile(0)
        assert prof.get("lbfgs_resident", (0, 0))[1] == 1, prof
        d = x.cpu().numpy().astype(np.float64) - case["X"][:B]
        assert (d[:, 45:82] == 0).all()
        moved = np.abs(d).max(axis=1) > 0
        assert moved[list(CHECK_FRAMES)].all(), (wname, "frames that did not step", np.flatnonzero(~moved))
        for i in CHECK_FRAMES:
            g = -oracle_vp(syn_model, case, i, wname)["grad"]
            cos = lambda a, b: float(a @ b / (np.linalg.norm(a) * np.linalg.norm(b)))
            worst.add("1 - cos all", 1.0 - cos(d[i], g), BAR_COS_ALL, (wname, i))
            worst.add("1 - cos latent", 1.0 - cos(d[i, 13:45], g[13:45]), BAR_COS_LATENT, (wname, i))
    ctx.close()
    worst.report()


# ----------------------------------------------------------------------------------------------------------------- E
def _rotmat(aa):
    """Rodrigues in float64, aa [..., 3] -> [..., 3, 3]"""
    th = np.linalg.norm(aa, axis=-1)[..., None, None]
    k = aa / np.maximum(np.linalg.norm(aa, axis=-1, keepdims=True), 1e-300)
    K = np.zeros(aa.shape[:-1] + (3, 3))
    K[..., 0, 1], K[..., 0, 2], K[..., 1, 2] = -k[..., 2], k[..., 1], -k[..., 0]
    K = K - np.swapaxes(K, -1, -2)
    return np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * (K @ K)


@pytest.mark.parametrize("decoder", VC.DECODERS)
def test_vposer_decode_entry_point_matches_float64(decoder, syn_model):
    """mvs_vposer_decode at B = 1, 33 and 257: every decoded joint rotation against the float64 decode, and the axis-angle
    itself (no rotation of the cases lies within 1e-2 of an angle of pi, where the axis flips); frame i decodes to the
    same bits at every B"""
    from mvsmplfitting_b200.context import FittingContext
    case = VC.make_case(decoder)
    ref = case["pose"].reshape(-1, 23, 3)
    assert (np.pi - np.linalg.norm(ref, axis=2)).min() > VC.PI_MARGIN
    Rref = _rotmat(ref)
    worst = Worst("E " + decoder)
    first = None
    for B in (1, 33, 257):
        ctx = FittingContext(0)
        ctx.set_model(syn_model)
        ctx.set_vposer(case["w"])
        ctx.set_batch(B)
        aa = ctx.vposer_decode(torch.tensor(case["X"][:B], device="cuda")).cpu().numpy().reshape(B, 23, 3)
        ctx.close()
        first = aa[0] if first is None else first
        assert np.array_equal(aa[0], first), B
        worst.add("rotation", float(np.abs(_rotmat(aa.astype(np.float64)) - Rref[:B]).max()), BAR_ROT, B)
        err = np.abs(aa - ref[:B]).max(axis=2) / np.maximum(1.0, np.linalg.norm(ref[:B], axis=2))
        worst.add("axis-angle / max(1, angle)", float(err.max()), BAR_AA, (B, np.unravel_index(err.argmax(), err.shape)))
    worst.report()


# ----------------------------------------------------------------------------------------------------------------- F
def test_dropin_decoded_pose_matches_float64_in_every_regime(syn_model, syn_gmm):
    """use_vposer = 1: the caller decodes the pose into the pose slot and owns the |z|^2 prior.  Exec modes 0
    (closure_resident_kernel), 1 (the batched chain, whose prior block runs in frame_bwd_kernel) and 3 (the dense closure,
    SDF weight CW_SMALL): the loss must be the oracle's total minus bpw^2 |z|^2 and the pose gradient the oracle's gradient
    with respect to the decoded pose.  The checked frames lie on both sides of the 1e4 bending cut-off at body_pose_weight
    57.4, which the drop-in mode must not apply either."""
    case = VC.make_case("synthetic", n=B_LARGE)
    B = B_LARGE
    pose32 = case["pose"][:B].astype(np.float32)
    X1 = case["X"][:B].copy()
    X1[:, 13:82] = pose32
    sw = WEIGHTS["s2"]
    bend = VC.angle_sum(pose32[list(CHECK_FRAMES)].astype(np.float64)) * sw["bending_prior_weight"]
    assert (bend > VC.ANGLE_CUT).sum() >= 3 and (bend < VC.ANGLE_CUT).sum() >= 3, bend
    worst = Worst("F")
    for mode, cw, kid in ((0, 0.0, "closure_resident"), (1, 0.0, "frame_bwd"), (3, CW_SMALL, "frame_step")):
        ctx = make_ctx(syn_model, syn_gmm, case["cams"], B, mode=mode)
        ctx.set_keypoints(*batch_frames(case["fr"], range(B)), case["fr"]["joint_weights"])
        ctx.set_loss(body_prior="l2", use_vposer=1, **loss_cfg("s2", cw))
        res = closure(ctx, X1, mode)
        ctx.close()
        assert kid in res["prof"], (mode, res["prof"])
        for i in CHECK_FRAMES:
            r = oracle_vp(syn_model, case, i, "s2", cw, body_pose=pose32[i].astype(np.float64))
            zz = float((case["Z"][i].astype(np.float64) ** 2).sum()) * sw["body_pose_weight"] ** 2
            g = r["grad"].copy()
            g[13:82] = r["g_body_pose"]
            compare(worst, "mode%d" % mode, dict(loss=r["loss"] - zz, grad=g), res["loss"][i], res["grad"][i], i,
                    BAR_V1_LOSS, BAR_V1_GRAD, SEGS_AA)
    worst.report()
