"""GPU: the 3-D joint term (mvs_set_joints3d, SMPLifyLoss(use_3d=True)) in every execution path, against the reference-run
fixtures of oracle/make_golden_3d.py (tests/golden/joints3d_*.npz).

Bars are the project's parity bar (1e-4 relative, max-norm per tensor); the worst value measured on the H100 is printed by
every comparison (run with -s) and written next to the bar."""
import json
import os

import numpy as np
import pytest
import torch

from mvsmplfitting_b200 import synthetic as S
from tests import golden_util as G
from tests.test_joints3d_golden import CASES, load

pytestmark = pytest.mark.gpu

TOL = 1e-4                 # parity bar; worst measured on an H100 80GB HBM3 (400 W): exec mode 0 2.7e-6 (scale gradient),
                           # mode 1 2.3e-6 (body_pose gradient), mode 3 1.1e-5 (global_orient gradient)
TOL_SATURATED = 1e-3       # gmm1_rho: rho = 0.05 saturates the 2-D GMoF too, so the scale / betas gradients are cancellations
                           # of near-zero terms in float32; measured 2.1e-4 in exec modes 0 and 1 on the same card
SEGS = dict(betas=(0, 10), global_orient=(10, 13), body_pose=(13, 82), transl=(82, 85), scale=(85, 86))
CW_SMALL = 3e-3            # SDF term on in exec mode 3, its value far below the compared losses (test_gpu_dense_parity.py)
SW = S.STAGE_WEIGHTS


def make_ctx(model, gmm, cams, B, model_type="smpllsp", mode=0):
    from mvsmplfitting_b200.context import FittingContext
    ctx = FittingContext(0)
    ctx.set_model(model, model_type=model_type)
    ctx.set_gmm_from_dict(gmm)
    ctx.set_cameras(cams["R"], cams["t"], cams["f"], cams["c"])
    ctx.set_batch(B)
    ctx.set_exec_mode(mode)
    return ctx


def case_loss(c, sdf):
    kw = dict(c["w"], body_prior=c["meta"]["body_prior"], rho=float(c["rho"]), fix_shape=c["meta"]["fix_shape"],
              frozen=("betas",) if c["meta"]["fix_shape"] else (), use_vposer=2 if c["meta"].get("use_vposer") else 0)
    if sdf:
        kw.update(interpenetration=True, coll_loss_weight=CW_SMALL, sdf_grid=128)
    return kw


def run_case(c, model, gmm, mode, conf3d=None, enable=True, perm=None):
    B = c["X"].shape[0]
    p = np.arange(B) if perm is None else np.asarray(perm)
    ctx = make_ctx(model, gmm, c["cams"], B, c["meta"]["model_type"], mode)
    ctx.set_keypoints(c["gt_uv"][:, p], c["conf"][:, p], c["joint_weights"])
    X = c["X"].copy()
    if c["meta"].get("use_vposer"):              # the latent code in the pose slot, decoded on the device (use_vposer = 2)
        ctx.set_vposer(G.snapshot_vposer_weights())
        X[:, 13:82] = 0.0
        X[:, 13:45] = c["Z"]
    if enable:
        ctx.set_joints3d(c["gt3d"][p], (c["conf3d"] if conf3d is None else conf3d)[p])
    ctx.set_loss(**case_loss(c, mode == 3))
    ctx.profile(0xFFFFFFFF)
    out = ctx.closure(torch.tensor(X[p], device="cuda"), want_joints=mode != 3)    # mode 3 serves loss and gradient only
    prof = ctx.profile_read()
    res = {k: v.cpu().numpy() for k, v in out.items()}
    ctx.close()
    return res, prof


@pytest.mark.parametrize("mode", [0, 1, 3])
@pytest.mark.parametrize("name", CASES)
def test_closure_matches_reference_fixture(name, mode, syn_model, syn_gmm):
    c = load(name)
    if mode == 1 and c["meta"].get("use_vposer"):
        pytest.skip("the batched reference chain has no device decoder (use_vposer = 2, include/mvsmpl.h)")
    if mode == 3 and name == "gmm1_rho":
        # its gradient is so small (both GMoF terms saturated) that the small SDF term exec mode 3 needs, and which the fixture
        # lacks, is visible in it (measured 8e-3 on betas / global_orient); gmm1_3donly_rho covers the saturated 3-D term there
        pytest.skip("gradient below the SDF term's")
    r, prof = run_case(c, syn_model, syn_gmm, mode)
    if mode == 3:
        assert prof.get("frame_step", (0, 0))[1] == 1 and "keypoint_loss" not in prof, prof
    elif mode == 1:
        assert "keypoint_loss" in prof, prof
    else:
        assert "closure_resident" in prof, prof
    worst = {}
    for tag in ("f64", "f32"):
        worst["loss " + tag] = G.relmax(r["loss"], c["loss_" + tag])
        for n, (a, e) in SEGS.items():
            if np.abs(c["grad_" + tag][:, a:e]).max() > 0:
                worst["grad %s %s" % (n, tag)] = G.relmax(r["grad"][:, a:e], c["grad_" + tag][:, a:e])
        if "joints" in r:
            worst["joints " + tag] = G.relmax(r["joints"], c["joints_" + tag])
    print("\n[%s mode %d] worst %s" % (name, mode, json.dumps({k: "%.2e" % v for k, v in worst.items()})))
    assert max(worst.values()) < (TOL_SATURATED if name == "gmm1_rho" else TOL), worst


@pytest.mark.parametrize("mode", [0, 1, 3])
def test_zero_confidence_is_bitwise_the_term_off(mode, syn_model, syn_gmm):
    c = load("gmm4_s3")
    on, _ = run_case(c, syn_model, syn_gmm, mode, conf3d=np.zeros_like(c["conf3d"]))
    off, _ = run_case(c, syn_model, syn_gmm, mode, enable=False)
    assert np.array_equal(on["loss"], off["loss"]) and np.array_equal(on["grad"], off["grad"])
    full, _ = run_case(c, syn_model, syn_gmm, mode)
    assert not np.array_equal(full["loss"], off["loss"])            # and the term does reach the result when on


def test_permuted_batch_gives_the_same_bits_per_frame_mode3(syn_model, syn_gmm):
    c = load("l2_4_scale")
    B = c["X"].shape[0]
    perm = np.roll(np.arange(B), 1)
    a, _ = run_case(c, syn_model, syn_gmm, 3)
    b, _ = run_case(c, syn_model, syn_gmm, 3, perm=perm)
    assert np.array_equal(a["loss"][perm], b["loss"]) and np.array_equal(a["grad"][perm], b["grad"])


def stage_cfgs(ctx, sdf_from=None):
    return [ctx.make_loss_config(body_prior="gmm", data_weight=500.0 / 1536, body_pose_weight=SW["body_pose_prior_weights"][i],
                                 shape_weight=SW["shape_weights"][i], bending_prior_weight=3.17 * SW["body_pose_prior_weights"][i],
                                 interpenetration=sdf_from is not None and i >= sdf_from, sdf_grid=128,
                                 coll_loss_weight=SW["coll_loss_weights"][i]) for i in range(4)]


def fit(model, gmm, cams, fr, X0, gt3d, conf3d, mode=0, sdf_from=None):
    B = X0.shape[0]
    ctx = make_ctx(model, gmm, cams, B, mode=mode)
    ctx.set_keypoints(fr["gt_uv"], fr["conf"], fr["joint_weights"])
    ctx.set_joints3d(gt3d, conf3d)
    x = torch.tensor(X0, device="cuda")
    final, st = ctx.fit(x, stage_cfgs(ctx, sdf_from))
    out = final.cpu().numpy(), x.cpu().numpy(), st
    ctx.close()
    return out


def fit_inputs(model, B, V, seed):
    from oracle.make_golden_3d import targets
    cams = {k: v[:V] for k, v in S.make_cameras(4).items() if isinstance(v, np.ndarray)}
    fr = S.make_frames(model, cams, B, seed=seed)
    return cams, fr, S.pack_params(fr["init"]), *targets(fr, seed + 1)


def test_fit_with_sdf_is_frame_indexed_through_compaction(syn_model, syn_gmm):
    """4-stage mvs_fit, SDF term in stages 2-3, B = 33 (crosses a compaction and a posedirs N-instance change): every frame's
    result is bitwise the same when the batch, detections and 3-D targets are permuted together"""
    cams, fr, X0, gt3d, conf3d = fit_inputs(syn_model, 33, 4, 4400)
    perm = np.random.RandomState(0).permutation(33)
    fa, xa, _ = fit(syn_model, syn_gmm, cams, fr, X0, gt3d, conf3d, sdf_from=2)
    frp = dict(fr, gt_uv=fr["gt_uv"][:, perm], conf=fr["conf"][:, perm])
    fb, xb, _ = fit(syn_model, syn_gmm, cams, frp, X0[perm], gt3d[perm], conf3d[perm], sdf_from=2)
    assert np.array_equal(fa[perm], fb) and np.array_equal(xa[perm], xb)


def test_merged_stages_equal_stage_barriers_bitwise(syn_model, syn_gmm):
    cams, fr, X0, gt3d, conf3d = fit_inputs(syn_model, 24, 4, 4410)
    fa, xa, sa = fit(syn_model, syn_gmm, cams, fr, X0, gt3d, conf3d, mode=0)
    fb, xb, sb = fit(syn_model, syn_gmm, cams, fr, X0, gt3d, conf3d, mode=2)
    assert np.array_equal(fa, fb) and np.array_equal(xa, xb)
    assert sa["frame_iterations"] == sb["frame_iterations"]


def test_lbfgs_step_runs_with_the_term(syn_model, syn_gmm):
    c = load("l2_4_3donly")
    B = c["X"].shape[0]
    ctx = make_ctx(syn_model, syn_gmm, c["cams"], B)
    ctx.set_keypoints(c["gt_uv"], c["conf"], c["joint_weights"])
    ctx.set_joints3d(c["gt3d"], c["conf3d"])
    ctx.set_loss(**case_loss(c, False))
    x = torch.tensor(c["X"], device="cuda")
    l0, _, _ = ctx.lbfgs_step(x, reset=True)
    for _ in range(5):
        l1, g, _ = ctx.lbfgs_step(x)
    l0, l1 = l0.cpu().numpy(), l1.cpu().numpy()
    ctx.close()
    assert np.allclose(l0, c["loss_f64"], rtol=TOL)                  # the loss at entry is the fixture's closure
    assert np.isfinite(l1).all() and (l1 < l0).all()


@pytest.mark.parametrize("tag", ["v4", "v1"])
def test_four_stage_fit_matches_reference_runs(tag, syn_model, syn_gmm):
    z = np.load(os.path.join(G.GOLD, "joints3d_fit_e2e.npz"))
    V, seed = int(z[tag + "_V"]), int(z[tag + "_seed"])
    cams, fr, X0, gt3d, conf3d = fit_inputs(syn_model, 8, V, seed)
    assert np.array_equal(X0, z[tag + "_X0"]) and np.array_equal(gt3d, z[tag + "_gt3d"])
    conf3d = conf3d.copy()
    conf3d[:, [11, 12]] = 0.0                                       # what the reference's solver does without use_hip
    final, x, st = fit(syn_model, syn_gmm, cams, fr, X0, gt3d, conf3d)
    ref_final = z[tag + "_final_loss"]
    it, ref_it = st["frame_iterations"] / 8, z[tag + "_iterations"].sum(1).mean()
    rel = np.abs(final - ref_final) / ref_final
    # the device closure at the reference's final parameters (last stage) reproduces the loss the reference reported there
    ctx = make_ctx(syn_model, syn_gmm, cams, 8)
    ctx.set_keypoints(fr["gt_uv"], fr["conf"], fr["joint_weights"])
    ctx.set_joints3d(gt3d, conf3d)
    ctx.set_loss(config=stage_cfgs(ctx)[3])
    at_ref = ctx.closure(torch.tensor(z[tag + "_params"], device="cuda"), want_grad=False)["loss"].cpu().numpy()
    ctx.close()
    rel_at = np.abs(at_ref - ref_final) / ref_final
    print("[e2e %s] iterations/frame device %.2f reference %.2f; final rel median %.2e max %.2e; at reference params max %.2e"
          % (tag, it, ref_it, np.median(rel), rel.max(), rel_at.max()))
    # measured on an H100 80GB HBM3 (400 W): iterations 2.1 % (v4) and 4.9 % (v1) below the reference; final losses at most
    # 8.9e-6 relative (median 1.8e-7); at the reference's parameters at most 2.5e-7
    assert abs(it - ref_it) / ref_it < 0.20, (it, ref_it)
    assert rel.max() < 4e-5, rel
    assert abs(final.mean() - ref_final.mean()) / ref_final.mean() < 4e-5
    assert rel_at.max() < 1e-6, rel_at


@pytest.mark.parametrize("V", [4, 1])
def test_init_guess_aligns_to_the_targets(V, syn_model, syn_gmm):
    """mvs_init_guess with the term on: the torso of the rest joints aligned to the targets' torso, not to the views
    (init_guess.py:85-86); one launch per repeated call.  The link to the reference's own run (joints3d_init.npz) is
    indirect, as in test_gpu_zz_init.py: the file's as-written alignment depends on the sign convention of the SVD behind
    numpy, so test_joints3d_golden.py pins the fixture to oracle/init_oracle.py under numpy's SVD, and this test pins the
    device to the same restatement under the convention the device implements, to test_gpu_zz_init.py's tolerances."""
    from oracle import init_oracle as IO
    g = np.load(os.path.join(G.GOLD, "joints3d_init.npz"))
    tag = "mv4" if V == 4 else "sv"
    cams = {k: v[:V] for k, v in S.make_cameras(4).items() if isinstance(v, np.ndarray)}
    fr = S.make_frames(syn_model, cams, 4, seed=int(g[tag + "_seed"]))
    ctx = make_ctx(syn_model, syn_gmm, cams, 4)
    ctx.set_keypoints(fr["gt_uv"], fr["conf"], fr["joint_weights"])
    ctx.set_joints3d(g[tag + "_gt3d"], g[tag + "_conf3d"])
    params, j3 = ctx.init_guess(estimate_scale=True, use_torso=True, umeyama_as_written=True)
    n0 = ctx.launch_count()
    ctx.init_guess(estimate_scale=True, use_torso=True, umeyama_as_written=True)
    torch.cuda.synchronize()
    assert ctx.launch_count() - n0 == 1
    params, j3 = params.cpu().numpy(), j3.cpu().numpy()
    ctx.close()
    assert np.array_equal(j3, g[tag + "_gt3d"])                       # the alignment target is the annotations
    z = lambda n: np.zeros((1, n))
    rest = S.model_keypoints_np(syn_model, z(10), z(3), z(69), z(3), np.ones((1, 1)), "smpllsp")[0].astype(np.float64)
    torso = [5, 6, 11, 12]
    for b in range(4):
        rot, tr, sc = IO.umeyama_as_written(rest[torso], g[tag + "_gt3d"][b].astype(np.float64)[torso], True,
                                            svd=IO.svd_sign_normalised)
        x = params[b]
        assert np.abs(x[10:13] - IO.rotmat_to_aa(rot)).max() < 2e-3
        assert np.abs(x[82:85] - np.reshape(tr, -1)).max() < 2e-3 * max(1.0, np.abs(tr).max())
        assert abs(x[85] - sc) < 1e-3 * sc
        assert (x[:10] == 0).all() and (x[13:19] == 1).all() and (x[19:82] == 0).all()


def test_dropin_init_guess_with_3d_joints(syn_model, syn_gmm, tmp_path):
    """utils.init_guess(setting, data, use_3d=True) with data['3d_joint'] (the reference's call, main.py:77): the model is
    aligned to the annotations, and the model's context has the term off again afterwards"""
    from mvsmplfitting_b200.fitting import model_context
    from mvsmplfitting_b200.utils import init_guess as IG
    from oracle import init_oracle as IO
    from tests.test_gpu_dropin import build_scene
    g = np.load(os.path.join(G.GOLD, "joints3d_init.npz"))
    cams = S.make_cameras(4)
    fr = S.make_frames(syn_model, cams, 4, seed=int(g["mv4_seed"]))
    model, _, _ = build_scene(syn_model, syn_gmm, tmp_path, cams, 1)
    ext = np.tile(np.eye(4), (4, 1, 1))
    ext[:, :3, :3], ext[:, :3, 3] = cams["R"], cams["t"]
    intr = np.tile(np.eye(3), (4, 1, 1))
    intr[:, 0, 0], intr[:, 1, 1], intr[:, 0, 2], intr[:, 1, 2] = cams["f"][:, 0], cams["f"][:, 1], cams["c"][:, 0], cams["c"][:, 1]
    z = lambda n: np.zeros((1, n))
    rest = S.model_keypoints_np(syn_model, z(10), z(3), z(69), z(3), np.ones((1, 1)), "smpllsp")[0].astype(np.float64)
    for b in range(2):
        kps = [np.concatenate([fr["gt_uv"][v, b], fr["conf"][v, b][:, None]], axis=1)[None] for v in range(4)]
        data = {"keypoints": kps, "3d_joint": [np.concatenate([g["mv4_gt3d"][b], g["mv4_conf3d"][b][:, None]], axis=1)]}
        setting = dict(model=model, dtype=torch.float32, extris=ext, intris=intr, fix_scale=False, fixed_scale=None)
        IG.init_guess(setting, data, use_torso=True, use_3d=True, model_type="smpllsp", umeyama_as_written=True)
        rot, tr, sc = IO.umeyama_as_written(rest[[5, 6, 11, 12]], g["mv4_gt3d"][b].astype(np.float64)[[5, 6, 11, 12]], True,
                                            svd=IO.svd_sign_normalised)
        assert np.abs(model.global_orient.detach().cpu().numpy().reshape(-1) - IO.rotmat_to_aa(rot)).max() < 2e-3
        assert np.abs(model.transl.detach().cpu().numpy().reshape(-1) - np.reshape(tr, -1)).max() < 2e-3
        assert abs(float(model.scale.detach().reshape(-1)[0]) - sc) < 1e-3 * sc
        assert model_context(model)._j3d_keep is None


def test_dropin_closure_reproduces_fixture(syn_model, syn_gmm, tmp_path):
    """the reference-style call create_fitting_closure(..., gt_joints3d, joints3d_conf, use_3d=True) with
    SMPLifyLoss(use_3d=True) reproduces a fixture; run_fitting through this package's LBFGS runs on the device; a missing
    joints3d_conf raises ValueError"""
    from mvsmplfitting_b200 import fitting, prior
    from mvsmplfitting_b200.optimizers import optim_factory
    from tests.test_gpu_dropin import build_scene
    c = load("l2_4_3donly")
    b = 0
    model, cams, bp = build_scene(syn_model, syn_gmm, tmp_path, c["cams"], 1, "smpllsp", "l2")
    model.reset_params(**{k: torch.tensor(v) for k, v in S.unpack_params(c["X"][b:b + 1]).items()})
    loss = fitting.create_loss("smplify", rho=float(c["rho"]), use_joints_conf=True, body_pose_prior=bp,
                               shape_prior=prior.create_prior("l2"), angle_prior=prior.create_prior("angle"),
                               interpenetration=False, use_3d=True).to("cuda")
    loss.reset_loss_weights({k: torch.tensor(v) for k, v in c["w"].items()})
    params = [p for p in model.parameters() if p.requires_grad]
    opt, cg = optim_factory.create_optimizer(params, optim_type="lbfgsls", lr=1.0, maxiters=30)
    mon = fitting.FittingMonitor(maxiters=30, ftol=1e-9, gtol=1e-9)
    V = c["gt_uv"].shape[0]
    kw = dict(camera=cams, gt_joints=torch.tensor(c["gt_uv"][:, b:b + 1]).cuda(),
              joints_conf=[torch.tensor(c["conf"][v, b:b + 1]).cuda() for v in range(V)],
              joint_weights=torch.tensor(c["joint_weights"]).unsqueeze(0).cuda(), loss=loss, create_graph=cg, use_vposer=False,
              vposer=None, pose_embedding=None, return_verts=True, return_full_pose=True)
    gt3d = torch.tensor(c["gt3d"][b]).cuda()                            # [K,3] and [1,K]: the reference's one-frame shapes
    with pytest.raises(ValueError):
        mon.create_fitting_closure(opt, model, gt_joints3d=gt3d, use_3d=True, **kw)
    closure = mon.create_fitting_closure(opt, model, gt_joints3d=gt3d, joints3d_conf=torch.tensor(c["conf3d"][b:b + 1]).cuda(),
                                         use_3d=True, **kw)
    total = float(closure())
    assert abs(total - c["loss_f32"][b]) / c["loss_f32"][b] < TOL
    for k, (a, e) in fitting.PARAM_SLICES.items():
        assert G.relmax(getattr(model, k).grad.cpu().numpy().reshape(-1), c["grad_f32"][b, a:e]) < TOL, k
    final = mon.run_fitting(opt, closure, params, model, use_vposer=False)
    assert final < total and mon.last_stats["frame_evals"] > 5


def test_errors(syn_model):
    from mvsmplfitting_b200 import _lib
    from mvsmplfitting_b200.context import FittingContext
    ctx = FittingContext(0)
    ctx.set_model(syn_model)
    lib, h = ctx.lib, ctx.h
    xyz, cf = np.zeros((2, 17, 3), np.float32), np.zeros((2, 17), np.float32)
    p = lambda a: a.ctypes.data_as(__import__("ctypes").c_void_p)
    assert lib.mvs_set_joints3d(h, p(xyz), p(cf), 1, 0, None) == -1           # before mvs_set_batch: MVS_ERR_INVALID
    ctx.set_batch(2)
    assert lib.mvs_set_joints3d(h, None, p(cf), 1, 0, None) == -1
    assert lib.mvs_set_joints3d(h, p(xyz), None, 1, 0, None) == -1
    assert lib.mvs_set_batch(h, 3) == -1                                       # the batch size (and the targets' rows) is fixed
    assert lib.mvs_set_joints3d(h, p(xyz), p(cf), 1, 0, None) == 0
    assert lib.mvs_set_joints3d(h, None, None, 0, 0, None) == 0
    with pytest.raises(ValueError):
        ctx.set_joints3d(np.zeros((3, 17, 3), np.float32), np.zeros((3, 17), np.float32))
    ctx.close()
    del _lib
