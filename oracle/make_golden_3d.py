"""TEST INFRASTRUCTURE -- writes tests/golden/joints3d_*.npz by RUNNING THE UNMODIFIED REFERENCE with 3-D joint supervision
(SMPLifyLoss(use_3d=True), fitting.py:318-324; targets as non_linear_solver.py:86-99 builds them) on the synthetic inputs of
mvsmplfitting_b200/synthetic.py.  Authoring container only (needs /root/reference):

    python -m oracle.make_golden_3d

* joints3d_closure_<case>.npz  one fitting_func() per frame, fp32 and fp64: loss, every gradient tensor, joints; two
                               cases with use_vposer=True and the reference's shipped VPoser snapshot
* joints3d_init.npz            the reference's own init_guess(use_3d=True) + fix_params, one and four views
* joints3d_fit_e2e.npz         the reference's own non_linear_solver with data['3d_joint'] set, SDF off, 8 frames x 4 views
                               and 8 frames x 1 view

The 3-D targets are the frames' true keypoints plus 2 cm of noise; their confidences are uniform in [0.5, 1] unless a case
says otherwise.  (The fixture names do not start with closure_: the 2-D-only closure tests glob those.)
"""
from __future__ import annotations

import json
import os
import sys
import types
import warnings

import numpy as np
import torch

warnings.filterwarnings("ignore")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from mvsmplfitting_b200 import synthetic as S  # noqa: E402
from oracle import ref_fit as RF               # noqa: E402
from oracle import ref_harness as H            # noqa: E402
from oracle.make_golden import model_checksum, stage_weights  # noqa: E402
from oracle.make_golden_vposer import reference_vposer       # noqa: E402
from tests import golden_util as G                            # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")


def targets(fr, seed, zero_frac=0.0):
    rng = np.random.RandomState(seed)
    gt3d = (fr["gt_joints3d"] + rng.normal(0, 0.02, size=fr["gt_joints3d"].shape)).astype(np.float32)
    conf3d = rng.uniform(0.5, 1.0, size=gt3d.shape[:2]).astype(np.float32)
    if zero_frac:
        conf3d[rng.rand(*conf3d.shape) < zero_frac] = 0.0
        conf3d[:, [11, 12]] = 0.0                               # non_linear_solver.py:92-94 without use_hip
    return gt3d, conf3d


def reference_closure_3d(rm, rc, fr, b, weights, bp, dt, params, gt3d, conf3d, rho, fix_shape, vp=None, z=None):
    """RH.reference_closure_eval with use_3d=True: the reference's create_fitting_closure / SMPLifyLoss.forward.  With a
    VPoser `vp` the pose is vp.decode(z, 'aa') (use_vposer=True, fitting.py:121-123) and the gradient's pose slot holds
    d loss / d z in its first 32 entries (the device layout of use_vposer = 2)."""
    ns = H.import_reference()
    H.set_model_params(rm, params, b)
    V = fr["gt_uv"].shape[0]
    gt = torch.tensor(fr["gt_uv"][:, b:b + 1], dtype=dt)
    conf = [torch.tensor(fr["conf"][v, b:b + 1], dtype=dt) for v in range(V)]
    jw = torch.tensor(fr["joint_weights"], dtype=dt).unsqueeze(0)
    loss = ns.fitting.create_loss("smplify", rho=rho, use_joints_conf=True, dtype=dt, body_pose_prior=bp,
                                  shape_prior=ns.prior.create_prior("l2"), angle_prior=ns.prior.create_prior("angle", dtype=dt),
                                  interpenetration=False, fix_shape=fix_shape, use_3d=True)
    loss.reset_loss_weights({k: torch.tensor(v, dtype=dt) for k, v in weights.items()})
    mon = ns.fitting.FittingMonitor(maxiters=30, ftol=1e-9, gtol=1e-9)
    emb = None
    if vp is not None:
        emb = torch.tensor(z[b], dtype=dt).view(1, 32).requires_grad_(True)
        rm.body_pose.requires_grad = False
    opt = torch.optim.SGD([q for q in rm.parameters() if q.requires_grad] + ([emb] if emb is not None else []), lr=0.0)
    closure = mon.create_fitting_closure(
        opt, rm, camera=rc, gt_joints=gt, joints_conf=conf, joint_weights=jw, loss=loss, create_graph=False,
        gt_joints3d=torch.tensor(gt3d[b], dtype=dt), joints3d_conf=torch.tensor(conf3d[b:b + 1], dtype=dt),
        use_vposer=vp is not None, vposer=vp, pose_embedding=emb, return_verts=True, return_full_pose=True, use_3d=True)
    total = closure()
    body_pose = None if vp is None else vp.decode(emb, output_type="aa").view(1, -1)
    out = rm(return_verts=True, body_pose=body_pose, return_full_pose=True)
    g = np.zeros(86)
    o = 0
    for k, n in zip(S.PARAM_ORDER, S.PARAM_SIZES):
        p = emb if (k == "body_pose" and emb is not None) else getattr(rm, k)
        if p.grad is not None:
            v = p.grad.detach().numpy().reshape(-1)
            g[o:o + v.shape[0]] = v
        o += n
    return float(total), g, out.joints.detach().numpy()[0].astype(np.float64)


def closure_case(name, model, gmm, cams, fr, params, weights, prior, gt3d, conf3d, rho=100.0, model_type="smpllsp",
                 fix_shape=False, Z=None):
    ns = H.import_reference()
    out = {}
    B = params["betas"].shape[0]
    for dt, tag in ((torch.float32, "f32"), (torch.float64, "f64")):
        rm = H.build_reference_model(model, dtype=dt, model_type=model_type)
        if fix_shape:
            rm.betas.requires_grad = False
        rc = H.build_reference_cameras(cams, dtype=dt)
        bp = H.build_reference_gmm(gmm, dtype=dt) if prior == "gmm" else ns.prior.create_prior("l2")
        vp = None if Z is None else reference_vposer(G.snapshot_vposer_weights(), dt)
        res = [reference_closure_3d(rm, rc, fr, b, weights, bp, dt, params, gt3d, conf3d, rho, fix_shape, vp, Z) for b in range(B)]
        out["loss_" + tag] = np.array([r[0] for r in res])
        out["grad_" + tag] = np.stack([r[1] for r in res])
        out["joints_" + tag] = np.stack([r[2] for r in res])
    out.update(X=S.pack_params(params), gt_uv=fr["gt_uv"], conf=fr["conf"], joint_weights=fr["joint_weights"],
               gt3d=gt3d, conf3d=conf3d, rho=np.float64(rho),
               weights=np.array([weights[k] for k in ("data_weight", "body_pose_weight", "shape_weight", "bending_prior_weight")]),
               meta=np.array(json.dumps(dict(name=name, body_prior=prior, model_type=model_type, fix_shape=fix_shape,
                                             use_vposer=Z is not None))),
               model_checksum=np.array(model_checksum(model)))
    if Z is not None:
        out["Z"] = Z
    for k in ("R", "t", "f", "c"):
        out["cam_" + k] = cams[k]
    np.savez_compressed(os.path.join(GOLD, "joints3d_closure_%s.npz" % name), **out)
    print("  case %-10s loss_f32 %s" % (name, out["loss_f32"]))


def closures(model, gmm):
    cams4, cams1 = S.make_cameras(4), {k: v[:1] for k, v in S.make_cameras(4).items() if isinstance(v, np.ndarray)}
    fr4 = S.make_frames(model, cams4, 3, seed=31)
    g4 = targets(fr4, 32)
    closure_case("gmm4_s3", model, gmm, cams4, fr4, fr4["init"], stage_weights(3), "gmm", *g4)
    closure_case("l2_4_fixshape", model, gmm, cams4, fr4, fr4["init"], stage_weights(2), "l2", *g4, fix_shape=True)
    closure_case("gmm4_zeroconf", model, gmm, cams4, fr4, fr4["init"], stage_weights(3), "gmm", *targets(fr4, 33, 0.3))
    rng = np.random.RandomState(34)                       # perturbed truth, non-unit scale
    pert = {k: (v + rng.normal(0, 0.02, size=v.shape)).astype(np.float32) for k, v in fr4["gt"].items()}
    pert["scale"] = (1.0 + rng.uniform(-0.2, 0.3, size=pert["scale"].shape)).astype(np.float32)
    closure_case("l2_4_scale", model, gmm, cams4, fr4, pert, stage_weights(3), "l2", *g4)
    fr1 = S.make_frames(model, cams1, 3, seed=35)
    g1 = targets(fr1, 36)
    closure_case("l2_1_s0", model, gmm, cams1, fr1, fr1["init"], stage_weights(0), "l2", *g1)
    # rho = 0.05: residuals of a few cm saturate the 3-D GMoF (at rho = 100 a residual in metres is purely quadratic)
    closure_case("gmm1_rho", model, gmm, cams1, fr1, fr1["init"], stage_weights(3), "gmm", *g1, rho=0.05)
    # In the cases above the 3-D term is a small share of the loss (metres against pixels, as in the reference's own use).
    # These two let it dominate: no 2-D confidence, light priors, data_weight 10.
    light = dict(data_weight=10.0, body_pose_weight=0.5, shape_weight=0.5, bending_prior_weight=3.17 * 0.5)
    closure_case("l2_4_3donly", model, gmm, cams4, dict(fr4, conf=np.zeros_like(fr4["conf"])), fr4["init"], light, "l2", *g4)
    closure_case("gmm1_3donly_rho", model, gmm, cams1, dict(fr1, conf=np.zeros_like(fr1["conf"])), fr1["init"], light, "gmm",
                 *g1, rho=0.05)
    fr_s = S.make_frames(model, cams4, 3, seed=37, model_type="smpl")
    closure_case("smpl4", model, gmm, cams4, fr_s, fr_s["init"], stage_weights(3), "gmm", *targets(fr_s, 38), model_type="smpl")


def vposer_closures(model, gmm):
    """use_vposer=True (the reference's shipped configuration) with its shipped snapshot (tests/golden/vposer_snapshot_*.npz):
    the 3-D term's adjoint goes on through the decoder to the latent code"""
    cams4 = S.make_cameras(4)
    fr4 = S.make_frames(model, cams4, 3, seed=31)
    g4 = targets(fr4, 32)
    light = dict(data_weight=10.0, body_pose_weight=0.5, shape_weight=0.5, bending_prior_weight=3.17 * 0.5)
    Zv = np.random.RandomState(39).normal(0, 0.8, size=(3, 32)).astype(np.float32)
    closure_case("vposer4_s3", model, gmm, cams4, fr4, fr4["init"], stage_weights(3), "l2", *g4, Z=Zv)
    closure_case("vposer4_3donly", model, gmm, cams4, dict(fr4, conf=np.zeros_like(fr4["conf"])), fr4["init"], light, "l2",
                 *g4, Z=Zv)


def init_runs(model):
    """the reference's init_guess(use_3d=True) + fix_params (init_guess.py:18-107,190-212), unmodified"""
    H.import_reference()
    with H.in_reference_dir():
        from utils import init_guess as RIG
    rm = H.build_reference_model(model)
    out = {}
    cuda = torch.Tensor.cuda
    torch.Tensor.cuda = lambda self, *a, **k: self            # init_guess.py:38 hard-codes .cuda(); a no-op here
    try:
        for tag, V in (("mv4", 4), ("sv", 1)):
            cams = {k: v[:V] for k, v in S.make_cameras(4).items() if isinstance(v, np.ndarray)}
            fr = S.make_frames(model, cams, 4, seed=800 + V)
            gt3d, conf3d = targets(fr, 810 + V)
            ext = np.tile(np.eye(4), (V, 1, 1))
            ext[:, :3, :3], ext[:, :3, 3] = cams["R"], cams["t"]
            intr = np.tile(np.eye(3), (V, 1, 1))
            intr[:, 0, 0], intr[:, 1, 1], intr[:, 0, 2], intr[:, 1, 2] = cams["f"][:, 0], cams["f"][:, 1], cams["c"][:, 0], cams["c"][:, 1]
            res = []
            for b in range(4):
                kps = [np.concatenate([fr["gt_uv"][v, b], fr["conf"][v, b][:, None]], axis=1)[None].astype(np.float32) for v in range(V)]
                setting = dict(model=rm, dtype=torch.float32, batch_size=1, device=torch.device("cpu"), fix_scale=False,
                               fixed_scale=None, extris=ext, intris=intr)
                data = {"keypoints": kps, "3d_joint": [np.concatenate([gt3d[b], conf3d[b][:, None]], axis=1)]}
                RIG.init_guess(setting, data, use_torso=True, model_type="smpllsp", use_vposer=False, use_3d=True)
                RIG.fix_params(setting, scale=None, shape=None)
                res.append(np.concatenate([getattr(rm, k).detach().numpy().reshape(-1) for k in S.PARAM_ORDER]))
            out[tag + "_V"] = np.int64(V)
            out[tag + "_seed"] = np.int64(800 + V)
            out[tag + "_gt3d"], out[tag + "_conf3d"] = gt3d, conf3d
            out[tag + "_params"] = np.stack(res)
    finally:
        torch.Tensor.cuda = cuda
    np.savez_compressed(os.path.join(GOLD, "joints3d_init.npz"), **out)
    print("wrote joints3d_init.npz")


def fit_frame_3d(sc, fr, b, gt3d, conf3d):
    """oracle/ref_fit.fit_frame with data['3d_joint'] set and use_3d=True (hips zeroed by the solver: no use_hip): the same
    call of the reference's own solver, with the annotations added to what fit_frame passes it"""
    solver = sc["nls"].non_linear_solver

    def with_joints3d(setting, data, **kw):
        data["3d_joint"] = [np.concatenate([gt3d[b], conf3d[b][:, None]], axis=1)]
        return solver(setting, data, **dict(kw, use_3d=True))
    r = RF.fit_frame(dict(sc, nls=types.SimpleNamespace(non_linear_solver=with_joints3d)), fr, b, S.STAGE_WEIGHTS)
    return r["per_stage"], r["final_loss"], r["params"]


def e2e(model, gmm):
    torch.set_num_threads(1)
    out = {}
    for tag, V, seed in (("v4", 4, 4300), ("v1", 1, 4310)):
        cams = {k: v[:V] for k, v in S.make_cameras(4).items() if isinstance(v, np.ndarray)}
        fr = S.make_frames(model, cams, 8, seed=seed)
        gt3d, conf3d = targets(fr, seed + 1)
        sc = RF.build_scene(model, gmm, cams)
        its, evs, fin, par = [], [], [], []
        for b in range(8):
            per_stage, final, params = fit_frame_3d(sc, fr, b, gt3d, conf3d)
            its.append([p[0] for p in per_stage]); evs.append([p[1] for p in per_stage]); fin.append(final); par.append(params)
            print(tag, b, per_stage, final)
        out.update({tag + "_V": np.int64(V), tag + "_seed": np.int64(seed), tag + "_X0": S.pack_params(fr["init"]),
                    tag + "_gt3d": gt3d, tag + "_conf3d": conf3d, tag + "_iterations": np.array(its), tag + "_evals": np.array(evs),
                    tag + "_final_loss": np.array(fin, np.float64), tag + "_params": np.stack(par)})
    np.savez_compressed(os.path.join(GOLD, "joints3d_fit_e2e.npz"), **out)
    print("wrote joints3d_fit_e2e.npz")


def main():
    model, gmm = S.make_model(0), S.make_gmm(7)
    what = sys.argv[1:] or ["closure", "vposer", "init", "e2e"]
    if "closure" in what:
        closures(model, gmm)
    if "vposer" in what:
        vposer_closures(model, gmm)
    if "init" in what:
        init_runs(model)
    if "e2e" in what:
        e2e(model, gmm)


if __name__ == "__main__":
    main()
