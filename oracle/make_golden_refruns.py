"""Writes the fixtures of the tests that compare with runs of the UNMODIFIED reference, so that those tests need neither
the reference checkout nor its compiled SDF kernel (oracle/_ref, oracle/stage_reference.py) at test time.

    python -m oracle.make_golden_refruns cpu OUT      # reference checkout present: shipped VPoser snapshot + demo data
    python -m oracle.make_golden_refruns gpu OUT      # CUDA device + oracle/_ref staged and built: reference SDF kernel
                                                      # grids, closures and fits; the demo-sequence reference fit

OUT is a directory; its .npz files (each < 1 MB) and demo/ tree go to tests/golden/.
"""
from __future__ import annotations

import json
import os
import shutil
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from mvsmplfitting_b200 import synthetic as S  # noqa: E402
from oracle import ref_harness as RH  # noqa: E402

SEG_NAMES = ("betas", "global_orient", "body_pose", "transl", "scale")
# grid cases of tests/test_gpu_sdf_refpin.py (grid, as_written, B, faces used); grids above FULL_MAX voxels are sampled
GRID_CASES = [(128, True, 2, None), (32, False, 1, None), (64, True, 3, None), (48, False, 1, 900)]
FULL_MAX = 1 << 17
SAMPLE = 1 << 14


def grid_key(grid, as_written, B, nf):
    return "g%d_%s_b%d_f%s" % (grid, "aw" if as_written else "all", B, "all" if nf is None else nf)


def cpu(out):
    """the snapshot's decoder weights (split in two files: each stays under 1 MB) and the demo data the reference ships,
    with what the reference's own readers make of it"""
    w = RH.vposer_weights_numpy(RH.load_reference_vposer())
    h = w["fc2_w"].shape[0] // 2
    np.savez_compressed(os.path.join(out, "vposer_snapshot_a.npz"), fc1_w=w["fc1_w"], fc1_b=w["fc1_b"], fc2_b=w["fc2_b"],
                        fc2_w_top=w["fc2_w"][:h])
    np.savez_compressed(os.path.join(out, "vposer_snapshot_b.npz"), fc2_w_bottom=w["fc2_w"][h:], out_w=w["out_w"], out_b=w["out_b"])
    demo = os.path.join(out, "demo")
    shutil.copytree(os.path.join(RH.REF_ROOT, "data", "keypoints"), os.path.join(demo, "keypoints"), dirs_exist_ok=True)
    shutil.copyfile(os.path.join(RH.REF_ROOT, "data", "3DOH50K_Parameters.txt"), os.path.join(demo, "3DOH50K_Parameters.txt"))
    RH.import_reference()
    with RH.in_reference_dir():
        from utils.utils import load_camera_para
        from utils.data_parser import read_keypoints
    e, i = load_camera_para(os.path.join(demo, "3DOH50K_Parameters.txt"))
    kp = {}
    for cam in sorted(os.listdir(os.path.join(demo, "keypoints", "0000"))):
        kp[cam] = read_keypoints(os.path.join(demo, "keypoints", "0000", cam, "00001_keypoints.json"),
                                 use_hands=False, use_face=False).keypoints[0]
    np.savez_compressed(os.path.join(out, "demo_readers_ref.npz"), extrinsics=e, intrinsics=i,
                        cameras=np.array(sorted(kp)), keypoints=np.stack([kp[c] for c in sorted(kp)]))


def gpu(out):
    import torch
    from oracle import closure_oracle as O, ref_fit as RF, ref_sdf, sdf_oracle, vposer_oracle as VO  # noqa: F401
    from tests.test_gpu_sdf_refpin import normalised_verts
    assert RH.available() and ref_sdf.available(), "stage and build oracle/_ref first (python -m oracle.stage_reference)"
    model, gmm = S.make_model(0), S.make_gmm(7)

    def ref_grid(faces, vn, G_, all_faces=False):
        return ref_sdf.grid(torch.tensor(np.asarray(faces, dtype=np.int32), device="cuda"),
                            torch.tensor(np.asarray(vn, dtype=np.float32), device="cuda"), G_, as_written=not all_faces).cpu().numpy()

    # 1. the reference kernel's grids: whole grids up to FULL_MAX voxels, else every inside voxel (up to SAMPLE) and a seeded
    #    sample of SAMPLE others
    grids = {}
    for grid, aw, B, nf in GRID_CASES:
        vn = normalised_verts(model, B, 3)
        faces = model["f"] if nf is None else model["f"][:nf]
        phi = ref_grid(faces, vn, grid, all_faces=not aw).reshape(-1)
        if phi.size <= FULL_MAX:
            idx = np.arange(phi.size)
        else:
            rng = np.random.RandomState(grid)
            inside = np.flatnonzero(phi > 0)
            if inside.size > SAMPLE:
                inside = np.sort(rng.choice(inside, SAMPLE, replace=False))
            rest = np.sort(rng.choice(np.flatnonzero(phi <= 0), SAMPLE, replace=False))
            idx = np.concatenate([inside, rest])
        k = grid_key(grid, aw, B, nf)
        grids[k + "_idx"] = idx.astype(np.int32)
        grids[k + "_phi"] = phi[idx].astype(np.float32)
        grids[k + "_inside_total"] = np.int64((phi > 0).sum())
    np.savez_compressed(os.path.join(out, "refpin_grids.npz"), **grids)

    # 2. the unmodified reference closure with interpenetration on (its own SDF kernel), and the float64 evaluation of its
    #    formulas on a grid from that kernel (tests/test_gpu_sdf_refpin.py, as-written semantics)
    B, grid, cw = 6, 128, 1000.0
    cams = S.make_cameras(4)
    fr = S.make_frames(model, cams, B, seed=2)
    w = dict(data_weight=500.0 / 1536, body_pose_weight=57.4, shape_weight=10.0, bending_prior_weight=3.17 * 57.4)
    ref_model, ref_cams, prior = RH.build_reference_model(model), RH.build_reference_cameras(cams), RH.build_reference_gmm(gmm)
    outs = [RH.reference_closure_eval(ref_model, ref_cams, fr, b, w, prior, device="cuda", interpenetration=True,
                                      coll_loss_weight=cw) for b in range(B)]
    outs0 = [RH.reference_closure_eval(ref_model, ref_cams, fr, b, w, prior, device="cuda", interpenetration=False)
             for b in range(B)]
    X = S.pack_params(fr["init"])
    old = sdf_oracle.GRID_FN
    sdf_oracle.GRID_FN = ref_grid
    try:
        om = O.OracleModel.from_numpy(model, dtype=torch.float64)
        arb = O.closure_eval_batch(om, O.LossConfig(interpenetration=True, coll_loss_weight=cw, sdf_grid=grid, **w),
                                   O.OraclePriors.gmm_from_dict(gmm, torch.float64), O.cams_to_torch(cams, torch.float64), X,
                                   fr["gt_uv"], fr["conf"], fr["joint_weights"])
        # intended semantics (every face) on a small grid from the reference kernel, oracle glue in fp32
        B2, grid2, cw2 = 2, 16, 0.05
        fr2 = S.make_frames(model, cams, B2, seed=2)
        om32 = O.OracleModel.from_numpy(model, dtype=torch.float32)
        allf = O.closure_eval_batch(om32, O.LossConfig(interpenetration=True, coll_loss_weight=cw2, sdf_grid=grid2, sdf_all_faces=True, **w),
                                    O.OraclePriors.gmm_from_dict(gmm, torch.float32), O.cams_to_torch(cams, torch.float32),
                                    S.pack_params(fr2["init"]), fr2["gt_uv"], fr2["conf"], fr2["joint_weights"])
    finally:
        sdf_oracle.GRID_FN = old
    np.savez_compressed(os.path.join(out, "refpin_closure.npz"), X=X,
                        ref_loss=np.array([o["loss"] for o in outs]), ref_loss0=np.array([o["loss"] for o in outs0]),
                        ref_grad=np.stack([np.concatenate([o["grads"][k] for k in SEG_NAMES]) for o in outs]),
                        arb_loss=np.asarray(arb["loss"]), arb_grad=np.asarray(arb["grad"]),
                        allfaces_loss=np.asarray(allf["loss"]), allfaces_grad=np.asarray(allf["grad"]))

    # 3. complete 4-stage fits by the reference on torch-CUDA with its SDF kernel (tests/test_gpu_fit_e2e.py)
    B, V = 16, 8
    cams8 = S.make_cameras(V)
    fr = S.make_frames(model, cams8, B, seed=4200)
    sc = RF.build_scene(model, gmm, cams8, device="cuda")
    runs = [RF.fit_frame(sc, fr, b, S.STAGE_WEIGHTS, interpenetration=True) for b in range(B)]
    np.savez_compressed(os.path.join(out, "fit_e2e_sdf_ref.npz"), B=B, V=V, seed=4200, X0=S.pack_params(fr["init"]),
                        iterations=np.array([r["iterations"] for r in runs]), evals=np.array([r["evals"] for r in runs]),
                        final_loss=np.array([r["final_loss"] for r in runs]), params=np.stack([r["params"] for r in runs]),
                        per_stage=np.array([r["per_stage"] for r in runs]))

    # 4. the demo sequence (tests/test_gpu_seq_demo.py): the reference solver from the device's initial guess
    from tests.test_gpu_seq_demo import demo_setup
    ctx, seq, cams6, stages, jw, vpw = demo_setup(model)
    p0, _ = ctx.init_guess(estimate_scale=True, fixed_scale=1.0, use_torso=True, hip_seed=1.0, want_joints3d=False)
    p0 = p0.cpu().numpy()
    ctx.close()
    vp = RH.load_reference_vposer()
    sc6 = RF.build_scene(model, gmm, cams6, device="cpu")
    init = S.unpack_params(p0)
    init["body_pose"] = np.zeros((1, 69), np.float32)
    init["body_pose"][:, :6] = 1.0                                               # fix_params; unused under VPoser
    frames = dict(gt_uv=seq["gt_uv"], conf=seq["conf"], joint_weights=jw, init=init)
    ref = RF.fit_frame(sc6, frames, 0, S.STAGE_WEIGHTS, interpenetration=False, image_height=1536, vposer=vp)
    np.savez_compressed(os.path.join(out, "seq_demo_ref.npz"), p0=p0, final_loss=ref["final_loss"], iterations=ref["iterations"],
                        evals=ref["evals"], params=ref["params"], pose_embedding=ref["pose_embedding"])
    print(json.dumps({"refpin_inside_totals": {k: int(v) for k, v in grids.items() if k.endswith("_inside_total")},
                      "fit_e2e_sdf_mean_iterations": float(np.mean([r["iterations"] for r in runs])),
                      "seq_demo_ref_loss": ref["final_loss"]}))


if __name__ == "__main__":
    mode, out = sys.argv[1], sys.argv[2]
    os.makedirs(out, exist_ok=True)
    {"cpu": cpu, "gpu": gpu}[mode](out)
