"""What refining the cameras from the fitted bodies (FittingContext.refine_cameras, seqio.fit_sequences(refine_cameras=n)) does
to a badly calibrated rig: rotation and centre errors of the views against the true calibration, keypoint error, mean final loss
and the refine pass's wall time, for the arms
  true        the true cameras, no refinement;
  perturbed   the perturbed cameras, no refinement;
  sweeps=n    the perturbed cameras, then one refine_cameras call of n sweeps over the perturbed fit's rows.

Synthetic smooth walks (synthetic.make_frames(smooth_walk=True), 5 px detection noise), S sequences x T frames, V views, in the
shipped configuration (VPoser latent pose, L2 prior, no SDF), fitted by fit_sequences on a context of S slots.  Calibration
errors: views 2 .. V-1 get a rotation update of N(0, --rot) rad per axis and a centre offset of N(0, --cen) scene units per axis;
view 1 the same rotation error and a move on its sphere about view 0 (the refinement's gauge); view 0 is exact.
Rotation error: mean over views 1 .. V-1 of the angle (deg) between fitted and true rotation; centre error: mean distance (mm)
between the camera centres.  Keypoint error: mean Euclidean distance (m) of the fitted 3-D keypoints to the true ones.  Final
loss: mean over frames.  Wall time: the refine_cameras call, ended by a device synchronisation (0 for the arms without one).
Needs a GPU; prints the card and its power limit, then one JSON line per arm, and writes them to --out."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from mvsmplfitting_b200 import seqio  # noqa: E402
from mvsmplfitting_b200 import synthetic as S  # noqa: E402
from oracle import camera_oracle as O  # noqa: E402
from scripts.seq_temporal_quality import keypoints, make_ctx, stages  # noqa: E402


def device_info():
    try:
        out = subprocess.check_output(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                      text=True, timeout=30).strip()
        name, limit = [s.strip() for s in out.split(",")]
        return {"gpu": name, "power_limit": limit}
    except Exception as e:  # noqa: BLE001
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": "unknown (%r)" % e}


def perturb(cams, seed, rot, cen):
    rng = np.random.RandomState(seed)
    out = {k: np.array(v) for k, v in cams.items()}
    for v in range(1, cams["R"].shape[0]):
        w = torch.tensor(rng.normal(0, rot, 3))
        if v == 1:
            E, n = O.sphere_basis(cams["R"][0], cams["t"][0], cams["R"][1], cams["t"][1])
            u = rng.normal(0, cen / np.linalg.norm(n), 2)
            R, t = O.cam_from_delta(cams["R"][v], cams["t"][v], w, torch.tensor([u[0], u[1], 0.0]), True, E, n)
        else:
            R, t = O.cam_from_delta(cams["R"][v], cams["t"][v], w, torch.tensor(rng.normal(0, cen, 3)))
        out["R"][v], out["t"][v] = R.numpy().astype(np.float32), t.numpy().astype(np.float32)
    return out


def cam_errors(cams, true):
    rot, cen = [], []
    for v in range(1, true["R"].shape[0]):
        M = cams["R"][v].astype(np.float64).T @ true["R"][v].astype(np.float64)
        s = np.linalg.norm([M[2, 1] - M[1, 2], M[0, 2] - M[2, 0], M[1, 0] - M[0, 1]]) / 2
        rot.append(np.degrees(np.arctan2(s, (np.trace(M) - 1) / 2)))
        cen.append(np.linalg.norm(O.centre(cams["R"][v], cams["t"][v]) - O.centre(true["R"][v], true["t"][v])) * 1000.0)
    return float(np.mean(rot)), float(np.mean(cen))


def fit(model, gmm, cams, seqs, opt):
    ctx = make_ctx(model, gmm, cams, len(seqs), True)
    res, _ = seqio.fit_sequences(ctx, seqs, stages(ctx, "shipped"), ctx.make_lbfgs_config(**opt), estimate_scale=True,
                                 pose_format="lsp14")
    ctx.close()
    return np.concatenate([r[0] for r in res]), np.concatenate([r[1] for r in res])


def refine(model, gmm, cams, seqs, x, sweeps, opt):
    ctx = make_ctx(model, gmm, cams, len(seqs), True)
    X = torch.tensor(x, device="cuda")
    gt_uv = np.concatenate([q["gt_uv"] for q in seqs], axis=1)
    conf = np.concatenate([q["conf"] for q in seqs], axis=1)
    jw = seqio.joint_weights("lsp14", True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    final, rigs, ca, po = ctx.refine_cameras(X, gt_uv, conf, jw, stages(ctx, "shipped")[-1], ctx.make_lbfgs_config(**opt),
                                             sweeps=sweeps)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    ctx.close()
    return X.cpu().numpy(), final.cpu().numpy(), rigs[0], wall, ca


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seqs", type=int, default=64)
    ap.add_argument("--frames", type=int, default=32)
    ap.add_argument("--views", type=int, default=8)
    ap.add_argument("--sweeps", default="1,2,3")
    ap.add_argument("--rot", type=float, default=0.01)
    ap.add_argument("--cen", type=float, default=0.15)
    ap.add_argument("--max-outer", type=int, default=30)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    info = device_info()
    print(json.dumps(info), flush=True)
    model, gmm, true = S.make_model(0), S.make_gmm(7), S.make_cameras(a.views)
    bad = perturb(true, 77, a.rot, a.cen)
    seqs, gt = [], []
    for s_ in range(a.seqs):
        fr = S.make_frames(model, true, a.frames, seed=5000 + s_, smooth_walk=True)
        seqs.append(dict(gt_uv=fr["gt_uv"], conf=fr["conf"], present=np.ones(fr["conf"].shape[:2], bool),
                         frames=["%05d" % t for t in range(a.frames)], serial="s%03d" % s_))
        gt.append(fr["gt_joints3d"])
    gt_j = np.concatenate(gt).astype(np.float64)
    opt = dict(max_outer=a.max_outer)
    out = open(a.out, "w") if a.out else None

    def emit(arm, cams, x, loss, wall, extra=None):
        rot, cen = cam_errors(cams, true)
        j = keypoints(model, gmm, true, x, True)
        r = dict(arm=arm, rot_err_deg=rot, centre_err_mm=cen, keypoint_err_m=float(np.linalg.norm(j - gt_j, axis=-1).mean()),
                 mean_final_loss=float(np.nanmean(loss)), wall_s=wall, seqs=a.seqs, frames=a.frames, views=a.views,
                 calib_rot=a.rot, calib_cen=a.cen, **info)
        r.update(extra or {})
        print(json.dumps(r), flush=True)
        if out:
            out.write(json.dumps(r) + "\n")
            out.flush()

    x, loss = fit(model, gmm, true, seqs, opt)
    emit("true", true, x, loss, 0.0)
    x, loss = fit(model, gmm, bad, seqs, opt)
    emit("perturbed", bad, x, loss, 0.0)
    for n in [int(v) for v in a.sweeps.split(",")]:
        x1, l1, cams, wall, ca = refine(model, gmm, bad, seqs, x, n, opt)
        emit("sweeps=%d" % n, cams, x1, l1, wall, dict(camera_evals=ca["frame_evals"]))


if __name__ == "__main__":
    main()
