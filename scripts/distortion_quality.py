"""Lens distortion (mvs_set_camera_rigs_dist): fit quality and cost on the wide-angle synthetic rig (synthetic.make_wide_cameras).

  quality  mean 3-D keypoint error of the fit with the coefficients and of the fit that ignores them, on distorted detections
           with 2 px noise, and of an undistorted control rig on undistorted detections with the same noise;
  cost     the shipped four-stage configuration (VPoser latent pose, no SDF) at 256 frames x 8 views, coefficients on against
           off (the same rig without them), alternating, median of --runs runs each: time per fit and frame-iterations/s.

Prints one JSON line.  Needs a GPU.

    python scripts/distortion_quality.py [--frames 256] [--views 8] [--runs 5]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from mvsmplfitting_b200 import synthetic as S  # noqa: E402
from mvsmplfitting_b200.context import FittingContext  # noqa: E402
from tests import golden_util as G  # noqa: E402


def stages(ctx, kind, n=4):
    sw = S.STAGE_WEIGHTS
    vp = kind == "vposer"
    return [ctx.make_loss_config(body_prior="l2" if vp else "gmm", use_vposer=2 if vp else 0, data_weight=500.0 / 1536,
                                 body_pose_weight=sw["body_pose_prior_weights"][i], shape_weight=sw["shape_weights"][i],
                                 bending_prior_weight=3.17 * sw["body_pose_prior_weights"][i]) for i in range(n)]


def make_ctx(model, gmm, cams, B, vposer):
    ctx = FittingContext(0)
    ctx.set_model(model)
    ctx.set_gmm_from_dict(gmm)
    ctx.set_camera_rigs([cams])
    ctx.set_batch(B)
    if vposer:
        ctx.set_vposer(G.snapshot_vposer_weights())
    return ctx


def fit(model, gmm, cams, fr, kind, max_outer=30):
    B = fr["gt_uv"].shape[1]
    ctx = make_ctx(model, gmm, cams, B, kind == "vposer")
    ctx.set_keypoints(fr["gt_uv"], fr["conf"], fr["joint_weights"])
    x0 = S.pack_params(fr["init"])
    if kind == "vposer":
        x0[:, 13:82] = 0.0
    x = torch.tensor(x0, device="cuda")
    torch.cuda.synchronize()
    t = time.perf_counter()
    _, st = ctx.fit(x, stages(ctx, kind), ctx.make_lbfgs_config(max_outer=max_outer))
    torch.cuda.synchronize()
    dt = time.perf_counter() - t
    out = x.cpu().numpy()
    if kind == "vposer":
        out[:, 13:82] = ctx.vposer_decode(x).cpu().numpy()
    ctx.close()
    return out, dt, st


def mpjpe(model, x, truth):
    p = S.unpack_params(x)
    j = S.model_keypoints_np(model, p["betas"], p["global_orient"], p["body_pose"], p["transl"], p["scale"], "smpllsp")
    return float(np.linalg.norm(j - truth, axis=-1).mean())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=256)
    ap.add_argument("--views", type=int, default=8)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--quality-frames", type=int, default=64)
    a = ap.parse_args()
    model, gmm = S.make_model(0), S.make_gmm(7)
    res = dict(gpu=torch.cuda.get_device_name(0))
    # quality (GMM prior, four stages)
    cams = S.make_wide_cameras(a.views)
    plain = {k: cams[k] for k in ("R", "t", "f", "c")}
    ctl = S.make_wide_cameras(a.views, distorted=False)
    fr = S.make_frames_wide(model, cams, a.quality_frames, seed=5, noise=2.0)
    fc = S.make_frames_wide(model, ctl, a.quality_frames, seed=5, noise=2.0)
    truth = fr["gt_joints3d"]
    res["mpjpe_with_coefficients"] = mpjpe(model, fit(model, gmm, cams, fr, "gmm")[0], truth)
    res["mpjpe_ignoring_coefficients"] = mpjpe(model, fit(model, gmm, plain, fr, "gmm")[0], truth)
    res["mpjpe_undistorted_control"] = mpjpe(model, fit(model, gmm, ctl, fc, "gmm")[0], truth)
    # cost: the shipped configuration, alternating on / off
    fr = S.make_frames_wide(model, cams, a.frames, seed=7, noise=2.0)
    fit(model, gmm, cams, fr, "vposer")
    fit(model, gmm, plain, fr, "vposer")                                     # warm-up of both arms
    t_on, t_off, it_on, it_off = [], [], [], []
    for _ in range(a.runs):
        _, dt, st = fit(model, gmm, cams, fr, "vposer")
        t_on.append(dt)
        it_on.append(st["frame_iterations"] / dt)
        _, dt, st = fit(model, gmm, plain, fr, "vposer")
        t_off.append(dt)
        it_off.append(st["frame_iterations"] / dt)
    res.update(frames=a.frames, views=a.views, runs=a.runs,
               fit_s_on=dict(median=float(np.median(t_on)), min=float(min(t_on)), max=float(max(t_on))),
               fit_s_off=dict(median=float(np.median(t_off)), min=float(min(t_off)), max=float(max(t_off))),
               frame_iters_per_s_on=float(np.median(it_on)), frame_iters_per_s_off=float(np.median(it_off)))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
