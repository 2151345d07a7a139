"""What one shared body shape per sequence (seqio.fit_sequences(shared_shape=n)) does to video fits: shape error against the true
shape, its spread within a sequence, keypoint error, acceleration error, final loss and wall time, for n = 0 (off), 1 and 2 sweeps.

Synthetic smooth walks (synthetic.make_frames(smooth_walk=True): one true betas row per sequence, 5 px detection noise), S
sequences x T frames, V views, in the shipped configuration (VPoser latent pose, L2 prior, no SDF), fitted by the sequence
stream on a context of S slots and, with n > 0, one fit_shared_shape call.
Shape error: mean per-vertex distance (mm) of the zero-pose, unit-scale, zero-translation mesh at the fitted betas to that mesh
at the true betas, over all frames; its spread: the mean over sequences of the standard deviation of that distance within the
sequence.  Keypoint error: mean Euclidean distance of the fitted 3-D keypoints to the true ones.  Acceleration error: mean
distance of the fitted keypoints' second differences to the true ones, over frames t whose t-1 and t are warm.  Final loss: mean
over frames (for n > 0: the pose step's).  Wall time: the whole fit_sequences pass (initial guesses included), ended by a device
synchronisation.  Needs a GPU; prints one JSON line per setting and writes them to --out."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from mvsmplfitting_b200 import seqio  # noqa: E402
from mvsmplfitting_b200 import synthetic as S  # noqa: E402
from scripts.seq_temporal_quality import keypoints, make_ctx, stages  # noqa: E402


def rest_verts(model, gmm, cams, betas):
    """vertices [F,N,3] of the zero-pose, unit-scale, zero-translation body with shapes betas [F,10]"""
    ctx = make_ctx(model, gmm, cams, betas.shape[0], False)
    p = torch.zeros(betas.shape[0], 86, device="cuda")
    p[:, :10] = torch.as_tensor(betas, dtype=torch.float32, device="cuda")
    p[:, 85] = 1.0
    v = ctx.forward_only(p, want_verts=True)["verts"].cpu().numpy().astype(np.float64)
    ctx.close()
    return v


def measure(model, gmm, cams, seqs, gt_j, gt_v, sweeps, opt):
    S_ = len(seqs)
    ctx = make_ctx(model, gmm, cams, S_, True)
    cfgs = stages(ctx, "shipped")
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    res, _ = seqio.fit_sequences(ctx, seqs, cfgs, ctx.make_lbfgs_config(**opt), estimate_scale=True, pose_format="lsp14",
                                 shared_shape=sweeps)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    ctx.close()
    x = np.concatenate([r[0] for r in res])
    loss = np.concatenate([r[1] for r in res])
    d = np.linalg.norm(rest_verts(model, gmm, cams, x[:, :10]) - gt_v, axis=-1).mean(axis=1) * 1000.0     # per frame, mm
    off = np.concatenate([[0], np.cumsum([len(q["frames"]) for q in seqs])])
    spread = float(np.mean([d[off[s]:off[s + 1]].std() for s in range(S_)]))
    j = keypoints(model, gmm, cams, x, True)
    acc = []
    for s in range(S_):
        f = off[s]
        for t in range(2, off[s + 1] - f):
            if loss[f + t - 2] <= 5000.0 and loss[f + t - 1] <= 5000.0:
                a_fit = j[f + t] - 2 * j[f + t - 1] + j[f + t - 2]
                a_gt = gt_j[f + t] - 2 * gt_j[f + t - 1] + gt_j[f + t - 2]
                acc.append(np.linalg.norm(a_fit - a_gt, axis=-1).mean())
    return dict(config="shipped", shared_shape=sweeps, shape_err_mm=float(d.mean()), shape_spread_mm=spread,
                keypoint_err_m=float(np.linalg.norm(j - gt_j, axis=-1).mean()), accel_err_m=float(np.mean(acc)),
                mean_final_loss=float(np.nanmean(loss)), wall_s=wall)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seqs", type=int, default=64)
    ap.add_argument("--frames", type=int, default=32)
    ap.add_argument("--views", type=int, default=8)
    ap.add_argument("--sweeps", default="0,1,2")
    ap.add_argument("--max-outer", type=int, default=30)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    model, gmm, cams = S.make_model(0), S.make_gmm(7), S.make_cameras(a.views)
    seqs, gt, gb = [], [], []
    for s_ in range(a.seqs):
        fr = S.make_frames(model, cams, a.frames, seed=5000 + s_, smooth_walk=True)
        seqs.append(dict(gt_uv=fr["gt_uv"], conf=fr["conf"], present=np.ones(fr["conf"].shape[:2], bool),
                         frames=["%05d" % t for t in range(a.frames)], serial="s%03d" % s_))
        gt.append(fr["gt_joints3d"])
        gb.append(fr["gt"]["betas"])
    gt_j = np.concatenate(gt).astype(np.float64)
    gt_v = rest_verts(model, gmm, cams, np.concatenate(gb))
    name = torch.cuda.get_device_name(0)
    out = open(a.out, "w") if a.out else None
    for n in [int(v) for v in a.sweeps.split(",")]:
        r = measure(model, gmm, cams, seqs, gt_j, gt_v, n, dict(max_outer=a.max_outer))
        r.update(device=name, seqs=a.seqs, frames=a.frames, views=a.views)
        print(json.dumps(r), flush=True)
        if out:
            out.write(json.dumps(r) + "\n")
            out.flush()


if __name__ == "__main__":
    main()
