"""What the causal temporal term (seqio.fit_sequences(temporal_weight=lam)) does to video fits: keypoint error against the
ground truth, acceleration error (jitter), final loss and wall time of the lock-step and the sequence stream, for a sweep of lam.

Synthetic smooth walks (synthetic.make_frames(smooth_walk=True): 5 px detection noise), S sequences x T frames, V views, in two
configurations: 'shipped' (VPoser latent pose, L2 prior, no SDF) and 'bench' (GMM prior, SDF term in stages 2-3, grid 64).
Keypoint error: mean Euclidean distance of the fitted 3-D keypoints to the true ones over all frames.  Acceleration error:
mean Euclidean distance of the fitted keypoints' second differences to the true ones, over frames t whose t-1 and t are warm.
Final loss: mean over frames (for lam > 0 it includes the temporal term of warm frames).  Lock-step: fit_sequences on a context
of S slots (initial guesses included); stream: one mvs_fit_seq_stream(_temporal) call on S slots (initial guesses excluded);
both end in a device synchronisation.  Needs a GPU; prints one JSON line per (configuration, lam) and writes them to --out."""
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
from mvsmplfitting_b200.context import FittingContext  # noqa: E402

GUESS = dict(estimate_scale=True, fixed_scale=1.0, use_torso=True, hip_seed=1.0, want_joints3d=False, umeyama_as_written=False)


def make_ctx(model, gmm, cams, B, vposer):
    ctx = FittingContext(0)
    ctx.set_model(model)
    ctx.set_gmm_from_dict(gmm)
    ctx.set_cameras(cams["R"], cams["t"], cams["f"], cams["c"])
    ctx.set_batch(B)
    if vposer:
        ctx.set_vposer(S.make_vposer(0))
    return ctx


def stages(ctx, kind):
    sw, vp, out = S.STAGE_WEIGHTS, kind == "shipped", []
    for i in range(4):
        on = kind == "bench" and i >= 2
        out.append(ctx.make_loss_config(body_prior="l2" if vp else "gmm", use_vposer=2 if vp else 0, interpenetration=on,
                                        sdf_grid=64, data_weight=500.0 / 1536, body_pose_weight=sw["body_pose_prior_weights"][i],
                                        shape_weight=sw["shape_weights"][i], bending_prior_weight=3.17 * sw["body_pose_prior_weights"][i],
                                        coll_loss_weight=sw["coll_loss_weights"][i] if on else 0.0))
    return out


def keypoints(model, gmm, cams, x, vposer):
    """the fitted 3-D keypoints of rows x [F,86] (latent codes decoded first)"""
    ctx = make_ctx(model, gmm, cams, x.shape[0], vposer)
    p = torch.tensor(x, device="cuda")
    if vposer:
        p[:, 13:82] = ctx.vposer_decode(p)
    j = ctx.forward_only(p.contiguous(), want_verts=False)["joints"].cpu().numpy().astype(np.float64)
    ctx.close()
    return j


def measure(model, gmm, cams, seqs, gt_j, kind, lam, opt):
    vp = kind == "shipped"
    S_, tw = len(seqs), (None if lam == 0 else lam)
    ctx = make_ctx(model, gmm, cams, S_, vp)
    cfgs = stages(ctx, kind)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    res, _ = seqio.fit_sequences(ctx, seqs, cfgs, ctx.make_lbfgs_config(**opt), estimate_scale=True, pose_format="lsp14",
                                 temporal_weight=tw)
    torch.cuda.synchronize()
    t_lock = time.perf_counter() - t0
    x = np.concatenate([r[0] for r in res])
    loss = np.concatenate([r[1] for r in res])
    # the stream on the same S slots
    gt_uv = np.concatenate([q["gt_uv"] for q in seqs], 1)
    conf = np.concatenate([q["conf"] for q in seqs], 1)
    jw = seqio.joint_weights("lsp14")
    xs = seqio._cold_guesses(ctx, gt_uv, conf, jw, cfgs, GUESS)
    kw = {} if tw is None else dict(temporal_weight=seqio.temporal_weight_vector(tw))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fs, _ = ctx.fit_seq_stream(xs, gt_uv, conf, jw, [len(q["frames"]) for q in seqs], cfgs, ctx.make_lbfgs_config(**opt), **kw)
    torch.cuda.synchronize()
    t_stream = time.perf_counter() - t0
    same = bool(np.array_equal(xs.cpu().numpy(), x))
    ctx.close()
    j = keypoints(model, gmm, cams, x, vp)
    kp_err = float(np.linalg.norm(j - gt_j, axis=-1).mean())
    acc, f = [], 0
    for q in seqs:
        T = len(q["frames"])
        for t in range(2, T):
            if loss[f + t - 2] <= 5000.0 and loss[f + t - 1] <= 5000.0:
                a_fit = j[f + t] - 2 * j[f + t - 1] + j[f + t - 2]
                a_gt = gt_j[f + t] - 2 * gt_j[f + t - 1] + gt_j[f + t - 2]
                acc.append(np.linalg.norm(a_fit - a_gt, axis=-1).mean())
        f += T
    return dict(config=kind, lam=lam, keypoint_err_m=kp_err, accel_err_m=float(np.mean(acc)), n_accel=len(acc),
                mean_final_loss=float(np.nanmean(loss)), lockstep_s=t_lock, stream_s=t_stream, stream_equals_lockstep=same)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seqs", type=int, default=64)
    ap.add_argument("--frames", type=int, default=32)
    ap.add_argument("--views", type=int, default=8)
    ap.add_argument("--lams", default="0,10,100,1000")
    ap.add_argument("--configs", default="shipped,bench")
    ap.add_argument("--max-outer", type=int, default=30)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    model, gmm, cams = S.make_model(0), S.make_gmm(7), S.make_cameras(a.views)
    seqs, gt = [], []
    for s_ in range(a.seqs):
        fr = S.make_frames(model, cams, a.frames, seed=5000 + s_, smooth_walk=True)
        seqs.append(dict(gt_uv=fr["gt_uv"], conf=fr["conf"], present=np.ones(fr["conf"].shape[:2], bool),
                         frames=["%05d" % t for t in range(a.frames)], serial="s%03d" % s_))
        gt.append(fr["gt_joints3d"])
    gt_j = np.concatenate(gt).astype(np.float64)
    name = torch.cuda.get_device_name(0)
    out = open(a.out, "w") if a.out else None
    for kind in a.configs.split(","):
        for lam in [float(v) for v in a.lams.split(",")]:
            r = measure(model, gmm, cams, seqs, gt_j, kind, lam, dict(max_outer=a.max_outer))
            r.update(device=name, seqs=a.seqs, frames=a.frames, views=a.views)
            print(json.dumps(r), flush=True)
            if out:
                out.write(json.dumps(r) + "\n")
                out.flush()


if __name__ == "__main__":
    main()
