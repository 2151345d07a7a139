"""per-kernel device time of ONE dense round (mvs_closure in exec mode 3 = the SDF-stage kernels with the optimiser step off)
at fixed batch sizes: python scripts/round_times.py [--joints3d] [B ...]
--joints3d: with the 3-D joint term on (targets = the frames' true keypoints, confidence 1)"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402
from mvsmplfitting_b200 import _lib, synthetic as S  # noqa: E402
if os.environ.get('MVS_LIB'):
    _lib.LIB_PATH = os.path.join(os.path.dirname(_lib.LIB_PATH), os.environ['MVS_LIB'])
from mvsmplfitting_b200.context import FittingContext  # noqa: E402

model, gmm, cams = S.make_model(0), S.make_gmm(7), S.make_cameras(8)
j3d = "--joints3d" in sys.argv[1:]
for B in [int(a) for a in sys.argv[1:] if a != "--joints3d"] or [256, 64, 5, 1]:
    fr = S.make_frames(model, cams, B, seed=1000)
    ctx = FittingContext(0)
    ctx.set_model(model); ctx.set_gmm_from_dict(gmm); ctx.set_cameras(cams["R"], cams["t"], cams["f"], cams["c"]); ctx.set_batch(B)
    ctx.set_keypoints(fr["gt_uv"], fr["conf"], fr["joint_weights"])
    if j3d:
        ctx.set_joints3d(fr["gt_joints3d"], np.ones(fr["gt_joints3d"].shape[:2], np.float32))
    ctx.set_exec_mode(3)
    ctx.set_loss(body_prior="gmm", interpenetration=True, coll_loss_weight=1000.0, sdf_grid=128, data_weight=500 / 1536,
                 body_pose_weight=57.4, shape_weight=10.0, bending_prior_weight=3.17 * 57.4)
    x = torch.tensor(S.pack_params(fr["init"]), device="cuda")
    for _ in range(3):
        ctx.closure(x)
    torch.cuda.synchronize()
    # un-instrumented wall time of the round (events around the whole call; includes the run's set-up launches)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(20):
        ctx.closure(x)
    e1.record(); torch.cuda.synchronize()
    ctx.profile(0xFFFFFFFF)
    for _ in range(20):
        ctx.closure(x)
    pr = ctx.profile_read()
    ctx.profile(0)
    print("B=%d%s: closure call %.1f us; per kernel (us): %s" % (B, " joints3d" if j3d else "", e0.elapsed_time(e1) * 1e3 / 20,
          {k: round(v[0] * 1e3 / max(v[1], 1), 1) for k, v in pr.items()}))
    ctx.close()
