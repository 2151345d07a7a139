"""How much of sdf_fused the cone cull leaves, as the device computed it: lane 0 of the bench.py workload (make_frames seed 1000,
8 views, grid 128) through one exec-mode-3 round at each batch size, at the initial guess and at the true poses.  Reads
every frame's SdfFrameSetup (mvs_debug_sdf_setup) and prints the fractions of 64-vertex chunks, 256-vertex blocks and
sdf_fused CTAs that survive the cull (a CTA survives when one of its blocks does; blocks per CTA from sdf_passes_for, as
the launch picks them), mean and largest over the frames.

    python scripts/sdf_cull_stats.py [--out DIR] [B ...]        (default B: 256 64 8)"""
import argparse
import ctypes
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402
from mvsmplfitting_b200 import synthetic as S  # noqa: E402
from mvsmplfitting_b200.context import FittingContext  # noqa: E402

REC_WORDS = 52                                      # sizeof(SdfFrameSetup) / 4: skip bits in words 44-51, live blocks in 42-43


def passes_for(na, nblocks, cta_slots):             # sdf_passes_for in mvs_internal.cuh
    return 2 if na * nblocks > 2 * cta_slots else 1


def frame_stats(rec, N, passes):
    nbox, nblocks = (N + 63) // 64, (N + 255) // 256
    words = rec[44:52].view(np.uint32)
    c = np.arange(nbox)
    chunk_live = ((words[c // 32] >> (c % 32).astype(np.uint32)) & 1) == 0
    lw = rec[42:44].view(np.uint32)
    mask = int(lw[0]) | (int(lw[1]) << 32)
    block_live = np.array([(mask >> b) & 1 for b in range(nblocks)], bool)
    nparts = (nblocks + passes - 1) // passes
    cta_live = np.array([block_live[p * passes:(p + 1) * passes].any() for p in range(nparts)])
    return chunk_live.mean(), block_live.mean(), cta_live.mean()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("B", type=int, nargs="*")
    args = ap.parse_args()
    model, gmm, cams = S.make_model(0), S.make_gmm(7), S.make_cameras(8)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    fr_all = S.make_frames(model, cams, 256, seed=1000)
    rows = []
    print(torch.cuda.get_device_properties(0).name)
    print("| B | poses | blocks / CTA | chunks live (mean / max) | blocks live (mean / max) | CTAs live (mean / max) |")
    print("|---|---|---|---|---|---|")
    for B in args.B or [256, 64, 8]:
        ctx = FittingContext(0)
        ctx.set_model(model); ctx.set_gmm_from_dict(gmm); ctx.set_cameras(cams["R"], cams["t"], cams["f"], cams["c"])
        ctx.set_batch(B)
        ctx.set_keypoints(np.ascontiguousarray(fr_all["gt_uv"][:, :B]), np.ascontiguousarray(fr_all["conf"][:, :B]),
                          fr_all["joint_weights"])
        ctx.set_exec_mode(3)
        ctx.set_loss(body_prior="gmm", interpenetration=True, coll_loss_weight=1000.0, sdf_grid=128, data_weight=500 / 1536,
                     body_pose_weight=57.4, shape_weight=10.0, bending_prior_weight=3.17 * 57.4)
        N = ctx.N
        forced = int(os.environ.get("MVS_SDF_PASSES", "0"))
        passes = forced if 1 <= forced <= 8 else passes_for(B, (N + 255) // 256, 3 * sms)
        for poses in ("init", "gt"):
            x = torch.tensor(S.pack_params(fr_all[poses])[:B], device="cuda")
            ctx.closure(x)
            rec = np.zeros((B, REC_WORDS), np.float32)
            assert ctx.lib.mvs_debug_sdf_setup(ctx.h, rec.ctypes.data_as(ctypes.c_void_p)) == 0
            st = np.array([frame_stats(rec[s], N, passes) for s in range(B)])
            row = dict(B=B, poses=poses, passes=passes, chunks=[st[:, 0].mean(), st[:, 0].max()],
                       blocks=[st[:, 1].mean(), st[:, 1].max()], ctas=[st[:, 2].mean(), st[:, 2].max()])
            rows.append(row)
            f = lambda v: "%.1f %% / %.0f %%" % (100 * v[0], 100 * v[1])
            print("| %d | %s | %d | %s | %s | %s |" % (B, poses, passes, f(row["chunks"]), f(row["blocks"]), f(row["ctas"])))
        ctx.close()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "sdf_cull_stats.json"), "w") as fh:
            json.dump(rows, fh, indent=1)


if __name__ == "__main__":
    main()
