"""GPU: the straggler tail of a dense fit.  During a dense-regime run frames converge at different times and are compacted
out of the active list once per chunk of 8 rounds; the survivors move to new slots, across 32-frame skinning groups and
128-frame posedirs column tiles, and the grids shrink with the host's (one chunk late) bound on the active count, down to
posedirs_gemm_tc's N = 8 instance and skin_small_kernel.  A frame's fitted parameters and final loss must depend on nothing
but the frame: not on its slot, not on its batch-mates, not on when they finish."""
import numpy as np
import pytest
import torch

from mvsmplfitting_b200 import synthetic as S

pytestmark = pytest.mark.gpu

B = 257


def make_ctx(model, gmm, cams, B):
    from mvsmplfitting_b200.context import FittingContext
    ctx = FittingContext(0)
    ctx.set_model(model)
    ctx.set_gmm_from_dict(gmm)
    ctx.set_cameras(cams["R"], cams["t"], cams["f"], cams["c"])
    ctx.set_batch(B)
    return ctx


def stages(ctx):
    """the four-stage fit_smpl.yaml schedule with the SDF term (as written, grid 128) in stages 2 and 3"""
    sw = S.STAGE_WEIGHTS
    return [ctx.make_loss_config(body_prior="gmm", interpenetration=i >= 2, sdf_grid=128, data_weight=500.0 / 1536,
                                 body_pose_weight=sw["body_pose_prior_weights"][i], shape_weight=sw["shape_weights"][i],
                                 bending_prior_weight=3.17 * sw["body_pose_prior_weights"][i],
                                 coll_loss_weight=sw["coll_loss_weights"][i] if i >= 2 else 0.0) for i in range(4)]


def fit(ctx, fr, X0, order):
    ctx.set_keypoints(np.ascontiguousarray(fr["gt_uv"][:, order]), np.ascontiguousarray(fr["conf"][:, order]),
                      fr["joint_weights"])
    x = torch.tensor(np.ascontiguousarray(X0[order]), device="cuda")
    final, st = ctx.fit(x, stages(ctx), ctx.make_lbfgs_config())
    return x.cpu().numpy(), final.cpu().numpy(), st


def test_dense_fit_frame_result_independent_of_slot_batch_and_tail(syn_model, syn_gmm):
    """Full four-stage fits (SDF term in stages 2-3) of 257 frames, in order and in a random permutation: every frame's
    parameters and final loss bit-identical.  Then every frame refitted alone (B = 1): bit-identical to its result at
    B = 257, slots 0, 31, 32, 127, 128, 129 and 256 included.

    The refits also give each frame's own dense evaluation count (mvs_lbfgs_stats.dense_frame_evals at B = 1).  Their sum
    must equal the B = 257 run's dense_frame_evals and their maximum its dense_rounds (the longest frame's count), so they
    are the counts of the batched run.  A frame is in the active list for exactly its count of rounds, so after the round
    count of the 9th-longest frame at most 8 frames are active.  The test requires that stretch to span more than three
    8-round chunks: compaction and the one-chunk-late host bound then bring the grids down to N = 8 and skin_small_kernel
    for at least one whole chunk at the end of the run.  Measured on an H100: 476 dense rounds, 129.7 evaluations per frame
    on average (39 at least), the 9th-longest frame at 289, so the last 187 rounds ran at most 8 frames and the last 277 at
    most 32."""
    cams = S.make_cameras(4)
    fr = S.make_frames(syn_model, cams, B, seed=2570)
    X0 = S.pack_params(fr["init"])
    ctx = make_ctx(syn_model, syn_gmm, cams, B)
    x_a, f_a, st = fit(ctx, fr, X0, np.arange(B))
    perm = np.random.RandomState(2571).permutation(B)
    x_p, f_p, st_p = fit(ctx, fr, X0, perm)
    ctx.close()
    inv = np.argsort(perm)
    x_p, f_p = x_p[inv], f_p[inv]
    same = (x_a == x_p).all(1) & ((f_a == f_p) | (np.isnan(f_a) & np.isnan(f_p)))
    assert same.all(), ("permuted batch", np.flatnonzero(~same)[:16])
    assert st["dense_rounds"] > 0 and st["frame_evals"] == st_p["frame_evals"], (st, st_p)
    c1 = make_ctx(syn_model, syn_gmm, cams, 1)
    evals = np.zeros(B, dtype=np.int64)
    for b in range(B):
        x1, f1, s1 = fit(c1, fr, X0, [b])
        assert np.array_equal(x1[0], x_a[b]) and (f1[0] == f_a[b] or (np.isnan(f1[0]) and np.isnan(f_a[b]))), ("alone", b)
        evals[b] = s1["dense_frame_evals"]
    c1.close()
    top = np.sort(evals)[::-1]
    tail = int(st["dense_rounds"] - top[8])
    print("[D] B=%d: dense_rounds %d, dense evaluations per frame mean %.1f min %d, 9th-longest frame %d -> %d rounds with "
          "<= 8 active frames; rounds with <= 32 active: %d" % (B, st["dense_rounds"], evals.mean(), evals.min(), top[8],
                                                                tail, int(st["dense_rounds"] - top[32])))
    assert evals.sum() == st["dense_frame_evals"] and top[0] == st["dense_rounds"], (evals.sum(), top[0], st)
    assert tail > 3 * 8, tail
