"""GPU: which kernels every entry point runs, for each execution mode x SDF term x pose encoding (the dispatch of
mvs_lbfgs.cu: stage_regime and evaluate_closure), and mvs_lbfgs_step with the SDF term in exec mode 3, which must run the
same optimiser as in exec mode 0 (exec mode 3 only changes what mvs_closure evaluates).

`python -m tests.test_gpu_dispatch` prints the table the current build produces."""
import itertools

import numpy as np
import pytest
import torch

from mvsmplfitting_b200 import synthetic as S

pytestmark = pytest.mark.gpu

B, V = 4, 4
WEIGHTS = dict(data_weight=500.0 / 1536, body_pose_weight=4.78, shape_weight=5.0, bending_prior_weight=3.17 * 4.78)
SDF_ON = dict(interpenetration=True, coll_loss_weight=1000.0, sdf_grid=32)
ENTRIES = ("closure", "closure_verts", "forward_only", "lbfgs_run", "lbfgs_step", "fit")
SINGLE = ("closure", "closure_verts", "forward_only")     # exact launch counts; the runs: the set of kernels they launch

_CHAIN = dict(frame_fwd=1, keypoint_loss=1, frame_bwd=1, vertex_bwd=1)
_SDF = dict(sdf_bbox=1, sdf_sample=1, sdf_finalize=1)
_TC = dict(posedirs_gemm_tc=1, skin=1)
_DENSE_RUN = ["frame_fwd", "frame_step", "lbfgs_compact", "misc", "posedirs_gemm_tc", "sdf_fused", "skin"]
_CHAIN_RUN = ["frame_bwd", "frame_fwd", "keypoint_loss", "lbfgs_advance", "lbfgs_compact", "misc", "vertex_bwd", "vertex_fwd"]
# what one call launches: {kernel name: launches} for single evaluations, sorted kernel names for runs
PATHS = {
    "error": "MvsError",
    "resident": {"closure_resident": 1},
    "chain": dict(_CHAIN, vertex_fwd=1),
    "chain_verts": dict(_CHAIN, vertex_fwd=1, misc=1),
    "chain_verts_tc": dict(_CHAIN, **_TC, misc=1),
    "chain_sdf": dict(_CHAIN, **_SDF, vertex_fwd=1),
    "chain_sdf_verts": dict(_CHAIN, **_SDF, vertex_fwd=1, misc=1),
    "dense_closure": dict(frame_fwd=1, **_TC, sdf_fused=1, frame_step=1, misc=2),
    "forward": dict(frame_fwd=1, vertex_fwd=1, keypoint_loss=1, misc=1),
    "forward_tc": dict(frame_fwd=1, **_TC, keypoint_loss=1, misc=1),
    "run_resident": ["lbfgs_resident", "misc"],
    "run_dense": _DENSE_RUN,
    "run_resident_dense": sorted(_DENSE_RUN + ["lbfgs_resident"]),
    "run_chain": _CHAIN_RUN,
    "run_chain_sdf": sorted(_CHAIN_RUN + ["sdf_bbox", "sdf_finalize", "sdf_sample"]),
    "run_chain_resident": ["closure_resident", "lbfgs_advance", "lbfgs_compact", "misc"],
}
# (exec mode, SDF term, use_vposer) -> path of each entry point, in the order of ENTRIES.  The fit has two stages, the
# SDF term off and then on, with the row's use_vposer.
_AUTO = {
    (False, 0): ("resident", "chain_verts_tc", "forward_tc", "run_resident", "run_chain_resident", "run_resident_dense"),
    (False, 2): ("resident", "error", "forward_tc", "run_resident", "run_chain_resident", "run_resident_dense"),
    (True, 0): ("chain_sdf", "chain_sdf_verts", "forward_tc", "run_dense", "run_chain_sdf", "run_resident_dense"),
    (True, 2): ("error", "error", "forward_tc", "run_dense", "run_dense", "run_resident_dense"),
}
TABLE = {
    **{(0,) + k: v for k, v in _AUTO.items()},
    (1, False, 0): ("chain", "chain_verts", "forward", "run_chain", "run_chain", "run_chain_sdf"),
    (1, False, 2): ("error", "error", "forward", "error", "error", "error"),
    (1, True, 0): ("chain_sdf", "chain_sdf_verts", "forward", "run_chain_sdf", "run_chain_sdf", "run_chain_sdf"),
    (1, True, 2): ("error", "error", "forward", "error", "error", "error"),
    **{(2,) + k: v for k, v in _AUTO.items()},
    (3, False, 0): _AUTO[(False, 0)],
    (3, False, 2): _AUTO[(False, 2)],
    # only mvs_closure differs from exec mode 0: one evaluation through the dense-round kernels
    (3, True, 0): ("dense_closure", "chain_sdf_verts", "forward_tc", "run_dense", "run_chain_sdf", "run_resident_dense"),
    (3, True, 2): ("dense_closure", "error", "forward_tc", "run_dense", "run_dense", "run_resident_dense"),
}


def _context(model, gmm, cams, fr, mode):
    from mvsmplfitting_b200.context import FittingContext
    ctx = FittingContext(0)
    ctx.set_model(model)
    ctx.set_gmm_from_dict(gmm)
    ctx.set_vposer(S.make_vposer(11))
    ctx.set_cameras(cams["R"], cams["t"], cams["f"], cams["c"])
    ctx.set_batch(B)
    ctx.set_keypoints(fr["gt_uv"], fr["conf"], fr["joint_weights"])
    ctx.set_exec_mode(mode)
    return ctx


def _loss(ctx, sdf, vposer):
    return ctx.make_loss_config(body_prior="l2", use_vposer=vposer, **WEIGHTS, **(SDF_ON if sdf else {}))


def observe(model, gmm, mode, sdf, vposer):
    """{entry point: "MvsError" | {kernel: launches} | sorted kernel names} for one row of TABLE"""
    from mvsmplfitting_b200._lib import MvsError
    cams = S.make_cameras(V)
    fr = S.make_frames(model, cams, B, seed=5)
    X = S.pack_params(fr["init"])
    ctx = _context(model, gmm, cams, fr, mode)
    ctx.set_loss(config=_loss(ctx, sdf, vposer))
    opt = ctx.make_lbfgs_config(max_outer=2, max_iter=4)
    calls = dict(
        closure=lambda x: ctx.closure(x),
        closure_verts=lambda x: ctx.closure(x, want_verts=True),
        forward_only=lambda x: ctx.forward_only(x),
        lbfgs_run=lambda x: ctx.lbfgs_run(x, opt),
        lbfgs_step=lambda x: ctx.lbfgs_step(x, opt, reset=True),
        fit=lambda x: ctx.fit(x, [_loss(ctx, False, vposer), _loss(ctx, True, vposer)], opt),
    )
    out = {}
    for name in ENTRIES:
        ctx.set_loss(config=_loss(ctx, sdf, vposer))
        x = torch.tensor(X, device="cuda")
        ctx.profile()
        try:
            calls[name](x)
            prof = ctx.profile_read()
            out[name] = {k: n for k, (_, n) in sorted(prof.items())} if name in SINGLE else sorted(prof)
        except MvsError:
            ctx.profile_read()
            out[name] = "MvsError"
    ctx.profile(0)
    ctx.close()
    return out


ROWS = list(itertools.product((0, 1, 2, 3), (False, True), (0, 2)))


@pytest.mark.parametrize("mode,sdf,vposer", ROWS)
def test_entry_points_run_the_kernels_of_their_path(mode, sdf, vposer, syn_model, syn_gmm):
    got = observe(syn_model, syn_gmm, mode, sdf, vposer)
    want = dict(zip(ENTRIES, (PATHS[p] for p in TABLE[(mode, sdf, vposer)])))
    assert got == want, {k: (got[k], want[k]) for k in ENTRIES if got[k] != want[k]}


def test_lbfgs_step_with_sdf_term_is_the_same_in_exec_mode_3(syn_model, syn_gmm):
    """exec mode 3 changes what mvs_closure evaluates, never the optimiser: three mvs_lbfgs_step calls with the SDF term on
    give the bits of exec mode 0 (both run the batched chain)"""
    cams = S.make_cameras(V)
    fr = S.make_frames(syn_model, cams, B, seed=5)
    res = []
    for mode in (3, 0):
        ctx = _context(syn_model, syn_gmm, cams, fr, mode)
        ctx.set_loss(config=_loss(ctx, True, 0))
        x = torch.tensor(S.pack_params(fr["init"]), device="cuda")
        cfg = ctx.make_lbfgs_config(max_outer=1, max_iter=8)
        steps = []
        for k in range(3):
            loss, grad, st = ctx.lbfgs_step(x, cfg, reset=(k == 0))
            steps.append((loss.cpu().numpy(), grad.cpu().numpy(), st))
        res.append((x.cpu().numpy(), steps))
        ctx.close()
    (xa, sa), (xb, sb) = res
    assert np.array_equal(xa, xb)
    for k, ((la, ga, sta), (lb, gb, stb)) in enumerate(zip(sa, sb)):
        assert np.array_equal(la, lb) and np.array_equal(ga, gb), k
        assert sta == stb, (k, sta, stb)
        assert sta["frame_iterations"] > 0 and sta["frames_nan"] == 0, (k, sta)


if __name__ == "__main__":
    model, gmm = S.make_model(0), S.make_gmm(7)
    for row in ROWS:
        print(row, observe(model, gmm, *row), flush=True)
