"""GPU: the wgmma / TMA dense vertex forward (mvs_tc.cu) against the fp32 SIMT kernel and the oracle."""
import numpy as np
import pytest
import torch

from mvsmplfitting_b200 import synthetic as S
from oracle import closure_oracle as O
from oracle.lbfgs_oracle import PARAM_SEGMENTS
from tests import golden_util as G

pytestmark = pytest.mark.gpu


def make_ctx(model, cams, B, gmm, mode):
    from mvsmplfitting_b200.context import FittingContext
    ctx = FittingContext(0)
    ctx.set_model(model)
    ctx.set_gmm_from_dict(gmm)
    ctx.set_cameras(cams["R"], cams["t"], cams["f"], cams["c"])
    ctx.set_batch(B)
    ctx.set_exec_mode(mode)
    return ctx


@pytest.mark.parametrize("B", [256, 70, 1, 300, 129])
def test_tensor_core_vertex_forward_matches_fp32_kernel(B, syn_model, syn_gmm):
    cams = S.make_cameras(4)
    fr = S.make_frames(syn_model, cams, B, seed=60 + B)
    w = dict(data_weight=500.0 / 1536, body_pose_weight=4.78, shape_weight=5.0, bending_prior_weight=3.17 * 4.78)
    X = S.pack_params(fr["gt"])           # large poses: the pose blend shapes matter
    outs = []
    for mode in (0, 1):
        ctx = make_ctx(syn_model, cams, B, syn_gmm, mode)
        ctx.set_keypoints(fr["gt_uv"], fr["conf"], fr["joint_weights"])
        ctx.set_loss(body_prior="gmm", **w)
        x = torch.tensor(X, device="cuda")
        o = ctx.closure(x, want_joints=True, want_verts=True)
        torch.cuda.synchronize()
        prof_names = None
        if mode == 0:
            ctx.profile(0xFFFFFFFF)
            ctx.closure(x, want_verts=True)
            prof_names = set(ctx.profile_read())
            assert "posedirs_gemm_tc" in prof_names and "skin" in prof_names and "vertex_fwd" not in prof_names
        outs.append({k: v.cpu().numpy().astype(np.float64) for k, v in o.items()})
        ctx.close()
    a, b = outs
    assert np.isfinite(a["verts"]).all()
    assert np.abs(a["verts"] - b["verts"]).max() < 2e-5 * np.abs(b["verts"]).max()
    assert G.relmax(a["loss"], b["loss"]) < 1e-4 and G.relmax(a["joints"], b["joints"]) < 2e-5
    for lo, hi in PARAM_SEGMENTS:
        assert G.relmax(a["grad"][:, lo:hi], b["grad"][:, lo:hi]) < 1e-4
    # and against the oracle (fp64) on a few frames
    om = O.OracleModel.from_numpy(syn_model, dtype=torch.float64)
    sel = sorted(set([0, B - 1, B // 2]))
    ref = O.closure_eval_batch(om, O.LossConfig(**w), O.OraclePriors.gmm_from_dict(syn_gmm, torch.float64),
                               O.cams_to_torch(cams, torch.float64), X[sel], fr["gt_uv"][:, sel], fr["conf"][:, sel],
                               fr["joint_weights"], want_verts=True)
    assert G.relmax(a["verts"][sel], ref["verts"]) < 1e-4
    assert G.relmax(a["loss"][sel], ref["loss"]) < 1e-4
