"""GPU: the tensor-core pose-offset contraction (posedirs_gemm_tc) at batch sizes on every wgmma N instance (8, 16, 32,
64, 128 frames) and column-tile boundary (128 frames per tile), and bitwise independence of a frame's vertices from its
slot and from the batch it runs in."""
import numpy as np
import pytest
import torch

from mvsmplfitting_b200 import synthetic as S
from tests import golden_util as G

pytestmark = pytest.mark.gpu

W = dict(data_weight=500.0 / 1536, body_pose_weight=4.78, shape_weight=5.0, bending_prior_weight=3.17 * 4.78)


def dense_verts(model, gmm, cams, X, mode=0):
    from mvsmplfitting_b200.context import FittingContext
    B = X.shape[0]
    fr = S.make_frames(model, cams, B, seed=5)
    ctx = FittingContext(0)
    try:
        ctx.set_model(model)
        ctx.set_gmm_from_dict(gmm)
        ctx.set_cameras(cams["R"], cams["t"], cams["f"], cams["c"])
        ctx.set_batch(B)
        ctx.set_exec_mode(mode)
        ctx.set_keypoints(fr["gt_uv"], fr["conf"], fr["joint_weights"])
        ctx.set_loss(body_prior="gmm", **W)
        o = ctx.closure(torch.tensor(X, device="cuda"), want_verts=True)
        torch.cuda.synchronize()
        return o["verts"].cpu().numpy()
    finally:
        ctx.close()


@pytest.mark.parametrize("B", [8, 9, 16, 17, 33, 64, 65, 128, 256, 257])
def test_tensor_core_vertices_match_fp32_kernel_on_tile_boundaries(B, syn_model, syn_gmm):
    cams = S.make_cameras(4)
    X = S.pack_params(S.make_frames(syn_model, cams, B, seed=300 + B)["gt"])     # large poses: the pose blend shapes matter
    a = dense_verts(syn_model, syn_gmm, cams, X, mode=0).astype(np.float64)     # tensor-core contraction + skin
    b = dense_verts(syn_model, syn_gmm, cams, X, mode=1).astype(np.float64)     # fp32 SIMT vertex kernel
    assert np.isfinite(a).all()
    assert np.abs(a - b).max() < 2e-5 * np.abs(b).max(), G.relmax(a, b)


def test_tensor_core_vertices_bitwise_independent_of_slot_and_batch(syn_model, syn_gmm):
    cams = S.make_cameras(4)
    probe = S.pack_params(S.make_frames(syn_model, cams, 3, seed=77)["gt"])     # the three frames followed everywhere
    ref = None
    for B in [8, 9, 64, 65, 128, 256, 257]:
        X = S.pack_params(S.make_frames(syn_model, cams, B, seed=400 + B)["gt"])
        for slots in ([0, 1, 2], [B - 1, B // 2, 3], [B - 2, 4, min(B - 1, 130)]):
            Xb = X.copy()
            Xb[slots] = probe
            v = dense_verts(syn_model, syn_gmm, cams, Xb)[slots]
            if ref is None:
                ref = v
            assert np.array_equal(v, ref), (B, slots, float(np.abs(v - ref).max()))
