"""GPU: bitwise pin of the dense rounds (frame_step_kernel) -- a few L-BFGS outer steps with the SDF term on for 16 frames
in three configurations (GMM prior, device-decoded VPoser, sequence anchor), then the dense closure and the frame-resident
closure at the point reached.  The fixture (golden/frame_step_pin.npz) was written by scripts/make_frame_step_pin.py on an
H100; any change of a floating-point operation or of its order in the closure, the priors or the optimiser step shows up
as a bit difference in the parameters, losses or gradients, or as different iteration / round counts."""
import os

import numpy as np
import pytest
import torch

from mvsmplfitting_b200 import synthetic as S

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "frame_step_pin.npz")
CASES = ("gmm", "vposer", "anchor")
B = 16
STATS = ("frame_iterations", "frame_evals", "rounds", "dense_rounds", "frames_nan")


def run_case(name, model, gmm):
    """-> dict of arrays: the fitted parameters, final losses and counts of a short dense-regime lbfgs_run, the dense closure
    (loss, gradient) at the parameters reached, and the loss of the same closure with the SDF term off"""
    from mvsmplfitting_b200.context import FittingContext
    cams = S.make_cameras(8)
    seed = 1000 + CASES.index(name)
    fr = S.make_frames(model, cams, B, seed=seed)
    X = S.pack_params(fr["init"])
    w = dict(data_weight=500.0 / 1536, body_pose_weight=57.4, shape_weight=10.0, bending_prior_weight=3.17 * 57.4)
    ctx = FittingContext(0)
    ctx.set_model(model); ctx.set_gmm_from_dict(gmm)
    ctx.set_cameras(cams["R"], cams["t"], cams["f"], cams["c"]); ctx.set_batch(B)
    ctx.set_keypoints(fr["gt_uv"], fr["conf"], fr["joint_weights"])
    loss_kw = dict(body_prior="gmm", **w)
    rng = np.random.RandomState(seed)
    if name == "vposer":                       # latent code in the first 32 entries of the pose slot
        ctx.set_vposer(S.make_vposer(11))
        X[:, 13:82] = 0.0
        X[:, 13:45] = rng.normal(0, 0.3, size=(B, 32))
        loss_kw = dict(body_prior="l2", use_vposer=2, **w)
    elif name == "anchor":
        anchor = (X + rng.normal(0, 0.05, X.shape)).astype(np.float32)
        weight = rng.uniform(0, 3, X.shape).astype(np.float32)
        ctx.set_anchor(torch.tensor(anchor), torch.tensor(weight))
    sdf = dict(interpenetration=True, coll_loss_weight=1000.0, sdf_grid=128)
    ctx.set_exec_mode(3)                       # closures with the SDF term run in the dense-regime kernels
    ctx.set_loss(**loss_kw, **sdf)
    x = torch.tensor(X, device="cuda")
    final, st = ctx.lbfgs_run(x, ctx.make_lbfgs_config(max_outer=3, max_iter=8))
    out = ctx.closure(x)
    ctx.set_exec_mode(0)
    ctx.set_loss(**loss_kw)
    nosdf = ctx.closure(x, want_grad=False)
    torch.cuda.synchronize()
    r = dict(params=x.cpu().numpy(), final=final.cpu().numpy(), loss=out["loss"].cpu().numpy(),
             grad=out["grad"].cpu().numpy(), loss_nosdf=nosdf["loss"].cpu().numpy(),
             stats=np.array([st[k] for k in STATS], dtype=np.int64))
    ctx.close()
    return r


@pytest.mark.parametrize("name", CASES)
def test_dense_rounds_bitwise(name, syn_model, syn_gmm):
    g = np.load(GOLD)
    r = run_case(name, syn_model, syn_gmm)
    assert (g[name + "/loss"] - g[name + "/loss_nosdf"] > 1e-3 * g[name + "/loss"]).any(), "the pinned frames must penetrate"
    assert np.array_equal(r["stats"], g[name + "/stats"]), (dict(zip(STATS, r["stats"])), dict(zip(STATS, g[name + "/stats"])))
    for k in ("params", "final", "loss", "grad", "loss_nosdf"):
        assert np.array_equal(r[k], g[name + "/" + k]), (k, np.abs(r[k] - g[name + "/" + k]).max())
