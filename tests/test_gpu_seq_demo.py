"""GPU: seqio.fit_sequence end to end on the data the original project ships (data/keypoints/0000: six cameras, one frame;
data/3DOH50K_Parameters.txt; copied to tests/golden/demo) with its default configuration (cfg_files/fit_smpl.yaml: VPoser
latent pose from the shipped snapshot, L2 body prior, four stages, no interpenetration), against a run of the UNMODIFIED
reference solver (oracle/ref_fit.py -> utils/non_linear_solver.py) started from the same initial guess, stored in
tests/golden/seq_demo_ref.npz by oracle/make_golden_refruns.py.  The body model is the synthetic SMPL-shaped one (the SMPL
pickle is not redistributable)."""
import os
import pickle

import numpy as np
import pytest
import torch

from mvsmplfitting_b200 import seqio
from mvsmplfitting_b200 import synthetic as S
from oracle import vposer_oracle as VO
from tests import golden_util as G

pytestmark = pytest.mark.gpu
H_IMG = 1536                                     # 3DOH50K images are 2048 x 1536; data_weight = 500 / H (non_linear_solver.py:149-151)


def _stages(ctx):
    sw = S.STAGE_WEIGHTS
    return [ctx.make_loss_config(body_prior="l2", use_vposer=2, data_weight=500.0 / H_IMG,
                                 body_pose_weight=sw["body_pose_prior_weights"][i], shape_weight=sw["shape_weights"][i],
                                 bending_prior_weight=3.17 * sw["body_pose_prior_weights"][i]) for i in range(4)]


def demo_setup(model):
    """context, sequence, cameras, stage configs, joint weights and VPoser weights of the demo fit"""
    from mvsmplfitting_b200.context import FittingContext
    ext, intr = seqio.load_camera_para(os.path.join(G.DEMO, "3DOH50K_Parameters.txt"))
    seq = seqio.load_sequence(os.path.join(G.DEMO, "keypoints"), "0000")
    V, B = len(seq["cameras"]), len(seq["frames"])
    assert (V, B) == (6, 1) and seq["present"].all()
    cams = seqio.camera_arrays(ext, intr, views=range(V))
    vpw = G.snapshot_vposer_weights()
    ctx = FittingContext(0)
    ctx.set_model(model)
    ctx.set_vposer(vpw)
    ctx.set_cameras(cams["R"], cams["t"], cams["f"], cams["c"])
    ctx.set_batch(B)
    stages = _stages(ctx)
    jw = seqio.joint_weights("coco17", True)
    ctx.set_keypoints(seq["gt_uv"], seq["conf"], jw)
    ctx.set_loss(config=stages[0])
    return ctx, seq, cams, stages, jw, vpw


def test_fit_sequence_on_the_reference_demo_data(syn_model, syn_gmm, tmp_path):
    ctx, seq, cams, stages, jw, vpw = demo_setup(syn_model)
    opt = ctx.make_lbfgs_config(max_outer=30, ftol=1e-9, gtol=1e-9)
    ref = np.load(os.path.join(G.GOLD, "seq_demo_ref.npz"))

    # the initial guess the batch starts from (main.py:76-82; fix_scale: false -> the scale is estimated); the reference run
    # started from this guess
    p0, _ = ctx.init_guess(estimate_scale=True, fixed_scale=1.0, use_torso=True, hip_seed=1.0, want_joints3d=False)
    p0 = p0.cpu().numpy()
    assert (p0[:, 13:82] == 0).all() and np.isfinite(p0).all()                   # latent code starts at zero
    assert np.abs(p0 - ref["p0"]).max() <= 1e-4 * max(1.0, np.abs(ref["p0"]).max())

    x, loss, st = seqio.fit_sequence(ctx, seq, stages, opt, estimate_scale=True, result_folder=str(tmp_path / "res"),
                                     mesh_folder=str(tmp_path / "mesh"), faces=syn_model["f"])
    assert st["frames_nan"] == 0 and st["frame_iterations"] > 30 and np.isfinite(loss).all()

    # the unmodified reference on the same frame from the same start
    ref = dict(final_loss=float(ref["final_loss"]), iterations=int(ref["iterations"]), evals=int(ref["evals"]),
               params=ref["params"], pose_embedding=ref["pose_embedding"])
    rel = abs(loss[0] - ref["final_loss"]) / abs(ref["final_loss"])
    print("demo fit: device loss %.4f (%d iterations, %d evals)  reference loss %.4f (%d iterations, %d evals)  rel %.2e" %
          (loss[0], st["frame_iterations"], st["frame_evals"], ref["final_loss"], ref["iterations"], ref["evals"], rel))
    assert rel < 0.05
    assert abs(st["frame_iterations"] - ref["iterations"]) <= 0.35 * ref["iterations"]
    # deterministic part: the device closure at the reference's final parameters reproduces its final loss
    xr = ref["params"].copy()[None]
    xr[:, 13:82] = 0.0
    xr[:, 13:45] = ref["pose_embedding"]
    ctx.set_loss(config=stages[-1])
    l_at_ref = float(ctx.closure(torch.tensor(xr, device="cuda"), want_grad=False)["loss"][0])
    assert abs(l_at_ref - ref["final_loss"]) / abs(ref["final_loss"]) < 1e-3

    # the result file of the frame (utils.py:741-759,856-863): decoded pose with zeroed extremities + the latent code
    got = pickle.load(open(tmp_path / "res" / "0000" / seq["frames"][0] / "000.pkl", "rb"))
    assert got["pose_embedding"].shape == (1, 32) and np.array_equal(got["pose_embedding"][0], x[0, 13:45])
    dec = VO.decode_aa(vpw, torch.tensor(x[:, 13:45], dtype=torch.float64)).reshape(1, -1).numpy()
    for a, b in ((18, 24), (27, 33), (57, 69)):
        dec[:, a:b] = 0.0
    assert np.abs(got["body_pose"] - dec).max() < 2e-4
    assert got["pose"].shape == (1, 72) and abs(got["loss"] - loss[0]) < 1e-6 * abs(loss[0])
    assert os.path.exists(tmp_path / "mesh" / "0000" / seq["frames"][0] / "000.obj")
    ctx.close()
