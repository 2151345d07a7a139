"""CPU: the oracle closure with the 3-D joint term (oracle/closure3d_oracle.py) against the reference-run fixtures
tests/golden/joints3d_closure_*.npz (oracle/make_golden_3d.py: SMPLifyLoss(use_3d=True) of the unmodified reference)."""
import glob
import json
import os

import numpy as np
import pytest
import torch

from oracle import closure3d_oracle as O3
from oracle import closure_oracle as O
from oracle import lbfgs_oracle as L
from tests import golden_util as G

CASES = sorted(os.path.basename(p)[len("joints3d_closure_"):-4] for p in glob.glob(G.GOLD + "/joints3d_closure_*.npz"))


def load(name):
    z = np.load(os.path.join(G.GOLD, "joints3d_closure_%s.npz" % name))
    d = {k: z[k] for k in z.files}
    d["meta"] = json.loads(str(d["meta"]))
    d["cams"] = {k: d["cam_" + k] for k in ("R", "t", "f", "c")}
    w = d["weights"]
    d["w"] = dict(data_weight=float(w[0]), body_pose_weight=float(w[1]), shape_weight=float(w[2]),
                  bending_prior_weight=float(w[3]))
    return d


def test_every_case_is_there():
    assert len(CASES) == 11


@pytest.mark.parametrize("name", CASES)
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_oracle_3d_closure_matches_reference(name, dtype, syn_model, syn_gmm):
    c = load(name)
    assert str(c["model_checksum"]) == G.model_checksum(syn_model)
    tag = "f32" if dtype == torch.float32 else "f64"
    om = O.OracleModel.from_numpy(syn_model, dtype=dtype, model_type=c["meta"]["model_type"])
    pri = O.OraclePriors.gmm_from_dict(syn_gmm, dtype) if c["meta"]["body_prior"] == "gmm" else O.OraclePriors("l2")
    vp = c["meta"].get("use_vposer", False)
    cfg = O.LossConfig(fix_shape=c["meta"]["fix_shape"], use_3d=True, use_vposer=vp, rho=float(c["rho"]), **c["w"])
    r = O3.closure_eval_batch_3d(om, cfg, pri, O.cams_to_torch(c["cams"], dtype), c["X"], c["gt_uv"], c["conf"],
                                 c["joint_weights"], c["gt3d"], c["conf3d"], Z=c.get("Z"),
                                 vposer_w=G.snapshot_vposer_weights() if vp else None)
    tol_loss, tol_grad = (2e-6, 1e-4) if dtype == torch.float32 else (1e-12, 1e-10)
    assert G.relmax(r["loss"], c["loss_" + tag]) < tol_loss
    g_ref = c["grad_" + tag]
    if c["meta"]["fix_shape"]:
        r["grad"][:, :10] = 0.0                  # frozen betas carry no grad in the reference
    for a, b in L.PARAM_SEGMENTS:
        if np.abs(g_ref[:, a:b]).max() > 0:
            assert G.relmax(r["grad"][:, a:b], g_ref[:, a:b]) < tol_grad, (a, b)
    assert G.relmax(r["joints"], c["joints_" + tag]) < tol_grad


def test_the_3d_term_carries_weight_in_the_dominated_cases(syn_model, syn_gmm):
    """l2_4_3donly: without the 3-D term the loss would be a fraction of the fixture's (the fixtures can tell a missing term)"""
    c = load("l2_4_3donly")
    om = O.OracleModel.from_numpy(syn_model, dtype=torch.float64)
    cfg = O.LossConfig(fix_shape=False, use_3d=False, **c["w"])
    r = O.closure_eval_batch(om, cfg, O.OraclePriors("l2"), O.cams_to_torch(c["cams"], torch.float64), c["X"], c["gt_uv"],
                             c["conf"], c["joint_weights"])
    assert (r["loss"] < 0.5 * c["loss_f64"]).all()


@pytest.mark.parametrize("tag", ["mv4", "sv"])
def test_reference_init_guess_aligns_to_the_annotations(tag, syn_model):
    """joints3d_init.npz (the reference's init_guess(use_3d=True)): its result is the as-written alignment of the rest joints'
    torso to the annotations' torso (init_guess.py:85-86), whatever the views say; numpy's own SVD, as in the authoring run"""
    from mvsmplfitting_b200 import synthetic as S
    from oracle import init_oracle as IO
    g = np.load(os.path.join(G.GOLD, "joints3d_init.npz"))
    z = lambda n: np.zeros((1, n))
    rest = S.model_keypoints_np(syn_model, z(10), z(3), z(69), z(3), np.ones((1, 1)), "smpllsp")[0].astype(np.float64)
    torso = [5, 6, 11, 12]
    for b in range(g[tag + "_params"].shape[0]):
        rot, tr, sc = IO.umeyama_as_written(rest[torso], g[tag + "_gt3d"][b].astype(np.float64)[torso], True)
        x = g[tag + "_params"][b]
        assert np.abs(IO.rotmat_to_aa(rot) - x[10:13]).max() < 2e-6
        assert np.abs(np.reshape(tr, -1) - x[82:85]).max() < 2e-6
        assert abs(sc - x[85]) < 1e-6 * x[85]
