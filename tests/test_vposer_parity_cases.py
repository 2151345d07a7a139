"""CPU: the frames and latent codes of tests/test_gpu_vposer_parity.py (tests/vposer_cases.py) reach what those tests are
meant to cover, and stay clear of the places where a float32 decode may legitimately differ from the float64 oracle."""
import numpy as np
import pytest
import torch

from oracle import vposer_oracle as VO
from tests import vposer_cases as VC


def _branches(decoder):
    with torch.no_grad():
        return VO.rotation_branches(VC.decoder_weights(decoder), VC.latent_codes(decoder).astype(np.float64))


@pytest.mark.parametrize("decoder", VC.DECODERS)
def test_rotations_clear_of_branch_surfaces_and_of_pi_and_well_conditioned(decoder):
    r = _branches(decoder)
    dist = r["margin"]
    assert dist.shape == (VC.POOL, 23)
    assert dist.min() > VC.BRANCH_MARGIN, dist.min()
    assert (np.pi - r["angle"]).min() > VC.PI_MARGIN, r["angle"].max()
    Z = VC.latent_codes(decoder)
    with torch.no_grad():
        pose32 = VO.decode_aa(VC.decoder_weights(decoder), torch.tensor(Z)).numpy()
    assert np.abs(pose32 - VC.decode64(VC.decoder_weights(decoder), Z)).max() < VC.DECODE32_MARGIN
    print("[%s] branches %s  cos < 0: %d  closest surface %.2e  largest angle %.4f" % (
        decoder, np.bincount(r["branch"].ravel(), minlength=4).tolist(), int(r["cos_neg"].sum()), dist.min(),
        r["angle"].max()))


def test_synthetic_decoder_reaches_every_quaternion_branch():
    """every branch with at least 10 joint rotations, among the frames every GPU case compares (B = 5 and 40 of
    test_gpu_dense_parity.CHECK_FRAMES), and both signs of the quaternion's scalar part"""
    from tests.test_gpu_dense_parity import CHECK_FRAMES, EDGE_FRAMES
    r = _branches("synthetic")
    for frames in (list(CHECK_FRAMES), EDGE_FRAMES):
        counts = np.bincount(r["branch"][frames].ravel(), minlength=4)
        assert counts.min() >= 10, counts
        assert r["cos_neg"][frames].any() and not r["cos_neg"][frames].all()


def test_snapshot_decoder_cases_are_built():
    """the shipped snapshot decodes nearly every rotation in branch 3: no coverage is asserted, only that its cases exist
    and decode to finite poses"""
    case = VC.make_case("snapshot", V=2, n=40)
    assert np.isfinite(case["pose"]).all() and (case["X"][:, 45:82] == 0).all()
    assert np.array_equal(case["X"][:, 13:45], case["Z"])


@pytest.mark.parametrize("decoder", VC.DECODERS)
def test_bending_term_clear_of_the_cut_off(decoder):
    """every stage-weight set: each frame's bending term at least GATE_MARGIN from 1e4.  Synthetic decoder at
    body_pose_weight 57.4: at least 3 compared frames on each side, so that a device applying the axis-angle cut-off to a
    latent pose fails"""
    from tests.test_gpu_dense_parity import CHECK_FRAMES, EDGE_FRAMES
    a = VC.angle_sum(VC.make_case(decoder)["pose"])
    for name, sw in VC.stage_weights().items():
        rel = sw["bending_prior_weight"] * a / VC.ANGLE_CUT
        assert np.abs(rel - 1.0).min() > VC.GATE_MARGIN, (name, np.abs(rel - 1.0).min())
        if decoder == "synthetic" and name == "s2":
            for frames in (list(CHECK_FRAMES), EDGE_FRAMES):
                above = rel[frames] > 1.0
                assert above.sum() >= 3 and (~above).sum() >= 3, (frames, np.round(rel[frames], 2))


def test_oracle_decoded_pose_gradient_matches_the_latent_gradient():
    """closure_eval_vposer: the gradient with respect to the decoded pose, pulled back through the decoder's Jacobian, is
    the latent gradient minus the |z|^2 prior's; and evaluating at a given pose (use_vposer = 1) returns the same loss and
    pose gradient as decoding it"""
    from mvsmplfitting_b200 import synthetic as S
    from oracle import closure_oracle as O
    case = VC.make_case("synthetic", V=2, n=8)
    om = O.OracleModel.from_numpy(S.make_model(0), dtype=torch.float64)
    sw = VC.stage_weights()["s2"]
    cfg = O.LossConfig(use_vposer=True, **sw)
    cams_t = O.cams_to_torch(case["cams"], torch.float64)
    fr, X, Z, w = case["fr"], case["X"], case["Z"], case["w"]
    for i in range(4):
        kp = (fr["gt_uv"][:, i], fr["conf"][:, i], fr["joint_weights"])
        r = O.closure_eval_vposer(om, cfg, O.OraclePriors("l2"), cams_t, X[i], Z[i], w, *kp)
        assert r["proj"].shape == (2, 17, 2) and set(r["terms"]) == {"data", "pprior", "shape", "angle", "pen"}
        assert abs(sum(r["terms"].values()) - r["loss"]) < 1e-12 * abs(r["loss"])
        z = torch.tensor(Z[i].astype(np.float64)).view(1, 32)
        J = torch.autograd.functional.jacobian(lambda zz: VO.decode_aa(w, zz).reshape(-1), z).reshape(69, 32).numpy()
        prior = 2 * sw["body_pose_weight"] ** 2 * Z[i].astype(np.float64)
        np.testing.assert_allclose(J.T @ r["g_body_pose"], r["g_pose_embedding"] - prior, rtol=0,
                                   atol=1e-9 * np.abs(r["g_pose_embedding"]).max())
        r1 = O.closure_eval_vposer(om, cfg, O.OraclePriors("l2"), cams_t, X[i], Z[i], w, *kp, body_pose=r["body_pose"])
        assert abs(r1["loss"] - r["loss"]) < 1e-12 * abs(r["loss"])
        np.testing.assert_allclose(r1["g_body_pose"], r["g_body_pose"], rtol=0, atol=1e-10 * np.abs(r["g_body_pose"]).max())
        np.testing.assert_allclose(r1["g_pose_embedding"], prior, rtol=1e-12)
