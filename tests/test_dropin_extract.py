"""CPU: the drop-in layer's mirror modules have the surface of the reference's modules, so that its init.py /
non_linear_solver.py can hand them over unchanged."""
import numpy as np
import pytest
import torch

from mvsmplfitting_b200 import synthetic as S


def test_mirror_modules_have_the_reference_surface(tmp_path, syn_model, syn_gmm):
    """constructor keywords / attribute names of the mirrors match what init.py and non_linear_solver.py use"""
    import pickle
    from mvsmplfitting_b200 import camera, prior, fitting
    from mvsmplfitting_b200 import smplx
    from mvsmplfitting_b200.optimizers import optim_factory
    from mvsmplfitting_b200.utils import utils
    ds = smplx.Struct(f=syn_model["f"], v_template=syn_model["v_template"], shapedirs=syn_model["shapedirs"],
                      posedirs=syn_model["posedirs"], J_regressor=syn_model["J_regressor"],
                      kintree_table=syn_model["kintree_table"], weights=syn_model["weights"])
    m = smplx.create_scale("unused", model_type="smpllsp", data_struct=ds, joint_mapper=utils.JointMapper(
        utils.smpl_to_annotation("smpllsp", pose_format="lsp14")), create_global_orient=True, create_body_pose=True,
        create_betas=True, create_transl=True, create_scale=True, dtype=torch.float32, batch_size=2,
        lsp_regressor_path="/nonexistent")
    assert [n for n, _ in m.named_parameters()] == ["betas", "global_orient", "body_pose", "transl", "scale"]
    assert tuple(m.posedirs.shape) == (207, 20670) and int(m.parents[0]) == -1 and tuple(m.scale.shape) == (2, 1)
    assert float(m.scale[0, 0]) == 1.0
    m.reset_params(transl=torch.ones(2, 3))
    assert float(m.transl.sum()) == 6.0 and float(m.scale.sum()) == 0.0      # reference semantics: others -> 0
    with open(tmp_path / "gmm_06.pkl", "wb") as f:
        pickle.dump({k: np.asarray(v) for k, v in syn_gmm.items()}, f)
    gp = prior.create_prior("gmm", prior_folder=str(tmp_path), num_gaussians=6, dtype=torch.float32)
    means, prec, nllw = S.gmm_buffers(syn_gmm)
    assert np.allclose(gp.nll_weights.numpy().reshape(-1), nllw, rtol=1e-5)
    cam = camera.create_camera(focal_length_x=2400.0, focal_length_y=2400.0, translation=torch.zeros(1, 3),
                               rotation=torch.eye(3).unsqueeze(0), center=torch.tensor([[1024.0, 768.0]]))
    uv = cam(torch.tensor([[[0.1, -0.2, 4.0]]]))
    assert np.allclose(uv.detach().numpy(), [[[1024 + 60.0, 768 - 120.0]]])
    loss = fitting.create_loss("smplify", rho=100, body_pose_prior=gp, shape_prior=prior.create_prior("l2"),
                               angle_prior=prior.create_prior("angle"), interpenetration=False, use_joints_conf=True,
                               fix_shape=False)
    loss.reset_loss_weights({"body_pose_weight": torch.tensor(57.4), "data_weight": 0.33, "coll_loss_weight": 3.0})
    assert abs(float(loss.body_pose_weight) - 57.4) < 1e-5 and not hasattr(loss, "coll_loss_weight")
    opt, cg = optim_factory.create_optimizer([p for p in m.parameters()], optim_type="lbfgsls", lr=1.0, maxiters=30)
    assert cg is False and opt.param_groups[0]["max_eval"] == 37 and opt.param_groups[0]["history_size"] == 100
    mon = fitting.FittingMonitor(maxiters=30, ftol=1e-9, gtol=1e-9)
    with pytest.raises(RuntimeError):
        mon.create_fitting_closure(opt, m, camera=[cam], gt_joints=torch.zeros(1, 2, 17, 2), loss=loss,
                                   joints_conf=[torch.ones(2, 17)], joint_weights=torch.ones(1, 17))   # CPU model: no fallback
