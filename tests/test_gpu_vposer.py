"""GPU: VPoser.decode on the device (use_vposer = 2) -- closure loss / gradients / joints against fixtures written by the
unmodified reference fitting closure with use_vposer=True (oracle/make_golden_vposer.py), and the optimiser on top."""
import os

import numpy as np
import pytest
import torch

from mvsmplfitting_b200 import synthetic as S
from tests import golden_util as G

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "vposer_s11.npz")


REAL = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "vposer_real.npz")


def _ctx(model, c, B, weights=None):
    from mvsmplfitting_b200.context import FittingContext
    ctx = FittingContext(0)
    ctx.set_model(model)
    ctx.set_vposer(S.make_vposer(11) if weights is None else weights)
    ctx.set_cameras(c["cam_R"], c["cam_t"], c["cam_f"], c["cam_c"])
    ctx.set_batch(B)
    ctx.set_keypoints(c["gt_uv"], c["conf"], c["joint_weights"])
    return ctx


def _x_with_latent(c):
    X = c["X"].copy()
    X[:, 13:82] = 0.0
    X[:, 13:45] = c["closure_Z"]                  # latent code in the first 32 entries of the pose slot
    return X


@pytest.mark.parametrize("stage", [3, 0])
def test_closure_with_device_vposer_matches_reference(stage, syn_model):
    c = np.load(GOLD)
    ctx = _ctx(syn_model, c, 2)
    dw, bpw, sw, bend = [float(v) for v in c["w%d" % stage]]
    ctx.set_loss(body_prior="l2", use_vposer=2, data_weight=dw, body_pose_weight=bpw, shape_weight=sw, bending_prior_weight=bend)
    out = ctx.closure(torch.tensor(_x_with_latent(c), device="cuda"), want_joints=True)
    loss, g, joints = out["loss"].cpu().numpy(), out["grad"].cpu().numpy(), out["joints"].cpu().numpy()
    for b in range(2):
        pre = "s%d_b%d_f32_" % (stage, b)
        assert abs(loss[b] - float(c[pre + "loss"])) / abs(float(c[pre + "loss"])) < 1e-4
        assert G.relmax(joints[b], c[pre + "joints"]) < 1e-4
        for name, (a, e) in (("betas", (0, 10)), ("global_orient", (10, 13)), ("transl", (82, 85)), ("scale", (85, 86)),
                             ("pose_embedding", (13, 45))):
            assert G.relmax(g[b, a:e], c[pre + "g_" + name]) < 2e-4, (stage, b, name)
        assert (g[b, 45:82] == 0).all()
    ctx.close()


@pytest.mark.parametrize("stage", [3, 0])
def test_closure_with_the_shipped_snapshot_matches_reference(stage, syn_model):
    """the decoder weights of the reference's own priors/snapshots/poser_epoch091.pkl (read from the staged tree
    oracle/_ref/reference by the reference's loader; the fixture holds inputs / outputs only)"""
    from tests.test_vposer_golden import _real_weights
    c = np.load(REAL)
    ctx = _ctx(syn_model, c, 2, weights=_real_weights())
    dw, bpw, sw, bend = [float(v) for v in c["w%d" % stage]]
    ctx.set_loss(body_prior="l2", use_vposer=2, data_weight=dw, body_pose_weight=bpw, shape_weight=sw, bending_prior_weight=bend)
    out = ctx.closure(torch.tensor(_x_with_latent(c), device="cuda"), want_joints=True)
    loss, g, joints = out["loss"].cpu().numpy(), out["grad"].cpu().numpy(), out["joints"].cpu().numpy()
    for b in range(2):
        pre = "s%d_b%d_f32_" % (stage, b)
        assert abs(loss[b] - float(c[pre + "loss"])) / abs(float(c[pre + "loss"])) < 1e-4
        assert G.relmax(joints[b], c[pre + "joints"]) < 1e-4
        for name, (a, e) in (("betas", (0, 10)), ("global_orient", (10, 13)), ("transl", (82, 85)), ("scale", (85, 86)),
                             ("pose_embedding", (13, 45))):
            assert G.relmax(g[b, a:e], c[pre + "g_" + name]) < 2e-4, (stage, b, name)
    ctx.close()


def test_vposer_decode_entry_point_matches_the_reference_class(syn_model):
    """mvs_vposer_decode (what save_results does before writing a result, utils.py:741-743) against decode outputs of the
    unmodified reference class, synthetic weights and the shipped snapshot (incl. decode(0): max |aa| = 0.8225)"""
    from tests.test_vposer_golden import _real_weights
    for gold, weights in ((GOLD, None), (REAL, _real_weights())):
        c = np.load(gold)
        Z = c["Z"]
        from mvsmplfitting_b200.context import FittingContext
        ctx = FittingContext(0)
        ctx.set_model(syn_model)
        ctx.set_vposer(S.make_vposer(11) if weights is None else weights)
        ctx.set_batch(Z.shape[0])
        x = np.zeros((Z.shape[0], 86), np.float32)
        x[:, 13:45] = Z
        aa = ctx.vposer_decode(torch.tensor(x, device="cuda")).cpu().numpy()
        ref = c["aa_f64"]
        # rotations near pi flip the axis sign with the last bit: compare as rotations there
        ang = np.linalg.norm(ref.reshape(-1, 23, 3), axis=2)
        err = np.abs(aa - ref).reshape(-1, 23, 3).max(axis=2)
        assert (err[ang < 3.0] < 2e-4 * np.maximum(1.0, ang[ang < 3.0])).all(), gold
        assert (np.abs(np.linalg.norm(aa.reshape(-1, 23, 3), axis=2) - ang)[ang >= 3.0] < 1e-3).all()
        if weights is not None:
            assert abs(np.abs(aa[0]).max() - 0.8225) < 1e-4
        ctx.close()


def test_lbfgs_in_latent_space(syn_model):
    c = np.load(GOLD)
    ctx = _ctx(syn_model, c, 2)
    dw, bpw, sw, bend = [float(v) for v in c["w3"]]
    ctx.set_loss(body_prior="l2", use_vposer=2, data_weight=dw, body_pose_weight=bpw, shape_weight=sw, bending_prior_weight=bend)
    X0 = _x_with_latent(c)
    x = torch.tensor(X0, device="cuda")
    l0 = ctx.closure(x, want_grad=False)["loss"].cpu().numpy()
    n0 = ctx.launch_count()
    final, st = ctx.lbfgs_run(x, ctx.make_lbfgs_config(max_outer=5))
    assert ctx.launch_count() - n0 <= 4                      # frame-resident: the whole stage is one launch
    l1 = ctx.closure(x, want_grad=False)["loss"].cpu().numpy()
    assert (l1 < l0).all() and st["frames_nan"] == 0 and st["frame_iterations"] > 10
    xn = x.cpu().numpy()
    assert np.array_equal(xn[:, 45:82], X0[:, 45:82])        # only the latent code moves inside the pose slot
    assert not np.array_equal(xn[:, 13:45], X0[:, 13:45])
    ctx.close()


@pytest.mark.parametrize("sdf", [False, True])
def test_lbfgs_step_in_latent_space(sdf, syn_model):
    """mvs_lbfgs_step with use_vposer = 2 (one LBFGS.step per call, state persistent): k calls walk the same path as
    mvs_lbfgs_run with max_outer = k and the monitor's tests off; the value returned is the loss at entry of the step.
    The two entry points evaluate the closure in different kernels, so their fp32 results differ in the last bits, and the
    line searches amplify that from step to step (max |x difference| after 1 / 2 / 3 steps: 2e-6 / 3e-4 / 4e-2, measured on
    an H100): the parameters are compared after two steps, the iteration counts after three."""
    c = np.load(GOLD)
    dw, bpw, sw, bend = [float(v) for v in c["w3"]]
    kw = dict(body_prior="l2", use_vposer=2, data_weight=dw, body_pose_weight=bpw, shape_weight=sw, bending_prior_weight=bend)
    if sdf:
        kw.update(interpenetration=True, coll_loss_weight=1000.0, sdf_grid=128)
    X0 = _x_with_latent(c)
    l_run, it_run = {}, {}
    for k in (2, 3):
        ctx = _ctx(syn_model, c, 2)
        ctx.set_exec_mode(3 if sdf else 0)          # closures with the SDF term + latent pose exist in the dense-regime kernels only
        ctx.set_loss(**kw)
        xr = torch.tensor(X0, device="cuda")
        _, st = ctx.lbfgs_run(xr, ctx.make_lbfgs_config(max_outer=k, max_iter=8, ftol=0.0, gtol=0.0))
        l_run[k], it_run[k] = ctx.closure(xr, want_grad=False)["loss"].cpu().numpy(), st["frame_iterations"]
        ctx.close()
    ctx = _ctx(syn_model, c, 2)
    ctx.set_exec_mode(3 if sdf else 0)
    ctx.set_loss(**kw)
    xs = torch.tensor(X0, device="cuda")
    l_entry0 = ctx.closure(xs, want_grad=False)["loss"].cpu().numpy()
    cfg = ctx.make_lbfgs_config(max_outer=1, max_iter=8)
    entry, its, x_after = [], 0, {}
    for k in range(3):
        loss, grad, st = ctx.lbfgs_step(xs, cfg, reset=(k == 0))
        entry.append(loss.cpu().numpy().copy())
        its += st["frame_iterations"]
        x_after[k + 1] = xs.clone()
        assert st["frame_iterations"] > 0 and torch.isfinite(grad).all()
        assert (grad[:, 45:82] == 0).all()
    assert np.abs(entry[0] - l_entry0).max() / np.abs(l_entry0).max() < 2e-4
    assert (entry[1] < entry[0]).all() and (entry[2] <= entry[1]).all()
    l_step = ctx.closure(x_after[2], want_grad=False)["loss"].cpu().numpy()
    assert np.abs(l_step - l_run[2]).max() / np.abs(l_run[2]).max() < 1e-3, (l_step, l_run[2])
    assert its == it_run[3], (its, it_run[3])
    assert np.array_equal(xs.cpu().numpy()[:, 45:82], X0[:, 45:82])
    ctx.close()


def test_device_vposer_guards(syn_model):
    from mvsmplfitting_b200.context import FittingContext
    from mvsmplfitting_b200._lib import MvsError
    c = np.load(GOLD)
    ctx = FittingContext(0)
    ctx.set_model(syn_model)
    ctx.set_cameras(c["cam_R"], c["cam_t"], c["cam_f"], c["cam_c"])
    ctx.set_batch(2)
    with pytest.raises(MvsError):
        ctx.set_loss(body_prior="l2", use_vposer=2)          # no decoder weights yet
    ctx.set_vposer(S.make_vposer(11))
    ctx.set_keypoints(c["gt_uv"], c["conf"], c["joint_weights"])
    ctx.set_loss(body_prior="l2", use_vposer=2)
    with pytest.raises(MvsError):                            # vertices requested -> batched chain, which has no decoder
        ctx.closure(torch.tensor(_x_with_latent(c), device="cuda"), want_verts=True)
    ctx.set_exec_mode(1)
    with pytest.raises(MvsError):
        ctx.closure(torch.tensor(_x_with_latent(c), device="cuda"))
    ctx.close()


def test_dense_regime_with_device_vposer_matches_oracle(syn_model):
    """SDF term + latent-space pose: the dense rounds decode the pose for the vertex kernels and back-propagate through the
    decoder in frame_step.  Pinned like the axis-angle dense regime: loss at entry and first search direction."""
    from oracle import closure_oracle as O
    c = np.load(GOLD)
    ctx = _ctx(syn_model, c, 2)
    dw, bpw, sw, bend = [float(v) for v in c["w3"]]
    cw = 1000.0
    ctx.set_loss(body_prior="l2", use_vposer=2, interpenetration=True, coll_loss_weight=cw, sdf_grid=128, data_weight=dw,
                 body_pose_weight=bpw, shape_weight=sw, bending_prior_weight=bend)
    X0 = _x_with_latent(c)
    x = torch.tensor(X0, device="cuda")
    n0 = ctx.launch_count()
    final, st = ctx.lbfgs_run(x, ctx.make_lbfgs_config(max_outer=1, max_iter=1))
    assert ctx.launch_count() - n0 > 8                       # dense rounds
    om = O.OracleModel.from_numpy(syn_model, dtype=torch.float32)
    cfg = O.LossConfig(data_weight=dw, body_pose_weight=bpw, shape_weight=sw, bending_prior_weight=bend, use_vposer=True,
                       interpenetration=True, coll_loss_weight=cw, sdf_grid=128)
    cams = dict(R=c["cam_R"], t=c["cam_t"], f=c["cam_f"], c=c["cam_c"])
    w = S.make_vposer(11)
    d = x.cpu().numpy().astype(np.float64) - X0
    for b in range(2):
        r = O.closure_eval_vposer(om, cfg, O.OraclePriors(kind="l2"), O.cams_to_torch(cams, torch.float32), X0[b],
                                  c["closure_Z"][b], w, c["gt_uv"][:, b], c["conf"][:, b], c["joint_weights"])
        assert abs(float(final[b]) - r["loss"]) / abs(r["loss"]) < 2e-4
        g = np.zeros(86)
        g[0:10], g[10:13], g[13:45], g[82:85], g[85:86] = r["g_betas"], r["g_global_orient"], r["g_pose_embedding"], r["g_transl"], r["g_scale"]
        cos = -(d[b] * g).sum() / (np.linalg.norm(d[b]) * np.linalg.norm(g))
        assert cos > 1 - 1e-6, (b, cos)
        assert (d[b, 45:82] == 0).all()
    ctx.close()


class _Decoder(torch.nn.Module):
    """a VPoser-shaped module: the reference's decoder layer names + decode(z, 'aa') (restated in oracle/vposer_oracle.py)"""

    def __init__(self, w, native_names=True):
        super().__init__()
        pre = "bodyprior_dec_" if native_names else "dec_"
        self._pre = pre
        for name, (o, i) in (("fc1", (512, 32)), ("fc2", (512, 512)), ("out", (138, 512))):
            lin = torch.nn.Linear(i, o)
            lin.weight.data = torch.tensor(w[name + "_w"])
            lin.bias.data = torch.tensor(w[name + "_b"])
            setattr(self, pre + name, lin)

    def decode(self, z, output_type="aa"):
        from oracle import vposer_oracle as VO
        g = lambda n: getattr(self, self._pre + n)
        h = torch.nn.functional.leaky_relu(g("fc1")(z), 0.2)
        h = torch.nn.functional.leaky_relu(g("fc2")(h), 0.2)
        R = VO.cont6d_to_matrot(g("out")(h))
        return VO.quaternion_to_angle_axis(VO.matrot_to_quaternion(R)).reshape(z.shape[0], 1, -1, 3)


def test_dropin_closure_native_decode_equals_host_decode(syn_model, syn_gmm, tmp_path):
    """FittingMonitor.create_fitting_closure(use_vposer=True): with the reference's decoder layers the decode runs on the
    device; with any other module PyTorch decodes upstream.  Same loss and gradients; the fused run_fitting works."""
    from mvsmplfitting_b200 import fitting, prior
    from mvsmplfitting_b200.optimizers import optim_factory
    from tests.test_gpu_dropin import build_scene
    c = np.load(GOLD)
    cams = dict(R=c["cam_R"], t=c["cam_t"], f=c["cam_f"], c=c["cam_c"])
    w = S.make_vposer(11)
    res = {}
    for native in (True, False):
        model, cam_list, _ = build_scene(syn_model, syn_gmm, tmp_path, cams, 1, "smpllsp", "l2")
        x = S.unpack_params(c["X"][:1])
        model.reset_params(**{k: torch.tensor(v) for k, v in x.items()})
        vp = _Decoder(w, native_names=native).cuda()
        emb = torch.tensor(c["closure_Z"][:1], device="cuda").requires_grad_(True)
        loss = fitting.create_loss("smplify", rho=100.0, use_joints_conf=True, body_pose_prior=prior.create_prior("l2"),
                                   shape_prior=prior.create_prior("l2"), angle_prior=prior.create_prior("angle"),
                                   interpenetration=False).to("cuda")
        dw, bpw, sw, bend = [float(v) for v in c["w3"]]
        loss.reset_loss_weights(dict(data_weight=torch.tensor(dw), body_pose_weight=torch.tensor(bpw),
                                     shape_weight=torch.tensor(sw), bending_prior_weight=torch.tensor(bend)))
        model.body_pose.requires_grad = False
        params = [p for p in model.parameters() if p.requires_grad] + [emb]
        opt, cg = optim_factory.create_optimizer(params, optim_type="lbfgsls", lr=1.0, maxiters=30)
        mon = fitting.FittingMonitor(maxiters=3, ftol=1e-9, gtol=1e-9)
        closure = mon.create_fitting_closure(
            opt, model, camera=cam_list, gt_joints=torch.tensor(c["gt_uv"][:, :1]).cuda(),
            joints_conf=[torch.tensor(c["conf"][v, :1]).cuda() for v in range(4)],
            joint_weights=torch.tensor(c["joint_weights"]).unsqueeze(0).cuda(), loss=loss, create_graph=cg, use_vposer=True,
            vposer=vp, pose_embedding=emb, return_verts=True, return_full_pose=True, use_3d=False)
        assert closure.vposer_native == native
        total = float(closure())
        res[native] = (total, emb.grad.detach().cpu().numpy().copy(), model.betas.grad.detach().cpu().numpy().copy())
        if native:
            assert abs(total - float(c["s3_b0_f32_loss"])) / float(c["s3_b0_f32_loss"]) < 1e-4
            assert G.relmax(res[True][1].reshape(-1), c["s3_b0_f32_g_pose_embedding"]) < 2e-4
            z0 = emb.detach().clone()
            entry = float(opt.step(closure))                 # one LBFGS.step on the device, in latent space
            assert abs(entry - total) / total < 1e-5 and not torch.equal(emb.detach(), z0) and float(closure()) < total
            final = mon.run_fitting(opt, closure, params, model, use_vposer=True, pose_embedding=emb, vposer=vp)
            assert final <= total and not torch.equal(emb.detach(), z0)
        else:
            with pytest.raises(NotImplementedError):         # no host-driven optimiser: the decoder must be on the device
                opt.step(closure)
    assert abs(res[True][0] - res[False][0]) / res[False][0] < 1e-4
    assert G.relmax(res[True][1], res[False][1]) < 2e-4 and G.relmax(res[True][2], res[False][2]) < 2e-4
