"""FittingMonitor / SMPLifyLoss / create_loss with the reference's call signatures
(code/utils/fitting.py:36-415), backed by the fused CUDA closure and the device-resident L-BFGS.

    monitor.create_fitting_closure(optimizer, body_model, camera=[...], gt_joints=[V,B,17,2],
        joints_conf=[V x [B,17]], joint_weights=[1,17], loss=SMPLifyLoss, use_vposer=...,
        gt_joints3d=[B,17,3], joints3d_conf=[B,17] (3-D joint term, SMPLifyLoss(use_3d=True)), ...)
        -> fitting_func(backward=True) -> 0-dim loss tensor, gradients written to p.grad
    monitor.run_fitting(optimizer, closure, params, body_model, ...) -> final loss

The closure reads the CURRENT values of the caller's nn.Parameter objects on every call and writes
`.grad` on those that require grad (frozen ones get none), exactly like the autograd closure it
replaces (fitting.py:162-203).  `body_model`, cameras, priors and the loss object are read by duck
typing, so the reference's own modules are accepted as well as the mirrors in this package.
The reference is fixed to one frame (non_linear_solver.py:56); here every tensor may carry B frames.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn as nn

from . import synthetic as S
from .context import FittingContext, SEGMENT_BITS
from .utils import utils

PARAM_SLICES = dict(betas=(0, 10), global_orient=(10, 13), body_pose=(13, 82), transl=(82, 85), scale=(85, 86))


# --------------------------------------------------------------------------- model -> context
def extract_model(body_model) -> tuple:
    """(model dict, model_type, joint_map, extra_vertex_ids) from a reference-style SMPL module"""
    mt = getattr(body_model, "model_type", "smpl")
    pd = body_model.posedirs.detach().cpu().numpy()
    d = dict(v_template=body_model.v_template.detach().cpu().numpy(), shapedirs=body_model.shapedirs.detach().cpu().numpy(),
             posedirs=pd, J_regressor=body_model.J_regressor.detach().cpu().numpy(),
             parents=body_model.parents.detach().cpu().numpy(), weights=body_model.lbs_weights.detach().cpu().numpy(),
             f=body_model.faces_tensor.detach().cpu().numpy().astype(np.int32).reshape(-1, 3))
    if mt == "smpllsp":
        d["lsp_regressor"] = body_model.joint_regressor.detach().cpu().numpy()
    extra = body_model.vertex_joint_selector.extra_joints_idxs.detach().cpu().numpy().astype(np.int32)
    jm = getattr(body_model, "joint_mapper", None)
    if jm is not None and getattr(jm, "joint_maps", None) is not None:
        jmap = jm.joint_maps.detach().cpu().numpy().astype(np.int32)
    else:
        jmap = np.arange((14 if mt == "smpllsp" else 24) + len(extra), dtype=np.int32)
    return d, mt, jmap, extra


def model_context(body_model) -> FittingContext:
    """one libmvsmpl context per (model object, device, batch size), built on first use"""
    dev = body_model.v_template.device
    if dev.type != "cuda":
        raise RuntimeError("the body model must live on a CUDA device: mvsmplfitting_b200 has no CPU path")
    B = int(getattr(body_model, "batch_size", 1))
    key = (dev.index or 0, B)
    cached = body_model.__dict__.get("_mvs_ctx")
    if cached is not None and cached[0] == key:
        return cached[1]
    d, mt, jmap, extra = extract_model(body_model)
    ctx = FittingContext(key[0])
    ctx.set_model(d, model_type=mt, joint_map=jmap, extra_vertex_ids=extra)
    ctx.set_batch(B)
    body_model.__dict__["_mvs_ctx"] = (key, ctx)
    return ctx


# --------------------------------------------------------------------------- loss container
def create_loss(loss_type="smplify", **kwargs):
    if loss_type == "smplify":
        return SMPLifyLoss(**kwargs)
    raise ValueError("Unknown loss type: {}".format(loss_type))


class SMPLifyLoss(nn.Module):
    """Weights + flags of the SMPLify energy (fitting.py:208-280).  The energy itself
    (fitting.py:290-415) is evaluated, together with its gradient, by the fused CUDA closure."""

    def __init__(self, search_tree=None, pen_distance=None, tri_filtering_module=None, rho=100, body_pose_prior=None,
                 shape_prior=None, angle_prior=None, use_joints_conf=True, interpenetration=True, dtype=torch.float32,
                 data_weight=1.0, body_pose_weight=0.0, shape_weight=0.0, bending_prior_weight=0.0,
                 coll_loss_weight=0.0, reduction="sum", use_3d=False, sdf_all_faces=False, **kwargs):
        super().__init__()
        self.use_joints_conf = use_joints_conf
        self.angle_prior = angle_prior
        self.use_3d = use_3d
        self.robustifier = utils.GMoF(rho=rho)
        self.rho = rho
        self.body_pose_prior = body_pose_prior
        self.shape_prior = shape_prior
        self.fix_shape = kwargs.get("fix_shape")
        self.interpenetration = interpenetration
        self.sdf_all_faces = sdf_all_faces
        if self.interpenetration:
            from .sdf import SDF
            self.sdf = SDF()
        for name, val in (("data_weight", data_weight), ("body_pose_weight", body_pose_weight),
                          ("shape_weight", shape_weight), ("bending_prior_weight", bending_prior_weight)):
            self.register_buffer(name, torch.tensor(val, dtype=dtype))
        if self.interpenetration:
            self.register_buffer("coll_loss_weight", torch.tensor(coll_loss_weight, dtype=dtype))

    def reset_loss_weights(self, loss_weight_dict):
        for key in loss_weight_dict:
            if hasattr(self, key):
                cur = getattr(self, key)
                val = loss_weight_dict[key]
                if torch.is_tensor(val):
                    new = val.clone().detach()
                else:
                    new = torch.tensor(val, dtype=cur.dtype, device=cur.device)
                setattr(self, key, new)

    def forward(self, *args, **kwargs):
        raise NotImplementedError("SMPLifyLoss is evaluated inside the fused CUDA closure "
                                  "(FittingMonitor.create_fitting_closure); it has no standalone torch forward")


def loss_config_from(loss, params_requires_grad: dict, use_vposer: bool):
    """mvs_loss_config from a (reference-style) SMPLifyLoss object"""
    prior = getattr(loss, "body_pose_prior", None)
    if prior is not None and hasattr(prior, "precisions"):
        kind = "gmm"
    elif prior is not None and isinstance(prior, nn.Module):
        kind = "l2"
    else:
        kind = "none"
    shape_prior = getattr(loss, "shape_prior", None)
    if shape_prior is not None and hasattr(shape_prior, "precisions"):
        raise NotImplementedError("only the L2 shape prior is on the B200 path")
    frozen = [k for k, rg in params_requires_grad.items() if not rg]
    f = lambda name: float(getattr(loss, name)) if hasattr(loss, name) else 0.0
    return FittingContext.make_loss_config(
        data_weight=f("data_weight"), body_pose_weight=f("body_pose_weight"), shape_weight=f("shape_weight"),
        bending_prior_weight=f("bending_prior_weight"), coll_loss_weight=f("coll_loss_weight"), rho=float(loss.rho),
        body_prior=kind, use_joints_conf=bool(loss.use_joints_conf), use_vposer=bool(use_vposer),
        fix_shape=bool(getattr(loss, "fix_shape", False)), interpenetration=bool(getattr(loss, "interpenetration", False)),
        sdf_grid=128, sdf_all_faces=bool(getattr(loss, "sdf_all_faces", False)), frozen=frozen), kind


# --------------------------------------------------------------------------- closure
class FittingClosure:
    """Callable returned by FittingMonitor.create_fitting_closure."""

    def __init__(self, optimizer, body_model, camera, gt_joints, loss, joints_conf, joint_weights, use_vposer, vposer,
                 pose_embedding, return_verts=True, gt_joints3d=None, joints3d_conf=None):
        self.optimizer = optimizer
        self.body_model = body_model
        self.loss = loss
        self.use_vposer = bool(use_vposer)
        self.vposer = vposer
        self.pose_embedding = pose_embedding
        self.ctx = model_context(body_model)
        B, dev = self.ctx.B, self.ctx.device
        cams = [c.numpy_params() if hasattr(c, "numpy_params") else _camera_params(c) for c in camera]
        self.ctx.set_cameras(np.stack([c[0] for c in cams]), np.stack([c[1] for c in cams]),
                             np.array([c[2] for c in cams], np.float32), np.stack([c[3] for c in cams]))
        V = len(cams)
        gt = torch.as_tensor(gt_joints).to(dev, torch.float32).reshape(V, B, -1, 2).contiguous()
        K = gt.shape[2]
        if joints_conf is None:
            conf = torch.ones(V, B, K, device=dev)
        else:
            conf = torch.stack([torch.as_tensor(c).to(dev, torch.float32).reshape(B, K) for c in joints_conf]).contiguous()
        jw = torch.as_tensor(joint_weights).to(dev, torch.float32).reshape(-1)[:K].contiguous()
        self.ctx.set_keypoints(gt, conf, jw)
        # 3-D joint term: on when the loss says so (SMPLifyLoss.use_3d, fitting.py:320), with the targets passed here
        if getattr(loss, "use_3d", False):
            if gt_joints3d is None or joints3d_conf is None:
                raise ValueError("use_3d needs gt_joints3d and joints3d_conf (non_linear_solver.py:86-99)")
            self.ctx.set_joints3d(torch.as_tensor(gt_joints3d).to(dev, torch.float32).reshape(B, K, 3),
                                  torch.as_tensor(joints3d_conf).to(dev, torch.float32).reshape(B, K))
        elif getattr(self.ctx, "_j3d_keep", None) is not None:      # the model's context had the term on: off again
            self.ctx.set_joints3d(None)
        self._gmm_of = None
        self.last = None
        # VPoser: when the module exposes the reference's decoder layers (model/VPoser.py:190-197) the decode runs on
        # the device inside the closure (mvs_set_vposer / use_vposer = 2); any other module is decoded by PyTorch upstream
        self.vposer_native = False
        if self.use_vposer and all(hasattr(vposer, n) for n in ("bodyprior_dec_fc1", "bodyprior_dec_fc2", "bodyprior_dec_out")) \
                and pose_embedding is not None and tuple(pose_embedding.shape[-1:]) == (32,):
            g = lambda layer, what: getattr(getattr(vposer, layer), what).detach().float().cpu().numpy()
            self.ctx.set_vposer(dict(fc1_w=g("bodyprior_dec_fc1", "weight"), fc1_b=g("bodyprior_dec_fc1", "bias"),
                                     fc2_w=g("bodyprior_dec_fc2", "weight"), fc2_b=g("bodyprior_dec_fc2", "bias"),
                                     out_w=g("bodyprior_dec_out", "weight"), out_b=g("bodyprior_dec_out", "bias")))
            self.vposer_native = True

    # -- parameter plumbing: the caller's nn.Parameters are the single source of truth
    def _named(self):
        # under VPoser the pose slot belongs to the decoder (decoded pose or latent code), not to body_model.body_pose
        return {k: getattr(self.body_model, k) for k in PARAM_SLICES
                if hasattr(self.body_model, k) and not (self.use_vposer and k == "body_pose")}

    def gather_params(self, body_pose=None) -> torch.Tensor:
        B, dev = self.ctx.B, self.ctx.device
        x = torch.zeros(B, S.NUM_PARAMS, dtype=torch.float32, device=dev)
        x[:, 85] = 1.0
        for k, p in self._named().items():
            a, e = PARAM_SLICES[k]
            x[:, a:e] = p.detach().reshape(B, e - a)
        if body_pose is not None:
            x[:, 13:82] = body_pose.detach().reshape(B, 69)
        elif self.vposer_native:
            x[:, 13:82] = 0.0
            x[:, 13:45] = self.pose_embedding.detach().reshape(B, 32)       # latent code in the pose slot (use_vposer = 2)
        return x.contiguous()

    @torch.no_grad()
    def scatter_params(self, x: torch.Tensor, grad: torch.Tensor | None = None):
        for k, p in self._named().items():
            a, e = PARAM_SLICES[k]
            if p.requires_grad:
                p.copy_(x[:, a:e].reshape(p.shape))
                if grad is not None:
                    p.grad = grad[:, a:e].reshape(p.shape).clone()
        if self.vposer_native and self.pose_embedding.requires_grad:
            self.pose_embedding.copy_(x[:, 13:45].reshape(self.pose_embedding.shape))
            if grad is not None:
                self.pose_embedding.grad = grad[:, 13:45].reshape(self.pose_embedding.shape).clone()

    def sync_loss_config(self):
        rg = {k: bool(p.requires_grad) for k, p in self._named().items()}
        if self.use_vposer:
            rg["body_pose"] = True          # driven through the decoder
        for k in PARAM_SLICES:
            rg.setdefault(k, False)
        cfg, kind = loss_config_from(self.loss, rg, self.use_vposer)
        if self.vposer_native:
            cfg.use_vposer = 2
        if kind == "gmm" and not self.use_vposer and self._gmm_of is not self.loss.body_pose_prior:
            pr = self.loss.body_pose_prior
            self.ctx.set_gmm(pr.means.detach().cpu().numpy(), pr.precisions.detach().cpu().numpy(),
                             pr.nll_weights.detach().cpu().numpy().reshape(-1))
            self._gmm_of = pr
        self.ctx.set_loss(config=cfg)
        return cfg

    def __call__(self, backward=True):
        if backward:
            self.optimizer.zero_grad()
        B = self.ctx.B
        body_pose = None
        if self.use_vposer and not self.vposer_native:
            body_pose = self.vposer.decode(self.pose_embedding, output_type="aa").view(B, -1)
        self.sync_loss_config()
        x = self.gather_params(body_pose=body_pose)
        out = self.ctx.closure(x, want_grad=backward)
        total = out["loss"].sum()
        if self.use_vposer and not self.vposer_native:
            bpw = float(self.loss.body_pose_weight)
            total = total + (self.pose_embedding.detach() ** 2).sum() * bpw ** 2      # fitting.py:327-329
        if backward:
            g = out["grad"]
            for k, p in self._named().items():
                if p.requires_grad:
                    a, e = PARAM_SLICES[k]
                    p.grad = g[:, a:e].reshape(p.shape).clone()
            if self.vposer_native:
                if self.pose_embedding.requires_grad:
                    self.pose_embedding.grad = g[:, 13:45].reshape(self.pose_embedding.shape).clone()
            elif self.use_vposer and self.pose_embedding.requires_grad:
                body_pose.backward(gradient=g[:, 13:82].reshape(body_pose.shape))
                with torch.no_grad():
                    self.pose_embedding.grad += 2.0 * float(self.loss.body_pose_weight) ** 2 * self.pose_embedding
        self.last = out
        return total


def _camera_params(cam):
    R = cam.rotation.detach()[0].cpu().numpy()
    t = cam.translation.detach()[0].cpu().numpy()
    f = [float(cam.focal_length_x.reshape(-1)[0]), float(cam.focal_length_y.reshape(-1)[0])]
    c = cam.center.detach().reshape(-1, 2)[0].cpu().numpy()
    return R, t, f, c


# --------------------------------------------------------------------------- monitor
class FittingMonitor(object):
    def __init__(self, summary_steps=1, visualize=False, maxiters=100, ftol=2e-09, gtol=1e-05,
                 body_color=(1.0, 1.0, 0.9, 1.0), model_type="smpl", **kwargs):
        self.maxiters = maxiters
        self.ftol = ftol
        self.gtol = gtol
        self.visualize = visualize
        self.summary_steps = summary_steps
        self.body_color = body_color
        self.model_type = model_type
        self.last_stats = None

    def create_fitting_closure(self, optimizer, body_model, camera=None, gt_joints=None, loss=None, joints_conf=None,
                               gt_joints3d=None, joints3d_conf=None, joint_weights=None, return_verts=True,
                               return_full_pose=False, use_vposer=False, vposer=None, pose_embedding=None,
                               create_graph=False, use_3d=False, **kwargs):
        if create_graph:
            raise NotImplementedError("create_graph=True (second-order) is not on the B200 path")
        if use_3d and (gt_joints3d is None or joints3d_conf is None):
            raise ValueError("use_3d needs gt_joints3d and joints3d_conf (non_linear_solver.py:86-99)")
        return FittingClosure(optimizer, body_model, camera, gt_joints, loss, joints_conf, joint_weights, use_vposer,
                              vposer, pose_embedding, return_verts=return_verts, gt_joints3d=gt_joints3d,
                              joints3d_conf=joints3d_conf)

    def run_fitting_stages(self, optimizer, closure, opt_weights):
        """The stage loop of non_linear_solver.py:109-203 in ONE call.  The reference does, per entry of
        `opt_weights`: loss.reset_loss_weights(weights); new optimiser; run_fitting.  Here the stages go to mvs_fit,
        where every frame moves to its next stage as soon as ITS current stage stops (same per-frame schedule and bits
        as the loop, no waiting for the slowest frame at a stage boundary).  Returns the last stage's final loss."""
        from .optimizers.lbfgs_ls import LBFGS
        if not (isinstance(optimizer, LBFGS) and isinstance(closure, FittingClosure) and
                (not closure.use_vposer or closure.vposer_native)):
            raise NotImplementedError("run_fitting_stages needs this package's LBFGS and closure (VPoser: the reference's "
                                      "decoder layers, so that the decode runs on the device)")
        cfgs = []
        for w in opt_weights:
            closure.loss.reset_loss_weights(w)
            cfgs.append(closure.sync_loss_config())
        x = closure.gather_params()
        cfg = optimizer.lbfgs_config(closure.ctx, max_outer=self.maxiters, ftol=self.ftol, gtol=self.gtol)
        final, st = closure.ctx.fit(x, cfgs, cfg)
        self.last_stats = st
        closure.scatter_params(x)
        vals = final.detach().cpu().numpy()
        return float(vals[0]) if vals.shape[0] == 1 else vals

    def run_fitting(self, optimizer, closure, params, body_model, use_vposer=True, pose_embedding=None, vposer=None,
                    camera=None, img_path=None, **kwargs):
        """fitting.py:71-142.  With this package's LBFGS + closure the whole loop (all outer steps, all
        frames) runs on the GPU in one call; any other optimiser is driven step by step from the host."""
        from .optimizers.lbfgs_ls import LBFGS
        if isinstance(optimizer, LBFGS) and isinstance(closure, FittingClosure) and \
                (not closure.use_vposer or closure.vposer_native):
            x = closure.gather_params()
            closure.sync_loss_config()
            cfg = optimizer.lbfgs_config(closure.ctx, max_outer=self.maxiters, ftol=self.ftol, gtol=self.gtol)
            final, st = closure.ctx.lbfgs_run(x, cfg)
            self.last_stats = st
            closure.scatter_params(x)
            vals = final.detach().cpu().numpy()
            return float(vals[0]) if vals.shape[0] == 1 else vals
        prev_loss = None
        for n in range(self.maxiters):
            loss = optimizer.step(closure)
            if torch.isnan(loss).sum() > 0:
                print("NaN loss value, stopping!")
                break
            if torch.isinf(loss).sum() > 0:
                print("Infinite loss value, stopping!")
                break
            if n > 0 and prev_loss is not None and self.ftol > 0:
                if utils.rel_change(prev_loss, loss.item()) <= self.ftol:
                    break
            if all([torch.abs(var.grad.view(-1).max()).item() < self.gtol for var in params if var.grad is not None]):
                break
            prev_loss = loss.item()
        return prev_loss
