"""Float64 restatement of the lens-distortion model of mvs_set_camera_rigs_dist (PyTorch autograd): OpenCV's projectPoints
with coefficients (k1, k2, p1, p2, k3) per view, its Newton inverse, and closure_oracle's loss with the distorted projection in
its 2-D term.  The model, the priors and every other term are closure_oracle's (and vposer_oracle's) own functions: the 2-D
term is added to closure_oracle.smplify_loss evaluated with zero joint weights, which leaves only its other terms."""
from __future__ import annotations

import numpy as np
import torch

from . import closure_oracle as O


def distort_norm(xn, yn, d):
    """(x', y') -> (x'', y''), d = (k1, k2, p1, p2, k3) (tensors or arrays, broadcasting)"""
    k1, k2, p1, p2, k3 = (d[..., i] for i in range(5))
    r2 = xn * xn + yn * yn
    a = 1 + k1 * r2 + k2 * r2 * r2 + k3 * r2 * r2 * r2
    xd = xn * a + 2 * p1 * xn * yn + p2 * (r2 + 2 * xn * xn)
    yd = yn * a + p1 * (r2 + 2 * yn * yn) + 2 * p2 * xn * yn
    return xd, yd


def project_distorted(cam_R, cam_t, cam_f, cam_c, dist, pts):
    """closure_oracle.project with the view's distortion dist [5]; pts [K,3] -> [K,2]"""
    x = torch.einsum("ki,ji->jk", cam_R, pts) + cam_t
    xd, yd = distort_norm(x[:, 0] / x[:, 2], x[:, 1] / x[:, 2], torch.as_tensor(np.asarray(dist, np.float64), dtype=x.dtype))
    return torch.stack([xd, yd], -1) * cam_f + cam_c


def undistort(uv, f, c, dist, steps=50):
    """Float64 Newton inverse of the distortion: pixels uv [...,2] of a view (f [2], c [2], dist [5]) -> ideal pixels [...,2]"""
    uv = np.asarray(uv, np.float64)
    f, c, d = np.asarray(f, np.float64), np.asarray(c, np.float64), np.asarray(dist, np.float64)
    td = (uv - c) / f
    x = torch.tensor(td.copy(), dtype=torch.float64)
    dt = torch.tensor(d)
    for _ in range(steps):
        x = x.detach().requires_grad_(True)
        xd, yd = distort_norm(x[..., 0], x[..., 1], dt)
        e = torch.stack([xd, yd], -1) - torch.tensor(td)
        J = torch.stack([torch.stack(torch.autograd.grad(e[..., i].sum(), x, retain_graph=True)[0].unbind(-1), -1)
                         for i in range(2)], -2)                                  # [..., 2 (out), 2 (in)]
        x = x.detach() - torch.linalg.solve(J, e.detach().unsqueeze(-1)).squeeze(-1)
    return x.detach().numpy() * f + c


def data_term(cfg, cams, dist, joints, gt_uv, conf, joint_weights):
    """fitting.py:312-316 with the distorted projection: (loss, proj [V,K,2]) for one frame"""
    dw = torch.tensor(cfg.data_weight, dtype=joints.dtype)
    loss, projs = 0.0, []
    for v in range(gt_uv.shape[0]):
        uv = project_distorted(cams["R"][v], cams["t"][v], cams["f"][v], cams["c"][v], dist[v], joints)
        projs.append(uv)
        w = (joint_weights * conf[v] if cfg.use_joints_conf else joint_weights).unsqueeze(-1)
        loss = loss + torch.sum(w ** 2 * O.gmof(gt_uv[v] - uv, cfg.rho)) * dw ** 2
    return loss, torch.stack(projs)


def closure_eval(om, cfg, pri, cams_t, dist, x86, gt_uv, conf, joint_weights, gt3d=None, conf3d=None, z=None, vposer_w=None):
    """closure_oracle.closure_eval for ONE frame with each view's distortion dist [V,5]; gt3d [K,3] / conf3d [K] add the 3-D
    term (cfg.use_3d); with vposer_w the body pose is VPoser.decode(z, 'aa') and the gradient's pose slot holds d loss / d z in
    its first 32 entries (the device's use_vposer = 2 layout).  Returns dict(loss, grad [86], joints, proj [V,K,2])."""
    dt = om.dtype
    x = torch.tensor(np.asarray(x86, dtype=np.float64), dtype=dt)
    parts, o = [], 0
    for n in O.PARAM_SIZES:
        parts.append(x[o:o + n].clone().view(1, n).requires_grad_(True))
        o += n
    betas, go, bp, tr, sc = parts
    emb = None
    if vposer_w is not None:
        from . import vposer_oracle as VO
        emb = torch.tensor(np.asarray(z, dtype=np.float64), dtype=dt).view(1, 32).requires_grad_(True)
        parts[2] = emb
        bp = VO.decode_aa(vposer_w, emb)
    verts, joints, full_pose = O.smpl_forward(om, betas, go, bp, tr, sc)
    T = lambda a: None if a is None else torch.tensor(np.asarray(a, np.float64), dtype=dt)
    jw, gt, cf = T(joint_weights), T(gt_uv), T(conf)
    rest, _ = O.smplify_loss(om, cfg, pri, cams_t, verts, joints, full_pose, betas, bp, gt, cf, torch.zeros_like(jw),
                             pose_embedding=emb, gt3d=T(gt3d), conf3d=T(conf3d))
    data, proj = data_term(cfg, cams_t, np.asarray(dist, np.float64), joints, gt, cf, jw)
    total = data + rest
    grads = torch.autograd.grad(total, parts, allow_unused=True)
    g = np.zeros(86)
    o = 0
    for n, gg in zip(O.PARAM_SIZES, grads):
        if gg is not None:
            v = gg.reshape(-1).numpy()
            g[o:o + v.shape[0]] = v
        o += n
    return dict(loss=float(total), grad=g, joints=joints.detach().numpy().copy(), proj=proj.detach().numpy().copy())


def closure_eval_batch(om, cfg, pri, cams_t, dist, X, gt_uv, conf, joint_weights, gt3d=None, conf3d=None, Z=None, vposer_w=None):
    """X [B,86], gt_uv [V,B,K,2], conf [V,B,K]; gt3d [B,K,3], conf3d [B,K], Z [B,32] as closure_eval.  proj [V,B,K,2]."""
    outs = [closure_eval(om, cfg, pri, cams_t, dist, X[b], gt_uv[:, b], conf[:, b], joint_weights,
                         None if gt3d is None else gt3d[b], None if conf3d is None else conf3d[b],
                         None if Z is None else Z[b], vposer_w) for b in range(X.shape[0])]
    return dict(loss=np.array([r["loss"] for r in outs]), grad=np.stack([r["grad"] for r in outs]),
                joints=np.stack([r["joints"] for r in outs]), proj=np.stack([r["proj"] for r in outs], 1))



def view_term(R, t, f, c, dist, q, gt_uv, conf, jw, dw, rho, use_conf):
    """camera_oracle.view_term with the view's distortion dist [5]: q [F,K,3], gt_uv [F,K,2], conf [F,K] (float64 tensors)"""
    from . import camera_oracle as CO
    x = q @ R.T + t
    xd, yd = distort_norm(x[..., 0] / x[..., 2], x[..., 1] / x[..., 2], torch.as_tensor(np.asarray(dist, np.float64)))
    uv = torch.stack([xd, yd], -1) * torch.as_tensor(np.asarray(f, np.float64)) + torch.as_tensor(np.asarray(c, np.float64))
    w = torch.as_tensor(np.asarray(jw, np.float64))[None, :] * (conf if use_conf else 1.0)
    w2 = w * w
    rho2 = float(rho) ** 2
    e = gt_uv - uv
    return ((w2 * CO.gmof(e[..., 0], rho2) + w2 * CO.gmof(e[..., 1], rho2)).sum(1) * float(dw) ** 2).sum()


def view_problem(cams, view, q, gt_uv, conf, jw, dw, rho, use_conf):
    """camera_oracle.ViewProblem of view `view` whose 2-D term projects through the view's distortion cams["dist"][view] (the
    coefficients are held, like f and c): called at an 86-entry row it returns (loss, gradient [86]) in float64"""
    from . import camera_oracle as CO

    class DistortedViewProblem(CO.ViewProblem):
        def __call__(self, row):
            x = torch.as_tensor(np.asarray(row, np.float64)).clone().requires_grad_(True)
            R, t = CO.cam_from_delta(self.R0, self.t0, x[CO.ROT], x[CO.CEN], self.sphere, self.E, self.n)
            loss = view_term(R, t, self.f, self.c, cams["dist"][view], self.q, self.gt_uv, self.conf, self.jw, self.dw, self.rho,
                             self.use_conf)
            loss.backward()
            g = torch.zeros(86, dtype=torch.float64)
            g[CO.ROT], g[CO.CEN] = x.grad[CO.ROT], x.grad[CO.CEN]
            if self.sphere:
                g[84] = 0
            return float(loss.detach()), g.numpy()

    return DistortedViewProblem(cams, view, q, gt_uv, conf, jw, dw, rho, use_conf)
