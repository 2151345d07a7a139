"""TEST INFRASTRUCTURE -- the oracle closure (oracle/closure_oracle.py) with the 3-D joint term of SMPLifyLoss(use_3d=True)
(fitting.py:318-324): closure_oracle.smplify_loss already restates the term; this passes the targets through to it, for the
axis-angle pose and for the VPoser latent code (fitting.py:121-123).  The model, loss and decoder are closure_oracle's and
vposer_oracle's own functions.  Pinned against the unmodified reference by the fixtures oracle/make_golden_3d.py writes
(tests/golden/joints3d_*.npz)."""
from __future__ import annotations

import numpy as np
import torch

from . import closure_oracle as O


def closure_eval_3d(om, cfg, pri, cams_t, x86, gt_uv, conf, joint_weights, gt3d, conf3d, z=None, vposer_w=None):
    """closure_oracle.closure_eval for ONE frame plus the 3-D term: gt3d [K,3], conf3d [K].  With vposer_w the body pose is
    VPoser.decode(z, 'aa') (cfg.use_vposer must be set) and the gradient's pose slot holds d loss / d z in its first 32
    entries, zeros after them: the layout of the device closure with use_vposer = 2.  Returns dict(loss, grad[86], joints)."""
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
    total, _ = O.smplify_loss(om, cfg, pri, cams_t, verts, joints, full_pose, betas, bp, torch.tensor(gt_uv, dtype=dt),
                              torch.tensor(conf, dtype=dt), torch.tensor(joint_weights, dtype=dt), pose_embedding=emb,
                              gt3d=torch.tensor(gt3d, dtype=dt), conf3d=torch.tensor(conf3d, dtype=dt))
    grads = torch.autograd.grad(total, parts, allow_unused=True)
    g = np.zeros(86)
    o = 0
    for n, gg in zip(O.PARAM_SIZES, grads):
        if gg is not None:
            v = gg.reshape(-1).numpy()
            g[o:o + v.shape[0]] = v
        o += n
    return dict(loss=float(total), grad=g, joints=joints.detach().numpy().copy())


def closure_eval_batch_3d(om, cfg, pri, cams_t, X, gt_uv, conf, joint_weights, gt3d, conf3d, Z=None, vposer_w=None):
    """X [B,86], gt_uv [V,B,K,2], conf [V,B,K], gt3d [B,K,3], conf3d [B,K]; Z [B,32] latent codes with vposer_w"""
    outs = [closure_eval_3d(om, cfg, pri, cams_t, X[b], gt_uv[:, b], conf[:, b], joint_weights, gt3d[b], conf3d[b],
                            None if Z is None else Z[b], vposer_w) for b in range(X.shape[0])]
    return dict(loss=np.array([r["loss"] for r in outs]), grad=np.stack([r["grad"] for r in outs]),
                joints=np.stack([r["joints"] for r in outs]))
