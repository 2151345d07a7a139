"""TEST INFRASTRUCTURE -- CPU restatement (PyTorch autograd, fp32 or fp64) of the
reference's per-frame fitting closure.  It is the parity oracle for the CUDA path
and the `cpu_baseline` "port" leg of bench.py; it is NOT a product path and is
never imported by `mvsmplfitting_b200`.

Pinned against the unmodified reference by tests/test_oracle_vs_reference.py
(when /root/reference is present) and by the committed fixtures under
tests/golden/ written by oracle/make_golden.py from the reference itself.

Every function cites the reference lines it restates (paths relative to the
reference root).  The reference is batch-size-1 only (non_linear_solver.py:56);
this restatement evaluates one frame per call and callers loop over frames.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import numpy as np
import torch

FACE_IDS = (332, 2800, 6260, 583, 4071)          # smplx/vertex_ids.py:25-29 in selector order
MAP_LSP14 = (14, 15, 16, 17, 18, 9, 8, 10, 7, 11, 6, 3, 2, 4, 1, 5, 0)      # utils/utils.py:455-457
MAP_COCO17 = (24, 25, 26, 27, 28, 16, 17, 18, 19, 20, 21, 1, 2, 4, 5, 7, 8)  # utils/utils.py:447-449
ANGLE_IDX = (52, 55, 9, 12)                       # prior.py:62,87 (55,58,12,15 minus 3)
ANGLE_SIGN = (1.0, -1.0, -1.0, -1.0)              # prior.py:66


@dataclass
class OracleModel:
    """Model constants as the reference registers them (body_models_scale.py:270-305)."""
    v_template: torch.Tensor      # [N,3]
    shapedirs: torch.Tensor       # [N,3,10]
    posedirs: torch.Tensor        # [207, 3N]   (reshape(-1,207).T, body_models_scale.py:293-297)
    J_regressor: torch.Tensor     # [24,N]
    parents: list
    lbs_weights: torch.Tensor     # [N,24]
    lsp_regressor: torch.Tensor   # [14,N]
    faces: torch.Tensor | None
    model_type: str = "smpllsp"
    dtype: torch.dtype = torch.float32
    joint_map: tuple | None = None          # keypoint k = source joint_map[k]; None: MAP_LSP14 / MAP_COCO17 by model_type
    extra_vertex_ids: tuple | None = None   # vertices appended to the source joints; None: FACE_IDS

    @staticmethod
    def from_numpy(model: dict, dtype=torch.float32, model_type="smpllsp", joint_map=None,
                   extra_vertex_ids=None) -> "OracleModel":
        t = lambda a: torch.tensor(np.asarray(a, dtype=np.float64), dtype=dtype)
        pd = np.reshape(np.asarray(model["posedirs"]), [-1, model["posedirs"].shape[-1]]).T
        parents = [int(x) for x in np.asarray(model["kintree_table"][0]).astype(np.int64)]
        parents[0] = -1
        return OracleModel(
            v_template=t(model["v_template"]), shapedirs=t(model["shapedirs"]), posedirs=t(pd),
            J_regressor=t(model["J_regressor"]), parents=parents, lbs_weights=t(model["weights"]),
            lsp_regressor=t(model["lsp_regressor"]),
            faces=None if model.get("f") is None else torch.tensor(np.asarray(model["f"], dtype=np.int64)),
            model_type=model_type, dtype=dtype,
            joint_map=None if joint_map is None else tuple(int(j) for j in joint_map),
            extra_vertex_ids=None if extra_vertex_ids is None else tuple(int(v) for v in extra_vertex_ids))


def rodrigues(rot_vecs: torch.Tensor) -> torch.Tensor:
    """lbs.py:269-300.  Note the 1e-8 is added to every component before the norm
    and the direction is r / angle without epsilon."""
    n = rot_vecs.shape[0]
    angle = torch.norm(rot_vecs + 1e-8, dim=1, keepdim=True)
    axis = rot_vecs / angle
    c = torch.cos(angle).unsqueeze(1)
    s = torch.sin(angle).unsqueeze(1)
    x, y, z = axis[:, 0:1], axis[:, 1:2], axis[:, 2:3]
    o = torch.zeros((n, 1), dtype=rot_vecs.dtype)
    K = torch.cat([o, -z, y, z, o, -x, -y, x, o], dim=1).view(n, 3, 3)
    eye = torch.eye(3, dtype=rot_vecs.dtype).unsqueeze(0)
    return eye + s * K + (1 - c) * torch.bmm(K, K)


def _hom(R, t):
    """lbs.py:303-313: [R t; 0 1]."""
    top = torch.cat([R, t], dim=2)
    bot = torch.zeros((R.shape[0], 1, 4), dtype=R.dtype)
    bot[:, 0, 3] = 1
    return torch.cat([top, bot], dim=1)


def rigid_chain(rot_mats, joints, parents, scale):
    """lbs.py:316-370 for one frame: rot_mats [24,3,3], joints [24,3], scale [1,1].
    Root 3x3 block is multiplied by `scale` before chaining (lbs.py:348)."""
    nj = joints.shape[0]
    rel = joints.clone()
    rel[1:] = joints[1:] - joints[parents[1:]]
    mats = _hom(rot_mats, rel.unsqueeze(-1))                      # [24,4,4]
    root = torch.cat([torch.cat([mats[0][:3, :3] * scale.reshape(()), mats[0][:3, 3:4]], dim=1),
                      mats[0][3:4]], dim=0)
    chain = [root]
    for i in range(1, nj):
        chain.append(torch.matmul(chain[parents[i]], mats[i]))
    G = torch.stack(chain, dim=0)
    posed = G[:, :3, 3]
    jh = torch.cat([joints, torch.zeros((nj, 1), dtype=joints.dtype)], dim=1).unsqueeze(-1)
    corr = torch.matmul(G, jh)                                     # [24,4,1]
    A = G - torch.cat([torch.zeros((nj, 4, 3), dtype=joints.dtype), corr], dim=2)
    return posed, A


def smpl_forward(om: OracleModel, betas, global_orient, body_pose, transl, scale):
    """body_models_scale.py:327-412 + lbs.py:135-222 for ONE frame.
    Inputs are [1,10],[1,3],[1,69],[1,3],[1,1].  Returns vertices [N,3] (with transl),
    keypoints [K,3] (K = 17 for the default keypoint maps), full_pose [1,72]."""
    full_pose = torch.cat([global_orient, body_pose], dim=1)
    v_shaped = om.v_template + torch.einsum("bl,mkl->bmk", betas, om.shapedirs)[0]   # lbs.py:179,265
    J = torch.einsum("ik,ji->jk", v_shaped, om.J_regressor)                           # lbs.py:183,242
    R = rodrigues(full_pose.view(-1, 3))                                              # lbs.py:189
    feat = (R[1:] - torch.eye(3, dtype=R.dtype)).reshape(1, -1)                       # lbs.py:192
    v_posed = v_shaped + torch.matmul(feat, om.posedirs).view(-1, 3)                  # lbs.py:194-203
    posed_joints, A = rigid_chain(R, J, om.parents, scale)                            # lbs.py:205
    T = torch.matmul(om.lbs_weights, A.view(-1, 16)).view(-1, 4, 4)                   # lbs.py:209-213
    vh = torch.cat([v_posed, torch.ones((v_posed.shape[0], 1), dtype=R.dtype)], dim=1)
    verts = torch.matmul(T, vh.unsqueeze(-1))[:, :3, 0]                               # lbs.py:215-220
    if om.model_type == "smpllsp":
        joints = torch.matmul(om.lsp_regressor, verts)                                # body_models_scale.py:393-394
        jmap = MAP_LSP14
    else:
        joints = posed_joints
        jmap = MAP_COCO17
    if om.joint_map is not None:
        jmap = om.joint_map
    extra = FACE_IDS if om.extra_vertex_ids is None else om.extra_vertex_ids
    joints = torch.cat([joints, verts[list(extra)]], dim=0)                           # vertex_joint_selector.py:73-77
    joints = joints[list(jmap)]                                                       # utils/utils.py:420-424
    joints = joints + transl                                                          # body_models_scale.py:401-403
    verts = verts + transl
    return verts, joints, full_pose


def project(cam_R, cam_t, cam_f, cam_c, pts):
    """camera.py:93-117 for one camera; pts [K,3] -> [K,2]."""
    x = torch.einsum("ki,ji->jk", cam_R, pts) + cam_t
    uv = x[:, :2] / x[:, 2:3]
    return uv * cam_f + cam_c


def gmof(res, rho):
    """utils/utils.py:427-438."""
    sq = res ** 2
    return rho ** 2 * (sq / (sq + rho ** 2))


@dataclass
class OraclePriors:
    kind: str = "l2"                      # 'l2' | 'gmm'
    means: torch.Tensor | None = None     # [M,69]
    precisions: torch.Tensor | None = None  # [M,69,69]
    nll_weights: torch.Tensor | None = None  # [1,M]

    @staticmethod
    def gmm_from_dict(gmm: dict, dtype=torch.float32) -> "OraclePriors":
        """prior.py:127-160 (same numpy dtype path: float32 casts then float64 dets)."""
        np_dtype = np.float32 if dtype == torch.float32 else np.float64
        means = gmm["means"].astype(np_dtype)
        covs = gmm["covars"].astype(np_dtype)
        precisions = np.stack([np.linalg.inv(c) for c in covs]).astype(np_dtype)
        sqrdets = np.array([np.sqrt(np.linalg.det(c)) for c in gmm["covars"]])
        const = (2 * np.pi) ** (69 / 2.0)
        nllw = np.asarray(gmm["weights"] / (const * (sqrdets / sqrdets.min())))
        return OraclePriors("gmm", torch.tensor(means, dtype=dtype), torch.tensor(precisions, dtype=dtype),
                            torch.tensor(nllw, dtype=dtype).unsqueeze(0))


def gmm_min_nll(pr: OraclePriors, pose):
    """prior.py:181-196 (merged, min over components)."""
    diff = pose.unsqueeze(1) - pr.means
    pd = torch.einsum("mij,bmj->bmi", pr.precisions, diff)
    quad = (pd * diff).sum(-1)
    ll = 0.5 * quad - torch.log(pr.nll_weights)
    return torch.min(ll, dim=1)[0]


@dataclass
class LossConfig:
    """Stage weights + flags (fitting.py:208-280, non_linear_solver.py:150,177-180)."""
    data_weight: float = 1.0
    body_pose_weight: float = 0.0
    shape_weight: float = 0.0
    bending_prior_weight: float = 0.0
    coll_loss_weight: float = 0.0
    rho: float = 100.0
    use_joints_conf: bool = True
    use_vposer: bool = False
    fix_shape: bool = False
    interpenetration: bool = False
    use_3d: bool = False
    sdf_grid: int = 128
    sdf_all_faces: bool = False        # False = as written (triangle 0 only, SURVEY A12)


def smplify_loss(om, cfg: LossConfig, pri: OraclePriors, cams: dict, verts, joints, full_pose,
                 betas, body_pose, gt_uv, conf, joint_weights, pose_embedding=None,
                 gt3d=None, conf3d=None, return_terms=False):
    """fitting.py:290-415 for one frame.  gt_uv [V,17,2], conf [V,17], joint_weights [17]."""
    dt = joints.dtype
    V = gt_uv.shape[0]
    dw = torch.tensor(cfg.data_weight, dtype=dt)
    bpw = torch.tensor(cfg.body_pose_weight, dtype=dt)
    sw = torch.tensor(cfg.shape_weight, dtype=dt)
    bend = torch.tensor(cfg.bending_prior_weight, dtype=dt)
    projs = []
    joint_loss = 0.0
    for v in range(V):
        uv = project(cams["R"][v], cams["t"][v], cams["f"][v], cams["c"][v], joints)
        projs.append(uv)
        w = (joint_weights * conf[v] if cfg.use_joints_conf else joint_weights).unsqueeze(-1)
        joint_loss = joint_loss + torch.sum(w ** 2 * gmof(gt_uv[v] - uv, cfg.rho)) * dw ** 2
    loss3d = 0.0
    if cfg.use_3d:
        loss3d = torch.sum(conf3d.unsqueeze(-1) ** 2 * gmof(gt3d - joints, cfg.rho)) * dw ** 2
    if cfg.use_vposer:
        pprior = pose_embedding.pow(2).sum() * bpw ** 2
    else:
        if pri.kind == "gmm":
            pprior = torch.sum(gmm_min_nll(pri, body_pose)) * bpw ** 2
        else:
            pprior = torch.sum(body_pose.pow(2)) * bpw ** 2                # prior.py:92-97
        if float(pprior) > 5e4:                                           # fitting.py:334-335
            pprior = 0.0
        pprior = pprior + body_pose.pow(2).sum() * (bpw * 4) ** 2          # fitting.py:336-337
    shape_loss = 0.0
    if not cfg.fix_shape:
        shape_loss = torch.sum(betas.pow(2)) * sw ** 2                    # fitting.py:339-342
    bp = full_pose[:, 3:66]
    sign = torch.tensor(ANGLE_SIGN, dtype=dt)
    angle = torch.sum(torch.exp(bp[:, list(ANGLE_IDX)] * sign).pow(2)) * bend   # prior.py:87-89
    if float(angle) > 1e4 and not cfg.use_vposer:                         # fitting.py:349-350
        angle = 0.0
    pen = 0.0
    if cfg.interpenetration and cfg.coll_loss_weight > 0:
        from . import sdf_oracle
        pen = sdf_oracle.penetration_loss(verts, om.faces, cfg.coll_loss_weight, cfg.sdf_grid,
                                          all_faces=cfg.sdf_all_faces)
    total = joint_loss + loss3d + pprior + shape_loss + angle + pen
    if return_terms:
        f = lambda t: float(t) if not isinstance(t, float) else t
        return total, torch.stack(projs), dict(data=f(joint_loss), pprior=f(pprior), shape=f(shape_loss),
                                               angle=f(angle), pen=f(pen))
    return total, torch.stack(projs)


PARAM_ORDER = ("betas", "global_orient", "body_pose", "transl", "scale")
PARAM_SIZES = (10, 3, 69, 3, 1)


def cams_to_torch(cams: dict, dtype):
    return {k: torch.tensor(np.asarray(cams[k], dtype=np.float64), dtype=dtype) for k in ("R", "t", "f", "c")}


def closure_eval(om: OracleModel, cfg: LossConfig, pri: OraclePriors, cams_t: dict,
                 x86: np.ndarray, gt_uv: np.ndarray, conf: np.ndarray, joint_weights: np.ndarray,
                 backward: bool = True, want_verts: bool = False):
    """One fitting_func() (fitting.py:162-203) for ONE frame given the flat 86-vector
    [betas|global_orient|body_pose|transl|scale].  Returns dict(loss, grad[86], joints, proj)."""
    dt = om.dtype
    x = torch.tensor(np.asarray(x86, dtype=np.float64), dtype=dt)
    parts, o = [], 0
    for n in PARAM_SIZES:
        parts.append(x[o:o + n].clone().view(1, n).requires_grad_(True))
        o += n
    betas, go, bp, tr, sc = parts
    verts, joints, full_pose = smpl_forward(om, betas, go, bp, tr, sc)
    total, proj = smplify_loss(
        om, cfg, pri, cams_t, verts, joints, full_pose, betas, bp,
        torch.tensor(gt_uv, dtype=dt), torch.tensor(conf, dtype=dt), torch.tensor(joint_weights, dtype=dt))
    out = dict(loss=float(total), joints=joints.detach().numpy().copy(), proj=proj.detach().numpy().copy())
    if want_verts:
        out["verts"] = verts.detach().numpy().copy()
    if backward:
        grads = torch.autograd.grad(total, parts, allow_unused=True)
        out["grad"] = np.concatenate([
            (g if g is not None else torch.zeros_like(p)).reshape(-1).numpy() for g, p in zip(grads, parts)])
    return out


def closure_eval_batch(om, cfg, pri, cams_t, X, gt_uv, conf, joint_weights, backward=True, want_verts=False):
    """Loop of closure_eval over frames: X [B,86], gt_uv [V,B,17,2], conf [V,B,17]."""
    outs = [closure_eval(om, cfg, pri, cams_t, X[b], gt_uv[:, b], conf[:, b], joint_weights,
                         backward=backward, want_verts=want_verts) for b in range(X.shape[0])]
    res = {k: np.stack([o[k] for o in outs]) for k in outs[0] if k != "loss"}
    res["loss"] = np.array([o["loss"] for o in outs])
    if "proj" in res:
        res["proj"] = np.ascontiguousarray(np.transpose(res["proj"], (1, 0, 2, 3)))   # [V,B,17,2]
    return res


def closure_eval_vposer(om: OracleModel, cfg: LossConfig, pri: OraclePriors, cams_t: dict, x86: np.ndarray, z: np.ndarray,
                        vposer_w: dict, gt_uv: np.ndarray, conf: np.ndarray, joint_weights: np.ndarray, body_pose=None):
    """fitting_func() with use_vposer=True for ONE frame (fitting.py:162-203): body_pose = VPoser.decode(z, 'aa');
    the 69 pose entries of x86 are ignored.  Returns dict(loss, grad_* for betas / global_orient / transl / scale /
    pose_embedding / body_pose (the decoded pose), joints, proj [V,K,2], body_pose, terms (per-term values of
    smplify_loss)).

    The decoder runs in om.dtype: float32 weights (what a device context uploads) are widened exactly to float64.
    body_pose [69]: evaluate at this pose instead of decode(z) -- the caller decoded it (use_vposer = 1, the drop-in
    mode); z then only enters the |z|^2 prior, and g_pose_embedding is that prior's gradient alone."""
    from . import vposer_oracle as VO
    dt = om.dtype
    x = torch.tensor(np.asarray(x86, dtype=np.float64), dtype=dt)
    betas = x[0:10].clone().view(1, 10).requires_grad_(True)
    go = x[10:13].clone().view(1, 3).requires_grad_(True)
    tr = x[82:85].clone().view(1, 3).requires_grad_(True)
    sc = x[85:86].clone().view(1, 1).requires_grad_(True)
    emb = torch.tensor(np.asarray(z, dtype=np.float64), dtype=dt).view(1, 32).requires_grad_(True)
    if body_pose is None:
        bp = VO.decode_aa(vposer_w, emb)
    else:
        bp = torch.tensor(np.asarray(body_pose, dtype=np.float64), dtype=dt).view(1, 69).requires_grad_(True)
    verts, joints, full_pose = smpl_forward(om, betas, go, bp, tr, sc)
    total, proj, terms = smplify_loss(om, cfg, pri, cams_t, verts, joints, full_pose, betas, bp,
                                      torch.tensor(gt_uv, dtype=dt), torch.tensor(conf, dtype=dt),
                                      torch.tensor(joint_weights, dtype=dt), pose_embedding=emb, return_terms=True)
    g = torch.autograd.grad(total, [betas, go, tr, sc, emb, bp])
    names = ("betas", "global_orient", "transl", "scale", "pose_embedding", "body_pose")
    out = dict(loss=float(total), joints=joints.detach().numpy().copy(), body_pose=bp.detach().numpy()[0].copy(),
               proj=proj.detach().numpy().copy(), terms=terms)
    for n, gg in zip(names, g):
        out["g_" + n] = gg.reshape(-1).numpy().copy()
    return out
