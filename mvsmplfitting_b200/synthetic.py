"""Deterministic synthetic inputs for the multi-view SMPL fitting path.

The licensed SMPL pickle and the GMM prior pickle are not redistributable, so every
test and benchmark in this repo runs on an SMPL-*shaped* model generated here
(6890 vertices, 13776 faces, 10 betas, 207 pose blendshapes, the 24-joint SMPL
kinematic tree) and on synthetic multi-view keypoints.  The generator is pure
numpy (float64 internally, float32 outputs) and has no dependency on the CUDA
library or on the oracle; it only *produces inputs*.

Definitions follow SURVEY.md section 8(d).  The arrays mirror what the reference
reads from its `data_struct` (reference code/smplx/body_models_scale.py:169-302).
"""
from __future__ import annotations

import os

import numpy as np

NUM_VERTS = 6890
NUM_JOINTS = 24
NUM_BETAS = 10
NUM_POSE_BASIS = 207
NUM_KEYPOINTS = 17

# SMPL kinematic tree (kintree_table[0]); reference body_models_scale.py:300-302
SMPL_PARENTS = np.array(
    [-1, 0, 0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 9, 9, 12, 13, 14, 16, 17, 18, 19, 20, 21],
    dtype=np.int64)

# Extra "face" vertices appended by the vertex-joint selector, in selector order
# nose, leye, reye, lear, rear (reference smplx/vertex_ids.py:25-29,
# vertex_joint_selector.py:38-43).
FACE_VERTEX_IDS = np.array([332, 2800, 6260, 583, 4071], dtype=np.int32)

# model-joint -> keypoint maps (reference utils/utils.py:447-449 and :455-457)
JOINT_MAP_LSP14 = np.array([14, 15, 16, 17, 18, 9, 8, 10, 7, 11, 6, 3, 2, 4, 1, 5, 0],
                           dtype=np.int32)
JOINT_MAP_COCO17_SMPL = np.array([24, 25, 26, 27, 28, 16, 17, 18, 19, 20, 21, 1, 2, 4, 5, 7, 8],
                                 dtype=np.int32)

# cfg_files/fit_smpl.yaml:40-68 of the reference (the four optimisation stages)
STAGE_WEIGHTS = dict(
    data_weights=[1.0, 1.0, 1.0, 1.0],
    body_pose_prior_weights=[404.0, 404.0, 57.4, 4.78],
    shape_weights=[100.0, 50.0, 10.0, 5.0],
    coll_loss_weights=[0.0, 0.0, 1000.0, 4500.0],
    rho=100.0,
    maxiters=30,
    ftol=1e-9,
    gtol=1e-9,
)

_DATA_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "data")


def load_lsp_regressor(path: str | None = None) -> np.ndarray:
    """Dense [14, 6890] float32 LSP joint regressor.

    The reference loads it from `data/J_regressor_lsp.npz`
    (body_models_scale.py:283-286).  We ship the same 81 non-zeros as COO
    triplets (written by oracle/make_golden.py) because the matrix is data the
    path cannot run without.
    """
    if path is not None and os.path.exists(path):
        z = np.load(path)
        if "joint_regressor" in z.files:
            return np.asarray(z["joint_regressor"], dtype=np.float32)
    z = np.load(os.path.join(_DATA_DIR, "lsp_regressor_coo.npz"))
    dense = np.zeros((14, NUM_VERTS), dtype=np.float32)
    dense[z["rows"], z["cols"]] = z["vals"]
    return dense


def _fibonacci_sphere(n: int) -> np.ndarray:
    i = np.arange(n, dtype=np.float64) + 0.5
    phi = np.arccos(1.0 - 2.0 * i / n)
    theta = np.pi * (1.0 + 5.0 ** 0.5) * i
    return np.stack([np.cos(theta) * np.sin(phi), np.cos(phi), np.sin(theta) * np.sin(phi)], axis=1)


def _skeleton_rest() -> np.ndarray:
    """24 joint centres of a humanoid that fits the (0.25, 0.85, 0.15) ellipsoid."""
    c = np.zeros((24, 3))
    c[0] = (0.00, -0.10, 0.00)   # pelvis
    c[1] = (0.07, -0.18, 0.00)   # l hip
    c[2] = (-0.07, -0.18, 0.00)  # r hip
    c[3] = (0.00, 0.02, 0.00)    # spine1
    c[4] = (0.08, -0.48, 0.01)   # l knee
    c[5] = (-0.08, -0.48, 0.01)  # r knee
    c[6] = (0.00, 0.15, 0.00)    # spine2
    c[7] = (0.07, -0.74, 0.00)   # l ankle
    c[8] = (-0.07, -0.74, 0.00)  # r ankle
    c[9] = (0.00, 0.25, 0.00)    # spine3
    c[10] = (0.07, -0.79, 0.04)  # l foot
    c[11] = (-0.07, -0.79, 0.04)  # r foot
    c[12] = (0.00, 0.45, 0.00)   # neck
    c[13] = (0.05, 0.38, 0.00)   # l collar
    c[14] = (-0.05, 0.38, 0.00)  # r collar
    c[15] = (0.00, 0.60, 0.01)   # head
    c[16] = (0.13, 0.40, 0.00)   # l shoulder
    c[17] = (-0.13, 0.40, 0.00)  # r shoulder
    c[18] = (0.18, 0.20, 0.00)   # l elbow
    c[19] = (-0.18, 0.20, 0.00)  # r elbow
    c[20] = (0.20, 0.00, 0.01)   # l wrist
    c[21] = (-0.20, 0.00, 0.01)  # r wrist
    c[22] = (0.20, -0.08, 0.01)  # l hand
    c[23] = (-0.20, -0.08, 0.01)  # r hand
    return c


def make_model(seed: int = 0, with_faces: bool = True) -> dict:
    """SMPL-shaped model in the reference's `data_struct` field layout.

    Returns float32/int arrays:
      v_template [6890,3], f [13776,3] (int32), shapedirs [6890,3,10],
      posedirs [6890,3,207], J_regressor [24,6890], kintree_table [2,24] (uint32,
      root parent = 2**32-1 like the SMPL pickle), weights [6890,24],
      lsp_regressor [14,6890].
    """
    rng = np.random.RandomState(seed)
    pts = _fibonacci_sphere(NUM_VERTS)
    pts = pts + rng.normal(0.0, 2e-3, size=pts.shape)
    pts /= np.linalg.norm(pts, axis=1, keepdims=True)
    # spatially coherent vertex order (bands in height, then azimuth), like a real mesh
    band = np.floor((pts[:, 1] + 1.0) * 20.0)
    az = np.arctan2(pts[:, 2], pts[:, 0])
    order = np.lexsort((az, band))
    pts = pts[order]
    v_template = pts * np.array([0.25, 0.85, 0.15])

    faces = None
    if with_faces:
        from scipy.spatial import ConvexHull
        hull = ConvexHull(pts)
        faces = hull.simplices.astype(np.int64)
        # consistent outward orientation
        a, b, c = pts[faces[:, 0]], pts[faces[:, 1]], pts[faces[:, 2]]
        nrm = np.cross(b - a, c - a)
        flip = np.einsum("ij,ij->i", nrm, a + b + c) < 0
        faces[flip] = faces[flip][:, [0, 2, 1]]
        faces = faces[np.lexsort((faces[:, 2], faces[:, 1], faces[:, 0]))]
        assert faces.shape == (2 * NUM_VERTS - 4, 3)

    centres = _skeleton_rest()
    d2 = ((v_template[None, :, :] - centres[:, None, :]) ** 2).sum(-1)  # [24, N]

    # rest-joint regressor: peaky positive rows, top-64 support, rows sum to 1
    J_regressor = np.zeros((NUM_JOINTS, NUM_VERTS))
    for j in range(NUM_JOINTS):
        idx = np.argsort(d2[j])[:64]
        w = np.exp(-(d2[j, idx] - d2[j, idx].min()) / (2 * 0.05 ** 2)) * rng.uniform(0.5, 1.0, size=64)
        J_regressor[j, idx] = w / w.sum()

    # skinning weights: <= 4 non-zeros per vertex, like the real model
    weights = np.zeros((NUM_VERTS, NUM_JOINTS))
    near = np.argsort(d2.T, axis=1)[:, :4]  # [N,4]
    dn = np.take_along_axis(d2.T, near, axis=1)
    w = np.exp(-(dn - dn[:, :1]) / (2 * 0.06 ** 2))
    w[w < 1e-3] = 0.0
    w /= w.sum(1, keepdims=True)
    np.put_along_axis(weights, near, w, axis=1)

    shapedirs = rng.normal(0.0, 0.01, size=(NUM_VERTS, 3, NUM_BETAS))
    posedirs = rng.normal(0.0, 0.001, size=(NUM_VERTS, 3, NUM_POSE_BASIS))

    kintree = np.zeros((2, NUM_JOINTS), dtype=np.uint32)
    kintree[0] = SMPL_PARENTS.astype(np.int64) % (2 ** 32)
    kintree[1] = np.arange(NUM_JOINTS)

    return dict(
        v_template=v_template.astype(np.float32),
        f=None if faces is None else faces.astype(np.int32),
        shapedirs=shapedirs.astype(np.float32),
        posedirs=posedirs.astype(np.float32),
        J_regressor=J_regressor.astype(np.float32),
        kintree_table=kintree,
        weights=weights.astype(np.float32),
        lsp_regressor=load_lsp_regressor(),
    )


def make_gmm(seed: int = 7, num_gaussians: int = 6, dim: int = 69) -> dict:
    """Synthetic GMM pose prior in the dict format the reference accepts
    (prior.py:130-133): means [M,69], covars [M,69,69] SPD, weights [M]."""
    rng = np.random.RandomState(seed)
    means = rng.normal(0.0, 0.15, size=(num_gaussians, dim))
    covars = np.zeros((num_gaussians, dim, dim))
    for m in range(num_gaussians):
        a = rng.normal(0.0, 1.0, size=(dim, dim)) * 0.05
        covars[m] = a @ a.T + np.diag(rng.uniform(0.02, 0.08, size=dim))
    w = rng.uniform(0.5, 1.5, size=num_gaussians)
    return dict(means=means, covars=covars, weights=w / w.sum())


def make_vposer(seed: int = 11, num_neurons: int = 512, latent: int = 32, num_joints: int = 23) -> dict:
    """Synthetic VPoser DECODER weights with the shapes of the reference's module (model/VPoser.py:190-197:
    bodyprior_dec_fc1 [512,32], bodyprior_dec_fc2 [512,512], bodyprior_dec_out [138,512]).  The trained snapshot the
    reference ships is its data, not ours; a seeded network of the same architecture exercises the same arithmetic."""
    rng = np.random.RandomState(seed)
    lin = lambda o, i, gain: (rng.normal(0.0, gain / np.sqrt(i), size=(o, i)).astype(np.float32),
                              rng.normal(0.0, 0.05, size=o).astype(np.float32))
    w1, b1 = lin(num_neurons, latent, 1.2)
    w2, b2 = lin(num_neurons, num_neurons, 1.3)
    w3, b3 = lin(num_joints * 6, num_neurons, 1.0)
    # bias the 6-D heads towards (1,0,0 | 0,1,0) so that decoded poses stay moderate rotations, as a trained prior's do
    b3 = b3.reshape(num_joints, 3, 2)
    b3[:, 0, 0] += 1.0
    b3[:, 1, 1] += 1.0
    return dict(fc1_w=w1, fc1_b=b1, fc2_w=w2, fc2_b=b2, out_w=w3, out_b=b3.reshape(-1).astype(np.float32))


def gmm_buffers(gmm: dict):
    """(means[M,69], precisions[M,69,69], nll_weights[M]) as float64, following
    reference prior.py:142-160 (precision = inv(cov); nll_weights = w / ((2pi)^34.5 *
    sqrt(det)/min sqrt(det)))."""
    means = np.asarray(gmm["means"], dtype=np.float64)
    covs = np.asarray(gmm["covars"], dtype=np.float64)
    weights = np.asarray(gmm["weights"], dtype=np.float64)
    precisions = np.stack([np.linalg.inv(c) for c in covs])
    sqrdets = np.array([np.sqrt(np.linalg.det(c)) for c in covs])
    const = (2 * np.pi) ** (69 / 2.0)
    nll_weights = weights / (const * (sqrdets / sqrdets.min()))
    return means, precisions, nll_weights


def make_cameras(num_views: int, radius: float = 20.0, focal: float = 2400.0,
                 center=(1024.0, 768.0), height: float = 0.5) -> dict:
    """Ring of calibrated cameras looking at the origin (world->camera R, t).
    Image y points down (camera y = -world up), x_cam.z > 0 in front."""
    R = np.zeros((num_views, 3, 3))
    t = np.zeros((num_views, 3))
    for v in range(num_views):
        ang = 2 * np.pi * (v + 0.25) / num_views
        pos = np.array([radius * np.cos(ang), height + 0.3 * np.sin(3 * ang), radius * np.sin(ang)])
        zc = -pos / np.linalg.norm(pos)
        up = np.array([0.0, 1.0, 0.0])
        xc = np.cross(zc, up)  # image x to the right
        xc /= np.linalg.norm(xc)
        yc = np.cross(zc, xc)  # image y down
        R[v] = np.stack([xc, yc, zc])
        t[v] = -R[v] @ pos
    return dict(
        R=R.astype(np.float32), t=t.astype(np.float32),
        f=np.full((num_views, 2), focal, dtype=np.float32),
        c=np.tile(np.asarray(center, dtype=np.float32), (num_views, 1)),
        H=1536, W=2048)


def rodrigues_np(r: np.ndarray) -> np.ndarray:
    """[...,3] -> [...,3,3]; same expression as reference lbs.py:284-299."""
    a = np.linalg.norm(r + 1e-8, axis=-1, keepdims=True)
    k = r / a
    K = np.zeros(r.shape[:-1] + (3, 3))
    K[..., 0, 1], K[..., 0, 2] = -k[..., 2], k[..., 1]
    K[..., 1, 0], K[..., 1, 2] = k[..., 2], -k[..., 0]
    K[..., 2, 0], K[..., 2, 1] = -k[..., 1], k[..., 0]
    s, c = np.sin(a)[..., None], np.cos(a)[..., None]
    return np.eye(3) + s * K + (1 - c) * (K @ K)


def model_keypoints_np(model: dict, betas, global_orient, body_pose, transl, scale,
                       model_type: str = "smpllsp"):
    """float64 forward used ONLY to synthesise ground-truth keypoints for the
    generator (not a product path, not the oracle).  Returns joints [B,17,3]."""
    vt = model["v_template"].astype(np.float64)
    S = model["shapedirs"].astype(np.float64)
    P = model["posedirs"].astype(np.float64).reshape(-1, NUM_POSE_BASIS)  # [3N,207]
    Jr = model["J_regressor"].astype(np.float64)
    W = model["weights"].astype(np.float64)
    L = model["lsp_regressor"].astype(np.float64)
    B = betas.shape[0]
    out = np.zeros((B, NUM_KEYPOINTS, 3))
    for b in range(B):
        v_s = vt + S @ betas[b]
        J = Jr @ v_s
        pose = np.concatenate([global_orient[b], body_pose[b]]).reshape(24, 3)
        Rm = rodrigues_np(pose)
        pf = (Rm[1:] - np.eye(3)).reshape(-1)
        v_p = v_s + (P @ pf).reshape(-1, 3)
        G = np.zeros((24, 4, 4))
        for j in range(24):
            M = np.eye(4)
            M[:3, :3] = Rm[j]
            if j == 0:
                M[:3, :3] *= scale[b]
                M[:3, 3] = J[0]
                G[0] = M
            else:
                M[:3, 3] = J[j] - J[SMPL_PARENTS[j]]
                G[j] = G[SMPL_PARENTS[j]] @ M
        A = G.copy()
        A[:, :3, 3] -= np.einsum("jab,jb->ja", G[:, :3, :3], J)
        T = np.einsum("nj,jab->nab", W, A)
        v = np.einsum("nab,nb->na", T[:, :3, :3], v_p) + T[:, :3, 3]
        if model_type == "smpllsp":
            q = np.concatenate([L @ v, v[FACE_VERTEX_IDS]])[JOINT_MAP_LSP14]
        else:
            q = np.concatenate([G[:, :3, 3], v[FACE_VERTEX_IDS]])[JOINT_MAP_COCO17_SMPL]
        out[b] = q + transl[b]
    return out


def project_np(cams: dict, joints: np.ndarray) -> np.ndarray:
    """[B,K,3] -> [V,B,K,2] (reference camera.py:102-116); with cams["dist"] [V,5] through each view's lens distortion
    (OpenCV's k1, k2, p1, p2, k3, as mvs_set_camera_rigs_dist)."""
    x = np.einsum("vab,nkb->vnka", cams["R"].astype(np.float64), joints) + \
        cams["t"].astype(np.float64)[:, None, None, :]
    uv = x[..., :2] / x[..., 2:3]
    if cams.get("dist") is not None:
        d = np.asarray(cams["dist"], np.float64)[:, None, None, :]
        k1, k2, p1, p2, k3 = (d[..., i] for i in range(5))
        xn, yn = uv[..., 0], uv[..., 1]
        r2 = xn * xn + yn * yn
        a = 1 + k1 * r2 + k2 * r2 * r2 + k3 * r2 * r2 * r2
        uv = np.stack([xn * a + 2 * p1 * xn * yn + p2 * (r2 + 2 * xn * xn),
                       yn * a + p1 * (r2 + 2 * yn * yn) + 2 * p2 * xn * yn], -1)
    return uv * cams["f"].astype(np.float64)[:, None, None, :] + \
        cams["c"].astype(np.float64)[:, None, None, :]


WIDE_OFFSET = (0.6, 0.0, 0.3)            # where make_frames_wide puts the bodies: off the wide rig's common optical centre


def make_wide_cameras(num_views: int, radius: float = 2.5, focal: float = 1000.0, distorted: bool = True) -> dict:
    """A wide-angle test rig: make_cameras' ring, close (radius 2.5 m) and short (f = 1000 px on a 2048 x 1536 image), so that
    a body make_frames_wide places off-centre reaches normalised image radius >= 0.4, where lens distortion moves detections by
    tens of pixels.  distorted: "dist" [V,5] (float32) holds each view's coefficients, mid-range barrel lenses
    (k1 -0.18 .. -0.26) with small tangential terms."""
    cams = make_cameras(num_views, radius=radius, focal=focal)
    if distorted:
        v = np.arange(num_views)
        cams["dist"] = np.ascontiguousarray(np.stack([-0.18 - 0.08 * (v % 3) / 2, 0.04 + 0.02 * (v % 2), 6e-4 * np.cos(v),
                                                      -4e-4 * np.sin(v), -0.004 * (v % 2)], 1), dtype=np.float32)
    return cams


def make_frames_wide(model: dict, cams: dict, num_frames: int, seed: int = 1, noise: float = 2.0,
                     model_type: str = "smpllsp") -> dict:
    """make_frames for make_wide_cameras: bodies off-centre by WIDE_OFFSET, detections projected through cams (with its "dist",
    if any) plus `noise` px of Gaussian noise.  Same keys as make_frames."""
    rng = np.random.RandomState(seed)
    B = num_frames
    body_pose = rng.normal(0, 0.15, size=(B, 69))
    global_orient = rng.normal(0, 0.2, size=(B, 3))
    transl = np.asarray(WIDE_OFFSET)[None, :] + rng.normal(0, 0.1, size=(B, 3))
    betas = rng.normal(0, 1.0, size=(B, 10))
    scale = np.ones((B, 1))
    joints = model_keypoints_np(model, betas, global_orient, body_pose, transl, scale, model_type)
    V = cams["R"].shape[0]
    gt_uv = project_np(cams, joints) + rng.normal(0, noise, size=(V, B, NUM_KEYPOINTS, 2))
    conf = rng.uniform(0.6, 0.95, size=(V, B, NUM_KEYPOINTS))
    init = dict(betas=np.zeros((B, 10)), global_orient=0.5 * global_orient, body_pose=0.5 * body_pose,
                transl=transl + rng.normal(0, 0.05, size=(B, 3)), scale=np.ones((B, 1)))
    f32 = lambda d: {k: np.ascontiguousarray(v, dtype=np.float32) for k, v in d.items()}
    return dict(gt=f32(dict(betas=betas, global_orient=global_orient, body_pose=body_pose, transl=transl, scale=scale)),
                init=f32(init), gt_uv=gt_uv.astype(np.float32), conf=conf.astype(np.float32),
                joint_weights=np.ones(NUM_KEYPOINTS, dtype=np.float32), gt_joints3d=joints.astype(np.float32))


def make_frames(model: dict, cams: dict, num_frames: int, seed: int = 1,
                smooth_walk: bool = False, model_type: str = "smpllsp") -> dict:
    """Ground-truth parameters, noisy multi-view keypoints and the initial guess
    for `num_frames` independent frames (SURVEY.md section 8d "Frames")."""
    rng = np.random.RandomState(seed)
    B = num_frames
    if smooth_walk:
        body_pose = np.cumsum(rng.normal(0, 0.02, size=(B, 69)), axis=0) + rng.normal(0, 0.2, size=(1, 69))
        global_orient = np.cumsum(rng.normal(0, 0.02, size=(B, 3)), axis=0) + rng.normal(0, 0.3, size=(1, 3))
        transl = np.cumsum(rng.normal(0, 0.02, size=(B, 3)), axis=0) + rng.normal(0, 0.5, size=(1, 3))
        betas = np.tile(rng.normal(0, 1.0, size=(1, 10)), (B, 1))
    else:
        body_pose = rng.normal(0, 0.2, size=(B, 69))
        global_orient = rng.normal(0, 0.3, size=(B, 3))
        transl = rng.normal(0, 0.5, size=(B, 3))
        betas = rng.normal(0, 1.0, size=(B, 10))
    scale = np.ones((B, 1))
    joints = model_keypoints_np(model, betas, global_orient, body_pose, transl, scale, model_type)
    V = cams["R"].shape[0]
    gt_uv = project_np(cams, joints) + rng.normal(0, 5.0, size=(V, B, NUM_KEYPOINTS, 2))
    conf = rng.uniform(0.6, 0.95, size=(V, B, NUM_KEYPOINTS))
    init = dict(
        betas=np.zeros((B, 10)),
        global_orient=0.5 * global_orient,
        body_pose=0.5 * body_pose,
        transl=transl + rng.normal(0, 0.05, size=(B, 3)),
        scale=np.ones((B, 1)),
    )
    f32 = lambda d: {k: np.ascontiguousarray(v, dtype=np.float32) for k, v in d.items()}
    return dict(
        gt=f32(dict(betas=betas, global_orient=global_orient, body_pose=body_pose,
                    transl=transl, scale=scale)),
        init=f32(init),
        gt_uv=gt_uv.astype(np.float32),
        conf=conf.astype(np.float32),
        joint_weights=np.ones(NUM_KEYPOINTS, dtype=np.float32),
        gt_joints3d=joints.astype(np.float32),
    )


PARAM_ORDER = ("betas", "global_orient", "body_pose", "transl", "scale")
PARAM_SIZES = (10, 3, 69, 3, 1)
NUM_PARAMS = 86


def pack_params(p: dict) -> np.ndarray:
    """dict of [B,*] -> [B,86] in the reference's L-BFGS flat order
    (registration order body_models_scale.py:213,232,244,255,266)."""
    return np.ascontiguousarray(
        np.concatenate([np.asarray(p[k], dtype=np.float32).reshape(len(p["betas"]), -1)
                        for k in PARAM_ORDER], axis=1))


def unpack_params(x: np.ndarray) -> dict:
    out, o = {}, 0
    for k, n in zip(PARAM_ORDER, PARAM_SIZES):
        out[k] = x[:, o:o + n]
        o += n
    return out
