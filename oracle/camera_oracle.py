"""Float64 restatement of mvs_refine_cameras' camera step (PyTorch autograd): the camera map from a view's update, view 1's
sphere basis, and each view problem's loss -- the 2-D data term of one view over the frames of its rig at held keypoints.

The map (DESIGN.md section 4):  R = Rod(w) R0,  t = Rod(w) (t0 - R0 dC),  Rod(w) = I + A K + B K^2 (K = [w]x, A = sin th / th,
B = (1 - cos th) / th^2), dC = c for a free view and dC = (E u - n (s - 1)) / s, s = sqrt(1 + |u|^2), for view 1."""
import numpy as np
import torch

ROT = slice(10, 13)                    # the problem's variables in its 86-entry row
CEN = slice(82, 85)


def rod(w: torch.Tensor) -> torch.Tensor:
    th2 = (w * w).sum()
    K = torch.zeros(3, 3, dtype=w.dtype)
    K[0, 1], K[0, 2], K[1, 0], K[1, 2], K[2, 0], K[2, 1] = -w[2], w[1], w[2], -w[0], -w[1], w[0]
    if float(th2.detach()) < 0.1:      # series (exact derivatives at 0)
        A = 1 - th2 / 6 + th2 ** 2 / 120 - th2 ** 3 / 5040 + th2 ** 4 / 362880
        B = 0.5 - th2 / 24 + th2 ** 2 / 720 - th2 ** 3 / 40320 + th2 ** 4 / 3628800
    else:
        th = torch.sqrt(th2)
        A, B = torch.sin(th) / th, (1 - torch.cos(th)) / th2
    return torch.eye(3, dtype=w.dtype) + A * K + B * (K @ K)


def delta_centre(c: torch.Tensor, sphere: bool, E=None, n=None) -> torch.Tensor:
    if not sphere:
        return c
    E, n = torch.as_tensor(np.asarray(E, np.float64).reshape(3, 2)), torch.as_tensor(np.asarray(n, np.float64))
    u = c[:2]
    s = torch.sqrt(1 + (u * u).sum())
    return (E @ u - n * (s - 1)) / s


def cam_from_delta(R0, t0, w, c, sphere=False, E=None, n=None):
    """(R [3,3], t [3]) float64 tensors; R0, t0 numpy (float32 values), w [3], c [3] float64 tensors"""
    R0, t0 = torch.as_tensor(np.asarray(R0, np.float64)), torch.as_tensor(np.asarray(t0, np.float64))
    Q = rod(w)
    dC = delta_centre(c, sphere, E, n)
    return Q @ R0, Q @ (t0 - R0 @ dC)


def centre(R, t):
    return -np.asarray(R, np.float64).T @ np.asarray(t, np.float64)


def sphere_basis(R_0, t_0, R_1, t_1):
    """(E [3,2], n [3]) float32 as the driver builds them for view 1 from views 0 and 1 of the table"""
    d = centre(R_1, t_1) - centre(R_0, t_0)
    r = np.sqrt((d * d).sum())
    if not r > 0:
        return np.zeros((3, 2), np.float32), np.zeros(3, np.float32)
    d = d / r
    k = 0 if abs(d[0]) <= abs(d[1]) and abs(d[0]) <= abs(d[2]) else 1 if abs(d[1]) <= abs(d[2]) else 2
    a = np.zeros(3)
    a[k] = 1.0
    e1 = np.cross(d, a)
    e1 = e1 / np.sqrt((e1 * e1).sum())
    e2 = np.cross(d, e1)
    return np.stack([r * e1, r * e2], 1).astype(np.float32), (r * d).astype(np.float32)


def gmof(e, rho2):
    return rho2 * (e * e) / (e * e + rho2)


def view_term(R, t, f, c, q, gt_uv, conf, jw, dw, rho, use_conf):
    """sum over frames of resident_closure P6's term of one view: q [F,K,3], gt_uv [F,K,2], conf [F,K] (float64 tensors)"""
    x = q @ R.T + t
    uv = x[..., :2] / x[..., 2:3] * torch.as_tensor(np.asarray(f, np.float64)) + torch.as_tensor(np.asarray(c, np.float64))
    w = torch.as_tensor(np.asarray(jw, np.float64))[None, :] * (conf if use_conf else 1.0)
    w2 = w * w
    rho2 = float(rho) ** 2
    e = gt_uv - uv
    return ((w2 * gmof(e[..., 0], rho2) + w2 * gmof(e[..., 1], rho2)).sum(1) * float(dw) ** 2).sum()


class ViewProblem:
    """One view problem in float64: view `view` of a rig with cameras cams (dict R, t, f, c of the table), data weight dw (the
    stage's times the rig's scale), over frames with held keypoints q [F,K,3] and the view's detections gt_uv [F,K,2],
    conf [F,K]"""

    def __init__(self, cams, view, q, gt_uv, conf, jw, dw, rho, use_conf):
        self.R0, self.t0 = np.asarray(cams["R"][view]), np.asarray(cams["t"][view])
        self.f, self.c = cams["f"][view], cams["c"][view]
        self.sphere = view == 1
        self.E, self.n = sphere_basis(cams["R"][0], cams["t"][0], cams["R"][1], cams["t"][1]) if self.sphere else (None, None)
        t64 = lambda a: torch.as_tensor(np.asarray(a, np.float64))
        self.q, self.gt_uv, self.conf = t64(q), t64(gt_uv), t64(conf)
        self.jw, self.dw, self.rho, self.use_conf = jw, dw, rho, use_conf

    def camera(self, row):
        row = torch.as_tensor(np.asarray(row, np.float64))
        return cam_from_delta(self.R0, self.t0, row[ROT], row[CEN], self.sphere, self.E, self.n)

    def __call__(self, row):
        """(loss, gradient [86]) at an 86-entry row (float64)"""
        x = torch.as_tensor(np.asarray(row, np.float64)).clone().requires_grad_(True)
        R, t = cam_from_delta(self.R0, self.t0, x[ROT], x[CEN], self.sphere, self.E, self.n)
        loss = view_term(R, t, self.f, self.c, self.q, self.gt_uv, self.conf, self.jw, self.dw, self.rho, self.use_conf)
        loss.backward()
        g = x.grad.clone()
        keep = torch.zeros(86, dtype=torch.bool)
        keep[ROT] = True
        keep[CEN] = True
        if self.sphere:
            keep[84] = False
        g[~keep] = 0
        return float(loss.detach()), g.numpy()
