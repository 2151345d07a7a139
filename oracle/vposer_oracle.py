"""TEST INFRASTRUCTURE -- CPU restatement of VPoser.decode(z, 'aa') (reference model/VPoser.py), pinned against the
unmodified reference class by oracle/make_golden_vposer.py -> tests/golden/vposer_s11.npz.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may import this module.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F


def decode_6d(w: dict, z: torch.Tensor) -> torch.Tensor:
    """VPoser.py:218-224: leaky-ReLU(0.2) MLP 32 -> 512 -> 512 -> 138 (dropout is the identity in eval mode)."""
    t = lambda a: torch.as_tensor(np.asarray(a), dtype=z.dtype)
    h = F.leaky_relu(z @ t(w["fc1_w"]).T + t(w["fc1_b"]), negative_slope=0.2)
    h = F.leaky_relu(h @ t(w["fc2_w"]).T + t(w["fc2_b"]), negative_slope=0.2)
    return h @ t(w["out_w"]).T + t(w["out_b"])


def cont6d_to_matrot(x6: torch.Tensor) -> torch.Tensor:
    """ContinousRotReprDecoder.forward, VPoser.py:165-174.  x6 [n, 6] -> R [n, 3, 3] with columns b1, b2, b3."""
    r = x6.reshape(-1, 3, 2)
    b1 = F.normalize(r[:, :, 0], dim=1)
    dot = torch.sum(b1 * r[:, :, 1], dim=1, keepdim=True)
    b2 = F.normalize(r[:, :, 1] - dot * b1, dim=-1)
    b3 = torch.cross(b1, b2, dim=1)
    return torch.stack([b1, b2, b3], dim=-1)


def matrot_to_quaternion(R: torch.Tensor, eps: float = 1e-6) -> torch.Tensor:
    """rotation_matrix_to_quaternion, VPoser.py:29-98 (works on the transposed matrix; four branches)."""
    m = R.transpose(1, 2)
    d2 = m[:, 2, 2] < eps
    d0_d1 = m[:, 0, 0] > m[:, 1, 1]
    d0_nd1 = m[:, 0, 0] < -m[:, 1, 1]
    t0 = 1 + m[:, 0, 0] - m[:, 1, 1] - m[:, 2, 2]
    q0 = torch.stack([m[:, 1, 2] - m[:, 2, 1], t0, m[:, 0, 1] + m[:, 1, 0], m[:, 2, 0] + m[:, 0, 2]], -1)
    t1 = 1 - m[:, 0, 0] + m[:, 1, 1] - m[:, 2, 2]
    q1 = torch.stack([m[:, 2, 0] - m[:, 0, 2], m[:, 0, 1] + m[:, 1, 0], t1, m[:, 1, 2] + m[:, 2, 1]], -1)
    t2 = 1 - m[:, 0, 0] - m[:, 1, 1] + m[:, 2, 2]
    q2 = torch.stack([m[:, 0, 1] - m[:, 1, 0], m[:, 2, 0] + m[:, 0, 2], m[:, 1, 2] + m[:, 2, 1], t2], -1)
    t3 = 1 + m[:, 0, 0] + m[:, 1, 1] + m[:, 2, 2]
    q3 = torch.stack([t3, m[:, 1, 2] - m[:, 2, 1], m[:, 2, 0] - m[:, 0, 2], m[:, 0, 1] - m[:, 1, 0]], -1)
    c0 = (d2 & d0_d1).to(R.dtype).view(-1, 1)
    c1 = (d2 & ~d0_d1).to(R.dtype).view(-1, 1)
    c2 = (~d2 & d0_nd1).to(R.dtype).view(-1, 1)
    c3 = (~d2 & ~d0_nd1).to(R.dtype).view(-1, 1)
    q = q0 * c0 + q1 * c1 + q2 * c2 + q3 * c3
    q = q / torch.sqrt(t0.view(-1, 1) * c0 + t1.view(-1, 1) * c1 + t2.view(-1, 1) * c2 + t3.view(-1, 1) * c3)
    return q * 0.5


def quaternion_to_angle_axis(q: torch.Tensor) -> torch.Tensor:
    """VPoser.py:101-156"""
    q1, q2, q3 = q[..., 1], q[..., 2], q[..., 3]
    sin2 = q1 * q1 + q2 * q2 + q3 * q3
    sin_t = torch.sqrt(sin2)
    cos_t = q[..., 0]
    two_theta = 2.0 * torch.where(cos_t < 0.0, torch.atan2(-sin_t, -cos_t), torch.atan2(sin_t, cos_t))
    k = torch.where(sin2 > 0.0, two_theta / sin_t, 2.0 * torch.ones_like(sin_t))
    return torch.stack([q1 * k, q2 * k, q3 * k], dim=-1)


def decode_aa(w: dict, z: torch.Tensor) -> torch.Tensor:
    """VPoser.decode(z, output_type='aa') flattened to [n, 69] (fitting.py:121-123 view(1, -1))."""
    n = z.shape[0]
    R = cont6d_to_matrot(decode_6d(w, z))
    return quaternion_to_angle_axis(matrot_to_quaternion(R)).reshape(n, -1)


def rotation_branches(w: dict, z, eps: float = 1e-6) -> dict:
    """Where each decoded joint rotation of decode(z, 'aa') sits in the branch structure of matrot_to_quaternion and
    quaternion_to_angle_axis, in float64 (float32 weights are widened exactly).  z [n, 32] -> arrays [n, 23]:

    branch    0-3, the quaternion formula rotation_matrix_to_quaternion picks (m = R^T: 0 if m22 < eps and m00 > m11,
              1 if m22 < eps otherwise, 2 if m22 >= eps and m00 < -m11, 3 otherwise)
    surface   [n, 23, 3] signed distances to the three branch surfaces: m22 - eps, m00 - m11, m00 + m11.  Rotation-matrix
              entries lie in [-1, 1], so these are relative distances as they stand
    margin    distance to the nearest surface that decides this rotation's branch: m22 = eps, and m00 = m11 below it or
              m00 = -m11 above it (the other one is not tested, so a rotation may sit on it: the identity has m00 = m11)
    cos_neg   the quaternion's scalar part is negative (the atan2(-sin, -cos) side of quaternion_to_angle_axis)
    angle     the rotation angle |aa| in [0, pi]"""
    z = torch.as_tensor(np.asarray(z, dtype=np.float64))
    n = z.shape[0]
    R = cont6d_to_matrot(decode_6d(w, z))
    m = R.transpose(1, 2)
    d2 = m[:, 2, 2] < eps
    br = torch.where(d2, torch.where(m[:, 0, 0] > m[:, 1, 1], 0, 1), torch.where(m[:, 0, 0] < -m[:, 1, 1], 2, 3))
    surface = torch.stack([m[:, 2, 2] - eps, m[:, 0, 0] - m[:, 1, 1], m[:, 0, 0] + m[:, 1, 1]], -1)
    margin = torch.minimum(surface[:, 0].abs(), torch.where(d2, surface[:, 1], surface[:, 2]).abs())
    q = matrot_to_quaternion(R)
    aa = quaternion_to_angle_axis(q)
    return dict(branch=br.reshape(n, -1).numpy(), surface=surface.reshape(n, -1, 3).numpy(), margin=margin.reshape(n, -1).numpy(),
                cos_neg=(q[:, 0] < 0).reshape(n, -1).numpy(), angle=aa.norm(dim=-1).reshape(n, -1).numpy())
