"""CPU: the lens-distortion blocks of mvs_math.cuh (project_fwd / project_bwd with coefficients) and mvs_init.cuh (undistort_px),
compiled with g++ in float and double: the forward against the float64 oracle (oracle/distortion_oracle.py) and OpenCV's
projectPoints, the adjoint against central differences, all-zero coefficients bit for bit the pinhole projection, and the Newton
undistortion against the forward and OpenCV's undistortPointsIter."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from mvsmplfitting_b200 import synthetic as S
from oracle import distortion_oracle as D

HERE = os.path.dirname(os.path.abspath(__file__))
f32p, f64p = ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_double)
# wide and mid-range lenses: barrel, pincushion, with tangential terms and a strong k3
COEFFS = [np.array([-0.25, 0.08, 0.0, 0.0, 0.0]), np.array([-0.18, 0.05, 1.5e-3, -8e-4, -0.01]),
          np.array([0.12, -0.03, -1e-3, 2e-3, 0.004])]


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    cxx = shutil.which("g++")
    if cxx is None:
        pytest.skip("no g++")
    so = str(tmp_path_factory.mktemp("distsim") / "libdistsim.so")
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-x", "c++", "-o", so,
                           os.path.join(HERE, "hostsim", "distortion_hostsim.cpp")])
    return ctypes.CDLL(so)


def _p(a):
    if a is None:
        return None
    return a.ctypes.data_as(f64p if a.dtype == np.float64 else f32p)


def _cam():
    cams = S.make_wide_cameras(4)
    return {k: np.ascontiguousarray(cams[k][1], np.float32) for k in ("R", "t", "f", "c")}


def _points(cam, n=200, r_max=0.55, seed=0):
    """world points whose normalised image radius is up to r_max"""
    rng = np.random.RandomState(seed)
    xn = rng.uniform(-r_max / np.sqrt(2), r_max / np.sqrt(2), size=(n, 2))
    z = rng.uniform(2.0, 5.0, size=n)
    xc = np.concatenate([xn * z[:, None], z[:, None]], 1)
    R, t = cam["R"].astype(np.float64), cam["t"].astype(np.float64)
    return (xc - t) @ R                       # R^T (xc - t)


def fwd(lib, cam, d, q, dtype):
    q = np.ascontiguousarray(q, dtype)
    n = q.shape[0]
    x, uv = np.zeros((n, 3), dtype), np.zeros((n, 2), dtype)
    dd = None if d is None else np.ascontiguousarray(d, np.float32)
    (lib.dist_fwd_f if dtype == np.float32 else lib.dist_fwd_d)(_p(cam["R"]), _p(cam["t"]), _p(cam["f"]), _p(cam["c"]), _p(dd), n,
                                                                 _p(q), _p(x), _p(uv))
    return x, uv


def bwd(lib, cam, d, x, duv, dtype):
    x, duv = np.ascontiguousarray(x, dtype), np.ascontiguousarray(duv, dtype)
    dq = np.zeros((x.shape[0], 3), dtype)
    dd = None if d is None else np.ascontiguousarray(d, np.float32)
    (lib.dist_bwd_f if dtype == np.float32 else lib.dist_bwd_d)(_p(cam["R"]), _p(cam["t"]), _p(cam["f"]), _p(cam["c"]), _p(dd),
                                                                 x.shape[0], _p(x), _p(duv), _p(dq))
    return dq


def undist(lib, cam, d, uv, dtype):
    uv = np.ascontiguousarray(uv, dtype)
    out = np.zeros_like(uv)
    dd = np.ascontiguousarray(d, np.float32)
    (lib.undist_f if dtype == np.float32 else lib.undist_d)(_p(cam["f"]), _p(cam["c"]), _p(dd), uv.shape[0], _p(uv), _p(out))
    return out


def test_wide_rig_reaches_the_lens_border():
    cams = S.make_wide_cameras(4)
    model = S.make_model(0)
    fr = S.make_frames_wide(model, cams, 4, seed=3)
    x = np.einsum("vab,nkb->vnka", cams["R"].astype(np.float64), fr["gt_joints3d"]) + cams["t"][:, None, None, :]
    r = np.sqrt((x[..., 0] / x[..., 2]) ** 2 + (x[..., 1] / x[..., 2]) ** 2)
    assert r.max() >= 0.4 and (x[..., 2] > 0.5).all()


@pytest.mark.parametrize("ci", range(len(COEFFS)))
def test_forward_against_float64_and_opencv(lib, ci):
    cam, d = _cam(), COEFFS[ci].astype(np.float32)
    q = _points(cam)
    d32 = d.astype(np.float64)
    want = D.project_distorted(*[torch.tensor(cam[k], dtype=torch.float64) for k in ("R", "t", "f", "c")], d32,
                               torch.tensor(q)).numpy()
    _, uv64 = fwd(lib, cam, d, q, np.float64)
    _, uv32 = fwd(lib, cam, d, q, np.float32)
    np.testing.assert_allclose(uv64, want, rtol=0, atol=1e-9)
    np.testing.assert_allclose(uv32, want, rtol=0, atol=2e-3 * max(1.0, float(cam["f"].max()) / 1000))
    cv2 = pytest.importorskip("cv2")
    K = np.array([[cam["f"][0], 0, cam["c"][0]], [0, cam["f"][1], cam["c"][1]], [0, 0, 1]], np.float64)
    rv, _ = cv2.Rodrigues(cam["R"].astype(np.float64))
    uv_cv, _ = cv2.projectPoints(q.reshape(-1, 1, 3), rv, cam["t"].astype(np.float64), K, d32)
    np.testing.assert_allclose(uv64, uv_cv.reshape(-1, 2), rtol=0, atol=5e-5)   # cv2 takes R through a rotation vector


@pytest.mark.parametrize("ci", range(len(COEFFS)))
def test_adjoint_against_central_differences(lib, ci):
    cam, d = _cam(), COEFFS[ci].astype(np.float32)
    q = _points(cam, n=40, seed=ci + 1)
    rng = np.random.RandomState(7)
    duv = rng.normal(size=(q.shape[0], 2))
    x, _ = fwd(lib, cam, d, q, np.float64)
    dq = bwd(lib, cam, d, x, duv, np.float64)
    h = 1e-6
    num = np.zeros_like(q)
    for j in range(3):
        e = np.zeros(3)
        e[j] = h
        up = fwd(lib, cam, d, q + e, np.float64)[1]
        um = fwd(lib, cam, d, q - e, np.float64)[1]
        num[:, j] = ((up - um) / (2 * h) * duv).sum(1)
    np.testing.assert_allclose(dq, num, rtol=1e-6, atol=1e-6 * np.abs(num).max())
    # the float build follows the double one to float precision
    dq32 = bwd(lib, cam, d, x.astype(np.float32), duv.astype(np.float32), np.float32)
    np.testing.assert_allclose(dq32, dq, rtol=0, atol=1e-4 * np.abs(dq).max())


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_zero_coefficients_are_the_pinhole_bits(lib, dtype):
    cam = _cam()
    q = _points(cam, n=300, r_max=0.8)
    z = np.zeros(5, np.float32)
    x0, uv0 = fwd(lib, cam, None, q, dtype)
    x1, uv1 = fwd(lib, cam, z, q, dtype)
    assert x0.tobytes() == x1.tobytes() and uv0.tobytes() == uv1.tobytes()
    duv = np.random.RandomState(1).normal(size=(q.shape[0], 2))
    assert bwd(lib, cam, None, x0, duv, dtype).tobytes() == bwd(lib, cam, z, x0, duv, dtype).tobytes()


@pytest.mark.parametrize("ci", range(len(COEFFS)))
def test_undistort_inverts_the_forward(lib, ci):
    cam, d = _cam(), COEFFS[ci].astype(np.float32)
    q = _points(cam, n=300, r_max=0.6, seed=ci)
    x, uv = fwd(lib, cam, d, q, np.float64)
    ideal = np.stack([x[:, 0] / x[:, 2], x[:, 1] / x[:, 2]], 1) * cam["f"].astype(np.float64) + cam["c"].astype(np.float64)
    got = undist(lib, cam, d, uv, np.float64)
    np.testing.assert_allclose(got, ideal, rtol=0, atol=1e-9 * float(cam["f"].max()))
    np.testing.assert_allclose(D.undistort(uv, cam["f"], cam["c"], d.astype(np.float64)), ideal, rtol=0,
                               atol=1e-9 * float(cam["f"].max()))
    got32 = undist(lib, cam, d, uv.astype(np.float32), np.float32)
    np.testing.assert_allclose(got32, ideal, rtol=0, atol=2e-3 * float(cam["f"].max()) / 1000)
    cv2 = pytest.importorskip("cv2")
    K = np.array([[cam["f"][0], 0, cam["c"][0]], [0, cam["f"][1], cam["c"][1]], [0, 0, 1]], np.float64)
    crit = (cv2.TERM_CRITERIA_COUNT | cv2.TERM_CRITERIA_EPS, 200, 1e-15)
    ucv = cv2.undistortPointsIter(uv.reshape(-1, 1, 2), K, d.astype(np.float64), None, K, crit).reshape(-1, 2)
    np.testing.assert_allclose(got, ucv, rtol=0, atol=1e-6)
