"""CPU: the camera-refinement block of mvs_math.cuh (cam_from_delta and its adjoint), compiled with g++ in float and double,
against the float64 restatement of oracle/camera_oracle.py and central differences: at random updates, small ones and exactly
0; the calibrated camera bit for bit at 0; view 1's centre at its calibrated distance from view 0 along a random path."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from mvsmplfitting_b200 import synthetic as S
from oracle import camera_oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
f32p, f64p = ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_double)


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    cxx = shutil.which("g++")
    if cxx is None:
        pytest.skip("no g++")
    so = str(tmp_path_factory.mktemp("camsim") / "libcamsim.so")
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-x", "c++", "-o", so,
                           os.path.join(HERE, "hostsim", "camera_hostsim.cpp")])
    return ctypes.CDLL(so)


def _p(a):
    return a.ctypes.data_as(f64p if a.dtype == np.float64 else f32p)


def cams8():
    return S.make_cameras(8)


def refine_of(cams, view):
    R0, t0 = np.ascontiguousarray(cams["R"][view], np.float32), np.ascontiguousarray(cams["t"][view], np.float32)
    if view == 1:
        E, n = O.sphere_basis(cams["R"][0], cams["t"][0], cams["R"][1], cams["t"][1])
    else:
        E, n = np.zeros((3, 2), np.float32), np.zeros(3, np.float32)
    return R0, t0, np.ascontiguousarray(E), np.ascontiguousarray(n), int(view == 1)


def fwd(lib, ref, w, c, dtype):
    R0, t0, E, n, sph = ref
    w, c = np.ascontiguousarray(w, dtype), np.ascontiguousarray(c, dtype)
    R, t = np.zeros(9, dtype), np.zeros(3, dtype)
    (lib.cam_fwd_f if dtype == np.float32 else lib.cam_fwd_d)(_p(R0), _p(t0), _p(E), _p(n), sph, _p(w), _p(c), _p(R), _p(t))
    return R.reshape(3, 3), t


def bwd(lib, ref, w, c, dR, dt, dtype):
    R0, t0, E, n, sph = ref
    a = [np.ascontiguousarray(v, dtype) for v in (w, c, np.reshape(dR, 9), dt)]
    gw, gc = np.zeros(3, dtype), np.zeros(3, dtype)
    (lib.cam_bwd_f if dtype == np.float32 else lib.cam_bwd_d)(_p(R0), _p(t0), _p(E), _p(n), sph, *[_p(v) for v in a], _p(gw), _p(gc))
    return gw, gc


def oracle(ref, w, c, dR, dt):
    R0, t0, E, n, sph = ref
    wt = torch.tensor(np.asarray(w, np.float64), requires_grad=True)
    ct = torch.tensor(np.asarray(c, np.float64), requires_grad=True)
    R, t = O.cam_from_delta(R0, t0, wt, ct, bool(sph), E, n)
    ((R * torch.tensor(np.reshape(dR, (3, 3)))).sum() + (t * torch.tensor(dt)).sum()).backward()
    gc = ct.grad.numpy().copy()
    if sph:
        gc[2] = 0
    return R.detach().numpy(), t.detach().numpy(), wt.grad.numpy(), gc


DELTAS = {"zero": 0.0, "tiny": 1e-6, "small": 1e-2, "large": 0.6}


@pytest.mark.parametrize("view", [1, 2, 5])
@pytest.mark.parametrize("size", list(DELTAS))
def test_map_and_adjoint_against_float64(lib, view, size):
    rng = np.random.RandomState(7 + view)
    ref = refine_of(cams8(), view)
    for _ in range(4):
        w, c = rng.normal(0, DELTAS[size], 3), rng.normal(0, DELTAS[size] * 0.5, 3)
        if ref[4]:
            c[2] = 0.0
        dR, dt = rng.normal(0, 1, (3, 3)), rng.normal(0, 1, 3)
        Ro, to, gwo, gco = oracle(ref, w, c, dR, dt)
        Rd, td = fwd(lib, ref, w, c, np.float64)
        assert np.allclose(Rd, Ro, rtol=0, atol=1e-12) and np.allclose(td, to, rtol=0, atol=1e-10)
        gwd, gcd = bwd(lib, ref, w, c, dR, dt, np.float64)
        assert np.allclose(gwd, gwo, rtol=1e-9, atol=1e-9), (gwd, gwo)
        assert np.allclose(gcd, gco, rtol=1e-9, atol=1e-9), (gcd, gco)
        Rf, tf = fwd(lib, ref, w, c, np.float32)
        assert np.abs(Rf - Ro).max() < 4e-7 and np.abs(tf - to).max() < 2e-6 * max(1.0, np.abs(to).max())
        gwf, gcf = bwd(lib, ref, w, c, dR, dt, np.float32)
        scale = 1.0 + np.abs(np.concatenate([gwo, gco])).max()
        assert np.abs(gwf - gwo).max() < 2e-5 * scale and np.abs(gcf - gco).max() < 2e-5 * scale, (gwf, gwo, gcf, gco)


@pytest.mark.parametrize("view", [1, 3])
def test_adjoint_against_central_differences(lib, view):
    rng = np.random.RandomState(11)
    ref = refine_of(cams8(), view)
    w, c = rng.normal(0, 0.05, 3), rng.normal(0, 0.05, 3)
    if ref[4]:
        c[2] = 0.0
    dR, dt = rng.normal(0, 1, (3, 3)), rng.normal(0, 1, 3)
    gw, gc = bwd(lib, ref, w, c, dR, dt, np.float64)
    J = lambda w_, c_: (lambda Rt: (Rt[0] * dR).sum() + (Rt[1] * dt).sum())(fwd(lib, ref, w_, c_, np.float64))
    h = 1e-6
    for i in range(3):
        e = np.zeros(3)
        e[i] = h
        assert abs((J(w + e, c) - J(w - e, c)) / (2 * h) - gw[i]) < 1e-6 * (1 + abs(gw[i]))
        if not (ref[4] and i == 2):
            assert abs((J(w, c + e) - J(w, c - e)) / (2 * h) - gc[i]) < 1e-6 * (1 + abs(gc[i]))
    if ref[4]:
        assert gc[2] == 0.0


@pytest.mark.parametrize("view", range(1, 8))
def test_zero_update_is_the_calibrated_camera_bit_for_bit(lib, view):
    cams = cams8()
    ref = refine_of(cams, view)
    R0, t0 = ref[0], ref[1]
    R0 = R0.copy()
    R0[0, 1] = -0.0 if R0[0, 1] == 0 else R0[0, 1]          # a -0 entry stays -0
    ref = (np.ascontiguousarray(R0),) + ref[1:]
    R, t = fwd(lib, ref, np.zeros(3), np.zeros(3), np.float32)
    assert R.tobytes() == R0.astype(np.float32).tobytes() and t.tobytes() == t0.tobytes()
    neg = ref[:1] + (np.ascontiguousarray(np.where(t0 == 0, np.float32(-0.0), t0)),) + ref[2:]
    R, t = fwd(lib, neg, -np.zeros(3), -np.zeros(3), np.float32)
    assert R.tobytes() == R0.astype(np.float32).tobytes() and t.tobytes() == neg[1].tobytes()


def test_view_one_keeps_its_distance_to_view_zero(lib):
    cams = cams8()
    ref = refine_of(cams, 1)
    C0 = O.centre(cams["R"][0], cams["t"][0])
    r0 = np.linalg.norm(O.centre(cams["R"][1], cams["t"][1]) - C0)
    rng = np.random.RandomState(3)
    w, c = np.zeros(3), np.zeros(3)
    for _ in range(50):                                       # a random walk of updates, up to tens of degrees
        w += rng.normal(0, 0.02, 3)
        c[:2] += rng.normal(0, 0.05, 2)
        R, t = fwd(lib, ref, w, c, np.float32)
        r = np.linalg.norm(O.centre(R, t) - C0)
        assert abs(r - r0) <= 8 * np.finfo(np.float32).eps * (r0 + np.abs(C0).max()), (r, r0)
