"""CPU: the float64 render oracle (oracle/render_oracle.py) on scenes with known answers -- watertight top-left coverage of a
split rectangle, exact perspective depth on a plane, the shading formula on a plane facing the camera -- and the per-pixel routines
of mvs_render_dev.cuh, compiled with g++ (tests/hostsim/render_hostsim.cpp), against the oracle on the synthetic body."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

from mvsmplfitting_b200 import synthetic as S
from oracle import render_oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    cxx = shutil.which("g++")
    if cxx is None:
        pytest.skip("no g++")
    so = str(tmp_path_factory.mktemp("rendersim") / "librendersim.so")
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-x", "c++", "-o", so,
                           os.path.join(HERE, "hostsim", "render_hostsim.cpp")])
    return ctypes.CDLL(so)


def _identity_cam(f=100.0, c=(8.0, 6.0)):
    return dict(R=np.eye(3, dtype=np.float32)[None], t=np.zeros((1, 3), np.float32), f=np.full((1, 2), f, np.float32),
                c=np.asarray([c], np.float32))


@pytest.mark.parametrize("diag", [0, 1])
def test_split_rectangle_covers_its_pixels_once(diag):
    """a rectangle with corners on samples, split along either diagonal: every sample inside or on its top / left edge is
    covered by exactly one of the two triangles, no sample on its bottom / right edge or outside is covered"""
    W, H = 16, 12
    uv = np.array([[2.0, 3.0], [10.0, 3.0], [10.0, 8.0], [2.0, 8.0]])
    faces = np.array([[0, 1, 2], [0, 2, 3]]) if diag == 0 else np.array([[0, 1, 3], [1, 2, 3]])
    for fc in (faces, faces[:, ::-1].copy()):               # both windings
        r = O.rasterize(uv, np.ones(4), fc, W, H)
        want = np.zeros((H, W), np.int64)
        want[3:8, 2:10] = 1
        np.testing.assert_array_equal(r["count"], want)
        assert ((r["face"] >= 0) == (want == 1)).all()


def test_fan_around_a_vertex_is_watertight():
    """a fan of 8 triangles around a vertex on a sample, with spokes through samples: every sample of the polygon's interior
    is covered exactly once"""
    W, H = 24, 24
    ang = np.arange(8) * np.pi / 4
    rim = np.stack([12 + 8 * np.cos(ang), 12 + 8 * np.sin(ang)], 1)
    uv = np.concatenate([[[12.0, 12.0]], rim])
    faces = np.array([[0, 1 + k, 1 + (k + 1) % 8] for k in range(8)])
    r = O.rasterize(uv, np.ones(9), faces, W, H)
    yy, xx = np.mgrid[0:H, 0:W]
    inner = np.ones((H, W), bool)
    for k in range(8):                                      # strictly inside the octagon
        a, b = rim[k], rim[(k + 1) % 8]
        inner &= (b[0] - a[0]) * (yy - a[1]) - (b[1] - a[1]) * (xx - a[0]) > 1e-9
    assert r["count"][inner].min() == 1 and r["count"].max() == 1


@pytest.mark.parametrize("flip", [False, True])
def test_sample_aligned_meshes_are_watertight(lib, flip):
    """a grid and a fan whose vertices and shared edges lie on samples, in both windings: the oracle and the header's routines
    (host build) cover every sample inside exactly once and the outline's boundary samples as the fill rule says"""
    uv, faces, outlines = O.sample_meshes()
    if flip:
        faces = faces[:, ::-1].copy()
    W, H = 44, 24
    want = O.expected_coverage(outlines, W, H)
    r = O.rasterize(uv, np.ones(len(uv)), faces, W, H)
    np.testing.assert_array_equal(r["count"], want)
    sv = np.zeros((len(uv), 4), np.float32)
    sv[:, :2], sv[:, 2] = uv, 1.0
    f = np.ascontiguousarray(faces, np.int32)
    count, face = np.zeros((H, W), np.int32), np.zeros((H, W), np.int32)
    P = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    lib.render_count_host(f.shape[0], P(sv), P(f), W, H, P(count), P(face))
    np.testing.assert_array_equal(count, want)
    np.testing.assert_array_equal(face, r["face"])
    # samples on the boundary: top and left rows of the grid, upper edges of the diamond are drawn; the others are not
    assert want[2, 2:14].all() and want[2:14, 2].all() and not want[14, 2:15].any() and not want[2:15, 14].any()
    assert want[8, 26] and want[8, 34] and want[4, 30] and not want[16, 26] and not want[16, 34] and not want[20, 30]
    assert not want[12, 22] and not want[12, 38]


def test_compare_catches_cracks(lib):
    """the comparison the GPU tests use fails a rendering with holes along shared edges"""
    uv, faces, _ = O.sample_meshes()
    W, H = 44, 24
    cam = _identity_cam(f=1.0, c=(0.0, 0.0))
    verts = np.concatenate([uv, np.ones((len(uv), 1))], 1)
    r = O.render_view(verts, faces, cam, 0, W, H, ambient=1.0)
    bg = np.zeros((H, W, 3), np.uint8)
    O.compare(r, r["image"], r["face"].astype(np.int32), r["depth"].astype(np.float32), bg)
    cracked = r["face"].copy()
    edge = np.zeros((H, W), bool)
    edge[4, 2:13] = True                                    # a row of samples on shared grid edges
    cracked[edge] = -1
    img = r["image"].copy()
    img[edge] = 0
    depth = r["depth"].astype(np.float32)
    depth[edge] = np.inf
    assert r["ambiguous"][edge].all()
    with pytest.raises(AssertionError, match="crack"):
        O.compare(r, img, cracked.astype(np.int32), depth, bg)


def test_depth_exact_on_a_plane():
    """perspective-correct depth of a tilted plane equals the ray-plane intersection at every covered sample"""
    W, H = 64, 48
    cam = _identity_cam(f=60.0, c=(32.0, 24.0))
    # plane z = 3 + 0.4 x - 0.2 y (camera coordinates), a quad on it
    X = np.array([[-1.0, -0.8], [1.0, -0.8], [1.0, 0.8], [-1.0, 0.8]])
    verts = np.concatenate([X, (3 + 0.4 * X[:, 0] - 0.2 * X[:, 1])[:, None]], 1)
    r = O.render_view(verts, np.array([[0, 1, 2], [0, 2, 3]]), cam, 0, W, H)
    yy, xx = np.mgrid[0:H, 0:W]
    dx, dy = (xx - 32.0) / 60.0, (yy - 24.0) / 60.0
    z = 3.0 / (1 - 0.4 * dx + 0.2 * dy)                     # z = 3 + 0.4 z dx - 0.2 z dy
    cov = r["face"] >= 0
    assert cov.sum() > 500
    np.testing.assert_allclose(r["depth"][cov], z[cov], rtol=1e-12)


def test_shading_of_a_plane_facing_the_camera():
    W, H = 40, 30
    cam = _identity_cam(f=40.0, c=(20.0, 15.0))
    verts = np.array([[-1.0, -1.0, 2.0], [1.0, -1.0, 2.0], [1.0, 1.0, 2.0], [-1.0, 1.0, 2.0]])
    faces = np.array([[0, 2, 1], [0, 3, 2]])                # normal (0, 0, -1): towards the camera
    r = O.render_view(verts, faces, cam, 0, W, H, base_color=(0.5, 0.8, 1.0), ambient=0.3)
    yy, xx = np.mgrid[0:H, 0:W]
    p = np.stack([(xx - 20.0) / 40.0 * 2, (yy - 15.0) / 40.0 * 2, np.full((H, W), 2.0)], -1)
    I = 0.3 + 0.7 * 2.0 / np.linalg.norm(p, axis=-1)        # n.l = z / |p|
    cov = r["face"] >= 0
    for c, b in enumerate((0.5, 0.8, 1.0)):
        want = np.minimum(255, np.floor(255 * b * I + 0.5))
        np.testing.assert_array_equal(r["image"][..., c][cov], want[cov])
    assert (r["image"][~cov] == 0).all()


def _scene(distorted, W=256, H=192, seed=3):
    """the synthetic body, posed rigidly, in the views of a pinhole or a distorted rig with intrinsics scaled to W x H (the
    pinhole ring at 4 m, so that the body spans ~60 px there)"""
    model = S.make_model(0)
    cams = S.make_wide_cameras(4, distorted=distorted) if distorted else S.make_cameras(4, radius=4.0)
    s = W / 2048.0
    cams = dict(cams, f=cams["f"] * s, c=cams["c"] * s)
    rng = np.random.RandomState(seed)
    Rm = S.rodrigues_np(rng.normal(0, 0.4, 3))
    off = np.asarray(S.WIDE_OFFSET) if distorted else np.zeros(3)
    verts = (model["v_template"].astype(np.float64) @ Rm.T + off).astype(np.float32)
    kps = verts[[100, 2000, 4000, 6000]]
    return model, cams, verts, kps


def _host_render(lib, verts, faces, cam, view, W, H, kps, bg, base=(0.5, 0.5, 0.5), ambient=0.3, radius=3.0):
    uv, x = O.project(verts, cam, view)
    sv = np.zeros((verts.shape[0], 4), np.float32)
    sv[:, :2], sv[:, 2] = uv, x[:, 2]
    kuv, kx = O.project(kps, cam, view)
    kv = np.zeros((kps.shape[0], 4), np.float32)
    kv[:, :2], kv[:, 2] = kuv, kx[:, 2]
    pc = np.ascontiguousarray(x, np.float32)
    ns = np.ascontiguousarray(O.normal_sums(verts, faces), np.float32)
    R = np.ascontiguousarray(cam["R"][view], np.float32)
    f = np.ascontiguousarray(faces, np.int32)
    img = np.zeros((H, W, 3), np.uint8)
    face = np.zeros((H, W), np.int32)
    depth = np.zeros((H, W), np.float32)
    P = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    lib.render_view_host(verts.shape[0], f.shape[0], P(sv), P(f), W, H, P(pc), P(ns), P(R), kv.shape[0], P(kv),
                         P(np.asarray(base, np.float32)), ctypes.c_float(ambient), ctypes.c_float(radius),
                         P(np.array([0, 0, 255], np.uint8)), P(bg), P(img), P(face), P(depth))
    # the oracle sees the same float32 screen positions and camera-space points the routines saw
    return img, face, depth, sv


@pytest.mark.parametrize("distorted", [False, True])
def test_host_routines_match_oracle(lib, distorted):
    W, H = 256, 192
    model, cams, verts, kps = _scene(distorted, W, H)
    faces = model["f"].astype(np.int64)
    rng = np.random.RandomState(0)
    for view in range(4):
        bg = rng.randint(0, 256, size=(H, W, 3)).astype(np.uint8)
        img, face, depth, sv = _host_render(lib, verts, faces, cams, view, W, H, kps, bg)
        r = O.render_view(verts, faces, cams, view, W, H, keypoints=kps, background=bg, marker_radius=3.0)
        assert (r["face"] >= 0).sum() > 50
        share = O.compare(r, img, face, depth, bg)
        print("view %d: ambiguous %.3f %% of %d covered pixels" % (view, 100 * share, (r["face"] >= 0).sum()))
        # 13 776 faces on a body ~60 px tall are a fraction of a pixel each, so a sample is often within 0.01 px of an edge
        assert share < 0.25
