"""GPU: mvs_render against the float64 oracle (oracle/render_oracle.py) -- visibility, depth, composite and markers on pinhole and
distorted rigs at reduced and full resolution, determinism and independence of the call's size, rigs of different view counts,
all-zero distortion, frames behind the camera or off-screen, meshes of other sizes -- and every refusal of the C entry point."""
import ctypes

import numpy as np
import pytest
import torch

from mvsmplfitting_b200 import synthetic as S
from oracle import render_oracle as O
from tests import model_variants as MV

pytestmark = pytest.mark.gpu


def scaled(cams, W, H=None):
    s = W / 2048.0
    return dict(cams, f=np.ascontiguousarray(cams["f"] * s), c=np.ascontiguousarray(cams["c"] * s))


def make_ctx(model, cams, B, extra=None):
    from mvsmplfitting_b200.context import FittingContext
    ctx = FittingContext(0)
    if extra is None:
        ctx.set_model(model)
    else:
        ctx.set_model(model, extra_vertex_ids=extra)
    if isinstance(cams, list):
        ctx.set_camera_rigs(cams)
    else:
        ctx.set_camera_rigs([cams])
    ctx.set_batch(B)
    return ctx


def posed(ctx, model, cams, n, seed=1, wide=False):
    """verts [n,N,3], joints [n,K,3] of n synthetic frames (their ground-truth parameters) on the device"""
    fr = (S.make_frames_wide if wide else S.make_frames)(model, cams, n, seed=seed)
    x = torch.tensor(S.pack_params(fr["gt"]), device="cuda")
    out = ctx.forward_only(x, want_verts=True)
    return out["verts"], out["joints"]


def backgrounds(n, V, H, W, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, (n, V, H, W, 3), generator=g, dtype=torch.uint8).cuda()


def check_views(model, cams, verts, joints, bg, out, frames, W, H, radius=8.0, views=None):
    faces = np.asarray(model["f"], np.int64)
    shares = []
    V = cams["R"].shape[0]
    for f in frames:
        for v in (range(V) if views is None else views):
            r = O.render_view(verts[f].cpu().numpy(), faces, cams, v, W, H, keypoints=joints[f].cpu().numpy(),
                              background=bg[f, v].cpu().numpy(), marker_radius=radius)
            shares.append(O.compare(r, out["image"][f, v].cpu().numpy(), out["face"][f, v].cpu().numpy(),
                                    out["depth"][f, v].cpu().numpy(), bg[f, v].cpu().numpy()))
    return shares


ALL = ("image", "face", "depth")


@pytest.mark.parametrize("wide", [False, True])
def test_parity_reduced_resolution(syn_model, wide):
    W, H = 256, 192
    cams = scaled(S.make_wide_cameras(4) if wide else S.make_cameras(4), W)
    n = 3
    ctx = make_ctx(syn_model, cams, n)
    verts, joints = posed(ctx, syn_model, cams, n, wide=wide)
    bg = backgrounds(n, 4, H, W)
    out = ctx.render(verts, joints, background=bg, outputs=ALL, marker_radius=3.0)
    torch.cuda.synchronize()
    shares = check_views(syn_model, cams, verts, joints, bg, out, range(n), W, H, radius=3.0)
    print("wide" if wide else "pinhole", "ambiguous share per frame-view (%):", np.round(100 * np.array(shares), 2).tolist())
    # 13 776 faces on a body < 100 px tall are fractions of a pixel, so many samples lie within 0.01 px of an edge
    assert max(shares) < 0.25
    assert (out["face"] >= 0).sum() > 500
    ctx.close()


def test_parity_full_resolution(syn_model):
    W, H = 2048, 1536
    cams = S.make_wide_cameras(4)
    ctx = make_ctx(syn_model, cams, 1)
    verts, joints = posed(ctx, syn_model, cams, 1, seed=4, wide=True)
    bg = backgrounds(1, 4, H, W, seed=1)
    out = ctx.render(verts, joints, background=bg, outputs=ALL)
    torch.cuda.synchronize()
    shares = check_views(syn_model, cams, verts, joints, bg, out, [0], W, H, views=[1])
    print("full resolution: ambiguous %.3f %% of %d covered pixels" % (100 * shares[0], int((out["face"][0, 1] >= 0).sum())))
    assert shares[0] < 0.02
    ctx.close()


@pytest.mark.parametrize("flip", [False, True])
def test_sample_aligned_meshes_are_watertight(syn_model, flip):
    """a grid and a fan whose vertices and shared edges lie on samples (oracle.render_oracle.sample_meshes), in both windings:
    every sample inside is drawn, by the face the oracle's fill rule gives it, and the outline's boundary samples as the rule
    says -- no exemption for ambiguous pixels, since the positions are exact"""
    uv, faces, outlines = O.sample_meshes()
    if flip:
        faces = faces[:, ::-1].copy()
    W, H = 44, 24
    cam = dict(R=np.eye(3, dtype=np.float32)[None], t=np.zeros((1, 3), np.float32), f=np.ones((1, 2), np.float32),
               c=np.zeros((1, 2), np.float32))
    ctx = make_ctx(dict(syn_model, f=faces.astype(np.int32)), cam, 1)
    verts = np.zeros((1, syn_model["v_template"].shape[0], 3), np.float32)
    verts[0, :, 2] = -1.0
    verts[0, :len(uv), :2], verts[0, :len(uv), 2] = uv, 1.0
    out = ctx.render(torch.tensor(verts, device="cuda"), width=W, height=H, outputs=ALL)
    torch.cuda.synchronize()
    r = O.rasterize(uv, np.ones(len(uv)), faces, W, H)
    want = O.expected_coverage(outlines, W, H)
    np.testing.assert_array_equal(r["count"], want)
    got = out["face"][0, 0].cpu().numpy()
    np.testing.assert_array_equal(got >= 0, want == 1)
    np.testing.assert_array_equal(got, r["face"])
    ctx.close()


def test_determinism_and_independence_of_call_size(syn_model):
    W, H = 256, 192
    cams = scaled(S.make_cameras(4), W)
    ctx = make_ctx(syn_model, cams, 256)
    verts, joints = posed(ctx, syn_model, cams, 256, seed=7)
    bg = backgrounds(256, 4, H, W, seed=2)
    full = ctx.render(verts, joints, background=bg, outputs=ALL)
    again = ctx.render(verts, joints, background=bg, outputs=ALL)
    for k in ALL:
        assert torch.equal(full[k], again[k]), k
    for n in (1, 3, 64):
        for f0 in (0, 256 - n):
            part = ctx.render(verts[f0:f0 + n].contiguous(), joints[f0:f0 + n].contiguous(), background=bg[f0:f0 + n].contiguous(),
                              outputs=ALL)
            for k in ALL:
                assert torch.equal(part[k], full[k][f0:f0 + n]), (k, n, f0)
    ctx.close()


def test_rigs_sentinel_zero_distortion_and_offscreen(syn_model):
    from mvsmplfitting_b200 import _lib
    W, H = 192, 160
    pin = scaled(S.make_cameras(4, radius=4.0), W)
    two = scaled(S.make_cameras(2, radius=5.0), W)
    zero = dict(pin, dist=np.zeros((4, 5), np.float32))
    rigs = [dict(R=pin["R"], t=pin["t"], f=pin["f"], c=pin["c"]), dict(R=two["R"], t=two["t"], f=two["f"], c=two["c"]), zero]
    ctx = make_ctx(syn_model, rigs, 4)
    verts, joints = posed(ctx, syn_model, pin, 4, seed=5)
    rig = torch.tensor([0, 1, 2, 1], dtype=torch.int32, device="cuda")
    img = torch.full((4, 4, H, W, 3), 77, dtype=torch.uint8, device="cuda")
    face = torch.full((4, 4, H, W), -7, dtype=torch.int32, device="cuda")
    depth = torch.full((4, 4, H, W), -3.0, dtype=torch.float32, device="cuda")
    cfg = _lib.RenderConfig(W, H, (ctypes.c_float * 3)(0.5, 0.5, 0.5), 0.3, 8.0, (ctypes.c_ubyte * 3)(0, 0, 255))
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    rc = ctx.lib.mvs_render(ctx.h, 4, p(verts), p(joints), p(rig), None, p(img), p(face), p(depth), ctypes.byref(cfg), None)
    assert rc == 0, ctx.lib.mvs_last_error(ctx.h)
    torch.cuda.synchronize()
    for f in (1, 3):                                        # rig 1 has 2 views: rows 2, 3 untouched
        assert (img[f, 2:] == 77).all() and (face[f, 2:] == -7).all() and (depth[f, 2:] == -3.0).all()
        assert (face[f, :2] >= 0).any()
    for f in (0, 2):
        assert (face[f] >= -1).all()
    # rig 2 (all-zero coefficients) gives rig 0's bits
    same = ctx.render(verts[[2, 2]].contiguous(), joints[[2, 2]].contiguous(), rig=[0, 2], width=W, height=H, outputs=ALL)
    for k in ALL:
        assert torch.equal(same[k][0], same[k][1]), k
    # a frame far off-screen renders background, with no fault
    far = (verts[:1] + torch.tensor([0.0, 500.0, 0.0], device="cuda")).contiguous()
    bg = backgrounds(1, 4, H, W, seed=3)
    out = ctx.render(far, None, rig=[0], background=bg, outputs=ALL)
    torch.cuda.synchronize()
    assert (out["face"] == -1).all() and torch.equal(out["image"], bg) and torch.isinf(out["depth"]).all()
    ctx.close()


def test_behind_the_camera(syn_model):
    """a body straddling and behind view 0's image plane: triangles with a vertex at depth <= 1e-3 are not drawn"""
    W, H = 128, 96
    cams = scaled(S.make_cameras(2, radius=4.0), W)
    ctx = make_ctx(syn_model, cams, 2)
    verts, joints = posed(ctx, syn_model, cams, 2, seed=6)
    R, t = cams["R"][0].astype(np.float64), cams["t"][0].astype(np.float64)
    centre = -R.T @ t                                       # camera 0's position
    back = R[2]                                             # its optical axis in world space
    moved = verts.clone()
    moved[0] = verts[0] - verts[0].mean(0) + torch.tensor(centre, device="cuda", dtype=torch.float32)        # around the camera
    moved[1] = verts[1] - verts[1].mean(0) + torch.tensor(centre - 3 * back, device="cuda", dtype=torch.float32)  # behind it
    bg = backgrounds(2, 2, H, W, seed=4)
    out = ctx.render(moved.contiguous(), None, background=bg, outputs=ALL, marker_radius=0.0)
    torch.cuda.synchronize()
    assert (out["face"][1, 0] == -1).all() and torch.equal(out["image"][1, 0], bg[1, 0])
    for f in range(2):
        check_views(syn_model, cams, moved, joints, bg, out, [f], W, H, radius=0.0, views=[0])
    ctx.close()


@pytest.mark.parametrize("N", [431, 10475])
def test_other_model_sizes(N):
    model, extra = MV.make_sized_model(N)
    W, H = 256, 192
    cams = scaled(S.make_wide_cameras(3), W)
    ctx = make_ctx(model, cams, 2, extra=extra)
    x = torch.tensor(S.pack_params(S.make_frames_wide(S.make_model(0), cams, 2, seed=8)["gt"]), device="cuda")
    fwd = ctx.forward_only(x, want_verts=True)
    bg = backgrounds(2, 3, H, W, seed=5)
    out = ctx.render(fwd["verts"], fwd["joints"], background=bg, outputs=ALL, marker_radius=3.0)
    torch.cuda.synchronize()
    check_views(model, cams, fwd["verts"], fwd["joints"], bg, out, range(2), W, H, radius=3.0)
    assert (out["face"] >= 0).sum() > 200
    ctx.close()


def test_refusals_write_nothing(syn_model):
    from mvsmplfitting_b200 import _lib
    from mvsmplfitting_b200.context import FittingContext
    W, H = 64, 48
    cams = scaled(S.make_cameras(2), W)
    ctx = make_ctx(syn_model, [cams, cams], 2)
    verts, joints = posed(ctx, syn_model, cams, 2)
    img = torch.full((2, 2, H, W, 3), 9, dtype=torch.uint8, device="cuda")
    p = lambda t: None if t is None else ctypes.c_void_p(t.data_ptr())
    good = torch.tensor([0, 1], dtype=torch.int32, device="cuda")
    bad = torch.tensor([0, 2], dtype=torch.int32, device="cuda")

    def cfg(**kw):
        d = dict(width=W, height=H, base=(0.5, 0.5, 0.5), ambient=0.3, radius=8.0)
        d.update(kw)
        return _lib.RenderConfig(d["width"], d["height"], (ctypes.c_float * 3)(*d["base"]), d["ambient"], d["radius"],
                                 (ctypes.c_ubyte * 3)(0, 0, 255))

    def call(n=2, v=verts, rig=good, out=img, c=None, h=None):
        return ctx.lib.mvs_render(h or ctx.h, n, p(v), p(joints), p(rig), None, p(out), None, None,
                                  ctypes.byref(c or cfg()), None)

    cases = dict(n0=call(n=0), verts=call(v=None), outputs=call(out=None), rig=call(rig=bad), no_rig=call(rig=None),
                 w0=call(c=cfg(width=0)), h_big=call(c=cfg(height=8193)), base=call(c=cfg(base=(0.5, 1.5, 0.5))),
                 base_nan=call(c=cfg(base=(float("nan"), 0.5, 0.5))), amb=call(c=cfg(ambient=-0.1)),
                 amb_inf=call(c=cfg(ambient=float("inf"))), radius=call(c=cfg(radius=-1.0)), radius_nan=call(c=cfg(radius=float("nan"))))
    torch.cuda.synchronize()
    for k, rc in cases.items():
        assert rc == -1, (k, rc)                           # MVS_ERR_INVALID
    assert (img == 9).all()
    assert ctx.lib.mvs_render(ctx.h, 2, p(verts), None, p(bad), None, p(img), None, None, ctypes.byref(cfg()), None) == -1
    assert b"frame 1" in ctx.lib.mvs_last_error(ctx.h)
    # a model without faces
    nf = FittingContext(0)
    nf.set_model(dict(syn_model, f=None))
    nf.set_cameras(cams["R"], cams["t"], cams["f"], cams["c"])
    assert nf.lib.mvs_render(nf.h, 2, p(verts), None, None, None, p(img), None, None, ctypes.byref(cfg()), None) == -1
    assert (img == 9).all()
    nf.close()
    ctx.close()
