"""float64 restatement of mvs_render (include/mvsmpl.h, DESIGN.md section 4d), the checker of the device rasteriser.

Everything the kernels do, in numpy and float64: projection through a view (with OpenCV's radial-tangential distortion), vertex
normals (R . normalize(sum of the faces' cross products)), the fill rule (sample of pixel (x, y) at (x, y); an edge evaluated with
its endpoints in ascending vertex-id order; a sample exactly on an edge belongs to the triangle whose interior lies below the
edge -- whatever its slope -- or, for a vertical edge, to its right), perspective-correct depth z = 1 / sum lam_i / z_i, the
headlight shading and the keypoint markers.

Besides the picture it reports what a float32 implementation may legitimately decide otherwise: per pixel the candidate faces
(triangles whose sample lies inside or within `margin` px of their edges) and whether the pixel is ambiguous (its sample within
`margin` px of an edge of a candidate that is not behind the visible surface, or the two nearest depths within `depth_rel` of each
other).  Candidates behind the visible surface are left out of the first test because their edges cannot change which face is
seen: where the visible face's own edge is near, the sample is ambiguous through that face.  It also reports where an
implementation may show no face although the oracle shows one: only near a silhouette edge (an edge with one face, or whose two
faces lie on the same side of it on screen, or with a neighbour that is not drawn).  Anywhere else, on or near an edge two drawn
faces share, a missing face is a crack."""
from __future__ import annotations

import numpy as np

NEAR = 1e-3


def project(verts, cam: dict, view: int):
    """verts [N,3] -> (uv [N,2], x [N,3] camera-space) through view `view` of a camera dict (R, t, f, c and optional dist [V,5])"""
    R = np.asarray(cam["R"], np.float64)[view]
    t = np.asarray(cam["t"], np.float64)[view]
    x = np.asarray(verts, np.float64) @ R.T + t
    xn, yn = x[:, 0] / x[:, 2], x[:, 1] / x[:, 2]
    if cam.get("dist") is not None:
        k1, k2, p1, p2, k3 = np.asarray(cam["dist"], np.float64)[view]
        r2 = xn * xn + yn * yn
        a = 1 + r2 * (k1 + r2 * (k2 + r2 * k3))
        xn, yn = (xn * a + 2 * p1 * xn * yn + p2 * (r2 + 2 * xn * xn), yn * a + p1 * (r2 + 2 * yn * yn) + 2 * p2 * xn * yn)
    f = np.asarray(cam["f"], np.float64)[view]
    c = np.asarray(cam["c"], np.float64)[view]
    return np.stack([xn * f[0] + c[0], yn * f[1] + c[1]], 1), x


def normal_sums(verts, faces):
    """[N,3]: per vertex the sum of cross(b - a, c - a) over the faces around it (world space)"""
    v = np.asarray(verts, np.float64)
    f = np.asarray(faces, np.int64)
    cr = np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])
    s = np.zeros_like(v)
    for k in range(3):
        np.add.at(s, f[:, k], cr)
    return s


def camera_normals(sums, R):
    """R . normalize(sums), 0 where a sum is 0"""
    l = np.linalg.norm(sums, axis=1, keepdims=True)
    u = np.where(l > 0, sums / np.where(l > 0, l, 1), 0.0)
    return u @ np.asarray(R, np.float64).T


def _edges(P, ids):
    """per triangle and edge k (opposite vertex k): canonical endpoints a, b [T,3,2], sign s [T,3] making the edge function
    positive inside, ownership [T,3] (top-left), orientation valid [T]"""
    j, l = np.array([1, 2, 0]), np.array([2, 0, 1])
    Pj, Pl = P[:, j], P[:, l]
    ij, il = ids[:, j], ids[:, l]
    fwd = ij < il
    a = np.where(fwd[..., None], Pj, Pl)
    b = np.where(fwd[..., None], Pl, Pj)
    sig = np.where(fwd, 1.0, -1.0)
    e2 = (b[:, 2, 0] - a[:, 2, 0]) * (P[:, 2, 1] - a[:, 2, 1]) - (b[:, 2, 1] - a[:, 2, 1]) * (P[:, 2, 0] - a[:, 2, 0])
    o = sig[:, 2] * e2
    s = sig * np.sign(o)[:, None]
    gy = s * (b[..., 0] - a[..., 0])
    gx = -s * (b[..., 1] - a[..., 1])
    own = (gy > 0) | ((gy == 0) & (gx > 0))
    valid = (o != 0) & np.all(ij != il, axis=1)
    return a, b, s, own, valid


def rasterize(uv, z, faces, W: int, H: int, margin: float = 0.01, depth_rel: float = 1e-5):
    """Screen-space visibility of the triangles faces [F,3] over vertices uv [N,2] (pixels) at camera depths z [N].
    Returns dict(face [H,W] int (-1: none), depth [H,W] (inf: none), lam [H,W,3] screen barycentrics of the visible face,
    count [H,W] (triangles covering the sample), ambiguous [H,W] bool, silhouette [H,W] bool (the sample is within margin of a
    silhouette edge of a candidate that is not behind the visible surface), cand (pixel * F + face of every candidate pair,
    sorted))."""
    uv = np.asarray(uv, np.float64)
    z = np.asarray(z, np.float64)
    faces = np.asarray(faces, np.int64)
    F = faces.shape[0]
    P = uv[faces]                                       # [F,3,2]
    Z = z[faces]
    ok = np.all(Z > NEAR, axis=1) & np.all(np.isfinite(P), axis=(1, 2)) & np.all(np.isfinite(Z), axis=1)
    a, b, s, own, valid = _edges(P, faces)
    ok &= valid
    # silhouette edges: an edge is interior when exactly two drawn faces share it and they have the same screen orientation
    sgn = np.where(ok, np.sign(s[:, 0] * np.where(faces[:, 1] < faces[:, 2], 1.0, -1.0)), 0.0)   # orientation of each face
    ek = np.sort(np.stack([faces[:, [1, 2]], faces[:, [2, 0]], faces[:, [0, 1]]], 1), axis=-1).reshape(-1, 2)  # edge k of face t
    key = ek[:, 0] * (faces.max() + 1) + ek[:, 1]
    _, inv, cnt_e = np.unique(key, return_inverse=True, return_counts=True)
    fs = np.repeat(sgn, 3)
    sum_s = np.zeros(cnt_e.size)
    np.add.at(sum_s, inv, fs)
    drawn = np.zeros(cnt_e.size, np.int64)
    np.add.at(drawn, inv, (fs != 0).astype(np.int64))
    interior = (cnt_e == 2) & (drawn == 2) & (np.abs(sum_s) == 2)
    sil = ~interior[inv].reshape(F, 3)
    lo, hi = P.min(1), P.max(1)
    x0 = np.clip(np.ceil(lo[:, 0] - margin), 0, W)
    x1 = np.clip(np.floor(hi[:, 0] + margin), -1, W - 1)
    y0 = np.clip(np.ceil(lo[:, 1] - margin), 0, H)
    y1 = np.clip(np.floor(hi[:, 1] + margin), -1, H - 1)
    nx = np.where(ok, np.maximum(x1 - x0 + 1, 0), 0).astype(np.int64)
    ny = np.where(ok, np.maximum(y1 - y0 + 1, 0), 0).astype(np.int64)
    cnt = nx * ny
    tri = np.repeat(np.arange(F), cnt)
    loc = np.arange(cnt.sum()) - np.repeat(np.cumsum(cnt) - cnt, cnt)
    px = x0[tri] + loc % nx[tri]
    py = y0[tri] + loc // nx[tri]
    A, Bp, Sg, Ow = a[tri], b[tri], s[tri], own[tri]
    e = (Bp[..., 0] - A[..., 0]) * (py[:, None] - A[..., 1]) - (Bp[..., 1] - A[..., 1]) * (px[:, None] - A[..., 0])
    w = Sg * e                                          # [pairs,3]
    elen = np.linalg.norm(Bp - A, axis=-1)
    d = w / elen                                        # signed distance to each edge, positive inside
    cover = np.all((w > 0) | ((w == 0) & Ow), axis=1) & (w.sum(1) > 0)
    cand = np.all(d >= -margin, axis=1)
    near = cand & (np.abs(d).min(1) < margin)
    pix = (py * W + px).astype(np.int64)
    lam = w / np.where(w.sum(1) != 0, w.sum(1), 1)[:, None]
    dep = 1.0 / (lam / Z[tri]).sum(1)
    out_face = np.full(H * W, -1, np.int64)
    out_depth = np.full(H * W, np.inf)
    out_lam = np.zeros((H * W, 3))
    count = np.zeros(H * W, np.int64)
    amb = np.zeros(H * W, bool)
    np.add.at(count, pix[cover], 1)
    c = np.nonzero(cover)[0]
    if c.size:
        order = c[np.lexsort((tri[c], dep[c], pix[c]))]
        first = np.ones(order.size, bool)
        first[1:] = pix[order][1:] != pix[order][:-1]
        win = order[first]
        out_face[pix[win]] = tri[win]
        out_depth[pix[win]] = dep[win]
        out_lam[pix[win]] = lam[win]
        # the runner-up depth of every pixel with two or more covering triangles
        second = np.zeros(order.size, bool)
        second[1:] = first[:-1] & ~first[1:]
        run = order[second]
        d1 = out_depth[pix[run]]
        amb[pix[run]] |= np.abs(dep[run] - d1) <= depth_rel * d1
    # a sample near an edge of a candidate that is not behind the visible surface (its depth, extrapolated outside the triangle,
    # at most the visible one's): only there can float32 positions change the visible face
    front = near & (dep <= out_depth[pix] * (1 + depth_rel))
    amb[pix[front]] = True
    silh = np.zeros(H * W, bool)
    near_sil = front & np.any((np.abs(d) < margin) & sil[tri], axis=1)
    silh[pix[near_sil]] = True
    return dict(face=out_face.reshape(H, W), depth=out_depth.reshape(H, W), lam=out_lam.reshape(H, W, 3),
                count=count.reshape(H, W), ambiguous=amb.reshape(H, W), silhouette=silh.reshape(H, W),
                cand=np.unique(pix[cand] * F + tri[cand]), F=F)


def intensity(lam, z, p, n, ambient):
    """headlight intensity at covered pixels: lam [M,3], z [M,3], p / n [M,3,3] camera-space vertex positions / normals"""
    w = lam / z
    w = w / w.sum(1, keepdims=True)
    N = np.einsum("mk,mkc->mc", w, n)
    Pp = np.einsum("mk,mkc->mc", w, p)
    nl, pl = np.linalg.norm(N, axis=1), np.linalg.norm(Pp, axis=1)
    ok = (nl > 0) & (pl > 0)
    dd = np.where(ok, -(N * Pp).sum(1) / np.where(ok, nl * pl, 1), 0.0)
    return ambient + (1 - ambient) * np.maximum(0.0, dd)


def render_view(verts, faces, cam: dict, view: int, W: int, H: int, keypoints=None, background=None, base_color=(0.5, 0.5, 0.5),
                ambient: float = 0.3, marker_radius: float = 8.0, marker_color=(0, 0, 255), margin: float = 0.01,
                depth_rel: float = 1e-5):
    """One view of one frame as mvs_render draws it.  Returns rasterize's dict plus image [H,W,3] uint8, shade [H,W,3] (the
    unrounded 255 base I + 1/2, covered pixels), marker [H,W] bool and marker_edge [H,W] bool (samples within margin of a disc's
    rim, where float32 may decide either way)."""
    uv, x = project(verts, cam, view)
    r = rasterize(uv, x[:, 2], faces, W, H, margin, depth_rel)
    faces = np.asarray(faces, np.int64)
    nrm = camera_normals(normal_sums(verts, faces), np.asarray(cam["R"], np.float64)[view])
    img = np.zeros((H, W, 3), np.uint8) if background is None else np.array(background, np.uint8).reshape(H, W, 3)
    shade = np.zeros((H, W, 3))
    cov = r["face"] >= 0
    if cov.any():
        fi = faces[r["face"][cov]]
        I = intensity(r["lam"][cov], x[fi, 2], x[fi], nrm[fi], ambient)
        v = 255.0 * np.asarray(base_color, np.float64)[None] * I[:, None] + 0.5
        shade[cov] = v
        img[cov] = np.minimum(255, np.floor(v)).astype(np.uint8)
    mk = np.zeros((H, W), bool)
    edge = np.zeros((H, W), bool)
    if keypoints is not None and marker_radius > 0:
        kuv, kx = project(keypoints, cam, view)
        yy, xx = np.mgrid[0:H, 0:W]
        for (u, v_), zz in zip(kuv, kx[:, 2]):
            if not zz > NEAR:
                continue
            dist = np.hypot(xx - u, yy - v_)
            mk |= dist <= marker_radius
            edge |= np.abs(dist - marker_radius) < margin
        img[mk] = np.asarray(marker_color, np.uint8)
    r.update(image=img, shade=shade, marker=mk, marker_edge=edge, uv=uv, x=x, normals=nrm)
    return r


def compare(r, img, face, depth, bg, marker_color=(0, 0, 255)):
    """Checks a float32 rendering (image [H,W,3], face [H,W], depth [H,W]) of one view against render_view's result r over
    background bg [H,W,3]: face ids equal at every non-ambiguous pixel, a candidate at ambiguous ones (so a crack or a missing
    silhouette pixel away from an edge fails), depth within 1e-5 where the faces agree, background bytes equal, shaded pixels
    within 1 LSB, markers where the oracle puts them (up to samples on a disc's rim).  No face where the oracle has one is
    accepted only near a silhouette edge, so a crack along an edge two drawn faces share fails.  Raises AssertionError; returns
    the share of ambiguous pixels among covered ones."""
    amb, of = r["ambiguous"], r["face"]
    bad = (face != of) & ~amb
    assert not bad.any(), "%d non-ambiguous face mismatches, first at %s" % (bad.sum(), np.argwhere(bad)[:5].tolist())
    hole = (face < 0) & (of >= 0) & ~r["silhouette"]
    assert not hole.any(), "%d pixels without a face away from any silhouette edge (cracks), first at %s" % (
        hole.sum(), np.argwhere(hole)[:5].tolist())
    H, W = of.shape
    pix = np.arange(H * W).reshape(H, W)
    g = amb & (face >= 0)
    assert np.isin(pix[g] * r["F"] + face[g], r["cand"]).all(), "a face that is not a candidate at an ambiguous pixel"
    agree = (face == of) & (of >= 0)
    np.testing.assert_allclose(depth[agree], r["depth"][agree], rtol=1e-5)
    assert np.isinf(depth[face < 0]).all()
    mk, sure = r["marker"], ~r["marker_edge"]
    back = (face < 0) & (of < 0) & ~mk & sure
    np.testing.assert_array_equal(img[back], np.asarray(bg)[back])
    shaded = agree & ~mk & sure
    d = np.abs(img[shaded].astype(int) - r["image"][shaded].astype(int))
    assert d.max(initial=0) <= 1, "shaded pixels differ by %d" % d.max()
    np.testing.assert_array_equal(img[mk & sure], np.broadcast_to(np.asarray(marker_color, np.uint8), img[mk & sure].shape))
    return amb.sum() / max(1, (of >= 0).sum())


def sample_meshes():
    """Planar meshes whose vertices and shared edges pass through samples, side by side on a 44 x 24 image: a 6 x 6 grid of
    2-px quads split along alternating diagonals, and a fan of 8 triangles around the centre of a diamond whose rim vertices are
    samples.  Returns (uv [N,2], faces [F,3], outlines: the convex outline of each mesh, in order)."""
    g = np.array([[2 + 2 * i, 2 + 2 * j] for j in range(7) for i in range(7)], np.float64)
    faces = []
    for j in range(6):
        for i in range(6):
            a = 7 * j + i
            b, c, d = a + 1, a + 8, a + 7
            faces += [[a, b, c], [a, c, d]] if (i + j) % 2 == 0 else [[a, b, d], [b, c, d]]
    rim = np.array([[38, 12], [34, 16], [30, 20], [26, 16], [22, 12], [26, 8], [30, 4], [34, 8]], np.float64)
    uv = np.concatenate([g, [[30.0, 12.0]], rim])
    c0 = g.shape[0]
    faces += [[c0, c0 + 1 + k, c0 + 1 + (k + 1) % 8] for k in range(8)]
    outlines = [np.array([[2.0, 2.0], [14.0, 2.0], [14.0, 14.0], [2.0, 14.0]]), rim[[0, 2, 4, 6]]]
    return uv, np.array(faces, np.int64), outlines


def expected_coverage(outlines, W: int, H: int):
    """[H,W] 0/1: the samples a convex outline covers under the fill rule, computed on the outline alone: inside, or on its
    boundary where every boundary edge through the sample has the interior below it (a vertical one: to its right) -- the same
    as moving the sample down by an infinitesimal step and right by a much smaller one"""
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float64)
    out = np.zeros((H, W), np.int64)
    for poly in outlines:
        cen = poly.mean(0)
        inside = np.ones((H, W), bool)
        for k in range(len(poly)):
            a, b = poly[k], poly[(k + 1) % len(poly)]
            e = lambda x, y: (b[0] - a[0]) * (y - a[1]) - (b[1] - a[1]) * (x - a[0])
            s = np.sign(e(cen[0], cen[1]))
            w = s * e(xx, yy)
            gy, gx = s * (b[0] - a[0]), -s * (b[1] - a[1])
            own = gy > 0 or (gy == 0 and gx > 0)
            inside &= (w > 0) | ((w == 0) & own)
        out += inside
    return out
