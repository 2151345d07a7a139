"""Model, prior and keypoint-set variants that put the frame-resident kernels at their limits, and a host mirror of the
bookkeeping mvs_set_model does (csrc/mvs_api.cu), so that a test can tell which branch a variant reaches.

The frame-resident closure (csrc/mvs_resident_dev.cuh) has fixed shared-memory envelopes:
  nsup + 6 <= kResMaxSup       support vertices plus the SDF term's box-extreme vertices, else the batched chain
  V * K <= kResMaxVK           views x keypoints, else the batched chain
  M <= kResMaxM                GMM components, else the batched chain
  nkpe <= kResMaxKpE           keypoint entries staged in shared memory (kp_on), else read from global memory
  nsupj <= kResMaxSupJ         (support vertex, joint) skinning pairs staged (sj_on), else read from global memory
and skin_kernel (csrc/mvs_tc.cu) stages the ELL skinning weights only when KW <= kSkinEllMax (ell_smem).

Every variant starts from synthetic.make_model(0) / make_gmm(7) and changes one thing.  A grown regressor row keeps its
own non-zeros and spreads a small share of its weight over nearby vertices, so it stays non-negative, sums to 1 and regresses
nearly the same keypoint; replaced skinning rows stay normalised.  CPU only: imported by the variant / limit test and by
the GPU parity tests.
"""
from __future__ import annotations

import os
import re

import numpy as np

from mvsmplfitting_b200 import synthetic as S

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "mvsmplfitting_b200", "csrc")
LSP_ROWS = sorted({int(s) for s in S.JOINT_MAP_LSP14 if s < 14})        # the 12 regressor rows the LSP keypoint map reads


def limits() -> dict:
    """the kernels' envelope and tiling constants, read from the CUDA sources (`= 64;` and `= 1 << 17;` forms)"""
    out = {}
    for f in ("mvs_resident_dev.cuh", "mvs_tc_dev.cuh", "mvs_math.cuh", "mvs_tc.cu", "mvs_sdf_dev.cuh", "mvs_internal.cuh",
              "mvs_sdf_bins.cuh"):
        src = open(os.path.join(CSRC, f)).read()
        for k, a, s in re.findall(r"constexpr\s+int\s+(k\w+)\s*=\s*(\d+)\s*(?:<<\s*(\d+)\s*)?;", src):
            out[k] = int(a) << int(s or 0)
    m = re.search(r"m\.nsup\s*\+\s*(\d+)\s*<=\s*kResMaxSup", open(os.path.join(CSRC, "mvs_resident.cu")).read())
    out["kResExtraSup"] = int(m.group(1))          # resident_supported(): room for the box-extreme vertices
    return out


def tails(N: int, lim: dict | None = None) -> dict:
    """host mirror of the vertex-count-dependent tiling of the dense kernels at N vertices"""
    lim = lim or limits()
    rows = 3 * N
    last = rows % lim["kTcRows"] or lim["kTcRows"]          # rows of the last posedirs tile
    nbox = -(-N // lim["kSkinV"])                           # 64-vertex skinning chunks = chunk boxes
    return dict(
        tc_tiles=-(-rows // lim["kTcRows"]),                # posedirs_gemm_tc 128-row tiles
        tc_last_rows=last,
        tc_last_wg1_rows=max(0, last - lim["kTcRows"] // 2),   # rows of warpgroup 1 in the last tile (0: idle)
        nbox=nbox,
        chunk_tail=N % lim["kSkinV"],                       # vertices of a partial last chunk (0: none)
        setup_groups=-(-nbox // (32 * lim["kSetupCh"])),    # sdf_frame_setup fold-loop trips
        cull=nbox <= 32 * lim["kSdfSkipWords"],             # chunk-cull bits cover every chunk
        sdf_blocks=-(-N // lim["kSdfFThreads"]),            # 256-vertex blocks of sdf_fused = partials frame_step sums
        block_tail=N % lim["kSdfFThreads"],
        tb_chunks=-(-rows // lim["kTbRows"]),               # vertex_bwd_tc 32-row reduction chunks
        tb_pad=(rows + 3) // 4 * 4 - rows,                  # tb_dvp_ld(N) - 3N
        simt_tail=N % lim["kTileV"],                        # vertices of the SIMT kernels' partial last tile
    )


def sdf_passes_for(na: int, nblocks: int, cta_slots: int) -> int:
    """csrc/mvs_internal.cuh sdf_passes_for: 256-vertex blocks per sdf_fused CTA (cta_slots = 3 x SM count)"""
    return 2 if na * nblocks > 2 * cta_slots else 1


def bookkeeping(model, model_type="smpllsp", joint_map=None, extra_vertex_ids=None) -> dict:
    """mvs_set_model's sizes: K, support vertices nsup, keypoint entries nkpe, (support vertex, joint) skinning pairs nsupj,
    skinning non-zeros per vertex KW"""
    W = np.asarray(model["weights"], dtype=np.float32)
    KW = max(1, int((W != 0).sum(1).max()))
    if model_type == "smpllsp":
        reg = np.asarray(model["lsp_regressor"], dtype=np.float32)
        n_first = reg.shape[0]
        jmap = S.JOINT_MAP_LSP14 if joint_map is None else joint_map
    else:
        reg, n_first = None, S.NUM_JOINTS
        jmap = S.JOINT_MAP_COCO17_SMPL if joint_map is None else joint_map
    extra = S.FACE_VERTEX_IDS if extra_vertex_ids is None else extra_vertex_ids
    vidx = []
    for src in np.asarray(jmap):
        if src < n_first:
            if reg is not None:
                vidx += [int(n) for n in np.flatnonzero(reg[src])]
        else:
            vidx.append(int(extra[src - n_first]))
    sup = np.unique(np.asarray(vidx, dtype=np.int64))
    return dict(K=len(jmap), nsup=len(sup), nkpe=len(vidx), nsupj=int((W[sup] != 0).sum()), KW=KW, sup=sup)


def branches(bk: dict, V: int, M: int, lim: dict | None = None) -> dict:
    """which side of each limit a model with bookkeeping bk, V views and M GMM components is on"""
    lim = lim or limits()
    resident = (bk["nsup"] + lim["kResExtraSup"] <= lim["kResMaxSup"] and bk["K"] <= lim["kMaxKeypoints"] and
                V * bk["K"] <= lim["kResMaxVK"] and M <= lim["kResMaxM"])
    return dict(resident=resident, kp_on=bk["nkpe"] <= lim["kResMaxKpE"], sj_on=bk["nsupj"] <= lim["kResMaxSupJ"],
                ell_smem=bk["KW"] <= lim["kSkinEllMax"])


# ------------------------------------------------------------------------------------------------------------ builders
def _grow_row(row, vt, add, frac, sigma):
    """a regressor row that keeps its own non-zeros (scaled by 1 - frac) and spreads frac over the vertices `add`, with
    Gaussian weights around the row's keypoint: non-negative, sums to 1, the keypoint moves by at most frac x the spread"""
    own = np.flatnonzero(row)
    centre = row[own].astype(np.float64) @ vt[own]
    d2 = ((vt[add] - centre) ** 2).sum(1)
    w = np.exp(-d2 / (2 * sigma ** 2)) + 1e-3          # the floor keeps every added entry non-zero in float32
    out = np.zeros_like(row, dtype=np.float64)
    out[own] = row[own] * (1.0 - frac)
    out[add] += frac * w / w.sum()
    return (out / out.sum()).astype(np.float32), centre


def _nearest_free(vt, centre, n, taken):
    order = np.argsort(((vt - centre) ** 2).sum(1), kind="stable")
    return np.array([i for i in order if i not in taken][:n], dtype=np.int64)


def _spread_new_vertices(reg, vt, n_new):
    """n_new vertices outside every used row's support and the face vertices, round-robin over the used rows, each the
    free vertex nearest that row's keypoint"""
    taken = set(int(v) for v in S.FACE_VERTEX_IDS) | set(int(v) for r in LSP_ROWS for v in np.flatnonzero(reg[r]))
    per_row = {r: [] for r in LSP_ROWS}
    for q in range(n_new):
        r = LSP_ROWS[q % len(LSP_ROWS)]
        own = np.flatnonzero(reg[r])
        v = int(_nearest_free(vt, reg[r, own].astype(np.float64) @ vt[own], 1, taken)[0])
        taken.add(v)
        per_row[r].append(v)
    return per_row


def regressor_with_support(model, nsup):
    """the LSP regressor with the used rows grown by disjoint new vertices: nsup = 5 face vertices + their non-zeros"""
    vt = np.asarray(model["v_template"], dtype=np.float64)
    reg = np.array(model["lsp_regressor"], dtype=np.float32, copy=True)
    now = bookkeeping(model)["nsup"]
    assert nsup >= now
    for r, add in _spread_new_vertices(reg, vt, nsup - now).items():
        if add:
            reg[r] = _grow_row(reg[r], vt, np.asarray(add), 0.2, 0.05)[0]
    return reg


def regressor_wide(model, per_row=22, pool_size=84):
    """every used row draws `per_row` non-zeros from one shared pool (the used rows' supports plus new vertices, pool_size
    in all): many keypoint entries (12 x 22 + 5 = 269) over few support vertices (5 + 84 = 89)"""
    vt = np.asarray(model["v_template"], dtype=np.float64)
    reg = np.array(model["lsp_regressor"], dtype=np.float32, copy=True)
    own = {r: set(int(v) for v in np.flatnonzero(reg[r])) for r in LSP_ROWS}
    pool = sorted(set().union(*own.values()))
    pool = np.asarray(pool + [v for a in _spread_new_vertices(reg, vt, pool_size - len(pool)).values() for v in a])
    for r in LSP_ROWS:
        o = np.flatnonzero(reg[r])
        centre = reg[r, o].astype(np.float64) @ vt[o]
        cand = np.array([v for v in pool if v not in own[r]])
        add = cand[np.argsort(((vt[cand] - centre) ** 2).sum(1), kind="stable")[:per_row - len(o)]]
        reg[r] = _grow_row(reg[r], vt, add, 0.1, 0.1)[0]
    return reg


def _skin_rows(model, verts, counts):
    """normalised skinning rows over the `counts` joints nearest each vertex (rest joints of the model's own regressor)"""
    vt = np.asarray(model["v_template"], dtype=np.float64)
    J = np.asarray(model["J_regressor"], dtype=np.float64) @ vt
    W = np.array(model["weights"], dtype=np.float32, copy=True)
    for n, k in zip(verts, counts):
        d2 = ((J - vt[n]) ** 2).sum(1)
        js = np.argsort(d2, kind="stable")[:k]
        w = np.exp(-(d2[js] - d2[js].min()) / (2 * 0.1 ** 2)) + 1e-3
        W[n] = 0.0
        W[n, js] = (w / w.sum()).astype(np.float32)
    return W


# ------------------------------------------------------------------------------------------------- meshes of other sizes
# N -> what the size reaches in the dense kernels (tests/test_model_sizes.py asserts each from tails() and limits())
SIZES = (431, 1723, 6890, 6912, 6913, 6944, 10475, 27554)


def make_sized_model(n_verts: int, seed: int = 0):
    """(model, extra_vertex_ids): a body model of n_verts vertices built the way synthetic.make_model builds its own (a
    Fibonacci sphere in height bands, its convex hull with F = 2N - 4 outward faces, J_regressor, <= 4 skinning weights per
    vertex, shapedirs and posedirs from the same draws; at 6890 and seed 0 all of these are make_model(0)'s).  Keypoints: every
    non-zero LSP regressor row of make_model(0) is rebuilt on the vertices nearest the point it regresses in the rest pose
    (as many as it has non-zeros, Gaussian weights, non-negative, sums to 1), and the 5 face keypoints become the vertices
    nearest make_model(0)'s face vertices."""
    from scipy.spatial import ConvexHull
    N, J = n_verts, S.NUM_JOINTS
    rng = np.random.RandomState(seed)
    pts = S._fibonacci_sphere(N)
    pts = pts + rng.normal(0.0, 2e-3, size=pts.shape)
    pts /= np.linalg.norm(pts, axis=1, keepdims=True)
    band = np.floor((pts[:, 1] + 1.0) * 20.0)
    pts = pts[np.lexsort((np.arctan2(pts[:, 2], pts[:, 0]), band))]
    vt = pts * np.array([0.25, 0.85, 0.15])
    faces = ConvexHull(pts).simplices.astype(np.int64)
    a, b, c = pts[faces[:, 0]], pts[faces[:, 1]], pts[faces[:, 2]]
    flip = np.einsum("ij,ij->i", np.cross(b - a, c - a), a + b + c) < 0
    faces[flip] = faces[flip][:, [0, 2, 1]]
    faces = faces[np.lexsort((faces[:, 2], faces[:, 1], faces[:, 0]))]
    assert faces.shape == (2 * N - 4, 3)
    d2 = ((vt[None, :, :] - S._skeleton_rest()[:, None, :]) ** 2).sum(-1)          # [24, N]
    Jreg = np.zeros((J, N))
    for j in range(J):
        idx = np.argsort(d2[j])[:64]
        w = np.exp(-(d2[j, idx] - d2[j, idx].min()) / (2 * 0.05 ** 2)) * rng.uniform(0.5, 1.0, size=64)
        Jreg[j, idx] = w / w.sum()
    weights = np.zeros((N, J))
    near = np.argsort(d2.T, axis=1)[:, :4]
    dn = np.take_along_axis(d2.T, near, axis=1)
    w = np.exp(-(dn - dn[:, :1]) / (2 * 0.06 ** 2))
    w[w < 1e-3] = 0.0
    w /= w.sum(1, keepdims=True)
    np.put_along_axis(weights, near, w, axis=1)
    shapedirs = rng.normal(0.0, 0.01, size=(N, 3, S.NUM_BETAS))
    posedirs = rng.normal(0.0, 0.001, size=(N, 3, S.NUM_POSE_BASIS)).astype(np.float32)
    kintree = np.zeros((2, J), dtype=np.uint32)
    kintree[0] = S.SMPL_PARENTS.astype(np.int64) % (2 ** 32)
    kintree[1] = np.arange(J)
    # keypoints where make_model(0)'s regress them in the rest pose
    base_vt = S.make_model(0, with_faces=False)["v_template"].astype(np.float64)
    base_reg = S.load_lsp_regressor().astype(np.float64)
    lsp = np.zeros((base_reg.shape[0], N), dtype=np.float64)
    for r in range(base_reg.shape[0]):
        own = np.flatnonzero(base_reg[r])
        if len(own) == 0:
            continue
        centre = base_reg[r, own] @ base_vt[own]
        dd = ((vt - centre) ** 2).sum(1)
        idx = np.argsort(dd, kind="stable")[:len(own)]
        w = np.exp(-(dd[idx] - dd[idx].min()) / (2 * 0.03 ** 2)) + 1e-3
        lsp[r, idx] = w / w.sum()
    extra = tuple(int(np.argmin(((vt - base_vt[v]) ** 2).sum(1))) for v in S.FACE_VERTEX_IDS)
    model = dict(v_template=vt.astype(np.float32), f=faces.astype(np.int32), shapedirs=shapedirs.astype(np.float32),
                 posedirs=posedirs, J_regressor=Jreg.astype(np.float32), kintree_table=kintree,
                 weights=weights.astype(np.float32), lsp_regressor=lsp.astype(np.float32))
    return model, extra


FACE18 = tuple(int(v) for v in S.FACE_VERTEX_IDS)
# 15 more single-vertex keypoints spread over the mesh, none of them in the LSP rows' support
EXTRA20 = FACE18 + (101, 555, 1010, 1500, 2020, 2500, 3030, 3500, 4040, 4500, 5050, 5500, 6060, 6500, 6800)
# K = 32: the 12 LSP rows and the 20 single-vertex keypoints, interleaved
JMAP32 = tuple(int(j) for j in np.random.RandomState(32).permutation(list(LSP_ROWS) + list(range(14, 34))))
# K = 18: the LSP set plus regressor row 12
JMAP18 = tuple(int(j) for j in S.JOINT_MAP_LSP14) + (12,)
KEYPOINT_SETS = dict(K18=dict(joint_map=JMAP18, extra_vertex_ids=FACE18),
                     K32=dict(joint_map=JMAP32, extra_vertex_ids=EXTRA20))


def make_variant(name, base):
    """the model dict of variant `name` (None: the base model itself)"""
    if name is None:
        return base
    m = dict(base)
    if name.startswith("sup"):
        m["lsp_regressor"] = regressor_with_support(base, int(name[3:]))
    elif name == "kpe_wide":
        m["lsp_regressor"] = regressor_wide(base)
    elif name == "skin_dense":
        sup = bookkeeping(base)["sup"]
        # 8 joints on most support vertices, 6 and 7 on some: > 512 (support vertex, joint) pairs and KW = 8
        m["weights"] = _skin_rows(base, sup, [6 if i % 10 == 0 else 7 if i % 10 == 5 else 8 for i in range(len(sup))])
    elif name == "skin_kw9":
        sup = set(int(v) for v in bookkeeping(base)["sup"])
        verts = [n for n in range(0, S.NUM_VERTS, 97) if n not in sup]
        m["weights"] = _skin_rows(base, verts, [9] * len(verts))
    else:
        raise KeyError(name)
    return m


def gmm_nll_min(gmm_f32, pose):
    """min over components of the GMM negative log-likelihood of `pose` (float64 over the float32 buffers the context
    uploads) and the component that attains it"""
    means, prec, nllw = gmm_f32
    d = np.asarray(pose, dtype=np.float64)[None, :] - means
    ll = 0.5 * np.einsum("mi,mij,mj->m", d, prec, d) - np.log(nllw)
    return float(ll.min()), int(ll.argmin())


def gmm_buffers_f32(gmm):
    """(means, precisions, nll_weights) exactly as FittingContext.set_gmm_from_dict rounds them, widened to float64"""
    means = gmm["means"].astype(np.float32)
    prec = np.stack([np.linalg.inv(c) for c in gmm["covars"].astype(np.float32)]).astype(np.float32)
    sqrdets = np.array([np.sqrt(np.linalg.det(c)) for c in gmm["covars"]])
    nllw = np.asarray(gmm["weights"] / ((2 * np.pi) ** (69 / 2.0) * (sqrdets / sqrdets.min()))).astype(np.float32)
    return means.astype(np.float64), prec.astype(np.float64), nllw.astype(np.float64)


ANGLE_IDX, ANGLE_SIGN = (52, 55, 9, 12), (1.0, -1.0, -1.0, -1.0)     # the bending prior's entries of body_pose


def prior_gates(pose, kind, bpw, bend, gmm_f32=None):
    """the two gated terms before their gates (fitting.py:330-350): pose prior (GMM min NLL or |theta|^2, x bpw^2) and the
    bending term"""
    pose = np.asarray(pose, dtype=np.float64)
    if kind == "gmm":
        pprior = gmm_nll_min(gmm_f32, pose)[0] * bpw ** 2
    else:
        pprior = float((pose ** 2).sum()) * bpw ** 2
    angle = bend * float(sum(np.exp(pose[i] * s) ** 2 for i, s in zip(ANGLE_IDX, ANGLE_SIGN)))
    return pprior, angle
