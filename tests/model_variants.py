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
    """the kernels' envelope constants, read from the CUDA headers"""
    out = {}
    for f in ("mvs_resident_dev.cuh", "mvs_tc_dev.cuh", "mvs_math.cuh"):
        src = open(os.path.join(CSRC, f)).read()
        for k, v in re.findall(r"constexpr\s+int\s+(k\w+)\s*=\s*(\d+)\s*;", src):
            out[k] = int(v)
    m = re.search(r"m\.nsup\s*\+\s*(\d+)\s*<=\s*kResMaxSup", open(os.path.join(CSRC, "mvs_resident.cu")).read())
    out["kResExtraSup"] = int(m.group(1))          # resident_supported(): room for the box-extreme vertices
    return out


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
