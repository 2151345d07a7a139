"""ctypes driver of tests/hostsim/closure_hostsim.cpp (test infrastructure only)."""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "_build", "libhostsim.so")


class HostLoss(ctypes.Structure):
    _fields_ = [("data_weight", ctypes.c_double), ("body_pose_weight", ctypes.c_double),
                ("shape_weight", ctypes.c_double), ("bending_prior_weight", ctypes.c_double),
                ("rho", ctypes.c_double), ("body_prior", ctypes.c_int), ("use_conf", ctypes.c_int),
                ("fix_shape", ctypes.c_int), ("M", ctypes.c_int)]


def _build():
    src = os.path.join(_HERE, "closure_hostsim.cpp")
    csrc = os.path.join(_HERE, "..", "..", "mvsmplfitting_b200", "csrc")
    hdrs = [os.path.join(csrc, n) for n in ("mvs_math.cuh", "mvs_init.cuh", "mvs_sdf_geom.cuh", "mvs_sdf_bins.cuh")]
    os.makedirs(os.path.dirname(_SO), exist_ok=True)
    if (not os.path.exists(_SO) or os.path.getmtime(_SO) < max(os.path.getmtime(q) for q in [src] + hdrs)):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-x", "c++",
                               "-o", _SO, src])
    return ctypes.CDLL(_SO)


def keypoint_lists(model, model_type):
    """(kp_ptr, kp_v, kp_w, kp_chain) for the 17 keypoints, as mvs_set_model builds them"""
    from mvsmplfitting_b200 import synthetic as S
    ptr, vv, ww, chain = [0], [], [], []
    if model_type == "smpllsp":
        jmap, nfirst = S.JOINT_MAP_LSP14, 14
    else:
        jmap, nfirst = S.JOINT_MAP_COCO17_SMPL, 24
    for src in jmap:
        c = -1
        if src < nfirst:
            if model_type == "smpllsp":
                nz = np.nonzero(model["lsp_regressor"][src])[0]
                vv += list(nz)
                ww += list(model["lsp_regressor"][src][nz])
            else:
                c = int(src)
        else:
            vv.append(int(S.FACE_VERTEX_IDS[src - nfirst]))
            ww.append(1.0)
        chain.append(c)
        ptr.append(len(vv))
    return (np.array(ptr, np.int32), np.array(vv, np.int32), np.array(ww, np.float64), np.array(chain, np.int32))


class HostSim:
    def __init__(self, model, cams, model_type="smpllsp"):
        self.lib = _build()
        self.lib.hostsim_create.restype = ctypes.c_void_p
        f64 = lambda a: np.ascontiguousarray(a, dtype=np.float64)
        N = model["v_template"].shape[0]
        pd = f64(np.reshape(model["posedirs"], [-1, 207]).T)
        parents = np.asarray(model["kintree_table"][0]).astype(np.int64)
        parents[0] = -1
        parents = parents.astype(np.int32)
        ptr, vv, ww, chain = keypoint_lists(model, model_type)
        self.K, self.V, self.N = len(chain), cams["R"].shape[0], N
        arrs = [f64(model["v_template"]), f64(model["shapedirs"]), pd, f64(model["J_regressor"]), parents,
                f64(model["weights"]), ptr, vv, ww, chain, f64(cams["R"]), f64(cams["t"]), f64(cams["f"]), f64(cams["c"])]
        self._keep = arrs
        p = [a.ctypes.data_as(ctypes.c_void_p) for a in arrs]
        self.h = ctypes.c_void_p(self.lib.hostsim_create(
            N, p[0], p[1], p[2], p[3], p[4], p[5], self.K, p[6], p[7], p[8], p[9], self.V, p[10], p[11], p[12], p[13]))

    def eval(self, x86, gt_uv, conf, jw, w, body_prior="l2", gmm=None, use_conf=True, fix_shape=False,
             use_double=False, rho=100.0, want_verts=False):
        from mvsmplfitting_b200 import synthetic as S
        lp = HostLoss(w["data_weight"], w["body_pose_weight"], w["shape_weight"], w["bending_prior_weight"], rho,
                      1 if body_prior == "gmm" else 0, int(use_conf), int(fix_shape), 0)
        gm = gp = gl = np.zeros(1)
        if body_prior == "gmm":
            means, prec, nllw = S.gmm_buffers(gmm)
            if not use_double:   # the reference holds these buffers in fp32 (prior.py:142-160)
                means = means.astype(np.float32).astype(np.float64)
                prec = np.stack([np.linalg.inv(c) for c in gmm["covars"].astype(np.float32)]).astype(np.float32).astype(np.float64)
                nllw = nllw.astype(np.float32).astype(np.float64)
            prec = 0.5 * (prec + np.transpose(prec, (0, 2, 1)))
            gm, gp, gl = np.ascontiguousarray(means), np.ascontiguousarray(prec), np.ascontiguousarray(np.log(nllw))
            lp.M = means.shape[0]
        f64 = lambda a: np.ascontiguousarray(a, dtype=np.float64)
        x, gt, cf, jw_ = f64(x86), f64(gt_uv), f64(conf), f64(jw)
        loss = np.zeros(1)
        grad = np.zeros(86)
        joints = np.zeros((self.K, 3))
        verts = np.zeros((self.N, 3)) if want_verts else None
        P = lambda a: a.ctypes.data_as(ctypes.c_void_p)
        self.lib.hostsim_eval(self.h, int(use_double), ctypes.byref(lp), P(gm), P(gp), P(gl), P(x), P(gt), P(cf), P(jw_),
                              P(loss), P(grad), P(joints), P(verts) if want_verts else None)
        out = dict(loss=float(loss[0]), grad=grad, joints=joints)
        if want_verts:
            out["verts"] = verts
        return out

    def __del__(self):
        try:
            self.lib.hostsim_destroy(self.h)
        except Exception:
            pass


def cont6d_to_aa(o6, daa, use_double=True):
    """mvs_math.cuh cont6d_to_aa_fwd/_bwd run on the host: returns (aa [n,3], (d aa/d o)^T daa [n,6], branch [n])"""
    lib = _build()
    o6 = np.ascontiguousarray(o6, dtype=np.float64).reshape(-1, 6)
    daa = np.ascontiguousarray(daa, dtype=np.float64).reshape(-1, 3)
    n = o6.shape[0]
    aa, d_o, br = np.zeros((n, 3)), np.zeros((n, 6)), np.zeros(n, np.int32)
    P = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    lib.hostsim_cont6d(ctypes.c_int(n), ctypes.c_int(int(use_double)), P(o6), P(daa), P(aa), P(d_o), P(br))
    return aa, d_o, br


def _P(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def triangulate(cams, uv, conf, use_double=True):
    """mvs_init.cuh triangulate_point on the host.  cams dict (R [V,3,3], t, f, c), uv [V,K,2], conf [V,K] -> [K,3]"""
    lib = _build()
    f64 = lambda a: np.ascontiguousarray(a, dtype=np.float64)
    uv = np.ascontiguousarray(uv, dtype=np.float32)
    conf = np.ascontiguousarray(conf, dtype=np.float32)
    V, K = conf.shape
    X = np.zeros((K, 3))
    R, t, f, c = f64(cams["R"]), f64(cams["t"]), f64(cams["f"]), f64(cams["c"])
    lib.hostsim_triangulate(ctypes.c_int(V), ctypes.c_int(K), _P(R), _P(t), _P(f), _P(c), _P(uv), _P(conf),
                            ctypes.c_int(int(use_double)), _P(X))
    return X


def umeyama(src, dst, estimate_scale, use_double=True, as_written=False):
    """mvs_init.cuh umeyama_fit + rotmat_to_aa on the host -> (R [3,3], t [3], scale, aa [3]) or None if degenerate"""
    lib = _build()
    src = np.ascontiguousarray(src, dtype=np.float64)
    dst = np.ascontiguousarray(dst, dtype=np.float64)
    R, t, s, aa = np.zeros(9), np.zeros(3), np.zeros(1), np.zeros(3)
    lib.hostsim_umeyama.restype = ctypes.c_int
    ok = lib.hostsim_umeyama(ctypes.c_int(src.shape[0]), _P(src), _P(dst), ctypes.c_int(int(estimate_scale)),
                             ctypes.c_int(int(use_double)), _P(R), _P(t), _P(s), _P(aa), ctypes.c_int(int(as_written)))
    return (R.reshape(3, 3), t, float(s[0]), aa) if ok else None


def single_view_joints(cam, rest, uv, conf):
    """mvs_init.cuh single_view_depth on the host: cam dict of ONE view (R [3,3], t, f, c), rest [K,3] -> joints3d [K,3]"""
    lib = _build()
    rest = np.ascontiguousarray(rest, dtype=np.float64)
    uv = np.ascontiguousarray(uv, dtype=np.float32)
    conf = np.ascontiguousarray(conf, dtype=np.float32)
    R, t, f, c = (np.ascontiguousarray(np.asarray(cam[k], dtype=np.float32), dtype=np.float64) for k in ("R", "t", "f", "c"))
    X = np.zeros((rest.shape[0], 3))
    lib.hostsim_single_view(ctypes.c_int(rest.shape[0]), _P(R), _P(t), _P(f), _P(c), _P(rest), _P(uv), _P(conf), _P(X))
    return X


def rotmat_to_aa(R):
    lib = _build()
    R = np.ascontiguousarray(R, dtype=np.float64).reshape(-1, 9)
    aa = np.zeros((R.shape[0], 3))
    lib.hostsim_rotmat_to_aa(ctypes.c_int(R.shape[0]), _P(R), _P(aa))
    return aa


def sdf_bin_entries(tri):
    """the entry counts of mvs_sdf_bins.cuh's candidate lists for tri [F,3,3] float32 box coordinates, and which capacity they
    exceed: (cell_entries, ray_entries, rc) with rc 0 (both fit), 1 (kBinCapD) or 2 (kBinCapR)"""
    lib = _build()
    tri = np.ascontiguousarray(tri, dtype=np.float32).reshape(-1, 9)
    ev = np.zeros(4, np.int64)
    lib.hostsim_sdf_bins.restype = ctypes.c_int
    rc = lib.hostsim_sdf_bins(ctypes.c_int(tri.shape[0]), _P(tri), ctypes.c_int(16), ctypes.c_long(0), None, None, None, _P(ev))
    return int(ev[2]), int(ev[3]), int(rc)


def sdf_bins(tri, G, voxel_ids, brute=True):
    """mvs_sdf_bins.cuh on the host: tri [F,3,3] float32 box coordinates -> (phi over candidate lists, phi by brute force or None,
    dict(ray_evals, dist_evals, cell_entries, ray_entries))"""
    lib = _build()
    tri = np.ascontiguousarray(tri, dtype=np.float32).reshape(-1, 9)
    vox = np.ascontiguousarray(voxel_ids, dtype=np.int64)
    ob, of = np.zeros(vox.shape[0], np.float32), np.zeros(vox.shape[0], np.float32)
    ev = np.zeros(4, np.int64)
    lib.hostsim_sdf_bins.restype = ctypes.c_int
    rc = lib.hostsim_sdf_bins(ctypes.c_int(tri.shape[0]), _P(tri), ctypes.c_int(int(G)), ctypes.c_long(vox.shape[0]), _P(vox), _P(ob),
                              _P(of) if brute else None, _P(ev))
    assert rc == 0, "list capacity exceeded (%d)" % rc
    return ob, (of if brute else None), dict(ray_evals=int(ev[0]), dist_evals=int(ev[1]), cell_entries=int(ev[2]), ray_entries=int(ev[3]))
