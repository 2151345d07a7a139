"""Python face of one libmvsmpl context (one per GPU / process).

PyTorch is used only as the owner of device memory and streams; every computation
on the path goes through the C ABI in include/mvsmpl.h.
"""
from __future__ import annotations

import ctypes

import numpy as np
import torch

from . import _lib
from . import synthetic as S

PRIOR_CODES = {"l2": 0, "gmm": 1, "none": 2, None: 2}
SEGMENT_BITS = {"betas": 0, "global_orient": 1, "body_pose": 2, "transl": 3, "scale": 4}


def _f32(a):
    return np.ascontiguousarray(np.asarray(a), dtype=np.float32)


def _i32(a):
    return np.ascontiguousarray(np.asarray(a), dtype=np.int32)


def _ptr(a):
    if a is None:
        return None
    if isinstance(a, torch.Tensor):
        return ctypes.c_void_p(a.data_ptr())
    return a.ctypes.data_as(ctypes.c_void_p)


def _temporal_weight(w) -> np.ndarray:
    """a temporal weight as the C ABI takes it: 86 host float32 (checked there)"""
    w = _f32(w.cpu() if isinstance(w, torch.Tensor) else w).reshape(-1)
    if w.shape[0] != S.NUM_PARAMS:
        raise ValueError("temporal_weight: want %d entries, got %d" % (S.NUM_PARAMS, w.shape[0]))
    return w


def _stats_dict(st) -> dict:
    return dict(frame_iterations=st.frame_iterations, frame_evals=st.frame_evals, rounds=st.rounds, frames_nan=st.frames_nan,
                dense_frame_evals=st.dense_frame_evals, dense_rounds=st.dense_rounds)


class FittingContext:
    """Owns the device copies of the model / cameras / detections and launches the closure
    and the batched L-BFGS.  All tensors passed in must live on `device` and be contiguous fp32."""

    def __init__(self, device: int | torch.device = 0):
        self.lib = _lib.load()
        if not torch.cuda.is_available():
            raise _lib.MvsError("no CUDA device visible: mvsmplfitting_b200 has no CPU fallback")
        self.device = torch.device("cuda", device if isinstance(device, int) else (device.index or 0))
        h = ctypes.c_void_p()
        _lib.check(None, self.lib.mvs_create(self.device.index, ctypes.byref(h)), "mvs_create")
        self.h = h
        self.B = 0
        self.V = 0                        # view rows of every detection array: the rigs' largest view count
        self.rig_views = []               # view count of each camera rig
        self.K = 17
        self.N = 0
        self._loss_cfg = None
        self._j3d_keep = None             # the 3-D targets while the term is on (set_joints3d)
        self._rigs = []                   # the camera table as set: dict(R, t, f, c) float32 per rig (refine_cameras updates R, t)

    def close(self):
        if getattr(self, "h", None):
            self.lib.mvs_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ------------------------------------------------------------------ uploads
    def set_model(self, model: dict, model_type: str = "smpllsp", joint_map=None, extra_vertex_ids=None):
        """`model` holds the reference's data_struct fields (v_template, shapedirs, posedirs [N,3,207],
        J_regressor, kintree_table, weights, f) plus `lsp_regressor` for model_type 'smpllsp'."""
        N = model["v_template"].shape[0]
        posedirs = np.asarray(model["posedirs"])
        if posedirs.ndim == 3:                      # [N,3,207] -> the registered [207, 3N] layout
            posedirs = np.reshape(posedirs, [-1, posedirs.shape[-1]]).T
        parents = np.asarray(model["kintree_table"][0]).astype(np.int64) if "kintree_table" in model \
            else np.asarray(model["parents"]).astype(np.int64)
        parents = parents.copy()
        parents[0] = -1
        if model_type == "smpllsp":
            reg = _f32(model["lsp_regressor"])
            n_reg = reg.shape[0]
            jmap = S.JOINT_MAP_LSP14 if joint_map is None else joint_map
        else:
            reg, n_reg = None, 0
            jmap = S.JOINT_MAP_COCO17_SMPL if joint_map is None else joint_map
        extra = _i32(S.FACE_VERTEX_IDS if extra_vertex_ids is None else extra_vertex_ids)
        faces = _i32(model["f"]) if model.get("f") is not None else None
        keep = dict(vt=_f32(model["v_template"]), sd=_f32(model["shapedirs"]), pd=_f32(posedirs),
                    jr=_f32(model["J_regressor"]), par=_i32(parents), w=_f32(model["weights"]), faces=faces,
                    reg=reg, extra=extra, jmap=_i32(jmap))
        d = _lib.ModelDesc(
            n_verts=N, n_faces=0 if faces is None else faces.shape[0],
            v_template=_ptr(keep["vt"]), shapedirs=_ptr(keep["sd"]), posedirs=_ptr(keep["pd"]),
            J_regressor=_ptr(keep["jr"]), parents=_ptr(keep["par"]), lbs_weights=_ptr(keep["w"]),
            faces=_ptr(faces), n_keypoints=len(keep["jmap"]), n_reg=n_reg, joint_regressor=_ptr(reg),
            n_extra=len(extra), extra_vertex_ids=_ptr(extra), joint_map=_ptr(keep["jmap"]))
        _lib.check(self.h, self.lib.mvs_set_model(self.h, ctypes.byref(d)), "mvs_set_model")
        self.N, self.K = N, len(keep["jmap"])
        self.model_type = model_type

    def set_gmm(self, means, precisions, nll_weights):
        m, p, w = _f32(means), _f32(precisions), _f32(np.reshape(nll_weights, -1))
        _lib.check(self.h, self.lib.mvs_set_gmm_prior(self.h, m.shape[0], _ptr(m), _ptr(p), _ptr(w)), "mvs_set_gmm_prior")

    def set_gmm_from_dict(self, gmm: dict):
        """same float32 buffer path as the reference (prior.py:127-160)"""
        means = gmm["means"].astype(np.float32)
        covs = gmm["covars"].astype(np.float32)
        prec = np.stack([np.linalg.inv(c) for c in covs]).astype(np.float32)
        sqrdets = np.array([np.sqrt(np.linalg.det(c)) for c in gmm["covars"]])
        nllw = np.asarray(gmm["weights"] / ((2 * np.pi) ** (69 / 2.0) * (sqrdets / sqrdets.min())))
        self.set_gmm(means, prec, nllw.astype(np.float32))

    def set_vposer(self, weights: dict):
        """VPoser decoder weights (mvs_set_vposer): dict(fc1_w [512,32], fc1_b, fc2_w [512,512], fc2_b, out_w [138,512],
        out_b) -- e.g. the bodyprior_dec_* tensors of a loaded VPoser, or synthetic.make_vposer().  Enables
        use_vposer=2 loss configurations (pose decoded on the device from the latent code in the pose slot)."""
        arrs = [_f32(weights[k]) for k in ("fc1_w", "fc1_b", "fc2_w", "fc2_b", "out_w", "out_b")]
        assert arrs[0].shape == (512, 32) and arrs[2].shape == (512, 512) and arrs[4].shape == (138, 512)
        _lib.check(self.h, self.lib.mvs_set_vposer(self.h, *[_ptr(a) for a in arrs]), "mvs_set_vposer")

    def vposer_decode(self, params: torch.Tensor) -> torch.Tensor:
        """vposer.decode(z, 'aa') of the latent codes in params[:, 13:45] (mvs_vposer_decode) -> body_pose [B,69]"""
        assert params.is_cuda and params.dtype == torch.float32 and params.is_contiguous() and params.shape == (self.B, 86)
        out = torch.empty(self.B, 69, dtype=torch.float32, device=self.device)
        _lib.check(self.h, self.lib.mvs_vposer_decode(self.h, _ptr(params), _ptr(out), self._stream()), "mvs_vposer_decode")
        return out

    def set_cameras(self, R, t, f, c, dist=None):
        """One rig of V views (mvs_set_cameras); dist [V,5] OpenCV coefficients (k1, k2, p1, p2, k3) per view or None (none)"""
        if dist is not None:
            return self.set_camera_rigs([dict(R=R, t=t, f=f, c=c, dist=dist)])
        R, t, f, c = _f32(R), _f32(t), _f32(f), _f32(c)
        self.V = R.shape[0]
        _lib.check(self.h, self.lib.mvs_set_cameras(self.h, self.V, _ptr(R), _ptr(t), _ptr(f), _ptr(c)), "mvs_set_cameras")
        self.rig_views = [self.V]
        self._rigs = [dict(R=R.copy(), t=t.copy(), f=f.copy(), c=c.copy())]

    def set_camera_rigs(self, rigs, data_weight_scale=None):
        """A table of camera rigs (mvs_set_camera_rigs): rigs is a list of dict(R [V_r,3,3], t [V_r,3], f [V_r,2], c [V_r,2])
        such as seqio.camera_arrays returns; data_weight_scale [n_rigs] multiplies every stage's data_weight for the frames
        of each rig (None: all 1).  Detection arrays then have V = max V_r view rows; rows v >= V_r of a frame with rig r are
        not read.  Name each slot's rig with set_frame_rigs, or each frame's with fit_stream / fit_seq_stream(rig=...).
        A rig dict may carry "dist" [V_r,5]: its views' lens distortion, OpenCV's (k1, k2, p1, p2, k3)
        (mvs_set_camera_rigs_dist); a rig without it has none."""
        if not rigs:
            raise ValueError("set_camera_rigs: want at least one rig")
        nv = [int(np.asarray(r["R"]).shape[0]) for r in rigs]
        V = max(nv)
        pad = lambda a, n, shape: np.concatenate([_f32(a), np.zeros((V - n,) + shape, np.float32)]) if n < V else _f32(a)
        R = _f32(np.stack([pad(r["R"], n, (3, 3)) for r, n in zip(rigs, nv)]))
        t = _f32(np.stack([pad(r["t"], n, (3,)) for r, n in zip(rigs, nv)]))
        f = _f32(np.stack([pad(r["f"], n, (2,)) for r, n in zip(rigs, nv)]))
        c = _f32(np.stack([pad(r["c"], n, (2,)) for r, n in zip(rigs, nv)]))
        scale = None if data_weight_scale is None else _f32(np.reshape(data_weight_scale, -1))
        if scale is not None and scale.shape[0] != len(rigs):
            raise ValueError("set_camera_rigs: %d rigs, %d data-weight scales" % (len(rigs), scale.shape[0]))
        nva = _i32(nv)
        has_dist = [r.get("dist") is not None for r in rigs]
        if any(has_dist):
            for i, (r, n) in enumerate(zip(rigs, nv)):
                if r.get("dist") is not None and np.shape(r["dist"]) != (n, 5):
                    raise ValueError("set_camera_rigs: rig %d has %d views, dist of shape %s (want [%d,5])"
                                     % (i, n, np.shape(r["dist"]), n))
            dist = _f32(np.stack([pad(r["dist"] if h else np.zeros((n, 5)), n, (5,)) for r, n, h in zip(rigs, nv, has_dist)]))
            _lib.check(self.h, self.lib.mvs_set_camera_rigs_dist(self.h, len(rigs), _ptr(nva), _ptr(R), _ptr(t), _ptr(f), _ptr(c),
                                                                 _ptr(dist), _ptr(scale)), "mvs_set_camera_rigs_dist")
        else:
            _lib.check(self.h, self.lib.mvs_set_camera_rigs(self.h, len(rigs), _ptr(nva), _ptr(R), _ptr(t), _ptr(f), _ptr(c),
                                                            _ptr(scale)), "mvs_set_camera_rigs")
        self.V, self.rig_views = V, nv
        self._rigs = [dict(R=R[r, :n].copy(), t=t[r, :n].copy(), f=f[r, :n].copy(), c=c[r, :n].copy()) for r, n in enumerate(nv)]
        for r, h in enumerate(has_dist):
            if h:
                self._rigs[r]["dist"] = dist[r, :nv[r]].copy()

    def set_frame_rigs(self, rig):
        """the rig of every slot of the batch (mvs_set_frame_rigs): rig [B] ints in [0, n_rigs)"""
        r = _i32(np.reshape(rig, -1))
        if r.shape[0] != self.B:
            raise ValueError("set_frame_rigs: want %d rig indices, got %d" % (self.B, r.shape[0]))
        _lib.check(self.h, self.lib.mvs_set_frame_rigs(self.h, _ptr(r)), "mvs_set_frame_rigs")

    def set_batch(self, B: int):
        _lib.check(self.h, self.lib.mvs_set_batch(self.h, int(B)), "mvs_set_batch")
        self.B = int(B)

    def _stream(self):
        return ctypes.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def set_keypoints(self, gt_uv, conf, joint_weights):
        """gt_uv [V,B,K,2], conf [V,B,K], joint_weights [K]; numpy (host) or CUDA tensors."""
        on_dev = isinstance(gt_uv, torch.Tensor) and gt_uv.is_cuda
        if on_dev:
            gt_uv = gt_uv.contiguous().float()
            conf = conf.to(self.device).contiguous().float()
            joint_weights = torch.as_tensor(joint_weights).to(self.device).contiguous().float().reshape(-1)
        else:
            gt_uv, conf, joint_weights = _f32(gt_uv), _f32(conf), _f32(np.reshape(joint_weights, -1))
        assert tuple(gt_uv.shape) == (self.V, self.B, self.K, 2), (tuple(gt_uv.shape), (self.V, self.B, self.K, 2))
        assert tuple(conf.shape) == (self.V, self.B, self.K)
        self._kp_keep = (gt_uv, conf, joint_weights)
        _lib.check(self.h, self.lib.mvs_set_keypoints(self.h, _ptr(gt_uv), _ptr(conf), _ptr(joint_weights),
                                                      1 if on_dev else 0, self._stream()), "mvs_set_keypoints")

    @staticmethod
    def make_loss_config(data_weight=1.0, body_pose_weight=0.0, shape_weight=0.0, bending_prior_weight=0.0,
                         coll_loss_weight=0.0, rho=100.0, body_prior="l2", use_joints_conf=True, use_vposer=False,
                         fix_shape=False, interpenetration=False, sdf_grid=128, sdf_all_faces=False,
                         frozen=()) -> _lib.LossConfig:
        mask = 0
        for name in frozen:
            mask |= 1 << SEGMENT_BITS[name]
        return _lib.LossConfig(float(data_weight), float(body_pose_weight), float(shape_weight),
                               float(bending_prior_weight), float(coll_loss_weight), float(rho),
                               PRIOR_CODES[body_prior], int(use_joints_conf), int(use_vposer), int(fix_shape),
                               int(interpenetration), int(sdf_grid), int(sdf_all_faces), mask)

    def set_loss(self, **kw):
        cfg = kw.pop("config", None) or self.make_loss_config(**kw)
        _lib.check(self.h, self.lib.mvs_set_loss_config(self.h, ctypes.byref(cfg)), "mvs_set_loss_config")
        self._loss_cfg = cfg

    # ------------------------------------------------------------------ compute
    def closure(self, params: torch.Tensor, want_grad=True, want_joints=False, want_proj=False, want_verts=False):
        """One batched fitting_func(): params [B,86] (CUDA fp32) -> dict(loss [B], grad [B,86], ...)."""
        assert params.is_cuda and params.dtype == torch.float32 and params.is_contiguous()
        assert tuple(params.shape) == (self.B, S.NUM_PARAMS)
        new = lambda *s: torch.empty(*s, dtype=torch.float32, device=self.device)
        out = dict(loss=new(self.B))
        if want_grad:
            out["grad"] = new(self.B, S.NUM_PARAMS)
        if want_joints:
            out["joints"] = new(self.B, self.K, 3)
        if want_proj:
            out["proj"] = new(self.V, self.B, self.K, 2)
        if want_verts:
            out["verts"] = new(self.B, self.N, 3)
        _lib.check(self.h, self.lib.mvs_closure(self.h, _ptr(params), _ptr(out["loss"]), _ptr(out.get("grad")),
                                                _ptr(out.get("joints")), _ptr(out.get("proj")), _ptr(out.get("verts")),
                                                self._stream()), "mvs_closure")
        return out

    def forward_only(self, params: torch.Tensor, want_verts: bool = True):
        """SMPL.forward outside the closure: dict(joints [B,K,3], verts [B,N,3])"""
        assert params.is_cuda and params.dtype == torch.float32 and params.is_contiguous()
        out = dict(joints=torch.empty(self.B, self.K, 3, dtype=torch.float32, device=self.device))
        if want_verts:
            out["verts"] = torch.empty(self.B, self.N, 3, dtype=torch.float32, device=self.device)
        _lib.check(self.h, self.lib.mvs_forward(self.h, _ptr(params), _ptr(out["joints"]), _ptr(out.get("verts")),
                                                self._stream()), "mvs_forward")
        return out

    def forward_vjp(self, params: torch.Tensor, djoints: torch.Tensor | None = None,
                    dverts: torch.Tensor | None = None) -> torch.Tensor:
        """Vector-Jacobian product of forward_only (mvs_forward_vjp): dparams [B,86] = d<djoints, joints> + d<dverts, verts>
        with respect to params [B,86] (body_pose as axis-angle).  djoints [B,K,3] and dverts [B,N,3] may each be None, not
        both; every tensor is float32 on this context's device."""
        def check(name, t, shape):
            if not isinstance(t, torch.Tensor) or t.dtype != torch.float32 or t.device != self.device or tuple(t.shape) != shape:
                raise ValueError("forward_vjp: want %s as a float32 tensor of shape %s on %s, got %s" % (
                    name, shape, self.device, (t.dtype, tuple(t.shape), t.device) if isinstance(t, torch.Tensor) else type(t)))
            return t.contiguous()
        if djoints is None and dverts is None:
            raise ValueError("forward_vjp: give djoints, dverts or both")
        params = check("params", params, (self.B, S.NUM_PARAMS))
        djoints = None if djoints is None else check("djoints", djoints, (self.B, self.K, 3))
        dverts = None if dverts is None else check("dverts", dverts, (self.B, self.N, 3))
        out = torch.empty(self.B, S.NUM_PARAMS, dtype=torch.float32, device=self.device)
        _lib.check(self.h, self.lib.mvs_forward_vjp(self.h, _ptr(params), _ptr(djoints), _ptr(dverts), _ptr(out),
                                                    self._stream()), "mvs_forward_vjp")
        return out

    @staticmethod
    def make_lbfgs_config(max_outer=30, max_iter=30, max_eval=None, history_size=100, lr=1.0, tolerance_grad=1e-5,
                          tolerance_change=1e-9, ftol=1e-9, gtol=1e-9) -> _lib.LbfgsConfig:
        return _lib.LbfgsConfig(int(max_outer), int(max_iter), int(max_eval if max_eval is not None else max_iter * 5 // 4),
                                int(history_size), float(lr), float(tolerance_grad), float(tolerance_change),
                                float(ftol), float(gtol))

    def lbfgs_run(self, params: torch.Tensor, config: _lib.LbfgsConfig | None = None):
        """Runs FittingMonitor.run_fitting for every frame on the device; params updated in place.
        Returns (final_loss [B] tensor, stats dict)."""
        assert params.is_cuda and params.dtype == torch.float32 and params.is_contiguous()
        cfg = config or self.make_lbfgs_config()
        final = torch.empty(self.B, dtype=torch.float32, device=self.device)
        st = _lib.LbfgsStats()
        _lib.check(self.h, self.lib.mvs_lbfgs_run(self.h, _ptr(params), _ptr(final), ctypes.byref(cfg), ctypes.byref(st),
                                                  self._stream()), "mvs_lbfgs_run")
        return final, _stats_dict(st)

    def lbfgs_step(self, params: torch.Tensor, config=None, reset: bool = False):
        """one LBFGS.step() for every frame; returns (loss at entry [B], grads of the last closure call [B,86], stats)"""
        assert params.is_cuda and params.dtype == torch.float32 and params.is_contiguous()
        cfg = config or self.make_lbfgs_config()
        loss = torch.empty(self.B, dtype=torch.float32, device=self.device)
        grad = torch.empty(self.B, S.NUM_PARAMS, dtype=torch.float32, device=self.device)
        st = _lib.LbfgsStats()
        _lib.check(self.h, self.lib.mvs_lbfgs_step(self.h, _ptr(params), _ptr(loss), _ptr(grad), ctypes.byref(cfg),
                                                   1 if reset else 0, ctypes.byref(st), self._stream()), "mvs_lbfgs_step")
        return loss, grad, _stats_dict(st)

    def init_guess(self, estimate_scale: bool = True, fixed_scale: float = 1.0, use_torso: bool = True,
                   hip_seed: float = 1.0, want_joints3d: bool = True, umeyama_as_written: bool = False):
        """Initial parameter block of every frame from the uploaded detections (mvs_init_guess: triangulation -- or the
        single-view depth guess, or the 3-D targets of set_joints3d while they are on -- + similarity alignment,
        init_guess.py:18-107 + fix_params :190-212).
        umeyama_as_written: evaluate code/utils/umeyama.py as written (see include/mvsmpl.h) instead of the published
        algorithm.  Returns (params [B,86], joints3d [B,K,3])."""
        params = torch.empty(self.B, 86, dtype=torch.float32, device=self.device)
        j3 = torch.empty(self.B, self.K, 3, dtype=torch.float32, device=self.device) if want_joints3d else None
        cfg = _lib.InitConfig(int(bool(estimate_scale)), float(fixed_scale), int(bool(use_torso)), float(hip_seed),
                              int(bool(umeyama_as_written)))
        _lib.check(self.h, self.lib.mvs_init_guess(self.h, _ptr(params), _ptr(j3), ctypes.byref(cfg), self._stream()),
                   "mvs_init_guess")
        return params, j3

    def fit(self, params: torch.Tensor, stage_cfgs, opt_cfg=None, warm=None, prev=None, temporal_weight=None):
        """All stages of a fit on device buffers (mvs_fit): params [B,86] CUDA float32, updated in place.  Frames move
        from stage to stage on their own; returns (final_loss [B], stats).  warm [B] bool (mvs_fit_seq): frames that
        continue a video sequence from the previous frame's result skip stages 0, 1 and damp stage 2's pose prior
        (non_linear_solver.py:157-162).  temporal_weight [86] (mvs_fit_seq_temporal, needs warm and prev [B,86] CUDA float32,
        the previous frames' fitted rows): every warm frame's stages add sum_i w_i (x_i - prev_i)^2."""
        assert params.is_cuda and params.dtype == torch.float32 and params.is_contiguous()
        arr = (_lib.LossConfig * len(stage_cfgs))(*stage_cfgs)
        cfg = opt_cfg or self.make_lbfgs_config()
        final = torch.empty(self.B, dtype=torch.float32, device=self.device)
        st = _lib.LbfgsStats()
        tw = None
        if temporal_weight is not None:
            if warm is None or prev is None:
                raise ValueError("fit: temporal_weight needs warm and prev")
            assert prev.is_cuda and prev.dtype == torch.float32 and prev.is_contiguous() and tuple(prev.shape) == (self.B, 86)
            tw = _temporal_weight(temporal_weight)
        wm = None if warm is None else np.ascontiguousarray(np.asarray(warm).astype(np.uint8).reshape(self.B))
        _lib.check(self.h, self.lib.mvs_fit_seq_temporal(self.h, _ptr(params), len(stage_cfgs), arr, ctypes.byref(cfg), _ptr(wm),
                                                         _ptr(prev if tw is not None else None), _ptr(tw), _ptr(final),
                                                         ctypes.byref(st), self._stream()), "mvs_fit_seq_temporal")
        return final, _stats_dict(st)

    def _stream_rows(self, who, F, gt_uv, conf, joint_weights, joints3d, conf3d):
        """A stream's per-frame rows on the device, checked against F frames: gt_uv [V,F,K,2], conf [V,F,K], joint_weights
        [K], and joints3d [F,K,3] with conf3d [F,K] or neither (None, None).  who: the public method, for the errors."""
        dev = lambda a: None if a is None else torch.as_tensor(a).to(self.device, torch.float32).contiguous()
        gt_uv, conf, jw = dev(gt_uv), dev(conf), dev(joint_weights).reshape(-1)
        assert tuple(gt_uv.shape) == (self.V, F, self.K, 2) and tuple(conf.shape) == (self.V, F, self.K), \
            (tuple(gt_uv.shape), tuple(conf.shape), (self.V, F, self.K))
        if (joints3d is None) != (conf3d is None):
            raise ValueError("%s: joints3d and conf3d go together" % who)
        j3, c3 = dev(joints3d), dev(conf3d)
        if j3 is not None and (tuple(j3.shape) != (F, self.K, 3) or tuple(c3.shape) != (F, self.K)):
            raise ValueError("%s: want joints3d [%d,%d,3] and conf3d [%d,%d], got %s and %s"
                             % (who, F, self.K, F, self.K, tuple(j3.shape), tuple(c3.shape)))
        return gt_uv, conf, jw, j3, c3

    def _stream_rigs(self, who, F, rig):
        """a stream's per-frame rig indices [F] on the device (int32), or None"""
        if rig is None:
            return None
        r = torch.as_tensor(np.asarray(rig.cpu() if isinstance(rig, torch.Tensor) else rig).astype(np.int32).reshape(-1))
        if r.shape[0] != F:
            raise ValueError("%s: want %d rig indices, got %d" % (who, F, r.shape[0]))
        return r.to(self.device).contiguous()

    def fit_stream(self, params: torch.Tensor, gt_uv, conf, joint_weights, stage_cfgs, opt_cfg=None, joints3d=None,
                   conf3d=None, rig=None):
        """mvs_fit over F frames of any number through the context's B slots (mvs_fit_stream): params [F,86] CUDA float32,
        updated in place; gt_uv [V,F,K,2], conf [V,F,K], joint_weights [K] (numpy or tensors); joints3d [F,K,3] with conf3d
        [F,K] switch the 3-D joint term on for this call.  rig [F] (mvs_fit_stream_rigs) names each frame's camera rig
        (set_camera_rigs; None: rig 0, one rig only).  Every frame gets the bits mvs_fit gives it.  Afterwards the context
        holds no keypoints, no 3-D targets and no per-slot rigs (set_keypoints / set_joints3d / set_frame_rigs again before a
        closure or fit).  Returns (final_loss [F], stats)."""
        assert params.is_cuda and params.dtype == torch.float32 and params.is_contiguous() and params.dim() == 2
        F = params.shape[0]
        gt_uv, conf, jw, j3, c3 = self._stream_rows("fit_stream", F, gt_uv, conf, joint_weights, joints3d, conf3d)
        rg = self._stream_rigs("fit_stream", F, rig)
        final = torch.empty(F, dtype=torch.float32, device=self.device)
        s = _lib.FrameStream(F, _ptr(params), _ptr(gt_uv), _ptr(conf), _ptr(jw), _ptr(j3), _ptr(c3), _ptr(final))
        arr = (_lib.LossConfig * len(stage_cfgs))(*stage_cfgs)
        cfg = opt_cfg or self.make_lbfgs_config()
        st = _lib.LbfgsStats()
        self._j3d_keep = None
        _lib.check(self.h, self.lib.mvs_fit_stream_rigs(self.h, ctypes.byref(s), _ptr(rg), len(stage_cfgs), arr, ctypes.byref(cfg),
                                                        ctypes.byref(st), self._stream()), "mvs_fit_stream_rigs")
        return final, _stats_dict(st)

    def fit_seq_stream(self, params: torch.Tensor, gt_uv, conf, joint_weights, lengths, stage_cfgs, opt_cfg=None,
                       reinit_loss: float = 5000.0, joints3d=None, conf3d=None, rig=None, temporal_weight=None):
        """mvs_fit_seq over S video sequences through the context's B slots (mvs_fit_seq_stream): the frames of sequence s are
        the next lengths[s] rows, in time order.  params [F,86] CUDA float32 holds every frame's cold start point (init_guess)
        and is updated in place; gt_uv [V,F,K,2], conf [V,F,K], joint_weights [K] (numpy or tensors).  A frame after the first
        starts from its predecessor's result while that frame's final loss is <= reinit_loss (skipping stages 0 and 1), from
        its own row otherwise.  joints3d [F,K,3] with conf3d [F,K] switch the 3-D joint term on for every frame of the call
        (mvs_fit_seq_stream3d; zero-confidence rows for frames without annotations).  rig [F] (mvs_fit_seq_stream_rigs)
        names each frame's camera rig (set_camera_rigs; None: rig 0, one rig only).  Every frame gets the bits
        seqio.fit_sequences gives it with a batch of S.  temporal_weight [86] (mvs_fit_seq_stream_temporal): every warm frame's
        stages add sum_i w_i (x_i - x^_i)^2, x^ = its predecessor's fitted row.  Afterwards the context holds no keypoints,
        no 3-D targets and no per-slot rigs.  Returns (final_loss [F], stats)."""
        assert params.is_cuda and params.dtype == torch.float32 and params.is_contiguous() and params.dim() == 2
        F = params.shape[0]
        lengths = [int(n) for n in lengths]
        if not lengths or min(lengths) < 1 or sum(lengths) != F:
            raise ValueError("fit_seq_stream: want sequence lengths >= 1 that add up to %d frames, got %s" % (F, lengths))
        off = np.ascontiguousarray(np.concatenate([[0], np.cumsum(lengths)]), dtype=np.int32)
        gt_uv, conf, jw, j3, c3 = self._stream_rows("fit_seq_stream", F, gt_uv, conf, joint_weights, joints3d, conf3d)
        rg = self._stream_rigs("fit_seq_stream", F, rig)
        final = torch.empty(F, dtype=torch.float32, device=self.device)
        s = _lib.SequenceStream(len(lengths), _ptr(off), _ptr(params), _ptr(gt_uv), _ptr(conf), _ptr(jw), _ptr(final),
                                float(reinit_loss))
        arr = (_lib.LossConfig * len(stage_cfgs))(*stage_cfgs)
        cfg = opt_cfg or self.make_lbfgs_config()
        st = _lib.LbfgsStats()
        self._j3d_keep = None
        tw = None if temporal_weight is None else _temporal_weight(temporal_weight)
        _lib.check(self.h, self.lib.mvs_fit_seq_stream_temporal(self.h, ctypes.byref(s), _ptr(j3), _ptr(c3), _ptr(rg), _ptr(tw),
                                                                len(stage_cfgs), arr, ctypes.byref(cfg), ctypes.byref(st),
                                                                self._stream()), "mvs_fit_seq_stream_temporal")
        return final, _stats_dict(st)

    def fit_shared_shape(self, params: torch.Tensor, gt_uv, conf, joint_weights, lengths, stage_cfg, opt_cfg=None, sweeps=1,
                         joints3d=None, conf3d=None, rig=None):
        """One body shape per video sequence (mvs_fit_shared_shape): the frames of sequence s are the next lengths[s] rows of
        params [F,86] (CUDA float32, fitted rows in, result out).  `sweeps` rounds of: each sequence's betas (and scale, unless
        stage_cfg freezes it) fitted to all of its frames with the poses held, from the mean over its finite rows; then every
        frame refits stage_cfg with the shared entries frozen.  gt_uv [V,F,K,2], conf [V,F,K], joint_weights [K], joints3d /
        conf3d and rig as in fit_seq_stream.  Afterwards the context holds no keypoints, no 3-D targets and no per-slot rigs.
        Returns (final_loss [F], seq_loss [S], shape_stats, pose_stats)."""
        assert params.is_cuda and params.dtype == torch.float32 and params.is_contiguous() and params.dim() == 2
        F = params.shape[0]
        lengths = [int(n) for n in lengths]
        if not lengths or min(lengths) < 1 or sum(lengths) != F:
            raise ValueError("fit_shared_shape: want sequence lengths >= 1 that add up to %d frames, got %s" % (F, lengths))
        if int(sweeps) < 1:
            raise ValueError("fit_shared_shape: want sweeps >= 1, got %s" % sweeps)
        off = np.ascontiguousarray(np.concatenate([[0], np.cumsum(lengths)]), dtype=np.int32)
        gt_uv, conf, jw, j3, c3 = self._stream_rows("fit_shared_shape", F, gt_uv, conf, joint_weights, joints3d, conf3d)
        rg = self._stream_rigs("fit_shared_shape", F, rig)
        final = torch.empty(F, dtype=torch.float32, device=self.device)
        seq_loss = torch.empty(len(lengths), dtype=torch.float32, device=self.device)
        s = _lib.SequenceStream(len(lengths), _ptr(off), _ptr(params), _ptr(gt_uv), _ptr(conf), _ptr(jw), _ptr(final), 0.0)
        cfg = opt_cfg or self.make_lbfgs_config()
        sh, po = _lib.LbfgsStats(), _lib.LbfgsStats()
        self._j3d_keep = None
        _lib.check(self.h, self.lib.mvs_fit_shared_shape(self.h, ctypes.byref(s), _ptr(j3), _ptr(c3), _ptr(rg), ctypes.byref(stage_cfg),
                                                         ctypes.byref(cfg), int(sweeps), _ptr(seq_loss), ctypes.byref(sh),
                                                         ctypes.byref(po), self._stream()), "mvs_fit_shared_shape")
        return final, seq_loss, _stats_dict(sh), _stats_dict(po)

    def refine_cameras(self, params: torch.Tensor, gt_uv, conf, joint_weights, stage_cfg, opt_cfg=None, sweeps=1, joints3d=None,
                       conf3d=None, rig=None):
        """Refine every rig's extrinsics from fitted bodies (mvs_refine_cameras): `sweeps` rounds of: each view v >= 1 of every rig
        fitted to the keypoints of the frames with that rig, held from their rows (view 0 fixed, view 1 at its distance to
        view 0); then every frame refits stage_cfg from its row against the refined cameras.  params [F,86] CUDA float32, fitted
        rows in, result out; gt_uv [V,F,K,2], conf [V,F,K], joint_weights [K], joints3d / conf3d and rig as in fit_stream.  The
        context keeps the refined cameras; afterwards it holds no keypoints, no 3-D targets and no per-slot rigs.  Returns
        (final_loss [F], rigs, camera_stats, pose_stats), rigs: the refined table as the list of dict(R, t, f, c) that
        set_camera_rigs takes (same views per rig, f, c and any "dist" unchanged)."""
        assert params.is_cuda and params.dtype == torch.float32 and params.is_contiguous() and params.dim() == 2
        F = params.shape[0]
        if isinstance(sweeps, bool) or int(sweeps) != sweeps or sweeps < 1:
            raise ValueError("refine_cameras: want sweeps >= 1, got %r" % (sweeps,))
        gt_uv, conf, jw, j3, c3 = self._stream_rows("refine_cameras", F, gt_uv, conf, joint_weights, joints3d, conf3d)
        rg = self._stream_rigs("refine_cameras", F, rig)
        final = torch.empty(F, dtype=torch.float32, device=self.device)
        s = _lib.FrameStream(F, _ptr(params), _ptr(gt_uv), _ptr(conf), _ptr(jw), _ptr(j3), _ptr(c3), _ptr(final))
        cfg = opt_cfg or self.make_lbfgs_config()
        n = len(self.rig_views)
        R = np.zeros((n, self.V, 3, 3), np.float32)
        t = np.zeros((n, self.V, 3), np.float32)
        ca, po = _lib.LbfgsStats(), _lib.LbfgsStats()
        self._j3d_keep = None
        _lib.check(self.h, self.lib.mvs_refine_cameras(self.h, ctypes.byref(s), _ptr(rg), ctypes.byref(stage_cfg), ctypes.byref(cfg),
                                                       int(sweeps), _ptr(R), _ptr(t), ctypes.byref(ca), ctypes.byref(po),
                                                       self._stream()), "mvs_refine_cameras")
        for r, nv in enumerate(self.rig_views):
            self._rigs[r] = dict(self._rigs[r], R=R[r, :nv].copy(), t=t[r, :nv].copy())
        rigs = [{k: v.copy() for k, v in d.items()} for d in self._rigs]
        return final, rigs, _stats_dict(ca), _stats_dict(po)

    def fit_host(self, params_host: np.ndarray, gt_uv: np.ndarray, conf: np.ndarray, joint_weights: np.ndarray,
                 stage_cfgs, opt_cfg=None):
        """Host-buffer entry point (mvs_fit_host): params_host [B,86] float32 updated in place."""
        assert params_host.dtype == np.float32 and params_host.flags["C_CONTIGUOUS"]
        gt_uv, conf, jw = _f32(gt_uv), _f32(conf), _f32(np.reshape(joint_weights, -1))
        arr = (_lib.LossConfig * len(stage_cfgs))(*stage_cfgs)
        cfg = opt_cfg or self.make_lbfgs_config()
        final = np.zeros(self.B, dtype=np.float32)
        st = _lib.LbfgsStats()
        _lib.check(self.h, self.lib.mvs_fit_host(self.h, _ptr(params_host), _ptr(gt_uv), _ptr(conf), _ptr(jw),
                                                 len(stage_cfgs), arr, ctypes.byref(cfg), _ptr(final), ctypes.byref(st),
                                                 self._stream()), "mvs_fit_host")
        return final, _stats_dict(st)

    def sdf_grid(self, faces: torch.Tensor, verts: torch.Tensor, grid_size: int, num_faces: int | None = None):
        """The reference's `sdf.csrc.sdf` op: phi [B,G,G,G] for verts [B,N,3] normalised to [-1,1]."""
        assert verts.is_cuda and faces.is_cuda
        faces = faces.to(torch.int32).contiguous()
        verts = verts.float().contiguous()
        Bv, Nv = verts.shape[0], verts.shape[1]
        phi = torch.zeros(Bv, grid_size, grid_size, grid_size, dtype=torch.float32, device=self.device)
        nf = int(num_faces if num_faces is not None else faces.reshape(-1, 3).shape[0])
        _lib.check(self.h, self.lib.mvs_sdf_grid(self.h, _ptr(phi), _ptr(faces), nf, _ptr(verts), Bv, Nv, grid_size,
                                                 self._stream()), "mvs_sdf_grid")
        return phi

    def render(self, verts: torch.Tensor, keypoints: torch.Tensor | None = None, rig=None, background: torch.Tensor | None = None,
               width: int | None = None, height: int | None = None, outputs=("image",), base_color=(0.5, 0.5, 0.5),
               ambient: float = 0.3, marker_radius: float = 8.0, marker_color=(0, 0, 255)) -> dict:
        """The fitted meshes verts [n,N,3] (CUDA float32, e.g. forward_only's) drawn into every view of each frame's rig
        (mvs_render, DESIGN.md section 4d): shaded by a headlight plus ambient light over background [n,V,H,W,3] (CUDA uint8;
        None: black), with a disc of marker_radius px in marker_color around every keypoint of keypoints [n,K,3] (None: no
        markers).  rig [n] names each frame's camera rig (None: rig 0, one rig only).  width and height default to the
        background's.  outputs: any of "image" (uint8 [n,V,H,W,3]), "face" (int32 [n,V,H,W], -1 = background) and "depth"
        (float32 [n,V,H,W], +inf = background); rows v >= V_r of a frame with rig r hold what background holds: zeros (image), -1
        (face), +inf (depth).
        The defaults are the reference's renderer's numbers: base colour 0.5, ambient 0.3, markers red in cv2's BGR order.
        Returns a dict of the requested outputs."""
        def check(name, t, dtype, shape):
            if not isinstance(t, torch.Tensor) or t.dtype != dtype or t.device != self.device or tuple(t.shape) != shape:
                raise ValueError("render: want %s as a %s tensor of shape %s on %s, got %s" % (
                    name, dtype, shape, self.device, (t.dtype, tuple(t.shape), t.device) if isinstance(t, torch.Tensor) else type(t)))
            return t.contiguous()
        outputs = tuple(outputs)
        if not outputs or any(o not in ("image", "face", "depth") for o in outputs):
            raise ValueError("render: outputs must be a non-empty subset of ('image', 'face', 'depth'), got %r" % (outputs,))
        if verts.dim() != 3:
            raise ValueError("render: want verts [n,%d,3], got %s" % (self.N, tuple(verts.shape)))
        n = verts.shape[0]
        verts = check("verts", verts, torch.float32, (n, self.N, 3))
        if background is not None and background.dim() == 5:
            height = background.shape[2] if height is None else height
            width = background.shape[3] if width is None else width
        if width is None or height is None:
            raise ValueError("render: give width and height, or a background")
        W, H = int(width), int(height)
        if background is not None:
            background = check("background", background, torch.uint8, (n, self.V, H, W, 3))
        if keypoints is not None:
            keypoints = check("keypoints", keypoints, torch.float32, (n, self.K, 3))
        rg = self._stream_rigs("render", n, rig)
        out = {}
        if "image" in outputs:
            out["image"] = torch.zeros(n, self.V, H, W, 3, dtype=torch.uint8, device=self.device)
        if "face" in outputs:
            out["face"] = torch.full((n, self.V, H, W), -1, dtype=torch.int32, device=self.device)
        if "depth" in outputs:
            out["depth"] = torch.full((n, self.V, H, W), float("inf"), dtype=torch.float32, device=self.device)
        cfg = _lib.RenderConfig(W, H, (ctypes.c_float * 3)(*[float(c) for c in base_color]), float(ambient), float(marker_radius),
                                (ctypes.c_ubyte * 3)(*[int(c) for c in marker_color]))
        _lib.check(self.h, self.lib.mvs_render(self.h, n, _ptr(verts), _ptr(keypoints), _ptr(rg), _ptr(background), _ptr(out.get("image")),
                                               _ptr(out.get("face")), _ptr(out.get("depth")), ctypes.byref(cfg), self._stream()),
                   "mvs_render")
        return out

    def set_anchor(self, anchor: torch.Tensor | None, weight: torch.Tensor | None = None):
        """per-frame quadratic anchor sum_i w_i (x_i - a_i)^2 (sequence mode); anchor=None switches it off.
        Takes effect with the next set_loss()."""
        if anchor is None:
            _lib.check(self.h, self.lib.mvs_set_anchor(self.h, None, None, 0, self._stream()), "mvs_set_anchor")
            return
        anchor = anchor.to(self.device, torch.float32).contiguous()
        weight = weight.to(self.device, torch.float32).contiguous()
        if weight.dim() == 1:
            weight = weight[None].expand(self.B, -1).contiguous()
        assert tuple(anchor.shape) == (self.B, S.NUM_PARAMS) and tuple(weight.shape) == (self.B, S.NUM_PARAMS)
        _lib.check(self.h, self.lib.mvs_set_anchor(self.h, _ptr(anchor), _ptr(weight), 1, self._stream()), "mvs_set_anchor")

    def set_joints3d(self, gt_xyz, conf=None):
        """3-D joint targets of the SMPLifyLoss use_3d term (mvs_set_joints3d): gt_xyz [B,K,3], conf [B,K]; numpy (host) or
        CUDA tensors.  gt_xyz=None switches the term off.  Takes effect with the next set_loss() / fit() and at once in
        init_guess()."""
        if gt_xyz is None:
            _lib.check(self.h, self.lib.mvs_set_joints3d(self.h, None, None, 0, 0, self._stream()), "mvs_set_joints3d")
            self._j3d_keep = None
            return
        if conf is None:
            raise ValueError("set_joints3d: the 3-D term needs its confidences")
        on_dev = isinstance(gt_xyz, torch.Tensor) and gt_xyz.is_cuda
        if on_dev:
            gt_xyz = gt_xyz.to(self.device, torch.float32).contiguous()
            conf = torch.as_tensor(conf).to(self.device, torch.float32).contiguous()
        else:
            gt_xyz, conf = _f32(gt_xyz), _f32(conf)
        if tuple(gt_xyz.shape) != (self.B, self.K, 3) or tuple(conf.shape) != (self.B, self.K):
            raise ValueError("set_joints3d: want gt_xyz [%d,%d,3] and conf [%d,%d], got %s and %s"
                             % (self.B, self.K, self.B, self.K, tuple(gt_xyz.shape), tuple(conf.shape)))
        self._j3d_keep = (gt_xyz, conf)
        _lib.check(self.h, self.lib.mvs_set_joints3d(self.h, _ptr(gt_xyz), _ptr(conf), 1, 1 if on_dev else 0, self._stream()),
                   "mvs_set_joints3d")

    def set_exec_mode(self, mode: int):
        """0 = frame-resident kernels where they apply (default), 1 = batched kernels only"""
        _lib.check(self.h, self.lib.mvs_set_exec_mode(self.h, int(mode)), "mvs_set_exec_mode")

    def profile(self, mask: int = 0xFFFFFFFF):
        """start (mask != 0) / stop (0) per-kernel CUDA-event timing (see mvs_profile in mvsmpl.h)"""
        _lib.check(self.h, self.lib.mvs_profile(self.h, ctypes.c_uint(mask & 0xFFFFFFFF)), "mvs_profile")

    def profile_read(self) -> dict:
        """{kernel name: (total ms, launches)} since the last profile() call"""
        n = _lib.NUM_KERNEL_IDS
        ms = (ctypes.c_double * n)()
        cnt = (ctypes.c_longlong * n)()
        _lib.check(self.h, self.lib.mvs_profile_read(self.h, ms, cnt), "mvs_profile_read")
        return {self.lib.mvs_kernel_name(k).decode(): (ms[k], int(cnt[k])) for k in range(n) if cnt[k]}

    def launch_count(self) -> int:
        return int(self.lib.mvs_launch_count(self.h))
