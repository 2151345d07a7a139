"""ctypes binding of libmvsmpl.so (include/mvsmpl.h).

There is NO CPU fallback: if the shared library is missing, or no sm_100 device is
visible when a context is created, this raises -- it never silently routes around
the CUDA path.
"""
from __future__ import annotations

import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libmvsmpl.so")


class MvsError(RuntimeError):
    pass


class ModelDesc(ctypes.Structure):
    _fields_ = [
        ("n_verts", ctypes.c_int), ("n_faces", ctypes.c_int),
        ("v_template", ctypes.c_void_p), ("shapedirs", ctypes.c_void_p), ("posedirs", ctypes.c_void_p),
        ("J_regressor", ctypes.c_void_p), ("parents", ctypes.c_void_p), ("lbs_weights", ctypes.c_void_p),
        ("faces", ctypes.c_void_p),
        ("n_keypoints", ctypes.c_int), ("n_reg", ctypes.c_int), ("joint_regressor", ctypes.c_void_p),
        ("n_extra", ctypes.c_int), ("extra_vertex_ids", ctypes.c_void_p), ("joint_map", ctypes.c_void_p),
    ]


class LossConfig(ctypes.Structure):
    _fields_ = [
        ("data_weight", ctypes.c_float), ("body_pose_weight", ctypes.c_float), ("shape_weight", ctypes.c_float),
        ("bending_prior_weight", ctypes.c_float), ("coll_loss_weight", ctypes.c_float), ("rho", ctypes.c_float),
        ("body_prior", ctypes.c_int), ("use_joints_conf", ctypes.c_int), ("use_vposer", ctypes.c_int),
        ("fix_shape", ctypes.c_int), ("interpenetration", ctypes.c_int), ("sdf_grid", ctypes.c_int),
        ("sdf_all_faces", ctypes.c_int), ("frozen_mask", ctypes.c_uint),
    ]


class LbfgsConfig(ctypes.Structure):
    _fields_ = [
        ("max_outer", ctypes.c_int), ("max_iter", ctypes.c_int), ("max_eval", ctypes.c_int),
        ("history_size", ctypes.c_int), ("lr", ctypes.c_float), ("tolerance_grad", ctypes.c_float),
        ("tolerance_change", ctypes.c_float), ("ftol", ctypes.c_float), ("gtol", ctypes.c_float),
    ]


class LbfgsStats(ctypes.Structure):
    _fields_ = [("frame_iterations", ctypes.c_longlong), ("frame_evals", ctypes.c_longlong),
                ("rounds", ctypes.c_int), ("frames_nan", ctypes.c_int), ("dense_frame_evals", ctypes.c_longlong),
                ("dense_rounds", ctypes.c_int), ("reserved", ctypes.c_int)]


class RenderConfig(ctypes.Structure):
    """mvs_render_config (include/mvsmpl.h)"""
    _fields_ = [("width", ctypes.c_int), ("height", ctypes.c_int), ("base_color", ctypes.c_float * 3), ("ambient", ctypes.c_float),
                ("marker_radius", ctypes.c_float), ("marker_color", ctypes.c_ubyte * 3)]


class InitConfig(ctypes.Structure):
    """mvs_init_config (include/mvsmpl.h)"""
    _fields_ = [("estimate_scale", ctypes.c_int), ("fixed_scale", ctypes.c_float), ("use_torso", ctypes.c_int),
                ("hip_seed", ctypes.c_float), ("umeyama_as_written", ctypes.c_int)]


class FrameStream(ctypes.Structure):
    """mvs_frame_stream (include/mvsmpl.h)"""
    _fields_ = [("n_frames", ctypes.c_int), ("params", ctypes.c_void_p), ("gt_uv", ctypes.c_void_p), ("conf", ctypes.c_void_p),
                ("joint_weights", ctypes.c_void_p), ("gt_xyz", ctypes.c_void_p), ("conf3d", ctypes.c_void_p),
                ("final_loss", ctypes.c_void_p)]


class SequenceStream(ctypes.Structure):
    """mvs_sequence_stream (include/mvsmpl.h)"""
    _fields_ = [("n_sequences", ctypes.c_int), ("seq_offsets", ctypes.c_void_p), ("params", ctypes.c_void_p),
                ("gt_uv", ctypes.c_void_p), ("conf", ctypes.c_void_p), ("joint_weights", ctypes.c_void_p),
                ("final_loss", ctypes.c_void_p), ("reinit_loss", ctypes.c_float)]


EXPORTS = (
    "mvs_version", "mvs_build_id", "mvs_create", "mvs_destroy", "mvs_last_error", "mvs_launch_count", "mvs_set_model",
    "mvs_set_gmm_prior", "mvs_set_vposer", "mvs_vposer_decode", "mvs_set_cameras", "mvs_set_camera_rigs", "mvs_set_camera_rigs_dist", "mvs_set_frame_rigs", "mvs_set_batch", "mvs_set_keypoints", "mvs_set_loss_config",
    "mvs_closure", "mvs_forward", "mvs_forward_vjp", "mvs_lbfgs_run", "mvs_lbfgs_step", "mvs_fit", "mvs_fit_seq", "mvs_fit_stream", "mvs_fit_seq_stream", "mvs_fit_seq_stream3d",
    "mvs_fit_stream_rigs", "mvs_fit_seq_stream_rigs", "mvs_fit_host", "mvs_sdf_grid", "mvs_profile", "mvs_profile_read",
    "mvs_kernel_name", "mvs_set_exec_mode", "mvs_set_anchor", "mvs_set_joints3d", "mvs_init_guess", "mvs_fit_seq_temporal",
    "mvs_fit_seq_stream_temporal", "mvs_fit_shared_shape", "mvs_refine_cameras", "mvs_render",
)
NUM_KERNEL_IDS = 19

_lib = None


def load() -> ctypes.CDLL:
    """Load libmvsmpl.so; raises MvsError (never falls back) when it is not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise MvsError(
            "libmvsmpl.so is not built (%s). Build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "or `python -m mvsmplfitting_b200.build`; there is no CPU fallback." % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    vp, ci, cf = ctypes.c_void_p, ctypes.c_int, ctypes.c_float
    lib.mvs_version.restype = ci
    lib.mvs_create.argtypes = [ci, ctypes.POINTER(vp)]
    lib.mvs_destroy.argtypes = [vp]
    lib.mvs_destroy.restype = None
    lib.mvs_last_error.argtypes = [vp]
    lib.mvs_last_error.restype = ctypes.c_char_p
    lib.mvs_launch_count.argtypes = [vp]
    lib.mvs_launch_count.restype = ctypes.c_longlong
    lib.mvs_set_model.argtypes = [vp, ctypes.POINTER(ModelDesc)]
    lib.mvs_set_gmm_prior.argtypes = [vp, ci, vp, vp, vp]
    lib.mvs_set_cameras.argtypes = [vp, ci, vp, vp, vp, vp]
    lib.mvs_set_camera_rigs.argtypes = [vp, ci, vp, vp, vp, vp, vp, vp]
    lib.mvs_set_camera_rigs_dist.argtypes = [vp, ci, vp, vp, vp, vp, vp, vp, vp]
    lib.mvs_set_frame_rigs.argtypes = [vp, vp]
    lib.mvs_set_batch.argtypes = [vp, ci]
    lib.mvs_set_keypoints.argtypes = [vp, vp, vp, vp, ci, vp]
    lib.mvs_set_loss_config.argtypes = [vp, ctypes.POINTER(LossConfig)]
    lib.mvs_closure.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp]
    lib.mvs_forward.argtypes = [vp, vp, vp, vp, vp]
    lib.mvs_forward_vjp.argtypes = [vp, vp, vp, vp, vp, vp]
    lib.mvs_lbfgs_run.argtypes = [vp, vp, vp, ctypes.POINTER(LbfgsConfig), ctypes.POINTER(LbfgsStats), vp]
    lib.mvs_lbfgs_step.argtypes = [vp, vp, vp, vp, ctypes.POINTER(LbfgsConfig), ci, ctypes.POINTER(LbfgsStats), vp]
    lib.mvs_set_vposer.argtypes = [vp, vp, vp, vp, vp, vp, vp]
    lib.mvs_build_id.restype = ctypes.c_char_p
    lib.mvs_build_id.argtypes = []
    lib.mvs_vposer_decode.argtypes = [vp, vp, vp, vp]
    lib.mvs_init_guess.argtypes = [vp, vp, vp, ctypes.POINTER(InitConfig), vp]
    lib.mvs_fit.argtypes = [vp, vp, ci, ctypes.POINTER(LossConfig), ctypes.POINTER(LbfgsConfig), vp, ctypes.POINTER(LbfgsStats), vp]
    lib.mvs_fit_seq.argtypes = [vp, vp, ci, ctypes.POINTER(LossConfig), ctypes.POINTER(LbfgsConfig), vp, vp,
                                ctypes.POINTER(LbfgsStats), vp]
    lib.mvs_fit_seq_temporal.argtypes = [vp, vp, ci, ctypes.POINTER(LossConfig), ctypes.POINTER(LbfgsConfig), vp, vp, vp, vp,
                                         ctypes.POINTER(LbfgsStats), vp]
    lib.mvs_fit_stream.argtypes = [vp, ctypes.POINTER(FrameStream), ci, ctypes.POINTER(LossConfig), ctypes.POINTER(LbfgsConfig),
                                   ctypes.POINTER(LbfgsStats), vp]
    lib.mvs_fit_seq_stream.argtypes = [vp, ctypes.POINTER(SequenceStream), ci, ctypes.POINTER(LossConfig),
                                       ctypes.POINTER(LbfgsConfig), ctypes.POINTER(LbfgsStats), vp]
    lib.mvs_fit_seq_stream3d.argtypes = [vp, ctypes.POINTER(SequenceStream), vp, vp, ci, ctypes.POINTER(LossConfig),
                                         ctypes.POINTER(LbfgsConfig), ctypes.POINTER(LbfgsStats), vp]
    lib.mvs_fit_stream_rigs.argtypes = [vp, ctypes.POINTER(FrameStream), vp, ci, ctypes.POINTER(LossConfig),
                                        ctypes.POINTER(LbfgsConfig), ctypes.POINTER(LbfgsStats), vp]
    lib.mvs_fit_seq_stream_rigs.argtypes = [vp, ctypes.POINTER(SequenceStream), vp, vp, vp, ci, ctypes.POINTER(LossConfig),
                                            ctypes.POINTER(LbfgsConfig), ctypes.POINTER(LbfgsStats), vp]
    lib.mvs_fit_seq_stream_temporal.argtypes = [vp, ctypes.POINTER(SequenceStream), vp, vp, vp, vp, ci, ctypes.POINTER(LossConfig),
                                                ctypes.POINTER(LbfgsConfig), ctypes.POINTER(LbfgsStats), vp]
    lib.mvs_fit_shared_shape.argtypes = [vp, ctypes.POINTER(SequenceStream), vp, vp, vp, ctypes.POINTER(LossConfig),
                                         ctypes.POINTER(LbfgsConfig), ci, vp, ctypes.POINTER(LbfgsStats), ctypes.POINTER(LbfgsStats),
                                         vp]
    lib.mvs_refine_cameras.argtypes = [vp, ctypes.POINTER(FrameStream), vp, ctypes.POINTER(LossConfig), ctypes.POINTER(LbfgsConfig),
                                       ci, vp, vp, ctypes.POINTER(LbfgsStats), ctypes.POINTER(LbfgsStats), vp]
    lib.mvs_fit_host.argtypes = [vp, vp, vp, vp, vp, ci, ctypes.POINTER(LossConfig), ctypes.POINTER(LbfgsConfig), vp,
                                 ctypes.POINTER(LbfgsStats), vp]
    lib.mvs_sdf_grid.argtypes = [vp, vp, vp, ci, vp, ci, ci, ci, vp]
    lib.mvs_render.argtypes = [vp, ci, vp, vp, vp, vp, vp, vp, vp, ctypes.POINTER(RenderConfig), vp]
    lib.mvs_set_exec_mode.argtypes = [vp, ci]
    lib.mvs_set_anchor.argtypes = [vp, vp, vp, ci, vp]
    lib.mvs_set_joints3d.argtypes = [vp, vp, vp, ci, ci, vp]
    lib.mvs_profile.argtypes = [vp, ctypes.c_uint]
    lib.mvs_profile_read.argtypes = [vp, vp, vp]
    lib.mvs_kernel_name.argtypes = [ci]
    lib.mvs_kernel_name.restype = ctypes.c_char_p
    for name in EXPORTS:
        if name not in ("mvs_destroy", "mvs_last_error", "mvs_launch_count", "mvs_kernel_name", "mvs_build_id"):
            getattr(lib, name).restype = ci
    _lib = lib
    return lib


def check(ctx, rc: int, what: str):
    if rc != 0:
        msg = load().mvs_last_error(ctx)
        raise MvsError("%s failed (%d): %s" % (what, rc, msg.decode() if msg else "?"))
