"""Mirror of the reference's code/utils/init_guess.py (init_guess :18-107, load_init :140-187, fix_params :190-212)
with the same signatures, over the device path: the triangulation + similarity alignment run in `mvs_init_guess` for all
frames of the model's batch at once (the reference: one frame, numpy).

`setting` / `data` are the reference's dictionaries (init.py, data_parser.py): setting['model'] (SMPL module on CUDA),
setting['extris'] [V,4,4], setting['intris'] [V,3,3], setting['fix_scale'], setting['fixed_scale'],
setting['pose_embedding']; data['keypoints'] = list over views of [B,17,3] arrays (u, v, confidence).

Difference from the reference, documented in DESIGN.md §7: the alignment is the published Umeyama algorithm unless
`umeyama_as_written=True` is passed (keyword of init_guess / load_init; the reference's transposed-V variant depends on the
LAPACK build, see include/mvsmpl.h).  One view: the depth guess of :54-78, as written."""
from __future__ import annotations

import numpy as np
import torch

from ..fitting import model_context
from ..seqio import camera_arrays


def _run_device_guess(setting, data, use_torso, hip_seed, as_written=False, joints3d=None):
    model = setting["model"]
    keypoints = data["keypoints"]
    est_scale = not setting["fix_scale"]                                                   # init_guess.py:24
    fixed_scale = 1.0 if setting.get("fixed_scale") is None else float(setting["fixed_scale"])   # :25
    ctx = model_context(model)
    cams = camera_arrays(setting["extris"], setting["intris"])
    ctx.set_cameras(cams["R"], cams["t"], cams["f"], cams["c"])
    kp = np.stack([np.asarray(k, dtype=np.float32).reshape(ctx.B, -1, 3) for k in keypoints])      # [V,B,K,3]
    K = kp.shape[2]
    ctx.set_keypoints(np.ascontiguousarray(kp[..., :2]), np.ascontiguousarray(kp[..., 2]), np.ones(K, np.float32))
    if joints3d is not None:                  # only the xyz steer the alignment; the loss gets its targets from the closure
        ctx.set_joints3d(np.asarray(joints3d, dtype=np.float32).reshape(ctx.B, K, 3), np.ones((ctx.B, K), np.float32))
    elif getattr(ctx, "_j3d_keep", None) is not None:
        ctx.set_joints3d(None)
    params, joints3d = ctx.init_guess(estimate_scale=est_scale, fixed_scale=fixed_scale, use_torso=use_torso,
                                      hip_seed=hip_seed, umeyama_as_written=as_written)
    if getattr(ctx, "_j3d_keep", None) is not None:
        ctx.set_joints3d(None)                # the guess's stand-in confidences must not reach a later loss
    return params, joints3d, est_scale, fixed_scale


def init_guess(setting, data, use_torso=False, **kwargs):
    """init_guess.py:18-107: resets the model to zero pose / shape, then sets transl, global_orient and scale from the
    similarity transform between the model's rest joints and the triangulated detections."""
    j3 = None
    if kwargs.get("use_3d") and data.get("3d_joint") is not None:     # init_guess.py:85-86: align to the annotations
        j3 = np.asarray(data["3d_joint"][0])[..., :3]
    model = setting["model"]
    params, _, est_scale, fixed_scale = _run_device_guess(setting, data, use_torso, hip_seed=0.0,
                                                          as_written=bool(kwargs.get("umeyama_as_written", False)),
                                                          joints3d=j3)
    p = params.detach()
    dtype = setting.get("dtype", torch.float32)
    scale = p[:, 85:86].to(dtype) if est_scale else torch.full((p.shape[0], 1), fixed_scale, dtype=dtype, device=p.device)
    if tuple(model.scale.shape) != tuple(scale.shape):           # the reference's scale parameter is [1] (one frame)
        scale = scale.reshape(model.scale.shape)
    # reset_params zero-fills whatever is not passed (body_models_scale.py:310-316): betas and body_pose end up 0
    model.reset_params(transl=p[:, 82:85].to(dtype), global_orient=p[:, 10:13].to(dtype), scale=scale)
    if kwargs.get("use_vposer"):
        with torch.no_grad():
            setting["pose_embedding"].fill_(0)                                             # init_guess.py:96-98


def load_init(setting, data, results, use_torso=False, **kwargs):
    """init_guess.py:140-187: warm start from the previous frame's result unless its loss was above 5000"""
    if results["loss"] > 5000:
        init_guess(setting, data, use_torso=use_torso, **kwargs)
        setting["seq_start"] = True
        return
    model = setting["model"]
    dtype = setting.get("dtype", torch.float32)
    device = setting.get("device", None)
    t = lambda a: torch.as_tensor(a, dtype=dtype)
    if kwargs.get("use_vposer"):
        setting["pose_embedding"] = torch.tensor(np.asarray(results["pose_embedding"]), dtype=dtype, device=device,
                                                 requires_grad=True)
    model.reset_params(global_orient=t(results["global_orient"]), transl=t(results["transl"]), scale=t(results["scale"]),
                       betas=t(results["betas"]))


def fix_params(setting, scale=None, shape=None):
    """init_guess.py:190-212: keeps transl / global_orient / scale / betas, sets the body pose to zero except its first
    six entries (= 1), optionally pins scale and shape (requires_grad = False)"""
    model = setting["model"]
    dtype = setting.get("dtype", torch.float32)
    init_t, init_r, init_s, init_shape = model.transl, model.global_orient, model.scale, model.betas
    B = int(getattr(model, "batch_size", 1))
    body = torch.zeros(B, 69, dtype=dtype)
    body[:, :6] = 1.0
    if scale is not None:
        init_s = torch.tensor(scale, dtype=dtype)
        model.scale.requires_grad = False
    if shape is not None:
        init_shape = torch.tensor(shape, dtype=dtype)
        model.betas.requires_grad = False
    model.reset_params(transl=init_t, global_orient=init_r, scale=init_s, betas=init_shape, body_pose=body)
