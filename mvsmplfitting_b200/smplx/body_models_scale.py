"""SMPL body model with the reference's extra `scale` parameter and `smpllsp` joint regressor,
computed by libmvsmpl (CUDA) instead of the PyTorch op chain.

Mirrors the public surface of reference code/smplx/body_models_scale.py for the SMPL class
(:39-89 create_scale, :92-412 SMPL): same constructor keywords, the same nn.Parameters
(betas, global_orient, body_pose, transl, scale, registered in that order), the same buffers,
reset_params(), and forward() -> ModelOutput.  SMPLH / SMPLX are out of scope (unreachable from
cfg_files/fit_smpl.yaml).

By default forward() returns DETACHED tensors: inside the fitting loop gradients come from the fused closure
(FittingMonitor.create_fitting_closure), which never builds an autograd graph.  With differentiable=True, forward() keeps
the module's parameters and the tensors passed to it in the graph and back-propagates through mvs_forward_vjp, like the
reference's autograd module (first derivatives only).
"""
from __future__ import annotations

import os
import pickle
from collections import namedtuple

import numpy as np
import torch
import torch.nn as nn

from .. import synthetic as S

ModelOutput = namedtuple("ModelOutput", ["vertices", "joints", "full_pose", "betas", "global_orient", "body_pose",
                                         "expression", "left_hand_pose", "right_hand_pose", "jaw_pose"])
ModelOutput.__new__.__defaults__ = (None,) * len(ModelOutput._fields)


class Struct(object):
    def __init__(self, **kwargs):
        for k, v in kwargs.items():
            setattr(self, k, v)


def _np(a, dtype=np.float32):
    if "scipy.sparse" in str(type(a)):
        a = a.todense()
    return np.array(a, dtype=dtype)


def create_scale(model_path, model_type="smpl", **kwargs):
    """Same dispatch as the reference factory (body_models_scale.py:39-89).  differentiable=True (passed on to SMPL) gives a
    module whose forward() back-propagates into its parameters and inputs."""
    if os.path.isdir(model_path):
        model_path = os.path.join(model_path, "smpl")
    mt = model_type.lower()
    if mt in ("smpl", "smpllsp"):
        return SMPL(model_path, model_type=model_type, **kwargs)
    if mt in ("smplh", "smplx"):
        raise ValueError("model type {} is outside the B200 fitting path (only 'smpl' / 'smpllsp')".format(model_type))
    raise ValueError("Unknown model type {}, exiting!".format(model_type))


class VertexJointSelector(nn.Module):
    """face keypoints appended after the joints (vertex_joint_selector.py:38-43)"""

    def __init__(self, vertex_ids=None, **kwargs):
        super().__init__()
        ids = S.FACE_VERTEX_IDS if vertex_ids is None else np.array(
            [vertex_ids[k] for k in ("nose", "leye", "reye", "lear", "rear")], dtype=np.int64)
        self.register_buffer("extra_joints_idxs", torch.tensor(np.asarray(ids), dtype=torch.long))


class SMPL(nn.Module):
    NUM_JOINTS = 23
    NUM_BODY_JOINTS = 23
    NUM_BETAS = 10

    def __init__(self, model_path, data_struct=None, create_betas=True, betas=None, create_global_orient=True,
                 global_orient=None, create_body_pose=True, body_pose=None, create_transl=True, transl=None,
                 create_scale=True, scale=None, dtype=torch.float32, batch_size=1, joint_mapper=None,
                 model_type="smpl", gender="neutral", vertex_ids=None, lsp_regressor_path="data/J_regressor_lsp.npz",
                 differentiable=False, **kwargs):
        self.model_type = model_type
        self.differentiable = bool(differentiable)
        self.gender = gender
        if data_struct is None:
            fn = os.path.join(model_path, "SMPL_{}.pkl".format(gender.upper())) if os.path.isdir(model_path) else model_path
            assert os.path.exists(fn), "Path {} does not exist!".format(fn)
            with open(fn, "rb") as f:
                data_struct = Struct(**pickle.load(f, encoding="latin1"))
        super().__init__()
        if dtype != torch.float32:
            raise ValueError("the B200 path computes in float32 (float_dtype: 'float32' in fit_smpl.yaml)")
        self.batch_size = batch_size
        self.dtype = dtype
        self.joint_mapper = joint_mapper
        self.vertex_joint_selector = VertexJointSelector(vertex_ids=vertex_ids, **kwargs)
        self.faces = data_struct.f
        self.register_buffer("faces_tensor", torch.tensor(_np(self.faces, np.int64), dtype=torch.long))

        def param(name, create, value, shape):
            if not create:
                return
            if value is None:
                t = torch.ones(shape, dtype=dtype) if name == "scale" else torch.zeros(shape, dtype=dtype)
            elif torch.is_tensor(value):
                t = value.clone().detach().to(dtype)
            else:
                t = torch.tensor(value, dtype=dtype)
            self.register_parameter(name, nn.Parameter(t, requires_grad=True))

        # registration order fixes the L-BFGS flat layout (body_models_scale.py:213,232,244,255,266)
        param("betas", create_betas, betas, [batch_size, self.NUM_BETAS])
        param("global_orient", create_global_orient, global_orient, [batch_size, 3])
        param("body_pose", create_body_pose, body_pose, [batch_size, self.NUM_BODY_JOINTS * 3])
        param("transl", create_transl, transl, [batch_size, 3])
        param("scale", create_scale, scale, [batch_size, 1])

        self.register_buffer("v_template", torch.tensor(_np(data_struct.v_template), dtype=dtype))
        self.register_buffer("shapedirs", torch.tensor(_np(data_struct.shapedirs), dtype=dtype))
        if self.model_type == "smpllsp":
            self.register_buffer("joint_regressor", torch.tensor(S.load_lsp_regressor(lsp_regressor_path), dtype=dtype))
        self.register_buffer("J_regressor", torch.tensor(_np(data_struct.J_regressor), dtype=dtype))
        pd = _np(data_struct.posedirs)
        self.register_buffer("posedirs", torch.tensor(np.reshape(pd, [-1, pd.shape[-1]]).T.copy(), dtype=dtype))
        parents = torch.tensor(_np(data_struct.kintree_table[0], np.int64)).long()
        parents[0] = -1
        self.register_buffer("parents", parents)
        self.register_buffer("lbs_weights", torch.tensor(_np(data_struct.weights), dtype=dtype))
        self._mvs = None          # (FittingContext, cache key) built lazily on the first CUDA use

    # ------------------------------------------------------------------ reference helpers
    @torch.no_grad()
    def reset_params(self, **params_dict):
        for name, p in self.named_parameters():
            if name in params_dict:
                p[:] = torch.as_tensor(params_dict[name]).clone().detach().to(p)
            else:
                p.fill_(0)

    def get_num_verts(self):
        return self.v_template.shape[0]

    def get_num_faces(self):
        return self.faces.shape[0]

    def extra_repr(self):
        return "Number of betas: {}".format(self.NUM_BETAS)

    # ------------------------------------------------------------------ CUDA context plumbing
    def model_dict(self) -> dict:
        """the arrays mvs_set_model needs, in the reference's data_struct layout"""
        N = self.v_template.shape[0]
        d = dict(v_template=self.v_template.cpu().numpy(), shapedirs=self.shapedirs.cpu().numpy(),
                 posedirs=self.posedirs.cpu().numpy(), J_regressor=self.J_regressor.cpu().numpy(),
                 parents=self.parents.cpu().numpy(), weights=self.lbs_weights.cpu().numpy(),
                 f=self.faces_tensor.cpu().numpy().astype(np.int32).reshape(-1, 3))
        if self.model_type == "smpllsp":
            d["lsp_regressor"] = self.joint_regressor.cpu().numpy()
        assert d["posedirs"].shape == (207, 3 * N)
        return d

    def joint_map(self):
        if self.joint_mapper is not None and getattr(self.joint_mapper, "joint_maps", None) is not None:
            return self.joint_mapper.joint_maps.cpu().numpy().astype(np.int32)
        n = (14 if self.model_type == "smpllsp" else 24) + len(self.vertex_joint_selector.extra_joints_idxs)
        return np.arange(n, dtype=np.int32)

    def flat_params(self, body_pose=None) -> torch.Tensor:
        """[B,86] in the library's order; missing tensors (e.g. body_pose under VPoser) come from arguments"""
        B = self.batch_size
        dev = self.v_template.device

        def get(name, n, default):
            t = getattr(self, name, None)
            if name == "body_pose" and body_pose is not None:
                t = body_pose
            if t is None:
                return torch.full((B, n), default, dtype=torch.float32, device=dev)
            return t.detach().reshape(B, n).to(torch.float32)
        return torch.cat([get("betas", 10, 0.0), get("global_orient", 3, 0.0), get("body_pose", 69, 0.0),
                          get("transl", 3, 0.0), get("scale", 1, 1.0)], dim=1).contiguous()

    def graph_params(self, betas=None, body_pose=None, global_orient=None, transl=None, scale=None) -> torch.Tensor:
        """[B,86] in the library's order from the tensors passed in, else the module's parameters, NOT detached
        (differentiable=True); a tensor missing from both is filled with its default (0, scale 1)"""
        B = self.batch_size
        dev = self.v_template.device

        def get(name, given, n, default):
            t = given if given is not None else getattr(self, name, None)
            if t is None:
                return torch.full((B, n), default, dtype=torch.float32, device=dev)
            return t.reshape(B, n).to(torch.float32)
        return torch.cat([get("betas", betas, 10, 0.0), get("global_orient", global_orient, 3, 0.0),
                          get("body_pose", body_pose, 69, 0.0), get("transl", transl, 3, 0.0),
                          get("scale", scale, 1, 1.0)], dim=1)

    def forward(self, betas=None, body_pose=None, global_orient=None, transl=None, scale=None, return_verts=True,
                return_full_pose=False, **kwargs):
        from ..fitting import model_context
        if not self.v_template.is_cuda:
            raise RuntimeError("mvsmplfitting_b200.SMPL.forward needs the model on a CUDA device (no CPU fallback)")
        ctx = model_context(self)
        if self.differentiable:
            from ..autograd import smpl_apply
            x = self.graph_params(betas=betas, body_pose=body_pose, global_orient=global_orient, transl=transl, scale=scale)
            joints, verts = smpl_apply(ctx, x, want_verts=return_verts)
            go, bp = x[:, 10:13], x[:, 13:82]
            return ModelOutput(vertices=verts, joints=joints, global_orient=go, body_pose=bp, betas=x[:, :10],
                               full_pose=torch.cat([go, bp], dim=1) if return_full_pose else None)
        x = self.flat_params(body_pose=body_pose)
        over = dict(betas=(betas, 0, 10), global_orient=(global_orient, 10, 13), transl=(transl, 82, 85), scale=(scale, 85, 86))
        for t, a, e in over.values():
            if t is not None:
                x[:, a:e] = t.detach().reshape(self.batch_size, e - a)
        out = ctx.forward_only(x, want_verts=return_verts)
        go, bp = x[:, 10:13], x[:, 13:82]
        return ModelOutput(vertices=out.get("verts") if return_verts else None, joints=out["joints"],
                           global_orient=go, body_pose=bp, betas=self.betas if hasattr(self, "betas") else x[:, :10],
                           full_pose=torch.cat([go, bp], dim=1) if return_full_pose else None)
