"""SMPL.forward as a torch.autograd.Function: the forward is mvs_forward, the backward mvs_forward_vjp.

For callers who put the body model inside their own PyTorch loss (a silhouette, contact or 3-D marker term), train a
regressor through it or check a fit by back-propagation.  The fitting paths do not use it: their gradients come from the
fused closure (mvs_closure / mvs_fit).
"""
from __future__ import annotations

import torch


class SMPLFunction(torch.autograd.Function):
    """(joints [B,K,3], verts [B,N,3] or None) = SMPL(params [B,86]) through a FittingContext.  The outputs are the bits
    FittingContext.forward_only returns.  First derivatives only: backward with create_graph=True raises
    NotImplementedError."""

    @staticmethod
    def forward(ctx, params, fctx, want_verts):
        out = fctx.forward_only(params.detach().contiguous(), want_verts=want_verts)
        ctx.fctx = fctx
        ctx.set_materialize_grads(False)
        ctx.save_for_backward(params)
        return out["joints"], out.get("verts")

    @staticmethod
    def backward(ctx, djoints, dverts):
        if torch.is_grad_enabled():
            raise NotImplementedError("SMPL through mvs_forward_vjp has first derivatives only (create_graph=True / double "
                                      "backward is not implemented)")
        if djoints is None and dverts is None:
            return None, None, None
        (params,) = ctx.saved_tensors
        dparams = ctx.fctx.forward_vjp(params.detach().contiguous(),
                                       None if djoints is None else djoints.contiguous(),
                                       None if dverts is None else dverts.contiguous())
        return dparams, None, None


def smpl_apply(fctx, params: torch.Tensor, want_verts: bool = True):
    """joints [B,K,3] and verts [B,N,3] (None without want_verts) of params [B,86], differentiable with respect to params"""
    return SMPLFunction.apply(params, fctx, bool(want_verts))
