"""GPU: the per-frame SDF set-up that the skinning kernels compute for sdf_fused (sdf_frame_setup in mvs_tc_dev.cuh).

* The FrameBox frame_step receives is, bit for bit, the fold of the frame's 64-vertex chunk boxes that sdf_fused used to do in
  every CTA (minimum / maximum per axis, ties -> lowest vertex index, then centre and scale in fp32), on batch sizes that run
  skin_small (<= 8 frames) and skin (partial and full 32-frame groups).
* The per-256-vertex-block sums and flags do not depend on how many blocks one sdf_fused CTA takes (MVS_SDF_PASSES, read
  once per process, so every setting runs in its own process).
* The arrival counters are back at zero after a round, and a round after a round with other parameters gives the outputs of
  a fresh context."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from mvsmplfitting_b200 import synthetic as S

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOSS = dict(body_prior="gmm", interpenetration=True, coll_loss_weight=1000.0, sdf_grid=128, data_weight=500 / 1536,
            body_pose_weight=57.4, shape_weight=10.0, bending_prior_weight=3.17 * 57.4)


def make_ctx(model, gmm, cams, B, seed):
    from mvsmplfitting_b200.context import FittingContext
    fr = S.make_frames(model, cams, B, seed=seed)
    ctx = FittingContext(0)
    ctx.set_model(model)
    ctx.set_gmm_from_dict(gmm)
    ctx.set_cameras(cams["R"], cams["t"], cams["f"], cams["c"])
    ctx.set_batch(B)
    ctx.set_keypoints(fr["gt_uv"], fr["conf"], fr["joint_weights"])
    ctx.set_exec_mode(3)                               # one dense round: posedirs_gemm_tc -> skin -> sdf_fused -> frame_step
    ctx.set_loss(**LOSS)
    return ctx, fr


def sdf_state(ctx, B, N):
    nbox, nblocks = (N + 63) // 64, (N + 255) // 256
    st = dict(bboxp=np.zeros((B, nbox, 12), np.float32), slot_tr=np.zeros((B, 4), np.float32),
              box=np.zeros((B, 12), np.float32), parts5=np.zeros((B, nblocks, 5), np.float32),
              pflag=np.zeros((B, nblocks), np.int32), arrive=np.ones(B, np.int32))
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    rc = ctx.lib.mvs_debug_sdf_state(ctx.h, p(st["bboxp"]), p(st["slot_tr"]), p(st["box"]), p(st["parts5"]), p(st["pflag"]),
                                     p(st["arrive"]))
    assert rc == 0
    return st


def canonical(v):
    return np.float32(v) + np.float32(0.0)               # the warp fold returns -0 as +0


def fold_box(bboxp, tr):
    """the fold sdf_fused did per CTA, restated on the host: FrameBox as 12 words (centre, scale, ilo, ihi, cmax, pad)"""
    out = np.zeros(12, np.float32)
    words = out.view(np.int32)
    lo, hi, ilo, ihi = [], [], [], []
    for c in range(3):
        l, h = bboxp[:, c], bboxp[:, 3 + c]
        il, ih = bboxp[:, 6 + c].view(np.int32), bboxp[:, 9 + c].view(np.int32)
        lo.append(canonical(l.min())); ilo.append(il[l == l.min()].min())
        hi.append(canonical(h.max())); ihi.append(ih[h == h.max()].min())
    ext, cmax = np.float32(-1.0), 0
    for c in range(3):
        lc, hc = np.float32(lo[c] + tr[c]), np.float32(hi[c] + tr[c])
        out[c] = np.float32(np.float32(lc + hc) / np.float32(2.0))
        words[4 + c], words[7 + c] = ilo[c], ihi[c]
        e = np.float32(hc - lc)
        if e > ext:
            ext, cmax = e, c
    out[3] = np.float32(np.float32(0.6) * ext)
    words[10] = cmax
    return out


@pytest.mark.parametrize("B", [1, 3, 8, 9, 33, 256, 257])
def test_frame_box_equals_chunk_box_fold(B, syn_model, syn_gmm):
    cams = S.make_cameras(4)
    ctx, fr = make_ctx(syn_model, syn_gmm, cams, B, seed=700 + B)
    try:
        x = torch.tensor(S.pack_params(fr["init"]), device="cuda")
        ctx.closure(x)
        st = sdf_state(ctx, B, ctx.N)
    finally:
        ctx.close()
    assert not st["arrive"].any(), "arrival counters not reset after the round"
    for s in range(B):
        want = fold_box(st["bboxp"][s], st["slot_tr"][s])
        assert want.view(np.int32)[:11].tobytes() == st["box"][s].view(np.int32)[:11].tobytes(), "slot %d" % s


PASSES_SCRIPT = r"""
import sys, numpy as np, torch
sys.path.insert(0, %(root)r)
from tests.test_gpu_sdf_setup import make_ctx, sdf_state
from mvsmplfitting_b200 import synthetic as S
model, gmm, cams = S.make_model(0), S.make_gmm(7), S.make_cameras(4)
res = {}
for B in (1, 8, 64):
    ctx, fr = make_ctx(model, gmm, cams, B, seed=900 + B)
    x = torch.tensor(S.pack_params(fr["init"]), device="cuda")
    o = ctx.closure(x)
    st = sdf_state(ctx, B, ctx.N)
    res["parts5_%%d" %% B] = st["parts5"]; res["pflag_%%d" %% B] = st["pflag"]
    res["loss_%%d" %% B] = o["loss"].cpu().numpy(); res["grad_%%d" %% B] = o["grad"].cpu().numpy()
    ctx.close()
np.savez(%(out)r, **res)
"""


def test_block_outputs_do_not_depend_on_blocks_per_cta(tmp_path):
    runs = {}
    for p in (1, 2, 4, 8):
        out = str(tmp_path / ("passes%d.npz" % p))
        env = dict(os.environ, MVS_SDF_PASSES=str(p))
        subprocess.run([sys.executable, "-c", PASSES_SCRIPT % dict(root=ROOT, out=out)], env=env, check=True, cwd=ROOT)
        runs[p] = np.load(out)
    ref = runs[1]
    assert any(ref["pflag_%d" % B].any() for B in (1, 8, 64)), "no block with a non-zero sample gradient: the case tests little"
    for p in (2, 4, 8):
        for k in ref.files:
            assert ref[k].tobytes() == runs[p][k].tobytes(), "MVS_SDF_PASSES=%d: %s differs" % (p, k)


def test_consecutive_rounds_leave_nothing_behind(syn_model, syn_gmm):
    cams = S.make_cameras(4)
    B = 40                                               # one full and one partial 32-frame group of skin_kernel
    fa = S.make_frames(syn_model, cams, B, seed=41)
    ctx, fr = make_ctx(syn_model, syn_gmm, cams, B, seed=42)
    fresh, _ = make_ctx(syn_model, syn_gmm, cams, B, seed=42)
    try:
        xa = torch.tensor(S.pack_params(fa["init"]), device="cuda")
        xb = torch.tensor(S.pack_params(fr["init"]), device="cuda")
        ctx.closure(xa)
        o1 = ctx.closure(xb)
        s1 = sdf_state(ctx, B, ctx.N)
        o2 = ctx.closure(xb)
        s2 = sdf_state(ctx, B, ctx.N)
        o3 = fresh.closure(xb)
        s3 = sdf_state(fresh, B, fresh.N)
    finally:
        ctx.close()
        fresh.close()
    for s in (s1, s2, s3):
        assert not s["arrive"].any()
    for o in (o2, o3):
        assert o1["loss"].cpu().numpy().tobytes() == o["loss"].cpu().numpy().tobytes()
        assert o1["grad"].cpu().numpy().tobytes() == o["grad"].cpu().numpy().tobytes()
    for k in ("box", "parts5", "pflag"):
        assert s1[k].tobytes() == s2[k].tobytes() == s3[k].tobytes(), k
