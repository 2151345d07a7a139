"""GPU: the per-frame SDF set-up of the dense rounds, computed by sdf_setup_kernel (one warp per frame, after the skinning
kernel) or, at <= 4 frames, at the end of skin_small_kernel, both through sdf_frame_setup.

* One exec-mode-3 round on both sides of the skin_small / skin switch (8 | 9 frames) and of the set-up switch (4 | 5): every
  frame's FrameBox is the host fold of its chunk boxes, the record carries the same box, its cone planes, triangle plane,
  margins and pads match a float64 recomputation from its triangle 0, and its chunk-cull bits are a host restatement of the
  verdict in sdf_frame_setup on those planes and margins.  sdf_setup_kernel runs exactly above 4 frames.
* A dense mvs_fit_stream whose slots are refilled and compacted gives every frame the bits mvs_fit gives it.  The host reads
  the active count one chunk late, so the rounds after a compaction run grids sized for more slots than are active, and
  warps of sdf_setup_kernel find no frame."""
import ctypes

import numpy as np
import pytest
import torch

from mvsmplfitting_b200 import synthetic as S
from tests.test_gpu_sdf_setup import LOSS, fold_box, make_ctx, sdf_state
from tests import test_gpu_stream as T

pytestmark = pytest.mark.gpu

SKIN_SETUP_MAX = 4                                      # kSkinSetupMax in mvs_tc.cu: set-ups in skin_small_kernel
REC_WORDS = 52                                          # sizeof(SdfFrameSetup) / 4
F32 = np.float32


def setup_records(ctx, B):
    rec = np.zeros((B, REC_WORDS), np.float32)
    assert ctx.lib.mvs_debug_sdf_setup(ctx.h, rec.ctypes.data_as(ctypes.c_void_p)) == 0
    return rec


def fma32(a, b, c):
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(F32)


def cull_bits(bboxp, tr, rec, G, fused):
    """the chunk-cull verdicts of sdf_frame_setup restated on the host, from the record's box, cone planes and margins.
    fused: (l + 1) * gs -/+ pad as one fused multiply-add (the compiler may contract it) or as two roundings."""
    centre, scale = rec[0:3], rec[3]
    cn, cm = rec[21:30].reshape(3, 3), rec[30:33]
    gs = F32(G) / F32(G - 1)
    pad = F32(F32(2.02) / F32(G - 1)) + F32(1e-5)
    lo = ((bboxp[:, 0:3] + tr[None, :3]) - centre[None]) / scale
    hi = ((bboxp[:, 3:6] + tr[None, :3]) - centre[None]) / scale
    one = F32(1.0)
    if fused:
        wlo, whi = fma32(lo + one, np.full_like(lo, gs), np.full_like(lo, -pad)), fma32(hi + one, np.full_like(hi, gs), np.full_like(hi, pad))
    else:
        wlo, whi = (lo + one) * gs - pad, (hi + one) * gs + pad
    neg = np.zeros(len(bboxp), bool)
    pos = np.zeros(len(bboxp), bool)
    for q in range(3):
        smin = np.zeros(len(bboxp), F32)
        smax = np.zeros(len(bboxp), F32)
        for c in range(3):
            a, b = cn[q, c] * wlo[:, c], cn[q, c] * whi[:, c]
            smin = smin + np.minimum(a, b)
            smax = smax + np.maximum(a, b)
        neg |= smax < -cm[q]
        pos |= smin > cm[q]
    return neg & pos


def check_planes(rec, G, what):
    """the record's cone planes, triangle plane, margins and pads against a float64 recomputation from its triangle 0
    (fitting.py:362-363 in box coordinates); tolerances scale with the products that form each entry"""
    tri = rec[12:21].astype(np.float64).reshape(3, 3)
    cn, cm = rec[21:30].astype(np.float64).reshape(3, 3), rec[30:33].astype(np.float64)
    pn, pd, pm = rec[33:36].astype(np.float64), float(rec[36]), float(rec[37])
    vpad, vpadp = rec[38:41].astype(np.float64), float(rec[41])
    vhalf = 2.02 / (G - 1) + 1e-5
    tol = 1e-5
    for q in range(3):
        ea, eb = tri[q] + 1.0, tri[(q + 1) % 3] + 1.0
        want = np.cross(ea, eb)
        mag = np.linalg.norm(ea) * np.linalg.norm(eb)
        assert np.abs(cn[q] - want).max() <= tol * mag, (what, "cone plane", q, cn[q], want)
        assert abs(cm[q] - 3.5e-4 * np.linalg.norm(want)) <= tol * 3.5e-4 * mag, (what, "cone margin", q)
        assert abs(vpad[q] - vhalf * np.abs(want).sum()) <= tol * vhalf * 3 * mag, (what, "vertex pad", q)
    e1, e2 = tri[1] - tri[0], tri[2] - tri[0]
    want = np.cross(e1, e2)
    mag = np.linalg.norm(e1) * np.linalg.norm(e2)
    assert np.abs(pn - want).max() <= tol * mag, (what, "triangle plane", pn, want)
    assert abs(pd - want @ (tri[0] + 1.0)) <= tol * mag * np.linalg.norm(tri[0] + 1.0) * 3, (what, "plane offset")
    assert abs(pm - 2e-3 * np.linalg.norm(want)) <= tol * 2e-3 * mag, (what, "plane margin")
    assert abs(vpadp - vhalf * np.abs(want).sum()) <= tol * vhalf * 3 * mag, (what, "plane pad")
    assert mag > 0 and np.linalg.norm(want) > 0, (what, "degenerate triangle 0: the case tests little")


def unpack_skip(rec, nbox):
    words = rec[44:52].view(np.uint32)
    c = np.arange(nbox)
    return (words[c // 32] >> (c % 32).astype(np.uint32)) & 1 == 1


@pytest.mark.parametrize("B", [1, 4, 5, 8, 9, 33, 256])
def test_round_setup_matches_host_restatement(B, syn_model, syn_gmm):
    cams = S.make_cameras(4)
    ctx, fr = make_ctx(syn_model, syn_gmm, cams, B, seed=1300 + B)
    try:
        x = torch.tensor(S.pack_params(fr["init"]), device="cuda")
        ctx.profile(0xFFFFFFFF)
        ctx.closure(x)
        prof = ctx.profile_read()
        ctx.profile(0)
        st = sdf_state(ctx, B, ctx.N)
        rec = setup_records(ctx, B)
    finally:
        ctx.close()
    assert prof.get("skin", (0, 0))[1] == 1, prof
    assert prof.get("sdf_setup", (0, 0))[1] == (0 if B <= SKIN_SETUP_MAX else 1), prof
    assert not st["arrive"].any(), "arrival counters not reset after the round"
    nbox = st["bboxp"].shape[1]
    assert nbox <= 256, "the mesh is too large for the chunk cull"
    G = LOSS["sdf_grid"]
    skipped = ambiguous = 0
    for s in range(B):
        want = fold_box(st["bboxp"][s], st["slot_tr"][s])
        assert want.view(np.int32)[:11].tobytes() == st["box"][s].view(np.int32)[:11].tobytes(), "slot %d: FrameBox" % s
        assert rec[s, :11].view(np.int32).tobytes() == st["box"][s].view(np.int32)[:11].tobytes(), "slot %d: record box" % s
        check_planes(rec[s], G, "slot %d" % s)
        got = unpack_skip(rec[s], nbox)
        a = cull_bits(st["bboxp"][s], st["slot_tr"][s], rec[s], G, fused=True)
        b = cull_bits(st["bboxp"][s], st["slot_tr"][s], rec[s], G, fused=False)
        sure = a == b
        assert np.array_equal(got[sure], a[sure]), ("slot %d: chunk-cull bits" % s, np.flatnonzero(got != a)[:16])
        assert (rec[s, 44:52].view(np.uint32)[(nbox + 31) // 32:] == 0).all(), "slot %d: bits past the last chunk" % s
        skipped += int(got.sum())
        ambiguous += int((~sure).sum())
    assert 0 < skipped < B * nbox, "the cull verdicts are all equal: the case tests little"
    assert ambiguous <= B, ambiguous


def test_dense_stream_with_refills_matches_fit(syn_model, syn_gmm):
    """40 frames through 16 slots: skin_kernel + sdf_setup_kernel rounds with refills and compactions, then the skin_small
    tail; against mvs_fit with all 40 frames in one context"""
    F, B = 40, 16
    cams, fr, X0 = T.inputs(syn_model, F, 4040)
    kw = dict(sdf=True, grid=64)
    ref = T.reference(syn_model, syn_gmm, cams, fr, X0, kw)
    assert ref[2]["dense_rounds"] > 0
    ctx = T.make_ctx(syn_model, syn_gmm, cams, B)
    try:
        ctx.profile(0xFFFFFFFF)
        got = T.stream(ctx, fr, X0, kw)
        prof = ctx.profile_read()
        ctx.profile(0)
    finally:
        ctx.close()
    assert prof.get("sdf_setup", (0, 0))[1] > 0, prof
    T.assert_same(ref, got, "F=%d B=%d" % (F, B))
