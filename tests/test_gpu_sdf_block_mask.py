"""GPU: the live-block mask of the per-frame SDF set-up (SdfFrameSetup::live_blocks, words 42-43 of the record) and the
CTAs of sdf_fused that retire on it.

* One exec-mode-3 round at batch sizes on both sides of the set-up switch (4 | 5) and of the skinning switch (8 | 9): bit b
  of every frame's mask is set exactly when 256-vertex block b has a chunk (of 64 vertices) that its own skip bits do not
  cull.  The mask is all ones in the all-faces modes (1 and 2) and on a mesh of more than 256 chunks, where nothing is culled.
* sdf_fused with the mask (MVS_SDF_BLOCK_SKIP=1, the default) and without it (=0) writes the same bytes: the per-block sums
  and flags, the flagged blocks' adjoint partials, the loss and the gradient of a round, and every frame of a dense
  mvs_fit_stream of 40 frames through 16 slots with refills.  The knob is read once per process, so each setting runs in a
  process of its own."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from mvsmplfitting_b200 import synthetic as S
from tests.test_gpu_sdf_setup import LOSS, make_ctx
from tests.test_gpu_sdf_setup_kernel import setup_records, unpack_skip

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ALL_ONES = (1 << 64) - 1


def live_mask(rec):
    w = rec[42:44].view(np.uint32)
    return int(w[0]) | (int(w[1]) << 32)


def want_mask(rec, N):
    """bit b: one of block b's chunks below nbox is not culled by the record's own skip bits"""
    nbox, nblocks = (N + 63) // 64, (N + 255) // 256
    skip = unpack_skip(rec, nbox)
    m = 0
    for b in range(nblocks):
        if not skip[4 * b:min(4 * b + 4, nbox)].all():
            m |= 1 << b
    return m


def one_round(ctx, fr):
    x = torch.tensor(S.pack_params(fr["init"]), device="cuda")
    return ctx.closure(x)


@pytest.mark.parametrize("B", [1, 4, 5, 9, 33, 256])
def test_mask_is_the_or_of_the_chunk_verdicts(B, syn_model, syn_gmm):
    ctx, fr = make_ctx(syn_model, syn_gmm, S.make_cameras(4), B, seed=1500 + B)
    try:
        one_round(ctx, fr)
        rec = setup_records(ctx, B)
        N = ctx.N
    finally:
        ctx.close()
    nblocks = (N + 255) // 256
    live = dead = 0
    for s in range(B):
        want = want_mask(rec[s], N)
        assert live_mask(rec[s]) == want, ("slot %d" % s, hex(live_mask(rec[s])), hex(want))
        n = bin(want).count("1")
        live += n
        dead += nblocks - n
    if B >= 5:
        assert live > 0 and dead > 0, ("every block live or every block culled: the case tests little", live, dead)


@pytest.mark.parametrize("all_faces", [1, 2])
def test_mask_all_ones_in_the_all_faces_modes(all_faces, syn_model, syn_gmm):
    B = 2
    ctx, fr = make_ctx(syn_model, syn_gmm, S.make_cameras(4), B, seed=1600 + all_faces)
    try:
        ctx.set_loss(**dict(LOSS, sdf_all_faces=all_faces))
        one_round(ctx, fr)
        rec = setup_records(ctx, B)
    finally:
        ctx.close()
    for s in range(B):
        assert live_mask(rec[s]) == ALL_ONES, ("slot %d" % s, hex(live_mask(rec[s])))
        assert not rec[s, 44:52].view(np.uint32).any(), "slot %d: chunks culled with every face on" % s


def test_mask_all_ones_above_256_chunks(syn_gmm):
    from tests.test_gpu_model_sizes import sized_ctx, sized_frames
    N, B = 27554, 2
    assert (N + 63) // 64 > 256
    cams = S.make_cameras(4)
    fr = sized_frames(N, cams, B, seed=1700)
    ctx = sized_ctx(N, syn_gmm, cams, B, mode=3)
    try:
        ctx.set_keypoints(fr["gt_uv"], fr["conf"], fr["joint_weights"])
        ctx.set_loss(**LOSS)
        ctx.closure(torch.tensor(fr["init"], device="cuda"))
        rec = setup_records(ctx, B)
    finally:
        ctx.close()
    for s in range(B):
        assert live_mask(rec[s]) == ALL_ONES, ("slot %d" % s, hex(live_mask(rec[s])))


BOTH_PATHS_SCRIPT = r"""
import ctypes, sys, numpy as np, torch
sys.path.insert(0, %(root)r)
from tests.test_gpu_sdf_setup import make_ctx, sdf_state
from tests.test_gpu_sdf_setup_kernel import setup_records
from tests.test_gpu_sdf_block_mask import live_mask
from tests import test_gpu_stream as T
from mvsmplfitting_b200 import synthetic as S
model, gmm, cams = S.make_model(0), S.make_gmm(7), S.make_cameras(4)
res = {}
live = dead = 0
for B in (1, 5, 9, 33, 256):
    ctx, fr = make_ctx(model, gmm, cams, B, seed=1800 + B)
    x = torch.tensor(S.pack_params(fr["gt"] if B %% 2 else fr["init"]), device="cuda")
    o = ctx.closure(x)
    N = ctx.N
    nblocks = (N + 255) // 256
    st = sdf_state(ctx, B, N)
    kp = ctx.lib.mvs_debug_sdf_part(ctx.h, None)
    part = np.zeros((B, nblocks, kp), np.float32)
    assert ctx.lib.mvs_debug_sdf_part(ctx.h, part.ctypes.data_as(ctypes.c_void_p)) == 0
    part[st["pflag"] == 0] = 0.0                     # only the flagged blocks' rows are written by a round
    rec = setup_records(ctx, B)
    for s in range(B):
        n = bin(live_mask(rec[s])).count("1")
        live += n; dead += nblocks - n
    res["parts5_%%d" %% B] = st["parts5"]; res["pflag_%%d" %% B] = st["pflag"]; res["part_%%d" %% B] = part
    res["loss_%%d" %% B] = o["loss"].cpu().numpy(); res["grad_%%d" %% B] = o["grad"].cpu().numpy()
    ctx.close()
res["live"] = np.array([live, dead])
cams, fr, X0 = T.inputs(model, 40, 4040)
ctx = T.make_ctx(model, gmm, cams, 16)
ctx.profile(0xFFFFFFFF)
xs, fs, ss = T.stream(ctx, fr, X0, dict(sdf=True, grid=64))
prof = ctx.profile_read()
ctx.close()
res["stream_x"] = xs; res["stream_final"] = fs
res["stream_sums"] = np.array([ss[k] for k in T.SUMS], np.float64)
res["stream_sdf_launches"] = np.array([prof.get("sdf_fused", (0, 0))[1]])
np.savez(%(out)r, **res)
"""


def test_both_paths_write_the_same_bytes(tmp_path):
    runs = {}
    for knob in (0, 1):
        out = str(tmp_path / ("block_skip%d.npz" % knob))
        env = dict(os.environ, MVS_SDF_BLOCK_SKIP=str(knob))
        subprocess.run([sys.executable, "-c", BOTH_PATHS_SCRIPT % dict(root=ROOT, out=out)], env=env, check=True, cwd=ROOT)
        runs[knob] = np.load(out)
    ref, got = runs[0], runs[1]
    live, dead = got["live"]
    assert live > 0 and dead > 0, ("every block live or every block culled: the case tests little", live, dead)
    assert any(ref["pflag_%d" % B].any() for B in (1, 5, 9, 33, 256)), "no flagged block: the adjoint rows test nothing"
    assert ref["stream_sdf_launches"][0] > 0, "the stream ran no dense SDF round"
    for k in ref.files:
        assert ref[k].tobytes() == got[k].tobytes(), "MVS_SDF_BLOCK_SKIP=0 vs 1: %s differs" % k
