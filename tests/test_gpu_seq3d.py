"""GPU: video sequences with 3-D joint annotations (use_3d x is_seq).  mvs_fit_seq_stream3d through a context of B slots, and
seqio's drivers with use_3d=True.  Oracle: seqio.fit_sequences on a context with B == S (lock-step, one mvs_fit_seq per time
step after mvs_set_joints3d with that step's rows).  Every frame must get the same parameters (np.array_equal) and final loss
(NaN equal to NaN)."""
import ctypes
import os

import numpy as np
import pytest
import torch

from mvsmplfitting_b200 import seqio
from mvsmplfitting_b200 import synthetic as S
from tests import golden_util as G
from tests.test_gpu_joints3d import stage_cfgs as gmm_stages
from tests.test_gpu_seq_stream import GUESS, OPT, assert_same, cold_after_first, make_ctx, reinit_between, stages

pytestmark = pytest.mark.gpu

LENGTHS = (1, 3, 4, 6, 9)
NO3D = ((1, 1), (3, 0), (3, 4), (4, 8))          # (sequence, frame) pairs without an annotation


def make_seqs(model, cams, lengths, seed, no3d=NO3D):
    """smooth walks with 3-D annotations: true keypoints + 2 cm noise, confidences in [0.5, 1]; the `no3d` frames have
    none (their rows hold values that must not be read)"""
    out = []
    for s_, T in enumerate(lengths):
        fr = S.make_frames(model, cams, T, seed=seed + s_, smooth_walk=True)
        rng = np.random.RandomState(seed + 50 + s_)
        has = np.array([(s_, t) not in no3d for t in range(T)])
        out.append(dict(gt_uv=fr["gt_uv"], conf=fr["conf"], present=np.ones(fr["conf"].shape[:2], bool),
                        frames=["%05d" % t for t in range(T)], serial="s%02d" % s_, has3d=has,
                        joints3d=(fr["gt_joints3d"] + rng.normal(0, 0.02, fr["gt_joints3d"].shape)).astype(np.float32),
                        conf3d=rng.uniform(0.5, 1.0, (T, 17)).astype(np.float32)))
    return out


def lockstep(model, gmm, cams, seqs, sdf=False, vposer=False, reinit=5000.0, use_3d=True):
    ctx = make_ctx(model, gmm, cams, len(seqs), vposer=vposer)
    res, tot = seqio.fit_sequences(ctx, seqs, stages(ctx, sdf, vposer), ctx.make_lbfgs_config(**OPT), estimate_scale=True,
                                   pose_format="lsp14", use_hip=False, reinit_loss=reinit, use_3d=use_3d)
    ctx.close()
    return np.concatenate([r[0] for r in res]), np.concatenate([r[1] for r in res]), tot


def cold_points(ctx, seqs, cfgs):
    gt_uv = np.concatenate([q["gt_uv"] for q in seqs], 1)
    conf = np.concatenate([q["conf"] for q in seqs], 1)
    jw = seqio.joint_weights("lsp14", False)
    t3 = seqio._targets_3d(seqs, cfgs, use_hip=False)
    return gt_uv, conf, jw, t3, seqio._cold_guesses(ctx, gt_uv, conf, jw, cfgs, GUESS, t3)


def seq_stream(model, gmm, cams, seqs, B, sdf=False, vposer=False, reinit=5000.0, launches=None, conf3d=None, joints3d=None):
    """cold start points as fit_sequences computes them, then one mvs_fit_seq_stream3d call on a context of B slots"""
    ctx = make_ctx(model, gmm, cams, B, vposer=vposer)
    cfgs = stages(ctx, sdf, vposer)
    gt_uv, conf, jw, t3, x = cold_points(ctx, seqs, cfgs)
    l0 = ctx.launch_count()
    final, st = ctx.fit_seq_stream(x, gt_uv, conf, jw, [len(q["frames"]) for q in seqs], cfgs, ctx.make_lbfgs_config(**OPT),
                                   reinit_loss=reinit, joints3d=t3[0] if joints3d is None else joints3d,
                                   conf3d=t3[1] if conf3d is None else conf3d)
    if launches is not None:
        launches.append(ctx.launch_count() - l0)
    out = x.cpu().numpy(), final.cpu().numpy(), st
    ctx.close()
    return out


def test_shipped_configuration_frame_resident(syn_model, syn_gmm):
    """VPoser latent pose, L2 prior, SDF off: the frame-resident chaining run reads the F-stride 3-D rows"""
    cams = S.make_cameras(4)
    seqs = make_seqs(syn_model, cams, LENGTHS, 1100)
    ref = lockstep(syn_model, syn_gmm, cams, seqs, vposer=True)
    launches = []
    for B in (1, 2, len(seqs), 8):
        assert_same(ref, seq_stream(syn_model, syn_gmm, cams, seqs, B, vposer=True, launches=launches), "B=%d" % B)
    assert set(launches) == {1}, launches                      # one lbfgs_resident_seq launch per call


def test_benchmark_stages_with_reinitialisation(syn_model, syn_gmm):
    """SDF in stages 2-3: dense chaining, and re-initialised frames take the parking passes with their 3-D rows"""
    cams = S.make_cameras(4)
    seqs = make_seqs(syn_model, cams, LENGTHS, 1200)
    first = lockstep(syn_model, syn_gmm, cams, seqs, sdf=True)
    reinit = reinit_between(first[1])
    ref = lockstep(syn_model, syn_gmm, cams, seqs, sdf=True, reinit=reinit)
    assert cold_after_first(seqs, ref[1], reinit) >= 1
    for B in (1, 3, 8):
        got = seq_stream(syn_model, syn_gmm, cams, seqs, B, sdf=True, reinit=reinit)
        assert_same(ref, got, "B=%d" % B)
        assert got[2]["dense_rounds"] > 0


@pytest.mark.parametrize("sdf", [False, True])
def test_frames_without_annotation(sdf, syn_model, syn_gmm):
    cams = S.make_cameras(4)
    seqs = make_seqs(syn_model, cams, LENGTHS, 1300)
    has = np.concatenate([q["has3d"] for q in seqs])
    base = seq_stream(syn_model, syn_gmm, cams, seqs, 3, sdf=sdf)
    # the zero rows of frames without annotation give the bits of arbitrary targets at confidence 0
    j3 = np.concatenate([q["joints3d"] for q in seqs])
    c3 = np.concatenate([q["conf3d"] for q in seqs])
    c3[:, 11:13] = 0.0
    c3[~has] = 0.0
    assert (j3[~has] != 0).all()
    assert_same(base, seq_stream(syn_model, syn_gmm, cams, seqs, 3, sdf=sdf, joints3d=j3, conf3d=c3), "zero confidence")
    # the term is really on: annotated frames end elsewhere than without the term
    plain = lockstep(syn_model, syn_gmm, cams, seqs, sdf=sdf, use_3d=False)
    assert (base[1][has] != plain[1][has]).all()
    assert (base[0][has] != plain[0][has]).any(1).all()


def test_fit_sequence_batch_equals_stream(syn_model, syn_gmm):
    cams = S.make_cameras(4)
    seq = make_seqs(syn_model, cams, (9,), 1400, no3d=((0, 2), (0, 5)))[0]
    out = []
    for B in (9, 4):
        ctx = make_ctx(syn_model, syn_gmm, cams, B)
        x, loss, _ = seqio.fit_sequence(ctx, seq, stages(ctx, sdf=True), ctx.make_lbfgs_config(**OPT), estimate_scale=True,
                                        pose_format="lsp14", use_hip=False, use_3d=True)
        ctx.close()
        out.append((x, loss))
    assert_same(out[0], out[1], "fit_sequence B=F vs B<F")


def test_refusals_and_context_state(syn_model, syn_gmm):
    from mvsmplfitting_b200 import _lib
    cams = S.make_cameras(4)
    seqs = make_seqs(syn_model, cams, (2, 3), 1500, no3d=((1, 0),))
    F = 5
    ctx = make_ctx(syn_model, syn_gmm, cams, 2)
    cfgs = stages(ctx)
    gt_uv, conf, jw, t3, x = cold_points(ctx, seqs, cfgs)
    dev = lambda a: torch.tensor(a, device="cuda").contiguous()
    g, c, w, j3, c3 = dev(gt_uv), dev(conf), dev(jw), dev(t3[0]), dev(t3[1])
    fin = torch.empty(F, device="cuda")
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    opt = ctx.make_lbfgs_config(**OPT)
    off = np.ascontiguousarray([0, 2, 5], dtype=np.int32)
    s = _lib.SequenceStream(2, off.ctypes.data_as(ctypes.c_void_p), p(x), p(g), p(c), p(w), p(fin), 5000.0)
    arr = (_lib.LossConfig * len(cfgs))(*cfgs)
    call = lambda a, b: ctx.lib.mvs_fit_seq_stream3d(ctx.h, ctypes.byref(s), a, b, len(cfgs), arr, ctypes.byref(opt), None, None)
    assert call(p(j3), None) == -1 and call(None, p(c3)) == -1           # MVS_ERR_INVALID
    with pytest.raises(ValueError):
        ctx.fit_seq_stream(x, g, c, w, [2, 3], cfgs, opt, joints3d=j3)
    with pytest.raises(ValueError):
        ctx.fit_seq_stream(x, g, c, w, [2, 3], cfgs, opt, joints3d=j3[:4], conf3d=c3[:4])
    # a call that runs, with the context's own 3-D term on before it: afterwards no keypoints and the term off
    ctx.set_keypoints(gt_uv[:, :2], conf[:, :2], jw)
    ctx.set_joints3d(t3[0][:2], t3[1][:2])
    assert call(p(j3), p(c3)) == 0
    ctx.set_loss(config=cfgs[3])
    out = torch.empty(2, device="cuda")
    xs = x[:2].contiguous()
    assert ctx.lib.mvs_closure(ctx.h, p(xs), p(out), None, None, None, None, None) == -1
    ctx.set_keypoints(gt_uv[:, :2], conf[:, :2], jw)
    ctx.set_loss(config=cfgs[3])
    assert ctx.lib.mvs_closure(ctx.h, p(xs), p(out), None, None, None, None, None) == 0
    ref = make_ctx(syn_model, syn_gmm, cams, 2)
    ref.set_keypoints(gt_uv[:, :2], conf[:, :2], jw)
    ref.set_loss(config=stages(ref)[3])
    out_ref = torch.empty(2, device="cuda")
    assert ref.lib.mvs_closure(ref.h, p(xs), p(out_ref), None, None, None, None, None) == 0
    assert torch.equal(out, out_ref)                                    # the 3-D term is off
    ref.close()
    ctx.close()


# Bars of the end-to-end comparison with the reference's own main loop (tests/golden/seq3d_e2e.npz).  Measured on an
# NVIDIA H100 80GB HBM3 (700 W); each bar is 4x the worst measured value.
E2E_LOSS_REL = 1.2e-6      # per-frame final loss, relative; measured 3.1e-7 (median 3.1e-8)
E2E_ITER_REL = 0.02        # L-BFGS iterations summed over the frames, relative; measured 0.005 (601 against 604)
E2E_AT_REF_REL = 5e-7      # device closure at the reference's final parameters against the reference's SMPLifyLoss there;
                           # measured 1.3e-7


def test_end_to_end_against_the_reference(syn_model, syn_gmm):
    """the reference's main loop with is_seq and use_3d (oracle/make_golden_seq3d.py), fitted by one mvs_fit_seq_stream3d call
    from the reference's own cold start points (which takes the Umeyama variant out of the comparison)"""
    z = np.load(os.path.join(G.GOLD, "seq3d_e2e.npz"))
    n = int(z["n_seq"])
    cams = {k: z["cam_" + k] for k in ("R", "t", "f", "c")}
    tags = ["s%d_" % s_ for s_ in range(n)]
    seqs = [dict(gt_uv=z[t + "gt_uv"], conf=z[t + "conf"], present=np.ones(z[t + "conf"].shape[:2], bool),
                 frames=["%05d" % i for i in range(z[t + "conf"].shape[1])], serial=t, has3d=z[t + "has3d"],
                 joints3d=z[t + "gt3d"], conf3d=z[t + "conf3d"]) for t in tags]
    assert not np.concatenate([q["has3d"] for q in seqs]).all()
    lengths = [len(q["frames"]) for q in seqs]
    F = sum(lengths)
    jw = z["joint_weights"]
    ctx = make_ctx(syn_model, syn_gmm, cams, 3)
    cfgs = gmm_stages(ctx)
    j3, c3, _ = seqio._targets_3d(seqs, cfgs, use_hip=False)
    gt_uv = np.concatenate([q["gt_uv"] for q in seqs], 1)
    conf = np.concatenate([q["conf"] for q in seqs], 1)
    x = torch.tensor(np.concatenate([z[t + "cold"] for t in tags]), device="cuda")
    final, st = ctx.fit_seq_stream(x, gt_uv, conf, jw, lengths, cfgs, ctx.make_lbfgs_config(), reinit_loss=5000.0,
                                   joints3d=j3, conf3d=c3)
    final = final.cpu().numpy()
    ctx.close()
    ref_final = np.concatenate([z[t + "final_loss"] for t in tags])
    ref_warm = np.concatenate([z[t + "warm"] for t in tags])
    first = np.concatenate([[0], np.cumsum(lengths)[:-1]])
    warm = np.ones(F, bool)
    warm[first] = False
    warm[1:] &= final[:-1] <= np.float32(5000.0)
    assert np.array_equal(warm, ref_warm), (warm, ref_warm)
    rel = np.abs(final - ref_final) / ref_final
    ref_it = sum(int(z[t + "iterations"].sum()) for t in tags)
    it_rel = abs(st["frame_iterations"] - ref_it) / ref_it
    # the device closure at the reference's final parameters, last stage, the same 3-D rows
    ctx = make_ctx(syn_model, syn_gmm, cams, F)
    ctx.set_keypoints(gt_uv, conf, jw)
    ctx.set_joints3d(j3, c3)
    ctx.set_loss(config=gmm_stages(ctx)[3])
    ref_x = np.concatenate([z[t + "params"] for t in tags])
    at = ctx.closure(torch.tensor(ref_x, device="cuda"), want_grad=False)["loss"].cpu().numpy()
    ctx.close()
    ref_at = np.concatenate([z[t + "loss_at_final"] for t in tags])
    at_rel = np.abs(at - ref_at) / np.abs(ref_at)
    print("[seq3d e2e] warm %s; final loss rel max %.2e (median %.2e); iterations device %d reference %d (rel %.3f); "
          "closure at reference params rel max %.2e" % (warm.tolist(), rel.max(), np.median(rel), st["frame_iterations"], ref_it,
                                                        it_rel, at_rel.max()))
    assert rel.max() < E2E_LOSS_REL, rel
    assert it_rel < E2E_ITER_REL, (st["frame_iterations"], ref_it)
    assert at_rel.max() < E2E_AT_REF_REL, at_rel
