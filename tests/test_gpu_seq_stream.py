"""GPU: mvs_fit_seq_stream fits S warm-started video sequences through a context of B slots, a slot taking the next frame of
its sequence as soon as a frame is done.  Oracle: seqio.fit_sequences on a context with B == S (lock-step, one mvs_fit_seq per
time step).  Every frame must get the same parameters (np.array_equal) and final loss (NaN equal to NaN)."""
import ctypes

import numpy as np
import pytest
import torch

from mvsmplfitting_b200 import seqio
from mvsmplfitting_b200 import synthetic as S
from tests import golden_util as G

pytestmark = pytest.mark.gpu

LENGTHS = (1, 3, 4, 6, 9)
OPT = dict(max_outer=10)
GUESS = dict(estimate_scale=True, fixed_scale=1.0, use_torso=True, hip_seed=1.0, want_joints3d=False, umeyama_as_written=False)


def make_ctx(model, gmm, cams, B, mode=0, vposer=False):
    from mvsmplfitting_b200.context import FittingContext
    ctx = FittingContext(0)
    ctx.set_model(model)
    ctx.set_gmm_from_dict(gmm)
    ctx.set_cameras(cams["R"], cams["t"], cams["f"], cams["c"])
    ctx.set_batch(B)
    ctx.set_exec_mode(mode)
    if vposer:
        ctx.set_vposer(G.snapshot_vposer_weights())
    return ctx


def stages(ctx, sdf=False, vposer=False, n=4):
    """the fit_smpl.yaml schedule; the SDF term (grid 64) in stages 2 and 3 when on"""
    sw = S.STAGE_WEIGHTS
    out = []
    for i in range(n):
        on = sdf and i >= 2
        out.append(ctx.make_loss_config(body_prior="l2" if vposer else "gmm", use_vposer=2 if vposer else 0,
                                        interpenetration=on, sdf_grid=64, data_weight=500.0 / 1536,
                                        body_pose_weight=sw["body_pose_prior_weights"][i], shape_weight=sw["shape_weights"][i],
                                        bending_prior_weight=3.17 * sw["body_pose_prior_weights"][i],
                                        coll_loss_weight=sw["coll_loss_weights"][i] if on else 0.0))
    return out


def make_seqs(model, cams, lengths, seed):
    out = []
    for s_, T in enumerate(lengths):
        fr = S.make_frames(model, cams, T, seed=seed + s_, smooth_walk=True)
        out.append(dict(gt_uv=fr["gt_uv"], conf=fr["conf"], present=np.ones(fr["conf"].shape[:2], bool),
                        frames=["%05d" % t for t in range(T)], serial="s%02d" % s_))
    return out


def lockstep(model, gmm, cams, seqs, sdf=False, vposer=False, reinit=5000.0):
    """the oracle: fit_sequences with one slot per sequence"""
    ctx = make_ctx(model, gmm, cams, len(seqs), vposer=vposer)
    res, tot = seqio.fit_sequences(ctx, seqs, stages(ctx, sdf, vposer), ctx.make_lbfgs_config(**OPT), estimate_scale=True,
                                   pose_format="lsp14", reinit_loss=reinit)
    ctx.close()
    return np.concatenate([r[0] for r in res]), np.concatenate([r[1] for r in res]), tot


def seq_stream(model, gmm, cams, seqs, B, sdf=False, vposer=False, reinit=5000.0, launches=None):
    """cold start points as fit_sequences computes them, then one mvs_fit_seq_stream call on a context of B slots"""
    ctx = make_ctx(model, gmm, cams, B, vposer=vposer)
    cfgs = stages(ctx, sdf, vposer)
    gt_uv = np.concatenate([q["gt_uv"] for q in seqs], 1)
    conf = np.concatenate([q["conf"] for q in seqs], 1)
    jw = seqio.joint_weights("lsp14")
    x = seqio._cold_guesses(ctx, gt_uv, conf, jw, cfgs, GUESS)
    l0 = ctx.launch_count()
    final, st = ctx.fit_seq_stream(x, gt_uv, conf, jw, [len(q["frames"]) for q in seqs], cfgs, ctx.make_lbfgs_config(**OPT),
                                   reinit_loss=reinit)
    if launches is not None:
        launches.append(ctx.launch_count() - l0)
    out = x.cpu().numpy(), final.cpu().numpy(), st
    ctx.close()
    return out


def assert_same(ref, got, what):
    xr, lr = ref[:2]
    xs, ls = got[:2]
    bad = ~((xr == xs).all(1) & ((lr == ls) | (np.isnan(lr) & np.isnan(ls))))
    assert not bad.any(), (what, "frames differ", np.flatnonzero(bad)[:16])


def cold_after_first(seqs, loss, reinit):
    """frames after a sequence's first whose predecessor's final loss fails loss <= reinit"""
    n, f = 0, 0
    for q in seqs:
        T = len(q["frames"])
        n += int((~(loss[f:f + T - 1] <= np.float32(reinit))).sum())
        f += T
    return n


def reinit_between(loss):
    """a re-initialisation threshold between the smallest and the largest final loss (float32, as the device compares)"""
    fin = np.sort(loss[np.isfinite(loss)])
    return float(np.float32(0.5 * (fin[len(fin) // 2] + fin[len(fin) // 2 - 1])))


def test_frame_resident_sequences_one_launch(syn_model, syn_gmm):
    cams = S.make_cameras(4)
    seqs = make_seqs(syn_model, cams, LENGTHS, 100)
    ref = lockstep(syn_model, syn_gmm, cams, seqs)
    launches = []
    for B in (1, 2, 5, 8):
        assert_same(ref, seq_stream(syn_model, syn_gmm, cams, seqs, B, launches=launches), "B=%d" % B)
    # one lbfgs_resident launch for the whole call, whatever F is
    seq_stream(syn_model, syn_gmm, cams, seqs[:2], 2, launches=launches)
    assert set(launches) == {1}, launches


def test_sdf_sequences_dense_chaining(syn_model, syn_gmm):
    cams = S.make_cameras(4)
    seqs = make_seqs(syn_model, cams, LENGTHS, 200)
    ref = lockstep(syn_model, syn_gmm, cams, seqs, sdf=True)
    for B in (2, 5, 8):
        got = seq_stream(syn_model, syn_gmm, cams, seqs, B, sdf=True)
        assert_same(ref, got, "B=%d" % B)
        assert got[2]["dense_rounds"] > 0


@pytest.mark.parametrize("sdf", [False, True])
def test_reinitialisation(sdf, syn_model, syn_gmm):
    """frames whose predecessor ended above reinit_loss start cold (with SDF stages: they park and take a second pass)"""
    cams = S.make_cameras(4)
    seqs = make_seqs(syn_model, cams, LENGTHS, 300)
    first = lockstep(syn_model, syn_gmm, cams, seqs, sdf=sdf)
    reinit = reinit_between(first[1])
    ref = lockstep(syn_model, syn_gmm, cams, seqs, sdf=sdf, reinit=reinit)
    assert cold_after_first(seqs, ref[1], reinit) >= 1
    for B in (2, 5):
        assert_same(ref, seq_stream(syn_model, syn_gmm, cams, seqs, B, sdf=sdf, reinit=reinit), "reinit B=%d" % B)


def test_vposer_latent_pose_carries_the_whole_row(syn_model, syn_gmm):
    cams = S.make_cameras(4)
    seqs = make_seqs(syn_model, cams, LENGTHS, 400)
    ref = lockstep(syn_model, syn_gmm, cams, seqs, vposer=True)
    for B in (2, 8):
        assert_same(ref, seq_stream(syn_model, syn_gmm, cams, seqs, B, vposer=True), "vposer B=%d" % B)


def test_stat_sums_equal_the_lockstep(syn_model, syn_gmm):
    cams = S.make_cameras(4)
    seqs = make_seqs(syn_model, cams, (4, 4, 4), 500)
    for sdf in (False, True):
        ref = lockstep(syn_model, syn_gmm, cams, seqs, sdf=sdf)
        got = seq_stream(syn_model, syn_gmm, cams, seqs, 2, sdf=sdf)
        assert_same(ref, got, "sdf=%s" % sdf)
        for k in ("frame_iterations", "frame_evals", "frames_nan"):
            assert ref[2][k] == got[2][k], (sdf, k, ref[2][k], got[2][k])


def test_one_long_video_and_single_frame_sequences(syn_model, syn_gmm):
    cams = S.make_cameras(4)
    video = make_seqs(syn_model, cams, (12,), 600)
    for sdf in (False, True):
        assert_same(lockstep(syn_model, syn_gmm, cams, video, sdf=sdf),
                    seq_stream(syn_model, syn_gmm, cams, video, 4, sdf=sdf), "S=1 sdf=%s" % sdf)
    # sequences of one frame: every frame cold, as mvs_fit gives it
    singles = make_seqs(syn_model, cams, (1,) * 6, 700)
    for sdf in (False, True):
        ctx = make_ctx(syn_model, syn_gmm, cams, 6)
        cfgs = stages(ctx, sdf)
        gt_uv = np.concatenate([q["gt_uv"] for q in singles], 1)
        conf = np.concatenate([q["conf"] for q in singles], 1)
        x = seqio._cold_guesses(ctx, gt_uv, conf, seqio.joint_weights("lsp14"), cfgs, GUESS)
        ctx.set_keypoints(gt_uv, conf, seqio.joint_weights("lsp14"))
        final, _ = ctx.fit(x, cfgs, ctx.make_lbfgs_config(**OPT))
        ref = x.cpu().numpy(), final.cpu().numpy()
        ctx.close()
        for B in (4, 8):
            assert_same(ref, seq_stream(syn_model, syn_gmm, cams, singles, B, sdf=sdf), "singles B=%d sdf=%s" % (B, sdf))


def test_refusals_and_context_state(syn_model, syn_gmm):
    from mvsmplfitting_b200 import _lib
    cams = S.make_cameras(4)
    seqs = make_seqs(syn_model, cams, (2, 3), 800)
    F = 5
    ctx = make_ctx(syn_model, syn_gmm, cams, 2, vposer=True)
    gt_uv = torch.tensor(np.concatenate([q["gt_uv"] for q in seqs], 1), device="cuda")
    conf = torch.tensor(np.concatenate([q["conf"] for q in seqs], 1), device="cuda")
    jw = torch.tensor(seqio.joint_weights("lsp14"), device="cuda")
    x = torch.zeros(F, 86, device="cuda")
    x[:, 85] = 1.0
    fin = torch.empty(F, device="cuda")
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    opt = ctx.make_lbfgs_config(**OPT)

    def raw(offsets, cfgs, n_seq=None):
        off = np.ascontiguousarray(offsets, dtype=np.int32)
        s = _lib.SequenceStream(len(off) - 1 if n_seq is None else n_seq, off.ctypes.data_as(ctypes.c_void_p), p(x), p(gt_uv),
                                p(conf), p(jw), p(fin), 5000.0)
        arr = (_lib.LossConfig * len(cfgs))(*cfgs)
        return ctx.lib.mvs_fit_seq_stream(ctx.h, ctypes.byref(s), len(cfgs), arr, ctypes.byref(opt), None, None)

    cfgs = stages(ctx)
    assert raw([0, 2, 5], cfgs[:2]) == -1                               # n_stages <= 2
    assert raw([0, 2, 2, 5], cfgs) == -1                                # an empty sequence
    assert raw([1, 2, 5], cfgs) == -1                                   # does not start at 0
    assert raw([0, 3, 2], cfgs) == -1                                   # descending
    assert raw([0, 2, 5], cfgs, n_seq=0) == -1
    assert raw([0, 2, 5], cfgs[:1] + stages(ctx, vposer=True)[1:]) == -1       # use_vposer 0 and 2 mixed
    ctx.set_anchor(torch.zeros(2, 86, device="cuda"), torch.ones(2, 86, device="cuda"))
    assert raw([0, 2, 5], cfgs) == -4
    ctx.set_anchor(None)
    for mode in (1, 2):                                                 # batched chain; stages 2 and 3 in separate runs
        ctx.set_exec_mode(mode)
        assert raw([0, 2, 5], cfgs) == -4, mode
    ctx.set_exec_mode(0)
    with pytest.raises(_lib.MvsError):
        ctx.fit_seq_stream(x, gt_uv, conf, jw, [2, 3], cfgs[:2], opt)
    with pytest.raises(ValueError):                                     # lengths that do not add up to F
        ctx.fit_seq_stream(x, gt_uv, conf, jw, [2, 2], cfgs, opt)
    # a call that runs: afterwards the context holds no keypoints
    ctx.set_keypoints(gt_uv[:, :2].cpu().numpy(), conf[:, :2].cpu().numpy(), jw.cpu().numpy())
    assert raw([0, 2, 5], cfgs) == 0
    ctx.set_loss(config=cfgs[0])
    out = torch.empty(2, device="cuda")
    assert ctx.lib.mvs_closure(ctx.h, p(x[:2].contiguous()), p(out), None, None, None, None, None) == -1
    ctx.close()


@pytest.mark.parametrize("B", [2, 7])
def test_fit_sequences_with_another_batch(B, syn_model, syn_gmm, tmp_path):
    import pickle
    cams = S.make_cameras(4)
    seqs = make_seqs(syn_model, cams, (3, 1, 4), 900)
    xr, lr, _ = lockstep(syn_model, syn_gmm, cams, seqs, sdf=True)
    ctx = make_ctx(syn_model, syn_gmm, cams, B)
    res, st = seqio.fit_sequences(ctx, seqs, stages(ctx, sdf=True), ctx.make_lbfgs_config(**OPT), estimate_scale=True,
                                  pose_format="lsp14", result_folder=str(tmp_path))
    ctx.close()
    xs, ls = np.concatenate([r[0] for r in res]), np.concatenate([r[1] for r in res])
    assert_same((xr, lr), (xs, ls), "fit_sequences B=%d" % B)
    f = 0
    for q in seqs:
        for fr in q["frames"]:
            got = pickle.load(open(tmp_path / q["serial"] / fr / "000.pkl", "rb"))
            assert got["loss"] == float(ls[f]) and np.array_equal(got["transl"][0], xs[f, 82:85])
            f += 1
