"""GPU: mvs_fit_stream fits F frames through a context of B < F (or >= F) slots, refilling a slot as soon as its frame is done.
Every frame must get the bits mvs_fit gives it: each case compares against mvs_fit on one context that holds all F frames
(params and final losses np.array_equal, NaN equal to NaN) and requires the same stat sums."""
import ctypes

import numpy as np
import pytest
import torch

from mvsmplfitting_b200 import synthetic as S
from tests import golden_util as G

pytestmark = pytest.mark.gpu

SUMS = ("frame_iterations", "frame_evals", "frames_nan", "dense_frame_evals")


def make_ctx(model, gmm, cams, B, mode=0):
    from mvsmplfitting_b200.context import FittingContext
    ctx = FittingContext(0)
    ctx.set_model(model)
    ctx.set_gmm_from_dict(gmm)
    ctx.set_cameras(cams["R"], cams["t"], cams["f"], cams["c"])
    ctx.set_batch(B)
    ctx.set_exec_mode(mode)
    return ctx


def stages(ctx, sdf=True, grid=64, all_faces=0, vposer=False):
    """the four-stage fit_smpl.yaml schedule, the SDF term (if on) in stages 2 and 3"""
    sw = S.STAGE_WEIGHTS
    out = []
    for i in range(4):
        on = sdf and i >= 2
        out.append(ctx.make_loss_config(body_prior="l2" if vposer else "gmm", use_vposer=2 if vposer else 0,
                                        interpenetration=on, sdf_grid=grid, sdf_all_faces=all_faces,
                                        data_weight=500.0 / 1536, body_pose_weight=sw["body_pose_prior_weights"][i],
                                        shape_weight=sw["shape_weights"][i],
                                        bending_prior_weight=3.17 * sw["body_pose_prior_weights"][i],
                                        coll_loss_weight=sw["coll_loss_weights"][i] if on else 0.0))
    return out


def inputs(model, F, seed, V=4, vposer=False):
    cams = S.make_cameras(V)
    fr = S.make_frames(model, cams, F, seed=seed)
    X0 = S.pack_params(fr["init"])
    if vposer:
        X0[:, 13:82] = 0.0
        X0[:, 13:45] = np.random.RandomState(seed).normal(0, 0.3, size=(F, 32)).astype(np.float32)
    return cams, fr, X0


def prep(ctx, vposer):
    if vposer:
        ctx.set_vposer(G.snapshot_vposer_weights())


def reference(model, gmm, cams, fr, X0, cfg_kw, mode=0, vposer=False, j3d=None, opt=None):
    """mvs_fit with all F frames in one context"""
    F = X0.shape[0]
    ctx = make_ctx(model, gmm, cams, F, mode)
    prep(ctx, vposer)
    ctx.set_keypoints(fr["gt_uv"], fr["conf"], fr["joint_weights"])
    if j3d is not None:
        ctx.set_joints3d(*j3d)
    x = torch.tensor(X0, device="cuda")
    final, st = ctx.fit(x, stages(ctx, **cfg_kw), ctx.make_lbfgs_config(**(opt or {})))
    out = x.cpu().numpy(), final.cpu().numpy(), st
    ctx.close()
    return out


def stream(ctx, fr, X0, cfg_kw, j3d=None, opt=None):
    x = torch.tensor(X0, device="cuda")
    kw = dict(joints3d=j3d[0], conf3d=j3d[1]) if j3d is not None else {}
    final, st = ctx.fit_stream(x, fr["gt_uv"], fr["conf"], fr["joint_weights"], stages(ctx, **cfg_kw),
                               ctx.make_lbfgs_config(**(opt or {})), **kw)
    return x.cpu().numpy(), final.cpu().numpy(), st


def assert_same(ref, got, what):
    xr, fr_, sr = ref
    xs, fs, ss = got
    bad = ~((xr == xs).all(1) & ((fr_ == fs) | (np.isnan(fr_) & np.isnan(fs))))
    assert not bad.any(), (what, "frames differ", np.flatnonzero(bad)[:16])
    for k in SUMS:
        assert sr[k] == ss[k], (what, k, sr[k], ss[k])


def run_stream(model, gmm, cams, fr, X0, B, cfg_kw, mode=0, vposer=False, j3d=None, opt=None):
    ctx = make_ctx(model, gmm, cams, B, mode)
    prep(ctx, vposer)
    out = stream(ctx, fr, X0, cfg_kw, j3d, opt)
    ctx.close()
    return out


def test_sdf_schedule_257_frames_through_64_and_32_slots(syn_model, syn_gmm):
    """refills across skinning groups and down to the N = 8 / skin_small tail; the stream overlaps the chunks' tails"""
    F = 257
    cams, fr, X0 = inputs(syn_model, F, 2570)
    kw = dict(sdf=True, grid=64)
    ref = reference(syn_model, syn_gmm, cams, fr, X0, kw)
    assert ref[2]["dense_rounds"] > 0
    for B in (64, 32):
        got = run_stream(syn_model, syn_gmm, cams, fr, X0, B, kw)
        assert_same(ref, got, "B=%d" % B)
        # the same frames as ceil(F / B) separate mvs_fit calls, one per chunk of B frames
        chunk_rounds = 0
        for c0 in range(0, F, B):
            n = min(B, F - c0)
            sub = dict(gt_uv=np.ascontiguousarray(fr["gt_uv"][:, c0:c0 + n]), conf=np.ascontiguousarray(fr["conf"][:, c0:c0 + n]),
                       joint_weights=fr["joint_weights"])
            xc, fc, sc = reference(syn_model, syn_gmm, cams, sub, X0[c0:c0 + n], kw)
            assert np.array_equal(xc, ref[0][c0:c0 + n])
            chunk_rounds += sc["dense_rounds"]
        print("[stream] F=%d B=%d: dense rounds stream %d, %d chunks one after another %d, one batch of %d: %d"
              % (F, B, got[2]["dense_rounds"], (F + B - 1) // B, chunk_rounds, F, ref[2]["dense_rounds"]))
        assert got[2]["dense_rounds"] < chunk_rounds, (got[2]["dense_rounds"], chunk_rounds)


def test_frame_resident_stream_bitwise_and_one_launch_per_group(syn_model, syn_gmm):
    F = 100
    cams, fr, X0 = inputs(syn_model, F, 1000)
    kw = dict(sdf=False)
    ref = reference(syn_model, syn_gmm, cams, fr, X0, kw)
    ctx = make_ctx(syn_model, syn_gmm, cams, 16)
    launches = []
    for n in (F, 20):
        sub = dict(gt_uv=np.ascontiguousarray(fr["gt_uv"][:, :n]), conf=np.ascontiguousarray(fr["conf"][:, :n]),
                   joint_weights=fr["joint_weights"])
        l0 = ctx.launch_count()
        got = stream(ctx, sub, X0[:n], kw)
        launches.append(ctx.launch_count() - l0)
        if n == F:
            assert_same(ref, got, "resident")
        else:
            assert np.array_equal(got[0], ref[0][:n])
    ctx.close()
    assert launches[0] == launches[1], launches


@pytest.mark.parametrize("F,B", [(5, 8), (8, 8), (1, 8), (19, 8)])
def test_stream_sizes(F, B, syn_model, syn_gmm):
    cams, fr, X0 = inputs(syn_model, F, 700 + F)
    kw = dict(sdf=True, grid=64)
    assert_same(reference(syn_model, syn_gmm, cams, fr, X0, kw), run_stream(syn_model, syn_gmm, cams, fr, X0, B, kw), (F, B))


def test_stream_vposer_decoder_with_sdf(syn_model, syn_gmm):
    F, B = 24, 8
    cams, fr, X0 = inputs(syn_model, F, 2401, vposer=True)
    kw = dict(sdf=True, grid=64, vposer=True)
    assert_same(reference(syn_model, syn_gmm, cams, fr, X0, kw, vposer=True),
                run_stream(syn_model, syn_gmm, cams, fr, X0, B, kw, vposer=True), "vposer")


def test_stream_3d_joint_term(syn_model, syn_gmm):
    F, B = 21, 8
    cams, fr, X0 = inputs(syn_model, F, 3301)
    rng = np.random.RandomState(3302)
    gt3d = (fr["gt_joints3d"] + rng.normal(0, 0.02, size=fr["gt_joints3d"].shape)).astype(np.float32)
    conf3d = rng.uniform(0.5, 1.0, size=gt3d.shape[:2]).astype(np.float32)
    kw = dict(sdf=True, grid=64)
    ref = reference(syn_model, syn_gmm, cams, fr, X0, kw, j3d=(gt3d, conf3d))
    assert_same(ref, run_stream(syn_model, syn_gmm, cams, fr, X0, B, kw, j3d=(gt3d, conf3d)), "3-D term")
    plain = reference(syn_model, syn_gmm, cams, fr, X0, kw)
    assert not np.array_equal(plain[0], ref[0])                       # the term reached the result


def test_stream_all_faces_candidate_lists(syn_model, syn_gmm):
    F, B = 12, 4
    cams, fr, X0 = inputs(syn_model, F, 1212)
    kw = dict(sdf=True, grid=64, all_faces=1)
    opt = dict(max_outer=4)                 # every round evaluates all 13776 faces: a shortened fit keeps the test quick
    assert_same(reference(syn_model, syn_gmm, cams, fr, X0, kw, opt=opt), run_stream(syn_model, syn_gmm, cams, fr, X0, B, kw, opt=opt),
                "all faces")


def test_stream_exec_mode_2_same_bits_as_mode_0(syn_model, syn_gmm):
    F, B = 20, 8
    cams, fr, X0 = inputs(syn_model, F, 2020)
    kw = dict(sdf=True, grid=64)
    a = run_stream(syn_model, syn_gmm, cams, fr, X0, B, kw, mode=0)
    b = run_stream(syn_model, syn_gmm, cams, fr, X0, B, kw, mode=2)
    assert_same(a, b, "exec mode 2")
    assert_same(reference(syn_model, syn_gmm, cams, fr, X0, kw, mode=2), b, "exec mode 2 vs mvs_fit")


def test_stream_refusals_and_context_state(syn_model, syn_gmm):
    from mvsmplfitting_b200 import _lib
    F, B = 6, 4
    cams, fr, X0 = inputs(syn_model, F, 606)
    ctx = make_ctx(syn_model, syn_gmm, cams, B)
    x = torch.tensor(X0, device="cuda")
    args = (fr["gt_uv"], fr["conf"], fr["joint_weights"])
    opt = ctx.make_lbfgs_config()
    lib = ctx.lib

    def raw(s, cfgs, o=opt):
        arr = (_lib.LossConfig * len(cfgs))(*cfgs)
        return lib.mvs_fit_stream(ctx.h, s, len(cfgs), arr, ctypes.byref(o), None, None)

    ctx.set_exec_mode(1)                                               # the batched reference chain has no stream
    with pytest.raises(_lib.MvsError):
        ctx.fit_stream(x, *args, stages(ctx, sdf=True))
    ctx.set_exec_mode(0)
    with pytest.raises(_lib.MvsError):                                 # history 110 without the SDF term: batched chain
        ctx.fit_stream(x, *args, stages(ctx, sdf=False), ctx.make_lbfgs_config(history_size=110))
    anchor = torch.zeros(B, 86, device="cuda")
    ctx.set_anchor(anchor, torch.ones(B, 86, device="cuda"))
    with pytest.raises(_lib.MvsError):
        ctx.fit_stream(x, *args, stages(ctx, sdf=True))
    ctx.set_anchor(None)
    g, c, w = (torch.tensor(a, device="cuda") for a in args)
    j3 = torch.zeros(F, ctx.K, 3, device="cuda")
    fin = torch.empty(F, device="cuda")
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    cfgs = stages(ctx, sdf=True)
    s = _lib.FrameStream(F, p(x), p(g), p(c), p(w), p(j3), None, p(fin))          # gt_xyz without conf3d
    assert raw(ctypes.byref(s), cfgs) == -1
    s = _lib.FrameStream(0, p(x), p(g), p(c), p(w), None, None, p(fin))           # F = 0
    assert raw(ctypes.byref(s), cfgs) == -1
    s = _lib.FrameStream(F, None, p(g), p(c), p(w), None, None, p(fin))           # no parameters
    assert raw(ctypes.byref(s), cfgs) == -1
    assert raw(None, cfgs) == -1
    # after a stream the context holds no keypoints: closures and fits are refused until set_keypoints
    xb = torch.tensor(X0[:B], device="cuda")
    ctx.set_keypoints(fr["gt_uv"][:, :B].copy(), fr["conf"][:, :B].copy(), fr["joint_weights"])
    ctx.fit_stream(x, *args, cfgs)
    ctx.set_loss(config=cfgs[0])
    with pytest.raises(_lib.MvsError):
        ctx.closure(xb)
    with pytest.raises(_lib.MvsError):
        ctx.fit(xb.clone(), cfgs)
    ctx.set_keypoints(fr["gt_uv"][:, :B].copy(), fr["conf"][:, :B].copy(), fr["joint_weights"])
    out = ctx.closure(xb)
    assert torch.isfinite(out["loss"]).all()
    ctx.close()


def test_fit_sequence_through_a_smaller_context(syn_model, syn_gmm):
    from mvsmplfitting_b200 import seqio
    F = 20
    cams = S.make_cameras(4)
    fr = S.make_frames(syn_model, cams, F, seed=2020, smooth_walk=True)
    seq = dict(gt_uv=fr["gt_uv"], conf=fr["conf"], present=np.ones(fr["conf"].shape[:2], bool),
               frames=["%05d" % i for i in range(F)], serial="syn")
    res = []
    for B in (F, 8):
        ctx = make_ctx(syn_model, syn_gmm, cams, B)
        x, loss, st = seqio.fit_sequence(ctx, seq, stages(ctx, sdf=True), ctx.make_lbfgs_config(), estimate_scale=True,
                                         pose_format="lsp14")
        ctx.close()
        res.append((x, loss, st))
    (xa, la, sa), (xb, lb, sb) = res
    assert xa.shape == xb.shape == (F, 86)
    assert np.array_equal(xa, xb) and np.array_equal(la, lb)
    for k in SUMS:
        assert sa[k] == sb[k], (k, sa[k], sb[k])
