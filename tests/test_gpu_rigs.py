"""GPU: frames of one context seen by different camera rigs (mvs_set_camera_rigs, mvs_set_frame_rigs, mvs_fit_stream_rigs,
mvs_fit_seq_stream_rigs).  Three synthetic rigs differ in view count, intrinsics, placement and data-weight scale; frames are
interleaved over them, and the padded view rows (v >= V_r) of gt_uv and conf hold NaN, which proves they are never read.
Oracle for every frame: a context with set_cameras(its rig), detections sliced to the rig's views and every stage's
data_weight = fl32(data_weight x s_r).  Every comparison is exact (np.array_equal; NaN equal to NaN for losses)."""

import numpy as np
import pytest
import torch

from mvsmplfitting_b200 import _lib, seqio
from mvsmplfitting_b200 import synthetic as S
from mvsmplfitting_b200.context import FittingContext, _ptr
from tests import golden_util as G

pytestmark = pytest.mark.gpu

# (views, radius, focal, centre, data-weight scale)
RIGS = ((4, 20.0, 2400.0, (1024.0, 768.0), 1.0), (6, 17.0, 2000.0, (960.0, 540.0), 0.75), (8, 23.0, 2800.0, (1100.0, 820.0), 1.3))
DW = 500.0 / 1536
OPT = dict(max_outer=10)
GUESS = dict(estimate_scale=True, fixed_scale=1.0, use_torso=True, hip_seed=1.0, want_joints3d=False, umeyama_as_written=False)
SENTINEL = 12345.0


def rig_cams(specs=RIGS):
    return [S.make_cameras(V, radius=r, focal=f, center=c) for V, r, f, c, _ in specs]


def rig_scales(specs=RIGS):
    return np.array([s for *_, s in specs], np.float32)


def rig_dw(scale):
    return float(np.float32(np.float32(DW) * np.float32(scale)))


def make_data(model, cams, rig, seed, smooth=False):
    """detections of frames whose rigs are rig [F]: rows v >= V_r are NaN; x0: the synthetic initial guesses; j3 / c3: 3-D
    targets (true joints + noise) and confidences"""
    rig = np.asarray(rig, np.int32)
    F, Vm = len(rig), max(c["R"].shape[0] for c in cams)
    gt = np.full((Vm, F, 17, 2), np.nan, np.float32)
    cf = np.full((Vm, F, 17), np.nan, np.float32)
    x0 = np.zeros((F, 86), np.float32)
    j3 = np.zeros((F, 17, 3), np.float32)
    for r in range(len(cams)):
        fr = S.make_frames(model, cams[r], F, seed=seed, smooth_walk=smooth)        # the same walk, seen by rig r
        idx = np.flatnonzero(rig == r)
        V = cams[r]["R"].shape[0]
        gt[:V, idx], cf[:V, idx] = fr["gt_uv"][:, idx], fr["conf"][:, idx]
        x0[idx] = S.pack_params(fr["init"])[idx]
        j3[idx] = fr["gt_joints3d"][idx]
        jw = fr["joint_weights"]
    rng = np.random.RandomState(seed + 7)
    j3 = (j3 + rng.normal(0, 0.02, j3.shape)).astype(np.float32)
    c3 = rng.uniform(0.5, 1.0, (F, 17)).astype(np.float32)
    return dict(rig=rig, gt_uv=gt, conf=cf, x0=x0, jw=np.asarray(jw, np.float32), j3=j3, c3=c3)


def stage_cfgs(ctx, kind, dw=DW, n=4):
    """'vposer': the shipped configuration (latent pose, L2 prior, no SDF); 'bench': GMM prior, SDF in stages 2-3 (grid 64);
    'gmm': GMM prior, no SDF"""
    sw = S.STAGE_WEIGHTS
    out = []
    for i in range(n):
        on = kind == "bench" and i >= 2
        vp = kind == "vposer"
        out.append(ctx.make_loss_config(body_prior="l2" if vp else "gmm", use_vposer=2 if vp else 0, interpenetration=on,
                                        sdf_grid=64, data_weight=dw, body_pose_weight=sw["body_pose_prior_weights"][i],
                                        shape_weight=sw["shape_weights"][i],
                                        bending_prior_weight=3.17 * sw["body_pose_prior_weights"][i],
                                        coll_loss_weight=sw["coll_loss_weights"][i] if on else 0.0))
    return out


def new_ctx(model, gmm, B, cams=None, rigs=None, scales=None, mode=0, vposer=False):
    ctx = FittingContext(0)
    ctx.set_model(model)
    ctx.set_gmm_from_dict(gmm)
    if rigs is not None:
        ctx.set_camera_rigs(rigs, scales)
    else:
        ctx.set_cameras(cams["R"], cams["t"], cams["f"], cams["c"])
    ctx.set_batch(B)
    ctx.set_exec_mode(mode)
    if vposer:
        ctx.set_vposer(G.snapshot_vposer_weights())
    return ctx


def per_rig(d, cams, r):
    """frames of rig r: their indices and detections sliced to the rig's views"""
    idx = np.flatnonzero(d["rig"] == r)
    V = cams[r]["R"].shape[0]
    return idx, d["gt_uv"][:V, idx], d["conf"][:V, idx]


def closure_raw(ctx, x, joints=True, proj=True):
    B, K = ctx.B, ctx.K
    dev = ctx.device
    out = dict(loss=torch.empty(B, device=dev), grad=torch.empty(B, 86, device=dev))
    out["joints"] = torch.empty(B, K, 3, device=dev) if joints else None
    out["proj"] = torch.full((ctx.V, B, K, 2), SENTINEL, device=dev) if proj else None
    _lib.check(ctx.h, ctx.lib.mvs_closure(ctx.h, _ptr(x), _ptr(out["loss"]), _ptr(out["grad"]), _ptr(out["joints"]),
                                          _ptr(out["proj"]), None, ctx._stream()), "mvs_closure")
    torch.cuda.synchronize()
    return {k: (None if v is None else v.cpu().numpy()) for k, v in out.items()}


def same_loss(a, b):
    return np.array_equal(a, b) or bool(((a == b) | (np.isnan(a) & np.isnan(b))).all())


INTERLEAVED = np.array([0, 1, 2, 2, 0, 1, 1, 2, 0], np.int32)


@pytest.mark.parametrize("mode,kind,j3d", [(0, "gmm", False), (0, "gmm", True), (1, "gmm", True), (3, "bench", False)])
def test_closure(mode, kind, j3d, syn_model, syn_gmm):
    """frame-resident (0), batched chain (1) and dense-round (3, SDF term) closures: loss, gradient, joints, and projections of
    the rig's views; the projection rows of the other views keep their sentinel"""
    cams, sc = rig_cams(), rig_scales()
    d = make_data(syn_model, cams, INTERLEAVED, 11)
    B = len(INTERLEAVED)
    ctx = new_ctx(syn_model, syn_gmm, B, rigs=cams, scales=sc, mode=mode)
    ctx.set_frame_rigs(d["rig"])
    ctx.set_keypoints(d["gt_uv"], d["conf"], d["jw"])
    if j3d:
        ctx.set_joints3d(d["j3"], d["c3"])
    ctx.set_loss(config=stage_cfgs(ctx, kind)[3 if kind == "bench" else 1])
    x = torch.tensor(d["x0"], device="cuda")
    want = mode != 3
    got = closure_raw(ctx, x, joints=want, proj=want)
    ctx.close()
    for r in range(3):
        idx, gt, cf = per_rig(d, cams, r)
        ref = new_ctx(syn_model, syn_gmm, len(idx), cams=cams[r], mode=mode)
        ref.set_keypoints(gt, cf, d["jw"])
        if j3d:
            ref.set_joints3d(d["j3"][idx], d["c3"][idx])
        ref.set_loss(config=stage_cfgs(ref, kind, rig_dw(sc[r]))[3 if kind == "bench" else 1])
        want_ = closure_raw(ref, torch.tensor(d["x0"][idx], device="cuda"), joints=want, proj=want)
        ref.close()
        assert np.array_equal(got["loss"][idx], want_["loss"]), (r, got["loss"][idx], want_["loss"])
        assert np.array_equal(got["grad"][idx], want_["grad"]), r
        if want:
            V = cams[r]["R"].shape[0]
            assert np.array_equal(got["joints"][idx], want_["joints"]), r
            assert np.array_equal(got["proj"][:V, idx], want_["proj"]), r
            assert (got["proj"][V:, idx] == SENTINEL).all(), r


def fit_multi(model, gmm, d, cams, sc, kind, warm=None, vposer=False):
    ctx = new_ctx(model, gmm, len(d["rig"]), rigs=cams, scales=sc, vposer=vposer)
    ctx.set_frame_rigs(d["rig"])
    ctx.set_keypoints(d["gt_uv"], d["conf"], d["jw"])
    x = torch.tensor(d["x0"], device="cuda")
    final, st = ctx.fit(x, stage_cfgs(ctx, kind), ctx.make_lbfgs_config(**OPT), warm=warm)
    out = x.cpu().numpy(), final.cpu().numpy(), st
    ctx.close()
    return out


def fit_per_rig(model, gmm, d, cams, sc, kind, warm=None, vposer=False):
    x = np.zeros_like(d["x0"])
    loss = np.zeros(len(d["rig"]), np.float32)
    tot = dict(frame_iterations=0, frame_evals=0)
    for r in range(len(cams)):
        idx, gt, cf = per_rig(d, cams, r)
        ctx = new_ctx(model, gmm, len(idx), cams=cams[r], vposer=vposer)
        ctx.set_keypoints(gt, cf, d["jw"])
        xr = torch.tensor(d["x0"][idx], device="cuda")
        final, st = ctx.fit(xr, stage_cfgs(ctx, kind, rig_dw(sc[r])), ctx.make_lbfgs_config(**OPT),
                            warm=None if warm is None else np.asarray(warm)[idx])
        x[idx], loss[idx] = xr.cpu().numpy(), final.cpu().numpy()
        for k in tot:
            tot[k] += st[k]
        ctx.close()
    return x, loss, tot


@pytest.mark.parametrize("kind", ["vposer", "bench"])
def test_fit(kind, syn_model, syn_gmm):
    """mvs_fit: the shipped configuration (frame-resident only) and the benchmark schedule (frame-resident + dense rounds)"""
    cams, sc = rig_cams(), rig_scales()
    d = make_data(syn_model, cams, INTERLEAVED, 21)
    vp = kind == "vposer"
    if vp:
        d["x0"][:, 13:82] = 0.0
    got = fit_multi(syn_model, syn_gmm, d, cams, sc, kind, vposer=vp)
    ref = fit_per_rig(syn_model, syn_gmm, d, cams, sc, kind, vposer=vp)
    assert np.array_equal(got[0], ref[0]) and same_loss(got[1], ref[1])
    for k in ref[2]:
        assert got[2][k] == ref[2][k], k
    if kind == "bench":
        assert got[2]["dense_rounds"] > 0


def test_fit_seq_warm_frames(syn_model, syn_gmm):
    cams, sc = rig_cams(), rig_scales()
    d = make_data(syn_model, cams, INTERLEAVED, 31)
    warm = np.arange(len(INTERLEAVED)) % 2 == 1
    got = fit_multi(syn_model, syn_gmm, d, cams, sc, "gmm", warm=warm)
    ref = fit_per_rig(syn_model, syn_gmm, d, cams, sc, "gmm", warm=warm)
    assert np.array_equal(got[0], ref[0]) and same_loss(got[1], ref[1])
    assert got[2]["frame_iterations"] == ref[2]["frame_iterations"] and got[2]["frame_evals"] == ref[2]["frame_evals"]


def test_lbfgs_step(syn_model, syn_gmm):
    cams, sc = rig_cams(), rig_scales()
    d = make_data(syn_model, cams, INTERLEAVED, 41)
    B = len(INTERLEAVED)

    def steps(ctx, x, cfg):
        ctx.set_loss(config=cfg)
        outs = []
        for i in range(3):
            loss, grad, _ = ctx.lbfgs_step(x, ctx.make_lbfgs_config(**OPT), reset=i == 0)
            outs.append((loss.cpu().numpy(), grad.cpu().numpy(), x.cpu().numpy().copy()))
        return outs

    ctx = new_ctx(syn_model, syn_gmm, B, rigs=cams, scales=sc)
    ctx.set_frame_rigs(d["rig"])
    ctx.set_keypoints(d["gt_uv"], d["conf"], d["jw"])
    got = steps(ctx, torch.tensor(d["x0"], device="cuda"), stage_cfgs(ctx, "gmm")[1])
    ctx.close()
    for r in range(3):
        idx, gt, cf = per_rig(d, cams, r)
        ref = new_ctx(syn_model, syn_gmm, len(idx), cams=cams[r])
        ref.set_keypoints(gt, cf, d["jw"])
        want = steps(ref, torch.tensor(d["x0"][idx], device="cuda"), stage_cfgs(ref, "gmm", rig_dw(sc[r]))[1])
        ref.close()
        for (lg, gg, xg), (lw, gw, xw) in zip(got, want):
            assert np.array_equal(lg[idx], lw) and np.array_equal(gg[idx], gw) and np.array_equal(xg[idx], xw), r


@pytest.mark.parametrize("j3d", [False, True])
def test_init_guess_with_a_one_view_rig(j3d, syn_model, syn_gmm):
    """triangulation for the multi-view rigs, the depth guess for the one-view rig -- per frame -- and the 3-D targets when on"""
    specs = ((1, 20.0, 2400.0, (1024.0, 768.0), 1.0),) + RIGS[1:]
    cams, sc = rig_cams(specs), rig_scales(specs)
    d = make_data(syn_model, cams, INTERLEAVED, 51)
    ctx = new_ctx(syn_model, syn_gmm, len(INTERLEAVED), rigs=cams, scales=sc)
    ctx.set_frame_rigs(d["rig"])
    ctx.set_keypoints(d["gt_uv"], d["conf"], d["jw"])
    ctx.set_loss(config=stage_cfgs(ctx, "gmm")[0])
    if j3d:
        ctx.set_joints3d(d["j3"], d["c3"])
    x, j = ctx.init_guess(**dict(GUESS, want_joints3d=True))
    x, j = x.cpu().numpy(), j.cpu().numpy()
    ctx.close()
    for r in range(3):
        idx, gt, cf = per_rig(d, cams, r)
        ref = new_ctx(syn_model, syn_gmm, len(idx), cams=cams[r])
        ref.set_keypoints(gt, cf, d["jw"])
        ref.set_loss(config=stage_cfgs(ref, "gmm")[0])
        if j3d:
            ref.set_joints3d(d["j3"][idx], d["c3"][idx])
        xr, jr = ref.init_guess(**dict(GUESS, want_joints3d=True))
        ref.close()
        assert np.array_equal(x[idx], xr.cpu().numpy()) and np.array_equal(j[idx], jr.cpu().numpy()), r


def test_fit_stream_rigs(syn_model, syn_gmm):
    """F > B frames over three rigs through mvs_fit_stream_rigs, benchmark schedule (frame-resident + dense lanes)"""
    cams, sc = rig_cams(), rig_scales()
    rig = np.array([2, 0, 1, 1, 2, 0, 0, 2, 1, 2, 0, 1, 2, 1], np.int32)
    d = make_data(syn_model, cams, rig, 61)
    ctx = new_ctx(syn_model, syn_gmm, 4, rigs=cams, scales=sc)
    x = torch.tensor(d["x0"], device="cuda")
    final, st = ctx.fit_stream(x, d["gt_uv"], d["conf"], d["jw"], stage_cfgs(ctx, "bench"), ctx.make_lbfgs_config(**OPT),
                               rig=rig)
    got = x.cpu().numpy(), final.cpu().numpy()
    ctx.close()
    ref = fit_per_rig(syn_model, syn_gmm, d, cams, sc, "bench")
    assert np.array_equal(got[0], ref[0]) and same_loss(got[1], ref[1])
    assert st["frame_iterations"] == ref[2]["frame_iterations"] and st["frame_evals"] == ref[2]["frame_evals"]
    assert st["dense_rounds"] > 0


# sequences: the rig of every frame; the last one changes rig from frame to frame
SEQ_RIGS = ([0, 0, 0], [1, 1, 1, 1, 1], [2, 2], [1, 1, 1, 1], [0, 2, 1, 0, 2])


def seq_data(model, cams, seed, no3d=((1, 2), (4, 1))):
    lengths = [len(r) for r in SEQ_RIGS]
    off = np.concatenate([[0], np.cumsum(lengths)])
    parts = [make_data(model, cams, r, seed + s_, smooth=True) for s_, r in enumerate(SEQ_RIGS)]
    d = {k: np.concatenate([p[k] for p in parts], axis=1 if k in ("gt_uv", "conf") else 0) for k in parts[0] if k != "jw"}
    d["jw"] = parts[0]["jw"]
    d["has"] = np.ones(off[-1], bool)
    for s_, t in no3d:
        d["has"][off[s_] + t] = False
    d["j3"][~d["has"]], d["c3"][~d["has"]] = 0.0, 0.0
    return d, lengths, off


def seq_oracle(model, gmm, cams, sc, d, lengths, kind, reinit, j3d):
    """frame by frame on one-slot contexts with only the frame's rig: the cold start point (init_guess, aligned to the 3-D
    target when the frame has one), the warm start from the predecessor's result (load_init + fix_params), mvs_fit_seq"""
    ctxs = {r: new_ctx(model, gmm, 1, cams=cams[r]) for r in range(len(cams))}
    x = np.zeros((len(d["rig"]), 86), np.float32)
    loss = np.zeros(len(d["rig"]), np.float32)
    f = 0
    for T in lengths:
        prev, prev_loss = None, np.float32(np.inf)
        for t in range(T):
            r = int(d["rig"][f])
            ctx, V = ctxs[r], cams[r]["R"].shape[0]
            cfgs = stage_cfgs(ctx, kind, rig_dw(sc[r]))
            ctx.set_keypoints(d["gt_uv"][:V, f:f + 1], d["conf"][:V, f:f + 1], d["jw"])
            ctx.set_loss(config=cfgs[0])
            if j3d and d["has"][f]:
                ctx.set_joints3d(d["j3"][f:f + 1], d["c3"][f:f + 1])
            else:
                ctx.set_joints3d(None)
            cold, _ = ctx.init_guess(**GUESS)
            if j3d:
                ctx.set_joints3d(d["j3"][f:f + 1], d["c3"][f:f + 1])
            warm = prev is not None and prev_loss <= np.float32(reinit)
            params = cold
            if warm:
                params = torch.tensor(prev, device="cuda")
                params[:, 13:82] = cold[:, 13:82]
                params = params.contiguous()
            final, _ = ctx.fit(params, cfgs, ctx.make_lbfgs_config(**OPT), warm=[True] if warm else None)
            x[f], loss[f] = params.cpu().numpy()[0], final.cpu().numpy()[0]
            prev, prev_loss = x[f:f + 1].copy(), loss[f]
            f += 1
    for c in ctxs.values():
        c.close()
    return x, loss


def seq_stream_rigs(model, gmm, cams, sc, d, lengths, kind, reinit, j3d, B=3):
    ctx = new_ctx(model, gmm, B, rigs=cams, scales=sc)
    cfgs = stage_cfgs(ctx, kind)
    t3 = (d["j3"], d["c3"], d["has"]) if j3d else None
    x = seqio._cold_guesses(ctx, d["gt_uv"], d["conf"], d["jw"], cfgs, GUESS, t3, d["rig"], [c["R"].shape[0] for c in cams])
    kw = dict(joints3d=d["j3"], conf3d=d["c3"]) if j3d else {}
    final, st = ctx.fit_seq_stream(x, d["gt_uv"], d["conf"], d["jw"], lengths, cfgs, ctx.make_lbfgs_config(**OPT),
                                   reinit_loss=reinit, rig=d["rig"], **kw)
    out = x.cpu().numpy(), final.cpu().numpy(), st
    ctx.close()
    return out


@pytest.mark.parametrize("kind,j3d", [("gmm", False), ("gmm", True), ("bench", False), ("bench", True)])
def test_fit_seq_stream_rigs(kind, j3d, syn_model, syn_gmm):
    """chaining run c = 0 (every stage frame-resident) and c > 0 (SDF stages 2-3: cold successors park for the earlier run),
    with sequences whose frames change rig"""
    cams, sc = rig_cams(), rig_scales()
    d, lengths, _ = seq_data(syn_model, cams, 71)
    reinit = 5000.0
    if kind == "bench":           # a threshold between the final losses: some later frames start cold and park
        _, l0 = seq_oracle(syn_model, syn_gmm, cams, sc, d, lengths, "gmm", 5000.0, j3d)
        fin = np.sort(l0[np.isfinite(l0)])
        reinit = float(np.float32(0.5 * (fin[len(fin) // 2] + fin[len(fin) // 2 - 1])))
    ref = seq_oracle(syn_model, syn_gmm, cams, sc, d, lengths, kind, reinit, j3d)
    got = seq_stream_rigs(syn_model, syn_gmm, cams, sc, d, lengths, kind, reinit, j3d)
    bad = ~((ref[0] == got[0]).all(1) & ((ref[1] == got[1]) | (np.isnan(ref[1]) & np.isnan(got[1]))))
    assert not bad.any(), np.flatnonzero(bad)


def test_fit_sequences_rigs_against_per_rig_lockstep(syn_model, syn_gmm):
    """seqio.fit_sequences(rigs=...): lock-step (B = S) and stream (B != S) against one lock-step call per rig"""
    cams, sc = rig_cams(), rig_scales()
    seq_rig = [0, 1, 2, 1, 0]
    seqs = []
    for s_, (r, T) in enumerate(zip(seq_rig, (3, 4, 2, 5, 3))):
        fr = S.make_frames(syn_model, cams[r], T, seed=80 + s_, smooth_walk=True)
        seqs.append(dict(gt_uv=fr["gt_uv"], conf=fr["conf"], present=np.ones(fr["conf"].shape[:2], bool),
                         frames=["%05d" % t for t in range(T)], serial="s%02d" % s_, rig=r))
    ref = [None] * len(seqs)
    for r in range(3):
        mine = [s_ for s_, q in enumerate(seqs) if q["rig"] == r]
        ctx = new_ctx(syn_model, syn_gmm, len(mine), cams=cams[r])
        res, _ = seqio.fit_sequences(ctx, [seqs[s_] for s_ in mine], stage_cfgs(ctx, "gmm", rig_dw(sc[r])),
                                     ctx.make_lbfgs_config(**OPT), estimate_scale=True, pose_format="lsp14")
        ctx.close()
        for s_, rr in zip(mine, res):
            ref[s_] = rr
    for B in (len(seqs), 2):
        ctx = new_ctx(syn_model, syn_gmm, B, rigs=cams, scales=sc)
        res, _ = seqio.fit_sequences(ctx, seqs, stage_cfgs(ctx, "gmm"), ctx.make_lbfgs_config(**OPT), estimate_scale=True,
                                     pose_format="lsp14", rigs=cams, rig_data_weight_scale=sc)
        ctx.close()
        for s_ in range(len(seqs)):
            assert np.array_equal(res[s_][0], ref[s_][0]) and same_loss(res[s_][1], ref[s_][1]), (B, s_)


def test_one_rig_equals_set_cameras(syn_model, syn_gmm):
    cams = S.make_cameras(6)
    fr = S.make_frames(syn_model, cams, 6, seed=91)
    outs = []
    for use_rigs in (False, True):
        ctx = new_ctx(syn_model, syn_gmm, 6, rigs=[cams] if use_rigs else None, cams=None if use_rigs else cams)
        ctx.set_keypoints(fr["gt_uv"], fr["conf"], fr["joint_weights"])
        x = torch.tensor(S.pack_params(fr["init"]), device="cuda")
        final, st = ctx.fit(x, stage_cfgs(ctx, "bench"), ctx.make_lbfgs_config(**OPT))
        outs.append((x.cpu().numpy(), final.cpu().numpy(), st))
        ctx.close()
    assert np.array_equal(outs[0][0], outs[1][0]) and same_loss(outs[0][1], outs[1][1]) and outs[0][2] == outs[1][2]


def test_refusals(syn_model, syn_gmm):
    cams, sc = rig_cams(), rig_scales()
    d = make_data(syn_model, cams, INTERLEAVED, 101)
    B = len(INTERLEAVED)
    ctx = new_ctx(syn_model, syn_gmm, 3, rigs=cams, scales=sc)
    cfgs = stage_cfgs(ctx, "gmm")
    # a stream frame naming a rig the context does not have: refused before any fitting work, nothing read out of bounds
    x = torch.tensor(d["x0"], device="cuda")
    x_before = x.clone()
    bad = d["rig"].copy()
    bad[5] = 3
    with pytest.raises(_lib.MvsError, match="frame 5"):
        ctx.fit_stream(x, d["gt_uv"], d["conf"], d["jw"], cfgs, ctx.make_lbfgs_config(**OPT), rig=bad)
    bad[5], bad[2] = 1, -1
    with pytest.raises(_lib.MvsError, match="frame 2"):
        ctx.fit_seq_stream(x, d["gt_uv"], d["conf"], d["jw"], [4, 5], cfgs, ctx.make_lbfgs_config(**OPT), rig=bad)
    assert torch.equal(x, x_before)
    # several rigs and no per-frame rigs
    with pytest.raises(_lib.MvsError, match="camera rigs"):
        ctx.fit_stream(x, d["gt_uv"], d["conf"], d["jw"], cfgs, ctx.make_lbfgs_config(**OPT))
    with pytest.raises(_lib.MvsError, match="camera rigs"):
        ctx.fit_seq_stream(x, d["gt_uv"], d["conf"], d["jw"], [4, 5], cfgs, ctx.make_lbfgs_config(**OPT))
    ctx.close()
    # several rigs and no per-slot rigs: every batch entry point refuses; after set_frame_rigs they run; a stream clears them
    ctx = new_ctx(syn_model, syn_gmm, B, rigs=cams, scales=sc)
    ctx.set_keypoints(d["gt_uv"], d["conf"], d["jw"])
    ctx.set_loss(config=cfgs[0])
    x = torch.tensor(d["x0"], device="cuda")
    for call in (lambda: ctx.closure(x), lambda: ctx.lbfgs_run(x.clone()), lambda: ctx.fit(x.clone(), cfgs),
                 lambda: ctx.init_guess(**GUESS), lambda: ctx.lbfgs_step(x.clone(), reset=True),
                 lambda: ctx.fit(x.clone(), cfgs, warm=np.zeros(B, bool))):
        with pytest.raises(_lib.MvsError, match="per-slot rigs"):
            call()
    ctx.set_frame_rigs(d["rig"])
    ctx.closure(x)
    with pytest.raises(_lib.MvsError):
        ctx.set_frame_rigs(np.full(B, 3))
    ctx.fit_stream(x.clone(), d["gt_uv"], d["conf"], d["jw"], cfgs, ctx.make_lbfgs_config(max_outer=1), rig=d["rig"])
    ctx.set_keypoints(d["gt_uv"], d["conf"], d["jw"])
    with pytest.raises(_lib.MvsError, match="per-slot rigs"):
        ctx.closure(x)
    ctx.close()
    # more than 16 views in a rig
    ctx = FittingContext(0)
    ctx.set_model(syn_model)
    with pytest.raises(_lib.MvsError, match="views"):
        ctx.set_camera_rigs([S.make_cameras(17)])
    ctx.close()
