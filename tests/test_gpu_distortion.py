"""GPU: lens distortion (mvs_set_camera_rigs_dist) on a wide-angle synthetic rig (synthetic.make_wide_cameras: detections out
to normalised radius >= 0.4, tens of pixels of distortion) next to an undistorted rig in the same table.

  * all-zero coefficients give the bits of mvs_set_camera_rigs through the closures, the fitting drivers, the initial guess and
    camera refinement;
  * with coefficients, mvs_closure against the float64 oracle (oracle/distortion_oracle.py) in the frame-resident closure, the
    dense rounds (the SDF term on), the batched chain, VPoser (use_vposer = 2) and use_3d;
  * every frame of a mixed table gets the bits of a context whose only rig is its own;
  * the initial guess undistorts the detections (and leaves confidence-0 rows alone);
  * the camera-refinement view closure against the float64 distorted view term; refinement keeps the coefficients and stays
    at the truth;
  * fit quality with and without the coefficients."""
import numpy as np
import pytest
import torch

from mvsmplfitting_b200 import synthetic as S
from oracle import closure_oracle as O
from oracle import distortion_oracle as D
from tests import golden_util as G
from mvsmplfitting_b200.context import FittingContext
from tests.test_gpu_rigs import DW, GUESS, OPT, closure_raw, new_ctx, same_loss, stage_cfgs

pytestmark = pytest.mark.gpu

TOL = 1e-4                     # the float64 closure comparisons' bar (tests/test_gpu_closure.py)
SEG = ((0, 10), (10, 13), (13, 82), (82, 85), (85, 86))
WIDE_V = 4


def wide(distorted=True):
    return {k: v for k, v in S.make_wide_cameras(WIDE_V, distorted=distorted).items() if k in ("R", "t", "f", "c", "dist")}


def zero_dist(cams):
    return dict(cams, dist=np.zeros((cams["R"].shape[0], 5), np.float32))


def pinhole(cams):
    return {k: cams[k] for k in ("R", "t", "f", "c")}


def table():
    """rig 0: the distorted wide rig; rig 1: an undistorted ring of 3 views"""
    return [wide(), {k: v for k, v in S.make_cameras(3).items() if k in ("R", "t", "f", "c")}]


def data(model, cams_list, rig, seed, noise=2.0):
    """detections of frames with rigs rig [F] (padded rows: zeros), initial rows and 3-D targets"""
    rig = np.asarray(rig, np.int32)
    F, Vm = len(rig), max(c["R"].shape[0] for c in cams_list)
    gt, cf = np.zeros((Vm, F, 17, 2), np.float32), np.zeros((Vm, F, 17), np.float32)
    x0, j3 = np.zeros((F, 86), np.float32), np.zeros((F, 17, 3), np.float32)
    for r, cams in enumerate(cams_list):
        fr = S.make_frames_wide(model, cams, F, seed=seed, noise=noise)
        idx = np.flatnonzero(rig == r)
        V = cams["R"].shape[0]
        gt[:V, idx], cf[:V, idx] = fr["gt_uv"][:, idx], fr["conf"][:, idx]
        x0[idx], j3[idx] = S.pack_params(fr["init"])[idx], fr["gt_joints3d"][idx]
        jw, xt = fr["joint_weights"], S.pack_params(fr["gt"])
    rng = np.random.RandomState(seed + 3)
    return dict(rig=rig, gt_uv=gt, conf=cf, x0=x0, jw=jw, j3=(j3 + rng.normal(0, 0.02, j3.shape)).astype(np.float32),
                c3=rng.uniform(0.5, 1.0, (F, 17)).astype(np.float32), truth=fr["gt_joints3d"], xt=xt)


def ctx_for(model, gmm, B, rigs, mode=0, vposer=False, rig=None):
    ctx = new_ctx(model, gmm, B, rigs=rigs, mode=mode, vposer=vposer)
    if rig is not None and len(rigs) > 1:
        ctx.set_frame_rigs(rig)
    return ctx


def closure_of(model, gmm, rigs, d, cfg_kind, stage, mode, vposer=False, j3d=False, x=None):
    B = len(d["rig"])
    ctx = ctx_for(model, gmm, B, rigs, mode, vposer, d["rig"])
    ctx.set_keypoints(d["gt_uv"], d["conf"], d["jw"])
    if j3d:
        ctx.set_joints3d(d["j3"], d["c3"])
    ctx.set_loss(config=stage_cfgs(ctx, cfg_kind)[stage])
    want = mode != 3
    out = closure_raw(ctx, torch.tensor(d["x0"] if x is None else x, device="cuda"), joints=want, proj=want)
    ctx.close()
    return out


MIXED = np.array([0, 1, 0, 0, 1, 0, 1, 0], np.int32)


@pytest.mark.parametrize("mode,kind,stage,j3d", [(0, "gmm", 1, False), (0, "gmm", 1, True), (1, "gmm", 1, True),
                                                 (3, "bench", 3, False)])
def test_zero_coefficients_closure_bits(mode, kind, stage, j3d, syn_model, syn_gmm):
    cams = table()
    d = data(syn_model, cams, MIXED, 5)
    plain = [pinhole(cams[0]), cams[1]]
    a = closure_of(syn_model, syn_gmm, plain, d, kind, stage, mode, j3d=j3d)
    b = closure_of(syn_model, syn_gmm, [zero_dist(plain[0]), zero_dist(cams[1])], d, kind, stage, mode, j3d=j3d)
    for k in a:
        assert (a[k] is None and b[k] is None) or a[k].tobytes() == b[k].tobytes(), k


def _fit(model, gmm, rigs, d, kind, vposer=False):
    ctx = ctx_for(model, gmm, len(d["rig"]), rigs, vposer=vposer, rig=d["rig"])
    ctx.set_keypoints(d["gt_uv"], d["conf"], d["jw"])
    x = torch.tensor(d["x0"], device="cuda")
    final, st = ctx.fit(x, stage_cfgs(ctx, kind), ctx.make_lbfgs_config(**OPT))
    out = x.cpu().numpy(), final.cpu().numpy()
    ctx.close()
    return out


def _stream(model, gmm, rigs, d, kind, seq=False):
    ctx = ctx_for(model, gmm, 3, rigs)
    x = torch.tensor(d["x0"], device="cuda")
    if seq:
        final, st = ctx.fit_seq_stream(x, d["gt_uv"], d["conf"], d["jw"], [3, 2, 3], stage_cfgs(ctx, kind),
                                       ctx.make_lbfgs_config(**OPT), rig=d["rig"])
    else:
        final, st = ctx.fit_stream(x, d["gt_uv"], d["conf"], d["jw"], stage_cfgs(ctx, kind), ctx.make_lbfgs_config(**OPT),
                                   rig=d["rig"])
    out = x.cpu().numpy(), final.cpu().numpy()
    ctx.close()
    return out


@pytest.mark.parametrize("kind", ["gmm", "bench"])
def test_zero_coefficients_fit_bits(kind, syn_model, syn_gmm):
    """mvs_fit, mvs_fit_stream_rigs and mvs_fit_seq_stream_rigs with the SDF stages off (gmm) and on (bench)"""
    cams = table()
    d = data(syn_model, cams, MIXED, 9)
    plain = [pinhole(cams[0]), cams[1]]
    zero = [zero_dist(plain[0]), cams[1]]
    for run in (lambda r: _fit(syn_model, syn_gmm, r, d, kind), lambda r: _stream(syn_model, syn_gmm, r, d, kind),
                lambda r: _stream(syn_model, syn_gmm, r, d, kind, seq=True)):
        a, b = run(plain), run(zero)
        assert a[0].tobytes() == b[0].tobytes() and same_loss(a[1], b[1])


def _init(model, gmm, rigs, d, rig=None):
    ctx = ctx_for(model, gmm, len(d["rig"]), rigs, rig=d["rig"] if rig is None else rig)
    ctx.set_keypoints(d["gt_uv"], d["conf"], d["jw"])
    ctx.set_loss(config=stage_cfgs(ctx, "gmm")[0])
    x, j = ctx.init_guess(**dict(GUESS, want_joints3d=True))
    out = x.cpu().numpy(), j.cpu().numpy()
    ctx.close()
    return out


def test_zero_coefficients_init_and_refine_bits(syn_model, syn_gmm):
    cams = table()
    d = data(syn_model, cams, MIXED, 13)
    plain = [pinhole(cams[0]), cams[1]]
    zero = [zero_dist(plain[0]), zero_dist(cams[1])]
    a, b = _init(syn_model, syn_gmm, plain, d), _init(syn_model, syn_gmm, zero, d)
    assert a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes()
    ra, rb = _refine(syn_model, syn_gmm, plain, d), _refine(syn_model, syn_gmm, zero, d)
    assert ra[0].tobytes() == rb[0].tobytes() and same_loss(ra[1], rb[1])
    for r in range(2):
        for k in ("R", "t"):
            assert ra[2][r][k].tobytes() == rb[2][r][k].tobytes(), (r, k)
        assert rb[2][r]["dist"].tobytes() == zero[r]["dist"].tobytes()


def _refine(model, gmm, rigs, d, x=None, sweeps=1):
    ctx = ctx_for(model, gmm, 4, rigs)
    xx = torch.tensor(d["x0"] if x is None else x, device="cuda")
    final, out, ca, po = ctx.refine_cameras(xx, d["gt_uv"], d["conf"], d["jw"], stage_cfgs(ctx, "gmm")[3],
                                            ctx.make_lbfgs_config(**OPT), sweeps=sweeps, rig=d["rig"])
    res = xx.cpu().numpy(), final.cpu().numpy(), out
    ctx.close()
    return res


def _oracle(model, gmm, cams, d, kind, stage, j3d=False, vposer_w=None, x=None):
    cfg = stage_cfgs(FittingContext, kind)[stage]
    lc = O.LossConfig(data_weight=cfg.data_weight, body_pose_weight=cfg.body_pose_weight, shape_weight=cfg.shape_weight,
                      bending_prior_weight=cfg.bending_prior_weight, use_vposer=vposer_w is not None, use_3d=j3d)
    om = O.OracleModel.from_numpy(model, dtype=torch.float64)
    pri = O.OraclePriors("l2") if vposer_w is not None else O.OraclePriors.gmm_from_dict(gmm, torch.float64)
    X = d["x0"] if x is None else x
    Z = X[:, 13:45] if vposer_w is not None else None
    return D.closure_eval_batch(om, lc, pri, O.cams_to_torch(cams, torch.float64), cams["dist"], X, d["gt_uv"], d["conf"], d["jw"],
                                d["j3"] if j3d else None, d["c3"] if j3d else None, Z, vposer_w)


def _check(got, ref, joints=True, tag=""):
    errs = dict(loss=G.relmax(got["loss"], ref["loss"]))
    if joints:
        errs["joints"] = G.relmax(got["joints"], ref["joints"])
        errs["proj"] = G.relmax(got["proj"], ref["proj"])
    for a, e in SEG:
        if np.abs(ref["grad"][:, a:e]).max() > 0:
            errs["grad%d" % a] = G.relmax(got["grad"][:, a:e], ref["grad"][:, a:e])
    print(tag, {k: "%.2e" % v for k, v in errs.items()})
    for k, v in errs.items():
        assert v < TOL, (tag, k, v)


@pytest.mark.parametrize("mode,j3d", [(0, False), (0, True), (1, False), (1, True)])
def test_closure_against_float64(mode, j3d, syn_model, syn_gmm):
    """frame-resident closure (0) and batched chain (1), with and without the 3-D term"""
    cams = wide()
    d = data(syn_model, [cams], np.zeros(6, np.int32), 17)
    got = closure_of(syn_model, syn_gmm, [cams], d, "gmm", 1, mode, j3d=j3d)
    _check(got, _oracle(syn_model, syn_gmm, cams, d, "gmm", 1, j3d=j3d), tag="mode %d j3d %d" % (mode, j3d))


def test_closure_against_float64_vposer(syn_model, syn_gmm):
    cams = wide()
    d = data(syn_model, [cams], np.zeros(5, np.int32), 19)
    rng = np.random.RandomState(4)
    d["x0"][:, 13:82] = 0.0
    d["x0"][:, 13:45] = rng.normal(0, 0.3, (5, 32)).astype(np.float32)
    got = closure_of(syn_model, syn_gmm, [cams], d, "vposer", 2, 0, vposer=True)
    ref = _oracle(syn_model, syn_gmm, cams, d, "vposer", 2, vposer_w=G.snapshot_vposer_weights())
    _check(got, ref, tag="vposer")


def test_dense_closure_against_float64(syn_model, syn_gmm):
    """exec mode 3 with the SDF term: the SDF term is camera-free, so the change the coefficients make to the loss and gradient
    is the change they make to the float64 2-D term"""
    cams = wide()
    d = data(syn_model, [cams], np.zeros(6, np.int32), 23)
    a = closure_of(syn_model, syn_gmm, [cams], d, "bench", 3, 3)
    b = closure_of(syn_model, syn_gmm, [pinhole(cams)], d, "bench", 3, 3)
    ra = _oracle(syn_model, syn_gmm, cams, d, "bench", 3)
    rb = _oracle(syn_model, syn_gmm, zero_dist(cams), d, "bench", 3)
    # mode 3 against mode 0 / 1 (SDF off) would not cover the dense rounds: compare the differences
    dl, rl = a["loss"].astype(np.float64) - b["loss"], ra["loss"] - rb["loss"]
    assert G.relmax(dl, rl) < 10 * TOL, (dl, rl)
    # each device gradient is a float32 sum of terms as large as the frame's largest entry (the penetration adjoint, up to 1e6 and
    # more): an entry where they cancel keeps their rounding, so 64 ulps of the frame's largest entry are part of the allowance
    row = np.maximum(np.abs(a["grad"]), np.abs(b["grad"])).max(1, keepdims=True)
    for s, e in SEG:
        dg, rg = a["grad"][:, s:e].astype(np.float64) - b["grad"][:, s:e], ra["grad"][:, s:e] - rb["grad"][:, s:e]
        noise = 64 * np.spacing(row)
        bar = 10 * TOL * max(np.abs(ra["grad"][:, s:e]).max(), 1e-30) + noise
        print("dense segment %d: largest error / allowance %.3f" % (s, float((np.abs(dg - rg) / bar).max())))
        assert (np.abs(dg - rg) < bar).all(), (s, dg, rg, row)
    # and the dense rounds' distorted data term is the frame-resident one's (SDF off): same bits for the same frame
    c0 = closure_of(syn_model, syn_gmm, [cams], d, "gmm", 1, 0)
    c3 = closure_of(syn_model, syn_gmm, [cams], d, "gmm", 1, 3)
    assert np.allclose(c0["loss"], c3["loss"], rtol=1e-5) and np.allclose(c0["grad"], c3["grad"], rtol=1e-4,
                                                                           atol=1e-4 * np.abs(c0["grad"]).max())


@pytest.mark.parametrize("mode", [0, 1])
def test_mixed_table_frames_get_their_rigs_bits(mode, syn_model, syn_gmm):
    cams = table()
    d = data(syn_model, cams, MIXED, 29)
    got = closure_of(syn_model, syn_gmm, cams, d, "gmm", 1, mode, j3d=True)
    for r in range(2):
        idx = np.flatnonzero(MIXED == r)
        V = cams[r]["R"].shape[0]
        dr = dict(d, rig=np.zeros(len(idx), np.int32), gt_uv=d["gt_uv"][:V, idx], conf=d["conf"][:V, idx], x0=d["x0"][idx],
                  j3=d["j3"][idx], c3=d["c3"][idx])
        ref = closure_of(syn_model, syn_gmm, [cams[r]], dr, "gmm", 1, mode, j3d=True)
        for k in ("loss", "grad", "joints"):
            assert got[k][idx].tobytes() == ref[k].tobytes(), (r, k)
        assert got["proj"][:V, idx].tobytes() == ref["proj"].tobytes(), r


@pytest.mark.parametrize("kind", ["gmm", "bench"])
def test_stream_drivers_give_each_frame_its_fit(kind, syn_model, syn_gmm):
    cams = table()
    d = data(syn_model, cams, MIXED, 31)
    ref = _fit(syn_model, syn_gmm, cams, d, kind)
    got = _stream(syn_model, syn_gmm, cams, d, kind)
    assert got[0].tobytes() == ref[0].tobytes() and same_loss(got[1], ref[1])


def _ideal(cams, d):
    """the detections undistorted in float64 (the oracle's Newton inverse), float32"""
    out = d["gt_uv"].copy()
    for v in range(cams["R"].shape[0]):
        out[v] = D.undistort(d["gt_uv"][v], cams["f"][v], cams["c"][v], cams["dist"][v]).astype(np.float32)
    return out


@pytest.mark.parametrize("V", [WIDE_V, 1])
def test_init_guess_undistorts(V, syn_model, syn_gmm):
    """noise-free distorted detections: the guess equals the pinhole guess from the float64-undistorted detections"""
    cams = {k: v[:V] for k, v in wide().items()}
    d = data(syn_model, [cams], np.zeros(8, np.int32), 37, noise=0.0)
    got = _init(syn_model, syn_gmm, [cams], d)
    ref = _init(syn_model, syn_gmm, [pinhole(cams)], dict(d, gt_uv=_ideal(cams, d)))
    assert G.relmax(got[1], ref[1]) < 1e-4 and G.relmax(got[0], ref[0]) < 1e-4, (G.relmax(got[1], ref[1]), G.relmax(got[0], ref[0]))
    # the pinhole guess from the distorted detections is clearly off
    naive = _init(syn_model, syn_gmm, [pinhole(cams)], d)
    assert G.relmax(naive[1], ref[1]) > 1e-3


def test_init_guess_leaves_confidence_0_rows_as_they_stand(syn_model, syn_gmm):
    """a row with confidence 0 is not undistorted: frames whose view 0 saw nothing (every row confidence 0, at arbitrary
    pixels) get the bits of a rig whose view 0 has no distortion; in a one-view rig, frames whose torso rows 5 and 11 have
    confidence 0 get the bits of the pinhole rig.  Frames with confident rows differ (the coefficients are in use)."""
    cams = wide()
    d = data(syn_model, [cams], np.zeros(8, np.int32), 39)
    miss = np.arange(8) % 2 == 0
    d["conf"][0, miss] = 0.0
    d["gt_uv"][0, miss] = np.random.RandomState(2).uniform(-3000, 5000, d["gt_uv"][0, miss].shape).astype(np.float32)
    d["gt_uv"][0, np.flatnonzero(miss)[0]] = 0.0                                          # zero rows too
    view0_plain = dict(cams, dist=cams["dist"].copy())
    view0_plain["dist"][0] = 0.0
    got, ref = _init(syn_model, syn_gmm, [cams], d), _init(syn_model, syn_gmm, [view0_plain], d)
    assert np.isfinite(got[0]).all() and np.isfinite(got[1]).all()
    assert got[0][miss].tobytes() == ref[0][miss].tobytes() and got[1][miss].tobytes() == ref[1][miss].tobytes()
    assert not np.array_equal(got[1][~miss], ref[1][~miss])
    one = {k: v[:1] for k, v in cams.items()}
    d1 = data(syn_model, [one], np.zeros(8, np.int32), 41)
    c = d1["conf"][0].copy()
    c[np.ix_(miss, [5, 11])] = 0.0
    d1["conf"][0] = c
    d1["gt_uv"][0, np.flatnonzero(miss)[0], 5] = 0.0
    got, ref = _init(syn_model, syn_gmm, [one], d1), _init(syn_model, syn_gmm, [pinhole(one)], d1)
    assert np.isfinite(got[0]).all() and np.isfinite(got[1]).all()
    assert got[0][miss].tobytes() == ref[0][miss].tobytes() and got[1][miss].tobytes() == ref[1][miss].tobytes()
    assert not np.array_equal(got[1][~miss], ref[1][~miss])


def _perturbed_table():
    from tests.test_gpu_camera_refine import perturb
    return [perturb(c, 60 + i) for i, c in enumerate(table())]


@pytest.mark.parametrize("at", ["zero", "random"])
def test_camera_closure_against_float64(at, syn_model, syn_gmm):
    """the view closure of mvs_refine_cameras (mvs_debug_camera_closure) on a table of a distorted wide rig and an undistorted
    rig, both miscalibrated, with noisy detections: loss and gradient of every view problem against the float64 view term
    through the view's distortion (distortion_oracle.view_problem), at a zero update and at random updates, to the bars of
    tests/test_gpu_camera_refine.py (1e-5 loss, 1e-4 gradient); the pinhole view term misses the distorted rig's by 10x the bars"""
    from oracle import camera_oracle as CO
    from tests.test_gpu_camera_refine import debug_closure, held, random_rows
    true = table()
    rig = (np.arange(12) % 2).astype(np.int32)
    d = data(syn_model, true, rig, 47)
    d.update(cams=_perturbed_table(), kind="gmm")
    sc = np.array([1.0, 0.75], np.float32)
    q = held(syn_model, syn_gmm, d, d["x0"])
    vps, pin = {}, {}
    for r, cm in enumerate(d["cams"]):
        idx = np.flatnonzero(rig == r)
        dw = np.float32(np.float32(DW) * sc[r])
        for v in range(1, cm["R"].shape[0]):
            args = (cm, v, q[idx], d["gt_uv"][v, idx], d["conf"][v, idx], d["jw"], dw, 100.0, True)
            pin[(r, v)] = CO.ViewProblem(*args)
            vps[(r, v)] = D.view_problem(*args) if "dist" in cm else pin[(r, v)]
    keys = sorted(vps)
    rows_of = (lambda P: np.zeros((P, 86), np.float32)) if at == "zero" else \
        (lambda P: random_rows(P, 7, lambda p: keys[p][1] == 1))
    probs, loss, grad = debug_closure(syn_model, syn_gmm, d, rows_of, sc)
    assert probs == keys
    rows = rows_of(len(keys))
    for p, k in enumerate(keys):
        L, g = vps[k](rows[p])
        gs = np.abs(g).max()
        print(k, "loss %.2e grad %.2e" % (abs(loss[p] - L) / abs(L), np.abs(grad[p] - g).max() / gs))
        assert abs(loss[p] - L) <= 1e-5 * abs(L), (k, loss[p], L)
        assert np.abs(grad[p] - g).max() <= 1e-4 * gs, (k, grad[p][[10, 11, 12, 82, 83, 84]], g[[10, 11, 12, 82, 83, 84]])
        if k[0] == 0:                   # the pinhole view term (and its adjoint) misses the bars by 10x or more: the check bites
            Lp, gp = pin[k](rows[p])
            assert abs(loss[p] - Lp) > 10 * 1e-5 * abs(L) and np.abs(grad[p] - gp).max() > 10 * 1e-4 * gs, k


def test_refinement_keeps_the_coefficients_and_the_truth(syn_model, syn_gmm):
    """exact distorted projections of the true rows: the refined table keeps the coefficients bit for bit and its cameras stay
    at the truth (the closure itself is checked against float64 by test_camera_closure_against_float64)"""
    cams = wide()
    d = data(syn_model, [cams], np.zeros(8, np.int32), 41, noise=0.0)
    d["conf"][:] = 1.0
    x, final, rigs = _refine(syn_model, syn_gmm, [cams], d, x=d["xt"])
    assert rigs[0]["dist"].tobytes() == cams["dist"].tobytes()
    for v in range(WIDE_V):
        dR = np.abs(rigs[0]["R"][v] - cams["R"][v]).max()
        dt = np.abs(rigs[0]["t"][v] - cams["t"][v]).max()
        assert dR < 5e-4 and dt < 5e-3, (v, dR, dt)


def _mpjpe(x, truth, model):
    p = S.unpack_params(x)
    j = S.model_keypoints_np(model, p["betas"], p["global_orient"], p["body_pose"], p["transl"], p["scale"], "smpllsp")
    return float(np.linalg.norm(j - truth, axis=-1).mean())


def test_quality(syn_model, syn_gmm):
    """2 px noise on a wide rig: the fit with the coefficients is as good as an undistorted rig's; ignoring them is not"""
    F = 24
    cams = wide()
    d = data(syn_model, [cams], np.zeros(F, np.int32), 43)
    ctl = data(syn_model, [wide(distorted=False)], np.zeros(F, np.int32), 43)
    on = _fit(syn_model, syn_gmm, [cams], d, "gmm")[0]
    off = _fit(syn_model, syn_gmm, [pinhole(cams)], d, "gmm")[0]
    ctrl = _fit(syn_model, syn_gmm, [wide(distorted=False)], ctl, "gmm")[0]
    e_on, e_off, e_ctl = (_mpjpe(x, d["truth"], syn_model) for x in (on, off, ctrl))
    print("quality: mean 3-D joint error with %.4f, ignoring %.4f, undistorted control %.4f" % (e_on, e_off, e_ctl))
    # first H100 run: 0.0136 with, 0.0242 ignoring, 0.0131 control (model units); bars with margin, each one apart from the
    # fit that ignores the coefficients
    assert e_on < 1.25 * e_ctl
    assert e_off > 1.4 * e_on
