"""GPU: the vertex forward and the dense SDF rounds against the float64 oracle (oracle/closure_oracle.py), at every batch size
where the kernel selection changes, across loss configurations and view counts; and bitwise independence of a frame's result
from its slot and from the batch it runs in.

A dense round runs posedirs_gemm_tc, then skin_small_kernel (at most 8 frames) or skin_kernel (32-frame groups, the last CTA
of a group builds the group's SDF set-up), then sdf_fused (1 or 2 blocks per CTA, switching near 29 active frames), then
frame_step.  posedirs_gemm_tc picks its wgmma N instance (8, 16, 32, 64 or 128 frames) from the bound on the active count and
runs column tiles of 128 frames above that.  BATCHES crosses every one of these switches; EDGE_FRAMES holds the first and
last frame of every batch and both sides of every 32-frame edge (so of every 128-frame edge too).

The oracle is fed exactly the float32 constants the context uploads (model, cameras, GMM buffers as set_gmm_from_dict builds
them, parameters), so its float64 result is the same operation carried out in high precision.  Each frame is compared on its
own: vertices and joints relative to that frame's largest |coordinate|, the loss relative to itself, and every gradient
segment (betas, orient, pose, transl, scale) relative to its own largest entry.

The same matrix runs at the limits of the frame-resident kernels (EDGE_CONFIGS, built by tests/model_variants.py): 1, 8 and
9 GMM components, 86, 90 and 91 support vertices, keypoint entries and support-joint pairs past what shared memory stages,
9 skinning weights per vertex, custom keypoint sets of 18 and 32 keypoints on both sides of the view-keypoint limit, and
poses on both sides of the pose-prior and bending cut-offs.  Each case asserts which kernels ran.

Each bar below is at most about 4x the worst value measured on an NVIDIA H100 80GB HBM3 (400 W power limit) and never
looser than the 1e-4 parity bar used elsewhere in the suite; the measured worst case is written next to it.  Every test
prints its worst errors next to its bars (run with -s).
"""
import numpy as np
import pytest
import torch

from mvsmplfitting_b200 import synthetic as S
from oracle import closure_oracle as O
from oracle import sdf_oracle
from tests import golden_util as G
from tests import model_variants as MV

pytestmark = pytest.mark.gpu

BATCHES = (1, 7, 8, 9, 16, 17, 31, 32, 33, 64, 65, 128, 129, 256, 257)
BMAX = max(BATCHES)
EDGE_FRAMES = sorted({0} | {b - 1 for b in BATCHES} | {e + d for e in range(32, BMAX, 32) for d in (-1, 0)})
SEGS = dict(betas=(0, 10), global_orient=(10, 13), body_pose=(13, 82), transl=(82, 85), scale=(85, 86))
# bench.py's stage 2 (cfg_files/fit_smpl.yaml stage 3 of 4), the first stage with the SDF term
W2 = dict(data_weight=500.0 / 1536, body_pose_weight=57.4, shape_weight=10.0, bending_prior_weight=3.17 * 57.4)
# bench.py's last stage (4 of 4): the GMM pose prior is active (its minimum NLL x 4.78^2 stays under the 5e4 cut-off)
W3 = dict(data_weight=500.0 / 1536, body_pose_weight=4.78, shape_weight=5.0, bending_prior_weight=3.17 * 4.78)
F64 = torch.float64

# ---- bars (measured worst on the H100 in the comment)
BAR_GEOM = 1e-6            # A: vertices / joints, both exec modes, both joint sets (worst 2.9e-7)
BAR_LOSS = 1.5e-6          # B: loss, exec modes 0, 1 and 3 (worst 4.4e-7)
BAR_GRAD = dict(betas=5e-6, global_orient=1e-4, body_pose=1e-6, transl=1e-4, scale=1e-4)
#                 B: per segment (worst 1.4e-6, 5.0e-5, 2.5e-7, 2.9e-5, 7.8e-5)
# B at the limits of the frame-resident kernels (EDGE_CONFIGS), exec modes 0, 1 and 3.  The active GMM prior adds a
# 69-term product with the float32 precision matrices to the pose gradient, and the cut-off cases run extreme poses.
BAR_EDGE_LOSS = 1.5e-6     # worst 4.1e-7 (K32_V9)
BAR_EDGE_GRAD = dict(betas=1e-5, global_orient=2e-5, body_pose=5e-6, transl=1.5e-5, scale=1e-4)
#                 worst 2.6e-6 (gmm1), 4.7e-6 (kpe_wide), 1.3e-6 (gmm8), 4.5e-6 (gmm8), 5.2e-5 (cut_l2_s2)
BAR_EDGE_JOINTS = 5e-6     # keypoints relative to the frame's largest |coordinate| (worst 1.3e-6, cut_l2_s3)
BAR_PROJ = 5e-7            # projections relative to the frame's largest |uv| (worst 1.2e-7, cut_l2_s3)
BAR_SDF_LOSS = 2e-5        # C: loss with the real SDF weight (worst 5.2e-6)
BAR_SDF_GRAD = 4e-4        # C: per segment, plus float32 noise (FP32_NOISE); worst 1.4e-4 without the noise allowance,
#                            0.64 of the allowance with it (scale, frame 159)


def make_ctx(model, gmm, cams, B, model_type="smpllsp", mode=0, jmap=None):
    from mvsmplfitting_b200.context import FittingContext
    ctx = FittingContext(0)
    ctx.set_model(model, model_type=model_type, **(jmap or {}))
    ctx.set_gmm_from_dict(gmm)
    ctx.set_cameras(cams["R"], cams["t"], cams["f"], cams["c"])
    ctx.set_batch(B)
    ctx.set_exec_mode(mode)
    return ctx


_OM = {}


def oracle_model(model, model_type, dtype=F64, variant=None, jmap=None):
    key = (model_type, dtype, variant, jmap)
    if key not in _OM:
        kp = MV.KEYPOINT_SETS[jmap] if jmap else {}
        _OM[key] = O.OracleModel.from_numpy(MV.make_variant(variant, model), dtype=dtype, model_type=model_type, **kp)
    return _OM[key]


def oracle_priors(gmm, kind):
    """the float32 buffers FittingContext.set_gmm_from_dict uploads, widened to float64"""
    if kind == "l2":
        return O.OraclePriors("l2")
    means = gmm["means"].astype(np.float32)
    covs = gmm["covars"].astype(np.float32)
    prec = np.stack([np.linalg.inv(c) for c in covs]).astype(np.float32)
    sqrdets = np.array([np.sqrt(np.linalg.det(c)) for c in gmm["covars"]])
    nllw = np.asarray(gmm["weights"] / ((2 * np.pi) ** (69 / 2.0) * (sqrdets / sqrdets.min()))).astype(np.float32)
    t = lambda a: torch.tensor(np.asarray(a, dtype=np.float64), dtype=F64)
    return O.OraclePriors("gmm", t(means), t(prec), t(nllw).unsqueeze(0))


def oracle_forward(om, x):
    parts = [torch.tensor(np.asarray(x[a:e], dtype=np.float64), dtype=om.dtype).view(1, -1) for a, e in SEGS.values()]
    with torch.no_grad():
        v, j, _ = O.smpl_forward(om, *parts)
    return v, j


def oracle_penetration(om, x, coll_loss_weight, grid, all_faces=False):
    v, _ = oracle_forward(om, x)
    return float(sdf_oracle.penetration_loss(v, om.faces, coll_loss_weight, grid, all_faces=all_faces))


class Worst:
    """largest error per quantity, with the frame it came from; printed next to its bar"""

    def __init__(self, title):
        self.title, self.w, self.fail = title, {}, []

    def add(self, key, err, bar, where):
        if key not in self.w or err > self.w[key][0]:
            self.w[key] = (err, bar, where)
        if not err < bar:
            self.fail.append((key, err, bar, where))

    def report(self):
        for k in sorted(self.w, key=str):
            e, bar, where = self.w[k]
            print("[%s] %-34s worst %.3e  bar %.0e  at %s" % (self.title, k, e, bar, where))
        assert not self.fail, self.fail[:8]


def batch_frames(fr, idx):
    idx = np.asarray(idx)
    return np.ascontiguousarray(fr["gt_uv"][:, idx]), np.ascontiguousarray(fr["conf"][:, idx])


# ----------------------------------------------------------------------------------------------------------------- A
@pytest.mark.parametrize("model_type", ["smpllsp", "smpl"])
def test_vertices_and_joints_match_float64_at_every_batch_size(model_type, syn_model, syn_gmm):
    """mvs_forward and closure(want_verts, want_joints) in exec mode 0 (tensor-core posedirs contraction) and exec mode 1
    (fp32 SIMT vertex kernel): all 6890 vertices and all keypoints of the edge frames against smpl_forward in float64, at
    every kernel-selection batch size.  Frame i of every batch is the same frame (the first B of one 257-frame pool), so one
    oracle evaluation checks it everywhere.  Every frame of every batch is also compared bit for bit with the same frame in a
    permuted batch.  Inputs: the generator's ground-truth poses (large rotations, so the pose blend shapes and the partial
    last 128-row posedirs tile matter), betas ~ N(0, 1), scale in [0.85, 1.15]."""
    cams = S.make_cameras(4)
    fr = S.make_frames(syn_model, cams, BMAX, seed=610, model_type=model_type)
    X = S.pack_params(fr["gt"])
    X[:, 85] = np.random.RandomState(611).uniform(0.85, 1.15, BMAX).astype(np.float32)
    om = oracle_model(syn_model, model_type)
    ref = {}
    for i in EDGE_FRAMES:
        v, j = oracle_forward(om, X[i])
        ref[i] = (v.numpy(), j.numpy())
    worst = Worst("A " + model_type)
    for B in BATCHES:
        ctx = make_ctx(syn_model, syn_gmm, cams, B, model_type)
        ctx.set_loss(body_prior="gmm", **W2)
        orders = dict(id=np.arange(B), perm=np.random.RandomState(B).permutation(B)[::-1].copy())
        for mode in (0, 1):
            ctx.set_exec_mode(mode)
            res = {}
            for name, order in orders.items():
                ctx.set_keypoints(*batch_frames(fr, order), fr["joint_weights"])
                x = torch.tensor(np.ascontiguousarray(X[order]), device="cuda")
                f = ctx.forward_only(x)
                c = ctx.closure(x, want_verts=True, want_joints=True)
                torch.cuda.synchronize()
                inv = np.argsort(order)
                res[name] = dict(fwd_v=f["verts"].cpu().numpy()[inv], fwd_j=f["joints"].cpu().numpy()[inv],
                                 cl_v=c["verts"].cpu().numpy()[inv], cl_j=c["joints"].cpu().numpy()[inv])
            for k, a in res["id"].items():
                assert np.isfinite(a).all(), (B, mode, k)
                same = np.array([np.array_equal(a[b], res["perm"][k][b]) for b in range(B)])
                assert same.all(), ("slot dependence", B, mode, k, np.flatnonzero(~same)[:8])
            for i in (i for i in EDGE_FRAMES if i < B):
                vo, jo = ref[i]
                for k in ("fwd", "cl"):
                    ev = np.abs(res["id"][k + "_v"][i] - vo).max() / np.abs(vo).max()
                    ej = np.abs(res["id"][k + "_j"][i] - jo).max() / np.abs(jo).max()
                    worst.add("mode%d verts" % mode, ev, BAR_GEOM, (B, i, k))
                    worst.add("mode%d joints" % mode, ej, BAR_GEOM, (B, i, k))
        ctx.close()
    worst.report()


# ----------------------------------------------------------------------------------------------------------------- B
# one change each from the bench stage-2 configuration (GMM prior, joint confidences, smpllsp, 4 views, rho 100)
CONFIGS = dict(
    base=dict(),
    l2=dict(loss=dict(body_prior="l2")),
    noconf=dict(loss=dict(use_joints_conf=False)),
    fix_shape=dict(loss=dict(fix_shape=True, frozen=("betas",))),
    frozen_scale=dict(loss=dict(frozen=("scale",))),
    frozen_transl=dict(loss=dict(frozen=("transl",))),
    rho10=dict(loss=dict(rho=10.0)),
    smpl=dict(model_type="smpl"),
    anchor=dict(anchor=True),
    V1=dict(V=1),
    V2=dict(V=2),
    V16=dict(V=16),
)
_SEED_INDEX = {n: i for i, n in enumerate(sorted(CONFIGS))}
# The limits of the frame-resident kernels (tests/model_variants.py), each from one side or both.  Keys: model (a variant of
# make_model(0)), gmm_m (components of make_gmm(7, M)), jmap (a custom keypoint set), V, pose (how the checked frames' poses
# are chosen), cut (prior cut-off case: prior kind and body_pose_weight).  The GMM variants run at the last stage's weights
# (W3), where the prior is active, with each checked frame posed near one component's mean so that every component index
# (the last one included) is the minimum somewhere.
EDGE_CONFIGS = dict(
    gmm1=dict(gmm_m=1, weights=W3, pose="gmm_means"),
    gmm8=dict(gmm_m=8, weights=W3, pose="gmm_means"),                    # M = kResMaxM
    gmm9=dict(gmm_m=9, weights=W3, pose="gmm_means"),                    # batched chain
    sup86=dict(model="sup86"),                                           # the real SMPL's support size
    sup90=dict(model="sup90"),                                           # nsup + 6 = kResMaxSup: full support arrays
    sup91=dict(model="sup91"),                                           # batched chain
    kpe_wide=dict(model="kpe_wide"),                                     # 269 keypoint entries: kp_on = 0
    skin_dense=dict(model="skin_dense"),                                 # 531 support-joint pairs: sj_on = 0; KW = 8
    skin_kw9=dict(model="skin_kw9"),                                     # KW = 9: skin_kernel reads the ELL from global
    K18_V15=dict(jmap="K18", V=15),                                      # 270 view-keypoints
    K18_V16=dict(jmap="K18", V=16),                                      # 288: batched chain
    K32_V8=dict(jmap="K32", V=8),                                        # 256
    K32_V9=dict(jmap="K32", V=9),                                        # 288: batched chain
    V16_smpl=dict(model_type="smpl", V=16),                              # 272 with the chain-joint keypoints
    cut_gmm_s3=dict(cut=("gmm", 4.78)),
    cut_gmm_s2=dict(cut=("gmm", 57.4)),
    cut_l2_s3=dict(cut=("l2", 4.78)),
    cut_l2_s2=dict(cut=("l2", 57.4)),
)
_SEED_INDEX.update({n: 100 + i for i, n in enumerate(EDGE_CONFIGS)})
CONFIGS.update(EDGE_CONFIGS)
B_SMALL, B_LARGE = 5, 40            # skin_small_kernel + N = 8;  skin_kernel over two 32-frame groups + N = 64
CHECK_FRAMES = (0, 1, 2, 3, 4, 30, 31, 32, 33, 39)
CW_SMALL = 3e-3                   # SDF term on, but its oracle value stays below 1e-7 of every frame's loss
PPRIOR_CUT, ANGLE_CUT = 5e4, 1e4  # fitting.py:334-335, :349-350
GATE_MARGIN = 1e-3                # no checked frame this close (relative) to a cut-off: the terms are discontinuous there

_VARIANTS, _GMMS = {}, {}


def variant_model(model, name):
    if name not in _VARIANTS:
        _VARIANTS[name] = MV.make_variant(name, model)
    return _VARIANTS[name]


def variant_gmm(gmm, M):
    if M is None:
        return gmm
    if M not in _GMMS:
        _GMMS[M] = S.make_gmm(7, num_gaussians=M)
    return _GMMS[M]


def _frame_rank(i):
    """position of frame i among the checked frames (its own index for the others)"""
    return CHECK_FRAMES.index(i) if i in CHECK_FRAMES else i


def _custom_keypoints(case, rng):
    """detections for a custom keypoint set: the float64 oracle keypoints of the generator's ground truth, projected, plus
    noise; confidences with zeros, one whole view of frame 2 among them; joint_weights of length K"""
    om = oracle_model(case["base"], case["model_type"], variant=case["variant"], jmap=case["jmap"])
    Xg = S.pack_params(case["fr"]["gt"])
    joints = np.stack([oracle_forward(om, Xg[i])[1].numpy() for i in range(B_LARGE)])
    V, K = case["V"], joints.shape[1]
    uv = S.project_np(case["cams"], joints) + rng.normal(0, 5.0, size=(V, B_LARGE, K, 2))
    conf = rng.uniform(0.6, 0.95, size=(V, B_LARGE, K))
    conf[rng.uniform(size=conf.shape) < 0.1] = 0.0
    conf[V - 1, 2] = 0.0
    fr = dict(case["fr"], gt_uv=uv.astype(np.float32), conf=conf.astype(np.float32),
              joint_weights=rng.uniform(0.5, 1.5, K).astype(np.float32))
    return fr


def _pose_at_gates(X, i, kind, bpw, gmm32, rng):
    """pose of frame i with its pose prior and bending term on chosen sides of their cut-offs: the bending entry
    (52, 55, 9 or 12 by frame) sets the bending term, then the other entries are scaled until the pose prior hits its target"""
    k = _frame_rank(i)
    bend = 3.17 * bpw
    p_above, a_above = k % 2 == 1, (k // 2) % 2 == 1
    pose = X[i, 13:82].astype(np.float64)
    e = MV.ANGLE_IDX[k % 4]
    sg = MV.ANGLE_SIGN[k % 4]
    r_a = rng.uniform(1.5, 3.0) if a_above else rng.uniform(0.2, 0.6)
    rest = pose.copy()
    rest[list(MV.ANGLE_IDX)] = 0.0
    base = np.zeros(69)
    base[list(MV.ANGLE_IDX)] = pose[list(MV.ANGLE_IDX)] * 0.1
    others = bend * sum(np.exp(base[j] * s) ** 2 for j, s in zip(MV.ANGLE_IDX, MV.ANGLE_SIGN) if j != e)
    base[e] = sg * 0.5 * np.log((r_a * ANGLE_CUT - others) / bend)
    f = lambda s: MV.prior_gates(base + s * rest, kind, bpw, bend, gmm32)[0]
    if kind == "gmm" and bpw > 10:            # min NLL >= 65 for make_gmm: always above the cut-off at this weight
        s = 1.0
    else:
        target = PPRIOR_CUT * (rng.uniform(2.0, 4.0) if p_above else rng.uniform(0.5, 0.9))
        lo, hi = 0.0, 1.0
        assert f(lo) < target, (i, f(lo), target)
        while f(hi) < target:
            hi *= 2.0
        for _ in range(80):
            mid = 0.5 * (lo + hi)
            lo, hi = (mid, hi) if f(mid) < target else (lo, mid)
        s = 0.5 * (lo + hi)
    X[i, 13:82] = (base + s * rest).astype(np.float32)


def config_case(model, gmm, name, V=None, seed=700):
    """frames, parameters and loss settings of configuration `name`: the model variant, GMM and keypoint set it names, and
    which side of each kernel limit it is on"""
    c = CONFIGS[name]
    V = V if V is not None else c.get("V", 4)
    model_type = c.get("model_type", "smpllsp")
    variant, jmap, M = c.get("model"), c.get("jmap"), c.get("gmm_m")
    mdl, gm = variant_model(model, variant), variant_gmm(gmm, M)
    weights = c.get("weights", W2)
    if "cut" in c:
        kind, bpw = c["cut"]
        weights = dict(W2 if bpw > 10 else W3, body_pose_weight=bpw, bending_prior_weight=3.17 * bpw)
    loss = dict(body_prior="gmm", **weights)
    if "cut" in c:
        loss["body_prior"] = c["cut"][0]
    loss.update(c.get("loss", {}))
    frozen = loss.get("frozen", ())
    cams = S.make_cameras(V)
    fr = S.make_frames(mdl, cams, B_LARGE, seed=seed + _SEED_INDEX[name], model_type=model_type)
    rng = np.random.RandomState(seed)
    X = S.pack_params(fr["init"])
    X[:, 0:10] = 0.5 * fr["gt"]["betas"]
    X[:, 85] = rng.uniform(0.9, 1.1, B_LARGE)
    anchor = weight = None
    if c.get("anchor"):
        anchor = (X + rng.normal(0, 0.05, X.shape)).astype(np.float32)
        weight = rng.uniform(0, 3, X.shape).astype(np.float32)
    kp = MV.KEYPOINT_SETS[jmap] if jmap else {}
    bk = MV.bookkeeping(mdl, model_type, **kp)
    case = dict(name=name, V=V, model_type=model_type, loss=loss, frozen=frozen, cams=cams, fr=fr, X=X, anchor=anchor,
                weight=weight, base=model, variant=variant, jmap=jmap, model=mdl, gmm=gm, kp=kp, bk=bk,
                branches=MV.branches(bk, V, gm["means"].shape[0]))
    if jmap:
        case["fr"] = _custom_keypoints(case, rng)
    gmm32 = MV.gmm_buffers_f32(gm)
    if c.get("pose") == "gmm_means":          # frame i near component (its rank mod M)
        for i in range(B_LARGE):
            X[i, 13:82] = gm["means"][_frame_rank(i) % M] + rng.normal(0, 0.05, 69)
        best = [MV.gmm_nll_min(gmm32, X[i, 13:82])[1] for i in CHECK_FRAMES]
        assert best == [k % M for k in range(len(CHECK_FRAMES))], best
        assert max(MV.prior_gates(X[i, 13:82], "gmm", loss["body_pose_weight"], loss["bending_prior_weight"], gmm32)[0]
                   for i in CHECK_FRAMES) < 0.5 * PPRIOR_CUT
    if "cut" in c:
        kind, bpw = c["cut"]
        for i in range(B_LARGE):
            _pose_at_gates(X, i, kind, bpw, gmm32, rng)
        g = np.array([MV.prior_gates(X[i, 13:82], kind, bpw, 3.17 * bpw, gmm32) for i in CHECK_FRAMES])
        for col, cut in ((0, PPRIOR_CUT), (1, ANGLE_CUT)):
            assert np.abs(g[:, col] / cut - 1.0).min() > GATE_MARGIN, (name, col, g[:, col])
        above = g / np.array([PPRIOR_CUT, ANGLE_CUT]) > 1.0
        assert (above[:, 1].sum() >= 3 and (~above[:, 1]).sum() >= 3), (name, g[:, 1])
        if kind == "gmm" and bpw > 10:
            assert above[:, 0].all(), (name, g[:, 0])            # the GMM term is always cut at this weight
        else:
            assert above[:, 0].sum() >= 3 and (~above[:, 0]).sum() >= 3, (name, g[:, 0])
        case["gates"] = g
    return case


def oracle_case(case):
    """the float64 oracle of the CHECK_FRAMES of a case"""
    om = oracle_model(case["base"], case["model_type"], variant=case["variant"], jmap=case["jmap"])
    lo = case["loss"]
    cfg = O.LossConfig(rho=lo.get("rho", 100.0), use_joints_conf=lo.get("use_joints_conf", True),
                       fix_shape=lo.get("fix_shape", False),
                       **{k: lo[k] for k in ("data_weight", "body_pose_weight", "shape_weight", "bending_prior_weight")})
    pri = oracle_priors(case["gmm"], lo["body_prior"])
    cams_t = O.cams_to_torch(case["cams"], F64)
    fr, X = case["fr"], case["X"]
    ref = {}
    for i in CHECK_FRAMES:
        r = O.closure_eval(om, cfg, pri, cams_t, X[i], fr["gt_uv"][:, i], fr["conf"][:, i], fr["joint_weights"])
        loss, grad = r["loss"], r["grad"].astype(np.float64)
        if case["anchor"] is not None:
            d = X[i].astype(np.float64) - case["anchor"][i].astype(np.float64)
            w = case["weight"][i].astype(np.float64)
            loss = loss + float((w * d * d).sum())
            grad = grad + 2 * w * d
        for f in case["frozen"]:
            a, e = SEGS[f]
            grad[a:e] = 0.0
        res = np.abs(fr["gt_uv"][:, i].astype(np.float64) - r["proj"]).max()
        ref[i] = dict(loss=loss, grad=grad, res=res, joints=r["joints"], proj=r["proj"])
    return ref


def case_ctx(case, B, mode=0):
    return make_ctx(case["model"], case["gmm"], case["cams"], B, case["model_type"], mode, case["kp"])


def run_closure(ctx, case, B, mode, sdf, want_geom=False):
    fr, X = case["fr"], case["X"]
    ctx.set_exec_mode(mode)
    ctx.set_keypoints(*batch_frames(fr, range(B)), fr["joint_weights"])
    if case["anchor"] is not None:
        ctx.set_anchor(torch.tensor(case["anchor"][:B]), torch.tensor(case["weight"][:B]))
    kw = dict(case["loss"])
    if sdf:
        kw.update(interpenetration=True, coll_loss_weight=CW_SMALL, sdf_grid=128)
    ctx.set_loss(**kw)
    x = torch.tensor(X[:B], device="cuda")
    ctx.profile(0xFFFFFFFF)
    out = ctx.closure(x, want_joints=want_geom, want_proj=want_geom)
    prof = ctx.profile_read()
    ctx.profile(0)
    res = (out["loss"].cpu().numpy(), out["grad"].cpu().numpy(), prof)
    if want_geom:
        res += (out["joints"].cpu().numpy(), out["proj"].cpu().numpy())
    return res


def compare_case(worst, tag, case, ref, loss, grad, B):
    edge = case["name"] in EDGE_CONFIGS
    bar_loss, bar_grad = (BAR_EDGE_LOSS, BAR_EDGE_GRAD) if edge else (BAR_LOSS, BAR_GRAD)
    for i in (i for i in CHECK_FRAMES if i < B):
        worst.add(tag + " loss", abs(float(loss[i]) - ref[i]["loss"]) / abs(ref[i]["loss"]), bar_loss, (B, i))
        for n, (a, e) in SEGS.items():
            if n in case["frozen"]:
                assert np.all(grad[i, a:e] == 0.0), (tag, B, i, n, "frozen segment must be exactly zero")
                continue
            worst.add(tag + " grad " + n, G.relmax(grad[i, a:e], ref[i]["grad"][a:e]), bar_grad[n], (B, i))


@pytest.mark.parametrize("name", list(CONFIGS))
def test_dense_closure_matches_float64(name, syn_model, syn_gmm):
    """Exec mode 3 (one evaluation through posedirs_gemm_tc -> skin -> sdf_fused -> frame_step) against closure_eval in
    float64: loss and each gradient segment of frames 0-4 at B = 5 (skin_small_kernel, N = 8) and of frames on both sides of
    the 32-frame edge at B = 40 (skin_kernel, N = 64, 2 blocks per sdf_fused CTA).  The SDF term is on with a weight so small
    that the oracle's penetration term stays below 1e-7 of every compared loss (asserted), so the comparison isolates the
    data and prior arithmetic from the discontinuous as-written SDF field.  Frozen segments must be exactly zero, and frames
    0-4 must give the same bits at B = 5 and at B = 40.  A configuration outside the frame-resident envelope (more support
    vertices, view-keypoints or GMM components than frame_step holds) must run the batched chain instead."""
    case = config_case(syn_model, syn_gmm, name)
    ref = oracle_case(case)
    om = oracle_model(syn_model, case["model_type"], variant=case["variant"], jmap=case["jmap"])
    pen_ratio = max(oracle_penetration(om, case["X"][i], CW_SMALL, 128) / ref[i]["loss"] for i in CHECK_FRAMES)
    assert pen_ratio < 1e-7, pen_ratio
    if name == "rho10":         # frames whose residuals reach GMoF's saturating region
        assert max(r["res"] for r in ref.values()) > 3 * case["loss"]["rho"]
    worst = Worst("B dense " + name)
    bits = {}
    for B in (B_SMALL, B_LARGE):
        ctx = case_ctx(case, B)
        loss, grad, prof = run_closure(ctx, case, B, 3, sdf=True)
        ctx.close()
        if case["branches"]["resident"]:
            assert prof.get("frame_step", (0, 0))[1] == 1 and prof.get("skin", (0, 0))[1] == 1, prof
            assert "keypoint_loss" not in prof, prof                # not the batched reference chain
        else:
            assert "keypoint_loss" in prof and "frame_step" not in prof and "skin" not in prof, prof
        compare_case(worst, "mode3", case, ref, loss, grad, B)
        bits[B] = (loss[:B_SMALL], grad[:B_SMALL])
    assert np.array_equal(bits[B_SMALL][0], bits[B_LARGE][0]) and np.array_equal(bits[B_SMALL][1], bits[B_LARGE][1])
    print("[B dense %s] oracle penetration / loss <= %.2e" % (name, pen_ratio))
    worst.report()


@pytest.mark.parametrize("V", [1, 2])
@pytest.mark.parametrize("name", [n for n in CONFIGS if not n.startswith("V") and n not in EDGE_CONFIGS])
def test_resident_and_batched_closure_match_float64_few_views(name, V, syn_model, syn_gmm):
    """The configuration matrix of test_dense_closure_matches_float64 without the SDF term, at one and two views, through the
    frame-resident closure (exec mode 0) and the batched kernel chain (exec mode 1), against closure_eval in float64."""
    case = config_case(syn_model, syn_gmm, name, V=V)
    ref = oracle_case(case)
    worst = Worst("B V=%d %s" % (V, name))
    for B in (B_SMALL, B_LARGE):
        ctx = case_ctx(case, B)
        for mode, kid in ((0, "closure_resident"), (1, "keypoint_loss")):
            loss, grad, prof = run_closure(ctx, case, B, mode, sdf=False)
            assert kid in prof, (mode, prof)
            compare_case(worst, "mode%d" % mode, case, ref, loss, grad, B)
        ctx.close()
    worst.report()


@pytest.mark.parametrize("name", list(EDGE_CONFIGS))
def test_closure_at_the_resident_limits_matches_float64(name, syn_model, syn_gmm):
    """Exec mode 0 (the frame-resident closure where the configuration fits it, the batched chain where it does not) and
    exec mode 1 (the batched chain) at the limits of the frame-resident kernels: loss, keypoints, projections and every
    gradient segment of the checked frames against closure_eval in float64, at B = 5 and B = 40.  Which kernel ran is read
    from the profile; the branch each configuration reaches inside the kernel is asserted from the host mirror of
    mvs_set_model (tests/test_model_variants.py)."""
    case = config_case(syn_model, syn_gmm, name)
    ref = oracle_case(case)
    br = case["branches"]
    if "gates" in case:
        print("[B limits %s] pose prior / 5e4: %s   bending / 1e4: %s" % (
            name, np.round(case["gates"][:, 0] / PPRIOR_CUT, 2).tolist(), np.round(case["gates"][:, 1] / ANGLE_CUT, 2).tolist()))
    worst = Worst("B limits " + name)
    for B in (B_SMALL, B_LARGE):
        ctx = case_ctx(case, B)
        for mode in (0, 1):
            loss, grad, prof, joints, proj = run_closure(ctx, case, B, mode, sdf=False, want_geom=True)
            if mode == 0 and br["resident"]:
                assert "closure_resident" in prof and "keypoint_loss" not in prof, prof
            else:
                assert "keypoint_loss" in prof and "closure_resident" not in prof, (mode, prof)
            tag = "mode%d" % mode
            compare_case(worst, tag, case, ref, loss, grad, B)
            for i in (i for i in CHECK_FRAMES if i < B):
                jo, po = ref[i]["joints"], ref[i]["proj"]
                worst.add(tag + " joints", np.abs(joints[i] - jo).max() / np.abs(jo).max(), BAR_EDGE_JOINTS, (B, i))
                worst.add(tag + " proj", np.abs(proj[:, i] - po).max() / np.abs(po).max(), BAR_PROJ, (B, i))
        ctx.close()
    worst.report()


# ----------------------------------------------------------------------------------------------------------------- C
# A frame is left out of the oracle comparison only where the oracle's own float32 and float64 penetration values differ by
# more than this (relative): a voxel whose inside / outside parity flips between the two.  Ordinary float32 rounding of the
# term, a sum of 6890 sampled distances with cancellation, stays below about 4e-5 on the edge frames.
PARITY_REL = 1e-4
# The as-written term is invariant, in exact arithmetic, under the scale and translation of the body (every vertex is sampled
# in the normalised coordinates of the frame's own bounding box).  Its contributions to the scale and transl gradients cancel
# to rounding noise, which in float32 is large where the term dominates the loss: the float32 oracle's own scale gradient is
# 8e-2 off the float64 value on frame 223, where the kernel is 6e-2 off.  A gradient segment may therefore differ from the
# float64 oracle by BAR_SDF_GRAD times its largest |entry| plus FP32_NOISE times the float32 oracle's own deviation, so that
# the bar measures the kernel against what float32 can resolve.
FP32_NOISE = 4.0
SDF_CASES = dict(as_written=dict(coll_loss_weight=1000.0, sdf_grid=128, sdf_all_faces=0),
                 all_faces=dict(coll_loss_weight=0.05, sdf_grid=16, sdf_all_faces=1))


@pytest.mark.parametrize("sdf", list(SDF_CASES))
def test_dense_closure_with_sdf_slot_independent_and_matches_float64(sdf, syn_model, syn_gmm):
    """Exec mode 3 with the real SDF weight at every kernel-selection batch size.  Frame i of every batch is frame i of one
    257-frame pool.  Every frame's loss and gradient must be bit-identical in the batch reversed; the edge frames must be
    bit-identical to the same frame evaluated alone (B = 1).  The edge frames are compared with the float64 oracle; a frame
    is left out only where the oracle's own float32 and float64 penetration values differ by more than PARITY_REL (the
    as-written field can flip a voxel's inside / outside parity), at least 90 % of them must be compared, and the compared
    ones must include penetrating frames."""
    sc = SDF_CASES[sdf]
    cams = S.make_cameras(4)
    fr = S.make_frames(syn_model, cams, BMAX, seed=820)
    X = S.pack_params(fr["init"])
    rng = np.random.RandomState(821)
    X[:, 0:10] = 0.5 * fr["gt"]["betas"]
    X[:, 85] = rng.uniform(0.9, 1.1, BMAX)
    loss_kw = dict(body_prior="gmm", interpenetration=True, **sc, **W2)
    # the float64 oracle of the edge frames, and the float32 / float64 penetration agreement that decides exclusion
    om64, om32 = oracle_model(syn_model, "smpllsp"), oracle_model(syn_model, "smpllsp", torch.float32)
    cfg = O.LossConfig(interpenetration=True, coll_loss_weight=sc["coll_loss_weight"], sdf_grid=sc["sdf_grid"],
                       sdf_all_faces=bool(sc["sdf_all_faces"]), **W2)
    pri, pri32 = oracle_priors(syn_gmm, "gmm"), O.OraclePriors.gmm_from_dict(syn_gmm, torch.float32)
    cams_t, cams32 = O.cams_to_torch(cams, F64), O.cams_to_torch(cams, torch.float32)
    ref, excluded = {}, []
    for i in EDGE_FRAMES:
        args = (sc["coll_loss_weight"], sc["sdf_grid"], bool(sc["sdf_all_faces"]))
        p64, p32 = oracle_penetration(om64, X[i], *args), oracle_penetration(om32, X[i], *args)
        if abs(p32 - p64) > PARITY_REL * abs(p64) and p32 != p64:
            excluded.append(i)
            continue
        kp = (fr["gt_uv"][:, i], fr["conf"][:, i], fr["joint_weights"])
        r = O.closure_eval(om64, cfg, pri, cams_t, X[i], *kp)
        r32 = O.closure_eval(om32, cfg, pri32, cams32, X[i], *kp)
        # allowed error per segment: BAR_SDF_GRAD x its largest |entry| + FP32_NOISE x the float32 oracle's own deviation
        allow = {n: BAR_SDF_GRAD * np.abs(r["grad"][a:e]).max() + FP32_NOISE * np.abs(r32["grad"][a:e] - r["grad"][a:e]).max()
                 for n, (a, e) in SEGS.items()}
        ref[i] = dict(loss=r["loss"], grad=r["grad"], pen=p64, allow=allow)
    print("[C %s] oracle-compared edge frames %d, excluded %d %s" % (sdf, len(ref), len(excluded), excluded))
    assert len(ref) >= 0.9 * len(EDGE_FRAMES), excluded
    assert sum(r["pen"] > 0 for r in ref.values()) >= 3, "the compared frames must penetrate"
    # each edge frame alone
    alone = {}
    ctx = make_ctx(syn_model, syn_gmm, cams, 1, mode=3)
    ctx.set_loss(**loss_kw)
    for i in EDGE_FRAMES:
        ctx.set_keypoints(*batch_frames(fr, [i]), fr["joint_weights"])
        out = ctx.closure(torch.tensor(X[i:i + 1], device="cuda"))
        alone[i] = (out["loss"].cpu().numpy()[0], out["grad"].cpu().numpy()[0])
    ctx.close()
    worst = Worst("C " + sdf)
    for B in BATCHES:
        ctx = make_ctx(syn_model, syn_gmm, cams, B, mode=3)
        res = {}
        for name, order in (("id", np.arange(B)), ("rev", np.arange(B)[::-1].copy())):
            ctx.set_keypoints(*batch_frames(fr, order), fr["joint_weights"])
            ctx.set_loss(**loss_kw)
            ctx.profile(0xFFFFFFFF)
            out = ctx.closure(torch.tensor(np.ascontiguousarray(X[order]), device="cuda"))
            prof = ctx.profile_read()
            ctx.profile(0)
            assert prof.get("frame_step", (0, 0))[1] == 1 and "keypoint_loss" not in prof, prof
            inv = np.argsort(order)
            res[name] = (out["loss"].cpu().numpy()[inv], out["grad"].cpu().numpy()[inv])
        ctx.close()
        loss, grad = res["id"]
        assert np.isfinite(loss).all() and np.isfinite(grad).all(), B
        same = (loss == res["rev"][0]) & (grad == res["rev"][1]).all(1)
        assert same.all(), ("reversed batch", B, np.flatnonzero(~same)[:8])
        for i in (i for i in EDGE_FRAMES if i < B):
            assert loss[i] == alone[i][0] and np.array_equal(grad[i], alone[i][1]), ("alone", B, i)
            if i not in ref:
                continue
            worst.add("loss", abs(float(loss[i]) - ref[i]["loss"]) / abs(ref[i]["loss"]), BAR_SDF_LOSS, (B, i))
            for n, (a, e) in SEGS.items():
                err = np.abs(grad[i, a:e] - ref[i]["grad"][a:e]).max() / ref[i]["allow"][n]
                worst.add("grad %s / allowed" % n, err, 1.0, (B, i))
    worst.report()
