"""GPU: mvs_forward_vjp, the vector-Jacobian product of mvs_forward, and the differentiable SMPL module built on it.

The oracle is oracle.closure_oracle.smpl_forward (the reference's lbs.py restated) run in float64 with torch autograd: the
VJP of <gv, verts> + <gj, joints> with respect to betas, global_orient, body_pose, transl and scale.  It is fed exactly the
float32 constants and parameters the context sees.  Each gradient segment of each checked frame is compared relative to its
own largest float64 entry; the bar of a segment is BAR_MULT times the error the same oracle makes in float32 on that frame
and segment, and never tighter than BAR_FLOOR.  Every test prints its worst ratios (run with -s).

Batch sizes cross the forward's kernel choices (skin_small_kernel up to 8 frames, 64-frame tiles of the SIMT kernels and of
the part layout) and the wgmma N instances of vertex_bwd_tc_kernel (8, 16, 32, 64 frames per column tile).
"""
import ctypes

import numpy as np
import pytest
import torch

from mvsmplfitting_b200 import synthetic as S
from oracle import closure_oracle as O

pytestmark = pytest.mark.gpu

BATCHES = (1, 4, 8, 9, 64, 65, 256)
BMAX = max(BATCHES)
CHECK = (0, 1, 2, 3, 7, 8, 63, 64, 255)           # frames compared with float64 (those below B)
SEGS = dict(betas=(0, 10), global_orient=(10, 13), body_pose=(13, 82), transl=(82, 85), scale=(85, 86))
KINDS = ("verts", "joints", "both")
BAR_MULT = 16.0
BAR_FLOOR = 2e-6


def make_params(seed=910):
    """BMAX frames: the generator's ground-truth poses, non-unit scale; frame 0 with every rotation near 0 (Rodrigues'
    small-angle branch), frame 1 with every rotation near pi, frame 2 with a mix"""
    cams = S.make_cameras(2)
    fr = S.make_frames(S.make_model(0), cams, BMAX, seed=seed)
    X = S.pack_params(fr["gt"]).astype(np.float32)
    rng = np.random.RandomState(seed + 1)
    X[:, 85] = rng.uniform(0.85, 1.15, BMAX).astype(np.float32)
    X[:, :10] = rng.normal(0, 1, (BMAX, 10)).astype(np.float32)
    axes = rng.normal(0, 1, (BMAX, 24, 3))
    axes /= np.linalg.norm(axes, axis=2, keepdims=True)
    X[0, 10:82] = (axes[0] * rng.uniform(1e-7, 1e-5, (24, 1))).reshape(-1)
    X[1, 10:82] = (axes[1] * (np.pi - rng.uniform(1e-4, 1e-2, (24, 1)))).reshape(-1)
    X[2, 10:82] = (axes[2] * rng.choice([1e-6, 1.0, np.pi - 1e-3], (24, 1))).reshape(-1)
    return X


def cotangents(N, K, seed=911):
    rng = np.random.RandomState(seed)
    return rng.normal(0, 1, (BMAX, N, 3)).astype(np.float32), rng.normal(0, 1, (BMAX, K, 3)).astype(np.float32)


def make_ctx(model, B, model_type, mode=0):
    from mvsmplfitting_b200.context import FittingContext
    ctx = FittingContext(0)
    ctx.set_model(model, model_type=model_type)
    ctx.set_batch(B)
    ctx.set_exec_mode(mode)
    return ctx


def oracle_vjp(om, x, gv, gj):
    parts = [torch.tensor(np.asarray(x[a:e], dtype=np.float64), dtype=om.dtype).view(1, -1).requires_grad_(True)
             for a, e in SEGS.values()]
    v, j, _ = O.smpl_forward(om, *parts)
    s = 0.0
    if gv is not None:
        s = s + (v * torch.tensor(gv, dtype=om.dtype)).sum()
    if gj is not None:
        s = s + (j * torch.tensor(gj, dtype=om.dtype)).sum()
    g = torch.autograd.grad(s, parts)
    return np.concatenate([t.detach().double().numpy().reshape(-1) for t in g])


def seg_err(g, ref):
    return {k: np.abs(g[a:e].astype(np.float64) - ref[a:e]).max() / max(np.abs(ref[a:e]).max(), 1e-30)
            for k, (a, e) in SEGS.items()}


def kind_args(kind, gv, gj):
    return (gv if kind != "joints" else None), (gj if kind != "verts" else None)


class Worst:
    def __init__(self, title):
        self.title, self.w, self.fail = title, {}, []

    def add(self, key, ratio, where):
        if key not in self.w or ratio > self.w[key][0]:
            self.w[key] = (ratio, where)
        if not ratio <= 1.0:
            self.fail.append((key, ratio, where))

    def report(self):
        for k in sorted(self.w, key=str):
            print("[%s] %-28s worst err/bar %.3f at %s" % (self.title, k, *self.w[k]))
        assert not self.fail, self.fail[:8]


@pytest.mark.parametrize("model_type", ["smpllsp", "smpl"])
def test_vjp_matches_float64_in_both_exec_modes(model_type, syn_model):
    X = make_params()
    gv_all, gj_all = cotangents(syn_model["v_template"].shape[0], 17)
    om64 = O.OracleModel.from_numpy(syn_model, dtype=torch.float64, model_type=model_type)
    om32 = O.OracleModel.from_numpy(syn_model, dtype=torch.float32, model_type=model_type)
    ref, bar = {}, {}
    for i in CHECK:
        for kind in KINDS:
            gv, gj = kind_args(kind, gv_all[i], gj_all[i])
            r64 = oracle_vjp(om64, X[i], gv, gj)
            e32 = seg_err(oracle_vjp(om32, X[i], gv, gj), r64)
            ref[i, kind] = r64
            bar[i, kind] = {k: max(BAR_MULT * e, BAR_FLOOR) for k, e in e32.items()}
    worst = Worst("vjp " + model_type)
    for B in BATCHES:
        ctx = make_ctx(syn_model, B, model_type)
        x = torch.tensor(X[:B], device="cuda")
        gv_t, gj_t = torch.tensor(gv_all[:B], device="cuda"), torch.tensor(gj_all[:B], device="cuda")
        for kind in KINDS:
            out = {}
            for mode in (0, 1):
                ctx.set_exec_mode(mode)
                gv, gj = kind_args(kind, gv_t, gj_t)
                out[mode] = ctx.forward_vjp(x, djoints=gj, dverts=gv).cpu().numpy()
                assert np.isfinite(out[mode]).all(), (B, kind, mode)
            for i in (i for i in CHECK if i < B):
                for mode in (0, 1):
                    for k, e in seg_err(out[mode][i], ref[i, kind]).items():
                        worst.add("mode%d %s %s" % (mode, kind, k), e / bar[i, kind][k], (B, i))
                # cross-check: the tensor-core path against the SIMT chain, within the same bar
                for k, e in seg_err(out[0][i], out[1][i].astype(np.float64)).items():
                    worst.add("mode0-vs-1 %s %s" % (kind, k), e / bar[i, kind][k], (B, i))
        ctx.close()
    worst.report()


def test_vjp_is_deterministic(syn_model):
    B = 256
    X = make_params()
    gv, gj = cotangents(syn_model["v_template"].shape[0], 17)
    ctx = make_ctx(syn_model, B, "smpllsp")
    x = torch.tensor(X, device="cuda")
    gv, gj = torch.tensor(gv, device="cuda"), torch.tensor(gj, device="cuda")
    a = ctx.forward_vjp(x, gj, gv)
    b = ctx.forward_vjp(x, gj, gv)
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    ctx.close()


def fit_scene(syn_model, syn_gmm, B, sdf=False):
    from mvsmplfitting_b200.context import FittingContext
    cams = S.make_cameras(4)
    fr = S.make_frames(syn_model, cams, B, seed=77)
    ctx = FittingContext(0)
    ctx.set_model(syn_model, model_type="smpllsp")
    ctx.set_gmm_from_dict(syn_gmm)
    ctx.set_cameras(cams["R"], cams["t"], cams["f"], cams["c"])
    ctx.set_batch(B)
    ctx.set_keypoints(fr["gt_uv"], fr["conf"], fr["joint_weights"])
    w = dict(data_weight=500.0 / 1536, body_pose_weight=57.4, shape_weight=10.0, bending_prior_weight=3.17 * 57.4)
    if sdf:
        w.update(interpenetration=True, coll_loss_weight=1.0)
    ctx.set_loss(body_prior="gmm", **w)
    return ctx, torch.tensor(S.pack_params(fr["init"]), device="cuda"), w


def bits(t):
    return t.contiguous().view(torch.int32).cpu()


@pytest.mark.parametrize("sdf", [False, True])
def test_vjp_leaves_the_optimiser_state_alone(sdf, syn_model, syn_gmm):
    """mvs_lbfgs_step, mvs_forward_vjp, mvs_lbfgs_step gives the bits of two steps without the VJP in between"""
    B = 8
    res = []
    for with_vjp in (False, True):
        ctx, x, _ = fit_scene(syn_model, syn_gmm, B, sdf=sdf)
        cfg = ctx.make_lbfgs_config(max_iter=5)
        l0, g0, _ = ctx.lbfgs_step(x, cfg, reset=True)
        if with_vjp:
            probe = torch.randn(B, ctx.N, 3, device="cuda")
            ctx.forward_vjp(x.clone(), torch.randn(B, ctx.K, 3, device="cuda"), probe)
        l1, g1, _ = ctx.lbfgs_step(x, cfg)
        torch.cuda.synchronize()
        res.append([bits(t) for t in (x, l0, g0, l1, g1)])
        ctx.close()
    for a, b in zip(*res):
        assert torch.equal(a, b)


def test_fit_and_sdf_closure_after_a_vjp_are_unchanged(syn_model, syn_gmm):
    """mvs_fit after a VJP on the same context, and mvs_closure with the SDF term after a VJP, give the bits without it"""
    B = 8
    res = []
    for with_vjp in (False, True):
        ctx, x, w = fit_scene(syn_model, syn_gmm, B, sdf=True)
        probe = (torch.randn(B, ctx.K, 3, device="cuda"), torch.randn(B, ctx.N, 3, device="cuda"))
        if with_vjp:
            ctx.forward_vjp(x, *probe)
        c = ctx.closure(x, want_grad=True)
        if with_vjp:
            ctx.forward_vjp(x, *probe)
        stages = [ctx.make_loss_config(body_prior="gmm", **w), ctx.make_loss_config(body_prior="gmm", **dict(w, interpenetration=False))]
        xf = x.clone()
        final, _ = ctx.fit(xf, stages, ctx.make_lbfgs_config(max_outer=3, max_iter=5))
        torch.cuda.synchronize()
        res.append([bits(t) for t in (c["loss"], c["grad"], xf, final)])
        ctx.close()
    for a, b in zip(*res):
        assert torch.equal(a, b)


def make_module(syn_model, B, differentiable, model_type="smpllsp"):
    from mvsmplfitting_b200 import smplx
    from mvsmplfitting_b200.utils import utils
    ds = smplx.Struct(f=syn_model["f"], v_template=syn_model["v_template"], shapedirs=syn_model["shapedirs"],
                      posedirs=syn_model["posedirs"], J_regressor=syn_model["J_regressor"],
                      kintree_table=syn_model["kintree_table"], weights=syn_model["weights"])
    fmt = "lsp14" if model_type == "smpllsp" else "coco17"
    return smplx.create_scale("unused", model_type=model_type, data_struct=ds, differentiable=differentiable,
                              joint_mapper=utils.JointMapper(utils.smpl_to_annotation(model_type, pose_format=fmt)),
                              batch_size=B, dtype=torch.float32).to("cuda")


def test_differentiable_module_backpropagates_into_its_parameters_and_inputs(syn_model):
    from mvsmplfitting_b200.fitting import model_context
    B = 9
    X = make_params()[:B]
    p = S.unpack_params(X)
    plain, diff = make_module(syn_model, B, False), make_module(syn_model, B, True)
    for m in (plain, diff):
        m.reset_params(betas=p["betas"], global_orient=p["global_orient"], body_pose=p["body_pose"], transl=p["transl"],
                       scale=p["scale"])
    o_plain, o_diff = plain(), diff()
    assert not o_plain.vertices.requires_grad and not o_plain.joints.requires_grad
    assert o_diff.vertices.requires_grad and o_diff.joints.requires_grad
    assert torch.equal(bits(o_plain.vertices), bits(o_diff.vertices)) and torch.equal(bits(o_plain.joints), bits(o_diff.joints))
    gv = torch.randn_like(o_diff.vertices)
    gj = torch.randn_like(o_diff.joints)
    ((o_diff.vertices * gv).sum() + (o_diff.joints * gj).sum()).backward()
    ctx = model_context(diff)
    ref = ctx.forward_vjp(diff.graph_params().detach().contiguous(), gj, gv)
    for name, (a, e) in SEGS.items():
        g = getattr(diff, name).grad
        assert g is not None, name
        assert torch.equal(bits(g.reshape(B, e - a)), bits(ref[:, a:e])), name
    # a body_pose passed in (e.g. decoded from a VPoser code in torch) receives its gradient
    bp = torch.tensor(p["body_pose"], device="cuda", requires_grad=True)
    out = diff(body_pose=bp * 1.0)
    (out.joints * gj).sum().backward()
    ref = ctx.forward_vjp(diff.graph_params(body_pose=bp).detach().contiguous(), gj, None)
    assert torch.equal(bits(bp.grad), bits(ref[:, 13:82]))
    # second derivatives are not implemented
    out = diff()
    with pytest.raises(NotImplementedError):
        torch.autograd.grad((out.vertices * gv).sum(), [diff.betas], create_graph=True)


def test_refusals_leave_a_working_context(syn_model):
    B = 4
    ctx = make_ctx(syn_model, B, "smpllsp")
    x = torch.tensor(make_params()[:B], device="cuda")
    gv, gj = torch.randn(B, ctx.N, 3, device="cuda"), torch.randn(B, ctx.K, 3, device="cuda")
    good = ctx.forward_vjp(x, gj, gv)
    out = torch.empty(B, 86, device="cuda")
    p = lambda t: None if t is None else ctypes.c_void_p(t.data_ptr())
    f = ctx.lib.mvs_forward_vjp
    assert f(None, p(x), p(gj), p(gv), p(out), None) == -1
    assert f(ctx.h, None, p(gj), p(gv), p(out), None) == -1
    assert f(ctx.h, p(x), p(gj), p(gv), None, None) == -1
    assert f(ctx.h, p(x), None, None, p(out), None) == -1
    from mvsmplfitting_b200.context import FittingContext
    bare = FittingContext(0)
    assert bare.lib.mvs_forward_vjp(bare.h, p(x), p(gj), p(gv), p(out), None) == -1       # no model, no batch
    bare.set_model(syn_model)
    assert bare.lib.mvs_forward_vjp(bare.h, p(x), p(gj), p(gv), p(out), None) == -1       # no batch
    bare.close()
    assert torch.equal(bits(ctx.forward_vjp(x, gj, gv)), bits(good))
    for bad in (dict(djoints=gj[:, :5]), dict(dverts=gv[:, :100]), dict(dverts=gv.double()), dict()):
        with pytest.raises(ValueError):
            ctx.forward_vjp(x, **bad)
    with pytest.raises(ValueError):
        ctx.forward_vjp(x[:2], gj)
    ctx.close()
