"""GPU: seqio's image_folder / render_folder (the reference's save_images) through fit_sequence (batch = F and stream) and
fit_sequences (lock-step and stream): exactly the expected overlays are written, each is cv2's JPEG of FittingContext.render on
the saved pose, and the result pickles and meshes are byte-identical to a run without rendering."""
import os

import numpy as np
import pytest
import torch

from mvsmplfitting_b200 import seqio
from mvsmplfitting_b200 import synthetic as S

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")

W, H = 160, 120
OPT = dict(max_outer=3)


def make_ctx(model, gmm, cams, B):
    from mvsmplfitting_b200.context import FittingContext
    ctx = FittingContext(0)
    ctx.set_model(model)
    ctx.set_gmm_from_dict(gmm)
    ctx.set_cameras(cams["R"], cams["t"], cams["f"], cams["c"])
    ctx.set_batch(B)
    return ctx


def stages(ctx):
    sw = S.STAGE_WEIGHTS
    return [ctx.make_loss_config(body_prior="gmm", data_weight=500.0 / 1536, body_pose_weight=sw["body_pose_prior_weights"][i],
                                 shape_weight=sw["shape_weights"][i], bending_prior_weight=3.17 * sw["body_pose_prior_weights"][i])
            for i in range(3)]


def make_seqs(model, cams, lengths, seed, image_root):
    """sequences with a missing detection and a missing image, and random images of W x H under image_root"""
    rng = np.random.RandomState(seed)
    out = []
    for s_, T in enumerate(lengths):
        fr = S.make_frames(model, cams, T, seed=seed + s_, smooth_walk=True)
        V = cams["R"].shape[0]
        present = np.ones((V, T), bool)
        present[1, 0] = False
        conf = fr["conf"].copy()
        conf[~present] = 0.0
        q = dict(gt_uv=fr["gt_uv"], conf=conf, present=present, frames=["%05d" % t for t in range(T)], serial="s%02d" % s_,
                 cameras=["Camera%02d" % v for v in range(V)])
        for v, cam in enumerate(q["cameras"]):
            os.makedirs(os.path.join(image_root, q["serial"], cam), exist_ok=True)
            for t, name in enumerate(q["frames"]):
                if (v, t) == (2, T - 1):
                    continue                                  # no image: no overlay
                ext = ".png" if v == 0 else ".jpg"
                cv2.imwrite(os.path.join(image_root, q["serial"], cam, name + ext), rng.randint(0, 256, (H, W, 3)).astype(np.uint8))
        out.append(q)
    return out


def expected(seqs, image_root):
    want = set()
    for q in seqs:
        for v, cam in enumerate(q["cameras"]):
            for t, name in enumerate(q["frames"]):
                if q["present"][v, t] and any(os.path.exists(os.path.join(image_root, q["serial"], cam, name + e)) for e in (".jpg", ".png")):
                    want.add(os.path.join(q["serial"], name, cam + ".jpg"))
    return want


def written(root):
    return {os.path.relpath(os.path.join(d, f), root) for d, _, fs in os.walk(root) for f in fs}


def check_overlays(ctx, seqs, xs, image_root, render_root):
    """every overlay equals cv2.imencode of ctx.render on the saved pose (extremities zeroed) over the frame's images, drawn
    through the sequence's rig (q["rig"], when the sequences name rigs)"""
    assert written(render_root) == expected(seqs, image_root)
    f = 0
    for q, x in zip(seqs, xs):
        for t, name in enumerate(q["frames"]):
            saved = torch.zeros(ctx.B, 86, device="cuda")
            saved[0] = torch.as_tensor(x[t], device="cuda")
            for a, b in ((18, 24), (27, 33), (57, 69)):
                saved[:, 13 + a:13 + b] = 0.0
            fwd = ctx.forward_only(saved.contiguous(), want_verts=True)
            bg = np.zeros((1, ctx.V, H, W, 3), np.uint8)
            for v, cam in enumerate(q["cameras"]):
                for e in (".jpg", ".png"):
                    p = os.path.join(image_root, q["serial"], cam, name + e)
                    if os.path.exists(p):
                        bg[0, v] = cv2.imread(p, cv2.IMREAD_COLOR)
                        break
            img = ctx.render(fwd["verts"][:1].contiguous(), fwd["joints"][:1].contiguous(), background=torch.as_tensor(bg).cuda(),
                             rig=[q["rig"]] if "rig" in q else None)
            img = img["image"][0].cpu().numpy()
            for v, cam in enumerate(q["cameras"]):
                p = os.path.join(render_root, q["serial"], name, cam + ".jpg")
                if os.path.exists(p):
                    assert open(p, "rb").read() == cv2.imencode(".jpg", img[v])[1].tobytes(), p
            f += 1


def same_tree(a, b):
    fa, fb = written(a), written(b)
    assert fa == fb
    for p in fa:
        assert open(os.path.join(a, p), "rb").read() == open(os.path.join(b, p), "rb").read(), p


@pytest.mark.parametrize("B", [5, 2])
def test_fit_sequence(B, syn_model, syn_gmm, tmp_path):
    cams = S.make_cameras(3, radius=5.0)
    cams = dict(cams, f=cams["f"] * W / 2048, c=cams["c"] * W / 2048)
    seq = make_seqs(syn_model, cams, [5], 40, str(tmp_path / "img"))[0]
    faces = syn_model["f"]
    runs = {}
    for tag, kw in (("plain", {}), ("render", dict(image_folder=str(tmp_path / "img"), render_folder=str(tmp_path / "ovl")))):
        ctx = make_ctx(syn_model, syn_gmm, cams, B)
        x, loss, _ = seqio.fit_sequence(ctx, seq, stages(ctx), ctx.make_lbfgs_config(**OPT), pose_format="lsp14",
                                        result_folder=str(tmp_path / tag / "res"), mesh_folder=str(tmp_path / tag / "mesh"),
                                        faces=faces, **kw)
        runs[tag] = (ctx, x)
    same_tree(str(tmp_path / "plain"), str(tmp_path / "render"))
    check_overlays(runs["render"][0], [seq], [runs["render"][1]], str(tmp_path / "img"), str(tmp_path / "ovl"))
    for ctx, _ in runs.values():
        ctx.close()
    ctx = make_ctx(syn_model, syn_gmm, cams, B)
    with pytest.raises(ValueError):
        seqio.fit_sequence(ctx, seq, stages(ctx), ctx.make_lbfgs_config(**OPT), pose_format="lsp14", image_folder=str(tmp_path))
    ctx.close()


@pytest.mark.parametrize("B,rigs", [(2, False), (3, False), (2, True), (3, True)])
def test_fit_sequences(B, rigs, syn_model, syn_gmm, tmp_path):
    """B = 2 sequences: lock-step; B = 3: the sequence stream.  rigs: the two sequences were seen by rigs of 3 and 2 views
    (fit_sequences(rigs=)), so each overlay is drawn through its sequence's rig"""
    cams = S.make_cameras(3, radius=5.0)
    cams = dict(cams, f=cams["f"] * W / 2048, c=cams["c"] * W / 2048)
    if rigs:
        two = S.make_cameras(2, radius=6.0)
        two = dict(two, f=two["f"] * W / 2048, c=two["c"] * W / 2048)
        seqs = make_seqs(syn_model, cams, [3], 50, str(tmp_path / "img")) + make_seqs(syn_model, two, [2], 51, str(tmp_path / "img2"))
        seqs[1] = dict(seqs[1], serial="s01")
        os.rename(str(tmp_path / "img2" / "s00"), str(tmp_path / "img" / "s01"))
        for r, q in enumerate(seqs):
            q["rig"] = r
        table = [{k: cams[k] for k in ("R", "t", "f", "c")}, {k: two[k] for k in ("R", "t", "f", "c")}]
        extra = dict(rigs=table)
    else:
        seqs = make_seqs(syn_model, cams, [3, 2], 50, str(tmp_path / "img"))
        extra = {}
    runs = {}
    for tag, kw in (("plain", {}), ("render", dict(image_folder=str(tmp_path / "img"), render_folder=str(tmp_path / "ovl")))):
        kw.update(extra)
        ctx = make_ctx(syn_model, syn_gmm, cams, B)
        res, _ = seqio.fit_sequences(ctx, seqs, stages(ctx), ctx.make_lbfgs_config(**OPT), pose_format="lsp14",
                                     result_folder=str(tmp_path / tag / "res"), mesh_folder=str(tmp_path / tag / "mesh"),
                                     faces=syn_model["f"], **kw)
        runs[tag] = (ctx, [r[0] for r in res])
    same_tree(str(tmp_path / "plain"), str(tmp_path / "render"))
    check_overlays(runs["render"][0], seqs, runs["render"][1], str(tmp_path / "img"), str(tmp_path / "ovl"))
    for ctx, _ in runs.values():
        ctx.close()


def test_mixed_image_sizes_refused(syn_model, syn_gmm, tmp_path):
    cams = S.make_cameras(2, radius=5.0)
    cams = dict(cams, f=cams["f"] * W / 2048, c=cams["c"] * W / 2048)
    seq = make_seqs(syn_model, cams, [2], 60, str(tmp_path / "img"))[0]
    cv2.imwrite(str(tmp_path / "img" / seq["serial"] / "Camera01" / "00001.jpg"), np.zeros((H + 2, W, 3), np.uint8))
    ctx = make_ctx(syn_model, syn_gmm, cams, 2)
    with pytest.raises(ValueError, match="one image size"):
        seqio.fit_sequence(ctx, seq, stages(ctx), ctx.make_lbfgs_config(**OPT), pose_format="lsp14",
                           image_folder=str(tmp_path / "img"), render_folder=str(tmp_path / "ovl"))
    ctx.close()
