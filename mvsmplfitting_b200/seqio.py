"""Host-side data formats on either side of the fitting path (SURVEY §8f row N4): the reference's camera file,
per-view keypoint JSON files and per-frame result pickles / meshes, read and written for WHOLE SEQUENCES so that the
frames of a sequence go through `mvs_init_guess` + `mvs_fit` as one batch instead of the reference's per-frame loop
(code/main.py:32-89).

Reference interfaces mirrored (file:line of /root/reference/code):
  load_camera_para     utils/utils.py:352-394      camera file -> extrinsics [V,4,4], intrinsics [V,3,3]
                                                   (load_camera_distortion reads the distortion lines it skips)
  read_keypoints       utils/data_parser.py:42-90  OpenPose-style JSON -> [17,3] (u, v, confidence), body part only
                                                   (use_hands = use_face = False is the only configuration of the path)
  FittingData          utils/data_parser.py:257-433  folder layout <keypoints>/<serial>/<camera>/<frame>_keypoints.json,
                                                   joint weights (:340-358)
  save_results         utils/utils.py:729-761,856-890  result dict, pickle protocol 2 at <results>/<serial>/<frame>/000.pkl,
                                                   optional .obj mesh

Plain numpy / stdlib for the formats; the device work is behind FittingContext (torch only carries its buffers)."""
from __future__ import annotations

import json
import os
import pickle

import numpy as np
import torch

NUM_BODY_JOINTS = 17                     # data_parser.py:259


def load_camera_para(path: str):
    """utils.py:352-394: lines of 3 numbers build the intrinsics, lines of 4 numbers the [R | t] rows of the
    extrinsics (a [0, 0, 0, 1] row is appended), anything else (camera index lines, blanks) is skipped."""
    intr_rows, ext_rows = [], []
    with open(path) as f:
        for line in f:
            words = line.split()
            if len(words) == 3:
                intr_rows.append([float(w) for w in words])
            elif len(words) == 4:
                ext_rows.append([float(w) for w in words])
    intris = [intr_rows[i:i + 3] for i in range(0, len(intr_rows) - len(intr_rows) % 3, 3)]
    extris = [ext_rows[i:i + 3] + [[0.0, 0.0, 0.0, 1.0]] for i in range(0, len(ext_rows) - len(ext_rows) % 3, 3)]
    return np.array(extris), np.array(intris)


def load_camera_distortion(path: str) -> np.ndarray:
    """The lens distortion of every view of a camera file, [V,5] float64 (k1, k2, p1, p2, k3) in OpenCV's order: the line
    between a view's three intrinsic rows and its [R | t] rows, which load_camera_para skips.  A line of 2 numbers is
    (k1, k2); a line of 5 numbers is OpenCV's (k1, k2, p1, p2, k3); a view without such a line has zeros."""
    n_intr, dist = 0, {}
    with open(path) as f:
        for line in f:
            words = line.split()
            if len(words) == 3:
                n_intr += 1
            elif len(words) in (2, 5) and n_intr > 0 and n_intr % 3 == 0:
                d = [float(w) for w in words]
                dist[n_intr // 3 - 1] = d + [0.0] * (5 - len(d))
    out = np.zeros((n_intr // 3, 5))
    for v, d in dist.items():
        out[v] = d
    return out


def camera_arrays(extris, intris, views=None, dist=None) -> dict:
    """(extrinsics, intrinsics) -> the R [V,3,3], t [V,3], f [V,2], c [V,2] float32 arrays FittingContext.set_cameras
    takes (what create_camera receives per view at init.py:108-131).  dist [V,5] (load_camera_distortion) adds the key
    "dist" (float32), the views' lens distortion; without it the dict has no such key."""
    extris, intris = np.asarray(extris, np.float64), np.asarray(intris, np.float64)
    if views is not None:
        extris, intris = extris[list(views)], intris[list(views)]
    f32 = lambda a: np.ascontiguousarray(a, dtype=np.float32)
    out = dict(R=f32(extris[:, :3, :3]), t=f32(extris[:, :3, 3]), f=f32(np.stack([intris[:, 0, 0], intris[:, 1, 1]], 1)),
               c=f32(np.stack([intris[:, 0, 2], intris[:, 1, 2]], 1)))
    if dist is not None:
        dist = np.asarray(dist, np.float64).reshape(-1, 5)
        out["dist"] = f32(dist[list(views)] if views is not None else dist)
    return out


def camera_matrices(cams: dict):
    """The inverse of camera_arrays: a camera dict R [V,3,3], t [V,3], f [V,2], c [V,2] -> (extrinsics [V,4,4], intrinsics
    [V,3,3]) float64, the layout load_camera_para returns"""
    R, t = np.asarray(cams["R"], np.float64), np.asarray(cams["t"], np.float64)
    f, c = np.asarray(cams["f"], np.float64), np.asarray(cams["c"], np.float64)
    V = R.shape[0]
    extris = np.zeros((V, 4, 4))
    extris[:, :3, :3], extris[:, :3, 3], extris[:, 3, 3] = R, t, 1.0
    intris = np.zeros((V, 3, 3))
    intris[:, 0, 0], intris[:, 1, 1], intris[:, 0, 2], intris[:, 1, 2], intris[:, 2, 2] = f[:, 0], f[:, 1], c[:, 0], c[:, 1], 1.0
    return extris, intris


def write_camera_para(path: str, extris, intris, dist=None) -> None:
    """A camera file in the reference's layout (what load_camera_para reads): per view its index line, the three intrinsic
    rows, the distortion line, the three [R | t] rows and a blank line.  The distortion line is '0 0' when dist is None;
    with dist [V,5] (k1, k2, p1, p2, k3) it is 'k1 k2', or all five numbers when p1, p2 or k3 is non-zero
    (load_camera_distortion reads both).  Numbers are written with repr, so float32 inputs read back as the same float32
    values."""
    extris, intris = np.asarray(extris), np.asarray(intris)
    row = lambda r: " ".join(repr(float(x)) for x in r) + " \n"
    with open(path, "w") as fh:
        for v in range(extris.shape[0]):
            fh.write("%d\n" % v)
            for r in intris[v]:
                fh.write(row(r))
            if dist is None:
                fh.write("0 0\n")
            else:
                d = np.asarray(dist)[v]
                fh.write(row(d if np.any(d[2:] != 0) else d[:2]))
            for r in extris[v][:3]:
                fh.write(row(r))
            fh.write("\n")


def read_keypoints(path: str, person: int = 0):
    """data_parser.py:42-90 with use_hands = use_face = False: the first 17 (u, v, confidence) triplets of
    `pose_keypoints_2d` of one person as float32 [17,3]; None if the file lists fewer people."""
    with open(path) as f:
        data = json.load(f)
    people = data.get("people", [])
    if person >= len(people):
        return None
    kp = np.array(people[person]["pose_keypoints_2d"], dtype=np.float32).reshape(-1, 3)[:NUM_BODY_JOINTS]
    return kp


def read_joints(path: str, person: int = 0):
    """data_parser.py:93-146 with use_hands = use_face = False: the 3-D annotation of one person, `pose_keypoints_3d` as
    float32 rows (x, y, z, confidence) [N,4], N as the file gives it (unlike the 2-D reader, no truncation).  None where the
    reference's reader gives None for the file: some person without `pose_keypoints_3d`, or with a length that does not
    reshape to [-1,4] (its try / except drops the whole file); also None when the file lists fewer people.  A file without a
    'people' list raises KeyError, as the reference's reader does."""
    with open(path) as f:
        data = json.load(f)
    rows = []
    for p in data["people"]:
        try:
            rows.append(np.array(p["pose_keypoints_3d"], dtype=np.float32).reshape([-1, 4]))
        except Exception:
            return None
    return rows[person] if person < len(rows) else None


def joint_weights(pose_format: str = "coco17", use_hip: bool = True) -> np.ndarray:
    """FittingData.get_joint_weights, data_parser.py:340-358: hips (11, 12) are ignored unless lsp14 with use_hip"""
    w = np.ones(NUM_BODY_JOINTS, dtype=np.float32)
    if pose_format != "lsp14" or not use_hip:
        w[11] = 0.0
        w[12] = 0.0
    return w


def list_sequence(keyp_folder: str, serial: str):
    """(cameras, frames): sorted camera folders of one serial and the sorted union of frame names seen in any of them
    (FittingData.__init__ sorts the same way, data_parser.py:296-313, on the image folders)."""
    root = os.path.join(keyp_folder, serial)
    cameras = sorted(d for d in os.listdir(root) if os.path.isdir(os.path.join(root, d)))
    frames = set()
    for cam in cameras:
        for fn in os.listdir(os.path.join(root, cam)):
            if fn.endswith("_keypoints.json") and not fn.startswith("."):
                frames.add(fn[: -len("_keypoints.json")])
    return cameras, sorted(frames)


def load_sequence(keyp_folder: str, serial: str, cameras=None, frames=None, person: int = 0, use_3d: bool = False) -> dict:
    """All detections of a sequence as the arrays the device path takes: gt_uv [V,B,17,2], conf [V,B,17] float32.
    A (view, frame) without a keypoint file or without that person gets confidence 0 for every joint -- the reference
    drops such a view for that frame (main.py:45-56); with confidence 0 it weighs (w * conf)^2 = 0 in the data term
    and 1e-6 in the triangulation (recompute3D.py:49).
    use_3d: also the 3-D annotations (data_parser.py:398-402): a frame's annotation is read_joints of the first of
    `cameras`, in order, whose keypoint file exists and gives one.  Adds joints3d [B,17,3], conf3d [B,17] (column 3 as
    written) and has3d [B] bool; a frame without annotation has zero rows and has3d False.  An annotation of other than 17
    rows raises ValueError (the reference cannot broadcast it against the 17 keypoints, fitting.py:318-324)."""
    all_cams, all_frames = list_sequence(keyp_folder, serial)
    cameras = list(cameras) if cameras is not None else all_cams
    frames = list(frames) if frames is not None else all_frames
    V, B = len(cameras), len(frames)
    gt_uv = np.zeros((V, B, NUM_BODY_JOINTS, 2), dtype=np.float32)
    conf = np.zeros((V, B, NUM_BODY_JOINTS), dtype=np.float32)
    present = np.zeros((V, B), dtype=bool)
    for v, cam in enumerate(cameras):
        for b, fr in enumerate(frames):
            fn = os.path.join(keyp_folder, serial, cam, fr + "_keypoints.json")
            if not os.path.exists(fn):
                continue
            kp = read_keypoints(fn, person)
            if kp is None or kp.shape[0] < NUM_BODY_JOINTS:
                continue
            gt_uv[v, b], conf[v, b], present[v, b] = kp[:, :2], kp[:, 2], True
    out = dict(gt_uv=gt_uv, conf=conf, present=present, cameras=cameras, frames=frames, serial=serial)
    if use_3d:
        joints3d = np.zeros((B, NUM_BODY_JOINTS, 3), dtype=np.float32)
        conf3d = np.zeros((B, NUM_BODY_JOINTS), dtype=np.float32)
        has3d = np.zeros(B, dtype=bool)
        for b, fr in enumerate(frames):
            for cam in cameras:
                fn = os.path.join(keyp_folder, serial, cam, fr + "_keypoints.json")
                j = read_joints(fn, person) if os.path.exists(fn) else None
                if j is None:
                    continue
                if j.shape[0] != NUM_BODY_JOINTS:
                    raise ValueError("%s: pose_keypoints_3d has %d rows, want %d" % (fn, j.shape[0], NUM_BODY_JOINTS))
                joints3d[b], conf3d[b], has3d[b] = j[:, :3], j[:, 3], True
                break
        out.update(joints3d=joints3d, conf3d=conf3d, has3d=has3d)
    return out


PARAM_SLICES = (("betas", 0, 10), ("global_orient", 10, 13), ("body_pose", 13, 82), ("transl", 82, 85), ("scale", 85, 86))


def result_from_params(x, loss: float, pose_embedding=None, body_pose=None) -> dict:
    """One frame's 86-vector -> the dict non_linear_solver returns (non_linear_solver.py:283-287): the model's named
    parameters with their reference shapes ([1,10], [1,3], [1,69], [1,3], [1]), 'loss', 'pose_embedding'.  body_pose: the
    decoded pose when the pose slot of x holds a VPoser latent code."""
    x = np.asarray(x, dtype=np.float32).reshape(-1)
    out = {}
    for name, a, b in PARAM_SLICES:
        out[name] = x[a:b].copy() if name == "scale" else x[a:b].reshape(1, -1).copy()
    if body_pose is not None:
        out["body_pose"] = np.asarray(body_pose, np.float32).reshape(1, 69).copy()
    out["loss"] = float(loss)
    out["pose_embedding"] = None if pose_embedding is None else np.asarray(pose_embedding, np.float32).reshape(1, -1)
    return out


def finalize_result(result: dict) -> dict:
    """save_results' post-processing (utils.py:741-768): ankles (body_pose[18:24] = SMPL joints 7, 8), feet (27:33 = joints
    10, 11) and wrists + hands (57: = joints 20-23) are zeroed, 'pose' = [global_orient | body_pose].  With VPoser the
    'body_pose' entry must already hold the DECODED pose (result_from_params(..., body_pose=...)), as :741-743 decodes the
    latent code before zeroing; 'pose_embedding' keeps the code."""
    bp = result["body_pose"]
    bp[:, 18:24] = 0.0
    bp[:, 27:33] = 0.0
    bp[:, 57:] = 0.0
    result["pose"] = np.hstack((result["global_orient"], bp))
    return result


def write_obj(path: str, verts, faces) -> None:
    """Wavefront .obj as trimesh's exporter writes a bare mesh (utils.py:884-890): `v x y z` lines, 1-based `f a b c`"""
    verts, faces = np.asarray(verts, np.float64).reshape(-1, 3), np.asarray(faces, np.int64).reshape(-1, 3)
    with open(path, "w") as f:
        for v in verts:
            f.write("v %.8f %.8f %.8f\n" % (v[0], v[1], v[2]))
        for t in faces + 1:
            f.write("f %d %d %d\n" % (t[0], t[1], t[2]))


def save_results(result_folder: str, serial: str, fn: str, result: dict, person_id: int = 0, verts=None, faces=None,
                 mesh_folder: str | None = None) -> str:
    """utils.py:856-863 (+ :884-890 when a mesh is given): <result_folder>/<serial>/<fn>/000.pkl, pickle protocol 2"""
    d = os.path.join(result_folder, serial, fn)
    os.makedirs(d, exist_ok=True)
    out = os.path.join(d, "%03d.pkl" % person_id)
    with open(out, "wb") as f:
        pickle.dump(finalize_result(result), f, protocol=2)
    if verts is not None and faces is not None and mesh_folder is not None:
        md = os.path.join(mesh_folder, serial, fn)
        os.makedirs(md, exist_ok=True)
        write_obj(os.path.join(md, "%03d.obj" % person_id), verts, faces)
    return out


def _uses_latent_pose(stage_cfgs) -> bool:
    """True when the stages optimise VPoser's latent code on the device (use_vposer = 2); mixing encodings is refused"""
    kinds = {int(c.use_vposer) for c in stage_cfgs}
    if 1 in kinds:
        raise NotImplementedError("use_vposer = 1 (pose decoded by the caller) has no whole-sequence path: upload the decoder "
                                  "(FittingContext.set_vposer) and use use_vposer = 2")
    if kinds == {0, 2}:
        raise ValueError("stage configurations mix axis-angle and latent-code poses")
    return kinds == {2}


def _check_missing_views(seq: dict, stage_cfgs, views: int | None = None) -> None:
    """a (view, frame) without detections carries confidence 0; that only removes it from the data term when the loss uses the
    confidences (the reference drops such a view from the camera list instead, main.py:45-56).  views: the number of views
    of the sequence's rig (default: all rows), the only ones its frames have"""
    present = seq["present"] if views is None else seq["present"][:views]
    if not present.all() and not all(int(c.use_joints_conf) for c in stage_cfgs):
        raise ValueError("sequence has (view, frame) pairs without detections: every stage needs use_joints_conf = 1")


def _targets_3d(seqs, stage_cfgs, use_hip: bool):
    """use_3d (non_linear_solver.py:68-99) for sequences loaded with load_sequence(use_3d=True): per frame 3-D targets [F,17,3],
    confidences [F,17] and has3d [F], the sequences' frames back to back.  A frame without annotation has no 3-D term (:68-69):
    zero rows, which weigh nothing.  Hips 11 and 12 have confidence 0 unless use_hip (:92-94).  The confidences exist only
    with use_joints_conf (:90-91), so every stage needs it."""
    if not all(int(c.use_joints_conf) for c in stage_cfgs):
        raise ValueError("use_3d needs use_joints_conf = 1 in every stage (the 3-D confidences are read with the 2-D ones)")
    for q in seqs:
        if "has3d" not in q:
            raise ValueError("use_3d: sequence %s was loaded without its 3-D annotations (load_sequence(use_3d=True))"
                             % q.get("serial"))
    has = np.concatenate([q["has3d"] for q in seqs])
    j3 = np.concatenate([q["joints3d"] for q in seqs]).astype(np.float32)
    c3 = np.concatenate([q["conf3d"] for q in seqs]).astype(np.float32)
    j3[~has], c3[~has] = 0.0, 0.0
    if not use_hip:
        c3[:, 11] = c3[:, 12] = 0.0
    return j3, c3, has


def _init_guess_3d(ctx, guess: dict, j3, c3, has):
    """init_guess of one batch whose keypoints and loss configuration are set, under use_3d (init_guess.py:85-86): a frame
    with annotation aligns to its 3-D targets, one without triangulates (or takes the depth guess).  A batch that mixes the
    two runs the guess once with the targets and once without and takes each frame's row from its pass; the guess is per
    frame, so each pass gives a frame the bits it gets alone.  Leaves the 3-D term set as the last pass left it."""
    x = None
    if has.any():
        ctx.set_joints3d(j3, c3)
        x, _ = ctx.init_guess(**guess)
    if not has.all():
        ctx.set_joints3d(None)
        x0, _ = ctx.init_guess(**guess)
        x = x0 if x is None else torch.where(torch.as_tensor(has, device=x.device)[:, None], x, x0).contiguous()
    return x


def _pad_views(seq: dict, V: int) -> dict:
    """seq with its per-view arrays (gt_uv, conf, present) padded to V view rows (zeros; rows beyond the sequence's own views
    are never read)"""
    n = seq["gt_uv"].shape[0]
    if n == V:
        return seq
    pad = lambda a: np.concatenate([a, np.zeros((V - n,) + a.shape[1:], a.dtype)])
    return dict(seq, gt_uv=pad(seq["gt_uv"]), conf=pad(seq["conf"]), present=pad(seq["present"]))


def _export(ctx, seq, params, loss, latent, result_folder, mesh_folder, faces, frames=None, rows=None, plan=None, rig=None):
    """per-frame result pickles (+ meshes) of `rows` of the batch (default: all), named by `frames`; with plan (_render_plan)
    also the frames' overlays, rig: the sequence's camera rig (None: the context's only one)"""
    x = params.cpu().numpy()
    B = x.shape[0]
    rows = list(range(B)) if rows is None else list(rows)
    frames = seq["frames"] if frames is None else frames
    decoded = ctx.vposer_decode(params).cpu().numpy() if latent else None      # utils.py:741-743
    verts = None
    if mesh_folder is not None or plan is not None:   # the mesh is rebuilt from the SAVED pose (extremities zeroed), utils.py:865-871
        saved = params.clone()
        if latent:
            saved[:, 13:82] = torch.as_tensor(decoded, device=saved.device)
        for a, b in ((18, 24), (27, 33), (57, 69)):
            saved[:, 13 + a:13 + b] = 0.0
        fwd = ctx.forward_only(saved, want_verts=True)
        if plan is not None:
            _render_rows(ctx, plan, fwd["verts"], fwd["joints"], rows, frames, rig)
        verts = fwd["verts"].cpu().numpy() if mesh_folder is not None else None
    if result_folder is None:
        return
    for b, fr in zip(rows, frames):
        res = result_from_params(x[b], loss[b], pose_embedding=x[b, 13:45] if latent else None,
                                 body_pose=decoded[b] if latent else None)
        save_results(result_folder, seq["serial"], fr, res, verts=None if verts is None else verts[b], faces=faces,
                     mesh_folder=mesh_folder)


RENDER_CHUNK_BYTES = 1 << 30             # image buffers (background + overlay) of one render call


def _render_plan(seq: dict, image_folder, render_folder):
    """What the save_images option (utils.py:866-882) draws for a sequence: every (view, frame) with detections (present) and an
    image at <image_folder>/<serial>/<camera>/<frame>.jpg or .png (data_parser.py:296-323), whose overlay goes to
    <render_folder>/<serial>/<frame>/<camera>.jpg.  None when neither folder is given; ValueError when only one is.  Checked
    before any fitting: that cv2 imports and that the sequence's first image reads (its size is the sequence's image size)."""
    if image_folder is None and render_folder is None:
        return None
    if image_folder is None or render_folder is None:
        raise ValueError("image_folder and render_folder go together (got %r, %r)" % (image_folder, render_folder))
    import cv2                                            # the reference reads and writes its images with cv2
    images = {}
    for v, cam in enumerate(seq["cameras"]):
        for b, fr in enumerate(seq["frames"]):
            if not seq["present"][v, b]:
                continue
            for ext in (".jpg", ".png"):
                path = os.path.join(image_folder, seq["serial"], cam, fr + ext)
                if os.path.exists(path):
                    images[v, fr] = path
                    break
    plan = dict(serial=seq["serial"], cameras=list(seq["cameras"]), images=images, render_folder=render_folder, size=None)
    if images:
        _read_image(cv2, plan, next(iter(images.values())))
    return plan


def _read_image(cv2, plan: dict, path: str):
    """one image of a sequence (BGR uint8 [H,W,3]); ValueError when it does not read or its size is not the sequence's"""
    im = cv2.imread(path, cv2.IMREAD_COLOR)
    if im is None:
        raise ValueError("cannot read image %s" % path)
    if plan["size"] is None:
        plan["size"] = im.shape[:2]
    if im.shape[:2] != plan["size"]:
        raise ValueError("sequence %s: image %s is %dx%d, other views are %dx%d (one image size per sequence)"
                         % (plan["serial"], path, im.shape[1], im.shape[0], plan["size"][1], plan["size"][0]))
    return im


def _render_rows(ctx, plan: dict, verts, joints, rows, frames, rig=None):
    """Overlays of the batch rows `rows` (named `frames`) of verts [B,N,3] / joints [B,K,3]: FittingContext.render over each
    frame's images (markers on the keypoints), written as JPEG with cv2.  Frames go in chunks whose image buffers (the
    backgrounds and the overlays, on the host and on the device) stay under RENDER_CHUNK_BYTES each; a chunk's images are read
    when it is rendered."""
    import cv2
    todo = [(b, fr, [v for v in range(len(plan["cameras"])) if (v, fr) in plan["images"]]) for b, fr in zip(rows, frames)]
    todo = [t for t in todo if t[2]]
    if not todo:
        return
    H, W = plan["size"]
    chunk = max(1, RENDER_CHUNK_BYTES // (2 * ctx.V * H * W * 3))
    for c0 in range(0, len(todo), chunk):
        part = todo[c0:c0 + chunk]
        bg = np.zeros((len(part), ctx.V, H, W, 3), np.uint8)
        for i, (b, fr, views) in enumerate(part):
            for v in views:
                bg[i, v] = _read_image(cv2, plan, plan["images"][v, fr])
        idx = torch.as_tensor([b for b, _, _ in part], device=verts.device)
        out = ctx.render(verts[idx].contiguous(), keypoints=joints[idx].contiguous(),
                         rig=None if rig is None else np.full(len(part), rig, np.int32),
                         background=torch.as_tensor(bg, device=verts.device))["image"].cpu().numpy()
        del bg
        for i, (b, fr, views) in enumerate(part):
            d = os.path.join(plan["render_folder"], plan["serial"], fr)
            os.makedirs(d, exist_ok=True)
            for v in views:
                cv2.imwrite(os.path.join(d, plan["cameras"][v] + ".jpg"), out[i, v])


def fit_sequence(ctx, seq: dict, stage_cfgs, opt_cfg=None, estimate_scale: bool = False, fixed_scale: float = 1.0,
                 use_hip: bool = True, pose_format: str = "coco17", result_folder: str | None = None,
                 mesh_folder: str | None = None, faces=None, umeyama_as_written: bool = False, use_3d: bool = False,
                 shared_shape: int = 0, refine_cameras: int = 0, image_folder: str | None = None, render_folder: str | None = None):
    """The frame loop of main.py:32-89 for one sequence as ONE batch (every frame from its own initial guess, is_seq = False):
    upload the detections, initial guess on the device (init_guess + fix_params), all stages (`mvs_fit`), results per
    frame.  `ctx` is a FittingContext whose model, priors (GMM / VPoser decoder), cameras and batch (= number of frames) are
    set.  With use_vposer = 2 stage configurations (the reference's default, cfg_files/fit_smpl.yaml) the latent code
    starts at 0 (init_guess.py:96-98), and results carry the decoded pose plus 'pose_embedding' (utils.py:741-759).
    A context batch smaller than the sequence works as a pool of slots: the initial guesses are computed ctx.B frames at a
    time, then all frames go through ONE `mvs_fit_stream` call, which refills a slot as soon as its frame is done (the same
    results bit for bit).
    use_3d (the sequence loaded with load_sequence(use_3d=True)): the 3-D joint term for every frame with an annotation,
    whose initial guess also aligns to it; frames without one fit as without the term (_targets_3d, _init_guess_3d).  The
    context has the 3-D term off afterwards.
    shared_shape (sweeps, 0: off): the sequence is one subject -- after the fit, one fit_shared_shape call gives all of its
    frames one betas (and scale) under the last stage, see share_shape; results are written after it.
    refine_cameras (sweeps, 0: off): after the fit, one FittingContext.refine_cameras call over all frames refines the context's
    camera extrinsics from them (before shared_shape when both are given), see refine_rigs; the refined rigs go into stats and,
    with result_folder, into cameras_rig<r>.txt there.
    image_folder with render_folder (the reference's save_images): every (view, frame) with detections and an image
    <image_folder>/<serial>/<camera>/<frame>.jpg|.png gets the fitted mesh (the saved pose, as the .obj) and keypoint markers
    drawn over it by FittingContext.render, written to <render_folder>/<serial>/<frame>/<camera>.jpg (cv2).
    Returns (params [F,86] numpy -- pose slot = latent code under VPoser --, final_loss [F], stats)."""
    _check_sweeps("shared_shape", shared_shape, None, "the shared shape's pose step")
    _check_sweeps("refine_cameras", refine_cameras, None, "the camera refinement's body step")
    plan = _render_plan(seq, image_folder, render_folder)
    F = len(seq["frames"])
    assert ctx.B <= F, "context batch %d > frames %d" % (ctx.B, F)
    latent = _uses_latent_pose(stage_cfgs)
    _check_missing_views(seq, stage_cfgs)
    t3 = _targets_3d([seq], stage_cfgs, use_hip) if use_3d else None
    jw = joint_weights(pose_format, use_hip)
    guess = dict(estimate_scale=estimate_scale, fixed_scale=fixed_scale, use_torso=True, hip_seed=1.0, want_joints3d=False,
                 umeyama_as_written=umeyama_as_written)
    if ctx.B == F:
        ctx.set_keypoints(seq["gt_uv"], seq["conf"], jw)
        ctx.set_loss(config=stage_cfgs[0])           # mvs_init_guess zeroes the pose slot when it holds a latent code
        if t3 is None:
            params, _ = ctx.init_guess(**guess)
        else:
            params = _init_guess_3d(ctx, guess, *t3)
            ctx.set_joints3d(t3[0], t3[1])
        final, stats = ctx.fit(params, stage_cfgs, opt_cfg)
        if t3 is not None:
            ctx.set_joints3d(None)
        if refine_cameras:
            final = refine_rigs(ctx, params, seq["gt_uv"], seq["conf"], jw, stage_cfgs, opt_cfg, refine_cameras, t3, stats=stats,
                                result_folder=result_folder)
        if shared_shape:
            final = share_shape(ctx, params, seq["gt_uv"], seq["conf"], jw, [F], stage_cfgs, opt_cfg, shared_shape, t3, stats=stats)
        loss = final.cpu().numpy()
        if result_folder is not None or plan is not None:
            _export(ctx, seq, params, loss, latent, result_folder, mesh_folder, faces, plan=plan)
        return params.cpu().numpy(), loss, stats
    params = _cold_guesses(ctx, seq["gt_uv"], seq["conf"], jw, stage_cfgs, guess, t3)
    if t3 is None:
        final, stats = ctx.fit_stream(params, seq["gt_uv"], seq["conf"], jw, stage_cfgs, opt_cfg)
    else:
        final, stats = ctx.fit_stream(params, seq["gt_uv"], seq["conf"], jw, stage_cfgs, opt_cfg, joints3d=t3[0], conf3d=t3[1])
        ctx.set_joints3d(None)
    if refine_cameras:
        final = refine_rigs(ctx, params, seq["gt_uv"], seq["conf"], jw, stage_cfgs, opt_cfg, refine_cameras, t3, stats=stats,
                            result_folder=result_folder)
    if shared_shape:
        final = share_shape(ctx, params, seq["gt_uv"], seq["conf"], jw, [F], stage_cfgs, opt_cfg, shared_shape, t3, stats=stats)
    loss = final.cpu().numpy()
    if result_folder is not None or plan is not None:
        _export_rows(ctx, seq, params, loss, latent, result_folder, mesh_folder, faces, plan)
    return params.cpu().numpy(), loss, stats


def _cold_guesses(ctx, gt_uv, conf, jw, stage_cfgs, guess: dict, t3=None, rig=None, rig_views=None) -> torch.Tensor:
    """initial guesses (init_guess + fix_params) of F frames of any number, ctx.B frames at a time: params [F,86] on the
    device.  The last chunk is padded with zero-confidence rows, which are dropped.  t3: _targets_3d of the F frames (use_3d),
    each chunk's guesses then come from _init_guess_3d (padding rows count as frames without annotation only when the chunk
    needs that pass anyway).  rig [F] (the rig of each frame, views rig_views[r]): every chunk names its slots' rigs, and a
    frame's rows beyond its rig's views are not taken (padding rows take the chunk's first rig)."""
    F, B = gt_uv.shape[1], ctx.B
    params = torch.empty(F, 86, dtype=torch.float32, device=ctx.device)
    for c0 in range(0, F, B):
        n = min(B, F - c0)
        gt = np.zeros((gt_uv.shape[0], B) + gt_uv.shape[2:], np.float32)
        cf = np.zeros((conf.shape[0], B) + conf.shape[2:], np.float32)
        if rig is None:
            gt[:, :n], cf[:, :n] = gt_uv[:, c0:c0 + n], conf[:, c0:c0 + n]
        else:
            for j in range(n):
                nv = rig_views[rig[c0 + j]]
                gt[:nv, j], cf[:nv, j] = gt_uv[:nv, c0 + j], conf[:nv, c0 + j]
            ctx.set_frame_rigs(np.concatenate([rig[c0:c0 + n], np.full(B - n, rig[c0], np.int32)]))
        ctx.set_keypoints(gt, cf, jw)
        ctx.set_loss(config=stage_cfgs[0])           # mvs_init_guess zeroes the pose slot when it holds a latent code
        if t3 is None:
            x, _ = ctx.init_guess(**guess)
        else:
            j3 = np.zeros((B,) + t3[0].shape[1:], np.float32)
            c3 = np.zeros((B,) + t3[1].shape[1:], np.float32)
            has = np.full(B, bool(t3[2][c0:c0 + n].all()))
            j3[:n], c3[:n], has[:n] = t3[0][c0:c0 + n], t3[1][c0:c0 + n], t3[2][c0:c0 + n]
            x = _init_guess_3d(ctx, guess, j3, c3, has)
        params[c0:c0 + n] = x[:n]
    return params


def _export_rows(ctx, seq, params, loss, latent, result_folder, mesh_folder, faces, plan=None, rig=None):
    """_export of one sequence's F rows (params [F,86] on the device, loss [F]) in chunks of ctx.B rows, as the export takes
    whole batches; the last chunk is padded"""
    F, B = params.shape[0], ctx.B
    for c0 in range(0, F, B):
        n = min(B, F - c0)
        chunk = torch.zeros(B, 86, dtype=torch.float32, device=ctx.device)
        chunk[:n] = params[c0:c0 + n]
        lc = np.zeros(B, np.float32)
        lc[:n] = loss[c0:c0 + n]
        _export(ctx, seq, chunk, lc, latent, result_folder, mesh_folder, faces, frames=seq["frames"][c0:c0 + n], rows=range(n),
                plan=plan, rig=rig)


def _check_sweeps(option, sweeps, temporal_weight, step) -> None:
    """option: shared_shape or refine_cameras, a number of sweeps; step: the part of it that fits frames independently"""
    if isinstance(sweeps, bool) or int(sweeps) != sweeps or sweeps < 0:
        raise ValueError("%s: want a number of sweeps >= 0 (0: off), got %r" % (option, sweeps))
    if sweeps and temporal_weight is not None:
        raise ValueError("%s and temporal_weight do not combine: %s fits frames independently, so the causal temporal term "
                         "cannot be honoured" % (option, step))


def refine_rigs(ctx, params, gt_uv, conf, jw, stage_cfgs, opt_cfg, sweeps, t3=None, rig=None, stats=None, result_folder=None):
    """The camera refinement of fit_sequences / fit_sequence: ONE refine_cameras call over the fitted rows params [F,86]
    (device, updated in place) of all frames, under the last stage configuration; t3 (_targets_3d of the frames) adds the
    3-D term, rig [F] each frame's rig.  Returns the frames' final losses [F]; stats (a dict) gets 'refine_cameras': the
    refined rigs (camera dicts, as set_camera_rigs takes them) and the camera and body steps' counts.  With result_folder,
    rig r's refined calibration, with its lens distortion, is written to <result_folder>/cameras_rig<r>.txt (write_camera_para)."""
    kw = {} if rig is None else dict(rig=rig)
    if t3 is not None:
        kw.update(joints3d=t3[0], conf3d=t3[1])
    final, rigs, ca, po = ctx.refine_cameras(params, gt_uv, conf, jw, stage_cfgs[-1], opt_cfg, sweeps=int(sweeps), **kw)
    if stats is not None:
        stats["refine_cameras"] = dict(rigs=rigs, camera=ca, pose=po)
    if result_folder is not None:
        os.makedirs(result_folder, exist_ok=True)
        for r, cams in enumerate(rigs):
            write_camera_para(os.path.join(result_folder, "cameras_rig%d.txt" % r), *camera_matrices(cams), dist=cams.get("dist"))
    return final


def share_shape(ctx, params, gt_uv, conf, jw, lengths, stage_cfgs, opt_cfg, sweeps, t3=None, rig=None, stats=None):
    """The shared shape of fit_sequences / fit_sequence: ONE fit_shared_shape call over the fitted rows params [F,86] (device,
    updated in place) of all sequences (lengths), under the last stage configuration; t3 (_targets_3d of the frames) adds the
    3-D term, rig [F] each frame's rig.  Returns the frames' final losses [F]; stats (a dict) gets 'shared_shape': the shape
    and pose steps' counts."""
    kw = {} if rig is None else dict(rig=rig)
    if t3 is not None:
        kw.update(joints3d=t3[0], conf3d=t3[1])
    final, _, sh, po = ctx.fit_shared_shape(params, gt_uv, conf, jw, lengths, stage_cfgs[-1], opt_cfg, sweeps=int(sweeps), **kw)
    if stats is not None:
        stats["shared_shape"] = dict(shape=sh, pose=po)
    return final


def temporal_weight_vector(temporal_weight):
    """fit_sequences' temporal_weight as the 86 per-parameter weights the device takes: None stays None, a scalar lam is
    lam x sequence.smooth_mask() (global orientation, the pose slot and translation), an array is taken as the 86-vector"""
    if temporal_weight is None:
        return None
    if np.ndim(temporal_weight) == 0:
        from .sequence import smooth_mask
        return np.float32(temporal_weight) * smooth_mask().numpy().astype(np.float32)
    w = np.ascontiguousarray(temporal_weight, dtype=np.float32).reshape(-1)
    if w.shape[0] != 86:
        raise ValueError("temporal_weight: want a scalar or 86 entries, got %d" % w.shape[0])
    return w


def fit_sequences(ctx, seqs, stage_cfgs, opt_cfg=None, estimate_scale: bool = False, fixed_scale: float = 1.0,
                  use_hip: bool = True, pose_format: str = "coco17", result_folder: str | None = None,
                  mesh_folder: str | None = None, faces=None, umeyama_as_written: bool = False, reinit_loss: float = 5000.0,
                  use_3d: bool = False, rigs=None, rig_data_weight_scale=None, temporal_weight=None, shared_shape: int = 0,
                  refine_cameras: int = 0, image_folder: str | None = None, render_folder: str | None = None):
    """main.py:32-89 with is_seq = True for S sequences in lock-step: the batch of step t is frame t of every sequence
    (context batch = S).  A sequence's first frame gets the initial guess and every stage; a later frame
    starts from the previous frame's result as load_init + fix_params leave it (init_guess.py:137-166,190-212: betas,
    global_orient, transl, scale kept; body pose back to the hip seed, or the previous latent code under VPoser), skips
    stages 0 and 1 and damps stage 2's pose prior (non_linear_solver.py:157-162, `mvs_fit_seq`) -- unless the previous loss
    was above 5000, which re-runs the initial guess for that sequence (:141-144).  Sequences may differ in length.
    A context batch other than S works as a pool of slots: the initial guesses of all frames are computed ctx.B frames at a
    time, then all sequences go through ONE `mvs_fit_seq_stream` call, in which a slot takes the next frame of its sequence
    as soon as a frame is done (the same results bit for bit; stats then also carry the dense-round counts).
    use_3d (every sequence loaded with load_sequence(use_3d=True)): per frame, as non_linear_solver.py:68-99 decides it --
    a frame with an annotation has the 3-D joint term in every stage it runs, warm or cold, and its cold start point aligns
    to the annotation; a frame without one fits as without the term (_targets_3d, _init_guess_3d).  The context has the
    3-D term off afterwards.
    Without rigs every sequence was seen by the context's cameras.  rigs (a list of camera dicts, seqio.camera_arrays) fits
    sequences of several camera setups in the same call: sequence q was seen by rigs[q["rig"]] and has that rig's number of
    view rows; rig_data_weight_scale [n_rigs] (None: all 1) scales every stage's data_weight per rig (the reference's
    500 / H for rigs of different image heights).  The rigs are set on the context (set_camera_rigs), detections are padded
    to the largest view count, and every frame gets what a context with only its rig's cameras gives it.
    temporal_weight (None: off; a scalar lam, or 86 weights w, see temporal_weight_vector) pulls every warm frame towards its
    predecessor's fitted row: its stages add sum_i w_i (x_i - x^_{t-1,i})^2 (mvs_fit_seq_temporal in lock-step, after step
    t-1 with that step's fitted rows; mvs_fit_seq_stream_temporal otherwise, with the same bits).  Cold frames are fitted as
    without it.
    shared_shape (a number of sweeps, 0: off) gives every sequence one body shape: after the fit, ONE fit_shared_shape call
    over all frames under the last stage configuration (the same call in lock-step and stream mode; see share_shape), and the
    results and meshes are written after it.  It does not combine with temporal_weight (ValueError).
    refine_cameras (a number of sweeps, 0: off) refines every rig's camera extrinsics from the fitted bodies: after the fit, ONE
    refine_cameras call over all frames with each frame's rig (see refine_rigs), before shared_shape when both are given; the
    refined rigs go into stats['refine_cameras'] and, with result_folder, into cameras_rig<r>.txt there.  The context keeps
    the refined cameras.  It does not combine with temporal_weight (ValueError).
    image_folder with render_folder: every sequence's overlays, as fit_sequence writes them (each in its rig's cameras).
    Returns a list (per sequence) of (params [T_s,86], loss [T_s]) and the summed stats."""
    _check_sweeps("shared_shape", shared_shape, temporal_weight, "the shared shape's pose step")
    _check_sweeps("refine_cameras", refine_cameras, temporal_weight, "the camera refinement's body step")
    plans = [_render_plan(q, image_folder, render_folder) for q in seqs]
    S_ = len(seqs)
    tw = temporal_weight_vector(temporal_weight)
    latent = _uses_latent_pose(stage_cfgs)
    seq_rig = rig_views = None
    if rigs is not None:
        rig_views = [int(np.asarray(r["R"]).shape[0]) for r in rigs]
        seq_rig = np.array([int(q["rig"]) for q in seqs], np.int32)
        for q, r in zip(seqs, seq_rig):
            if not 0 <= r < len(rigs):
                raise ValueError("fit_sequences: sequence %s names rig %d of %d" % (q.get("serial"), r, len(rigs)))
            if q["gt_uv"].shape[0] != rig_views[r]:
                raise ValueError("fit_sequences: sequence %s has %d views, its rig %d has %d"
                                 % (q.get("serial"), q["gt_uv"].shape[0], r, rig_views[r]))
        ctx.set_camera_rigs(rigs, rig_data_weight_scale)
        V = max(rig_views)
        seqs = [_pad_views(q, V) for q in seqs]
    for s_, q in enumerate(seqs):
        _check_missing_views(q, stage_cfgs, None if seq_rig is None else rig_views[seq_rig[s_]])
    t3 = _targets_3d(seqs, stage_cfgs, use_hip) if use_3d else None
    if ctx.B != S_:
        return _fit_sequences_stream(ctx, seqs, stage_cfgs, opt_cfg, latent, reinit_loss, result_folder, mesh_folder, faces,
                                     pose_format, use_hip, dict(estimate_scale=estimate_scale, fixed_scale=fixed_scale,
                                                                use_torso=True, hip_seed=1.0, want_joints3d=False,
                                                                umeyama_as_written=umeyama_as_written), t3, seq_rig, rig_views, tw,
                                     shared_shape, refine_cameras, plans)
    T = max(len(q["frames"]) for q in seqs)
    V = seqs[0]["gt_uv"].shape[0]
    off = np.concatenate([[0], np.cumsum([len(q["frames"]) for q in seqs])])
    jw = joint_weights(pose_format, use_hip)
    prev = None
    prev_loss = np.full(S_, np.inf, np.float32)
    out_x = [np.zeros((len(q["frames"]), 86), np.float32) for q in seqs]
    out_l = [np.zeros(len(q["frames"]), np.float32) for q in seqs]
    tot = dict(frame_iterations=0, frame_evals=0, rounds=0, frames_nan=0)
    for t in range(T):
        live = np.array([t < len(q["frames"]) for q in seqs])
        gt = np.zeros((V, S_, NUM_BODY_JOINTS, 2), np.float32)
        cf = np.zeros((V, S_, NUM_BODY_JOINTS), np.float32)
        for s_, q in enumerate(seqs):
            if live[s_]:
                gt[:, s_], cf[:, s_] = q["gt_uv"][:, t], q["conf"][:, t]
            else:                              # a finished sequence idles on its last frame (results are not kept)
                gt[:, s_], cf[:, s_] = q["gt_uv"][:, -1], q["conf"][:, -1]
        if seq_rig is not None:
            ctx.set_frame_rigs(seq_rig)
        ctx.set_keypoints(gt, cf, jw)
        ctx.set_loss(config=stage_cfgs[0])
        guess = dict(estimate_scale=estimate_scale, fixed_scale=fixed_scale, use_torso=True, hip_seed=1.0,
                     want_joints3d=False, umeyama_as_written=umeyama_as_written)
        if t3 is None:
            cold, _ = ctx.init_guess(**guess)
        else:                                  # frame t's 3-D rows (the last frame's for a finished sequence)
            rows = [off[s_] + min(t, len(q["frames"]) - 1) for s_, q in enumerate(seqs)]
            j3, c3, has = t3[0][rows], t3[1][rows], t3[2][rows]
            cold = _init_guess_3d(ctx, guess, j3, c3, has)
            ctx.set_joints3d(j3, c3)
        warm = np.zeros(S_, bool) if prev is None else (prev_loss <= reinit_loss)
        params = cold
        if warm.any():
            carried = prev.clone()
            if not latent:                     # fix_params: the body pose restarts from the hip seed
                carried[:, 13:82] = cold[:, 13:82]
            wm = torch.as_tensor(warm, device=params.device)
            params = torch.where(wm[:, None], carried, cold).contiguous()
        if tw is not None and warm.any():      # prev: step t-1's fitted rows, before load_init / fix_params
            final, st = ctx.fit(params, stage_cfgs, opt_cfg, warm=warm, prev=prev, temporal_weight=tw)
        else:
            final, st = ctx.fit(params, stage_cfgs, opt_cfg, warm=warm if warm.any() else None)
        for k in tot:
            tot[k] += st[k]
        prev, prev_loss = params, final.cpu().numpy()
        x = params.cpu().numpy()
        for s_, q in enumerate(seqs):
            if live[s_]:
                out_x[s_][t], out_l[s_][t] = x[s_], prev_loss[s_]
        if (result_folder is not None or plans[0] is not None) and not (shared_shape or refine_cameras):
            for s_, q in enumerate(seqs):
                if live[s_]:
                    _export(ctx, q, params, prev_loss, latent, result_folder, mesh_folder, faces, frames=[q["frames"][t]], rows=[s_],
                            plan=plans[s_], rig=None if seq_rig is None else seq_rig[s_])
    if t3 is not None:
        ctx.set_joints3d(None)
    if shared_shape or refine_cameras:
        lengths = [len(q["frames"]) for q in seqs]
        x = torch.as_tensor(np.concatenate(out_x), device=ctx.device).contiguous()
        rig = None if seq_rig is None else np.repeat(seq_rig, lengths).astype(np.int32)
        gt_all = np.concatenate([q["gt_uv"] for q in seqs], axis=1)
        conf_all = np.concatenate([q["conf"] for q in seqs], axis=1)
        if refine_cameras:
            final = refine_rigs(ctx, x, gt_all, conf_all, jw, stage_cfgs, opt_cfg, refine_cameras, t3, rig, tot, result_folder)
        if shared_shape:
            final = share_shape(ctx, x, gt_all, conf_all, jw, lengths, stage_cfgs, opt_cfg, shared_shape, t3, rig, tot)
        final = final.cpu().numpy()
        xs = x.cpu().numpy()
        out_x = [xs[off[s_]:off[s_ + 1]] for s_ in range(S_)]
        out_l = [final[off[s_]:off[s_ + 1]] for s_ in range(S_)]
        if result_folder is not None or plans[0] is not None:
            for s_, q in enumerate(seqs):
                _export_rows(ctx, q, x[off[s_]:off[s_ + 1]], out_l[s_], latent, result_folder, mesh_folder, faces, plans[s_],
                             None if seq_rig is None else seq_rig[s_])
    return list(zip(out_x, out_l)), tot


def _fit_sequences_stream(ctx, seqs, stage_cfgs, opt_cfg, latent, reinit_loss, result_folder, mesh_folder, faces, pose_format,
                          use_hip, guess, t3=None, seq_rig=None, rig_views=None, tw=None, shared_shape=0, refine_cameras=0, plans=None):
    """fit_sequences through mvs_fit_seq_stream: the sequences' frames back to back, every frame's cold start point from
    _cold_guesses; t3: _targets_3d of those frames (mvs_fit_seq_stream3d); seq_rig [S]: each sequence's rig, which every
    one of its frames takes (mvs_fit_seq_stream_rigs); tw [86]: the temporal weight (mvs_fit_seq_stream_temporal);
    shared_shape: sweeps of share_shape after the fit (0: off); refine_cameras: sweeps of refine_rigs before it (0: off); plans:
    each sequence's _render_plan"""
    lengths = [len(q["frames"]) for q in seqs]
    off = np.concatenate([[0], np.cumsum(lengths)])
    gt_uv = np.concatenate([q["gt_uv"] for q in seqs], axis=1)
    conf = np.concatenate([q["conf"] for q in seqs], axis=1)
    jw = joint_weights(pose_format, use_hip)
    rig = None if seq_rig is None else np.repeat(seq_rig, lengths).astype(np.int32)
    params = _cold_guesses(ctx, gt_uv, conf, jw, stage_cfgs, guess, t3, rig, rig_views)
    kw = {} if rig is None else dict(rig=rig)
    if tw is not None:
        kw["temporal_weight"] = tw
    if t3 is not None:
        kw.update(joints3d=t3[0], conf3d=t3[1])
    final, stats = ctx.fit_seq_stream(params, gt_uv, conf, jw, lengths, stage_cfgs, opt_cfg, reinit_loss=reinit_loss, **kw)
    if t3 is not None:
        ctx.set_joints3d(None)
    if refine_cameras:
        final = refine_rigs(ctx, params, gt_uv, conf, jw, stage_cfgs, opt_cfg, refine_cameras, t3, rig, stats, result_folder)
    if shared_shape:
        final = share_shape(ctx, params, gt_uv, conf, jw, lengths, stage_cfgs, opt_cfg, shared_shape, t3, rig, stats)
    x, loss = params.cpu().numpy(), final.cpu().numpy()
    if result_folder is not None or (plans and plans[0] is not None):
        for s_, q in enumerate(seqs):
            _export_rows(ctx, q, params[off[s_]:off[s_ + 1]], loss[off[s_]:off[s_ + 1]], latent, result_folder, mesh_folder, faces,
                         None if plans is None else plans[s_], None if seq_rig is None else seq_rig[s_])
    return [(x[off[s_]:off[s_ + 1]], loss[off[s_]:off[s_ + 1]]) for s_ in range(len(seqs))], stats
