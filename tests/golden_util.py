"""helpers shared by the golden-fixture tests"""
import glob
import hashlib
import json
import os

import numpy as np

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
DEMO = os.path.join(GOLD, "demo")          # the data the original project ships (data/keypoints, data/3DOH50K_Parameters.txt)


def model_checksum(model):
    h = hashlib.sha256()
    for k in ("v_template", "shapedirs", "posedirs", "J_regressor", "weights", "lsp_regressor"):
        h.update(np.ascontiguousarray(model[k]).tobytes())
    return h.hexdigest()


def closure_cases():
    return sorted(os.path.basename(p)[len("closure_"):-4] for p in glob.glob(os.path.join(GOLD, "closure_*.npz")))


def load_case(name):
    z = np.load(os.path.join(GOLD, "closure_%s.npz" % name))
    d = {k: z[k] for k in z.files}
    d["meta"] = json.loads(str(d["meta"]))
    d["cams"] = {k: d["cam_" + k] for k in ("R", "t", "f", "c")}
    w = d["weights"]
    d["w"] = dict(data_weight=float(w[0]), body_pose_weight=float(w[1]), shape_weight=float(w[2]),
                  bending_prior_weight=float(w[3]))
    return d


def relmax(a, b):
    """max-norm relative error of a against reference b"""
    return float(np.abs(np.asarray(a, dtype=np.float64) - b).max() / max(np.abs(b).max(), 1e-30))


def snapshot_vposer_weights():
    """decoder weights of the VPoser snapshot the original project ships (priors/snapshots/poser_epoch091.pkl), as read by its
    own loader (oracle/make_golden_refruns.py); stored in two files so that each stays under 1 MB"""
    a, b = np.load(os.path.join(GOLD, "vposer_snapshot_a.npz")), np.load(os.path.join(GOLD, "vposer_snapshot_b.npz"))
    return dict(fc1_w=a["fc1_w"], fc1_b=a["fc1_b"], fc2_w=np.concatenate([a["fc2_w_top"], b["fc2_w_bottom"]]), fc2_b=a["fc2_b"],
                out_w=b["out_w"], out_b=b["out_b"])
