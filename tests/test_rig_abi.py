"""CPU: the ctypes signatures of the camera-rig entry points (mvsmplfitting_b200/_lib.py) match include/mvsmpl.h, as the host
compiler reads the header, and seqio.fit_sequences(rigs=...) drives a context as the rig contract says (recording stub)."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

from mvsmplfitting_b200 import seqio
from tests.test_seqio import StubCtx, _cfgs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ("mvs_set_cameras", "mvs_set_camera_rigs", "mvs_set_frame_rigs", "mvs_fit_stream", "mvs_fit_stream_rigs",
       "mvs_fit_seq_stream", "mvs_fit_seq_stream3d", "mvs_fit_seq_stream_rigs")


def _code(t) -> str:
    """one letter per ctypes argument type: i int, f float, u unsigned, p pointer"""
    if t is ctypes.c_int:
        return "i"
    if t is ctypes.c_float:
        return "f"
    if t is ctypes.c_uint:
        return "u"
    if t is ctypes.c_void_p or issubclass(t, ctypes._Pointer):
        return "p"
    raise AssertionError("unexpected argument type %r" % (t,))


def test_rig_entry_points_match_the_header(tmp_path):
    cxx = shutil.which("g++") or shutil.which("c++")
    if cxx is None:
        pytest.skip("no host C++ compiler")
    from mvsmplfitting_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("libmvsmpl.so is not built")
    lib = _lib.load()
    src = tmp_path / "probe.cpp"
    lines = ['#include <cstdio>', '#include <string>', '#include <type_traits>', '#include "mvsmpl.h"',
             "template <class T> char code() {",
             "    if (std::is_pointer<T>::value) return 'p';",
             "    if (std::is_same<T, int>::value) return 'i';",
             "    if (std::is_same<T, float>::value) return 'f';",
             "    if (std::is_same<T, unsigned>::value) return 'u';",
             "    return '?';", "}",
             "template <class R, class... A> std::string sig(R (*)(A...)) {",
             "    std::string s = std::is_same<R, int>::value ? \"i:\" : \"?:\";",
             "    ((s += code<A>()), ...);", "    return s;", "}", "int main() {"]
    lines += ['    std::printf("%s %%s\\n", sig(static_cast<decltype(&%s)>(nullptr)).c_str());' % (n, n) for n in NEW]
    lines += ["    return 0;", "}"]
    src.write_text("\n".join(lines) + "\n")
    exe = tmp_path / "probe"
    subprocess.check_call([cxx, "-std=c++17", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    want = dict(line.split() for line in subprocess.check_output([str(exe)], text=True).splitlines())
    for n in NEW:
        f = getattr(lib, n)
        got = ("i:" if f.restype is ctypes.c_int else "?:") + "".join(_code(t) for t in f.argtypes)
        assert got == want[n], (n, got, want[n])
        assert n in _lib.EXPORTS


class RigStub(StubCtx):
    """StubCtx with the rig entry points and the stream: records what the drivers upload"""

    def __init__(self, B):
        super().__init__(B)
        self.device = "cpu"

    def set_camera_rigs(self, rigs, scale=None):
        self.calls.append(("rigs", [np.asarray(r["R"]).shape[0] for r in rigs], None if scale is None else list(scale)))

    def set_frame_rigs(self, rig):
        self.calls.append(("frame_rigs", list(map(int, rig))))

    def set_keypoints(self, gt_uv, conf, jw):
        super().set_keypoints(gt_uv, conf, jw)
        self.kp = (np.array(gt_uv), np.array(conf))

    def fit_seq_stream(self, params, gt_uv, conf, jw, lengths, stage_cfgs, opt_cfg=None, reinit_loss=5000.0, rig=None, **kw):
        import torch
        self.calls.append(("seq_stream", np.array(gt_uv).shape, list(lengths), None if rig is None else list(map(int, rig))))
        self.stream_kp = (np.array(gt_uv), np.array(conf))
        return torch.zeros(params.shape[0]), dict(frame_iterations=1, frame_evals=1, rounds=1, frames_nan=0)


def _cams(V):
    return dict(R=np.tile(np.eye(3, dtype=np.float32), (V, 1, 1)), t=np.zeros((V, 3), np.float32),
                f=np.ones((V, 2), np.float32), c=np.zeros((V, 2), np.float32))


def _seq(V, T, rig, serial, missing=None):
    gt = np.full((V, T, 17, 2), float(V), np.float32)
    conf = np.ones((V, T, 17), np.float32)
    present = np.ones((V, T), bool)
    if missing is not None:
        present[missing] = False
        conf[missing] = 0.0
    return dict(gt_uv=gt, conf=conf, present=present, frames=["%05d" % t for t in range(T)], serial=serial, rig=rig)


def test_fit_sequences_with_rigs_lockstep_and_stream():
    rigs = [_cams(2), _cams(4), _cams(3)]
    seqs = [_seq(2, 3, 0, "a"), _seq(4, 2, 1, "b"), _seq(3, 2, 2, "c")]
    # lock-step (B = S): the rig table once, each step the slots' rigs before the keypoints; views padded to Vmax = 4
    ctx = RigStub(3)
    seqio.fit_sequences(ctx, seqs, _cfgs(4), rigs=rigs, rig_data_weight_scale=[1.0, 0.5, 2.0])
    names = [c[0] for c in ctx.calls]
    assert ctx.calls[0] == ("rigs", [2, 4, 3], [1.0, 0.5, 2.0])
    assert names.count("frame_rigs") == 3 and names.count("fit") == 3
    for i, n in enumerate(names):
        if n == "kp":
            assert names[i - 1] == "frame_rigs" and ctx.calls[i - 1][1] == [0, 1, 2] and ctx.calls[i][1] == (4, 3, 17, 2)
    # stream (B != S): per-frame rigs [F], each sequence's frames with its rig; cold guesses name the slots' rigs per chunk and
    # take no rows beyond a frame's own views
    ctx = RigStub(2)
    seqio.fit_sequences(ctx, seqs, _cfgs(4), rigs=rigs)
    st = [c for c in ctx.calls if c[0] == "seq_stream"]
    assert len(st) == 1 and st[0][1] == (4, 7, 17, 2) and st[0][2] == [3, 2, 2] and st[0][3] == [0, 0, 0, 1, 1, 2, 2]
    fr = [c[1] for c in ctx.calls if c[0] == "frame_rigs"]
    assert fr == [[0, 0], [0, 1], [1, 2], [2, 2]]                       # the last chunk's padding row takes its first rig
    gt, cf = ctx.stream_kp
    assert (gt[2:, :3] == 0).all() and (gt[:2, :3] == 2).all() and (gt[3:, 5:] == 0).all() and (gt[:3, 5:] == 3).all()
    assert (cf[2:, :3] == 0).all() and (cf[:, 3:5] == 1).all()
    # the last chunk's keypoints: frame 6 (rig 2, three views) and a zero padding row
    assert (ctx.kp[0][:3, 0] == 3).all() and (ctx.kp[0][3:, 0] == 0).all() and (ctx.kp[1][:, 1] == 0).all()


def test_fit_sequences_with_rigs_checks():
    rigs = [_cams(2), _cams(4)]
    # a missing view of the sequence's own rig needs use_joints_conf; its padding rows do not count
    seqs = [_seq(2, 2, 0, "a"), _seq(4, 2, 1, "b", missing=(3, 1))]
    with pytest.raises(ValueError, match="use_joints_conf"):
        seqio.fit_sequences(RigStub(2), seqs, _cfgs(4, use_joints_conf=0), rigs=rigs)
    seqio.fit_sequences(RigStub(2), [_seq(2, 2, 0, "a"), _seq(4, 2, 1, "b")], _cfgs(4, use_joints_conf=0), rigs=rigs)
    with pytest.raises(ValueError, match="views"):
        seqio.fit_sequences(RigStub(2), [_seq(3, 2, 0, "a")], _cfgs(4), rigs=rigs)
    with pytest.raises(ValueError, match="names rig"):
        seqio.fit_sequences(RigStub(2), [_seq(2, 2, 5, "a")], _cfgs(4), rigs=rigs)
    # without rigs nothing of the rig interface is touched
    ctx = RigStub(1)
    seqio.fit_sequences(ctx, [_seq(2, 2, 0, "a")], _cfgs(4))
    assert not any(c[0] in ("rigs", "frame_rigs") for c in ctx.calls)
