"""CPU: the ctypes mirror of mvs_sequence_stream (mvsmplfitting_b200/_lib.py) has the C struct's size and field offsets, as the
host compiler lays out include/mvsmpl.h; fit_sequences with a batch other than the number of sequences drives the sequence
stream with every frame's cold start point and exports one result per frame."""
import ctypes
import os
import pickle
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

FIELDS = ("n_sequences", "seq_offsets", "params", "gt_uv", "conf", "joint_weights", "final_loss", "reinit_loss")


def test_sequence_stream_layout_matches_the_header(tmp_path):
    cxx = shutil.which("g++") or shutil.which("c++")
    if cxx is None:
        pytest.skip("no host C++ compiler")
    from mvsmplfitting_b200 import _lib
    src = tmp_path / "probe.cpp"
    lines = ['#include <cstddef>', '#include <cstdio>', '#include "mvsmpl.h"', "int main() {",
             '    std::printf("sizeof %zu\\n", sizeof(mvs_sequence_stream));']
    lines += ['    std::printf("%s %%zu\\n", offsetof(mvs_sequence_stream, %s));' % (f, f) for f in FIELDS]
    lines += ["    return 0;", "}"]
    src.write_text("\n".join(lines) + "\n")
    exe = tmp_path / "probe"
    subprocess.check_call([cxx, "-std=c++17", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    out = dict(line.split() for line in subprocess.check_output([str(exe)], text=True).splitlines())
    assert int(out["sizeof"]) == ctypes.sizeof(_lib.SequenceStream)
    assert [name for name, _ in _lib.SequenceStream._fields_] == list(FIELDS)
    for f in FIELDS:
        assert int(out[f]) == getattr(_lib.SequenceStream, f).offset, f


class StreamStubCtx:
    """records what fit_sequences asks of a FittingContext whose batch differs from the number of sequences"""
    def __init__(self, B):
        self.B, self.calls, self.device = B, [], "cpu"

    def set_keypoints(self, gt_uv, conf, jw):
        self.calls.append(("kp", gt_uv.shape))

    def set_loss(self, config=None):
        self.calls.append(("loss",))

    def init_guess(self, **kw):
        import torch
        n = len([c for c in self.calls if c[0] == "init"])
        self.calls.append(("init",))
        return (torch.arange(self.B, dtype=torch.float32)[:, None] + 100 * n).expand(self.B, 86).contiguous(), None

    def fit_seq_stream(self, params, gt_uv, conf, jw, lengths, stage_cfgs, opt_cfg=None, reinit_loss=5000.0):
        import torch
        self.calls.append(("stream", gt_uv.shape, list(lengths), reinit_loss, params.clone()))
        params += 0.5
        return torch.arange(params.shape[0], dtype=torch.float32), dict(frame_iterations=3, frame_evals=4, rounds=1, frames_nan=0)

    def fit(self, *a, **k):
        raise AssertionError("the lock-step path is for a batch of one frame per sequence")


@pytest.mark.parametrize("B", [1, 3])
def test_fit_sequences_with_another_batch_uses_the_sequence_stream(B, tmp_path):
    from mvsmplfitting_b200 import seqio
    V, K = 2, 17

    def seq(T, serial):
        return dict(gt_uv=np.zeros((V, T, K, 2), np.float32), conf=np.ones((V, T, K), np.float32),
                    present=np.ones((V, T), bool), frames=["%05d" % t for t in range(T)], serial=serial)

    from types import SimpleNamespace
    cfgs = [SimpleNamespace(use_vposer=0, use_joints_conf=1) for _ in range(4)]
    seqs = [seq(3, "a"), seq(1, "b")]
    ctx = StreamStubCtx(B)
    res, st = seqio.fit_sequences(ctx, seqs, cfgs, result_folder=str(tmp_path), reinit_loss=7.0)
    stream = [c for c in ctx.calls if c[0] == "stream"]
    assert len(stream) == 1 and stream[0][1] == (V, 4, K, 2) and stream[0][2] == [3, 1] and stream[0][3] == 7.0
    # cold start points: ctx.B frames per init_guess call, frames back to back
    assert len([c for c in ctx.calls if c[0] == "init"]) == -(-4 // B)
    start = stream[0][4].numpy()[:, 0]
    assert start.tolist() == [(f % B) + 100 * (f // B) for f in range(4)]
    assert [r[0].shape for r in res] == [(3, 86), (1, 86)] and res[1][1].tolist() == [3.0] and st["frame_iterations"] == 3
    for q, (x, loss) in zip(seqs, res):
        for t, fr in enumerate(q["frames"]):
            got = pickle.load(open(tmp_path / q["serial"] / fr / "000.pkl", "rb"))
            assert got["loss"] == loss[t] and got["transl"][0, 0] == x[t, 82]
