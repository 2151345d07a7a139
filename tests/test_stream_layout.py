"""CPU: the ctypes mirror of mvs_frame_stream (mvsmplfitting_b200/_lib.py) has the C struct's size and field offsets, as
the host compiler lays out include/mvsmpl.h."""
import ctypes
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

FIELDS = ("n_frames", "params", "gt_uv", "conf", "joint_weights", "gt_xyz", "conf3d", "final_loss")


def test_frame_stream_layout_matches_the_header(tmp_path):
    cxx = shutil.which("g++") or shutil.which("c++")
    if cxx is None:
        pytest.skip("no host C++ compiler")
    from mvsmplfitting_b200 import _lib
    src = tmp_path / "probe.cpp"
    lines = ['#include <cstddef>', '#include <cstdio>', '#include "mvsmpl.h"', "int main() {",
             '    std::printf("sizeof %zu\\n", sizeof(mvs_frame_stream));']
    lines += ['    std::printf("%s %%zu\\n", offsetof(mvs_frame_stream, %s));' % (f, f) for f in FIELDS]
    lines += ["    return 0;", "}"]
    src.write_text("\n".join(lines) + "\n")
    exe = tmp_path / "probe"
    subprocess.check_call([cxx, "-std=c++17", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    out = dict(line.split() for line in subprocess.check_output([str(exe)], text=True).splitlines())
    assert int(out["sizeof"]) == ctypes.sizeof(_lib.FrameStream)
    assert [name for name, _ in _lib.FrameStream._fields_] == list(FIELDS)
    for f in FIELDS:
        assert int(out[f]) == getattr(_lib.FrameStream, f).offset, f
