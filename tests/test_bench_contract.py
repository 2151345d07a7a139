"""CPU: bench.py stays importable without a GPU and its bookkeeping covers every kernel the library can report."""
import importlib.util
import os

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _bench():
    spec = importlib.util.spec_from_file_location("bench", os.path.join(ROOT, "bench.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def test_stage_table_and_workload():
    b = _bench()
    st = b.stage_table()
    assert len(st) == 4 and st[2]["coll_loss_weight"] > 0 and st[0]["coll_loss_weight"] == 0
    cfg = b.workload_config(256, 8, True)
    assert "workload" in cfg and "model" in cfg and "cfg4" in cfg["workload"]
    assert b.METRIC and b.UNIT


def test_algorithmic_bytes_cover_every_kernel_id():
    from mvsmplfitting_b200 import _lib
    b = _bench()
    lib = _lib.load()
    names = [lib.mvs_kernel_name(k).decode() for k in range(_lib.NUM_KERNEL_IDS)]
    assert "sdf_fused" in names and "frame_step" in names and "posedirs_gemm_tc" in names and "skin" in names
    for n in names:
        assert b.algorithmic_bytes(n, 128.0, 8, dense=True) > 0, n
    assert b.gemm_flops(128.0) == 2.0 * 128 * 207 * 20670


def test_lanes_and_reference_worker_flags_parse():
    """--inflight (batches in flight) and the hidden --ref-worker mode are part of the command line the driver / the reference arm use"""
    import subprocess
    import sys
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--help"], capture_output=True, text=True).stdout
    assert "--inflight" in out and "--impl" in out and "--ref-device" in out and "--ref-worker " not in out
