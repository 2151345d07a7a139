"""per-phase wall time of frame_step_kernel (CTA 0) from the -DMVS_PHASE_DBG build: python scripts/phase_times.py"""
import sys, os, ctypes
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from mvsmplfitting_b200 import _lib, synthetic as S
_lib.LIB_PATH = os.path.join(os.path.dirname(_lib.LIB_PATH), "libmvsmpl_dbg.so")
from mvsmplfitting_b200.context import FittingContext
NAMES = {0: "start", 1: "prologue (frame state cp.async, history cp.async issue, SDF scalars)", 2: "P1 rodrigues/J", 3: "P2 chain",
         4: "P3 A/Phi", 5: "P4 vposed gather", 6: "P5", 7: "P6 keypoints", 8: "P6 projection", 9: "P6 reduce", 10: "P6 scatter",
         11: "P7 dvp/dA", 12: "P8 dPhi", 14: "P9 skin_transform_bwd", 15: "reverse sweep", 16: "P10a",
         17: "P10 rodrigues_bwd/betas, join with warps 6-7 (GMM, |theta|^2)", 21: "priors + angle", 22: "total/grad",
         23: "g_eval store + cp.async wait", 24: "L-BFGS advance", 26: "rodrigues (next) + write-back (warps 4-7)",
         27: "chain (next)", 28: "A/Phi store (next)"}
model = S.make_model(0); gmm = S.make_gmm(7); cams = S.make_cameras(8)
B = int(sys.argv[1]) if len(sys.argv) > 1 else 256
fr = S.make_frames(model, cams, B, seed=1000)
ctx = FittingContext(0)
ctx.set_model(model); ctx.set_gmm_from_dict(gmm)
ctx.set_cameras(cams["R"], cams["t"], cams["f"], cams["c"]); ctx.set_batch(B)
ctx.set_keypoints(fr["gt_uv"], fr["conf"], fr["joint_weights"])
x = torch.tensor(S.pack_params(fr["init"]), device="cuda")
SDF = not (len(sys.argv) > 2 and sys.argv[2] == "resident")      # "resident": the frame-resident kernel's last evaluation
ctx.set_loss(body_prior="gmm", interpenetration=SDF, coll_loss_weight=1000.0 if SDF else 0.0, data_weight=500 / 1536,
             body_pose_weight=57.4, shape_weight=10.0, bending_prior_weight=3.17 * 57.4)
ctx.lbfgs_run(x, ctx.make_lbfgs_config(max_outer=1, max_iter=12))
torch.cuda.synchronize()
buf = (ctypes.c_longlong * 64)()
lib = ctypes.CDLL(_lib.LIB_PATH)
assert lib.mvs_debug_clocks(buf, 64) == 0
clk = torch.cuda.get_device_properties(0).clock_rate if hasattr(torch.cuda.get_device_properties(0), "clock_rate") else 1.965e6
ghz = 1.965
prev = buf[0]
print("phase                                                        cycles      us (at %.3f GHz)" % ghz)
for i in sorted(NAMES)[1:]:
    if buf[i] == 0 or buf[i] < prev:
        print("%2d %-56s (not reached in the last launch)" % (i, NAMES.get(i, "")))
        continue
    d = buf[i] - prev
    print("%2d %-56s %8d %8.2f" % (i, NAMES.get(i, ""), d, d / ghz / 1e3))
    prev = buf[i]
print("total %.2f us" % ((prev - buf[0]) / ghz / 1e3))
print("max over all CTAs and launches (us): closure %.2f | history wait %.2f | advance (+ write-back) %.2f | next pose %.2f | "
      "start->advanced %.2f | start->end %.2f" % tuple(buf[32 + k] / ghz / 1e3 for k in range(6)))

print("longest two-loop recursion: %.2f us with %d history pairs" % (buf[40] / ghz / 1e3, buf[41]))
# tensor-core contraction: stamps of CTA (0, 0) in the last launch
tb = (ctypes.c_longlong * 32)()
if hasattr(lib, "mvs_debug_tc_clocks") and lib.mvs_debug_tc_clocks(tb, 32) == 0 and tb[0]:
    def us(i): return (tb[i] - tb[0]) / ghz / 1e3
    print("posedirs_gemm_tc CTA(0,0), us from kernel entry: setup done %.2f | first ring stage landed %.2f | row tiles done %s | "
          "epilogue (tile ready, stored) %s | exit %.2f" % (
              us(1), us(2), ["%.2f" % us(3 + i) for i in range(4) if tb[3 + i] > tb[0]],
              ["%.2f/%.2f" % (us(8 + 2 * i), us(9 + 2 * i)) for i in range(4) if tb[8 + 2 * i] > tb[0]], us(20)))
