"""per-CTA phase times of sdf_fused_kernel from the -DMVS_PHASE_DBG build (python -m mvsmplfitting_b200.build --debug first):

    python scripts/sdf_phase_times.py [B ...]

Runs dense-regime closures (exec mode 3: posedirs_gemm_tc -> skin -> sdf_setup -> sdf_fused -> frame_step, one round each) at every batch
size and prints, per CTA that ran to the end, the mean and the largest time of each phase (see the SDF_MARK stamps in
mvs_sdf.cu), then the CTAs per launch, the waves they make at 3 CTAs/SM and waves x mean CTA time against the kernel's event
time per launch (profiled in a separate loop of the same build)."""
import ctypes
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
from mvsmplfitting_b200 import _lib, synthetic as S  # noqa: E402
_lib.LIB_PATH = os.path.join(os.path.dirname(_lib.LIB_PATH), os.environ.get("MVS_LIB", "libmvsmpl_dbg.so"))
from mvsmplfitting_b200.context import FittingContext  # noqa: E402

PHASES = {1: "start -> pdl_wait returned", 2: "-> box folded (after the barrier)", 3: "-> cone/plane set-up + cull verdicts",
          4: "-> sampling done (after the barrier)", 5: "-> block reduction + adjoint done"}
REPS = 20
model, gmm, cams = S.make_model(0), S.make_gmm(7), S.make_cameras(8)
lib = ctypes.CDLL(_lib.LIB_PATH)
buf = (ctypes.c_ulonglong * 32)()
sms = torch.cuda.get_device_properties(0).multi_processor_count
print(torch.cuda.get_device_properties(0).name)
for B in [int(a) for a in sys.argv[1:]] or [256, 64, 8, 1]:
    fr = S.make_frames(model, cams, B, seed=1000)
    ctx = FittingContext(0)
    ctx.set_model(model); ctx.set_gmm_from_dict(gmm); ctx.set_cameras(cams["R"], cams["t"], cams["f"], cams["c"]); ctx.set_batch(B)
    ctx.set_keypoints(fr["gt_uv"], fr["conf"], fr["joint_weights"])
    ctx.set_exec_mode(3)
    ctx.set_loss(body_prior="gmm", interpenetration=True, coll_loss_weight=1000.0, sdf_grid=128, data_weight=500 / 1536,
                 body_pose_weight=57.4, shape_weight=10.0, bending_prior_weight=3.17 * 57.4)
    x = torch.tensor(S.pack_params(fr["init"]), device="cuda")
    for _ in range(3):
        ctx.closure(x)
    torch.cuda.synchronize()
    assert lib.mvs_debug_sdf_clocks(buf, 32, 1) == 0
    for _ in range(REPS):
        ctx.closure(x)
    torch.cuda.synchronize()
    assert lib.mvs_debug_sdf_clocks(buf, 32, 1) == 0
    ctas = buf[16]
    ghz = buf[18] / max(buf[17], 1)
    ctx.profile(0xFFFFFFFF)
    for _ in range(REPS):
        ctx.closure(x)
    pr = ctx.profile_read()
    ctx.profile(0)
    ev_us = pr["sdf_fused"][0] * 1e3 / pr["sdf_fused"][1]
    print("B=%d: %d CTAs per launch, SM clock %.3f GHz (clock64 / globaltimer)" % (B, ctas // REPS, ghz))
    tot = 0.0
    for k in range(1, 6):
        mean = buf[k] / ctas / ghz / 1e3
        tot += mean
        print("  %-42s mean %7.2f us   max %7.2f us" % (PHASES[k], mean, buf[8 + k] / ghz / 1e3))
    setup = (buf[2] + buf[3]) / ctas / ghz / 1e3
    post = tot - buf[1] / ctas / ghz / 1e3
    waves = -(-(ctas // REPS) // (3 * sms))
    print("  CTA total %.2f us (after pdl_wait %.2f us); set-up (box fold + cone/cull) %.2f us = %.0f %% of the CTA, %.0f %% after "
          "pdl_wait" % (tot, post, setup, 100 * setup / tot, 100 * setup / max(post, 1e-9)))
    print("  %d wave(s) at 3 CTAs/SM x %.2f us = %.1f us vs sdf_fused event time %.1f us per launch" % (waves, tot, waves * tot, ev_us))
    ctx.close()
