// Per-frame initial guess on the device, all frames at once (SURVEY §8f row N2; the reference does it per frame in
// numpy: code/utils/init_guess.py:18-107 + fix_params :190-212, called from main.py:76-82).
//
//   1. rest joints: the model's keypoints at zero pose, zero shape, scale = fixed_scale  (init_guess.py:29-52)
//      -- the library's own forward pass on a seeded parameter block;
//   2. triangulation of the K keypoints from the V views                                 (recompute3D.py:24-61)
//      (a rig with lens distortion: every detection with non-zero confidence undistorted first, mvs_init.cuh undistort_px)
//   3. similarity alignment rest joints -> triangulated joints, torso joints only by default (init_guess.py:80-85),
//      rotation -> axis-angle (:86), and the parameter block fix_params leaves behind (:190-212).
//
// One warp per frame: lane k triangulates keypoint k (double accumulation: two-camera rigs are ill-conditioned in
// float), lane 0 solves the 3x3 alignment.  The arithmetic is mvs_init.cuh, which tests/hostsim runs on the CPU against
// reference-run golden vectors.  HBM traffic is the detections once (V*K*12 B per frame) + 344 B of parameters out:
// the kernel is launch-latency sized, not bandwidth sized.
#include <string.h>

#include "mvs_internal.cuh"
#include "mvs_init.cuh"

namespace mvs {

__global__ void init_seed_kernel(float* __restrict__ params, int B, float scale) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * kParams) return;
    params[i] = (i % kParams == kOffScale) ? scale : 0.f;
}

// params [B,86] (written completely), rest [K,3] rest joints of the model (the same for every frame),
// gt_uv [Vmax,B,K,2], conf [Vmax,B,K] (rows v < the frame's rig's view count are read); targets [B,K,3] (3-D joint term on) or nullptr; joints3d [B,K,3] or nullptr
__global__ void __launch_bounds__(128) init_guess_kernel(float* __restrict__ params, const float* __restrict__ rest,
                                                         RigSet rigs, const float* __restrict__ gt_uv,
                                                         const float* __restrict__ conf, const float* __restrict__ targets,
                                                         int B, int K, int estimate_scale,
                                                         float fixed_scale, int use_torso, float hip_seed, int as_written,
                                                         float* __restrict__ joints3d) {
    __shared__ double s_dst[4][kMaxKeypoints * 3];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int b = blockIdx.x * 4 + warp;
    if (b >= B) return;                                   // whole warps leave together; only __syncwarp below
    double* dst = s_dst[warp];
    float* x = params + (size_t)b * kParams;
    for (int i = lane; i < kParams; i += 32) x[i] = 0.f;
    if (lane < K) {
        const FrameRig cams = frame_rig(rigs, b);            // this frame's rig: its views, or one view's depth guess
        double X[3];
        if (targets) {                                    // init_guess.py:85-86: the 3-D annotations replace both guesses
            for (int c = 0; c < 3; ++c) X[c] = (double)targets[((size_t)b * K + lane) * 3 + c];
        } else if (cams.num_views == 1) {                 // init_guess.py:54-78: depth guess along the optical axis
            double rj[kMaxKeypoints * 3];
            for (int i = 0; i < K * 3; ++i) rj[i] = (double)rest[i];
            const double d = single_view_depth<double>(cams.cam[0], rj, gt_uv + (size_t)b * K * 2, conf + (size_t)b * K,
                                                       cams.dist);
            for (int c = 0; c < 3; ++c) X[c] = rj[3 * lane + c] + d * (double)cams.cam[0].R[6 + c];
        } else {
            triangulate_point<double>(cams, gt_uv + ((size_t)b * K + lane) * 2, conf + (size_t)b * K + lane, (long)B * K * 2,
                                      (long)B * K, X, cams.dist);
        }
        dst[3 * lane] = X[0]; dst[3 * lane + 1] = X[1]; dst[3 * lane + 2] = X[2];
        if (joints3d) {
            float* o = joints3d + ((size_t)b * K + lane) * 3;
            o[0] = (float)X[0]; o[1] = (float)X[1]; o[2] = (float)X[2];
        }
    }
    __syncwarp();
    if (lane != 0) return;
    const int torso[4] = {5, 6, 11, 12};                  // init_guess.py:82-84
    double src[kMaxKeypoints * 3], sel[kMaxKeypoints * 3];
    const int n = use_torso ? 4 : K;
    for (int i = 0; i < n; ++i) {
        const int k = use_torso ? torso[i] : i;
        for (int c = 0; c < 3; ++c) {
            src[3 * i + c] = (double)rest[k * 3 + c];
            sel[3 * i + c] = dst[3 * k + c];
        }
    }
    double R[9], t[3], sc = 1.0, aa[3] = {0.0, 0.0, 0.0};
    if (umeyama_fit<double>(src, sel, n, estimate_scale != 0, R, t, &sc, as_written != 0)) {
        rotmat_to_aa<double>(R, aa);
    } else {                                              // degenerate detections (the reference raises): translate only
        sc = 1.0;
        for (int c = 0; c < 3; ++c) {
            double ms = 0.0, md = 0.0;
            for (int i = 0; i < n; ++i) { ms += src[3 * i + c]; md += sel[3 * i + c]; }
            t[c] = (md - ms) / n;
        }
    }
    for (int c = 0; c < 3; ++c) {
        x[kOffOrient + c] = (float)aa[c];
        x[kOffTransl + c] = (float)t[c];
    }
    for (int c = 0; c < 6; ++c) x[kOffPose + c] = hip_seed;        // fix_params, init_guess.py:198-201
    x[kOffScale] = estimate_scale ? (float)sc : fixed_scale;      // init_guess.py:88-91
}

}  // namespace mvs

using namespace mvs;

extern "C" int mvs_init_guess(mvs_ctx* ctx, float* params_dev, float* joints3d_dev, const mvs_init_config* cfg, void* stream) {
    if (!ctx) return set_error(nullptr, MVS_ERR_INVALID, "ctx is NULL");
    if (!(ctx->have_model && ctx->have_cams && ctx->have_kp && ctx->ws.B > 0))
        return set_error(ctx, MVS_ERR_INVALID, "mvs_init_guess: model, cameras, batch and keypoints must be set first");
    if (!params_dev || !cfg) return set_error(ctx, MVS_ERR_INVALID, "mvs_init_guess: NULL argument");
    if (int rc = batch_rigs(ctx, "mvs_init_guess")) return rc;
    const int K = ctx->m.K, B = ctx->ws.B;
    if (cfg->use_torso && K < 13) return set_error(ctx, MVS_ERR_INVALID, "mvs_init_guess: use_torso needs keypoints 5, 6, 11, 12");
    if (!(cfg->fixed_scale > 0.f)) return set_error(ctx, MVS_ERR_INVALID, "mvs_init_guess: fixed_scale must be positive");
    MVS_CUDA_OK(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = (cudaStream_t)stream;
    Workspace& w = ctx->ws;
    if (K * 3 > kParams) return set_error(ctx, MVS_ERR_INVALID, "mvs_init_guess: more than 28 keypoints");
    const bool j3d = ctx->j3d_enabled;
    if (!j3d && K < 13)                                    // per frame: the frames whose rig has one view
        for (int b = 0; b < B; ++b)
            if (ctx->rigs[ctx->slot_rigs ? ctx->slot_rig_host[b] : 0].num_views == 1)
                return set_error(ctx, MVS_ERR_INVALID, "mvs_init_guess: the single-view depth guess (frame %d) needs keypoints 5, 6, "
                                                       "11, 12", b);
    // Rest joints (zero pose, zero shape, scale = fixed_scale; init_guess.py:29-52) are a property of the model: computed once
    // per context and scale with the library's own forward pass (seed + the 3-kernel geometry chain), then cached, so that a
    // call is ONE launch afterwards.
    if (!ctx->rest_joints) {
        int rc = dev_alloc(ctx, &ctx->rest_joints, (size_t)kMaxKeypoints * 3);
        if (rc) return rc;
    }
    if (ctx->rest_scale != cfg->fixed_scale) {
        float* rest = w.grad_scratch;                      // [B,86] scratch of the closure; K*3 <= 86 floats per frame
        MVS_LAUNCH(ctx, KID_MISC, st, init_seed_kernel<<<(B * kParams + 255) / 256, 256, 0, st>>>(params_dev, B, cfg->fixed_scale));
        const int vposer = ctx->loss.use_vposer;           // the rest pose is body_pose = 0 whatever the pose encoding
        ctx->loss.use_vposer = 0;                          // (the geometry-only chain never reads the 3-D targets)
        const int rc = launch_closure(ctx, params_dev, nullptr, nullptr, rest, nullptr, nullptr, st, true);
        ctx->loss.use_vposer = vposer;
        if (rc) return rc;
        MVS_CUDA_OK(ctx, cudaMemcpyAsync(ctx->rest_joints, rest, (size_t)K * 3 * sizeof(float), cudaMemcpyDeviceToDevice, st));
        ctx->rest_scale = cfg->fixed_scale;
    }
    MVS_LAUNCH(ctx, KID_MISC, st,
               init_guess_kernel<<<(B + 3) / 4, 128, 0, st>>>(params_dev, ctx->rest_joints, slot_rig_set(ctx), w.gt_uv, w.conf,
                                                              j3d ? w.j3d_xyz : nullptr, B, K,
                                                              cfg->estimate_scale, cfg->fixed_scale, cfg->use_torso,
                                                              ctx->loss.use_vposer == 2 ? 0.f : cfg->hip_seed,
                                                              cfg->umeyama_as_written, joints3d_dev));
    MVS_CUDA_OK(ctx, cudaGetLastError());
    return MVS_OK;
}
