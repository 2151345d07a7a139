// The camera step of mvs_refine_cameras (DESIGN.md section 4): per view problem, the 2-D data term of one view of one rig over
// the frames with that rig, at keypoints held from the body fit, as a function of the view's extrinsics update.  The optimiser
// is the 86-vector state machine of mvs_lbfgs.cu; these kernels are its closure and the write-back into the rig table.
#include "mvs_internal.cuh"
#include "mvs_lbfgs_core.cuh"

namespace mvs {

// The camera of a view problem at its update (w, c): compiled once and called by both the closure and the write-back, so the
// table receives exactly the camera the closure evaluated.  S: the state of the adjoint (closure only).
__device__ __noinline__ void build_camera(const CamRefine& cr, const float* w, const float* c, float* R, float* t,
                                          CamDeltaState<float>* S) {
    cam_from_delta(cr, w, c, R, t, *S);
}

// One warp per work item (problem slot, frame of its rig), lane = keypoint.  The frame's view term is resident_closure P6's for
// that view: the same projection (with the view's distortion, held like f and c), weights, GMoF and dw^2, the keypoints' terms
// added in keypoint order.  Its gradient with respect to the camera (R, t) is summed over the keypoints, then taken back to the
// problem's variables.  At most 64 registers, so that eight 128-thread CTAs stay resident per SM: the out-of-line distorted
// projection would otherwise take the kernel to 68 (allocated as 72: seven CTAs); at 64 it does not spill.
__global__ void __launch_bounds__(128, 8)
camera_closure_kernel(LossParams lp, LbfgsState L, CameraArgs a, ProblemChunk ch) {
    const int lane = threadIdx.x & 31;
    const int item = ch.i0 + blockIdx.x * 4 + (threadIdx.x >> 5);
    if (item >= ch.i0 + ch.ni) return;
    const int p = ch.item_of[item], j = p - ch.base;
    if (L.sc[j].phase == PH_DONE) return;                                // the problem has finished
    const CameraProblem P = a.prob[p];
    const int f = a.frames[P.fbeg + item - ch.beg[p]], K = a.K, F = a.in.n;
    const CamRefine cr = a.cr[p];
    const float* xe = L.x_eval + (size_t)j * kParams;
    const float w[3] = {xe[kOffOrient], xe[kOffOrient + 1], xe[kOffOrient + 2]};
    const float c[3] = {xe[kOffTransl], xe[kOffTransl + 1], xe[kOffTransl + 2]};
    CamDeltaState<float> S;
    CamF cam;
    build_camera(cr, w, c, cam.R, cam.t, &S);
    const Rig& rig = a.rigs[P.rig];
    cam.f[0] = rig.cam[P.view].f[0]; cam.f[1] = rig.cam[P.view].f[1];
    cam.c[0] = rig.cam[P.view].c[0]; cam.c[1] = rig.cam[P.view].c[1];
    const Dist* dp = rig.distorted ? rig.dist + P.view : nullptr;    // the view's distortion (NULL: none), held like f and c
    const float dw = lp.data_weight * rig.dw_scale;
    const float rho2 = lp.rho * lp.rho, dw2 = dw * dw;
    float lterm = 0.f, g[12];
#pragma unroll
    for (int i = 0; i < 12; ++i) g[i] = 0.f;
    if (lane < K) {
        const float* q = a.q + ((size_t)f * K + lane) * 3;
        const float qk[3] = {q[0], q[1], q[2]};
        float xc[3], uv[2];
        project_fwd(cam, qk, xc, uv, dp);
        const size_t o = ((size_t)P.view * F + f) * K + lane;
        float wk = a.in.joint_w[lane];
        if (lp.use_joints_conf) wk *= a.in.conf[o];
        const float w2 = wk * wk;
        float d0, d1;
        const float g0 = gmof(a.in.gt_uv[2 * o] - uv[0], rho2, &d0);
        const float g1 = gmof(a.in.gt_uv[2 * o + 1] - uv[1], rho2, &d1);
        lterm = w2 * g0 + w2 * g1;
        const float duv[2] = {-(w2 * d0) * dw2, -(w2 * d1) * dw2};
        float dx[3];
        project_bwd_x(cam, xc, duv, dx, dp);
#pragma unroll
        for (int r = 0; r < 3; ++r) {
#pragma unroll
            for (int k = 0; k < 3; ++k) g[3 * r + k] = dx[r] * qk[k];
            g[9 + r] = dx[r];
        }
    }
    float acc = 0.f;                                                     // P6's order: keypoint 0, 1, ..., K-1
    for (int k = 0; k < K; ++k) acc += __shfl_sync(0xffffffffu, lterm, k);
#pragma unroll
    for (int i = 0; i < 12; ++i) g[i] = warp_sum(g[i]);
    if (lane == 0) {
        float gw[3], gc[3];
        cam_from_delta_bwd(cr, w, c, S, g, g + 9, gw, gc);
        float* out = ch.part + (size_t)item * kPartCols;
        out[0] = acc * dw2;
        out[1] = gw[0]; out[2] = gw[1]; out[3] = gw[2];
        out[4] = gc[0]; out[5] = gc[1]; out[6] = gc[2];
    }
}

// One thread per problem: the camera at the problem's row into its rig's view
__global__ void camera_write_kernel(Rig* __restrict__ rigs, const CamRefine* __restrict__ cr, const CameraProblem* __restrict__ prob,
                                    int P, const float* __restrict__ x) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= P) return;
    const float* xp = x + (size_t)p * kParams;
    const float w[3] = {xp[kOffOrient], xp[kOffOrient + 1], xp[kOffOrient + 2]};
    const float c[3] = {xp[kOffTransl], xp[kOffTransl + 1], xp[kOffTransl + 2]};
    const CamRefine crp = cr[p];
    CamDeltaState<float> S;
    float R[9], t[3];
    build_camera(crp, w, c, R, t, &S);
    CamF& cam = rigs[prob[p].rig].cam[prob[p].view];
    for (int i = 0; i < 9; ++i) cam.R[i] = R[i];
    for (int i = 0; i < 3; ++i) cam.t[i] = t[i];
}

// One warp per row
__global__ void row_finite_kernel(const float* __restrict__ params, int F, int* __restrict__ fin) {
    const int f = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (f >= F) return;
    bool ok = true;
    for (int i = lane; i < kParams; i += 32) ok = ok && isfinite(params[(size_t)f * kParams + i]);
    ok = __all_sync(0xffffffffu, ok);
    if (lane == 0) fin[f] = ok ? 1 : 0;
}

int launch_camera_closure(mvs_ctx* ctx, const CameraArgs& a, const ProblemChunk& c, const LossParams& lp, const LbfgsState& L,
                          cudaStream_t st) {
    if (c.ni > 0)
        MVS_LAUNCH(ctx, KID_MISC, st, camera_closure_kernel<<<(c.ni + 3) / 4, 128, 0, st>>>(lp, L, a, c));
    MVS_CUDA_OK(ctx, cudaGetLastError());
    return MVS_OK;
}

int launch_camera_write(mvs_ctx* ctx, const CamRefine* cr, const CameraProblem* prob, int P, const float* x, cudaStream_t st) {
    if (P > 0)
        MVS_LAUNCH(ctx, KID_MISC, st, camera_write_kernel<<<(P + 63) / 64, 64, 0, st>>>(ctx->rigs_dev.p, cr, prob, P, x));
    MVS_CUDA_OK(ctx, cudaGetLastError());
    return MVS_OK;
}

int launch_row_finite(mvs_ctx* ctx, const float* params, int F, int* fin, cudaStream_t st) {
    MVS_LAUNCH(ctx, KID_MISC, st, row_finite_kernel<<<(F + 3) / 4, 128, 0, st>>>(params, F, fin));
    MVS_CUDA_OK(ctx, cudaGetLastError());
    return MVS_OK;
}

}  // namespace mvs
