// The batched fitting closure: SMPL forward, keypoint loss and the hand-derived adjoint,
// for every frame in flight.  Replaces (reference paths under code/):
//   smplx/body_models_scale.py:327-412 + smplx/lbs.py:135-370  (SMPL forward)
//   camera.py:93-117, utils/utils.py:427-438, utils/fitting.py:290-350 (projection, GMoF data term, priors)
//   and the autograd backward of all of it (utils/fitting.py:190-192).
//
// Kernel chain for one evaluation (all on the caller's stream, no host sync):
//   frame_fwd     (CTA / frame)   Rodrigues, rest joints, kinematic chain -> Phi rows, skinning transforms
//   vertex_fwd    (64 frames x 32 vertices / CTA)   v_posed = Phi . Qk^T  (blend shapes as ONE contraction),
//                                 linear blend skinning fused in the epilogue, coalesced stores
//   [sdf_*        (mvs_sdf.cu)    interpenetration term, dense d loss / d vertex]
//   keypoint_loss (CTA / frame)   sparse joint regression, V-view projection, GMoF, d loss / d vertex
//   vertex_bwd    (strip of vertex tiles x 64 frames / CTA)   adjoint of skinning + contraction,
//                                 per-strip partials (deterministic, no float atomics)
//   frame_bwd     (CTA / frame)   partial reduction, chain + Rodrigues adjoints, priors, loss, grad[86]
//
// The vertex kernels run on a vertex LIST: all 6890 vertices when vertices / the SDF term are
// requested, otherwise only the <= 86 vertices the keypoints depend on (SURVEY H4).
#include <stdarg.h>
#include <stdio.h>

#include "mvs_internal.cuh"

namespace mvs {

struct PoseSmem {
    float x[kParams + 2];
    float R[kJoints * 9];
    float J[kJoints * 3];
    float Gam[kJoints * 9];
    float g[kJoints * 3];
};

// Rodrigues for 24 joints, rest joints from betas, kinematic chain with the scaled root.
// Must be called by all threads of a block with >= 104 threads.
__device__ __forceinline__ void pose_forward_block(const float* __restrict__ xf, const Parents& par,
                                                   const float* __restrict__ Jt, const float* __restrict__ JS,
                                                   PoseSmem& s) {
    const int t = threadIdx.x;
    for (int i = t; i < kParams; i += blockDim.x) s.x[i] = xf[i];
    __syncthreads();
    if (t < kJoints) {
        rodrigues_fwd(&s.x[kOffOrient + 3 * t], &s.R[9 * t]);
    } else if (t >= 32 && t < 32 + 72) {
        const int jc = t - 32;
        float a = Jt[jc];
#pragma unroll
        for (int l = 0; l < kBetas; ++l) a = fmaf(JS[jc * kBetas + l], s.x[kOffBetas + l], a);
        s.J[jc] = a;
    }
    __syncthreads();
    if (t == 0) {
        const float sc = s.x[kOffScale];
#pragma unroll
        for (int i = 0; i < 9; ++i) s.Gam[i] = sc * s.R[i];      // lbs.py:348
        s.g[0] = s.J[0]; s.g[1] = s.J[1]; s.g[2] = s.J[2];
        for (int j = 1; j < kJoints; ++j) {
            const int p = par.p[j];
            float rel[3] = {s.J[3 * j] - s.J[3 * p], s.J[3 * j + 1] - s.J[3 * p + 1], s.J[3 * j + 2] - s.J[3 * p + 2]};
            chain_step_fwd(&s.Gam[9 * p], &s.g[3 * p], &s.R[9 * j], rel, &s.Gam[9 * j], &s.g[3 * j]);
        }
    }
    __syncthreads();
}

// ------------------------------------------------------------------------------------------ K1
__global__ void __launch_bounds__(kFrameThreads)
frame_fwd_kernel(const float* __restrict__ x, const int* __restrict__ fidx, const int* __restrict__ na_ptr,
                 Parents par, const float* __restrict__ Jt, const float* __restrict__ JS,
                 float* __restrict__ Phi, float* __restrict__ PhiTc, float* __restrict__ At, int ldA,
                 float* __restrict__ gchain, float* __restrict__ slot_tr) {
    pdl_wait();
    const int slot = blockIdx.x;
    if (slot >= *na_ptr) return;
    const int b = fidx[slot];
    __shared__ PoseSmem s;
    pose_forward_block(x + (size_t)b * kParams, par, Jt, JS, s);
    const int t = threadIdx.x;
    if (slot_tr && t < 3) slot_tr[4 * slot + t] = x[(size_t)b * kParams + kOffTransl + t];
    for (int k = t; k < kFeatPad; k += blockDim.x) {
        float v;
        if (k < kPoseBasis) v = s.R[9 + k] - (((k % 9) % 4 == 0) ? 1.0f : 0.0f);   // lbs.py:192
        else if (k < kPoseBasis + kBetas) v = s.x[kOffBetas + k - kPoseBasis];
        else v = (k == kFeat - 1) ? 1.0f : 0.0f;
        Phi[(size_t)slot * kFeatPad + k] = v;
        if (PhiTc) {                 // A operand of the tensor-core contraction: pose feature only, v = hi + lo, both TF32
            float hi = 0.f, lo = 0.f;
            if (k < kPoseBasis) tf32_split(v, hi, lo);
            PhiTc[(size_t)slot * kFeatPad + k] = hi;
            PhiTc[((size_t)ldA + slot) * kFeatPad + k] = lo;
        }
    }
    if (t < kJoints) {
        float A[12];
        make_skin_transform(&s.Gam[9 * t], &s.g[3 * t], &s.J[3 * t], A);
#pragma unroll
        for (int c = 0; c < 12; ++c) At[(size_t)(t * 12 + c) * ldA + slot] = A[c];
        gchain[((size_t)slot * kJoints + t) * 3 + 0] = s.g[3 * t];
        gchain[((size_t)slot * kJoints + t) * 3 + 1] = s.g[3 * t + 1];
        gchain[((size_t)slot * kJoints + t) * 3 + 2] = s.g[3 * t + 2];
    }
}

// ------------------------------------------------------------------------------------------ K2
constexpr int kQsLd = kGemmKC + 4;      // 20: conflict-free LDS.128 for the strided thread->row map
constexpr int kVpLd = kTileC + 1;       // 97
constexpr size_t kVertFwdSmem = (size_t)(kTileC * kQsLd + kTileF * kQsLd + 2 * kTileF * kVpLd) * sizeof(float);

__global__ void __launch_bounds__(kVertThreads)
vertex_fwd_kernel(const float* __restrict__ Qk, const float* __restrict__ Phi, const float* __restrict__ At, int ldA,
                  const int* __restrict__ ell_j, const float* __restrict__ ell_w, int KW,
                  const int* __restrict__ vlist, int nv, const int* __restrict__ na_ptr,
                  float* __restrict__ vposed, float* __restrict__ verts) {
    extern __shared__ __align__(16) float smem[];
    float* Qs = smem;                         // [96][20]
    float* Ps = Qs + kTileC * kQsLd;          // [64][20]
    float* Vp = Ps + kTileF * kQsLd;          // [64][97]  v_posed tile
    float* Vo = Vp + kTileF * kVpLd;          // [64][97]  skinned tile
    __shared__ int s_n[kTileV];
    const int na = *na_ptr;
    const int f0 = blockIdx.y * kTileF;
    if (f0 >= na) return;
    const int v0 = blockIdx.x * kTileV;
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    if (tid < kTileV) {
        const int vi = v0 + tid;
        s_n[tid] = vi < nv ? (vlist ? vlist[vi] : vi) : -1;
    }
    __syncthreads();

    float acc[4][6];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 6; ++j) acc[i][j] = 0.f;

    for (int k0 = 0; k0 < kFeatPad; k0 += kGemmKC) {
        for (int idx = tid; idx < kTileC * 4; idx += kVertThreads) {
            const int row = idx >> 2, q = idx & 3;
            const int n = s_n[row / 3], c = row % 3;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (n >= 0) v = __ldg(reinterpret_cast<const float4*>(Qk + (size_t)(3 * n + c) * kFeatPad + k0 + 4 * q));
            *reinterpret_cast<float4*>(&Qs[row * kQsLd + 4 * q]) = v;
        }
        {
            const int row = tid >> 2, q = tid & 3, slot = f0 + row;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (slot < na) v = *reinterpret_cast<const float4*>(Phi + (size_t)slot * kFeatPad + k0 + 4 * q);
            *reinterpret_cast<float4*>(&Ps[row * kQsLd + 4 * q]) = v;
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < kGemmKC; kk += 4) {
            float4 p[4], q[6];
#pragma unroll
            for (int i = 0; i < 4; ++i) p[i] = *reinterpret_cast<const float4*>(&Ps[(ty + 16 * i) * kQsLd + kk]);
#pragma unroll
            for (int j = 0; j < 6; ++j) q[j] = *reinterpret_cast<const float4*>(&Qs[(tx + 16 * j) * kQsLd + kk]);
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 6; ++j) {
                    acc[i][j] = fmaf(p[i].x, q[j].x, acc[i][j]);
                    acc[i][j] = fmaf(p[i].y, q[j].y, acc[i][j]);
                    acc[i][j] = fmaf(p[i].z, q[j].z, acc[i][j]);
                    acc[i][j] = fmaf(p[i].w, q[j].w, acc[i][j]);
                }
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 6; ++j) Vp[(ty + 16 * i) * kVpLd + tx + 16 * j] = acc[i][j];
    __syncthreads();

    // linear blend skinning, lane = frame (coalesced reads of the frame-fastest transforms)
    {
        const int b = tid & 63, vg = tid >> 6;
        const int slotc = min(f0 + b, na - 1);
        for (int ii = 0; ii < 8; ++ii) {
            const int i = vg * 8 + ii;
            const int n = s_n[i];
            if (n < 0) continue;
            const float p0 = Vp[b * kVpLd + 3 * i], p1 = Vp[b * kVpLd + 3 * i + 1], p2 = Vp[b * kVpLd + 3 * i + 2];
            float T[12];
#pragma unroll
            for (int c = 0; c < 12; ++c) T[c] = 0.f;
            for (int e = 0; e < KW; ++e) {
                const float w = ell_w[(size_t)n * KW + e];
                if (w != 0.f) {
                    const int j = ell_j[(size_t)n * KW + e];
#pragma unroll
                    for (int c = 0; c < 12; ++c) T[c] = fmaf(w, At[(size_t)(j * 12 + c) * ldA + slotc], T[c]);
                }
            }
#pragma unroll
            for (int r = 0; r < 3; ++r)
                Vo[b * kVpLd + 3 * i + r] = T[4 * r] * p0 + T[4 * r + 1] * p1 + T[4 * r + 2] * p2 + T[4 * r + 3];
        }
    }
    __syncthreads();
    for (int idx = tid; idx < kTileF * kTileC; idx += kVertThreads) {
        const int b = idx / kTileC, col = idx % kTileC;
        const int slot = f0 + b, vi = v0 + col / 3;
        if (slot < na && vi < nv) {
            const size_t off = ((size_t)slot * nv + v0) * 3 + col;
            vposed[off] = Vp[b * kVpLd + col];
            verts[off] = Vo[b * kVpLd + col];
        }
    }
}

// ------------------------------------------------------------------------------------------ K3
struct KeypointModel {
    int K, nsup, N;
    const int* kp_ptr; const int* kp_vidx; const int* kp_spos; const float* kp_w; const int* kp_chain;
    const int* sup; const int* sup_ptr; const int* sup_k; const float* sup_w;
};

__global__ void __launch_bounds__(kFrameThreads)
keypoint_loss_kernel(const float* __restrict__ x, const int* __restrict__ fidx, const int* __restrict__ na_ptr,
                     KeypointModel km, const float* __restrict__ verts, int nv, int dense,
                     const float* __restrict__ gchain, CamSet cams, const float* __restrict__ gt_uv,
                     const float* __restrict__ conf, const float* __restrict__ joint_w, int B, LossParams lp,
                     float* __restrict__ data_loss, float* __restrict__ dtransl, float* __restrict__ dv,
                     int dv_stride, float* __restrict__ dgchain, float* __restrict__ joints_out,
                     float* __restrict__ proj_out) {
    const int slot = blockIdx.x;
    if (slot >= *na_ptr) return;
    const int b = fidx[slot];
    const int t = threadIdx.x;
    const int K = km.K, V = cams.num_views;
    __shared__ float q[kMaxKeypoints * 3];
    __shared__ float dq[kMaxKeypoints * 3];
    __shared__ float contrib[kMaxViews * kMaxKeypoints * 3];
    __shared__ float lterm[kMaxViews * kMaxKeypoints];
    __shared__ float vsum[kMaxViews];
    const float* vf = verts + (size_t)slot * nv * 3;
    if (t < K) {
        float a0 = 0.f, a1 = 0.f, a2 = 0.f;
        for (int e = km.kp_ptr[t]; e < km.kp_ptr[t + 1]; ++e) {
            const int pos = dense ? km.kp_vidx[e] : km.kp_spos[e];
            const float w = km.kp_w[e];
            a0 = fmaf(w, vf[3 * pos], a0); a1 = fmaf(w, vf[3 * pos + 1], a1); a2 = fmaf(w, vf[3 * pos + 2], a2);
        }
        const int cj = km.kp_chain[t];
        if (cj >= 0) {
            a0 += gchain[((size_t)slot * kJoints + cj) * 3]; a1 += gchain[((size_t)slot * kJoints + cj) * 3 + 1];
            a2 += gchain[((size_t)slot * kJoints + cj) * 3 + 2];
        }
        const float* tr = x + (size_t)b * kParams + kOffTransl;       // body_models_scale.py:401-402
        q[3 * t] = a0 + tr[0]; q[3 * t + 1] = a1 + tr[1]; q[3 * t + 2] = a2 + tr[2];
        if (joints_out) {
            joints_out[((size_t)b * K + t) * 3] = q[3 * t]; joints_out[((size_t)b * K + t) * 3 + 1] = q[3 * t + 1];
            joints_out[((size_t)b * K + t) * 3 + 2] = q[3 * t + 2];
        }
    }
    __syncthreads();
    const float rho2 = lp.rho * lp.rho;
    const float dw2 = lp.data_weight * lp.data_weight;
    for (int idx = t; idx < V * K; idx += blockDim.x) {
        const int v = idx / K, k = idx % K;
        float xc[3], uv[2];
        project_fwd(cams.cam[v], &q[3 * k], xc, uv);
        const size_t o = ((size_t)v * B + b) * K + k;
        if (proj_out) { proj_out[2 * o] = uv[0]; proj_out[2 * o + 1] = uv[1]; }
        float w = joint_w[k];
        if (lp.use_joints_conf) w *= conf[o];
        const float w2 = w * w;
        float d0, d1;
        const float g0 = gmof(gt_uv[2 * o] - uv[0], rho2, &d0);
        const float g1 = gmof(gt_uv[2 * o + 1] - uv[1], rho2, &d1);
        lterm[idx] = w2 * g0 + w2 * g1;
        const float duv[2] = {-(w2 * d0) * dw2, -(w2 * d1) * dw2};
        float dqv[3] = {0.f, 0.f, 0.f};
        project_bwd(cams.cam[v], xc, duv, dqv);
        contrib[3 * idx] = dqv[0]; contrib[3 * idx + 1] = dqv[1]; contrib[3 * idx + 2] = dqv[2];
    }
    __syncthreads();
    if (t < K) {
        float a0 = 0.f, a1 = 0.f, a2 = 0.f;
        for (int v = 0; v < V; ++v) {
            a0 += contrib[3 * (v * K + t)]; a1 += contrib[3 * (v * K + t) + 1]; a2 += contrib[3 * (v * K + t) + 2];
        }
        dq[3 * t] = a0; dq[3 * t + 1] = a1; dq[3 * t + 2] = a2;
    } else if (t >= 32 && t < 32 + V) {
        const int v = t - 32;
        float a = 0.f;
        for (int k = 0; k < K; ++k) a += lterm[v * K + k];
        vsum[v] = a * dw2;                                           // fitting.py:313-315
    }
    __syncthreads();
    if (t == 0) {
        float a = 0.f;
        for (int v = 0; v < V; ++v) a += vsum[v];
        data_loss[slot] = a;
    }
    if (t >= 32 && t < 35) {
        const int c = t - 32;
        float a = 0.f;
        for (int k = 0; k < K; ++k) a += dq[3 * k + c];
        dtransl[(size_t)slot * 3 + c] = a;
    }
    if (t >= 64 && t < 64 + kJoints) {
        const int j = t - 64;
        float a0 = 0.f, a1 = 0.f, a2 = 0.f;
        for (int k = 0; k < K; ++k)
            if (km.kp_chain[k] == j) { a0 += dq[3 * k]; a1 += dq[3 * k + 1]; a2 += dq[3 * k + 2]; }
        dgchain[((size_t)slot * kJoints + j) * 3] = a0; dgchain[((size_t)slot * kJoints + j) * 3 + 1] = a1;
        dgchain[((size_t)slot * kJoints + j) * 3 + 2] = a2;
    }
    for (int i = t; i < km.nsup; i += blockDim.x) {
        float a0 = 0.f, a1 = 0.f, a2 = 0.f;
        for (int e = km.sup_ptr[i]; e < km.sup_ptr[i + 1]; ++e) {
            const int k = km.sup_k[e];
            const float w = km.sup_w[e];
            a0 = fmaf(w, dq[3 * k], a0); a1 = fmaf(w, dq[3 * k + 1], a1); a2 = fmaf(w, dq[3 * k + 2], a2);
        }
        // keypoint gradients occupy the first nsup entries of the frame's backward list (the SDF term, when on,
        // appends one entry per vertex after them)
        float* d = dv + ((size_t)slot * dv_stride + i) * 3;
        d[0] = a0; d[1] = a1; d[2] = a2;
    }
}

// ------------------------------------------------------------------------------------------ K4
constexpr int kDvLd = kTileF + 1;        // 65
constexpr int kDvpLd = kTileF + 4;       // 68 (16-byte aligned rows)
constexpr int kBwdCols = 16;             // columns of Qk staged per step
constexpr int kQbLd = kFeatPad + 4;      // 228
constexpr size_t kVertBwdSmem =
    (size_t)(2 * kTileC * kDvLd + kTileC * kDvpLd + kTileV * kJoints + kBwdCols * kQbLd + kSkinFloats * kTileF) * sizeof(float);

__global__ void __launch_bounds__(kVertThreads, 1)
vertex_bwd_kernel(const float* __restrict__ Qk, const float* __restrict__ At, int ldA,
                  const int* __restrict__ ell_j, const float* __restrict__ ell_w, int KW,
                  const float* __restrict__ Wd, const int* __restrict__ blist_n, const int* __restrict__ blist_pos,
                  int nvb, int nv_fwd, const float* __restrict__ vposed, const float* __restrict__ dv,
                  const int* __restrict__ na_ptr, int tiles_per_strip, int ntiles, float* __restrict__ part) {
    extern __shared__ __align__(16) float smem[];
    float* DV = smem;                          // [96][65]   upstream d loss / d vertex, column-major
    float* VP = DV + kTileC * kDvLd;           // [96][65]   v_posed
    float* dVp = VP + kTileC * kDvLd;          // [96][68]   d loss / d v_posed
    float* Ws = dVp + kTileC * kDvpLd;         // [32][24]
    float* Qs = Ws + kTileV * kJoints;         // [16][228]
    float* Ats = Qs + kBwdCols * kQbLd;        // [288][64] this CTA's skinning transforms, frame fastest
    __shared__ int s_n[kTileV], s_pos[kTileV];
    const int na = *na_ptr;
    const int f0 = blockIdx.y * kTileF;
    if (f0 >= na) return;
    const int strip = blockIdx.x;
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int b = tid & 63, jg = tid >> 6;
    bool ats_loaded = false;            // the 73 KB of transforms are fetched when the first active tile shows up

    float accP[4][14];
    float accA[6][12];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int k = 0; k < 14; ++k) accP[i][k] = 0.f;
#pragma unroll
    for (int j = 0; j < 6; ++j)
#pragma unroll
        for (int c = 0; c < 12; ++c) accA[j][c] = 0.f;

    // strided tile -> strip map: neighbouring tiles (e.g. the three keypoint-support tiles that always carry
    // gradient) land in different CTAs instead of serialising inside one
    const int nstrips_g = gridDim.x;
    (void)tiles_per_strip;
    for (int tile = strip; tile < ntiles; tile += nstrips_g) {
        const int v0 = tile * kTileV;
        __syncthreads();
        if (tid < kTileV) {
            const int vi = v0 + tid;
            s_n[tid] = vi < nvb ? (blist_n ? blist_n[vi] : vi) : -1;
            s_pos[tid] = vi < nvb ? (blist_pos ? blist_pos[vi] : vi) : 0;
        }
        __syncthreads();
        int any = 0;
        for (int idx = tid; idx < kTileF * kTileC; idx += kVertThreads) {
            const int bb = idx / kTileC, col = idx % kTileC;
            const int slot = f0 + bb, vi = v0 + col / 3;
            float d = 0.f, p = 0.f;
            if (slot < na && vi < nvb) {
                d = dv[((size_t)slot * nvb + v0) * 3 + col];
                p = vposed[((size_t)slot * nv_fwd + s_pos[col / 3]) * 3 + col % 3];
            }
            DV[col * kDvLd + bb] = d;
            VP[col * kDvLd + bb] = p;
            any |= (d != 0.f);
        }
        for (int idx = tid; idx < kTileV * kJoints; idx += kVertThreads) {
            const int n = s_n[idx / kJoints];
            Ws[idx] = n >= 0 ? Wd[(size_t)n * kJoints + idx % kJoints] : 0.f;
        }
        if (!__syncthreads_or(any)) continue;          // no upstream gradient anywhere in this tile
        if (!ats_loaded) {
            for (int e = tid; e < kSkinFloats * kTileF; e += kVertThreads)
                Ats[e] = At[(size_t)(e >> 6) * ldA + min(f0 + (e & 63), na - 1)];
            ats_loaded = true;
            __syncthreads();
        }

        // d v_posed = T_3x3^T d v     (lane = frame)
        for (int ii = 0; ii < 8; ++ii) {
            const int i = jg * 8 + ii;
            const int n = s_n[i];
            float o0 = 0.f, o1 = 0.f, o2 = 0.f;
            if (n >= 0) {
                const float d0 = DV[(3 * i) * kDvLd + b], d1 = DV[(3 * i + 1) * kDvLd + b], d2 = DV[(3 * i + 2) * kDvLd + b];
                float G[9];
#pragma unroll
                for (int c = 0; c < 9; ++c) G[c] = 0.f;
                for (int e = 0; e < KW; ++e) {
                    const float w = ell_w[(size_t)n * KW + e];
                    if (w != 0.f) {
                        const int j = ell_j[(size_t)n * KW + e];
#pragma unroll
                        for (int r = 0; r < 3; ++r)
#pragma unroll
                            for (int c = 0; c < 3; ++c)
                                G[3 * r + c] = fmaf(w, Ats[(j * 12 + 4 * r + c) * kTileF + b], G[3 * r + c]);
                    }
                }
                o0 = G[0] * d0 + G[3] * d1 + G[6] * d2;
                o1 = G[1] * d0 + G[4] * d1 + G[7] * d2;
                o2 = G[2] * d0 + G[5] * d1 + G[8] * d2;
            }
            dVp[(3 * i) * kDvpLd + b] = o0; dVp[(3 * i + 1) * kDvpLd + b] = o1; dVp[(3 * i + 2) * kDvpLd + b] = o2;
        }
        // d A_j += W[n,j] * [d v (x) v_posed | d v]     (lane = frame, this thread owns joints 6jg..6jg+5)
        for (int i = 0; i < kTileV; ++i) {
            if (s_n[i] < 0) break;
            float d[3], p[3];
            bool loaded = false;
#pragma unroll
            for (int jj = 0; jj < 6; ++jj) {
                const float w = Ws[i * kJoints + 6 * jg + jj];
                if (w != 0.f) {
                    if (!loaded) {
#pragma unroll
                        for (int c = 0; c < 3; ++c) { d[c] = DV[(3 * i + c) * kDvLd + b]; p[c] = VP[(3 * i + c) * kDvLd + b]; }
                        loaded = true;
                    }
#pragma unroll
                    for (int r = 0; r < 3; ++r) {
                        const float wd = w * d[r];
                        accA[jj][4 * r] = fmaf(wd, p[0], accA[jj][4 * r]);
                        accA[jj][4 * r + 1] = fmaf(wd, p[1], accA[jj][4 * r + 1]);
                        accA[jj][4 * r + 2] = fmaf(wd, p[2], accA[jj][4 * r + 2]);
                        accA[jj][4 * r + 3] += wd;
                    }
                }
            }
        }
        // d Phi[b][k] += sum_col dVp[b][col] * Qk[col][k]; the next 16 Qk rows are fetched into registers while
        // the current ones are consumed from shared memory
        constexpr int kQv = (kBwdCols * (kFeatPad / 4) + kVertThreads - 1) / kVertThreads;      // float4 per thread (4)
        float4 qreg[kQv];
        auto fetch = [&](int c0) {
#pragma unroll
            for (int u = 0; u < kQv; ++u) {
                const int idx = tid + u * kVertThreads;
                qreg[u] = make_float4(0.f, 0.f, 0.f, 0.f);
                if (idx < kBwdCols * (kFeatPad / 4)) {
                    const int r = idx / (kFeatPad / 4), q4 = idx % (kFeatPad / 4);
                    const int col = c0 + r, n = s_n[col / 3];
                    if (n >= 0) qreg[u] = __ldg(reinterpret_cast<const float4*>(Qk + (size_t)(3 * n + col % 3) * kFeatPad + 4 * q4));
                }
            }
        };
        fetch(0);
        for (int c0 = 0; c0 < kTileC; c0 += kBwdCols) {
            __syncthreads();
#pragma unroll
            for (int u = 0; u < kQv; ++u) {
                const int idx = tid + u * kVertThreads;
                if (idx < kBwdCols * (kFeatPad / 4))
                    *reinterpret_cast<float4*>(&Qs[(idx / (kFeatPad / 4)) * kQbLd + 4 * (idx % (kFeatPad / 4))]) = qreg[u];
            }
            __syncthreads();
            if (c0 + kBwdCols < kTileC) fetch(c0 + kBwdCols);
#pragma unroll 4
            for (int r = 0; r < kBwdCols; ++r) {
                const float4 d = *reinterpret_cast<const float4*>(&dVp[(c0 + r) * kDvpLd + 4 * ty]);
#pragma unroll
                for (int m = 0; m < 7; ++m) {
                    const float2 qv = *reinterpret_cast<const float2*>(&Qs[r * kQbLd + 14 * tx + 2 * m]);
                    accP[0][2 * m] = fmaf(d.x, qv.x, accP[0][2 * m]); accP[0][2 * m + 1] = fmaf(d.x, qv.y, accP[0][2 * m + 1]);
                    accP[1][2 * m] = fmaf(d.y, qv.x, accP[1][2 * m]); accP[1][2 * m + 1] = fmaf(d.y, qv.y, accP[1][2 * m + 1]);
                    accP[2][2 * m] = fmaf(d.z, qv.x, accP[2][2 * m]); accP[2][2 * m + 1] = fmaf(d.z, qv.y, accP[2][2 * m + 1]);
                    accP[3][2 * m] = fmaf(d.w, qv.x, accP[3][2 * m]); accP[3][2 * m + 1] = fmaf(d.w, qv.y, accP[3][2 * m + 1]);
                }
            }
        }
    }
    // per-strip partials: [strip][slot][288 skin | 224 feature]
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int slot = f0 + 4 * ty + i;
        if (slot < na) {
            float* o = part + ((size_t)strip * ldA + slot) * kPartFloats + kSkinFloats + 14 * tx;
#pragma unroll
            for (int k = 0; k < 14; ++k) o[k] = accP[i][k];
        }
    }
    if (f0 + b < na) {
        float* o = part + ((size_t)strip * ldA + f0 + b) * kPartFloats + (6 * jg) * 12;
#pragma unroll
        for (int j = 0; j < 6; ++j)
#pragma unroll
            for (int c = 0; c < 12; ++c) o[j * 12 + c] = accA[j][c];
    }
}

// ------------------------------------------------------------------------------------------ K5
struct PriorModel {
    int M;
    const float* means; const float* prec; const float* lognllw;
};

__global__ void __launch_bounds__(kFrameThreads)
frame_bwd_kernel(const float* __restrict__ x, const int* __restrict__ fidx, const int* __restrict__ na_ptr,
                 Parents par, const float* __restrict__ Jt, const float* __restrict__ JS,
                 const float* __restrict__ part, int nstrips, int ldA, int have_grad,
                 const float* __restrict__ data_loss, const float* __restrict__ pen_loss /* NULL: term off */,
                 const float* __restrict__ dtransl, const float* __restrict__ dgchain, PriorModel pm, LossParams lp,
                 const float* __restrict__ anchor, const float* __restrict__ anchor_w,
                 float* __restrict__ loss_out, float* __restrict__ grad_out) {
    const int slot = blockIdx.x;
    if (slot >= *na_ptr) return;
    const int b = fidx[slot];
    const int t = threadIdx.x;
    __shared__ PoseSmem s;
    __shared__ float dA[kSkinFloats];
    __shared__ float dPhi[kFeatPad];
    __shared__ float dR[kJoints * 9], dGam[kJoints * 9], dg[kJoints * 3], dJ[kJoints * 3];
    __shared__ float grad[kParams + 2];
    __shared__ float gm_diff[kPoseBasis / 3];       // 69
    __shared__ float gm_y[kPoseBasis / 3];
    __shared__ float gm_ybest[kPoseBasis / 3];
    __shared__ float red[kFrameThreads];
    __shared__ float s_scalar[8];
    pose_forward_block(x + (size_t)b * kParams, par, Jt, JS, s);

    for (int i = t; i < kParams; i += blockDim.x) grad[i] = 0.f;
    if (have_grad) {
        for (int e = t; e < kPartFloats; e += blockDim.x) {
            float a = 0.f;
            const float* pp = part + (size_t)slot * kPartFloats + e;
            const size_t stride = (size_t)ldA * kPartFloats;
            int sidx = 0;
            for (; sidx + 8 <= nstrips; sidx += 8) {       // fixed order, 8 independent L2 reads in flight
                float v[8];
#pragma unroll
                for (int u = 0; u < 8; ++u) v[u] = pp[(size_t)(sidx + u) * stride];
#pragma unroll
                for (int u = 0; u < 8; ++u) a += v[u];
            }
            for (; sidx < nstrips; ++sidx) a += pp[(size_t)sidx * stride];
            if (e < kSkinFloats) dA[e] = a; else dPhi[e - kSkinFloats] = a;
        }
        for (int i = t; i < kJoints * 9; i += blockDim.x) { dGam[i] = 0.f; dR[i] = 0.f; }
        for (int i = t; i < kJoints * 3; i += blockDim.x) { dg[i] = dgchain[(size_t)slot * kJoints * 3 + i]; dJ[i] = 0.f; }
    }
    __syncthreads();
    if (have_grad) {
        if (t < kJoints) skin_transform_bwd(&dA[12 * t], &s.Gam[9 * t], &s.J[3 * t], &dGam[9 * t], &dg[3 * t], &dJ[3 * t]);
        __syncthreads();
        if (t == 0) {
            for (int j = kJoints - 1; j >= 1; --j) {
                const int p = par.p[j];
                float rel[3] = {s.J[3 * j] - s.J[3 * p], s.J[3 * j + 1] - s.J[3 * p + 1], s.J[3 * j + 2] - s.J[3 * p + 2]};
                float drel[3];
                chain_step_bwd(&dGam[9 * j], &dg[3 * j], &s.Gam[9 * p], &s.R[9 * j], rel, &dGam[9 * p], &dg[3 * p],
                               &dR[9 * j], drel);
#pragma unroll
                for (int c = 0; c < 3; ++c) { dJ[3 * j + c] += drel[c]; dJ[3 * p + c] -= drel[c]; }
            }
            const float sc = s.x[kOffScale];
            float ds = 0.f;
#pragma unroll
            for (int i = 0; i < 9; ++i) { dR[i] = sc * dGam[i]; ds = fmaf(dGam[i], s.R[i], ds); }
            dJ[0] += dg[0]; dJ[1] += dg[1]; dJ[2] += dg[2];
            grad[kOffScale] = ds;
        }
        __syncthreads();
        for (int k = t; k < kPoseBasis; k += blockDim.x) dR[9 + k] += dPhi[k];       // adjoint of lbs.py:192-195
        __syncthreads();
        if (t < kJoints) {
            float dr[3] = {0.f, 0.f, 0.f};
            rodrigues_bwd(&s.x[kOffOrient + 3 * t], &dR[9 * t], dr);
            grad[kOffOrient + 3 * t] = dr[0]; grad[kOffOrient + 3 * t + 1] = dr[1]; grad[kOffOrient + 3 * t + 2] = dr[2];
        } else if (t >= 32 && t < 32 + kBetas) {
            const int l = t - 32;
            float a = dPhi[kPoseBasis + l];
            for (int jc = 0; jc < kJoints * 3; ++jc) a = fmaf(JS[jc * kBetas + l], dJ[jc], a);
            grad[kOffBetas + l] = a;
        } else if (t >= 64 && t < 67) {
            grad[kOffTransl + t - 64] = dtransl[(size_t)slot * 3 + t - 64];
        }
        __syncthreads();
    }

    // ---------------- priors (fitting.py:327-350); value + gradient, data-dependent guards on device
    const float bpw = lp.body_pose_weight, bpw2 = bpw * bpw;
    const float* theta = &s.x[kOffPose];
    float pprior = 0.f;          // guarded part
    float l2extra = 0.f;
    float gscale_guarded = 0.f;  // multiplies the guarded gradient
    if (!lp.use_vposer) {
        if (lp.body_prior == MVS_PRIOR_GMM) {
            float best = 3.0e38f;
            for (int m = 0; m < pm.M; ++m) {
                if (t < 69) gm_diff[t] = theta[t] - pm.means[m * 69 + t];
                __syncthreads();
                float y = 0.f;
                if (t < 69) {
                    const float* P = pm.prec + (size_t)m * 69 * 69;
#pragma unroll 3
                    for (int j = 0; j < 69; ++j) y = fmaf(P[j * 69 + t], gm_diff[j], y);   // symmetric: column == row
                    gm_y[t] = y;
                    red[t] = y * gm_diff[t];
                }
                __syncthreads();
                if (t == 0) {
                    float qd = 0.f;
                    for (int i = 0; i < 69; ++i) qd += red[i];
                    s_scalar[0] = 0.5f * qd - pm.lognllw[m];                 // prior.py:188-189
                }
                __syncthreads();
                const float ll = s_scalar[0];
                if (ll < best) {                                             // torch.min keeps the first minimum
                    best = ll;
                    if (t < 69) gm_ybest[t] = gm_y[t];
                }
                __syncthreads();
            }
            pprior = best * bpw2;
        } else if (lp.body_prior == MVS_PRIOR_L2) {
            red[t] = (t < 69) ? theta[t] * theta[t] : 0.f;
            __syncthreads();
            if (t == 0) { float a = 0.f; for (int i = 0; i < 69; ++i) a += red[i]; s_scalar[0] = a; }
            __syncthreads();
            pprior = s_scalar[0] * bpw2;
            if (t < 69) gm_ybest[t] = 2.f * theta[t];
        }
        gscale_guarded = bpw2;
        if (pprior > 5e4f) { pprior = 0.f; gscale_guarded = 0.f; }          // fitting.py:334-335
        __syncthreads();
        red[t] = (t < 69) ? theta[t] * theta[t] : 0.f;
        __syncthreads();
        if (t == 0) { float a = 0.f; for (int i = 0; i < 69; ++i) a += red[i]; s_scalar[1] = a; }
        __syncthreads();
        const float w4 = (bpw * 4.f) * (bpw * 4.f);
        l2extra = s_scalar[1] * w4;                                          // fitting.py:336-337
        if (have_grad && t < 69) {
            float gth = 2.f * theta[t] * w4;
            if (lp.body_prior != MVS_PRIOR_NONE) gth = fmaf(gscale_guarded, gm_ybest[t], gth);
            grad[kOffPose + t] += gth;
        }
    }
    float shape_loss = 0.f;
    if (!lp.fix_shape) {
        const float sw2 = lp.shape_weight * lp.shape_weight;
        float a = 0.f;
        for (int l = 0; l < kBetas; ++l) a = fmaf(s.x[l], s.x[l], a);
        shape_loss = a * sw2;                                                // fitting.py:339-342
        if (have_grad && t < kBetas) grad[kOffBetas + t] += 2.f * s.x[t] * sw2;
    }
    // angle prior on full_pose[3:66][52,55,9,12] with signs (1,-1,-1,-1)  (prior.py:62-66,87-89)
    float angle = 0.f;
    {
        const int idx[4] = {52, 55, 9, 12};
        const float sg[4] = {1.f, -1.f, -1.f, -1.f};
        float ev[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) { const float e = mvs_exp(theta[idx[i]] * sg[i]); ev[i] = e * e; angle += ev[i]; }
        angle *= lp.bending_prior_weight;
        float gs = lp.bending_prior_weight;
        if (angle > 1e4f && !lp.use_vposer) { angle = 0.f; gs = 0.f; }      // fitting.py:349-350
        __syncthreads();
        if (have_grad && t < 4) grad[kOffPose + idx[t]] += 2.f * sg[t] * ev[t] * gs;
    }
    __syncthreads();
    float anchor_loss = 0.f;
    if (lp.anchor_on) {                                   // sequence mode: sum_i w_i (x_i - a_i)^2
        float dif = 0.f, wt = 0.f;
        if (t < kParams) { dif = s.x[t] - anchor[(size_t)b * kParams + t]; wt = anchor_w[(size_t)b * kParams + t]; }
        red[t] = wt * dif * dif;
        if (have_grad && t < kParams) grad[t] += 2.f * wt * dif;
        __syncthreads();
        if (t == 0) { float a = 0.f; for (int i = 0; i < kParams; ++i) a += red[i]; s_scalar[2] = a; }
        __syncthreads();
        anchor_loss = s_scalar[2];
    }
    if (t == 0) {
        // same order as fitting.py:411-413: joint + joints3d + pprior + shape + angle + pen
        float total = data_loss[slot];
        total += (pprior + l2extra);
        total += shape_loss;
        total += angle;
        if (pen_loss) total += pen_loss[slot];
        total += anchor_loss;
        loss_out[b] = total;
    }
    if (have_grad) {
        for (int i = t; i < kParams; i += blockDim.x) {
            int seg = i < kOffOrient ? 0 : i < kOffPose ? 1 : i < kOffTransl ? 2 : i < kOffScale ? 3 : 4;
            grad_out[(size_t)b * kParams + i] = ((lp.frozen_mask >> seg) & 1u) ? 0.f : grad[i];
        }
    }
}

// ------------------------------------------------------------------------------------------ misc
__global__ void verts_out_kernel(const float* __restrict__ verts, const float* __restrict__ x,
                                 const int* __restrict__ fidx, const int* __restrict__ na_ptr, int N,
                                 float* __restrict__ out) {
    const int slot = blockIdx.y;
    if (slot >= *na_ptr) return;
    const int b = fidx[slot];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < N * 3) out[(size_t)b * N * 3 + i] = verts[(size_t)slot * N * 3 + i] + x[(size_t)b * kParams + kOffTransl + i % 3];
}

__global__ void fill_kernel(float* p, float v, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = v;
}

int launch_closure(mvs_ctx* ctx, const float* x_dev, float* loss_dev, float* grad_dev, float* joints_dev,
                   float* proj_dev, float* verts_dev, cudaStream_t st, bool geometry_only) {
    DevModel& m = ctx->m;
    Workspace& w = ctx->ws;
    const LossParams& lp = ctx->loss;
    const int B = w.B;
    const bool sdf_on = !geometry_only && lp.interpenetration && lp.coll_loss_weight > 0.f;
    const bool dense = sdf_on || verts_dev != nullptr;
    const bool have_grad = grad_dev != nullptr;
    if (!dense && !geometry_only && resident_closure_available(ctx))     // sparse regime: one fused launch
        return launch_closure_resident(ctx, x_dev, loss_dev, grad_dev, joints_dev, proj_dev, st);
    if (sdf_on && ctx->exec_mode == 3 && !verts_dev && !joints_dev && !proj_dev && hybrid_available(ctx))
        return dense_regime_closure(ctx, x_dev, loss_dev, grad_dev, st);       // the optimiser's own SDF-stage kernels
    if (lp.use_vposer == 2 && !geometry_only)      // geometry only: the pose slot is axis-angle by definition (mvs_forward)
        return set_error(ctx, MVS_ERR_INVALID, "use_vposer = 2 (VPoser decode on the device) is implemented in the "
                                               "frame-resident closure only (no vertices, no SDF term, exec mode 0 or 2)");
    const int nv = dense ? m.N : m.nsup;
    const int* vlist = dense ? nullptr : m.sup;
    const Parents par = ctx->parents;
    const int ftiles = (B + kTileF - 1) / kTileF;

    if (!ctx->attr_done) {
        MVS_CUDA_OK(ctx, cudaFuncSetAttribute(vertex_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kVertFwdSmem));
        MVS_CUDA_OK(ctx, cudaFuncSetAttribute(vertex_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kVertBwdSmem));
        ctx->attr_done = true;
    }

    MVS_LAUNCH(ctx, KID_FRAME_FWD, st,
               frame_fwd_kernel<<<B, kFrameThreads, 0, st>>>(x_dev, w.fidx, w.na, par, m.Jt, m.JS, w.Phi, w.PhiTc, w.At, w.ldA,
                                                             w.gchain, w.slot_tr));
    if (dense) {
        // with the SDF term this chain is the plain-fp32 cross-check of the dense-regime kernels: the sampled distances are
        // voxel-sized numbers, TF32 pose offsets would cost them 1e-5 .. 1e-4 relative (the dense-regime kernels re-evaluate
        // the vertices that matter in fp32 instead, mvs_sdf_dev.cuh)
        int rc = launch_vertex_fwd_dense(ctx, st, !sdf_on);
        if (rc) return rc;
    } else {
        dim3 g2((nv + kTileV - 1) / kTileV, ftiles);
        MVS_LAUNCH(ctx, KID_VERTEX_FWD, st,
                   vertex_fwd_kernel<<<g2, kVertThreads, kVertFwdSmem, st>>>(m.Qk, w.Phi, w.At, w.ldA, m.ell_j, m.ell_w, m.KW,
                                                                             vlist, nv, w.na, w.vposed, w.verts));
    }
    if (sdf_on) {
        int rc = launch_sdf_terms(ctx, x_dev, st);          // writes dense dv and pen_loss
        if (rc) return rc;
    }
    KeypointModel km{m.K, m.nsup, m.N, m.kp_ptr, m.kp_vidx, m.kp_spos, m.kp_w, m.kp_chain, m.sup, m.sup_ptr, m.sup_k, m.sup_w};
    CamSet cams = ctx->cams;
    if (geometry_only) cams.num_views = 0;           // joints / vertices only: no projection, no detections read
    MVS_LAUNCH(ctx, KID_KEYPOINT, st,
               keypoint_loss_kernel<<<B, kFrameThreads, 0, st>>>(x_dev, w.fidx, w.na, km, w.verts, nv, dense ? 1 : 0,
                                                                 w.gchain, cams, w.gt_uv, w.conf, w.joint_w, B, lp,
                                                                 w.data_loss, w.dtransl, w.dv, sdf_on ? m.nsup + m.N : m.nsup,
                                                                 w.dgchain, joints_dev, proj_dev));
    if (geometry_only) {
        if (verts_dev) {
            dim3 g6((m.N * 3 + 255) / 256, B);
            MVS_LAUNCH(ctx, KID_MISC, st, verts_out_kernel<<<g6, 256, 0, st>>>(w.verts, x_dev, w.fidx, w.na, m.N, verts_dev));
        }
        MVS_CUDA_OK(ctx, cudaGetLastError());
        return MVS_OK;
    }
    int nstrips = 1;
    if (have_grad) {
        // backward list: the keypoint support (compact), then -- with the SDF term -- every vertex once more for the
        // dense penetration gradient (tiles without upstream gradient are skipped inside the kernel)
        const int nvb = sdf_on ? m.nsup + m.N : m.nsup;
        const int* blist_n = sdf_on ? m.sup_then_all : m.sup;
        const int* blist_pos = sdf_on ? m.sup_then_all : (dense ? m.sup : nullptr);
        const int ntiles = (nvb + kTileV - 1) / kTileV;
        int want = (ctx->sm_count + ftiles - 1) / ftiles;
        if (want < 1) want = 1;
        if (want > w.nstrips_max) want = w.nstrips_max;
        int tps = (ntiles + want - 1) / want;
        nstrips = (ntiles + tps - 1) / tps;
        dim3 g4(nstrips, ftiles);
        MVS_LAUNCH(ctx, KID_VERTEX_BWD, st,
                   vertex_bwd_kernel<<<g4, kVertThreads, kVertBwdSmem, st>>>(m.Qk, w.At, w.ldA, m.ell_j, m.ell_w, m.KW, m.Wd,
                                                                             blist_n, blist_pos, nvb, nv, w.vposed, w.dv,
                                                                             w.na, tps, ntiles, w.part));
    }
    PriorModel pm{m.M, m.gmm_means, m.gmm_prec, m.gmm_lognllw};
    MVS_LAUNCH(ctx, KID_FRAME_BWD, st,
               frame_bwd_kernel<<<B, kFrameThreads, 0, st>>>(x_dev, w.fidx, w.na, par, m.Jt, m.JS, w.part, nstrips, w.ldA,
                                                             have_grad ? 1 : 0, w.data_loss, sdf_on ? w.pen_loss : nullptr, w.dtransl,
                                                             w.dgchain, pm, lp, w.anchor, w.anchor_w,
                                                             loss_dev ? loss_dev : w.loss_scratch, grad_dev));
    if (verts_dev) {
        dim3 g6((m.N * 3 + 255) / 256, B);
        MVS_LAUNCH(ctx, KID_MISC, st, verts_out_kernel<<<g6, 256, 0, st>>>(w.verts, x_dev, w.fidx, w.na, m.N, verts_dev));
    }
    MVS_CUDA_OK(ctx, cudaGetLastError());
    return MVS_OK;
}

int launch_frame_fwd(mvs_ctx* ctx, const float* x_dev, cudaStream_t st) {
    DevModel& m = ctx->m;
    Workspace& w = ctx->ws;
    MVS_LAUNCH(ctx, KID_FRAME_FWD, st,
               frame_fwd_kernel<<<w.na_bound > 0 ? w.na_bound : w.B, kFrameThreads, 0, st>>>(x_dev, w.fidx, w.na, ctx->parents, m.Jt,
                                                              m.JS, w.Phi, w.PhiTc, w.At, w.ldA, w.gchain, w.slot_tr));
    MVS_CUDA_OK(ctx, cudaGetLastError());
    return MVS_OK;
}

// need_vposed = false: the caller's consumers recompute v_posed where they need it (the dense rounds: sdf_fused / frame_step read
// ST . [beta; 1] + pose offsets for their few vertices), so the skinning kernel does not write the [B][N][3] array at all
int launch_vertex_fwd_dense(mvs_ctx* ctx, cudaStream_t st, bool allow_tc, bool need_vposed) {
    DevModel& m = ctx->m;
    Workspace& w = ctx->ws;
    if (allow_tc && tc_available(ctx)) return launch_vertex_fwd_tc(ctx, st, need_vposed);     // wgmma / TMA path (mvs_tc.cu)
    if (!ctx->attr_done) {
        MVS_CUDA_OK(ctx, cudaFuncSetAttribute(vertex_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kVertFwdSmem));
        MVS_CUDA_OK(ctx, cudaFuncSetAttribute(vertex_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kVertBwdSmem));
        ctx->attr_done = true;
    }
    dim3 g2((m.N + kTileV - 1) / kTileV, (w.B + kTileF - 1) / kTileF);
    MVS_LAUNCH(ctx, KID_VERTEX_FWD, st,
               vertex_fwd_kernel<<<g2, kVertThreads, kVertFwdSmem, st>>>(m.Qk, w.Phi, w.At, w.ldA, m.ell_j, m.ell_w, m.KW,
                                                                         nullptr, m.N, w.na, w.vposed, w.verts));
    MVS_CUDA_OK(ctx, cudaGetLastError());
    return MVS_OK;
}

}  // namespace mvs
