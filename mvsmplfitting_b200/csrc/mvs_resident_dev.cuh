// Device side of the frame-resident kernels (mvs_resident.cu): shared-memory layout of one frame, level-parallel kinematic
// chain, VPoser decoder, the closure, the pose forward of the next trial point, and the per-frame half of a dense round
// (frame_step_kernel).
// A translation unit may define PHASE_MARK(i) before including this file (clock instrumentation); default: nothing.
#pragma once
#include <cstddef>
#include "mvs_internal.cuh"
#include "mvs_lbfgs_core.cuh"
#include "mvs_tc_dev.cuh"
#ifndef PHASE_MARK
#define PHASE_MARK(i) do {} while (0)
#endif

namespace mvs {

constexpr int kResThreads = 256;
constexpr int kResMaxSup = 96;            // support vertices (SMPL: 86)
constexpr int kResMaxSupJ = 512;          // (support vertex, joint) pairs with a non-zero skinning weight (SMPL: <= 344)
constexpr int kResMaxVK = 272;            // views x keypoints (16 x 17)
constexpr int kResMaxM = 8;               // GMM components
constexpr int kResMaxKpE = 256;           // (keypoint, support vertex) entries staged in shared memory
constexpr int kFlagList = 64;             // penetration-flagged 256-vertex blocks listed in shared memory (16384 vertices)
// resident_closure splits the CTA from P4 to P10: warps 0-5 run the data term and its adjoint, warps 6-7 the part of the
// priors that only needs the pose (GMM mat-vec and log-likelihoods, |theta|^2).  Each group syncs on its own named barrier;
// warp 6 then joins the data warps for P8.
constexpr int kDataThreads = 192;
constexpr int kPriorThreads = kResThreads - kDataThreads;

__device__ __forceinline__ void bar_sync_n(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }
__device__ __forceinline__ void data_sync() { bar_sync_n(1, kDataThreads); }
__device__ __forceinline__ void prior_sync() { bar_sync_n(2, kPriorThreads); }
// P8 (dPhi, kFeatPad columns) runs on the data warps and warp 6
constexpr int kP8Threads = kDataThreads + 32;
static_assert(kFeatPad == kP8Threads, "one P8 column per thread");
__device__ __forceinline__ void p8_sync() { bar_sync_n(3, kP8Threads); }

__device__ __forceinline__ void cp_async4(float* dst, const float* src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"((unsigned)__cvta_generic_to_shared(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async8(float* dst, const float* src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"((unsigned)__cvta_generic_to_shared(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async16(float* dst, const float* src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 16;" ::"r"((unsigned)__cvta_generic_to_shared(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait_group() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

// sum_{q < n} v(q) in ascending q -- the order of `for (q) a += v(q)` -- with eight loads in flight instead of one
template <class F>
__device__ __forceinline__ float serial_sum8(int n, F v) {
    float a = 0.f;
    for (int q0 = 0; q0 < n; q0 += 8) {
        float r[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) r[u] = q0 + u < n ? v(q0 + u) : 0.f;
#pragma unroll
        for (int u = 0; u < 8; ++u)
            if (q0 + u < n) a += r[u];
    }
    return a;
}

struct ResidentModel {                    // device pointers + sizes, by value
    const float* Qk; const float* Jt; const float* JS;
    const int* ell_j; const float* ell_w; int KW;
    int K, nsup;
    const int* kp_ptr; const int* kp_spos; const float* kp_w; const int* kp_chain; int nkpe;
    const int* sup; const int* sup_ptr; const int* sup_k; const float* sup_w;
    const int* supj_ptr; const int* supj_i; const float* supj_w;      // per joint: (support index, weight)
    int M; const float* gmm_means; const float* gmm_prec; const float* gmm_lognllw;
    const float* anchor; const float* anchor_w;     // sequence mode (mvs_set_anchor)
    const float* j3d_xyz; const float* j3d_conf;    // 3-D joint targets [B][K][3], [B][K] (mvs_set_joints3d)
    const float *vp_w1, *vp_w2, *vp_w3, *vp_w1t, *vp_w2t, *vp_w3t, *vp_b1, *vp_b2, *vp_b3;      // VPoser decoder
    Parents par;
    ChainSched cs;
};

struct ResidentSmem {
    // pose
    float x[88], R[216], J[72], Gam[216], g[72], A[288], Phi[224];
    // support vertices
    float vp[kResMaxSup * 3], v[kResMaxSup * 3], dv[kResMaxSup * 3], dvp[kResMaxSup * 3];
    int rowbase[kResMaxSup * 3];          // Qk row of column (3 i + c)
    // keypoints / data term
    float q[kMaxKeypoints * 3], dq[kMaxKeypoints * 3], contrib[kResMaxVK * 3], lterm[kResMaxVK], vsum[kMaxViews];
    // adjoint
    float dA[288], dPhi[224], dR[216], dGam[216], dg[72], dJ[72], grad[88];
    // priors
    float gm_diff[kResMaxM * 69], gm_y[kResMaxM * 69], gm_ll[kResMaxM];
    float red[kResThreads];
    float sc[16];                          // [0] data loss, [1] |theta|^2, [2] total loss, [3] anchor, [4] 3-D joint loss
    // optimiser vectors (lbfgs_resident_kernel only)
    float lx[88], lg[88], ld[88], lprev_g[88], lx_init[88], lg_prev[88], lbg0[88], lbg1[88], lx_eval[88], lg_new[88];
    float ro[128], al[128];
    float gram[kGramFloats];               // s_i . y_j within 8-slot blocks of the history ring (blocked two-loop recursion)
    float tl_scratch[96];
    // level schedule of the kinematic tree (copy of ResidentModel::cs / par: shared-memory latency instead of
    // dependent constant-bank loads inside the level loops)
    int nlev, lev_ptr[kJoints + 1], lev_j[kJoints], ch_ptr[kJoints + 1], ch_j[kJoints], par[kJoints];
    // per joint: the support vertices it skins (copy of supj_*: the dA loop of P7 is a chain of dependent list reads)
    int sj_ptr[kJoints + 1], sj_i[kResMaxSupJ], sj_on;
    float sj_w[kResMaxSupJ];
    // keypoint regressor over the support vertices and its transpose (copies of kp_* / sup_*: P6 would otherwise walk
    // chains of dependent list reads from L2); the entry lists only when they fit (kp_on)
    int sup[kResMaxSup], kp_ptr[kMaxKeypoints + 1], kp_chain[kMaxKeypoints], sup_ptr[kResMaxSup + 1], kp_on;
    int kp_spos[kResMaxKpE], sup_k[kResMaxKpE];
    float kp_w[kResMaxKpE], sup_w[kResMaxKpE];
    // dense regime: frame scalars of the SDF term and its box-extreme vertex list (frame_step_kernel)
    int ext_n[8];
    float ext_d[24];
    float sdf_sc[4];                       // [0] cg / scale, [1] pen loss, [2] number of extreme entries
    int fl[kFlagList], nfl;                // 256-vertex blocks with a penetration adjoint partial (the first kFlagList), count
    LossParams lp;                         // this frame's CURRENT stage (multi-stage kernels)
    FrameScalars fs;
};

constexpr int kPoseCacheFloats = 216 + 72 + 216 + 72 + 288;      // R | J | Gam | g | A
static_assert(offsetof(ResidentSmem, A) - offsetof(ResidentSmem, R) == (216 + 72 + 216 + 72) * sizeof(float), "pose cache layout");
static_assert(offsetof(ResidentSmem, gram) % 16 == 0, "cp.async 16-byte staging of the block Gram");
static_assert(sizeof(ResidentSmem) + 2 * 100 * kParams * sizeof(float) <= 112 * 1024, "two frame CTAs per SM (227 KB)");

// Inputs of the dense regime (SDF term on): the skinning kernel already produced every vertex of the frame, and
// sdf_fused_kernel the unit-factor adjoint of the vertices inside the penetration cone (per 1024-vertex part).
struct DenseIn {
    const float* verts;       // [N][3] this frame's skinned vertices, pre-transl (NULL: sparse regime, recompute the support vertices)
    const float* poffT;       // [3N][ldA] pose offsets of the tensor-core contraction; this frame is column `slot`
    const float* ST;          // [N][33] shapedirs rows | template: v_posed = vposed_of(ST row, betas, pose offset)
    int ldA, slot;
    const int* extra_n;       // [n_extra] box-extreme vertices that carry the gradient through the box centre / scale
    const float* extra_d;     // [n_extra][3] d pen / d vertex
    int n_extra;
    float pen_loss;
    const float* Wd;          // [N][24] dense skinning weights (adjoint of the extra vertices)
    const float* part;        // [nblocks][512] this frame's unit-factor partial adjoints, or NULL (no penetration)
    const int* fl;            // nfl <= kFlagList: [nfl] blocks that wrote partials, ascending; else [nblocks] flag per block
    int nfl;                  // number of blocks that wrote partials
    float factor;             // cg / scale: d pen / d (sum of samples) over the box scale
    bool pose_ready;          // R, J, Gam, g, A of this trial point are already in shared memory (frame_step's pose cache)
};

// ------------------------------------------------------------------------------------------------
// Kinematic chain by depth levels (lbs.py:348-374).  Every ROLE (rotation part, translation part, ...) has its own
// warps so that no warp executes more than one branch body: a level costs one short dependent chain plus a barrier.
// All kResThreads threads must call; ends with a barrier.
__device__ __forceinline__ void chain_fwd_levels(ResidentSmem& S) {
    const int t = threadIdx.x;
    if (t < 9) S.Gam[t] = S.x[kOffScale] * S.R[t];                               // lbs.py:348
    else if (t >= 64 && t < 67) S.g[t - 64] = S.J[t - 64];
    __syncthreads();
    for (int L = 1; L < S.nlev; ++L) {
        const int beg = S.lev_ptr[L], cnt = S.lev_ptr[L + 1] - beg;
        if (t < 63) {                                        // threads 0..62: Gam_j = Gam_p R_j, 9 lanes per joint
            const int l = t % 9;
            for (int q = t / 9; q < cnt; q += 7) {
                const int j = S.lev_j[beg + q], p = S.par[j];
                const float* Gp = &S.Gam[9 * p];
                const float* Rj = &S.R[9 * j];
                const int r = l / 3, c = l % 3;
                S.Gam[9 * j + l] = Gp[3 * r] * Rj[c] + Gp[3 * r + 1] * Rj[3 + c] + Gp[3 * r + 2] * Rj[6 + c];
            }
        } else if (t >= 64 && t < 64 + 30) {                 // threads 64..93: g_j = Gam_p (J_j - J_p) + g_p, 3 lanes per joint
            const int u = t - 64, r = u % 3;
            for (int q = u / 3; q < cnt; q += 10) {
                const int j = S.lev_j[beg + q], p = S.par[j];
                const float* Gp = &S.Gam[9 * p];
                const float r0 = S.J[3 * j] - S.J[3 * p], r1 = S.J[3 * j + 1] - S.J[3 * p + 1], r2 = S.J[3 * j + 2] - S.J[3 * p + 2];
                S.g[3 * j + r] = (Gp[3 * r] * r0 + Gp[3 * r + 1] * r1 + Gp[3 * r + 2] * r2) + S.g[3 * p + r];
            }
        }
        __syncthreads();
    }
}

// Adjoint of the chain, deepest level first.  Per level L (parents p with children j at level L + 1, already final):
//   role A (threads 0..62)     dGam_p += sum_j dGam_j R_j^T + dg_j rel_j^T      9 lanes per parent
//   role B (threads 64..126)   dR_j = Gam_p^T dGam_j                             9 lanes per child
//   role C (threads 128..157)  drel_j = Gam_p^T dg_j;  dJ_j += drel_j, dJ_p -= sum_j drel_j     3 lanes per parent
//   role D (threads 160..189)  dg_p += sum_j dg_j                                3 lanes per parent
// Children are gathered in descending index order = the summation order of the plain j = 23..1 sweep.
// The kDataThreads data-term threads call; ends with their barrier.
__device__ __forceinline__ void chain_bwd_levels(ResidentSmem& S) {
    const int t = threadIdx.x;
    for (int L = S.nlev - 2; L >= 0; --L) {
        const int beg = S.lev_ptr[L], cnt = S.lev_ptr[L + 1] - beg;
        if (t < 63) {
            const int l = t % 9, r = l / 3, c = l % 3;
            for (int q = t / 9; q < cnt; q += 7) {
                const int p = S.lev_j[beg + q];
                const int c0 = S.ch_ptr[p], c1 = S.ch_ptr[p + 1];
                if (c0 == c1) continue;
                float acc = S.dGam[9 * p + l];
                for (int ci = c0; ci < c1; ++ci) {
                    const int j = S.ch_j[ci];
                    const float* dGj = &S.dGam[9 * j];
                    const float* Rj = &S.R[9 * j];
                    const float rel = S.J[3 * j + c] - S.J[3 * p + c];
                    acc += (dGj[3 * r] * Rj[3 * c] + dGj[3 * r + 1] * Rj[3 * c + 1] + dGj[3 * r + 2] * Rj[3 * c + 2]) + S.dg[3 * j + r] * rel;
                }
                S.dGam[9 * p + l] = acc;
            }
        } else if (t >= 64 && t < 64 + 63) {
            const int u = t - 64, e = u % 9, r = e / 3, c = e % 3;
            const int cbeg = S.lev_ptr[L + 1], ccnt = S.lev_ptr[L + 2] - cbeg;
            for (int q = u / 9; q < ccnt; q += 7) {
                const int j = S.lev_j[cbeg + q], p = S.par[j];
                const float* Gp = &S.Gam[9 * p];
                const float* dGj = &S.dGam[9 * j];
                S.dR[9 * j + e] = Gp[r] * dGj[c] + Gp[3 + r] * dGj[3 + c] + Gp[6 + r] * dGj[6 + c];
            }
        } else if (t >= 128 && t < 128 + 30) {
            const int u = t - 128, r = u % 3;
            for (int q = u / 3; q < cnt; q += 10) {
                const int p = S.lev_j[beg + q];
                const int c0 = S.ch_ptr[p], c1 = S.ch_ptr[p + 1];
                if (c0 == c1) continue;
                const float* Gp = &S.Gam[9 * p];
                float acc = S.dJ[3 * p + r];
                for (int ci = c0; ci < c1; ++ci) {
                    const int j = S.ch_j[ci];
                    const float* dgj = &S.dg[3 * j];
                    const float out = Gp[r] * dgj[0] + Gp[3 + r] * dgj[1] + Gp[6 + r] * dgj[2];
                    S.dJ[3 * j + r] += out;
                    acc -= out;
                }
                S.dJ[3 * p + r] = acc;
            }
        } else if (t >= 160 && t < 160 + 30) {
            const int u = t - 160, r = u % 3;
            for (int q = u / 3; q < cnt; q += 10) {
                const int p = S.lev_j[beg + q];
                const int c0 = S.ch_ptr[p], c1 = S.ch_ptr[p + 1];
                if (c0 == c1) continue;
                float acc = S.dg[3 * p + r];
                for (int ci = c0; ci < c1; ++ci) acc += S.dg[3 * S.ch_j[ci] + r];
                S.dg[3 * p + r] = acc;
            }
        }
        data_sync();
    }
}

// ------------------------------------------------------------------------------------------------
// VPoser decoder on the device (use_vposer = 2): body_pose = VPoser.decode(z, 'aa') (model/VPoser.py:218-232,
// fitting.py:121-123) and its adjoint.  z = S.x[kOffPose .. kOffPose + 32).  The scratch lives in dynamic shared memory
// behind the curvature history (only kernels launched for this mode reserve it).
constexpr int kVpH = 512, kVpZ = 32, kVpO = 138;
struct VposerSmem {
    float h1[kVpH], h2[kVpH], o6[kVpO + 6], th[72], dth[72], dh[kVpH], red[256];
};

__device__ __forceinline__ float lrelu(float v) { return v > 0.f ? v : 0.2f * v; }

// all threads; ends with a barrier.  Leaves W.th = decoded axis-angle pose (69) and zeroes W.dth.
static __device__ void vposer_decode(const ResidentSmem& S, const ResidentModel& m, VposerSmem& W) {
    const int t = threadIdx.x;
    const float* z = &S.x[kOffPose];
#pragma unroll
    for (int o = t; o < kVpH; o += kResThreads) {
        float a = m.vp_b1[o];
#pragma unroll 8
        for (int i = 0; i < kVpZ; ++i) a = fmaf(__ldg(m.vp_w1t + (size_t)i * kVpH + o), z[i], a);
        W.h1[o] = lrelu(a);
    }
    __syncthreads();
    {
        float a0 = m.vp_b2[t], a1 = m.vp_b2[t + kResThreads];
#pragma unroll 32
        for (int i = 0; i < kVpH; ++i) {
            const float hi = W.h1[i];
            a0 = fmaf(__ldg(m.vp_w2t + (size_t)i * kVpH + t), hi, a0);
            a1 = fmaf(__ldg(m.vp_w2t + (size_t)i * kVpH + t + kResThreads), hi, a1);
        }
        W.h2[t] = lrelu(a0); W.h2[t + kResThreads] = lrelu(a1);
    }
    __syncthreads();
    if (t < kVpO) {
        float a = m.vp_b3[t];
#pragma unroll 32
        for (int i = 0; i < kVpH; ++i) a = fmaf(__ldg(m.vp_w3t + (size_t)i * kVpO + t), W.h2[i], a);
        W.o6[t] = a;
    }
    if (t < 72) W.dth[t] = 0.f;
    __syncthreads();
    if (t < kJoints - 1) {
        Cont6dState<float> st;
        cont6d_to_aa_fwd(&W.o6[6 * t], &W.th[3 * t], st);
    }
    __syncthreads();
}

// all threads; adjoint of vposer_decode: W.dth (d loss / d decoded pose, 69) -> dz[32] in W.red[0..31].  Ends with a barrier.
static __device__ void vposer_decode_bwd(const ResidentModel& m, VposerSmem& W) {
    const int t = threadIdx.x;
    if (t < kJoints - 1) {
        Cont6dState<float> st;
        float aa[3], d6[6];
        cont6d_to_aa_fwd(&W.o6[6 * t], aa, st);               // recompute the intermediates (cheaper than keeping 23 states)
        cont6d_to_aa_bwd(st, &W.dth[3 * t], d6);
#pragma unroll
        for (int c = 0; c < 6; ++c) W.red[6 * t + c] = d6[c];                     // d o6 (138 <= 256)
    }
    __syncthreads();
    {   // d h2 = lrelu'(h2) .* (W3^T d o6)
        float a0 = 0.f, a1 = 0.f;
#pragma unroll 23
        for (int o = 0; o < kVpO; ++o) {
            const float d = W.red[o];
            a0 = fmaf(__ldg(m.vp_w3 + (size_t)o * kVpH + t), d, a0);
            a1 = fmaf(__ldg(m.vp_w3 + (size_t)o * kVpH + t + kResThreads), d, a1);
        }
        W.dh[t] = (W.h2[t] > 0.f ? 1.f : 0.2f) * a0;
        W.dh[t + kResThreads] = (W.h2[t + kResThreads] > 0.f ? 1.f : 0.2f) * a1;
    }
    __syncthreads();
    {   // d h1 = lrelu'(h1) .* (W2^T d h2)   (result overwrites h2, no longer needed)
        float a0 = 0.f, a1 = 0.f;
#pragma unroll 32
        for (int o = 0; o < kVpH; ++o) {
            const float d = W.dh[o];
            a0 = fmaf(__ldg(m.vp_w2 + (size_t)o * kVpH + t), d, a0);
            a1 = fmaf(__ldg(m.vp_w2 + (size_t)o * kVpH + t + kResThreads), d, a1);
        }
        W.h2[t] = (W.h1[t] > 0.f ? 1.f : 0.2f) * a0;
        W.h2[t + kResThreads] = (W.h1[t + kResThreads] > 0.f ? 1.f : 0.2f) * a1;
    }
    __syncthreads();
    {   // d z = W1^T d h1: 8 partial sums of 64 terms per latent entry
        const int k = t & 31, part = t >> 5;
        float a = 0.f;
#pragma unroll 8
        for (int o = part * 64; o < part * 64 + 64; ++o) a = fmaf(__ldg(m.vp_w1 + (size_t)o * kVpZ + k), W.h2[o], a);
        W.dh[t] = a;
    }
    __syncthreads();
    if (t < kVpZ) {
        float a = 0.f;
#pragma unroll
        for (int part = 0; part < 8; ++part) a += W.dh[32 * part + t];
        W.red[t] = a;
    }
    __syncthreads();
}

// sum over the flagged blocks, ascending, of entry e of their unit-factor partials.  A frame with more flagged blocks than
// the list holds walks the blocks' flags up to the last flagged one: the same terms added in the same order.
__device__ __forceinline__ float pen_partial_sum(const DenseIn& din, int e) {
    if (din.nfl <= kFlagList)
        return serial_sum8(din.nfl, [&](int q) { return din.part[(size_t)din.fl[q] * kPartFloats + e]; });
    float a = 0.f;
#pragma unroll 1
    for (int p = 0, q = 0; q < din.nfl; ++p)
        if (din.fl[p] != 0) { a += din.part[(size_t)p * kPartFloats + e]; ++q; }
    return a;
}

// P8 of the closure for feature column k: dPhi[k] = sum_col dvp[col] Qk[row(col)][k] in ascending col, then the
// penetration partials.  32 independent L2 loads in flight: the phase is as long as its round trips to L2 (258 rows: 8
// instead of 21).
__device__ __forceinline__ void dphi_col(ResidentSmem& S, const ResidentModel& m, const DenseIn& din, int ncol_all, int k) {
    float a = 0.f;
    int col = 0;
    for (; col + 32 <= ncol_all; col += 32) {
        float qv[32];
#pragma unroll
        for (int u = 0; u < 32; ++u) qv[u] = __ldg(m.Qk + (size_t)S.rowbase[col + u] * kFeatPad + k);
#pragma unroll
        for (int u = 0; u < 32; ++u) a = fmaf(S.dvp[col + u], qv[u], a);
    }
    for (; col + 8 <= ncol_all; col += 8) {
        float qv[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) qv[u] = __ldg(m.Qk + (size_t)S.rowbase[col + u] * kFeatPad + k);
#pragma unroll
        for (int u = 0; u < 8; ++u) a = fmaf(S.dvp[col + u], qv[u], a);
    }
    for (; col < ncol_all; ++col) a = fmaf(S.dvp[col], __ldg(m.Qk + (size_t)S.rowbase[col] * kFeatPad + k), a);
    if (din.part) {
        a = fmaf(pen_partial_sum(din, kSkinFloats + k), din.factor, a);
    }
    S.dPhi[k] = a;
}

// ------------------------------------------------------------------------------------------------
// One closure evaluation at S.x (already loaded).  Writes S.sc[2] = total loss and S.lg_new = gradient
// (frozen segments zeroed).  All kResThreads threads must call it.
static __device__ void resident_closure(ResidentSmem& S, const ResidentModel& m, const FrameRig& rig, const LossParams& lp,
                                 const float* __restrict__ gt_uv, const float* __restrict__ conf,
                                 const float* __restrict__ joint_w, int B, int b, bool have_grad,
                                 float* __restrict__ joints_out, float* __restrict__ proj_out, const DenseIn& din,
                                 VposerSmem* W = nullptr) {
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const int nsup = m.nsup, K = m.K, V = rig.num_views, ncol = 3 * nsup;          // V: the views of this frame's rig
    // use_vposer == 2: the body pose is decoded from the latent code in the pose slot (fitting.py:121-123)
    const bool vp2 = (lp.use_vposer == 2) && W != nullptr;
    if (vp2) vposer_decode(S, m, *W);
    const float* theta = vp2 ? W->th : &S.x[kOffPose];          // the 69 body-pose entries the model sees
    const bool kp_sm = S.kp_on != 0;
    const int* kp_spos = kp_sm ? S.kp_spos : m.kp_spos;
    const float* kp_w = kp_sm ? S.kp_w : m.kp_w;
    const int* sup_k = kp_sm ? S.sup_k : m.sup_k;
    const float* sup_w = kp_sm ? S.sup_w : m.sup_w;

    // ---- P1 Rodrigues, rest joints (skipped when the caller restored them: the previous frame_step computed the pose
    //      forward of exactly this trial point for the dense kernels and parked it in the per-frame pose cache)
    if (!din.pose_ready) {
        if (t < kJoints) rodrigues_fwd(t == 0 ? &S.x[kOffOrient] : &theta[3 * (t - 1)], &S.R[9 * t]);
        else if (t >= 32 && t < 32 + 72) {
            const int jc = t - 32;
            float a = m.Jt[jc];
#pragma unroll
            for (int l = 0; l < kBetas; ++l) a = fmaf(m.JS[jc * kBetas + l], S.x[kOffBetas + l], a);
            S.J[jc] = a;
        }
    }
    for (int i = t; i < kJoints * 9; i += kResThreads) { S.dGam[i] = 0.f; S.dR[i] = 0.f; }
    for (int i = t; i < kJoints * 3; i += kResThreads) { S.dg[i] = 0.f; S.dJ[i] = 0.f; }
    for (int i = t; i < kParams; i += kResThreads) S.grad[i] = 0.f;
    __syncthreads();
    PHASE_MARK(2);
    if (!din.pose_ready) {
        // ---- P2 kinematic chain, level-parallel
        chain_fwd_levels(S);
        PHASE_MARK(3);
        // ---- P3 skinning transforms and the feature row
        if (t < kJoints) make_skin_transform(&S.Gam[9 * t], &S.g[3 * t], &S.J[3 * t], &S.A[12 * t]);
        else if (t >= 32) {
            const int k = t - 32;                                                      // 224 threads, 224 entries
            float v;
            if (k < kPoseBasis) v = S.R[9 + k] - (((k % 9) % 4 == 0) ? 1.0f : 0.0f);
            else if (k < kPoseBasis + kBetas) v = S.x[kOffBetas + k - kPoseBasis];
            else v = (k == kFeat - 1) ? 1.0f : 0.0f;
            S.Phi[k] = v;
        }
        __syncthreads();
    }
    PHASE_MARK(4);
    if (t >= kDataThreads) {
        const int M = m.M;
        const bool gmm = !lp.use_vposer && lp.body_prior == MVS_PRIOR_GMM;
        // ---- P11a priors (fitting.py:327-350) that need only the pose: GMM components and |theta|^2, on warps 6-7 while
        //      warps 0-5 run P4-P10.  Same expressions and orders as one phase per barrier on all warps.
        const int pt = t - kDataThreads;
        if (gmm)
            for (int e = pt; e < M * 69; e += kPriorThreads) S.gm_diff[e] = theta[e % 69] - m.gmm_means[e];
        for (int i = pt; i < 69; i += kPriorThreads)
            S.red[i] = vp2 ? ((i < kVpZ) ? S.x[kOffPose + i] * S.x[kOffPose + i] : 0.f) : theta[i] * theta[i];  // |z|^2 (fitting.py:327-329)
        prior_sync();
        if (gmm) {
            for (int e = pt; e < M * 69; e += kPriorThreads) {
                const int mm = e / 69, i = e % 69;
                const float* P = m.gmm_prec + (size_t)mm * 69 * 69 + i;
                const float* df = &S.gm_diff[mm * 69];
                float y = 0.f;
#pragma unroll
                for (int j = 0; j < 69; ++j) y = fmaf(__ldg(P + j * 69), df[j], y);       // all 69 loads of the row in flight
                S.gm_y[e] = y;
            }
        }
        if (pt == 0) { float a = 0.f; for (int i = 0; i < 69; ++i) a += S.red[i]; S.sc[1] = a; }
        prior_sync();
        if (gmm) {
            for (int mm = warp - kDataThreads / 32; mm < M; mm += kPriorThreads / 32) {
                float p = 0.f;
                for (int i = lane; i < 69; i += 32) p = fmaf(S.gm_y[mm * 69 + i], S.gm_diff[mm * 69 + i], p);
                p = warp_sum(p);
                if (lane == 0) S.gm_ll[mm] = 0.5f * p - m.gmm_lognllw[mm];
            }
        }
        if (have_grad && warp == kDataThreads / 32) {    // P8 for the feature columns 192 .. 223, between the data warps' barriers
            p8_sync();
            dphi_col(S, m, din, ncol + 3 * din.n_extra, kDataThreads + lane);
            p8_sync();
        }
    } else {
        // ---- P4 v_posed for the support columns
        if (din.verts) {                  // dense regime: the vertex kernels already have them (v_posed: bit for bit skin_vertex's)
            for (int col = t; col < ncol; col += kDataThreads) {
                const int n = S.sup[col / 3], c = col % 3;
                S.vp[col] = vposed_of(din.ST + (size_t)n * 33 + 11 * c, &S.x[kOffBetas], din.poffT[(size_t)(3 * n + c) * din.ldA + din.slot]);
                S.v[col] = din.verts[3 * n + c];
            }
            // the box-extreme vertices of the penetration term ride along as support entries nsup .. nsup + n_extra - 1
            if (t < 3 * din.n_extra) {
                const int n = din.extra_n[t / 3], c = t % 3;
                S.vp[ncol + t] = vposed_of(din.ST + (size_t)n * 33 + 11 * c, &S.x[kOffBetas], din.poffT[(size_t)(3 * n + c) * din.ldA + din.slot]);
                S.dv[ncol + t] = din.extra_d[t];
                S.rowbase[ncol + t] = 3 * n + c;
            }
        } else {
            // warp per Qk row (896 B = 2 x LDG.128 per lane), FOUR rows in flight per warp: the 231 KB slice comes from L2
            // and the phase is pure latency, so the depth of the load queue is what sets its length
            const float4 ph0 = *reinterpret_cast<const float4*>(&S.Phi[4 * lane]);
            const float4 ph1 = lane < 24 ? *reinterpret_cast<const float4*>(&S.Phi[128 + 4 * lane]) : make_float4(0.f, 0.f, 0.f, 0.f);
            constexpr int kW = kDataThreads / 32;
            for (int col0 = warp; col0 < ncol; col0 += 4 * kW) {
                float4 a[4], bq[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const int col = col0 + u * kW;
                    const float* r = m.Qk + (size_t)S.rowbase[col < ncol ? col : col0] * kFeatPad;
                    a[u] = __ldg(reinterpret_cast<const float4*>(r + 4 * lane));
                    bq[u] = lane < 24 ? __ldg(reinterpret_cast<const float4*>(r + 128 + 4 * lane)) : make_float4(0.f, 0.f, 0.f, 0.f);
                }
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    float p = a[u].x * ph0.x;
                    p = fmaf(a[u].y, ph0.y, p); p = fmaf(a[u].z, ph0.z, p); p = fmaf(a[u].w, ph0.w, p);
                    p = fmaf(bq[u].x, ph1.x, p); p = fmaf(bq[u].y, ph1.y, p); p = fmaf(bq[u].z, ph1.z, p); p = fmaf(bq[u].w, ph1.w, p);
                    p = warp_sum(p);
                    const int col = col0 + u * kW;
                    if (lane == 0 && col < ncol) S.vp[col] = p;
                }
            }
        }
        data_sync();
        PHASE_MARK(5);
        // ---- P5 linear blend skinning of the support vertices
        if (!din.verts && t < nsup) {
            const int n = S.sup[t];
            float T[12];
#pragma unroll
            for (int c = 0; c < 12; ++c) T[c] = 0.f;
            for (int e = 0; e < m.KW; ++e) {
                const float w = m.ell_w[(size_t)n * m.KW + e];
                if (w != 0.f) {
                    const float* Aj = &S.A[12 * m.ell_j[(size_t)n * m.KW + e]];
#pragma unroll
                    for (int c = 0; c < 12; ++c) T[c] = fmaf(w, Aj[c], T[c]);
                }
            }
            const float p0 = S.vp[3 * t], p1 = S.vp[3 * t + 1], p2 = S.vp[3 * t + 2];
#pragma unroll
            for (int r = 0; r < 3; ++r) S.v[3 * t + r] = T[4 * r] * p0 + T[4 * r + 1] * p1 + T[4 * r + 2] * p2 + T[4 * r + 3];
        }
        data_sync();
        PHASE_MARK(6);
        // ---- P6 keypoints, projection, GMoF data term and its adjoint down to the support vertices
        if (t < K) {
            float a0 = 0.f, a1 = 0.f, a2 = 0.f;
            for (int e = S.kp_ptr[t]; e < S.kp_ptr[t + 1]; ++e) {
                const int pos = kp_spos[e];
                const float w = kp_w[e];
                a0 = fmaf(w, S.v[3 * pos], a0); a1 = fmaf(w, S.v[3 * pos + 1], a1); a2 = fmaf(w, S.v[3 * pos + 2], a2);
            }
            const int cj = S.kp_chain[t];
            if (cj >= 0) { a0 += S.g[3 * cj]; a1 += S.g[3 * cj + 1]; a2 += S.g[3 * cj + 2]; }
            S.q[3 * t] = a0 + S.x[kOffTransl]; S.q[3 * t + 1] = a1 + S.x[kOffTransl + 1]; S.q[3 * t + 2] = a2 + S.x[kOffTransl + 2];
            if (joints_out) {
                joints_out[((size_t)b * K + t) * 3] = S.q[3 * t]; joints_out[((size_t)b * K + t) * 3 + 1] = S.q[3 * t + 1];
                joints_out[((size_t)b * K + t) * 3 + 2] = S.q[3 * t + 2];
            }
        }
        data_sync();
        PHASE_MARK(7);
        {
            const float dw = lp.data_weight * rig.dw_scale;                         // the rig's data weight (x 1: exact)
            const float rho2 = lp.rho * lp.rho, dw2 = dw * dw;
            for (int idx = t; idx < V * K; idx += kDataThreads) {
                const int v = idx / K, k = idx % K;
                float xc[3], uv[2];
                const CamF cam = rig_camera(rig, v);
                const Dist* dp = rig.dist ? rig.dist + v : nullptr;          // this view's distortion (NULL: none)
                project_fwd(cam, &S.q[3 * k], xc, uv, dp);
                const size_t o = ((size_t)v * B + b) * K + k;
                if (proj_out) { proj_out[2 * o] = uv[0]; proj_out[2 * o + 1] = uv[1]; }
                float w = joint_w[k];
                if (lp.use_joints_conf) w *= conf[o];
                const float w2 = w * w;
                float d0, d1;
                const float g0 = gmof(gt_uv[2 * o] - uv[0], rho2, &d0);
                const float g1 = gmof(gt_uv[2 * o + 1] - uv[1], rho2, &d1);
                S.lterm[idx] = w2 * g0 + w2 * g1;
                const float duv[2] = {-(w2 * d0) * dw2, -(w2 * d1) * dw2};
                float dqv[3] = {0.f, 0.f, 0.f};
                project_bwd(cam, xc, duv, dqv, dp);
                S.contrib[3 * idx] = dqv[0]; S.contrib[3 * idx + 1] = dqv[1]; S.contrib[3 * idx + 2] = dqv[2];
            }
            data_sync();
            PHASE_MARK(8);
            if (t < 32) {
                float l3 = 0.f;
                if (t < K) {
                    float a0 = 0.f, a1 = 0.f, a2 = 0.f;
                    for (int v = 0; v < V; ++v) {
                        a0 += S.contrib[3 * (v * K + t)]; a1 += S.contrib[3 * (v * K + t) + 1]; a2 += S.contrib[3 * (v * K + t) + 2];
                    }
                    if (lp.j3d_on) {          // 3-D joint term (fitting.py:318-324): targets of frame b, no joint_weights
                        const float c3 = m.j3d_conf[(size_t)b * K + t], c2 = c3 * c3;
                        const float* g3 = m.j3d_xyz + ((size_t)b * K + t) * 3;
                        float d0, d1, d2;
                        const float e0 = gmof(g3[0] - S.q[3 * t], rho2, &d0);
                        const float e1 = gmof(g3[1] - S.q[3 * t + 1], rho2, &d1);
                        const float e2 = gmof(g3[2] - S.q[3 * t + 2], rho2, &d2);
                        l3 = c2 * e0 + c2 * e1 + c2 * e2;
                        a0 += -(c2 * d0) * dw2; a1 += -(c2 * d1) * dw2; a2 += -(c2 * d2) * dw2;
                    }
                    S.dq[3 * t] = a0; S.dq[3 * t + 1] = a1; S.dq[3 * t + 2] = a2;
                }
                if (lp.j3d_on) {
                    l3 = warp_sum(l3);
                    if (t == 0) S.sc[4] = l3 * dw2;
                }
            } else if (t >= 32 && t < 32 + V) {
                const int v = t - 32;
                float a = 0.f;
                for (int k = 0; k < K; ++k) a += S.lterm[v * K + k];
                S.vsum[v] = a * dw2;
            }
            data_sync();
            PHASE_MARK(9);
            if (t == 0) {
                float a = 0.f;
                for (int v = 0; v < V; ++v) a += S.vsum[v];
                S.sc[0] = a;
            }
            if (t >= 32 && t < 35) {
                float a = 0.f;
                for (int k = 0; k < K; ++k) a += S.dq[3 * k + t - 32];
                S.grad[kOffTransl + t - 32] = a;
            }
            if (t >= 64 && t < 64 + kJoints) {
                const int j = t - 64;
                float a0 = 0.f, a1 = 0.f, a2 = 0.f;
                for (int k = 0; k < K; ++k)
                    if (S.kp_chain[k] == j) { a0 += S.dq[3 * k]; a1 += S.dq[3 * k + 1]; a2 += S.dq[3 * k + 2]; }
                S.dg[3 * j] = a0; S.dg[3 * j + 1] = a1; S.dg[3 * j + 2] = a2;
            }
            if (t >= 96 && t < 96 + nsup) {
                const int i = t - 96;
                float a0 = 0.f, a1 = 0.f, a2 = 0.f;
                for (int e = S.sup_ptr[i]; e < S.sup_ptr[i + 1]; ++e) {
                    const int k = sup_k[e];
                    const float w = sup_w[e];
                    a0 = fmaf(w, S.dq[3 * k], a0); a1 = fmaf(w, S.dq[3 * k + 1], a1); a2 = fmaf(w, S.dq[3 * k + 2], a2);
                }
                S.dv[3 * i] = a0; S.dv[3 * i + 1] = a1; S.dv[3 * i + 2] = a2;
            }
        }
        data_sync();
        PHASE_MARK(10);
        if (have_grad) {
            // ---- P7 adjoint of skinning: dvp = T3x3^T dv ; dA_j = sum_i W[i,j] [dv (x) vp | dv]
            const int nx = din.n_extra, ncol_all = ncol + 3 * nx;
            if (t < nsup + nx) {
                const int n = t < nsup ? S.sup[t] : din.extra_n[t - nsup];
                float G[9];
#pragma unroll
                for (int c = 0; c < 9; ++c) G[c] = 0.f;
                for (int e = 0; e < m.KW; ++e) {
                    const float w = m.ell_w[(size_t)n * m.KW + e];
                    if (w != 0.f) {
                        const float* Aj = &S.A[12 * m.ell_j[(size_t)n * m.KW + e]];
#pragma unroll
                        for (int r = 0; r < 3; ++r)
#pragma unroll
                            for (int c = 0; c < 3; ++c) G[3 * r + c] = fmaf(w, Aj[4 * r + c], G[3 * r + c]);
                    }
                }
                const float d0 = S.dv[3 * t], d1 = S.dv[3 * t + 1], d2 = S.dv[3 * t + 2];
                S.dvp[3 * t] = G[0] * d0 + G[3] * d1 + G[6] * d2;
                S.dvp[3 * t + 1] = G[1] * d0 + G[4] * d1 + G[7] * d2;
                S.dvp[3 * t + 2] = G[2] * d0 + G[5] * d1 + G[8] * d2;
            }
            for (int e = t; e < kSkinFloats; e += kDataThreads) {
                const int j = e / 12, r = (e % 12) / 4, c = e % 4;
                float a = 0.f;
                if (S.sj_on) {
#pragma unroll 4
                    for (int q2 = S.sj_ptr[j]; q2 < S.sj_ptr[j + 1]; ++q2) {
                        const int i = S.sj_i[q2];
                        const float wd = S.sj_w[q2] * S.dv[3 * i + r];
                        a = (c < 3) ? fmaf(wd, S.vp[3 * i + c], a) : a + wd;
                    }
                } else {
#pragma unroll 4
                    for (int q2 = m.supj_ptr[j]; q2 < m.supj_ptr[j + 1]; ++q2) {
                        const int i = m.supj_i[q2];
                        const float wd = m.supj_w[q2] * S.dv[3 * i + r];
                        a = (c < 3) ? fmaf(wd, S.vp[3 * i + c], a) : a + wd;
                    }
                }
                for (int k = 0; k < nx; ++k) {                     // box-extreme vertices: generic (dense-W) joint ownership
                    const float w = __ldg(din.Wd + (size_t)din.extra_n[k] * kJoints + j);
                    if (w != 0.f) {
                        const float wd = w * S.dv[3 * (nsup + k) + r];
                        a = (c < 3) ? fmaf(wd, S.vp[3 * (nsup + k) + c], a) : a + wd;
                    }
                }
                if (din.part) {                                    // penetration gradient: unit-factor block partials
                    a = fmaf(pen_partial_sum(din, e), din.factor, a);
                }
                S.dA[e] = a;
            }
            p8_sync();                                         // dvp ready for P8 (warp 6 included)
            PHASE_MARK(11);
            // ---- P8 dPhi[k] = sum_col dvp[col] Qk[row(col)][k]   (thread per k, coalesced rows; warp 6 takes k >= 192)
            dphi_col(S, m, din, ncol_all, t);
            p8_sync();
            PHASE_MARK(12);
            // ---- P9 adjoint of the skinning transforms
            if (t < kJoints)
                skin_transform_bwd(&S.dA[12 * t], &S.Gam[9 * t], &S.J[3 * t], &S.dGam[9 * t], &S.dg[3 * t], &S.dJ[3 * t]);
            data_sync();
            PHASE_MARK(14);
            // reverse sweep over the tree, level-parallel
            chain_bwd_levels(S);
            if (warp == 0) {
                const float sc = S.x[kOffScale];
                if (lane < 9) S.dR[lane] = sc * S.dGam[lane];
                if (lane == 0) {
                    float ds = 0.f;
#pragma unroll
                    for (int i = 0; i < 9; ++i) ds = fmaf(S.dGam[i], S.R[i], ds);
                    S.grad[kOffScale] = ds;
                }
                if (lane < 3) S.dJ[lane] += S.dg[lane];
            }
            data_sync();
            PHASE_MARK(15);
            // ---- P10 pose-feature adjoint, Rodrigues adjoint, shape gradient
            for (int k = t; k < kPoseBasis; k += kDataThreads) S.dR[9 + k] += S.dPhi[k];
            data_sync();
            PHASE_MARK(16);
            if (t < kJoints) {
                float dr[3] = {0.f, 0.f, 0.f};
                rodrigues_bwd(t == 0 ? &S.x[kOffOrient] : &theta[3 * (t - 1)], &S.dR[9 * t], dr);
                float* go = (vp2 && t > 0) ? &W->dth[3 * (t - 1)] : &S.grad[kOffOrient + 3 * t];     // decoded pose: adjoint goes on
                go[0] = dr[0]; go[1] = dr[1]; go[2] = dr[2];
            } else if (t >= 32 && t < 32 + kBetas) {
                const int l = t - 32;
                float a = S.dPhi[kPoseBasis + l];
                for (int jc = 0; jc < kJoints * 3; ++jc) a = fmaf(m.JS[jc * kBetas + l], S.dJ[jc], a);
                S.grad[kOffBetas + l] = a;
            }
        }
    }
    __syncthreads();                      // the two groups join: P11b applies the priors after the data-term gradient
    PHASE_MARK(17);
    const float bpw = lp.body_pose_weight, bpw2 = bpw * bpw;
    const int M = m.M;
    float pprior = 0.f, l2extra = 0.f;
    if (vp2) pprior = S.sc[1] * bpw2;
    if (!lp.use_vposer) {
        float gs = bpw2;
        int best_m = -1;
        if (lp.body_prior == MVS_PRIOR_GMM) {
            float best = 3.0e38f;
            for (int mm = 0; mm < M; ++mm) if (S.gm_ll[mm] < best) { best = S.gm_ll[mm]; best_m = mm; }
            pprior = best * bpw2;
        } else if (lp.body_prior == MVS_PRIOR_L2) {
            pprior = S.sc[1] * bpw2;
        }
        if (pprior > 5e4f) { pprior = 0.f; gs = 0.f; }
        const float w4 = (bpw * 4.f) * (bpw * 4.f);
        l2extra = S.sc[1] * w4;
        if (have_grad && t < 69) {
            float gth = 2.f * theta[t] * w4;
            if (lp.body_prior == MVS_PRIOR_GMM && best_m >= 0) gth = fmaf(gs, S.gm_y[best_m * 69 + t], gth);
            else if (lp.body_prior == MVS_PRIOR_L2) gth = fmaf(gs, 2.f * theta[t], gth);
            S.grad[kOffPose + t] += gth;
        }
    }
    float shape_loss = 0.f;
    if (!lp.fix_shape) {
        const float sw2 = lp.shape_weight * lp.shape_weight;
        float a = 0.f;
        for (int l = 0; l < kBetas; ++l) a = fmaf(S.x[l], S.x[l], a);
        shape_loss = a * sw2;
        if (have_grad && t >= 96 && t < 96 + kBetas) S.grad[kOffBetas + t - 96] += 2.f * S.x[t - 96] * sw2;
    }
    float angle = 0.f;
    {
        const int idx[4] = {52, 55, 9, 12};
        const float sg[4] = {1.f, -1.f, -1.f, -1.f};
        float ev[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) { const float e = mvs_exp(theta[idx[i]] * sg[i]); ev[i] = e * e; angle += ev[i]; }
        angle *= lp.bending_prior_weight;
        float gs = lp.bending_prior_weight;
        if (angle > 1e4f && !lp.use_vposer) { angle = 0.f; gs = 0.f; }
        if (have_grad) {                  // by the thread that added the pose prior to the same entry above: no barrier between
            float* gth = vp2 ? W->dth : &S.grad[kOffPose];
#pragma unroll
            for (int i = 0; i < 4; ++i)
                if (t == idx[i]) gth[idx[i]] += 2.f * sg[i] * ev[i] * gs;
        }
    }
    __syncthreads();
    PHASE_MARK(21);
    if (vp2 && have_grad) {               // d loss / d decoded pose -> d loss / d z, plus the prior's 2 bpw^2 z
        vposer_decode_bwd(m, *W);
        if (t < 69) S.grad[kOffPose + t] = (t < kVpZ) ? fmaf(2.f * bpw2, S.x[kOffPose + t], W->red[t]) : 0.f;
        __syncthreads();
    }
    float anchor_loss = 0.f;
    if (lp.anchor_on) {                                   // sequence mode: sum_i w_i (x_i - a_i)^2
        float dif = 0.f, wt = 0.f;
        if (t < kParams) { dif = S.x[t] - m.anchor[(size_t)b * kParams + t]; wt = m.anchor_w[(size_t)b * kParams + t]; }
        S.red[t] = wt * dif * dif;
        if (have_grad && t < kParams) S.grad[t] += 2.f * wt * dif;
        __syncthreads();
        if (t == 0) { float a = 0.f; for (int i = 0; i < kParams; ++i) a += S.red[i]; S.sc[3] = a; }
        __syncthreads();
        anchor_loss = S.sc[3];
    }
    // ---- P12 total (same order as fitting.py:411-413) and the masked gradient
    if (t == 0) {
        float total = S.sc[0];
        if (lp.j3d_on) total += S.sc[4];
        total += (pprior + l2extra);
        total += shape_loss;
        total += angle;
        if (din.verts) total += din.pen_loss;
        total += anchor_loss;
        S.sc[2] = total;
    }
    if (have_grad) {
        for (int i = t; i < kParams; i += kResThreads) {
            const int seg = i < kOffOrient ? 0 : i < kOffPose ? 1 : i < kOffTransl ? 2 : i < kOffScale ? 3 : 4;
            S.lg_new[i] = ((lp.frozen_mask >> seg) & 1u) ? 0.f : S.grad[i];
        }
    }
    __syncthreads();
    PHASE_MARK(22);
}

__device__ __forceinline__ void resident_setup(ResidentSmem& S, const ResidentModel& m) {
    for (int col = threadIdx.x; col < 3 * m.nsup; col += kResThreads) S.rowbase[col] = 3 * m.sup[col / 3] + col % 3;
    const int t = threadIdx.x;
    if (t < kJoints) { S.lev_j[t] = m.cs.lev_j[t]; S.ch_j[t] = m.cs.ch_j[t]; S.par[t] = m.par.p[t]; }
    else if (t >= 32 && t < 32 + kJoints + 1) { S.lev_ptr[t - 32] = m.cs.lev_ptr[t - 32]; S.ch_ptr[t - 32] = m.cs.ch_ptr[t - 32]; }
    else if (t == 64) S.nlev = m.cs.nlev;
    const int nsj = m.supj_ptr[kJoints];
    if (t == 65) S.sj_on = nsj <= kResMaxSupJ ? 1 : 0;
    if (nsj <= kResMaxSupJ) {
        if (t >= 96 && t < 96 + kJoints + 1) S.sj_ptr[t - 96] = m.supj_ptr[t - 96];
        for (int q = t; q < nsj; q += kResThreads) { S.sj_i[q] = m.supj_i[q]; S.sj_w[q] = m.supj_w[q]; }
    }
    if (t < m.nsup) S.sup[t] = m.sup[t];
    if (t <= m.nsup) S.sup_ptr[t] = m.sup_ptr[t];
    if (t < m.K) S.kp_chain[t] = m.kp_chain[t];
    if (t <= m.K) S.kp_ptr[t] = m.kp_ptr[t];
    if (t == 66) S.kp_on = m.nkpe <= kResMaxKpE ? 1 : 0;
    if (m.nkpe <= kResMaxKpE)
        for (int q = t; q < m.nkpe; q += kResThreads) {
            S.kp_spos[q] = m.kp_spos[q]; S.kp_w[q] = m.kp_w[q]; S.sup_k[q] = m.sup_k[q]; S.sup_w[q] = m.sup_w[q];
        }
}

// Pose forward of the trial point in S.x for the dense kernels of the next round: feature row (fp32 and TF32), skinning
// transforms (frame fastest), translation -- all addressed by the slot -- and the per-frame pose cache.  With vp2 the
// body pose is decoded from the latent code first.  All threads; no trailing barrier.
__device__ __forceinline__ void next_pose_forward(ResidentSmem& S, const ResidentModel& m, VposerSmem* W, bool vp2, int slot, int b,
                                                  float* __restrict__ Phi, float* __restrict__ PhiTc, float* __restrict__ At,
                                                  int ldA, float* __restrict__ slot_tr, float* __restrict__ pose_cache,
                                                  int* __restrict__ pose_valid) {
    const int t = threadIdx.x;
    if (vp2) vposer_decode(S, m, *W);
    const float* theta = vp2 ? W->th : &S.x[kOffPose];
    if (t < kJoints) rodrigues_fwd(t == 0 ? &S.x[kOffOrient] : &theta[3 * (t - 1)], &S.R[9 * t]);
    else if (t >= 32 && t < 32 + 72) {
        const int jc = t - 32;
        float a = m.Jt[jc];
#pragma unroll
        for (int l = 0; l < kBetas; ++l) a = fmaf(m.JS[jc * kBetas + l], S.x[kOffBetas + l], a);
        S.J[jc] = a;
    }
    __syncthreads();
    PHASE_MARK(26);
    chain_fwd_levels(S);
    PHASE_MARK(27);
    if (t < kJoints) {
        float* A = &S.A[12 * t];
        make_skin_transform(&S.Gam[9 * t], &S.g[3 * t], &S.J[3 * t], A);
#pragma unroll
        for (int c = 0; c < 12; ++c) At[(size_t)(t * 12 + c) * ldA + slot] = A[c];
        if (t < 3) slot_tr[4 * slot + t] = S.x[kOffTransl + t];
    } else if (t >= 32) {
        const int k = t - 32;
        float v;
        if (k < kPoseBasis) v = S.R[9 + k] - (((k % 9) % 4 == 0) ? 1.0f : 0.0f);
        else if (k < kPoseBasis + kBetas) v = S.x[kOffBetas + k - kPoseBasis];
        else v = (k == kFeat - 1) ? 1.0f : 0.0f;
        Phi[(size_t)slot * kFeatPad + k] = v;
        if (PhiTc) {                 // A operand of the tensor-core contraction: v = hi + lo, both TF32 (tf32_split)
            float hi = 0.f, lo = 0.f;
            if (k < kPoseBasis) tf32_split(v, hi, lo);
            PhiTc[(size_t)slot * kFeatPad + k] = hi;
            PhiTc[((size_t)ldA + slot) * kFeatPad + k] = lo;
        }
    }
    __syncthreads();
    if (pose_cache) {   // park R | J | Gam | g | A for the next round's closure adjoint
        const float* src = &S.R[0];
        float* dst = pose_cache + (size_t)b * kPoseCacheFloats;
        for (int i = t; i < kPoseCacheFloats; i += kResThreads) dst[i] = src[i];
        if (t == 0) pose_valid[b] = 1;
    }
}

// Arguments of frame_step_kernel
struct FrameStepArgs {
    ResidentModel m; RigSet rigs; const LossParams* lp_tab; int nstages; LbfgsCfg cfg; LbfgsState L; float* params;
    const float* gt_uv; const float* conf; const float* joint_w; int B, N;
    const float* verts_ws; const float* poffT; const float* ST;
    const float* parts5; const float* part; const int* pflag; const FrameBox* box; const float* Wd;
    float* Phi; float* PhiTc; float* At; int ldA; float* slot_tr; float* pose_cache; int* pose_valid; int with_vposer;
};

// One round of the dense regime for one frame: consumes the dense vertices + the SDF gradient list of this
// frame's trial point, finishes the closure (keypoint term, adjoint, priors), advances the frame's L-BFGS state
// machine and -- if the frame needs another evaluation -- runs the pose forward of the NEXT trial point and
// writes its feature row / skinning transforms for the next dense vertex launch.
// One CTA per slot; dynamic shared memory: sizeof(ResidentSmem) + 2 H 86 floats (+ VposerSmem).
__global__ void __launch_bounds__(kResThreads, 2)
frame_step_kernel(FrameStepArgs a, const int* __restrict__ fidx, const int* __restrict__ na_ptr) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    ResidentSmem& S = *reinterpret_cast<ResidentSmem*>(smem_raw);
    // the model tables are constants of the run: staged while the previous kernel of the round drains
    resident_setup(S, a.m);
    pdl_wait();
    const int slot = blockIdx.x;
    if (slot >= *na_ptr) return;
    const int b = fidx[slot];
    const FrameRig rig = frame_rig(a.rigs, b);                  // the cameras of this frame (issued ahead of the closure)
    const ResidentModel& m = a.m; const LossParams* lp_tab = a.lp_tab;
    const LbfgsCfg& cfg = a.cfg; const LbfgsState& L = a.L; float* params = a.params;
    const float* __restrict__ gt_uv = a.gt_uv; const float* __restrict__ conf = a.conf; const float* __restrict__ joint_w = a.joint_w;
    const int B = a.B, N = a.N, ldA = a.ldA, with_vposer = a.with_vposer;
    const float* verts_ws = a.verts_ws; const float* parts5 = a.parts5; const float* part = a.part; const int* pflag = a.pflag;
    const FrameBox* box = a.box; const float* __restrict__ Wd = a.Wd;
    float* Phi = a.Phi; float* PhiTc = a.PhiTc; float* At = a.At; float* slot_tr = a.slot_tr; float* pose_cache = a.pose_cache;
    int* pose_valid = a.pose_valid;
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const int nparts = (N + 255) / 256;                         // sdf_fused_kernel emits per 256-vertex block
    float* x_eval = L.x_eval + (size_t)b * kParams;
    float* hy = reinterpret_cast<float*>(smem_raw + sizeof(ResidentSmem));
    float* hs = hy + (size_t)L.H * kParams;
    VposerSmem* W = with_vposer ? reinterpret_cast<VposerSmem*>(hs + (size_t)L.H * kParams) : nullptr;
    const int phase0 = L.sc[b].phase, stage0 = L.sc[b].stage, hl = L.sc[b].hist_len;
    // Everything that needs only the frame index is requested at once, ahead of the branch on the frame's phase
    // (cp.async group 0): the frame's scalars (for the optimiser step; not kept in registers through the closure); the trial point; the optimiser's eight 86-vectors (one read now, one write-back after the step:
    // every dot product / axpy of the state machine then runs out of shared memory); and the pose forward of this trial
    // point, computed by the previous round's frame_step for the dense kernels (loaded next to its validity flag instead of
    // behind it: an invalid cache is simply overwritten by P1-P3 of the closure).
    if (t < kParams) {
        const size_t o = (size_t)b * kParams + t, o2 = (size_t)b * 2 * kParams + t;
        cp_async4(&S.x[t], x_eval + t);
        cp_async4(&S.lx[t], params + o);
        cp_async4(&S.lg[t], L.g + o);
        cp_async4(&S.ld[t], L.d + o);
        cp_async4(&S.lprev_g[t], L.prev_g + o);
        cp_async4(&S.lx_init[t], L.x_init + o);
        cp_async4(&S.lg_prev[t], L.g_prev + o);
        cp_async4(&S.lbg0[t], L.bg + o2);
        cp_async4(&S.lbg1[t], L.bg + o2 + kParams);
    }
    if (t >= 128 && t < 128 + (int)(sizeof(FrameScalars) / 4))
        cp_async4(reinterpret_cast<float*>(&S.fs) + (t - 128), reinterpret_cast<const float*>(&L.sc[b]) + (t - 128));
    {
        const float* src = pose_cache + (size_t)b * kPoseCacheFloats;      // R | J | Gam | g | A are contiguous (864 floats)
        for (int i = t; i < kPoseCacheFloats / 4; i += kResThreads) cp_async16(&S.R[4 * i], src + 4 * i);
    }
    cp_async_commit();
    const bool pose_ready = pose_valid[b] != 0;
    if (phase0 == PH_DONE) { cp_async_wait_all(); return; }
    PHASE_MARK(0);
    if (t < (int)(sizeof(LossParams) / 4))          // the loss parameters of the stage THIS frame is in
        reinterpret_cast<int*>(&S.lp)[t] = reinterpret_cast<const int*>(&lp_tab[stage0])[t];
    // Stage this frame's curvature history (<= 2 x 100 x 86 floats) into shared memory while the closure runs (cp.async
    // group 1): the two-loop recursion is ~200 DEPENDENT dot products, at L2 latency it costs ~80 us, from shared memory ~5 us.
    {
        const float* gy = L.hist_y + (size_t)b * L.H * kParams;
        const float* gs = L.hist_s + (size_t)b * L.H * kParams;
        // ring buffer: with hl < H the live rows are [0, hl); when full all rows are live.  8-byte packets
        // (rows are 344 B: 8-byte aligned)
        const int total = hl * kParams / 2;
        for (int i = t; i < total; i += kResThreads) {
            cp_async8(hy + 2 * i, gy + 2 * i);
            cp_async8(hs + 2 * i, gs + 2 * i);
        }
        for (int i = t; i < hl; i += kResThreads) cp_async4(&S.ro[i], L.ro + (size_t)b * L.H + i);
        {   // block Gram of the live part of the ring
            const float* gg = L.gram + (size_t)b * kGramFloats;
            const int nfl4 = ((hl == L.H ? L.H : hl) + 7) / 8 * 16;      // float4 packets
            for (int i = t; i < nfl4; i += kResThreads) cp_async16(S.gram + 4 * i, gg + 4 * i);
        }
        cp_async_commit();
    }
    if (warp == 7) {
        // frame scalars of the penetration term (fitting.py:386-392): total of the sampled values -> loss, the
        // factor of the listed vertices' adjoint, and the <= 6 box-extreme vertices that carry the gradient through
        // the box centre (mean of min / max vertex) and scale (0.6 x the largest extent)
        float a = 0.f;
        if (lane < 5) a = serial_sum8(nparts, [&](int p) { return parts5[((size_t)slot * nparts + p) * 5 + lane]; });
        float tot[5];
#pragma unroll
        for (int q = 0; q < 5; ++q) tot[q] = __shfl_sync(0xffffffffu, a, q);
        if (lane == 0) {
            const FrameBox fb = box[slot];
            const float coll_w = lp_tab[stage0].coll_loss_weight;
            const float wsum = coll_w * tot[0];                 // coll_loss_weight * cur_loss.sum() / 1
            const float cg = 2.f * wsum * coll_w;               // d pen / d (sum of samples)
            const float inv_s = 1.f / fb.scale;
            int cnt = 0;
            if (cg != 0.f) {
                const float dscale = -cg * tot[4] * inv_s;      // local = (v - c) / s  ->  d local / d s = -local / s
                for (int c = 0; c < 3; ++c) {
                    const float dcentre = -cg * tot[1 + c] * inv_s;
                    float dl = 0.5f * dcentre, dh = 0.5f * dcentre;
                    if (c == fb.cmax) { dh += 0.6f * dscale; dl -= 0.6f * dscale; }
                    if (dl != 0.f) { S.ext_n[cnt] = fb.ilo[c]; S.ext_d[3 * cnt] = 0.f; S.ext_d[3 * cnt + 1] = 0.f; S.ext_d[3 * cnt + 2] = 0.f; S.ext_d[3 * cnt + c] = dl; ++cnt; }
                    if (dh != 0.f) { S.ext_n[cnt] = fb.ihi[c]; S.ext_d[3 * cnt] = 0.f; S.ext_d[3 * cnt + 1] = 0.f; S.ext_d[3 * cnt + 2] = 0.f; S.ext_d[3 * cnt + c] = dh; ++cnt; }
                }
            }
            S.sdf_sc[0] = cg * inv_s;
            S.sdf_sc[1] = wsum * wsum;                          // fitting.py:391-392
            S.sdf_sc[2] = (float)cnt;
        }
        // blocks whose vertices carry a sample gradient (ascending), so the adjoint phases loop over those only
        int nfl = 0;
        for (int p0 = 0; p0 < nparts; p0 += 32) {
            const int p = p0 + lane;
            const bool f = p < nparts && pflag[(size_t)slot * nparts + p] != 0;
            const unsigned mk = __ballot_sync(0xffffffffu, f);
            if (f) { const int pos = nfl + __popc(mk & ((1u << lane) - 1u)); if (pos < kFlagList) S.fl[pos] = p; }
            nfl += __popc(mk);
        }
        if (lane == 0) S.nfl = nfl;
    }
    cp_async_wait_group<1>();                          // group 0: the frame state the closure starts from
    __syncthreads();
    PHASE_MARK(1);
    DenseIn din;
    din.verts = verts_ws + (size_t)slot * N * 3;
    din.poffT = a.poffT; din.ST = a.ST; din.ldA = ldA; din.slot = slot;
    din.extra_n = S.ext_n;
    din.extra_d = S.ext_d;
    din.n_extra = (int)S.sdf_sc[2];
    din.pen_loss = S.sdf_sc[1];
    din.Wd = Wd;
    din.factor = S.sdf_sc[0];
    din.part = (din.factor != 0.f && S.nfl > 0) ? part + (size_t)slot * nparts * kPartFloats : nullptr;
    din.fl = S.nfl <= kFlagList ? S.fl : pflag + (size_t)slot * nparts;
    din.nfl = S.nfl;
    din.pose_ready = pose_ready;
    resident_closure(S, m, rig, S.lp, gt_uv, conf, joint_w, B, b, true, nullptr, nullptr, din, W);
    for (int i = t; i < kParams; i += kResThreads) L.g_eval[(size_t)b * kParams + i] = S.lg_new[i];
    cp_async_wait_all();                               // group 1: history, curvature scalars, block Gram
    __syncthreads();
    PHASE_MARK(23);
    if (cfg.step_mode == 2) {                          // closure only (mvs_closure in exec mode 3): no optimiser step
        if (t == 0) L.loss_eval[b] = S.sc[2];
        return;
    }
    if (warp == 0) {
        FrameScalars s = S.fs;
        LbfgsPtrs P{S.lx, S.lg, S.ld, S.lprev_g, S.lx_init, S.lg_prev, S.lbg0, S.lbg1, hy, hs, S.ro, S.al, S.lx_eval,
                    S.lg_new, L.H, S.gram, S.tl_scratch};
        lbfgs_advance_core(s, P, S.sc[2], cfg, lane, S.lp.use_vposer == 2 ? 32 : kOffTransl - kOffPose);
        __syncwarp();
        advance_stage_if_done(s, S.lx_eval, S.lx, lane);
        VLOOP(i) S.x[i] = S.lx_eval[i];                // the next trial point: input of next_pose_forward
        if (lane == 0) { L.sc[b] = s; S.fs = s; }
    }
    __syncthreads();
    PHASE_MARK(24);
    // global write-back of the optimiser state, on warps 4-7: the first two phases of next_pose_forward run on warps 0-3
    if (warp >= 4) {
        const int u = t - 128;
        for (int i = u; i < kParams; i += kResThreads - 128) {
            params[(size_t)b * kParams + i] = S.lx[i];
            L.g[(size_t)b * kParams + i] = S.lg[i];
            L.d[(size_t)b * kParams + i] = S.ld[i];
            L.prev_g[(size_t)b * kParams + i] = S.lprev_g[i];
            L.x_init[(size_t)b * kParams + i] = S.lx_init[i];
            L.g_prev[(size_t)b * kParams + i] = S.lg_prev[i];
            L.bg[(size_t)b * 2 * kParams + i] = S.lbg0[i];
            L.bg[(size_t)b * 2 * kParams + kParams + i] = S.lbg1[i];
            x_eval[i] = S.lx_eval[i];
        }
        const int wslot = S.fs.pushed_slot;
        if (wslot >= 0) {                               // write the new curvature pair through to global memory
            for (int i = u; i < kParams; i += kResThreads - 128) {
                L.hist_y[((size_t)b * L.H + wslot) * kParams + i] = hy[(size_t)wslot * kParams + i];
                L.hist_s[((size_t)b * L.H + wslot) * kParams + i] = hs[(size_t)wslot * kParams + i];
            }
            if (u == 0) L.ro[(size_t)b * L.H + wslot] = S.ro[wslot];
            if (u < 64) L.gram[(size_t)b * kGramFloats + (wslot >> 3) * 64 + u] = S.gram[(wslot >> 3) * 64 + u];
        }
    }
    if (S.fs.phase == PH_DONE) return;
    // pose forward of the next trial point -> Phi row and skinning transforms for the next vertex launch (the frame keeps
    // its slot until the next compaction).  vp2n: the stage the NEXT evaluation belongs to (S.lp unless the frame just
    // changed stage).
    {
        const int nst = S.fs.stage;
        const bool vp2n = W != nullptr && (nst == stage0 ? S.lp.use_vposer : lp_tab[nst].use_vposer) == 2;
        next_pose_forward(S, m, W, vp2n, slot, b, Phi, PhiTc, At, ldA, slot_tr, pose_cache, pose_valid);
    }
    PHASE_MARK(28);
}

}  // namespace mvs
