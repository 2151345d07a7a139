// Frame-resident execution of the sparse regime (no vertices requested, no SDF term):
// ONE CTA owns ONE frame and runs the whole closure -- and, in lbfgs_resident_kernel, the whole
// L-BFGS / strong-Wolfe optimisation of that frame -- out of shared memory, without returning to
// the host or to other kernels between evaluations.
//
// Why: the loss of the sparse regime depends on only 86 of the 6890 vertices (SURVEY H4), so one
// closure is ~0.1 MFLOP + two passes over a 231 KB L2-resident slice of Qk.  Spread over five
// kernels per evaluation and ~900 rounds per fit, the batched path is bound by launch + dependent
// load latency.  Frames are independent
// optimisation problems, so nothing forces them into lock-step rounds: here every frame advances
// at its own pace, the optimiser state (7 vectors, 100-pair history = 69 KB) lives in shared
// memory, and a 256-frame stage is ONE kernel launch.
//
// The arithmetic is the same set of building blocks (mvs_math.cuh) in the same data flow as the
// batched kernels of mvs_closure.cu; only reduction orders differ (warp-tree vs serial sums).
#include <cstddef>
#include "mvs_internal.cuh"
#ifdef MVS_PHASE_DBG
namespace mvs { __device__ long long g_phase_clk[64];   /* [0..31] stamps of CTA 0; [32..39] max over CTAs of coarse segment times; [40,41] two-loop */ }
// longest two-loop recursion seen (cycles) and the history length it ran with
#define MVS_TL_MARK(dt, hl)                                                                                         \
    do {                                                                                                            \
        if ((unsigned long long)(dt) > atomicMax(reinterpret_cast<unsigned long long*>(&mvs::g_phase_clk[40]),      \
                                                 (unsigned long long)(dt)))                                         \
            mvs::g_phase_clk[41] = (hl);                                                                            \
    } while (0)
#endif
#include "mvs_lbfgs_core.cuh"

namespace mvs {

// -DMVS_PHASE_DBG (scripts/phase_times.py builds libmvsmpl_dbg.so with it): thread 0 of CTA 0 stamps clock64() after
// every barrier of frame_step_kernel, so the serial phases of one frame's round can be timed without a profiler.
#ifdef MVS_PHASE_DBG
__device__ __forceinline__ void phase_mark(int i) {
    if (threadIdx.x != 0) return;
    const long long c = clock64();
    if (blockIdx.x == 0) g_phase_clk[i] = c;
    // coarse segments of every CTA: start -> closure done (22) -> history ready (23) -> advanced (24) -> next pose (28)
    __shared__ long long seg_t0, seg_prev;
    if (i == 0) { seg_t0 = c; seg_prev = c; }
    const int k = (i == 22) ? 0 : (i == 23) ? 1 : (i == 24) ? 2 : (i == 28) ? 3 : -1;
    if (k >= 0) {
        atomicMax(reinterpret_cast<unsigned long long*>(&g_phase_clk[32 + k]), (unsigned long long)(c - seg_prev));
        seg_prev = c;
        if (i == 24 || i == 28) atomicMax(reinterpret_cast<unsigned long long*>(&g_phase_clk[36 + (i == 28)]), (unsigned long long)(c - seg_t0));
    }
}
#define PHASE_MARK(i) phase_mark(i)
#else
#define PHASE_MARK(i) do {} while (0)
#endif
}  // namespace mvs

#include "mvs_resident_dev.cuh"

namespace mvs {

// ------------------------------------------------------------------------------------------------ single closure
__global__ void __launch_bounds__(kResThreads, 2)
closure_resident_kernel(ResidentModel m, RigSet rigs, LossParams lp, const float* __restrict__ x,
                        const int* __restrict__ fidx, const int* __restrict__ na_ptr, const float* __restrict__ gt_uv,
                        const float* __restrict__ conf, const float* __restrict__ joint_w, int B, int have_grad,
                        float* __restrict__ loss_out, float* __restrict__ grad_out, float* __restrict__ joints_out,
                        float* __restrict__ proj_out) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    ResidentSmem& S = *reinterpret_cast<ResidentSmem*>(smem_raw);
    const int slot = blockIdx.x;
    if (slot >= *na_ptr) return;
    const int b = fidx[slot];
    const FrameRig rig = frame_rig(rigs, b);
    resident_setup(S, m);
    for (int i = threadIdx.x; i < kParams; i += kResThreads) S.x[i] = x[(size_t)b * kParams + i];
    __syncthreads();
    VposerSmem* W = lp.use_vposer == 2 ? reinterpret_cast<VposerSmem*>(smem_raw + sizeof(ResidentSmem)) : nullptr;
    resident_closure(S, m, rig, lp, gt_uv, conf, joint_w, B, b, have_grad != 0, joints_out, proj_out, DenseIn{}, W);
    if (threadIdx.x == 0) loss_out[b] = S.sc[2];
    if (have_grad)
        for (int i = threadIdx.x; i < kParams; i += kResThreads) grad_out[(size_t)b * kParams + i] = S.lg_new[i];
}

// The shape step of mvs_fit_shared_shape: ONE CTA per frame of chunk c (its sequence's problem in slot j).  The frame's row with
// its sequence's shared entries (betas, and scale with a.share_scale) taken from the slot's x_eval, evaluated by resident_closure
// under the stage lp; its part row: the loss, the betas' gradient, then scale's.
__device__ __forceinline__ bool shape_shared(int i, int share_scale) { return i < kOffOrient || (share_scale && i == kOffScale); }

__global__ void __launch_bounds__(kResThreads, 2)
shape_closure_kernel(ResidentModel m, RigSet rigs, LossParams lp, LbfgsState L, ShapeArgs a, ProblemChunk c) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    ResidentSmem& S = *reinterpret_cast<ResidentSmem*>(smem_raw);
    const int f = c.i0 + blockIdx.x;
    const int j = c.item_of[f] - c.base;
    if (L.sc[j].phase == PH_DONE) return;                               // the sequence's problem has finished
    const FrameRig rig = frame_rig(rigs, f);
    resident_setup(S, m);
    for (int i = threadIdx.x; i < kParams; i += kResThreads)
        S.x[i] = shape_shared(i, a.share_scale) ? L.x_eval[(size_t)j * kParams + i] : a.params[(size_t)f * kParams + i];
    __syncthreads();
    VposerSmem* W = lp.use_vposer == 2 ? reinterpret_cast<VposerSmem*>(smem_raw + sizeof(ResidentSmem)) : nullptr;
    resident_closure(S, m, rig, lp, a.in.gt_uv, a.in.conf, a.in.joint_w, a.in.n, f, true, nullptr, nullptr, DenseIn{}, W);
    float* row = c.part + (size_t)f * kPartCols;
    if (threadIdx.x == 0) row[0] = S.sc[2];
    if (threadIdx.x <= kOffOrient) row[1 + threadIdx.x] = S.lg_new[threadIdx.x < kOffOrient ? threadIdx.x : kOffScale];
}

// The held keypoints of mvs_refine_cameras: ONE CTA per frame of `frames`, resident_closure's joints output (the keypoints the
// 2-D term projects, with translation; VPoser decoded under use_vposer = 2) of the frame's row, into q [F][K][3]
__global__ void __launch_bounds__(kResThreads, 2)
camera_joints_kernel(ResidentModel m, RigSet rigs, LossParams lp, FrameInputs in, const float* __restrict__ params,
                     const int* __restrict__ frames, float* __restrict__ q) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    ResidentSmem& S = *reinterpret_cast<ResidentSmem*>(smem_raw);
    const int f = frames[blockIdx.x];
    const FrameRig rig = frame_rig(rigs, f);
    resident_setup(S, m);
    for (int i = threadIdx.x; i < kParams; i += kResThreads) S.x[i] = params[(size_t)f * kParams + i];
    __syncthreads();
    VposerSmem* W = lp.use_vposer == 2 ? reinterpret_cast<VposerSmem*>(smem_raw + sizeof(ResidentSmem)) : nullptr;
    resident_closure(S, m, rig, lp, in.gt_uv, in.conf, in.joint_w, in.n, f, false, q, nullptr, DenseIn{}, W);
}

// VPoser.decode(z, 'aa') alone (result export: code/utils/utils.py:741-743 decodes the fitted latent code before saving)
__global__ void __launch_bounds__(kResThreads, 2)
vposer_decode_kernel(ResidentModel m, const float* __restrict__ x, int B, float* __restrict__ body_pose) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    ResidentSmem& S = *reinterpret_cast<ResidentSmem*>(smem_raw);
    VposerSmem& W = *reinterpret_cast<VposerSmem*>(smem_raw + sizeof(ResidentSmem));
    const int b = blockIdx.x;
    if (b >= B) return;
    for (int i = threadIdx.x; i < kParams; i += kResThreads) S.x[i] = x[(size_t)b * kParams + i];
    __syncthreads();
    vposer_decode(S, m, W);
    if (threadIdx.x < 69) body_pose[(size_t)b * 69 + threadIdx.x] = W.th[threadIdx.x];
}

// ------------------------------------------------------------------------------------------------ whole stage
__global__ void __launch_bounds__(kResThreads, 2)
lbfgs_resident_kernel(ResidentModel m, RigSet rigs, const LossParams* __restrict__ lp_tab, int nstages, LbfgsCfg cfg,
                      float* __restrict__ params, const float* __restrict__ gt_uv, const float* __restrict__ conf,
                      const float* __restrict__ joint_w, int B, int H, FrameScalars* __restrict__ sc_out,
                      float* __restrict__ last_grad_out, int with_vposer, const int2* __restrict__ stage_rng) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    ResidentSmem& S = *reinterpret_cast<ResidentSmem*>(smem_raw);
    float* hy = reinterpret_cast<float*>(smem_raw + sizeof(ResidentSmem));
    float* hs = hy + (size_t)H * kParams;
    VposerSmem* W = with_vposer ? reinterpret_cast<VposerSmem*>(hs + (size_t)H * kParams) : nullptr;
    const int b = blockIdx.x, t = threadIdx.x, lane = t & 31, warp = t >> 5;
    if (b >= B) return;
    // this frame's slice of the stage table (all of it unless the run mixes cold and warm-started frames, mvs_fit_seq)
    const int st_begin = stage_rng ? stage_rng[b].x : 0, st_end = stage_rng ? stage_rng[b].y : nstages;
    if (st_begin >= st_end) {                                            // nothing to do in this run: parameters stay
        if (t == 0) sc_out[b] = fresh_frame_scalars(make_int2(st_begin, st_end));
        return;
    }
    const FrameRig rig = frame_rig(rigs, b);
    resident_setup(S, m);
    for (int i = t; i < kParams; i += kResThreads) { const float v = params[(size_t)b * kParams + i]; S.lx[i] = v; S.lx_eval[i] = v; }
    if (t == 0) S.fs = fresh_frame_scalars(make_int2(st_begin, st_end));
    if (t < (int)(sizeof(LossParams) / 4)) reinterpret_cast<int*>(&S.lp)[t] = reinterpret_cast<const int*>(&lp_tab[st_begin])[t];
    __syncthreads();
    LbfgsPtrs P{S.lx, S.lg, S.ld, S.lprev_g, S.lx_init, S.lg_prev, S.lbg0, S.lbg1, hy, hs, S.ro, S.al, S.lx_eval, S.lg_new, H,
                S.gram, S.tl_scratch};
    const long long eval_cap = stage_eval_cap(cfg);
    long long stage_ev0 = 0;
    int cur_stage = st_begin;
    while (true) {
        PHASE_MARK(0);
        for (int i = t; i < kParams; i += kResThreads) S.x[i] = S.lx_eval[i];
        __syncthreads();
        PHASE_MARK(1);
        resident_closure(S, m, rig, S.lp, gt_uv, conf, joint_w, B, b, true, nullptr, nullptr, DenseIn{}, W);
        PHASE_MARK(23);
        if (warp == 0) {
            FrameScalars s = S.fs;
            lbfgs_advance_core(s, P, S.sc[2], cfg, lane, S.lp.use_vposer == 2 ? 32 : kOffTransl - kOffPose);
            if (s.evals - stage_ev0 >= eval_cap && s.phase != PH_DONE) { s.phase = PH_DONE; s.nan_flag = 1; }
            advance_stage_if_done(s, S.lx_eval, S.lx, lane);
            if (lane == 0) S.fs = s;
        }
        __syncthreads();
        PHASE_MARK(24);
        if (S.fs.phase == PH_DONE) break;
        if (S.fs.stage != cur_stage) {                                   // a stage just started: its loss parameters
            cur_stage = S.fs.stage;
            stage_ev0 = S.fs.evals;
            if (t < (int)(sizeof(LossParams) / 4))
                reinterpret_cast<int*>(&S.lp)[t] = reinterpret_cast<const int*>(&lp_tab[cur_stage])[t];
            __syncthreads();
        }
    }
    for (int i = t; i < kParams; i += kResThreads) {
        params[(size_t)b * kParams + i] = S.lx[i];
        if (last_grad_out) last_grad_out[(size_t)b * kParams + i] = S.lg_new[i];
    }
    if (t == 0) sc_out[b] = S.fs;
}

// The chaining run of mvs_fit_seq_stream: ONE CTA owns ONE sequence (q.act[blockIdx.x]) and runs lbfgs_resident_kernel's
// per-frame optimisation for each of its frames in turn, from its pending frame q.cur[seq] (cold) on.  After a frame it
// writes the frame's parameters, final loss and counts, then starts the successor with a fresh optimiser: warm from the
// fitted row in shared memory, cold from the successor's own row -- or, with q.park, leaves a cold successor to the next
// pass.  B = F: the inputs' row stride.  A kernel of its own so that the sequence walk stays out of lbfgs_resident_kernel's
// registers.  Its stage loop repeats lbfgs_resident_kernel's: shared as one inlined function, it cost that kernel 20 B of spills.
__global__ void __launch_bounds__(kResThreads, 2)
lbfgs_resident_seq_kernel(ResidentModel m, RigSet rigs, const LossParams* __restrict__ lp_tab, LbfgsCfg cfg,
                          float* __restrict__ params, const float* __restrict__ gt_uv, const float* __restrict__ conf,
                          const float* __restrict__ joint_w, int B, int H, int with_vposer, SeqChain q) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    ResidentSmem& S = *reinterpret_cast<ResidentSmem*>(smem_raw);
    float* hy = reinterpret_cast<float*>(smem_raw + sizeof(ResidentSmem));
    float* hs = hy + (size_t)H * kParams;
    VposerSmem* W = with_vposer ? reinterpret_cast<VposerSmem*>(hs + (size_t)H * kParams) : nullptr;
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    if ((int)blockIdx.x >= q.n_act) return;
    const int seq = q.act[blockIdx.x], seq_end = q.off[seq + 1];
    int b = q.cur[seq];
    int2 rng = q.cold;
    long long seq_evals = 0;                                             // evaluations of this CTA's frames so far
    resident_setup(S, m);
    for (int i = t; i < kParams; i += kResThreads) { const float v = params[(size_t)b * kParams + i]; S.lx[i] = v; S.lx_eval[i] = v; }
    LbfgsPtrs P{S.lx, S.lg, S.ld, S.lprev_g, S.lx_init, S.lg_prev, S.lbg0, S.lbg1, hy, hs, S.ro, S.al, S.lx_eval, S.lg_new, H,
                S.gram, S.tl_scratch};
    const long long eval_cap = stage_eval_cap(cfg);
    while (true) {                                                       // frames of the sequence
        const FrameRig rig = frame_rig(rigs, b);                         // a sequence's frames may change rig
        if (t == 0) S.fs = fresh_frame_scalars(rng);
        if (t < (int)(sizeof(LossParams) / 4)) reinterpret_cast<int*>(&S.lp)[t] = reinterpret_cast<const int*>(&lp_tab[rng.x])[t];
        __syncthreads();
        long long stage_ev0 = 0;
        int cur_stage = rng.x;
        while (true) {                                                   // as lbfgs_resident_kernel
            for (int i = t; i < kParams; i += kResThreads) S.x[i] = S.lx_eval[i];
            __syncthreads();
            resident_closure(S, m, rig, S.lp, gt_uv, conf, joint_w, B, b, true, nullptr, nullptr, DenseIn{}, W);
            if (warp == 0) {
                FrameScalars s = S.fs;
                lbfgs_advance_core(s, P, S.sc[2], cfg, lane, S.lp.use_vposer == 2 ? 32 : kOffTransl - kOffPose);
                if (s.evals - stage_ev0 >= eval_cap && s.phase != PH_DONE) { s.phase = PH_DONE; s.nan_flag = 1; }
                advance_stage_if_done(s, S.lx_eval, S.lx, lane);
                if (lane == 0) S.fs = s;
            }
            __syncthreads();
            if (S.fs.phase == PH_DONE) break;
            if (S.fs.stage != cur_stage) {
                cur_stage = S.fs.stage;
                stage_ev0 = S.fs.evals;
                if (t < (int)(sizeof(LossParams) / 4))
                    reinterpret_cast<int*>(&S.lp)[t] = reinterpret_cast<const int*>(&lp_tab[cur_stage])[t];
                __syncthreads();
            }
        }
        for (int i = t; i < kParams; i += kResThreads) params[(size_t)b * kParams + i] = S.lx[i];
        const FrameScalars& s = S.fs;
        seq_evals += s.evals;
        if (t == 0) {                                                    // the frame's totals, as lbfgs_finalize_kernel counts them
            if (q.final_loss) q.final_loss[b] = s.final_loss;
            add_frame_totals(q.totals, s);
        }
        const int nx = b + 1;
        const bool more = nx < seq_end, warm = more && s.final_loss <= q.reinit_loss;   // NaN is not <= reinit_loss
        if (!more || (!warm && q.park)) {                                // sequence done, or parked for the earlier runs
            if (t == 0) {
                q.cur[seq] = more ? nx : -1;
                atomicMax((unsigned long long*)&q.totals[3], (unsigned long long)seq_evals);
            }
            break;
        }
        for (int i = t; i < kParams; i += kResThreads) {                 // the successor's start point
            const bool own = !warm || (q.keep_pose && i >= kOffPose && i < kOffTransl);
            const float v = own ? params[(size_t)nx * kParams + i] : S.lx[i];
            S.lx[i] = v; S.lx_eval[i] = v;
        }
        rng = warm ? q.warm : q.cold;
        b = nx;
        __syncthreads();                                                 // every thread has read S.fs before it is reset
    }
}

// The same for every active slot at the start of a run and after a compaction (slots changed): the VPoser-capable
// counterpart of frame_fwd_kernel (mvs_closure.cu), which only knows axis-angle poses.
__global__ void __launch_bounds__(kResThreads, 2)
frame_fwd_resident_kernel(ResidentModel m, const LossParams* __restrict__ lp_tab, const FrameScalars* __restrict__ sc,
                          const float* __restrict__ x, const int* __restrict__ fidx, const int* __restrict__ na_ptr,
                          float* __restrict__ Phi, float* __restrict__ PhiTc, float* __restrict__ At, int ldA,
                          float* __restrict__ slot_tr) {
    pdl_wait();
    extern __shared__ __align__(16) unsigned char smem_raw[];
    ResidentSmem& S = *reinterpret_cast<ResidentSmem*>(smem_raw);
    VposerSmem* W = reinterpret_cast<VposerSmem*>(smem_raw + sizeof(ResidentSmem));
    const int slot = blockIdx.x;
    if (slot >= *na_ptr) return;
    const int b = fidx[slot], t = threadIdx.x;
    resident_setup(S, m);
    for (int i = t; i < kParams; i += kResThreads) S.x[i] = x[(size_t)b * kParams + i];
    const bool vp2 = lp_tab[sc[b].stage].use_vposer == 2;
    __syncthreads();
    next_pose_forward(S, m, W, vp2, slot, b, Phi, PhiTc, At, ldA, slot_tr, nullptr, nullptr);
}

// ------------------------------------------------------------------------------------------------ host side
bool resident_supported(const mvs_ctx* ctx) {
    const DevModel& m = ctx->m;
    return m.supj_ptr != nullptr && m.nsup + 6 <= kResMaxSup && m.K <= kMaxKeypoints &&
           ctx->vmax * m.K <= kResMaxVK && m.M <= kResMaxM;
}

// dynamic shared memory of lbfgs_resident_kernel and frame_step_kernel: one frame, history H (+ the VPoser decoder)
static size_t frame_smem(int H, bool with_vposer) {
    return sizeof(ResidentSmem) + (size_t)2 * H * kParams * sizeof(float) + (with_vposer ? sizeof(VposerSmem) : 0);
}

// lbfgs_resident_kernel runs histories up to 100 (stage_regime), frame_step_kernel up to 128 (the history_size limit)
int resident_set_attributes(mvs_ctx* ctx) {
    const int one_frame = (int)(sizeof(ResidentSmem) + sizeof(VposerSmem));
    MVS_CUDA_OK(ctx, cudaFuncSetAttribute(closure_resident_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, one_frame));
    MVS_CUDA_OK(ctx, cudaFuncSetAttribute(shape_closure_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, one_frame));
    MVS_CUDA_OK(ctx, cudaFuncSetAttribute(camera_joints_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, one_frame));
    MVS_CUDA_OK(ctx, cudaFuncSetAttribute(vposer_decode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, one_frame));
    MVS_CUDA_OK(ctx, cudaFuncSetAttribute(frame_fwd_resident_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, one_frame));
    MVS_CUDA_OK(ctx, cudaFuncSetAttribute(lbfgs_resident_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          (int)frame_smem(100, true)));
    MVS_CUDA_OK(ctx, cudaFuncSetAttribute(lbfgs_resident_seq_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          (int)frame_smem(100, true)));
    MVS_CUDA_OK(ctx, cudaFuncSetAttribute(frame_step_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          (int)frame_smem(128, true)));
    return MVS_OK;
}

static ResidentModel make_resident_model(const mvs_ctx* ctx) {
    const DevModel& m = ctx->m;
    ResidentModel r;
    r.Qk = m.Qk; r.Jt = m.Jt; r.JS = m.JS; r.ell_j = m.ell_j; r.ell_w = m.ell_w; r.KW = m.KW;
    r.K = m.K; r.nsup = m.nsup; r.kp_ptr = m.kp_ptr; r.kp_spos = m.kp_spos; r.kp_w = m.kp_w; r.kp_chain = m.kp_chain;
    r.nkpe = m.n_kp_entries;
    r.sup = m.sup; r.sup_ptr = m.sup_ptr; r.sup_k = m.sup_k; r.sup_w = m.sup_w;
    r.supj_ptr = m.supj_ptr; r.supj_i = m.supj_i; r.supj_w = m.supj_w;
    r.M = m.M; r.gmm_means = m.gmm_means; r.gmm_prec = m.gmm_prec; r.gmm_lognllw = m.gmm_lognllw;
    r.anchor = ctx->ws.anchor; r.anchor_w = ctx->ws.anchor_w;
    r.j3d_xyz = ctx->ws.j3d_xyz; r.j3d_conf = ctx->ws.j3d_conf;
    r.vp_w1 = m.vp_w1; r.vp_w2 = m.vp_w2; r.vp_w3 = m.vp_w3; r.vp_w1t = m.vp_w1t; r.vp_w2t = m.vp_w2t; r.vp_w3t = m.vp_w3t;
    r.vp_b1 = m.vp_b1; r.vp_b2 = m.vp_b2; r.vp_b3 = m.vp_b3;
    r.par = ctx->parents;
    r.cs = ctx->chain;
    return r;
}

int launch_closure_resident(mvs_ctx* ctx, const float* x_dev, float* loss_dev, float* grad_dev, float* joints_dev,
                            float* proj_dev, cudaStream_t st) {
    Workspace& w = ctx->ws;
    const size_t smem = sizeof(ResidentSmem) + (ctx->loss.use_vposer == 2 ? sizeof(VposerSmem) : 0);
    MVS_LAUNCH(ctx, KID_RESIDENT_CLOSURE, st,
               closure_resident_kernel<<<w.B, kResThreads, smem, st>>>(make_resident_model(ctx), slot_rig_set(ctx), ctx->loss, x_dev,
                                                                       w.fidx, w.na, w.gt_uv, w.conf, w.joint_w, w.B,
                                                                       grad_dev ? 1 : 0, loss_dev ? loss_dev : w.loss_scratch,
                                                                       grad_dev, joints_dev, proj_dev));
    MVS_CUDA_OK(ctx, cudaGetLastError());
    return MVS_OK;
}

int launch_shape_closure(mvs_ctx* ctx, const ShapeArgs& a, const ProblemChunk& c, const LossParams& lp, const LbfgsState& L,
                         cudaStream_t st) {
    const size_t smem = sizeof(ResidentSmem) + (lp.use_vposer == 2 ? sizeof(VposerSmem) : 0);
    ResidentModel rm = make_resident_model(ctx);
    rm.j3d_xyz = a.in.j3d_xyz; rm.j3d_conf = a.in.j3d_conf;           // row stride a.in.n, as gt_uv / conf
    MVS_LAUNCH(ctx, KID_RESIDENT_CLOSURE, st,
               shape_closure_kernel<<<c.ni, kResThreads, smem, st>>>(rm, RigSet{ctx->rigs_dev.p, a.in.rig}, lp, L, a, c));
    MVS_CUDA_OK(ctx, cudaGetLastError());
    return MVS_OK;
}

int launch_camera_joints(mvs_ctx* ctx, const FrameInputs& in, const float* params, const int* frames, int n, const LossParams& lp,
                         float* q, cudaStream_t st) {
    if (n <= 0) return MVS_OK;
    LossParams l = lp;
    l.j3d_on = 0;                                                     // only the keypoints are read: no 3-D targets, no anchor
    l.anchor_on = 0;
    const size_t smem = sizeof(ResidentSmem) + (l.use_vposer == 2 ? sizeof(VposerSmem) : 0);
    MVS_LAUNCH(ctx, KID_RESIDENT_CLOSURE, st,
               camera_joints_kernel<<<n, kResThreads, smem, st>>>(make_resident_model(ctx), RigSet{ctx->rigs_dev.p, in.rig}, l, in,
                                                                  params, frames, q));
    MVS_CUDA_OK(ctx, cudaGetLastError());
    return MVS_OK;
}

int launch_vposer_decode(mvs_ctx* ctx, const float* x_dev, float* body_pose_dev, cudaStream_t st) {
    const size_t smem = sizeof(ResidentSmem) + sizeof(VposerSmem);
    MVS_LAUNCH(ctx, KID_MISC, st,
               vposer_decode_kernel<<<ctx->ws.B, kResThreads, smem, st>>>(make_resident_model(ctx), x_dev, ctx->ws.B, body_pose_dev));
    MVS_CUDA_OK(ctx, cudaGetLastError());
    return MVS_OK;
}

static int stages_with_vposer(const LbfgsState& L, int nstages) {
    int v = 0;
    for (int i = 0; i < nstages; ++i) v |= (L.lp_tab_host[i].use_vposer == 2);
    return v;
}

// The launch set-up of the frame-resident optimiser kernels over the frames `in`: the model with in's 3-D target rows (row
// stride in.n, as gt_uv / conf), in's rigs, and the shared memory of one frame with the run's history (and the VPoser decoder
// when a stage of the run's table, as begin_run stored it, decodes one)
struct ResidentLaunch { ResidentModel m; RigSet rigs; int with_vposer; size_t smem; };
static ResidentLaunch resident_launch(const mvs_ctx* ctx, const FrameInputs& in, int H, int nstages) {
    ResidentLaunch r;
    r.m = make_resident_model(ctx);
    r.m.j3d_xyz = in.j3d_xyz; r.m.j3d_conf = in.j3d_conf;
    r.rigs = RigSet{ctx->rigs_dev.p, in.rig};
    r.with_vposer = stages_with_vposer(*ctx->lbfgs, nstages);
    r.smem = frame_smem(H, r.with_vposer != 0);
    return r;
}

int launch_lbfgs_resident(mvs_ctx* ctx, float* params_dev, const LbfgsCfg& cfg, int nstages, const FrameInputs& in,
                          FrameScalars* sc_out, float* last_grad_dev, const int2* stage_rng_dev, cudaStream_t st) {
    const ResidentLaunch r = resident_launch(ctx, in, cfg.history, nstages);
    MVS_LAUNCH(ctx, KID_RESIDENT_LBFGS, st,
               lbfgs_resident_kernel<<<in.n, kResThreads, r.smem, st>>>(r.m, r.rigs, ctx->lbfgs->lp_tab, nstages, cfg, params_dev,
                                                                        in.gt_uv, in.conf, in.joint_w, in.n, cfg.history, sc_out,
                                                                        last_grad_dev, r.with_vposer, stage_rng_dev));
    MVS_CUDA_OK(ctx, cudaGetLastError());
    return MVS_OK;
}

int launch_lbfgs_resident_seq(mvs_ctx* ctx, float* params_dev, const LbfgsCfg& cfg, int nstages, const FrameInputs& in,
                              const SeqChain& q, cudaStream_t st, const float* temporal_w) {
    ResidentLaunch r = resident_launch(ctx, in, cfg.history, nstages);
    if (temporal_w) {
        // the closure reads frame b's anchor row at anchor + 86 b: here the row of frame b - 1 in params, which the CTA wrote
        // (the frame's fitted row) before the barrier that starts warm frame b.  Cold frames run no anchored stage, so the
        // row before params is never read.
        r.m.anchor = params_dev - kParams;
        r.m.anchor_w = temporal_w;
    }
    MVS_LAUNCH(ctx, KID_RESIDENT_LBFGS, st,
               lbfgs_resident_seq_kernel<<<q.n_act, kResThreads, r.smem, st>>>(r.m, r.rigs, ctx->lbfgs->lp_tab, cfg, params_dev,
                                                                              in.gt_uv, in.conf, in.joint_w, in.n, cfg.history,
                                                                              r.with_vposer, q));
    MVS_CUDA_OK(ctx, cudaGetLastError());
    return MVS_OK;
}

// per-frame pose cache of frame_step; invalidated at the start of every run (the first round recomputes the pose)
int frame_step_begin_run(mvs_ctx* ctx, cudaStream_t st) {
    Workspace& w = ctx->ws;
    if (!w.pose_cache) {
        int rc;
        if ((rc = dev_alloc(ctx, &w.pose_cache, (size_t)w.B * kPoseCacheFloats))) return rc;
        if ((rc = dev_alloc(ctx, &w.pose_valid, (size_t)w.B))) return rc;
    }
    MVS_CUDA_OK(ctx, cudaMemsetAsync(w.pose_valid, 0, (size_t)w.B * sizeof(int), st));
    return MVS_OK;
}

static FrameStepArgs make_frame_step_args(mvs_ctx* ctx, float* params_dev, const LbfgsState& L, const LbfgsCfg& cfg, int nstages) {
    Workspace& w = ctx->ws;
    const DevModel& dm = ctx->m;
    FrameStepArgs a;
    a.m = make_resident_model(ctx); a.rigs = slot_rig_set(ctx); a.lp_tab = L.lp_tab; a.nstages = nstages;
    a.cfg = cfg; a.L = L; a.params = params_dev;
    a.gt_uv = w.gt_uv; a.conf = w.conf; a.joint_w = w.joint_w; a.B = w.B; a.N = dm.N;
    a.verts_ws = w.verts; a.poffT = tc_poffT(ctx); a.ST = dm.ST;
    a.parts5 = w.sdf_parts5; a.part = w.sdf_part; a.pflag = w.sdf_pflag; a.box = w.sdf_box;
    a.Wd = dm.Wd; a.Phi = w.Phi; a.PhiTc = w.PhiTc; a.At = w.At; a.ldA = w.ldA; a.slot_tr = w.slot_tr;
    a.pose_cache = w.pose_cache; a.pose_valid = w.pose_valid; a.with_vposer = stages_with_vposer(L, nstages);
    return a;
}

int launch_frame_step(mvs_ctx* ctx, float* params_dev, const LbfgsState& L, const LbfgsCfg& cfg, int nstages, cudaStream_t st) {
    Workspace& w = ctx->ws;
    const FrameStepArgs a = make_frame_step_args(ctx, params_dev, L, cfg, nstages);
    const size_t smem = frame_smem(L.H, a.with_vposer != 0);
    MVS_LAUNCH(ctx, KID_FRAME_STEP, st,
               MVS_CUDA_OK(ctx, launch_pdl(frame_step_kernel, dim3(w.na_bound > 0 ? w.na_bound : w.B), dim3(kResThreads), smem, st,
                                           a, (const int*)w.fidx, (const int*)w.na)));
    MVS_CUDA_OK(ctx, cudaGetLastError());
    return MVS_OK;
}

// slot-indexed pose forward of every active frame (run start, after a compaction); the axis-angle-only frame_fwd_kernel
// serves runs without a device-decoded VPoser stage
int launch_frame_fwd_dense(mvs_ctx* ctx, const float* x_dev, const LbfgsState& L, int nstages, cudaStream_t st) {
    if (!stages_with_vposer(L, nstages)) return launch_frame_fwd(ctx, x_dev, st);
    Workspace& w = ctx->ws;
    MVS_LAUNCH(ctx, KID_FRAME_FWD, st,
               frame_fwd_resident_kernel<<<w.na_bound > 0 ? w.na_bound : w.B, kResThreads, sizeof(ResidentSmem) + sizeof(VposerSmem), st>>>(
                   make_resident_model(ctx), L.lp_tab, L.sc, x_dev, w.fidx, w.na, w.Phi, w.PhiTc, w.At, w.ldA, w.slot_tr));
    MVS_CUDA_OK(ctx, cudaGetLastError());
    return MVS_OK;
}

}  // namespace mvs

#ifdef MVS_PHASE_DBG
extern "C" int mvs_debug_clocks(long long* out, int n) {       // debug builds only; not part of the ABI
    long long h[64];
    if (cudaMemcpyFromSymbol(h, mvs::g_phase_clk, sizeof(h)) != cudaSuccess) return -1;
    for (int i = 0; i < n && i < 64; ++i) out[i] = h[i];
    return 0;
}
#endif
