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
closure_resident_kernel(ResidentModel m, CamSet cams, LossParams lp, const float* __restrict__ x,
                        const int* __restrict__ fidx, const int* __restrict__ na_ptr, const float* __restrict__ gt_uv,
                        const float* __restrict__ conf, const float* __restrict__ joint_w, int B, int have_grad,
                        float* __restrict__ loss_out, float* __restrict__ grad_out, float* __restrict__ joints_out,
                        float* __restrict__ proj_out) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    ResidentSmem& S = *reinterpret_cast<ResidentSmem*>(smem_raw);
    const int slot = blockIdx.x;
    if (slot >= *na_ptr) return;
    const int b = fidx[slot];
    resident_setup(S, m);
    for (int i = threadIdx.x; i < kParams; i += kResThreads) S.x[i] = x[(size_t)b * kParams + i];
    __syncthreads();
    VposerSmem* W = lp.use_vposer == 2 ? reinterpret_cast<VposerSmem*>(smem_raw + sizeof(ResidentSmem)) : nullptr;
    resident_closure(S, m, cams, lp, gt_uv, conf, joint_w, B, b, have_grad != 0, joints_out, proj_out, DenseIn{}, W);
    if (threadIdx.x == 0) loss_out[b] = S.sc[2];
    if (have_grad)
        for (int i = threadIdx.x; i < kParams; i += kResThreads) grad_out[(size_t)b * kParams + i] = S.lg_new[i];
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
lbfgs_resident_kernel(ResidentModel m, CamSet cams, const LossParams* __restrict__ lp_tab, int nstages, LbfgsCfg cfg,
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
        if (t == 0) {
            FrameScalars s;
            memset(&s, 0, sizeof(s));
            s.phase = PH_DONE;
            s.final_loss = __int_as_float(0x7fc00000);
            sc_out[b] = s;
        }
        return;
    }
    resident_setup(S, m);
    for (int i = t; i < kParams; i += kResThreads) { const float v = params[(size_t)b * kParams + i]; S.lx[i] = v; S.lx_eval[i] = v; }
    if (t == 0) {
        FrameScalars s;
        memset(&s, 0, sizeof(s));
        s.phase = PH_STEP_ENTRY;
        s.H_diag = 1.f;
        s.final_loss = __int_as_float(0x7fc00000);
        s.stage = st_begin; s.stage_end = st_end;
        S.fs = s;
    }
    if (t < (int)(sizeof(LossParams) / 4)) reinterpret_cast<int*>(&S.lp)[t] = reinterpret_cast<const int*>(&lp_tab[st_begin])[t];
    __syncthreads();
    LbfgsPtrs P{S.lx, S.lg, S.ld, S.lprev_g, S.lx_init, S.lg_prev, S.lbg0, S.lbg1, hy, hs, S.ro, S.al, S.lx_eval, S.lg_new, H,
                S.gram, S.tl_scratch};
    // hard bound on closure evaluations per frame and stage (never reached by a terminating line search; a guard
    // against hanging the GPU): every outer step costs at most 1 + max_eval + max_iter evaluations
    const long long eval_cap = (long long)cfg.max_outer * (cfg.max_eval + cfg.max_iter + 2) + 8;
    long long stage_ev0 = 0;
    int cur_stage = st_begin;
    while (true) {
        PHASE_MARK(0);
        for (int i = t; i < kParams; i += kResThreads) S.x[i] = S.lx_eval[i];
        __syncthreads();
        PHASE_MARK(1);
        resident_closure(S, m, cams, S.lp, gt_uv, conf, joint_w, B, b, true, nullptr, nullptr, DenseIn{}, W);
        PHASE_MARK(23);
        if (warp == 0) {
            FrameScalars s = S.fs;
            lbfgs_advance_core(s, P, S.sc[2], cfg, lane, S.lp.use_vposer == 2 ? 32 : kOffTransl - kOffPose);
            if (s.evals - stage_ev0 >= eval_cap && s.phase != PH_DONE) { s.phase = PH_DONE; s.nan_flag = 1; }
            if (s.phase == PH_DONE && s.stage + 1 < s.stage_end) {      // this frame moves on to its next stage
                next_stage_scalars(s);
                VLOOP(i) S.lx_eval[i] = S.lx[i];
            }
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

// ------------------------------------------------------------------------------------------------ dense regime
// One round of the dense regime for one frame (multi-kernel path): see frame_step_body.
__global__ void __launch_bounds__(kResThreads, 2)
frame_step_kernel(FrameStepArgs a, const int* __restrict__ fidx, const int* __restrict__ na_ptr) {
    pdl_wait();
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int slot = blockIdx.x;
    if (slot >= *na_ptr) return;
    frame_step_body(smem_raw, a, slot, fidx[slot]);
}

// ------------------------------------------------------------------------------------------------ host side
static bool resident_supported(const mvs_ctx* ctx) {
    const DevModel& m = ctx->m;
    return ctx->exec_mode != 1 && m.supj_ptr != nullptr && m.nsup + 6 <= kResMaxSup && m.K <= kMaxKeypoints &&
           ctx->cams.num_views * m.K <= kResMaxVK && m.M <= kResMaxM;
}

static ResidentModel make_resident_model(const mvs_ctx* ctx) {
    const DevModel& m = ctx->m;
    ResidentModel r;
    r.Qk = m.Qk; r.Jt = m.Jt; r.JS = m.JS; r.ell_j = m.ell_j; r.ell_w = m.ell_w; r.KW = m.KW;
    r.K = m.K; r.nsup = m.nsup; r.kp_ptr = m.kp_ptr; r.kp_spos = m.kp_spos; r.kp_w = m.kp_w; r.kp_chain = m.kp_chain;
    r.sup = m.sup; r.sup_ptr = m.sup_ptr; r.sup_k = m.sup_k; r.sup_w = m.sup_w;
    r.supj_ptr = m.supj_ptr; r.supj_i = m.supj_i; r.supj_w = m.supj_w;
    r.M = m.M; r.gmm_means = m.gmm_means; r.gmm_prec = m.gmm_prec; r.gmm_lognllw = m.gmm_lognllw;
    r.anchor = ctx->ws.anchor; r.anchor_w = ctx->ws.anchor_w;
    r.vp_w1 = m.vp_w1; r.vp_w2 = m.vp_w2; r.vp_w3 = m.vp_w3; r.vp_w1t = m.vp_w1t; r.vp_w2t = m.vp_w2t; r.vp_w3t = m.vp_w3t;
    r.vp_b1 = m.vp_b1; r.vp_b2 = m.vp_b2; r.vp_b3 = m.vp_b3;
    r.par = ctx->parents;
    // level schedule of the tree (parents[j] < j is checked in mvs_set_model)
    int depth[kJoints];
    depth[0] = 0;
    int maxd = 0;
    for (int j = 1; j < kJoints; ++j) { depth[j] = depth[r.par.p[j]] + 1; if (depth[j] > maxd) maxd = depth[j]; }
    r.cs.nlev = maxd + 1;
    int o = 0;
    for (int L = 0; L <= maxd; ++L) {
        r.cs.lev_ptr[L] = (unsigned char)o;
        for (int j = 0; j < kJoints; ++j) if (depth[j] == L) r.cs.lev_j[o++] = (unsigned char)j;
    }
    for (int L = maxd + 1; L <= kJoints; ++L) r.cs.lev_ptr[L] = (unsigned char)o;
    o = 0;
    for (int p = 0; p < kJoints; ++p) {
        r.cs.ch_ptr[p] = (unsigned char)o;
        for (int j = kJoints - 1; j >= 1; --j) if (r.par.p[j] == p) r.cs.ch_j[o++] = (unsigned char)j;
    }
    r.cs.ch_ptr[kJoints] = (unsigned char)o;
    for (int q = o; q < kJoints; ++q) r.cs.ch_j[q] = 0;
    return r;
}

bool resident_closure_available(const mvs_ctx* ctx) { return resident_supported(ctx); }

int launch_closure_resident(mvs_ctx* ctx, const float* x_dev, float* loss_dev, float* grad_dev, float* joints_dev,
                            float* proj_dev, cudaStream_t st) {
    Workspace& w = ctx->ws;
    const size_t smem = sizeof(ResidentSmem) + (ctx->loss.use_vposer == 2 ? sizeof(VposerSmem) : 0);
    if (!ctx->attr_done_res) {
        MVS_CUDA_OK(ctx, cudaFuncSetAttribute(closure_resident_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                              (int)(sizeof(ResidentSmem) + sizeof(VposerSmem))));
        ctx->attr_done_res = true;
    }
    MVS_LAUNCH(ctx, KID_RESIDENT_CLOSURE, st,
               closure_resident_kernel<<<w.B, kResThreads, smem, st>>>(make_resident_model(ctx), ctx->cams, ctx->loss, x_dev,
                                                                       w.fidx, w.na, w.gt_uv, w.conf, w.joint_w, w.B,
                                                                       grad_dev ? 1 : 0, loss_dev ? loss_dev : w.loss_scratch,
                                                                       grad_dev, joints_dev, proj_dev));
    MVS_CUDA_OK(ctx, cudaGetLastError());
    return MVS_OK;
}

int launch_vposer_decode(mvs_ctx* ctx, const float* x_dev, float* body_pose_dev, cudaStream_t st) {
    const size_t smem = sizeof(ResidentSmem) + sizeof(VposerSmem);
    MVS_CUDA_OK(ctx, cudaFuncSetAttribute(vposer_decode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    MVS_LAUNCH(ctx, KID_MISC, st,
               vposer_decode_kernel<<<ctx->ws.B, kResThreads, smem, st>>>(make_resident_model(ctx), x_dev, ctx->ws.B, body_pose_dev));
    MVS_CUDA_OK(ctx, cudaGetLastError());
    return MVS_OK;
}

bool resident_lbfgs_available_for(const mvs_ctx* ctx, const LossParams& lp, int H) {
    const bool sdf_on = lp.interpenetration && lp.coll_loss_weight > 0.f;
    return resident_supported(ctx) && !sdf_on && H <= 100;
}
bool resident_lbfgs_available(const mvs_ctx* ctx, int H) { return resident_lbfgs_available_for(ctx, ctx->loss, H); }

int launch_lbfgs_resident(mvs_ctx* ctx, float* params_dev, const void* cfg_ptr, int H, const void* lp_tab_dev,
                          const void* lp_tab_host, int nstages, void* sc_out, float* last_grad_dev, cudaStream_t st,
                          const void* stage_rng_dev) {
    Workspace& w = ctx->ws;
    const LbfgsCfg& cfg = *static_cast<const LbfgsCfg*>(cfg_ptr);
    const LossParams* lph = static_cast<const LossParams*>(lp_tab_host);
    int with_vposer = 0;
    for (int i = 0; i < nstages; ++i) with_vposer |= (lph[i].use_vposer == 2);
    const size_t smem = sizeof(ResidentSmem) + (size_t)2 * H * kParams * sizeof(float) + (with_vposer ? sizeof(VposerSmem) : 0);
    if (ctx->attr_res_lbfgs_smem < (int)smem) {
        MVS_CUDA_OK(ctx, cudaFuncSetAttribute(lbfgs_resident_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        ctx->attr_res_lbfgs_smem = (int)smem;
    }
    MVS_LAUNCH(ctx, KID_RESIDENT_LBFGS, st,
               lbfgs_resident_kernel<<<w.B, kResThreads, smem, st>>>(make_resident_model(ctx), ctx->cams,
                                                                     static_cast<const LossParams*>(lp_tab_dev), nstages, cfg,
                                                                     params_dev, w.gt_uv, w.conf, w.joint_w, w.B, H,
                                                                     static_cast<FrameScalars*>(sc_out), last_grad_dev, with_vposer,
                                                                     static_cast<const int2*>(stage_rng_dev)));
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

bool hybrid_available_for(const mvs_ctx* ctx, const LossParams& lp) {
    const bool sdf_on = lp.interpenetration && lp.coll_loss_weight > 0.f;
    return resident_supported(ctx) && sdf_on && (ctx->m.N + 255) / 256 <= 64;      // frame_step's block list holds 64 entries
}
bool hybrid_available(const mvs_ctx* ctx) { return hybrid_available_for(ctx, ctx->loss); }

static int stages_with_vposer(const LbfgsState& L, int nstages) {
    int v = 0;
    for (int i = 0; i < nstages; ++i) v |= (L.lp_tab_host[i].use_vposer == 2);
    return v;
}

FrameStepArgs make_frame_step_args(mvs_ctx* ctx, float* params_dev, const void* lbfgs_state, const void* lbfgs_cfg, int nstages) {
    Workspace& w = ctx->ws;
    const DevModel& dm = ctx->m;
    const LbfgsState& L = *static_cast<const LbfgsState*>(lbfgs_state);
    FrameStepArgs a;
    a.m = make_resident_model(ctx); a.cams = ctx->cams; a.lp_tab = L.lp_tab; a.nstages = nstages;
    a.cfg = *static_cast<const LbfgsCfg*>(lbfgs_cfg); a.L = L; a.params = params_dev;
    a.gt_uv = w.gt_uv; a.conf = w.conf; a.joint_w = w.joint_w; a.B = w.B; a.N = dm.N;
    a.verts_ws = w.verts; a.poffT = tc_poffT(ctx); a.ST = dm.ST;
    a.parts5 = w.sdf_parts5; a.part = w.sdf_part; a.pflag = w.sdf_pflag; a.box = reinterpret_cast<const FrameBox*>(w.sdf_box);
    a.Wd = dm.Wd; a.Phi = w.Phi; a.PhiTc = w.PhiTc; a.At = w.At; a.ldA = w.ldA; a.slot_tr = w.slot_tr;
    a.pose_cache = w.pose_cache; a.pose_valid = w.pose_valid; a.with_vposer = stages_with_vposer(L, nstages);
    return a;
}

size_t frame_step_smem(int H, bool with_vposer) {
    return sizeof(ResidentSmem) + (size_t)2 * H * kParams * sizeof(float) + (with_vposer ? sizeof(VposerSmem) : 0);
}

int launch_frame_step(mvs_ctx* ctx, float* params_dev, const void* lbfgs_state, const void* lbfgs_cfg, int nstages,
                      cudaStream_t st) {
    Workspace& w = ctx->ws;
    const LbfgsState& L = *static_cast<const LbfgsState*>(lbfgs_state);
    const FrameStepArgs a = make_frame_step_args(ctx, params_dev, lbfgs_state, lbfgs_cfg, nstages);
    const size_t smem = frame_step_smem(L.H, a.with_vposer != 0);
    if (!ctx->attr_done_step) {
        MVS_CUDA_OK(ctx, cudaFuncSetAttribute(frame_step_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                              (int)frame_step_smem(L.H, true)));
        MVS_CUDA_OK(ctx, cudaFuncSetAttribute(frame_fwd_resident_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                              (int)(sizeof(ResidentSmem) + sizeof(VposerSmem))));
        ctx->attr_done_step = true;
    }
    MVS_LAUNCH(ctx, KID_FRAME_STEP, st,
               MVS_CUDA_OK(ctx, launch_pdl(frame_step_kernel, dim3(w.na_bound > 0 ? w.na_bound : w.B), dim3(kResThreads), smem, st,
                                           a, (const int*)w.fidx, (const int*)w.na)));
    MVS_CUDA_OK(ctx, cudaGetLastError());
    return MVS_OK;
}

// slot-indexed pose forward of every active frame (run start, after a compaction); the axis-angle-only frame_fwd_kernel
// serves runs without a device-decoded VPoser stage
int launch_frame_fwd_dense(mvs_ctx* ctx, const float* x_dev, const void* lbfgs_state, int nstages, cudaStream_t st) {
    const LbfgsState& L = *static_cast<const LbfgsState*>(lbfgs_state);
    if (!stages_with_vposer(L, nstages)) return launch_frame_fwd(ctx, x_dev, st);
    Workspace& w = ctx->ws;
    if (!ctx->attr_done_step) {
        MVS_CUDA_OK(ctx, cudaFuncSetAttribute(frame_fwd_resident_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                              (int)(sizeof(ResidentSmem) + sizeof(VposerSmem))));
    }
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
