// Batched, device-resident L-BFGS with strong-Wolfe cubic line search: one independent
// optimisation problem per frame, advanced as a per-frame state machine between batched
// closure evaluations.  Replaces (reference paths under code/):
//   optimizers/lbfgs_ls.py:11-36   _cubic_interpolate
//   optimizers/lbfgs_ls.py:39-167  _strong_Wolfe
//   optimizers/lbfgs_ls.py:256-445 LBFGS.step   (history 100, persistent state across step() calls)
//   utils/fitting.py:71-142        FittingMonitor.run_fitting (NaN/Inf guard, ftol, gtol)
//
// The reference runs this loop in Python with a blocking float(closure()) per evaluation
// (lbfgs_ls.py:251,281).  Here no scalar leaves the GPU.  run_stage picks one of three execution regimes per
// group of stages (DESIGN.md section 4):
//   frame-resident   one CTA per frame runs closure + state machine for ALL stages of the group inside ONE launch
//                    (mvs_resident.cu: lbfgs_resident_kernel)
//   dense rounds     SDF term on: per round posedirs_gemm_tc -> skin -> sdf_fused -> frame_step; finished frames are
//                    compacted out every 8 rounds; the host reads the active count one chunk late (the next chunk is
//                    already enqueued) and only uses it to size grids and to stop
//   batched chain    the reference SIMT path (launch_closure + lbfgs_advance_kernel + lbfgs_compact_kernel), also
//                    what mvs_lbfgs_step (one LBFGS.step per call, state persistent in the context) uses
// run_fit hands consecutive stages of the same regime to one run in which every frame changes stage on its own.
//
// Arithmetic mirrors the reference's types: dot products, step lengths and directional
// derivatives are fp32 (0-dim fp32 tensors there), losses are Python floats there and are
// compared / subtracted in double here.
#include <math.h>
#include <stdio.h>

#include <chrono>
#include <cstdio>
#include <vector>
#include <cstdlib>
#include "mvs_internal.cuh"
#include "mvs_lbfgs_core.cuh"

namespace mvs {

// reset != 0: fresh optimiser (new stage).  reset == 0: next step() of the same optimiser: history, d, t,
// H_diag, prev_flat_grad, prev_loss and n_iter persist (lbfgs_ls.py:292-300,436-443).
__global__ void lbfgs_init_kernel(LbfgsState S, const float* __restrict__ params, int B, int reset, int nstages,
                                  const int2* __restrict__ stage_rng) {
    const int b = blockIdx.x, lane = threadIdx.x;
    if (b >= B) return;
    VLOOP(i) S.x_eval[(size_t)b * kParams + i] = params[(size_t)b * kParams + i];
    if (lane == 0) {
        FrameScalars s;
        if (reset) {
            memset(&s, 0, sizeof(s));
            s.H_diag = 1.f;
        } else {
            s = S.sc[b];
            s.outer_n = 0; s.have_prev = 0; s.nan_flag = 0; s.iters = 0; s.evals = 0;
        }
        s.phase = PH_STEP_ENTRY;
        s.final_loss = __int_as_float(0x7fc00000);
        if (reset) {                                        // this frame's slice of the stage table (mvs_fit_seq)
            s.stage = stage_rng ? stage_rng[b].x : 0;
            s.stage_end = stage_rng ? stage_rng[b].y : nstages;
            if (s.stage >= s.stage_end) s.phase = PH_DONE;  // no stage of this run is for this frame
        }
        S.sc[b] = s;
    }
}

__global__ void __launch_bounds__(32)
lbfgs_advance_kernel(LbfgsState S, LbfgsCfg cfg, float* __restrict__ params, const int* __restrict__ fidx,
                     const int* __restrict__ na_ptr, int pose_len) {
    const int slot = blockIdx.x;
    if (slot >= *na_ptr) return;
    const int b = fidx[slot];
    const int lane = threadIdx.x;
    __shared__ float al[128];
    __shared__ float scratch[96];
    FrameScalars s = S.sc[b];
    float* x = params + (size_t)b * kParams;
    float* g = S.g + (size_t)b * kParams;
    float* d = S.d + (size_t)b * kParams;
    float* prev_g = S.prev_g + (size_t)b * kParams;
    float* x_init = S.x_init + (size_t)b * kParams;
    float* g_prev = S.g_prev + (size_t)b * kParams;
    float* bg0 = S.bg + (size_t)b * 2 * kParams;
    float* bg1 = bg0 + kParams;
    float* hy = S.hist_y + (size_t)b * S.H * kParams;
    float* hs = S.hist_s + (size_t)b * S.H * kParams;
    float* ro = S.ro + (size_t)b * S.H;
    float* x_eval = S.x_eval + (size_t)b * kParams;
    const float* g_new = S.g_eval + (size_t)b * kParams;
    const float f_new = S.loss_eval[b];

    LbfgsPtrs P{x, g, d, prev_g, x_init, g_prev, bg0, bg1, hy, hs, ro, al, x_eval, g_new, S.H,
                S.gram + (size_t)b * kGramFloats, scratch};
    lbfgs_advance_core(s, P, f_new, cfg, lane, pose_len);
    __syncwarp();
    if (lane == 0) S.sc[b] = s;
}

// Ordered compaction of the frames that still need closure evaluations.
__global__ void __launch_bounds__(1024) lbfgs_compact_kernel(LbfgsState S, int B, int* __restrict__ fidx, int* __restrict__ na) {
    pdl_wait();
    if (threadIdx.x == 0 && *na > 0) S.totals[3] += 1;     // rounds that actually evaluated something
    __shared__ int wsum[32];
    __shared__ int base;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    if (tid == 0) base = 0;
    __syncthreads();
    for (int b0 = 0; b0 < B; b0 += 1024) {
        const int b = b0 + tid;
        const int act = (b < B && S.sc[b].phase != PH_DONE) ? 1 : 0;
        const unsigned m = __ballot_sync(0xffffffffu, act);
        const int pre = __popc(m & ((1u << lane) - 1));
        if (lane == 0) wsum[wid] = __popc(m);
        __syncthreads();
        int off = base;
        for (int w = 0; w < wid; ++w) off += wsum[w];
        if (act) fidx[off + pre] = b;
        __syncthreads();
        if (tid == 0) { int tot = 0; for (int w = 0; w < 32; ++w) tot += wsum[w]; base += tot; }
        __syncthreads();
    }
    if (tid == 0) *na = base;
}

__global__ void lbfgs_finalize_kernel(LbfgsState S, int B, float* __restrict__ final_loss, long long* __restrict__ totals,
                                      int max_evals_as_rounds) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const FrameScalars s = S.sc[b];
    if (final_loss) final_loss[b] = s.final_loss;
    atomicAdd((unsigned long long*)&totals[0], (unsigned long long)s.iters);
    atomicAdd((unsigned long long*)&totals[1], (unsigned long long)s.evals);
    atomicAdd((unsigned long long*)&totals[2], (unsigned long long)(s.nan_flag + s.nan_acc));
    if (max_evals_as_rounds) atomicMax((unsigned long long*)&totals[3], (unsigned long long)s.evals);
}

__global__ void iota2_kernel(int* p, int n, int* na) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = i;
    if (i == 0) *na = n;
}

static int ensure_state(mvs_ctx* ctx, int H) {
    LbfgsState* S = static_cast<LbfgsState*>(ctx->lbfgs);
    const int B = ctx->ws.B;
    if (S && S->B == B && S->H == H) return MVS_OK;
    if (S) return set_error(ctx, MVS_ERR_INVALID, "mvs_lbfgs_run: history_size changed between calls (%d -> %d)", S->H, H);
    S = new LbfgsState();
    S->B = B; S->H = H;
    int rc;
    const size_t V = (size_t)B * kParams;
    if ((rc = dev_alloc(ctx, &S->g, V))) return rc;
    if ((rc = dev_alloc(ctx, &S->d, V))) return rc;
    if ((rc = dev_alloc(ctx, &S->prev_g, V))) return rc;
    if ((rc = dev_alloc(ctx, &S->x_init, V))) return rc;
    if ((rc = dev_alloc(ctx, &S->g_prev, V))) return rc;
    if ((rc = dev_alloc(ctx, &S->bg, 2 * V))) return rc;
    if ((rc = dev_alloc(ctx, &S->hist_y, V * H))) return rc;
    if ((rc = dev_alloc(ctx, &S->hist_s, V * H))) return rc;
    if ((rc = dev_alloc(ctx, &S->ro, (size_t)B * H))) return rc;
    if ((rc = dev_alloc(ctx, &S->gram, (size_t)B * kGramFloats))) return rc;
    if ((rc = dev_alloc(ctx, &S->x_eval, V))) return rc;
    if ((rc = dev_alloc(ctx, &S->loss_eval, B))) return rc;
    if ((rc = dev_alloc(ctx, &S->g_eval, V))) return rc;
    if ((rc = dev_alloc(ctx, &S->x_fit, V))) return rc;
    if ((rc = dev_alloc(ctx, &S->final_fit, B))) return rc;
    unsigned char* raw = nullptr;
    if ((rc = dev_alloc(ctx, &raw, (size_t)B * sizeof(FrameScalars)))) return rc;
    S->sc = reinterpret_cast<FrameScalars*>(raw);
    unsigned char* raw2 = nullptr;
    if ((rc = dev_alloc(ctx, &raw2, 4 * sizeof(long long)))) return rc;
    S->totals = reinterpret_cast<long long*>(raw2);
    MVS_CUDA_OK(ctx, cudaMallocHost(&S->na_host, 8 * sizeof(long long)));
    MVS_CUDA_OK(ctx, cudaMallocHost(&S->lp_tab_host, kMaxStages * sizeof(LossParams)));
    unsigned char* raw3 = nullptr;
    if ((rc = dev_alloc(ctx, &raw3, kMaxStages * sizeof(LossParams)))) return rc;
    S->lp_tab = reinterpret_cast<LossParams*>(raw3);
    ctx->lbfgs = S;
    return MVS_OK;
}

// Runs the stages lps[0 .. nst) (nst == 1: ctx->loss).  nst > 1 requires that all of them run in the same regime
// (frame-resident or dense rounds, see run_fit): every frame then walks through the stages at its own pace.
static int run_stage(mvs_ctx* ctx, float* params_dev, float* final_loss_dev, const mvs_lbfgs_config* c,
                     mvs_lbfgs_stats* stats, cudaStream_t st, int step_mode = 0, int reset = 1,
                     float* last_grad_dev = nullptr, const LossParams* lps = nullptr, int nst = 1,
                     const int2* stage_rng = nullptr, bool some_inactive = false) {
    const int B = ctx->ws.B;
    const int H = c->history_size > 0 ? c->history_size : 100;
    if (H > 128) return set_error(ctx, MVS_ERR_INVALID, "mvs_lbfgs_run: history_size must be <= 128");
    int rc = ensure_state(ctx, H);
    if (rc) return rc;
    LbfgsState& S = *static_cast<LbfgsState*>(ctx->lbfgs);
    LbfgsCfg cfg;
    cfg.max_outer = c->max_outer > 0 ? c->max_outer : 30;
    cfg.max_iter = c->max_iter > 0 ? c->max_iter : 30;
    cfg.max_eval = c->max_eval > 0 ? c->max_eval : cfg.max_iter * 5 / 4;
    cfg.history = H;
    cfg.max_ls = 25;                                            // _strong_Wolfe default (lbfgs_ls.py:41)
    cfg.step_mode = step_mode;
    cfg.lr = c->lr > 0.f ? c->lr : 1.f;
    cfg.tol_grad = c->tolerance_grad; cfg.tol_change = c->tolerance_change;
    cfg.ftol = (double)c->ftol; cfg.gtol = (double)c->gtol;

    Workspace& w = ctx->ws;
    MVS_CUDA_OK(ctx, cudaMemsetAsync(S.totals, 0, 4 * sizeof(long long), st));
    if (!lps) { lps = &ctx->loss; nst = 1; }
    if (nst > kMaxStages) return set_error(ctx, MVS_ERR_INVALID, "at most %d stages per run", kMaxStages);
    // stage table for the multi-stage kernels (the previous run ended with a stream synchronisation, so the pinned
    // staging copy is free)
    for (int i = 0; i < nst; ++i) S.lp_tab_host[i] = lps[i];
    MVS_CUDA_OK(ctx, cudaMemcpyAsync(S.lp_tab, S.lp_tab_host, (size_t)nst * sizeof(LossParams), cudaMemcpyHostToDevice, st));
    if (!step_mode && resident_lbfgs_available(ctx, H)) {
        // sparse regime: every frame runs its whole stage inside one CTA (mvs_resident.cu): one launch, no rounds
        rc = launch_lbfgs_resident(ctx, params_dev, &cfg, H, S.lp_tab, lps, nst, S.sc, last_grad_dev, st, stage_rng);
        if (rc) return rc;
        MVS_LAUNCH(ctx, KID_MISC, st, lbfgs_finalize_kernel<<<(B + 255) / 256, 256, 0, st>>>(S, B, final_loss_dev, S.totals, 1));
        long long* th = reinterpret_cast<long long*>(S.na_host) + 1;
        MVS_CUDA_OK(ctx, cudaMemcpyAsync(th, S.totals, 4 * sizeof(long long), cudaMemcpyDeviceToHost, st));
        MVS_CUDA_OK(ctx, cudaStreamSynchronize(st));
        if (stats) {
            stats->frame_iterations += th[0]; stats->frame_evals += th[1]; stats->frames_nan += (int)th[2];
            stats->rounds += (int)th[3];          // critical path: the largest per-frame evaluation count
        }
        MVS_CUDA_OK(ctx, cudaGetLastError());
        return MVS_OK;
    }
    // use_vposer = 2 (VPoser decode on the device) exists in the frame-resident closure and in the dense-regime kernels, not in
    // the SIMT reference chain.  mvs_lbfgs_step therefore runs its one step() per call through the dense rounds when the SDF
    // term is on, and through launch_closure's frame-resident kernel + lbfgs_advance_kernel otherwise.
    const bool vp2 = ctx->loss.use_vposer == 2;
    const bool sdf_on = ctx->loss.interpenetration && ctx->loss.coll_loss_weight > 0.f;
    if (vp2 && (sdf_on ? !hybrid_available(ctx) : !resident_closure_available(ctx)))
        return set_error(ctx, MVS_ERR_INVALID, "use_vposer = 2 (VPoser decode on the device) is not implemented in the batched "
                                               "reference chain (exec mode 1): use use_vposer = 1 there");
    MVS_LAUNCH(ctx, KID_MISC, st, iota2_kernel<<<(B + 255) / 256, 256, 0, st>>>(w.fidx, B, w.na));
    MVS_LAUNCH(ctx, KID_MISC, st, lbfgs_init_kernel<<<B, 32, 0, st>>>(S, params_dev, B, reset, nst, stage_rng));
    if (some_inactive)                                      // frames without a stage in this run leave the active list now
        MVS_LAUNCH(ctx, KID_LBFGS_COMPACT, st, lbfgs_compact_kernel<<<1, 1024, 0, st>>>(S, B, w.fidx, w.na));
    if ((!step_mode || vp2) && hybrid_available(ctx)) {
        // dense regime (SDF term on): four launches per round -- pose blend shapes of the active frames (wgmma
        // GEMM), skinning + box partials, the SDF term with the adjoint of its (short) vertex list, and the per-frame
        // closure adjoint + optimiser step + next pose forward.  Finished frames are compacted out once per chunk.
        const int chunk = 8;
        const long long max_rounds = ((long long)cfg.max_outer * (cfg.max_eval + cfg.max_iter + 2) + 8) * nst;
        long long rounds = 0;
        int na_host = B;
        static const bool trace_na = getenv("MVS_TRACE_NA") != nullptr;       // debugging aid: active-list size per chunk
        // debugging aid: how long the host thread waited for the GPU inside the round loop (close to 0 = the GPU waits for the host)
        static const bool trace_host = getenv("MVS_TRACE_HOST") != nullptr;
        double blocked_us = 0.0;
        const auto loop_t0 = std::chrono::steady_clock::now();
        rc = launch_frame_fwd_dense(ctx, S.x_eval, &S, nst, st);
        if (rc) return rc;
        if ((rc = frame_step_begin_run(ctx, st))) return rc;
        // The host only needs the active count to know when to stop, so chunk k+1 is enqueued BEFORE the count of
        // chunk k is awaited (kernels exit at once when the list is empty): the GPU never idles on the host round trip.
        if (!S.na_event[0]) {
            // blocking sync: the host thread sleeps while it waits for a chunk (several contexts are driven by as many host
            // threads; spinning ones would compete with the threads that have launches to enqueue)
            MVS_CUDA_OK(ctx, cudaEventCreateWithFlags(&S.na_event[0], cudaEventDisableTiming | cudaEventBlockingSync));
            MVS_CUDA_OK(ctx, cudaEventCreateWithFlags(&S.na_event[1], cudaEventDisableTiming | cudaEventBlockingSync));
        }
        int* na_slots = reinterpret_cast<int*>(S.na_host);           // [0], [1]: two chunks in flight
        int pending = -1;                                             // chunk whose count has not been read yet
        long long chunk_idx = 0;
        w.na_bound = B;                                               // grids shrink with the (lagging) host view of the count
        while (rounds < max_rounds) {
            for (int r = 0; r < chunk; ++r) {
                if ((rc = launch_vertex_fwd_dense(ctx, st, true, false))) return rc;   // wgmma GEMM + LBS + bbox partials
                if ((rc = launch_sdf_fused(ctx, st))) return rc;   // samples + adjoint of the listed vertices
                if ((rc = launch_frame_step(ctx, params_dev, &S, &cfg, nst, st))) return rc;
                ++rounds;
            }
            // compaction changes slot -> frame, so the surviving frames' Phi / transforms are rebuilt for their new slots
            MVS_LAUNCH(ctx, KID_LBFGS_COMPACT, st, lbfgs_compact_kernel<<<1, 1024, 0, st>>>(S, B, w.fidx, w.na));
            if ((rc = launch_frame_fwd_dense(ctx, S.x_eval, &S, nst, st))) return rc;
            const int cur = (int)(chunk_idx & 1);
            MVS_CUDA_OK(ctx, cudaMemcpyAsync(&na_slots[cur], w.na, sizeof(int), cudaMemcpyDeviceToHost, st));
            MVS_CUDA_OK(ctx, cudaEventRecord(S.na_event[cur], st));
            if (pending >= 0) {
                const auto tb0 = std::chrono::steady_clock::now();
                MVS_CUDA_OK(ctx, cudaEventSynchronize(S.na_event[pending]));
                if (trace_host) blocked_us += std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - tb0).count();
                na_host = na_slots[pending];
                if (trace_na) fprintf(stderr, "[mvs] dense regime: chunk %lld, active frames %d\n", chunk_idx - 1, na_host);
                if (na_host <= 0) break;
                w.na_bound = na_host;                                 // the list only shrinks: still an upper bound
            }
            pending = cur;
            ++chunk_idx;
        }
        w.na_bound = B;
        if (trace_host) {
            const double enq = std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - loop_t0).count();
            const auto td0 = std::chrono::steady_clock::now();
            MVS_CUDA_OK(ctx, cudaStreamSynchronize(st));
            const double drain = std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - td0).count();
            fprintf(stderr, "[mvs] dense regime host loop: %lld rounds, %.0f us in the loop (%.0f us of it blocked on the GPU), %.0f us "
                            "draining afterwards\n", rounds, enq, blocked_us, drain);
        }
        MVS_CUDA_OK(ctx, cudaStreamSynchronize(st));
        if ((rc = tc_check_error(ctx))) return rc;
        MVS_LAUNCH(ctx, KID_MISC, st, lbfgs_finalize_kernel<<<(B + 255) / 256, 256, 0, st>>>(S, B, final_loss_dev, S.totals, 1));
        if (last_grad_dev)
            MVS_CUDA_OK(ctx, cudaMemcpyAsync(last_grad_dev, S.g_eval, (size_t)B * kParams * sizeof(float), cudaMemcpyDeviceToDevice, st));
        long long* th = reinterpret_cast<long long*>(S.na_host) + 1;
        MVS_CUDA_OK(ctx, cudaMemcpyAsync(th, S.totals, 4 * sizeof(long long), cudaMemcpyDeviceToHost, st));
        MVS_LAUNCH(ctx, KID_MISC, st, iota2_kernel<<<(B + 255) / 256, 256, 0, st>>>(w.fidx, B, w.na));
        MVS_CUDA_OK(ctx, cudaStreamSynchronize(st));
        if (stats) {
            stats->frame_iterations += th[0]; stats->frame_evals += th[1]; stats->frames_nan += (int)th[2];
            stats->rounds += (int)th[3];
            stats->dense_frame_evals += th[1]; stats->dense_rounds += (int)th[3];
        }
        MVS_CUDA_OK(ctx, cudaGetLastError());
        return MVS_OK;
    }
    const int chunk = 8;
    const long long max_rounds = (long long)cfg.max_outer * (cfg.max_eval + cfg.max_iter + 2) + 8;
    long long rounds = 0;
    int na_host = B;
    while (na_host > 0 && rounds < max_rounds) {
        for (int r = 0; r < chunk; ++r) {
            rc = launch_closure(ctx, S.x_eval, S.loss_eval, S.g_eval, nullptr, nullptr, nullptr, st);
            if (rc) return rc;
            MVS_LAUNCH(ctx, KID_LBFGS_ADVANCE, st, lbfgs_advance_kernel<<<B, 32, 0, st>>>(S, cfg, params_dev, w.fidx, w.na, vp2 ? 32 : kOffTransl - kOffPose));
            MVS_LAUNCH(ctx, KID_LBFGS_COMPACT, st, lbfgs_compact_kernel<<<1, 1024, 0, st>>>(S, B, w.fidx, w.na));
            ++rounds;
        }
        MVS_CUDA_OK(ctx, cudaMemcpyAsync(S.na_host, w.na, sizeof(int), cudaMemcpyDeviceToHost, st));
        MVS_CUDA_OK(ctx, cudaStreamSynchronize(st));
        na_host = *S.na_host;
    }
    MVS_LAUNCH(ctx, KID_MISC, st, lbfgs_finalize_kernel<<<(B + 255) / 256, 256, 0, st>>>(S, B, final_loss_dev, S.totals, 0));
    if (last_grad_dev)
        MVS_CUDA_OK(ctx, cudaMemcpyAsync(last_grad_dev, S.g_eval, (size_t)B * kParams * sizeof(float), cudaMemcpyDeviceToDevice, st));
    long long* tot_host = reinterpret_cast<long long*>(S.na_host) + 1;
    MVS_CUDA_OK(ctx, cudaMemcpyAsync(tot_host, S.totals, 4 * sizeof(long long), cudaMemcpyDeviceToHost, st));
    // leave the context usable for plain closures: full active list again
    MVS_LAUNCH(ctx, KID_MISC, st, iota2_kernel<<<(B + 255) / 256, 256, 0, st>>>(w.fidx, B, w.na));
    MVS_CUDA_OK(ctx, cudaStreamSynchronize(st));
    if (stats) {
        stats->frame_iterations += tot_host[0];
        stats->frame_evals += tot_host[1];
        stats->frames_nan += (int)tot_host[2];
        stats->rounds += (int)tot_host[3];
    }
    MVS_CUDA_OK(ctx, cudaGetLastError());
    return MVS_OK;
}

// One closure evaluation through the dense-regime kernels (posedirs_gemm_tc -> skin -> sdf_fused -> frame_step with the
// optimiser step switched off): mvs_closure in exec mode 3.  Exists so that parity tests can compare the loss and every
// gradient segment of the kernels the optimiser actually runs with the SDF term on (DESIGN.md section 2).
int dense_regime_closure(mvs_ctx* ctx, const float* x_dev, float* loss_dev, float* grad_dev, cudaStream_t st) {
    const int B = ctx->ws.B;
    int rc = ensure_state(ctx, static_cast<LbfgsState*>(ctx->lbfgs) ? static_cast<LbfgsState*>(ctx->lbfgs)->H : 100);
    if (rc) return rc;
    LbfgsState& S = *static_cast<LbfgsState*>(ctx->lbfgs);
    Workspace& w = ctx->ws;
    LbfgsCfg cfg{};
    cfg.max_outer = 1; cfg.max_iter = 1; cfg.max_eval = 1; cfg.history = S.H; cfg.max_ls = 25; cfg.step_mode = 2; cfg.lr = 1.f;
    S.lp_tab_host[0] = ctx->loss;
    MVS_CUDA_OK(ctx, cudaMemcpyAsync(S.lp_tab, S.lp_tab_host, sizeof(LossParams), cudaMemcpyHostToDevice, st));
    MVS_LAUNCH(ctx, KID_MISC, st, iota2_kernel<<<(B + 255) / 256, 256, 0, st>>>(w.fidx, B, w.na));
    MVS_LAUNCH(ctx, KID_MISC, st, lbfgs_init_kernel<<<B, 32, 0, st>>>(S, x_dev, B, 1, 1, nullptr));
    w.na_bound = B;
    if ((rc = launch_frame_fwd_dense(ctx, S.x_eval, &S, 1, st))) return rc;
    if ((rc = frame_step_begin_run(ctx, st))) return rc;
    if ((rc = launch_vertex_fwd_dense(ctx, st, true, false))) return rc;
    if ((rc = launch_sdf_fused(ctx, st))) return rc;
    if ((rc = launch_frame_step(ctx, const_cast<float*>(x_dev) /* read only in this mode */, &S, &cfg, 1, st))) return rc;
    if (loss_dev) MVS_CUDA_OK(ctx, cudaMemcpyAsync(loss_dev, S.loss_eval, (size_t)B * sizeof(float), cudaMemcpyDeviceToDevice, st));
    if (grad_dev) MVS_CUDA_OK(ctx, cudaMemcpyAsync(grad_dev, S.g_eval, (size_t)B * kParams * sizeof(float), cudaMemcpyDeviceToDevice, st));
    MVS_CUDA_OK(ctx, cudaStreamSynchronize(st));         // the pinned stage table is reused by the next call
    if ((rc = tc_check_error(ctx))) return rc;
    MVS_CUDA_OK(ctx, cudaGetLastError());
    return MVS_OK;
}

// All stages of a fit.  Consecutive stages that run in the same regime are handed to ONE multi-stage run in which
// every frame changes stage on its own (frames are independent problems, so a frame that converged need not wait at
// the stage boundary for the slowest one; the per-frame arithmetic is the sequential schedule's).  exec_mode 2 keeps
// the stage barrier (one run per stage).
static int run_fit(mvs_ctx* ctx, float* x_dev, int n_stages, const mvs_loss_config* stage_cfgs, const mvs_lbfgs_config* opt_cfg,
                   float* final_loss_dev, mvs_lbfgs_stats* stats, cudaStream_t st, const unsigned char* warm_host = nullptr) {
    if (n_stages > 64) return set_error(ctx, MVS_ERR_INVALID, "mvs_fit: at most 64 stages");
    std::vector<LossParams> lps(n_stages);
    for (int i = 0; i < n_stages; ++i) {
        const int rc = make_loss_params(ctx, &stage_cfgs[i], &lps[i]);
        if (rc) return rc;
    }
    const int B = ctx->ws.B;
    // warm-started frames (is_seq, non_linear_solver.py:157-162): no stage 0 and 1, stage 2 with 0.15 x body_pose_weight
    constexpr int kWarmSkip = 2;
    bool any_warm = false;
    if (warm_host)
        for (int b = 0; b < B; ++b) any_warm |= warm_host[b] != 0;
    if (any_warm && n_stages <= kWarmSkip)
        return set_error(ctx, MVS_ERR_INVALID, "mvs_fit_seq: warm-started frames skip the first %d stages, %d given", kWarmSkip, n_stages);
    std::vector<LossParams> wlps;
    if (any_warm) {
        wlps = lps;
        std::vector<mvs_loss_config> wc(stage_cfgs, stage_cfgs + n_stages);
        wc[kWarmSkip].body_pose_weight *= 0.15f;
        const int rc = make_loss_params(ctx, &wc[kWarmSkip], &wlps[kWarmSkip]);
        if (rc) return rc;
        if (!ctx->stage_rng) {
            const int rc2 = dev_alloc(ctx, &ctx->stage_rng, (size_t)B * 2);
            if (rc2) return rc2;
        }
    }
    const int H = opt_cfg->history_size > 0 ? opt_cfg->history_size : 100;
    auto regime = [&](const LossParams& lp) {
        if (resident_lbfgs_available_for(ctx, lp, H)) return 0;
        if (hybrid_available_for(ctx, lp)) return 1;
        return 2;
    };
    const int max_run = any_warm ? kMaxStages / 2 : kMaxStages;       // the table holds the cold and the warm slice of a run
    std::vector<int> rng;
    int i = 0;
    while (i < n_stages) {
        const int rg = regime(lps[i]);
        int j = i + 1;
        while (ctx->exec_mode != 2 && rg != 2 && j < n_stages && j - i < max_run && regime(lps[j]) == rg &&
               lps[j].sdf_grid == lps[i].sdf_grid && lps[j].sdf_all_faces == lps[i].sdf_all_faces)
            ++j;
        ctx->loss = lps[i];
        ctx->have_loss = true;
        int rc;
        if (!any_warm) {
            rc = run_stage(ctx, x_dev, final_loss_dev, opt_cfg, stats, st, 0, 1, nullptr, &lps[i], j - i);
        } else {
            if (rg == 2)
                return set_error(ctx, MVS_ERR_INVALID, "mvs_fit_seq: warm-started frames are not implemented in the batched "
                                                       "reference chain (exec mode 1 / a model the resident kernels do not take)");
            // table of this run: cold stages i .. j-1, then the warm slice max(i, 2) .. j-1
            std::vector<LossParams> tab(lps.begin() + i, lps.begin() + j);
            const int wi = i > kWarmSkip ? i : kWarmSkip;
            const int wbegin = (int)tab.size();
            for (int k = wi; k < j; ++k) tab.push_back(wlps[k]);
            const int wend = (int)tab.size();
            rng.assign((size_t)B * 2, 0);
            bool inactive = false;
            for (int b = 0; b < B; ++b) {
                const bool wm = warm_host[b] != 0;
                rng[2 * b] = wm ? wbegin : 0;
                rng[2 * b + 1] = wm ? wend : j - i;
                inactive |= wm && wbegin == wend;
            }
            MVS_CUDA_OK(ctx, cudaMemcpyAsync(ctx->stage_rng, rng.data(), rng.size() * sizeof(int), cudaMemcpyHostToDevice, st));
            MVS_CUDA_OK(ctx, cudaStreamSynchronize(st));           // rng is reused by the next run
            rc = run_stage(ctx, x_dev, final_loss_dev, opt_cfg, stats, st, 0, 1, nullptr, tab.data(), (int)tab.size(),
                           reinterpret_cast<const int2*>(ctx->stage_rng), inactive);
        }
        if (rc) return rc;
        i = j;
    }
    ctx->loss = lps[n_stages - 1];
    return MVS_OK;
}

}  // namespace mvs

using namespace mvs;

extern "C" {

int mvs_lbfgs_run(mvs_ctx* ctx, float* params_dev, float* final_loss_dev, const mvs_lbfgs_config* cfg,
                  mvs_lbfgs_stats* stats, void* stream) {
    if (!ctx) return set_error(nullptr, MVS_ERR_INVALID, "ctx is NULL");
    if (!(ctx->have_model && ctx->have_cams && ctx->have_kp && ctx->have_loss && ctx->ws.B > 0))
        return set_error(ctx, MVS_ERR_INVALID, "mvs_lbfgs_run: model, cameras, batch, keypoints and loss config must be set first");
    if (!params_dev || !cfg) return set_error(ctx, MVS_ERR_INVALID, "mvs_lbfgs_run: NULL argument");
    MVS_CUDA_OK(ctx, cudaSetDevice(ctx->device));
    if (stats) memset(stats, 0, sizeof(*stats));
    return run_stage(ctx, params_dev, final_loss_dev, cfg, stats, (cudaStream_t)stream);
}

int mvs_lbfgs_step(mvs_ctx* ctx, float* params_dev, float* loss_dev, float* last_grad_dev, const mvs_lbfgs_config* cfg,
                   int reset, mvs_lbfgs_stats* stats, void* stream) {
    if (!ctx) return set_error(nullptr, MVS_ERR_INVALID, "ctx is NULL");
    if (!(ctx->have_model && ctx->have_cams && ctx->have_kp && ctx->have_loss && ctx->ws.B > 0))
        return set_error(ctx, MVS_ERR_INVALID, "mvs_lbfgs_step: model, cameras, batch, keypoints and loss config must be set first");
    if (!params_dev || !cfg) return set_error(ctx, MVS_ERR_INVALID, "mvs_lbfgs_step: NULL argument");
    if (!reset && !ctx->lbfgs) return set_error(ctx, MVS_ERR_INVALID, "mvs_lbfgs_step: reset=0 before any step");
    MVS_CUDA_OK(ctx, cudaSetDevice(ctx->device));
    if (stats) memset(stats, 0, sizeof(*stats));
    return run_stage(ctx, params_dev, loss_dev, cfg, stats, (cudaStream_t)stream, 1, reset ? 1 : 0, last_grad_dev);
}

int mvs_fit_seq(mvs_ctx* ctx, float* params_dev, int n_stages, const mvs_loss_config* stage_cfgs, const mvs_lbfgs_config* opt_cfg,
                const unsigned char* warm_host, float* final_loss_dev, mvs_lbfgs_stats* stats, void* stream) {
    if (!ctx) return set_error(nullptr, MVS_ERR_INVALID, "ctx is NULL");
    if (!(ctx->have_model && ctx->have_cams && ctx->have_kp && ctx->ws.B > 0))
        return set_error(ctx, MVS_ERR_INVALID, "mvs_fit_seq: model, cameras, batch and keypoints must be set first");
    if (!params_dev || n_stages <= 0 || !stage_cfgs || !opt_cfg) return set_error(ctx, MVS_ERR_INVALID, "mvs_fit_seq: NULL / empty argument");
    MVS_CUDA_OK(ctx, cudaSetDevice(ctx->device));
    if (stats) memset(stats, 0, sizeof(*stats));
    return run_fit(ctx, params_dev, n_stages, stage_cfgs, opt_cfg, final_loss_dev, stats, (cudaStream_t)stream, warm_host);
}

int mvs_fit(mvs_ctx* ctx, float* params_dev, int n_stages, const mvs_loss_config* stage_cfgs, const mvs_lbfgs_config* opt_cfg,
            float* final_loss_dev, mvs_lbfgs_stats* stats, void* stream) {
    if (!ctx) return set_error(nullptr, MVS_ERR_INVALID, "ctx is NULL");
    if (!(ctx->have_model && ctx->have_cams && ctx->have_kp && ctx->ws.B > 0))
        return set_error(ctx, MVS_ERR_INVALID, "mvs_fit: model, cameras, batch and keypoints must be set first");
    if (!params_dev || n_stages <= 0 || !stage_cfgs || !opt_cfg) return set_error(ctx, MVS_ERR_INVALID, "mvs_fit: NULL / empty argument");
    MVS_CUDA_OK(ctx, cudaSetDevice(ctx->device));
    if (stats) memset(stats, 0, sizeof(*stats));
    return run_fit(ctx, params_dev, n_stages, stage_cfgs, opt_cfg, final_loss_dev, stats, (cudaStream_t)stream);
}

int mvs_fit_host(mvs_ctx* ctx, float* params_host, const float* gt_uv_host, const float* conf_host,
                 const float* joint_weights_host, int n_stages, const mvs_loss_config* stage_cfgs,
                 const mvs_lbfgs_config* opt_cfg, float* final_loss_host, mvs_lbfgs_stats* stats, void* stream) {
    if (!ctx) return set_error(nullptr, MVS_ERR_INVALID, "ctx is NULL");
    if (!(ctx->have_model && ctx->have_cams && ctx->ws.B > 0))
        return set_error(ctx, MVS_ERR_INVALID, "mvs_fit_host: model, cameras and batch must be set first");
    if (!params_host || !gt_uv_host || !conf_host || !joint_weights_host || n_stages <= 0 || !stage_cfgs || !opt_cfg)
        return set_error(ctx, MVS_ERR_INVALID, "mvs_fit_host: NULL / empty argument");
    MVS_CUDA_OK(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = (cudaStream_t)stream;
    const int B = ctx->ws.B;
    int rc = mvs_set_keypoints(ctx, gt_uv_host, conf_host, joint_weights_host, 0, stream);
    if (rc) return rc;
    {
        const int H = opt_cfg->history_size > 0 ? opt_cfg->history_size : 100;
        if (H > 128) return set_error(ctx, MVS_ERR_INVALID, "mvs_fit_host: history_size must be <= 128");
        rc = ensure_state(ctx, H);
        if (rc) return rc;
    }
    LbfgsState& S = *static_cast<LbfgsState*>(ctx->lbfgs);
    float* x = S.x_fit;                              // [B][86] device copy of the parameters
    MVS_CUDA_OK(ctx, cudaMemcpyAsync(x, params_host, (size_t)B * kParams * sizeof(float), cudaMemcpyHostToDevice, st));
    if (stats) memset(stats, 0, sizeof(*stats));
    rc = run_fit(ctx, x, n_stages, stage_cfgs, opt_cfg, S.final_fit, stats, st);
    if (rc) return rc;
    MVS_CUDA_OK(ctx, cudaMemcpyAsync(params_host, x, (size_t)B * kParams * sizeof(float), cudaMemcpyDeviceToHost, st));
    if (final_loss_host)
        MVS_CUDA_OK(ctx, cudaMemcpyAsync(final_loss_host, S.final_fit, (size_t)B * sizeof(float), cudaMemcpyDeviceToHost, st));
    MVS_CUDA_OK(ctx, cudaStreamSynchronize(st));
    return MVS_OK;
}

}  // extern "C"
