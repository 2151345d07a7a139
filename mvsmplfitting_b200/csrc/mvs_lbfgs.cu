// Batched, device-resident L-BFGS with strong-Wolfe cubic line search: one independent
// optimisation problem per frame, advanced as a per-frame state machine between batched
// closure evaluations.  Replaces (reference paths under code/):
//   optimizers/lbfgs_ls.py:11-36   _cubic_interpolate
//   optimizers/lbfgs_ls.py:39-167  _strong_Wolfe
//   optimizers/lbfgs_ls.py:256-445 LBFGS.step   (history 100, persistent state across step() calls)
//   utils/fitting.py:71-142        FittingMonitor.run_fitting (NaN/Inf guard, ftol, gtol)
//
// The reference runs this loop in Python with a blocking float(closure()) per evaluation
// (lbfgs_ls.py:251,281).  Here no scalar leaves the GPU.  stage_regime picks one of three execution regimes per
// group of stages (DESIGN.md section 4):
//   frame-resident   one CTA per frame runs closure + state machine for ALL stages of the group inside ONE launch
//                    (mvs_resident.cu: lbfgs_resident_kernel)
//   dense rounds     SDF term on: per round posedirs_gemm_tc -> skin -> sdf_setup (above 4 frames) -> sdf_fused ->
//                    frame_step; finished frames are compacted out every 8 rounds; the host reads the active count
//                    one chunk late (the next chunk is already enqueued) and only uses it to size grids and to stop
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
#include <functional>
#include <memory>
#include "mvs_internal.cuh"
#include "mvs_lbfgs_core.cuh"

namespace mvs {

// Start of frame b's run, one warp; x = its parameter row.  reset != 0: fresh optimiser (new stage).  reset == 0: next
// step() of the same optimiser: history, d, t, H_diag, prev_flat_grad, prev_loss and n_iter persist
// (lbfgs_ls.py:292-300,436-443).
__device__ __forceinline__ void init_frame_state(const LbfgsState& S, const float* __restrict__ x, int b, int reset, int nstages,
                                                 const int2* __restrict__ stage_rng, int lane) {
    VLOOP(i) S.x_eval[(size_t)b * kParams + i] = x[i];
    if (lane == 0) {
        FrameScalars s;
        if (reset) {                                        // this frame's slice of the stage table (mvs_fit_seq)
            s = fresh_frame_scalars(stage_rng ? stage_rng[b] : make_int2(0, nstages));
        } else {
            s = S.sc[b];
            s.outer_n = 0; s.have_prev = 0; s.nan_flag = 0; s.iters = 0; s.evals = 0;
            s.phase = PH_STEP_ENTRY;
            s.final_loss = __int_as_float(0x7fc00000);
        }
        S.sc[b] = s;
    }
}

__global__ void lbfgs_init_kernel(LbfgsState S, const float* __restrict__ params, int B, int reset, int nstages,
                                  const int2* __restrict__ stage_rng) {
    const int b = blockIdx.x;
    if (b >= B) return;
    init_frame_state(S, params + (size_t)b * kParams, b, reset, nstages, stage_rng, threadIdx.x);
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

__global__ void lbfgs_finalize_kernel(const FrameScalars* __restrict__ sc, int B, float* __restrict__ final_loss,
                                      long long* __restrict__ totals, int max_evals_as_rounds) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const FrameScalars s = sc[b];
    if (final_loss) final_loss[b] = s.final_loss;
    add_frame_totals(totals, s);
    if (max_evals_as_rounds) atomicMax((unsigned long long*)&totals[3], (unsigned long long)s.evals);
}

__global__ void iota2_kernel(int* p, int n, int* na) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = i;
    if (i == 0) *na = n;
}

// mvs_fit_stream / mvs_fit_seq_stream (DESIGN.md section 4): the context's B slots are lanes, each holding one frame of the
// call's F frames
struct StreamState {
    DevBuf<FrameScalars> sc;            // frame scalars of the frame-resident groups (one per frame of the stream)
    int* lane_frame = nullptr;          // [B] frame held by each lane of a dense group, -1: none
    long long* lane_start = nullptr;    // [B] round of the group in which the lane's frame started
    float* lane_params = nullptr;       // [B][86] the lanes' parameters (what params_dev is to mvs_fit)
    int* queue = nullptr;               // [1] next queue entry to enter a lane
    long long* end_round = nullptr;     // [1] max over retired frames of start round + evaluations: the rounds the group ran
    int* host = nullptr;                // pinned [2]: queue position of the two chunks in flight (next to their active counts)
};

// A dense run over the lanes, fed from a queue.  A frame stream is a sequence stream in which every sequence is one frame
// long: its frames have no successor, and queue entry k is frame k.
struct LaneArgs {
    int F, B, K;
    int n_queue;                        // queue entries: F (frame stream) or q.n_act (sequences of this pass)
    float* params;                      // [F][86] the call's parameters, in / out
    float* final_loss;                  // [F] or NULL
    const float *gt_uv, *conf;          // [V][F][K][2], [V][F][K]
    const float *j3d_xyz, *j3d_conf;    // [F][K][3], [F][K]; NULL: 3-D term off
    const Rig* rigs;                    // the context's rig table
    const int* rig;                     // [F] rig of each frame; NULL: every frame has rig 0
    float *ws_gt_uv, *ws_conf, *ws_j3d_xyz, *ws_j3d_conf;     // the lanes' rows, read by the dense kernels
    int* ws_rig;                        // [B] the rig of each lane's frame (with rig)
    int* lane_frame; long long* lane_start; float* lane_params; int* queue; long long* end_round;
    int* pose_valid;
    SeqChain q;                         // the sequences, queued by q.act; q.off == NULL: a frame stream (q.cold: its stage table)
    int* lane_seq;                      // [B] sequence of each lane's frame (sequence stream)
    float* anchor;                      // [B][86] the lanes' anchor rows (temporal term of a sequence stream), NULL: term off
};

// What follows a lane's finished frame `old` in the lane: its successor in the same sequence -- warm from the frame's
// fitted row when the frame's loss is <= reinit_loss, else cold -- or -1 when the lane is freed: a frame stream's frames have
// no successor, and a sequence that ends or parks a cold successor gives its lane up.
__device__ __forceinline__ int lane_successor(const LaneArgs& a, int l, int old, float loss, int flush, bool& warm) {
    warm = false;
    if (!a.q.off) return -1;
    const int sq = a.lane_seq[l], nx = old + 1;
    const bool more = !flush && nx < a.q.off[sq + 1];
    warm = more && loss <= a.q.reinit_loss;                         // NaN is not
    if (warm || (more && !a.q.park)) return nx;
    a.q.cur[sq] = more ? nx : -1;
    return -1;
}

// The frame that queue entry k brings into lane l: frame k of a frame stream, the pending frame of sequence q.act[k] otherwise
__device__ __forceinline__ int queued_frame(const LaneArgs& a, int l, int k) {
    if (!a.q.off) return k;
    const int sq = a.q.act[k];
    a.lane_seq[l] = sq;
    return a.q.cur[sq];
}

// Runs just before lbfgs_compact_kernel at every compaction point of a dense run over lanes (and once before the run's first
// round).  Every lane whose frame is done hands the frame's parameters, final loss and counts back to the call and takes the
// frame's successor in place (a lane that continues stays active).  The freed lanes then take the next queue entries in
// ascending lane order (ballot + prefix sum: no atomics decide which lane gets which frame), so freed lanes only take from
// the queue and the host's na_bound rule holds.  Every frame that enters a lane brings its rig index, the detections of its
// rig's views and, with the 3-D term on, its 3-D targets into the lane's rows, and starts as lbfgs_init_kernel starts a frame of mvs_fit, so that its bits do not
// depend on the lane or on when it entered.  round: rounds of the run so far (the new frames' first round).  flush != 0: hand
// back every frame still in a lane, take none.
__global__ void __launch_bounds__(1024) lane_refill_kernel(LbfgsState S, LaneArgs a, long long round, int flush) {
    __shared__ int wsum[32];
    __shared__ int qbase;
    __shared__ int s_old[1024], s_new[1024];
    __shared__ unsigned char s_warm[1024];
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    if (tid == 0) qbase = *a.queue;
    __syncthreads();
    for (int l0 = 0; l0 < a.B; l0 += 1024) {
        const int l = l0 + tid;
        int old = -1, fresh = -1;
        bool fin = false, freed = false, warm = false;
        if (l < a.B) {
            old = a.lane_frame[l];
            fin = old < 0 || flush || S.sc[l].phase == PH_DONE;
            if (old >= 0 && fin) {                        // the frame's totals, as lbfgs_finalize_kernel counts them
                const FrameScalars& s = S.sc[l];
                if (a.final_loss) a.final_loss[old] = s.final_loss;
                add_frame_totals(S.totals, s);
                atomicMax((unsigned long long*)a.end_round, (unsigned long long)(a.lane_start[l] + s.evals));
                fresh = lane_successor(a, l, old, s.final_loss, flush, warm);
                freed = fresh < 0;
            } else {
                freed = fin;
                old = -1;
            }
        }
        const unsigned m = __ballot_sync(0xffffffffu, freed);
        const int pre = __popc(m & ((1u << lane) - 1));
        if (lane == 0) wsum[wid] = __popc(m);
        __syncthreads();
        if (freed) {
            int k = qbase + pre;
            for (int w = 0; w < wid; ++w) k += wsum[w];
            if (!flush && k < a.n_queue) fresh = queued_frame(a, l, k);
        }
        if (fin) {
            a.lane_frame[l] = fresh;
            if (fresh >= 0) a.lane_start[l] = round;
            else S.sc[l].phase = PH_DONE;                 // an empty lane stays out of the active list
        }
        s_old[tid] = old;
        s_new[tid] = fresh;
        s_warm[tid] = warm ? 1 : 0;
        __syncthreads();
        if (tid == 0 && !flush) {
            int tot = qbase;
            for (int w = 0; w < 32; ++w) tot += wsum[w];
            qbase = tot < a.n_queue ? tot : a.n_queue;
        }
        // parameters out and in, the new frame's detections into the lane's rows: one warp per lane
        for (int j = wid; j < 1024 && l0 + j < a.B; j += 32) {
            const int ln = l0 + j, fo = s_old[j], fn = s_new[j];
            const bool wm = s_warm[j] != 0;
            float* xl = a.lane_params + (size_t)ln * kParams;
            if (fo >= 0) {
                VLOOP(i) a.params[(size_t)fo * kParams + i] = xl[i];
            }
            if (fn < 0) continue;
            VLOOP(i) {                                    // a warm frame keeps the fitted row (but its own body pose, keep_pose)
                if (wm && a.anchor) a.anchor[(size_t)ln * kParams + i] = xl[i];      // its anchor: the fitted row as returned
                if (!wm || (a.q.keep_pose && i >= kOffPose && i < kOffTransl)) xl[i] = a.params[(size_t)fn * kParams + i];
            }
            const int K = a.K, rg = a.rig ? a.rig[fn] : 0;
            if (a.rig && lane == 0) a.ws_rig[ln] = rg;
            const int nv = a.rigs[rg].num_views;          // rows v >= nv of the frame are not read
            for (int v = 0; v < nv; ++v) {
                const size_t dst = (size_t)v * a.B + ln, src = (size_t)v * a.F + fn;
                for (int k = lane; k < 2 * K; k += 32) a.ws_gt_uv[dst * 2 * K + k] = a.gt_uv[src * 2 * K + k];
                for (int k = lane; k < K; k += 32) a.ws_conf[dst * K + k] = a.conf[src * K + k];
            }
            if (a.j3d_xyz) {
                for (int k = lane; k < 3 * K; k += 32) a.ws_j3d_xyz[(size_t)ln * 3 * K + k] = a.j3d_xyz[(size_t)fn * 3 * K + k];
                for (int k = lane; k < K; k += 32) a.ws_j3d_conf[(size_t)ln * K + k] = a.j3d_conf[(size_t)fn * K + k];
            }
            __syncwarp();
            VLOOP(i) S.x_eval[(size_t)ln * kParams + i] = xl[i];
            if (lane == 0) {
                S.sc[ln] = fresh_frame_scalars(wm ? a.q.warm : a.q.cold);     // the frame's slice of the run's stage table
                a.pose_valid[ln] = 0;                     // the lane's pose cache belongs to its previous frame
            }
        }
        __syncthreads();
    }
    if (tid == 0) *a.queue = qbase;
}

// rows [0, n) of dst [n][86] = w (the temporal weight: the same for every frame of a call)
struct Row86 { float v[kParams]; };
__global__ void fill_rows_kernel(float* __restrict__ dst, Row86 w, int n) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < (size_t)n * kParams) dst[i] = w.v[i % kParams];
}

// rows idx[0 .. n) of full [V][n_full][L] <-> packed [V][n][L]; to_full = 0 gathers, 1 scatters.  With rig (per-view rows of
// frames with rigs rig[n_full]): view v of a frame whose rig has no view v is skipped.
template <class T>
__global__ void copy_rows_kernel(T* __restrict__ packed, T* __restrict__ full, const int* __restrict__ idx, int n, int n_full,
                                 int L, int to_full, const Rig* __restrict__ rigs = nullptr, const int* __restrict__ rig = nullptr) {
    const int i = blockIdx.x, v = blockIdx.y;
    if (rig && v >= rigs[rig[idx[i]]].num_views) return;
    T* p = packed + ((size_t)v * n + i) * L;
    T* g = full + ((size_t)v * n_full + idx[i]) * L;
    for (int k = threadIdx.x; k < L; k += blockDim.x) {
        if (to_full) g[k] = p[k];
        else p[k] = g[k];
    }
}

// The host resources of the state objects; their device arrays belong to ctx->allocs
static void release(LbfgsState* S) {
    if (!S) return;
    cudaFreeHost(S->na_host);
    cudaFreeHost(S->lp_tab_host);
    for (cudaEvent_t e : S->na_event)
        if (e) cudaEventDestroy(e);
    delete S;
}
static void release(StreamState* ss) {
    if (!ss) return;
    cudaFreeHost(ss->host);
    delete ss;
}
struct ReleaseState { template <class T> void operator()(T* p) const { release(p); } };

static int ensure_state(mvs_ctx* ctx, int H) {
    const int B = ctx->ws.B;
    if (ctx->lbfgs && ctx->lbfgs->B == B && ctx->lbfgs->H == H) return MVS_OK;
    if (ctx->lbfgs)
        return set_error(ctx, MVS_ERR_INVALID, "mvs_lbfgs_run: history_size changed between calls (%d -> %d)", ctx->lbfgs->H, H);
    std::unique_ptr<LbfgsState, ReleaseState> S(new LbfgsState());
    S->B = B; S->H = H;
    int rc;
    const size_t V = (size_t)B * kParams;
    if ((rc = dev_alloc(ctx, &S->g, V)) || (rc = dev_alloc(ctx, &S->d, V)) || (rc = dev_alloc(ctx, &S->prev_g, V)) ||
        (rc = dev_alloc(ctx, &S->x_init, V)) || (rc = dev_alloc(ctx, &S->g_prev, V)) || (rc = dev_alloc(ctx, &S->bg, 2 * V)) ||
        (rc = dev_alloc(ctx, &S->hist_y, V * H)) || (rc = dev_alloc(ctx, &S->hist_s, V * H)) ||
        (rc = dev_alloc(ctx, &S->ro, (size_t)B * H)) || (rc = dev_alloc(ctx, &S->gram, (size_t)B * kGramFloats)) ||
        (rc = dev_alloc(ctx, &S->x_eval, V)) || (rc = dev_alloc(ctx, &S->loss_eval, B)) || (rc = dev_alloc(ctx, &S->g_eval, V)) ||
        (rc = dev_alloc(ctx, &S->x_fit, V)) || (rc = dev_alloc(ctx, &S->final_fit, B)) || (rc = dev_alloc(ctx, &S->sc, B)) ||
        (rc = dev_alloc(ctx, &S->totals, 4)) || (rc = dev_alloc(ctx, &S->lp_tab, kMaxStages)))
        return rc;
    MVS_CUDA_OK(ctx, cudaMallocHost(&S->na_host, 8 * sizeof(long long)));
    MVS_CUDA_OK(ctx, cudaMallocHost(&S->lp_tab_host, kMaxStages * sizeof(LossParams)));
    // blocking sync: the host thread sleeps while it waits for a chunk of dense rounds (several contexts are driven by as many
    // host threads; spinning ones would compete with the threads that have launches to enqueue)
    for (cudaEvent_t& e : S->na_event)
        MVS_CUDA_OK(ctx, cudaEventCreateWithFlags(&e, cudaEventDisableTiming | cudaEventBlockingSync));
    ctx->lbfgs = S.release();
    return MVS_OK;
}

// What a run does beyond its optimiser configuration.  The defaults are one mvs_lbfgs_run: a fresh optimiser for the stage
// in ctx->loss, every frame active.
struct RunOpts {
    bool step = false;                // one LBFGS.step() per call, state kept in the context (mvs_lbfgs_step)
    bool reset = true;                // false: the next step() of the same optimiser (lbfgs_init_kernel)
    float* last_grad = nullptr;       // [B][86] gradient at the last evaluated point
    const LossParams* lps = nullptr;  // stage table lps[0 .. nst); nullptr: ctx->loss alone
    int nst = 1;
    const int2* stage_rng = nullptr;  // [B] per-frame slice of the stage table (mvs_fit_seq); nullptr: all of it
    bool some_inactive = false;       // some frame has no stage in this run
};

// How a run evaluates the stage lp (step: mvs_lbfgs_step).  The frame-resident optimiser holds histories up to 100 and runs
// whole stages; the dense rounds serve the SDF term, in step mode only with use_vposer = 2, which the batched chain lacks.
static Regime stage_regime(const mvs_ctx* ctx, const LossParams& lp, int history, bool step) {
    if (ctx->exec_mode == 1 || !resident_supported(ctx)) return kBatched;
    if (!sdf_term_on(lp)) return !step && history <= 100 ? kResident : kBatched;
    return !step || lp.use_vposer == 2 ? kDense : kBatched;
}

static bool resident_closure_applies(const mvs_ctx* ctx, bool want_verts) {
    return !want_verts && !sdf_term_on(ctx->loss) && ctx->exec_mode != 1 && resident_supported(ctx);
}

static int history_size(const mvs_lbfgs_config* c) { return c->history_size > 0 ? c->history_size : 100; }

// Shared set-up of a run: optimiser configuration, state for history size H, zeroed totals, stage table on the device
static int begin_run(mvs_ctx* ctx, const mvs_lbfgs_config* c, bool step, const LossParams* lps, int nst, LbfgsCfg* cfg,
                     cudaStream_t st) {
    const int H = history_size(c);
    if (H > 128) return set_error(ctx, MVS_ERR_INVALID, "mvs_lbfgs_run: history_size must be <= 128");
    int rc = ensure_state(ctx, H);
    if (rc) return rc;
    LbfgsState& S = *ctx->lbfgs;
    cfg->max_outer = c->max_outer > 0 ? c->max_outer : 30;
    cfg->max_iter = c->max_iter > 0 ? c->max_iter : 30;
    cfg->max_eval = c->max_eval > 0 ? c->max_eval : cfg->max_iter * 5 / 4;
    cfg->history = H;
    cfg->max_ls = 25;                                           // _strong_Wolfe default (lbfgs_ls.py:41)
    cfg->step_mode = step ? 1 : 0;
    cfg->lr = c->lr > 0.f ? c->lr : 1.f;
    cfg->tol_grad = c->tolerance_grad; cfg->tol_change = c->tolerance_change;
    cfg->ftol = (double)c->ftol; cfg->gtol = (double)c->gtol;
    MVS_CUDA_OK(ctx, cudaMemsetAsync(S.totals, 0, 4 * sizeof(long long), st));
    if (nst > kMaxStages) return set_error(ctx, MVS_ERR_INVALID, "at most %d stages per run", kMaxStages);
    // stage table for the multi-stage kernels (the previous run ended with a stream synchronisation, so the pinned
    // staging copy is free)
    for (int i = 0; i < nst; ++i) S.lp_tab_host[i] = lps[i];
    MVS_CUDA_OK(ctx, cudaMemcpyAsync(S.lp_tab, S.lp_tab_host, (size_t)nst * sizeof(LossParams), cudaMemcpyHostToDevice, st));
    return MVS_OK;
}

// Start of a dense run: pose forward of every active slot, frame_step's pose cache invalidated
static int dense_begin(mvs_ctx* ctx, const LbfgsState& S, int nst, cudaStream_t st) {
    const int rc = launch_frame_fwd_dense(ctx, S.x_eval, S, nst, st);
    return rc ? rc : frame_step_begin_run(ctx, st);
}

// One dense round: pose blend shapes of the active frames (wgmma GEMM), skinning + box partials, each frame's SDF set-up
// (sdf_setup, one warp per frame; at <= 4 frames the tail of skin_small instead), the SDF term with the adjoint of its
// (short) vertex list, and the per-frame closure adjoint + optimiser step + next pose forward
static int dense_round(mvs_ctx* ctx, float* params_dev, const LbfgsState& S, const LbfgsCfg& cfg, int nst, cudaStream_t st) {
    int rc;
    if ((rc = launch_vertex_fwd_tc(ctx, st, false, true))) return rc;
    if ((rc = launch_sdf_fused(ctx, st))) return rc;
    return launch_frame_step(ctx, params_dev, S, cfg, nst, st);
}

// Dense regime (SDF term on): rounds of dense_round until no frame is active.  Finished frames are compacted out once per
// chunk of rounds.  la (mvs_fit_stream, mvs_fit_seq_stream): the finished frames' lanes are refilled from la's queue just
// before each compaction.
static int run_dense(mvs_ctx* ctx, float* params_dev, const LbfgsCfg& cfg, int nst, cudaStream_t st,
                     const LaneArgs* la = nullptr) {
    LbfgsState& S = *ctx->lbfgs;
    Workspace& w = ctx->ws;
    const int B = w.B;
    const int chunk = 8;
    // (a lane of a sequence stream may carry every frame of the call)
    const long long frames_per_lane = !la ? 1 : la->q.off ? la->F + 1 : (la->F + B - 1) / B + 1;
    const long long max_rounds = stage_eval_cap(cfg) * nst * frames_per_lane;
    long long rounds = 0;
    int na_host = B;
    static const bool trace_na = getenv("MVS_TRACE_NA") != nullptr;       // debugging aid: active-list size per chunk
    // debugging aid: how long the host thread waited for the GPU inside the round loop (close to 0 = the GPU waits for the host)
    static const bool trace_host = getenv("MVS_TRACE_HOST") != nullptr;
    double blocked_us = 0.0;
    const auto loop_t0 = std::chrono::steady_clock::now();
    int rc = dense_begin(ctx, S, nst, st);
    if (rc) return rc;
    // The host only needs the active count to know when to stop, so chunk k+1 is enqueued BEFORE the count of
    // chunk k is awaited (kernels exit at once when the list is empty): the GPU never idles on the host round trip.
    int* na_slots = reinterpret_cast<int*>(S.na_host);           // [0], [1]: two chunks in flight
    int* queue_slots = la ? ctx->fstream->host : nullptr;         // the same chunks' queue positions
    bool drained = la == nullptr;                                 // the host has seen the queue empty
    int pending = -1;                                             // chunk whose count has not been read yet
    long long chunk_idx = 0;
    w.na_bound = B;                                               // grids shrink with the (lagging) host view of the count
    while (rounds < max_rounds) {
        for (int r = 0; r < chunk; ++r) {
            if ((rc = dense_round(ctx, params_dev, S, cfg, nst, st))) return rc;
            ++rounds;
        }
        if (la) MVS_LAUNCH(ctx, KID_LBFGS_COMPACT, st, lane_refill_kernel<<<1, 1024, 0, st>>>(S, *la, rounds, 0));
        // compaction changes slot -> frame, so the surviving frames' Phi / transforms are rebuilt for their new slots
        MVS_LAUNCH(ctx, KID_LBFGS_COMPACT, st, lbfgs_compact_kernel<<<1, 1024, 0, st>>>(S, B, w.fidx, w.na));
        if ((rc = launch_frame_fwd_dense(ctx, S.x_eval, S, nst, st))) return rc;
        const int cur = (int)(chunk_idx & 1);
        MVS_CUDA_OK(ctx, cudaMemcpyAsync(&na_slots[cur], w.na, sizeof(int), cudaMemcpyDeviceToHost, st));
        if (la) MVS_CUDA_OK(ctx, cudaMemcpyAsync(&queue_slots[cur], la->queue, sizeof(int), cudaMemcpyDeviceToHost, st));
        MVS_CUDA_OK(ctx, cudaEventRecord(S.na_event[cur], st));
        if (pending >= 0) {
            const auto tb0 = std::chrono::steady_clock::now();
            MVS_CUDA_OK(ctx, cudaEventSynchronize(S.na_event[pending]));
            if (trace_host) blocked_us += std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - tb0).count();
            na_host = na_slots[pending];
            if (!drained) drained = queue_slots[pending] >= la->n_queue;
            if (trace_na) fprintf(stderr, "[mvs] dense regime: chunk %lld, active frames %d\n", chunk_idx - 1, na_host);
            if (na_host <= 0) break;                              // (a refill leaves no lane idle while frames are queued)
            // Without refills the list only shrinks, so the count is an upper bound for every later round.  Refills add
            // frames back until the queue is empty: until the host has seen that, the grids keep all B slots.
            w.na_bound = drained ? na_host : B;
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
    return tc_check_error(ctx);
}

// Batched chain: the closure (frame-resident where it applies, launch_closure otherwise; closure: the caller's, which fills
// S.loss_eval / S.g_eval of the active slots) + lbfgs_advance_kernel + lbfgs_compact_kernel per round, the host reads the active
// count after every chunk of rounds
static int run_batched(mvs_ctx* ctx, float* params_dev, const LbfgsCfg& cfg, bool vp2, cudaStream_t st,
                       const std::function<int()>& closure = nullptr) {
    LbfgsState& S = *ctx->lbfgs;
    Workspace& w = ctx->ws;
    const int B = w.B;
    const int chunk = 8;
    const long long max_rounds = stage_eval_cap(cfg);
    long long rounds = 0;
    int na_host = B;
    const bool resident = resident_closure_applies(ctx, false);     // (not the dense-round closure: it restarts the optimiser)
    while (na_host > 0 && rounds < max_rounds) {
        for (int r = 0; r < chunk; ++r) {
            const int rc = closure ? closure()
                         : resident ? launch_closure_resident(ctx, S.x_eval, S.loss_eval, S.g_eval, nullptr, nullptr, st)
                         : launch_closure(ctx, S.x_eval, S.loss_eval, S.g_eval, nullptr, nullptr, nullptr, st);
            if (rc) return rc;
            MVS_LAUNCH(ctx, KID_LBFGS_ADVANCE, st, lbfgs_advance_kernel<<<B, 32, 0, st>>>(S, cfg, params_dev, w.fidx, w.na, vp2 ? 32 : kOffTransl - kOffPose));
            MVS_LAUNCH(ctx, KID_LBFGS_COMPACT, st, lbfgs_compact_kernel<<<1, 1024, 0, st>>>(S, B, w.fidx, w.na));
            ++rounds;
        }
        MVS_CUDA_OK(ctx, cudaMemcpyAsync(S.na_host, w.na, sizeof(int), cudaMemcpyDeviceToHost, st));
        MVS_CUDA_OK(ctx, cudaStreamSynchronize(st));
        na_host = *S.na_host;
    }
    return MVS_OK;
}

// End of every run: waits for st, then adds the run's totals (S.totals: iterations, evaluations, NaN / Inf stops) and its
// rounds (S.totals[3], or *rounds_dev when given) to stats, and to the dense counters for a dense run
static int read_totals(mvs_ctx* ctx, const long long* rounds_dev, bool dense, mvs_lbfgs_stats* stats, cudaStream_t st) {
    LbfgsState& S = *ctx->lbfgs;
    long long* th = reinterpret_cast<long long*>(S.na_host) + 1;
    MVS_CUDA_OK(ctx, cudaMemcpyAsync(th, S.totals, 4 * sizeof(long long), cudaMemcpyDeviceToHost, st));
    if (rounds_dev) MVS_CUDA_OK(ctx, cudaMemcpyAsync(th + 3, rounds_dev, sizeof(long long), cudaMemcpyDeviceToHost, st));
    MVS_CUDA_OK(ctx, cudaStreamSynchronize(st));
    MVS_CUDA_OK(ctx, cudaGetLastError());
    if (!stats) return MVS_OK;
    stats->frame_iterations += th[0]; stats->frame_evals += th[1]; stats->frames_nan += (int)th[2];
    stats->rounds += (int)th[3];
    if (dense) { stats->dense_frame_evals += th[1]; stats->dense_rounds += (int)th[3]; }
    return MVS_OK;
}

// End of a run of regime rg over n frames whose scalars are sc: their final losses (final_loss_dev [n], or NULL), and the
// run's totals added to stats.  The dense and frame-resident regimes report the largest per-frame evaluation count (the
// critical path) as rounds.
static int finish_run(mvs_ctx* ctx, Regime rg, const FrameScalars* sc, int n, float* final_loss_dev, mvs_lbfgs_stats* stats,
                      cudaStream_t st) {
    MVS_LAUNCH(ctx, KID_MISC, st, lbfgs_finalize_kernel<<<(n + 255) / 256, 256, 0, st>>>(sc, n, final_loss_dev, ctx->lbfgs->totals,
                                                                                         rg != kBatched));
    return read_totals(ctx, nullptr, rg == kDense, stats, st);
}

// End of a round-based run (batched chain, dense rounds): the gradient at the last evaluated point, the context left usable
// for plain closures (full active list), then finish_run over the slots
static int end_run(mvs_ctx* ctx, Regime rg, float* final_loss_dev, float* last_grad_dev, mvs_lbfgs_stats* stats, cudaStream_t st) {
    LbfgsState& S = *ctx->lbfgs;
    Workspace& w = ctx->ws;
    const int B = w.B;
    if (last_grad_dev)
        MVS_CUDA_OK(ctx, cudaMemcpyAsync(last_grad_dev, S.g_eval, (size_t)B * kParams * sizeof(float), cudaMemcpyDeviceToDevice, st));
    MVS_LAUNCH(ctx, KID_MISC, st, iota2_kernel<<<(B + 255) / 256, 256, 0, st>>>(w.fidx, B, w.na));
    return finish_run(ctx, rg, S.sc, B, final_loss_dev, stats, st);
}

// Runs the stages o.lps[0 .. o.nst) (default: ctx->loss).  nst > 1 requires that all of them run in the same regime
// (frame-resident or dense rounds, see run_fit): every frame then walks through the stages at its own pace.
static int run_stage(mvs_ctx* ctx, float* params_dev, float* final_loss_dev, const mvs_lbfgs_config* c, mvs_lbfgs_stats* stats,
                     cudaStream_t st, const RunOpts& o) {
    const LossParams* lps = o.lps ? o.lps : &ctx->loss;
    const int nst = o.lps ? o.nst : 1;
    LbfgsCfg cfg;
    int rc = begin_run(ctx, c, o.step, lps, nst, &cfg, st);
    if (rc) return rc;
    LbfgsState& S = *ctx->lbfgs;
    Workspace& w = ctx->ws;
    const int B = w.B;
    const Regime rg = stage_regime(ctx, ctx->loss, cfg.history, o.step);
    if (rg == kResident) {
        // sparse regime: every frame runs its whole stage inside one CTA (mvs_resident.cu): one launch, no rounds; the kernel
        // writes the last gradient itself and leaves the active list alone
        const FrameInputs in{B, w.gt_uv, w.conf, w.joint_w, w.j3d_xyz, w.j3d_conf, ctx->slot_rigs};
        rc = launch_lbfgs_resident(ctx, params_dev, cfg, nst, in, S.sc, o.last_grad, o.stage_rng, st);
        return rc ? rc : finish_run(ctx, kResident, S.sc, B, final_loss_dev, stats, st);
    }
    // use_vposer = 2 (VPoser decode on the device) exists in the frame-resident closure and in the dense-regime kernels, not in
    // the SIMT reference chain.  mvs_lbfgs_step therefore runs its one step() per call through the dense rounds when the SDF
    // term is on, and through the frame-resident closure + lbfgs_advance_kernel otherwise.
    const bool vp2 = ctx->loss.use_vposer == 2;
    if (rg == kBatched && vp2 && !resident_closure_applies(ctx, false))
        return set_error(ctx, MVS_ERR_INVALID, "use_vposer = 2 (VPoser decode on the device) is not implemented in the batched "
                                               "reference chain (exec mode 1): use use_vposer = 1 there");
    MVS_LAUNCH(ctx, KID_MISC, st, iota2_kernel<<<(B + 255) / 256, 256, 0, st>>>(w.fidx, B, w.na));
    MVS_LAUNCH(ctx, KID_MISC, st, lbfgs_init_kernel<<<B, 32, 0, st>>>(S, params_dev, B, o.reset ? 1 : 0, nst, o.stage_rng));
    if (o.some_inactive)                                    // frames without a stage in this run leave the active list now
        MVS_LAUNCH(ctx, KID_LBFGS_COMPACT, st, lbfgs_compact_kernel<<<1, 1024, 0, st>>>(S, B, w.fidx, w.na));
    rc = rg == kDense ? run_dense(ctx, params_dev, cfg, nst, st) : run_batched(ctx, params_dev, cfg, vp2, st);
    return rc ? rc : end_run(ctx, rg, final_loss_dev, o.last_grad, stats, st);
}

// One closure evaluation through the dense-regime kernels (dense_round: posedirs_gemm_tc -> skin -> sdf_setup -> sdf_fused
// -> frame_step, with the optimiser step switched off): mvs_closure in exec mode 3.  Exists so that parity tests can compare the loss and every
// gradient segment of the kernels the optimiser actually runs with the SDF term on (DESIGN.md section 2).
static int dense_regime_closure(mvs_ctx* ctx, const float* x_dev, float* loss_dev, float* grad_dev, cudaStream_t st) {
    const int B = ctx->ws.B;
    int rc = ensure_state(ctx, ctx->lbfgs ? ctx->lbfgs->H : 100);
    if (rc) return rc;
    LbfgsState& S = *ctx->lbfgs;
    Workspace& w = ctx->ws;
    LbfgsCfg cfg{};
    cfg.max_outer = 1; cfg.max_iter = 1; cfg.max_eval = 1; cfg.history = S.H; cfg.max_ls = 25; cfg.step_mode = 2; cfg.lr = 1.f;
    S.lp_tab_host[0] = ctx->loss;
    MVS_CUDA_OK(ctx, cudaMemcpyAsync(S.lp_tab, S.lp_tab_host, sizeof(LossParams), cudaMemcpyHostToDevice, st));
    MVS_LAUNCH(ctx, KID_MISC, st, iota2_kernel<<<(B + 255) / 256, 256, 0, st>>>(w.fidx, B, w.na));
    MVS_LAUNCH(ctx, KID_MISC, st, lbfgs_init_kernel<<<B, 32, 0, st>>>(S, x_dev, B, 1, 1, nullptr));
    w.na_bound = B;
    if ((rc = dense_begin(ctx, S, 1, st))) return rc;
    if ((rc = dense_round(ctx, const_cast<float*>(x_dev) /* read only in this mode */, S, cfg, 1, st))) return rc;
    if (loss_dev) MVS_CUDA_OK(ctx, cudaMemcpyAsync(loss_dev, S.loss_eval, (size_t)B * sizeof(float), cudaMemcpyDeviceToDevice, st));
    if (grad_dev) MVS_CUDA_OK(ctx, cudaMemcpyAsync(grad_dev, S.g_eval, (size_t)B * kParams * sizeof(float), cudaMemcpyDeviceToDevice, st));
    MVS_CUDA_OK(ctx, cudaStreamSynchronize(st));         // the pinned stage table is reused by the next call
    if ((rc = tc_check_error(ctx))) return rc;
    MVS_CUDA_OK(ctx, cudaGetLastError());
    return MVS_OK;
}

// mvs_closure: the frame-resident closure where it applies; in exec mode 3, loss and gradient with the SDF term through the
// dense-round kernels the optimiser runs; the batched chain otherwise
int evaluate_closure(mvs_ctx* ctx, const float* x_dev, float* loss_dev, float* grad_dev, float* joints_dev, float* proj_dev,
                     float* verts_dev, cudaStream_t st) {
    if (resident_closure_applies(ctx, verts_dev != nullptr))
        return launch_closure_resident(ctx, x_dev, loss_dev, grad_dev, joints_dev, proj_dev, st);
    if (ctx->exec_mode == 3 && sdf_term_on(ctx->loss) && !joints_dev && !proj_dev && !verts_dev && resident_supported(ctx))
        return dense_regime_closure(ctx, x_dev, loss_dev, grad_dev, st);
    if (ctx->loss.use_vposer == 2)
        return set_error(ctx, MVS_ERR_INVALID, "use_vposer = 2 (VPoser decode on the device) is implemented in the "
                                               "frame-resident closure (no vertices, no SDF term, exec mode 0, 2 or 3) and in "
                                               "the dense-round closure of exec mode 3 (SDF term, loss and gradient) only");
    return launch_closure(ctx, x_dev, loss_dev, grad_dev, joints_dev, proj_dev, verts_dev, st);
}

// One past the last stage of the run that starts at stage i: the following stages of the same regime, SDF grid and face
// mode, at most max_run of them (one stage per run in exec mode 2 and in the batched chain)
static int stage_group_end(const mvs_ctx* ctx, const std::vector<LossParams>& lps, int i, int H, int max_run) {
    const Regime rg = stage_regime(ctx, lps[i], H, false);
    int j = i + 1;
    while (ctx->exec_mode != 2 && rg != kBatched && j < (int)lps.size() && j - i < max_run &&
           stage_regime(ctx, lps[j], H, false) == rg && lps[j].sdf_grid == lps[i].sdf_grid &&
           lps[j].sdf_all_faces == lps[i].sdf_all_faces)
        ++j;
    return j;
}

// warm-started frames (is_seq, non_linear_solver.py:157-162): no stage 0 and 1, stage 2 with 0.15 x body_pose_weight
constexpr int kWarmSkip = 2;

// The LossParams of a call's stages (at most 64; who names the entry point in the error).  j3d >= 0 sets the 3-D joint term
// on (1) or off (0) in every stage: a stream's own targets, never the context's.
static int stage_table(mvs_ctx* ctx, const char* who, int n_stages, const mvs_loss_config* cfgs, int j3d,
                       std::vector<LossParams>* lps) {
    if (n_stages > 64) return set_error(ctx, MVS_ERR_INVALID, "%s: at most 64 stages", who);
    lps->resize(n_stages);
    for (int i = 0; i < n_stages; ++i) {
        const int rc = make_loss_params(ctx, &cfgs[i], &(*lps)[i]);
        if (rc) return rc;
        if (j3d >= 0) (*lps)[i].j3d_on = j3d;
    }
    return MVS_OK;
}

// The warm-started frames' copy of a stage table: stage kWarmSkip with 0.15 x its body-pose weight.  temporal: every stage
// the warm frames run (kWarmSkip .. n-1) carries the anchor term, whose rows and weights the caller has set up.
static int warm_stage_table(mvs_ctx* ctx, const mvs_loss_config* cfgs, int j3d, const std::vector<LossParams>& lps,
                            std::vector<LossParams>* wlps, bool temporal = false) {
    *wlps = lps;
    mvs_loss_config wc = cfgs[kWarmSkip];
    wc.body_pose_weight *= 0.15f;
    const int rc = make_loss_params(ctx, &wc, &(*wlps)[kWarmSkip]);
    if (!rc && j3d >= 0) (*wlps)[kWarmSkip].j3d_on = j3d;
    if (temporal)
        for (size_t k = kWarmSkip; k < wlps->size(); ++k) (*wlps)[k].anchor_on = 1;
    return rc;
}

// The runs of a stream's stages, grouped as run_fit groups them (at most max_run stages each): ends[g] is one past run g's
// last stage.  A stage of the batched reference chain is refused: that chain has no stream.
static int stream_runs(mvs_ctx* ctx, const char* who, const std::vector<LossParams>& lps, int H, int max_run,
                       std::vector<int>* ends) {
    for (int i = 0; i < (int)lps.size(); i = ends->back()) {
        if (stage_regime(ctx, lps[i], H, false) == kBatched)
            return set_error(ctx, MVS_ERR_UNSUPPORTED, "%s: stage %d would run in the batched reference chain (exec mode 1, "
                                                       "history_size > 100 without the SDF term, or a model the frame-resident "
                                                       "and dense kernels do not take), which has no stream", who, i);
        ends->push_back(stage_group_end(ctx, lps, i, H, max_run));
    }
    return MVS_OK;
}

// The stage a run starts with becomes the context's loss config (what the kernels and a later mvs_lbfgs_run read)
static void use_stage(mvs_ctx* ctx, const LossParams& lp) {
    ctx->loss = lp;
    ctx->have_loss = true;
}

// Each slot's slice [rng[2b], rng[2b+1]) of the next run's stage table, in ctx->stage_rng.  Synchronises: rng is reused.
static int upload_stage_rng(mvs_ctx* ctx, const std::vector<int>& rng, cudaStream_t st) {
    int rc;
    if (!ctx->stage_rng && (rc = dev_alloc(ctx, &ctx->stage_rng, (size_t)ctx->ws.B))) return rc;
    MVS_CUDA_OK(ctx, cudaMemcpyAsync(ctx->stage_rng, rng.data(), rng.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    MVS_CUDA_OK(ctx, cudaStreamSynchronize(st));
    return MVS_OK;
}

// All stages of a fit (who: the entry point called).  Consecutive stages that run in the same regime are handed to ONE
// multi-stage run in which every frame changes stage on its own (frames are independent problems, so a frame that converged
// need not wait at the stage boundary for the slowest one; the per-frame arithmetic is the sequential schedule's).  exec_mode 2
// keeps the stage barrier (one run per stage).
// temporal (mvs_fit_seq_temporal): the warm frames' stages carry the anchor term of the rows the caller put in ws.anchor / anchor_w.
static int run_fit(mvs_ctx* ctx, const char* who, float* x_dev, int n_stages, const mvs_loss_config* stage_cfgs,
                   const mvs_lbfgs_config* opt_cfg, float* final_loss_dev, mvs_lbfgs_stats* stats, cudaStream_t st,
                   const unsigned char* warm_host = nullptr, bool temporal = false) {
    std::vector<LossParams> lps;
    int rc = stage_table(ctx, who, n_stages, stage_cfgs, -1, &lps);
    if (rc) return rc;
    const int B = ctx->ws.B;
    bool any_warm = false;
    if (warm_host)
        for (int b = 0; b < B; ++b) any_warm |= warm_host[b] != 0;
    if (any_warm && n_stages <= kWarmSkip)
        return set_error(ctx, MVS_ERR_INVALID, "%s: warm-started frames skip the first %d stages, %d given", who, kWarmSkip, n_stages);
    std::vector<LossParams> wlps;
    if (any_warm && (rc = warm_stage_table(ctx, stage_cfgs, -1, lps, &wlps, temporal))) return rc;
    const int H = history_size(opt_cfg);
    const int max_run = any_warm ? kMaxStages / 2 : kMaxStages;       // the table holds the cold and the warm slice of a run
    std::vector<int> rng;
    std::vector<LossParams> tab;                                      // stage table of a warm run (read by run_stage)
    int i = 0;
    while (i < n_stages) {
        const Regime rg = stage_regime(ctx, lps[i], H, false);
        const int j = stage_group_end(ctx, lps, i, H, max_run);
        use_stage(ctx, lps[i]);
        RunOpts o;
        if (!any_warm) {
            o.lps = &lps[i];
            o.nst = j - i;
        } else {
            if (rg == kBatched)
                return set_error(ctx, MVS_ERR_INVALID, "%s: warm-started frames are not implemented in the batched reference "
                                                       "chain (exec mode 1 / a model the resident kernels do not take)", who);
            // table of this run: cold stages i .. j-1, then the warm slice max(i, 2) .. j-1
            tab.assign(lps.begin() + i, lps.begin() + j);
            const int wi = i > kWarmSkip ? i : kWarmSkip;
            const int wbegin = (int)tab.size();
            for (int k = wi; k < j; ++k) tab.push_back(wlps[k]);
            const int wend = (int)tab.size();
            rng.assign((size_t)B * 2, 0);
            for (int b = 0; b < B; ++b) {
                const bool wm = warm_host[b] != 0;
                rng[2 * b] = wm ? wbegin : 0;
                rng[2 * b + 1] = wm ? wend : j - i;
                o.some_inactive |= wm && wbegin == wend;
            }
            if ((rc = upload_stage_rng(ctx, rng, st))) return rc;
            o.lps = tab.data();
            o.nst = (int)tab.size();
            o.stage_rng = ctx->stage_rng;
        }
        const int rc = run_stage(ctx, x_dev, final_loss_dev, opt_cfg, stats, st, o);
        if (rc) return rc;
        i = j;
    }
    ctx->loss = lps[n_stages - 1];
    return MVS_OK;
}

// Lane state of the dense groups, and frame scalars for F frames when a frame-resident group runs (grow-only)
static int ensure_stream_state(mvs_ctx* ctx, int F_resident) {
    if (!ctx->fstream) {
        std::unique_ptr<StreamState, ReleaseState> ss(new StreamState());
        const size_t B = (size_t)ctx->ws.B;
        int rc;
        if ((rc = dev_alloc(ctx, &ss->lane_frame, B)) || (rc = dev_alloc(ctx, &ss->lane_start, B)) ||
            (rc = dev_alloc(ctx, &ss->lane_params, B * kParams)) || (rc = dev_alloc(ctx, &ss->queue, 1)) ||
            (rc = dev_alloc(ctx, &ss->end_round, 1)))
            return rc;
        MVS_CUDA_OK(ctx, cudaMallocHost(&ss->host, 2 * sizeof(int)));
        ctx->fstream = ss.release();
    }
    return dev_grow(ctx, ctx->fstream->sc, (size_t)F_resident);
}

// The lanes' keypoint rows, and their 3-D target rows when with_j3d
static int ensure_lane_rows(mvs_ctx* ctx, bool with_j3d) {
    Workspace& w = ctx->ws;
    int rc = ensure_keypoint_ws(ctx);
    if (!rc && with_j3d && !w.j3d_xyz) {
        const size_t n = (size_t)w.B * ctx->m.K;
        if (!(rc = dev_alloc(ctx, &w.j3d_xyz, n * 3))) rc = dev_alloc(ctx, &w.j3d_conf, n);
    }
    return rc;
}

// A dense run over the context's B lanes, fed from the queue that a describes (the caller sets F, n_queue, the call's arrays,
// q.cold and, for a sequence stream, q and lane_seq): the first fill, the rounds, and the hand-back of whatever the round
// limit left in the lanes.  Adds the run's totals to stats.
static int run_lanes(mvs_ctx* ctx, LaneArgs& a, const float* joint_weights, const LbfgsCfg& cfg, int nst, mvs_lbfgs_stats* stats,
                     cudaStream_t st) {
    LbfgsState& S = *ctx->lbfgs;
    StreamState& ss = *ctx->fstream;
    Workspace& w = ctx->ws;
    const int B = w.B, K = ctx->m.K;
    int rc;
    if ((rc = frame_step_begin_run(ctx, st))) return rc;                 // (allocates the pose cache on first use)
    a.B = B; a.K = K;
    a.rigs = ctx->rigs_dev.p;
    a.ws_gt_uv = w.gt_uv; a.ws_conf = w.conf; a.ws_j3d_xyz = w.j3d_xyz; a.ws_j3d_conf = w.j3d_conf; a.ws_rig = w.slot_rig;
    ctx->slot_rigs = a.rig ? w.slot_rig : nullptr;                       // the dense kernels read each lane's rig
    a.lane_frame = ss.lane_frame; a.lane_start = ss.lane_start; a.lane_params = ss.lane_params; a.queue = ss.queue;
    a.end_round = ss.end_round; a.pose_valid = w.pose_valid;
    MVS_CUDA_OK(ctx, cudaMemcpyAsync(w.joint_w, joint_weights, (size_t)K * sizeof(float), cudaMemcpyDeviceToDevice, st));
    MVS_CUDA_OK(ctx, cudaMemsetAsync(ss.lane_frame, 0xff, (size_t)B * sizeof(int), st));
    MVS_CUDA_OK(ctx, cudaMemsetAsync(ss.queue, 0, sizeof(int), st));
    MVS_CUDA_OK(ctx, cudaMemsetAsync(ss.end_round, 0, sizeof(long long), st));
    MVS_LAUNCH(ctx, KID_MISC, st, iota2_kernel<<<(B + 255) / 256, 256, 0, st>>>(w.fidx, B, w.na));
    // the first min(n_queue, B) queue entries enter through the same path as every later one
    MVS_LAUNCH(ctx, KID_LBFGS_COMPACT, st, lane_refill_kernel<<<1, 1024, 0, st>>>(S, a, 0, 0));
    MVS_LAUNCH(ctx, KID_LBFGS_COMPACT, st, lbfgs_compact_kernel<<<1, 1024, 0, st>>>(S, B, w.fidx, w.na));
    if ((rc = run_dense(ctx, ss.lane_params, cfg, nst, st, &a))) return rc;
    // whatever the round limit left in the lanes (nothing, when every frame finished)
    MVS_LAUNCH(ctx, KID_LBFGS_COMPACT, st, lane_refill_kernel<<<1, 1024, 0, st>>>(S, a, 0, 1));
    MVS_LAUNCH(ctx, KID_MISC, st, iota2_kernel<<<(B + 255) / 256, 256, 0, st>>>(w.fidx, B, w.na));
    return read_totals(ctx, ss.end_round, true, stats, st);
}

// One run of mvs_fit_stream: stages lps[0 .. nst) of one regime over all F frames of the stream
static int run_stream_group(mvs_ctx* ctx, const mvs_frame_stream* s, const int* rig, Regime rg, const LossParams* lps, int nst,
                            const mvs_lbfgs_config* c, mvs_lbfgs_stats* stats, cudaStream_t st) {
    use_stage(ctx, lps[0]);
    LbfgsCfg cfg;
    int rc = begin_run(ctx, c, false, lps, nst, &cfg, st);
    if (rc) return rc;
    const int F = s->n_frames;
    if (rg == kResident) {
        // one launch over all F frames, one CTA each: the block scheduler refills the SMs as frames finish
        FrameScalars* sc = ctx->fstream->sc.p;
        const FrameInputs in{F, s->gt_uv, s->conf, s->joint_weights, s->gt_xyz, s->conf3d, rig};
        rc = launch_lbfgs_resident(ctx, s->params, cfg, nst, in, sc, nullptr, nullptr, st);
        return rc ? rc : finish_run(ctx, kResident, sc, F, s->final_loss, stats, st);
    }
    LaneArgs a{};
    a.F = F; a.n_queue = F;
    a.params = s->params; a.final_loss = s->final_loss; a.gt_uv = s->gt_uv; a.conf = s->conf;
    a.j3d_xyz = s->gt_xyz; a.j3d_conf = s->conf3d; a.rig = rig;
    a.q.cold = make_int2(0, nst);                                     // every frame runs the whole table
    return run_lanes(ctx, a, s->joint_weights, cfg, nst, stats, st);
}

// A stream call's writes to the context.  Its dense runs overwrite the slots' keypoint, 3-D target and rig rows, so from the
// start the context holds none of them; at the end its loss config is the call's last stage, without the call's 3-D term.
static void stream_call_begin(mvs_ctx* ctx) {
    ctx->have_kp = false;
    ctx->j3d_enabled = false;
    ctx->slot_rigs = nullptr;
}
static void stream_call_end(mvs_ctx* ctx, const LossParams& last) {
    ctx->loss = last;
    ctx->loss.j3d_on = 0;
    ctx->slot_rigs = nullptr;
}

// mvs_fit_stream (who: the entry point called): the stage groups of run_fit, each over all F frames before the next starts
// (rig [F] or NULL: rig 0)
static int run_stream(mvs_ctx* ctx, const char* who, const mvs_frame_stream* s, const int* rig, int n_stages,
                      const mvs_loss_config* stage_cfgs, const mvs_lbfgs_config* opt_cfg, mvs_lbfgs_stats* stats, cudaStream_t st) {
    const int H = history_size(opt_cfg);
    std::vector<LossParams> lps;
    std::vector<int> ends;
    int rc = stage_table(ctx, who, n_stages, stage_cfgs, s->gt_xyz ? 1 : 0, &lps);
    if (!rc) rc = stream_runs(ctx, who, lps, H, kMaxStages, &ends);
    if (rc) return rc;
    bool any_dense = false, any_resident = false;
    for (int i = 0, g = 0; i < n_stages; i = ends[g++]) (stage_regime(ctx, lps[i], H, false) == kDense ? any_dense : any_resident) = true;
    rc = ensure_stream_state(ctx, any_resident ? s->n_frames : 0);
    if (!rc && any_dense) rc = ensure_lane_rows(ctx, s->gt_xyz != nullptr);
    if (rc) return rc;
    stream_call_begin(ctx);
    for (int i = 0, g = 0; i < n_stages && !rc; i = ends[g++])
        rc = run_stream_group(ctx, s, rig, stage_regime(ctx, lps[i], H, false), &lps[i], ends[g] - i, opt_cfg, stats, st);
    stream_call_end(ctx, lps[n_stages - 1]);
    return rc;
}

// mvs_fit_seq_stream, mvs_fit_shared_shape and mvs_refine_cameras scratch (DESIGN.md section 4), every array grow-only.  A
// context runs one call at a time, so they share it: the gathered frames (gather_frames) serve all three, and off, item_of,
// part, rows and seq_final describe the small problems of the two alternating calls (solve_problems).
struct SeqState {
    DevBuf<int> off;                    // [S+1] the call's sequence offsets; alternating calls: [P+1] problem p owns the
                                        // work items [off[p], off[p+1]) (shared shape: a problem per sequence, an item per frame)
    DevBuf<int> frames, packed_rig;     // [n] the gathered frames, their rigs
    DevBuf<float> packed;               // their packed rows (gather_floats)
    DevBuf<int> cur, act, lane_seq;     // sequence stream: [S], [S], [B] (SeqChain, LaneArgs)
    DevBuf<float> tw;                   // [F][86] the temporal weight, one row per frame (frame-resident chaining)
    DevBuf<int> item_of;                // [items] the problem of each work item
    DevBuf<float> part;                 // [items][kPartCols] each work item's loss and gradient entries
    DevBuf<float> rows;                 // [P + B][86] each problem's x (B rows of padding for the slots a last chunk leaves empty)
    DevBuf<float> seq_final;            // [B] run_fitting's value of each slot's problem
    DevBuf<int> ok;                     // shared shape: [S] the sequence has a finite row
    // camera refinement
    DevBuf<int> fin, body;              // [F] the row is all finite, [n] the frames with a finite row (ascending)
    DevBuf<float> held;                 // [F][K][3] held keypoints
    DevBuf<int> cam_frames;             // the rig-grouped frame list
    DevBuf<CameraProblem> prob;         // [P]
    DevBuf<CamRefine> cr;               // [P]
};

static SeqState& seq_state(mvs_ctx* ctx) {
    if (!ctx->sstream) ctx->sstream = new SeqState();
    return *ctx->sstream;
}

// The floats of n gathered frames' packed rows: params | gt_uv | conf, a final loss each with with_loss, then gt_xyz | conf3d
// with the 3-D term
static size_t gather_floats(const mvs_ctx* ctx, int n, bool with_loss, bool j3d) {
    const size_t K = (size_t)ctx->m.K;
    return (size_t)n * (kParams + (size_t)ctx->vmax * K * 3 + (with_loss ? 1 : 0) + (j3d ? K * 4 : 0));
}

// Frames idx[0 .. n) of a call's frames `in` and their rows params [in.n][86] packed into the scratch as the frame stream *fs of
// n frames, with final-loss rows when with_loss; *prig: their rigs, NULL without in.rig
static int gather_frames(mvs_ctx* ctx, const FrameInputs& in, float* params, const std::vector<int>& idx, bool with_loss,
                         mvs_frame_stream* fs, const int** prig, cudaStream_t st) {
    SeqState& q = *ctx->sstream;
    const int n = (int)idx.size(), F = in.n, V = ctx->vmax, K = ctx->m.K;
    const float *gt_xyz = in.j3d_xyz, *conf3d = in.j3d_conf;
    const int* rig = in.rig;
    int rc;
    if ((rc = dev_grow(ctx, q.frames, (size_t)n)) || (rc = dev_grow(ctx, q.packed_rig, (size_t)n)) ||
        (rc = dev_grow(ctx, q.packed, gather_floats(ctx, n, with_loss, gt_xyz != nullptr))))
        return rc;
    const int* fr = q.frames.p;
    const Rig* rigs = ctx->rigs_dev.p;
    MVS_CUDA_OK(ctx, cudaMemcpyAsync(q.frames.p, idx.data(), (size_t)n * sizeof(int), cudaMemcpyHostToDevice, st));
    float* px = q.packed.p;
    float* pg = px + (size_t)n * kParams;
    float* pc = pg + (size_t)V * n * K * 2;
    float* pf = pc + (size_t)V * n * K;
    float* pj = gt_xyz ? pf + (with_loss ? n : 0) : nullptr;
    float* pjc = gt_xyz ? pj + (size_t)n * K * 3 : nullptr;
    MVS_LAUNCH(ctx, KID_MISC, st, copy_rows_kernel<<<dim3(n, 1), 128, 0, st>>>(px, params, fr, n, F, kParams, 0));
    MVS_LAUNCH(ctx, KID_MISC, st, copy_rows_kernel<<<dim3(n, V), 128, 0, st>>>(pg, const_cast<float*>(in.gt_uv), fr, n, F, 2 * K, 0,
                                                                             rigs, rig));
    MVS_LAUNCH(ctx, KID_MISC, st, copy_rows_kernel<<<dim3(n, V), 128, 0, st>>>(pc, const_cast<float*>(in.conf), fr, n, F, K, 0,
                                                                             rigs, rig));
    if (rig)
        MVS_LAUNCH(ctx, KID_MISC, st, copy_rows_kernel<<<dim3(n, 1), 32, 0, st>>>(q.packed_rig.p, const_cast<int*>(rig), fr, n, F, 1, 0));
    if (gt_xyz) {
        MVS_LAUNCH(ctx, KID_MISC, st, copy_rows_kernel<<<dim3(n, 1), 128, 0, st>>>(pj, const_cast<float*>(gt_xyz), fr, n, F, 3 * K, 0));
        MVS_LAUNCH(ctx, KID_MISC, st, copy_rows_kernel<<<dim3(n, 1), 128, 0, st>>>(pjc, const_cast<float*>(conf3d), fr, n, F, K, 0));
    }
    *fs = mvs_frame_stream{n, px, pg, pc, in.joint_w, pj, pjc, with_loss ? pf : nullptr};
    *prig = rig ? q.packed_rig.p : nullptr;
    return MVS_OK;
}

// The gathered frames' rows (gather_frames) back to the call's rows params [F][86], and their final losses to final_loss [F]
// when fs has them and final_loss is not NULL
static void scatter_frames(mvs_ctx* ctx, int F, float* params, float* final_loss, const mvs_frame_stream& fs, cudaStream_t st) {
    const int n = fs.n_frames;
    const int* fr = ctx->sstream->frames.p;
    MVS_LAUNCH(ctx, KID_MISC, st, copy_rows_kernel<<<dim3(n, 1), 128, 0, st>>>(fs.params, params, fr, n, F, kParams, 1));
    if (fs.final_loss && final_loss)
        MVS_LAUNCH(ctx, KID_MISC, st, copy_rows_kernel<<<dim3(n, 1), 32, 0, st>>>(fs.final_loss, final_loss, fr, n, F, 1, 1));
}

// The slots' anchor rows and weights (as mvs_set_anchor allocates them), weights set to w for every slot
static int temporal_slot_rows(mvs_ctx* ctx, const float* w, cudaStream_t st) {
    Workspace& ws = ctx->ws;
    int rc;
    if (!ws.anchor) {
        if ((rc = dev_alloc(ctx, &ws.anchor, (size_t)ws.B * kParams))) return rc;
        if ((rc = dev_alloc(ctx, &ws.anchor_w, (size_t)ws.B * kParams))) return rc;
    }
    Row86 r;
    for (int i = 0; i < kParams; ++i) r.v[i] = w[i];
    MVS_LAUNCH(ctx, KID_MISC, st, fill_rows_kernel<<<(ws.B * kParams + 255) / 256, 256, 0, st>>>(ws.anchor_w, r, ws.B));
    return MVS_OK;
}

// The chaining run over the sequences of one pass (q.act): every frame of run `tab` from its sequence's pending frame on
// (in: the call's frames, F = in.n)
// temporal: the warm stages of tab carry the anchor term; its weight rows are set up (sstream->tw for the frame-resident
// regime, ws.anchor_w for the dense one), and the anchor rows are the predecessors' fitted rows, handed over on the device.
static int run_seq_chain(mvs_ctx* ctx, const mvs_sequence_stream* s, const FrameInputs& in, Regime rg,
                         const std::vector<LossParams>& tab, const SeqChain& q0, const mvs_lbfgs_config* c, mvs_lbfgs_stats* stats,
                         cudaStream_t st, bool temporal) {
    const int nst = (int)tab.size();
    use_stage(ctx, tab[0]);
    LbfgsCfg cfg;
    int rc = begin_run(ctx, c, false, tab.data(), nst, &cfg, st);
    if (rc) return rc;
    LbfgsState& S = *ctx->lbfgs;
    SeqChain q = q0;
    q.final_loss = s->final_loss;
    q.totals = S.totals;
    if (rg == kResident) {
        // one launch, one CTA per sequence; rounds: the largest number of evaluations one CTA ran (its frames' sum)
        if ((rc = launch_lbfgs_resident_seq(ctx, s->params, cfg, nst, in, q, st, temporal ? ctx->sstream->tw.p : nullptr)))
            return rc;
        return read_totals(ctx, nullptr, false, stats, st);
    }
    LaneArgs a{};
    a.F = in.n; a.n_queue = q.n_act;
    a.params = s->params; a.final_loss = s->final_loss; a.gt_uv = in.gt_uv; a.conf = in.conf;
    a.j3d_xyz = in.j3d_xyz; a.j3d_conf = in.j3d_conf; a.rig = in.rig;
    a.q = q;
    a.lane_seq = ctx->sstream->lane_seq.p;
    a.anchor = temporal ? ctx->ws.anchor : nullptr;
    return run_lanes(ctx, a, in.joint_w, cfg, nst, stats, st);
}

// mvs_fit_seq_stream (DESIGN.md section 4; who: the entry point called).  Stages are grouped into runs as mvs_fit_seq groups
// them; run c holds stages 2 .. n-1 and is the chaining run.  Each pass takes the pending cold frames P (at first: every
// sequence's first frame) through the runs before c (as a frame stream of P's rows), then runs c over their sequences; a
// sequence whose next frame turns out cold parks it for the next pass (c > 0 only: with c == 0 the cold frame stays in its slot
// with the cold slice).
// gt_xyz / conf3d ([F][K][3] / [F][K], both NULL or both set): the 3-D joint term is on in every stage, cold and warm, iff set;
// they travel with the frames as gt_uv / conf do, and so does rig ([F] or NULL: every frame has rig 0).
// tw ([86] host, NULL: off): the temporal weight; every warm frame's stages carry sum_i tw_i (x_i - predecessor's fitted x_i)^2.
static int run_seq_stream(mvs_ctx* ctx, const char* who, const mvs_sequence_stream* s, const float* gt_xyz, const float* conf3d,
                          const int* rig, int n_stages, const mvs_loss_config* stage_cfgs, const mvs_lbfgs_config* opt_cfg,
                          mvs_lbfgs_stats* stats, cudaStream_t st, const float* tw) {
    const int NS = s->n_sequences;
    const std::vector<int> off(s->seq_offsets, s->seq_offsets + NS + 1);
    const int F = off[NS];
    const FrameInputs in{F, s->gt_uv, s->conf, s->joint_weights, gt_xyz, conf3d, rig};
    const int j3d = gt_xyz ? 1 : 0;                                   // the call's own targets, never the context's
    std::vector<LossParams> lps, wlps;
    int rc = stage_table(ctx, who, n_stages, stage_cfgs, j3d, &lps);
    if (rc) return rc;
    int n_vp2 = 0;
    for (const LossParams& lp : lps) n_vp2 += lp.use_vposer == 2;
    if (n_vp2 > 0 && n_vp2 < n_stages)
        return set_error(ctx, MVS_ERR_INVALID, "%s: stages mix latent-code (use_vposer = 2) and axis-angle poses", who);
    if ((rc = warm_stage_table(ctx, stage_cfgs, j3d, lps, &wlps, tw != nullptr))) return rc;
    const int H = history_size(opt_cfg);
    std::vector<int> ends;
    if ((rc = stream_runs(ctx, who, lps, H, kMaxStages / 2, &ends))) return rc;
    int c = -1, ic = 0;
    bool any_dense = false, resident_before = false;
    for (int i = 0, g = 0; i < n_stages; i = ends[g++]) {
        const Regime rg = stage_regime(ctx, lps[i], H, false);
        any_dense |= rg == kDense;
        if (i <= kWarmSkip && kWarmSkip < ends[g]) { c = g; ic = i; }
        else if (c < 0) resident_before |= rg == kResident;
    }
    if (ends[c] != n_stages)
        return set_error(ctx, MVS_ERR_UNSUPPORTED, "%s: stages %d .. %d do not form one run (the run holding stage %d ends at %d; "
                                                   "exec mode 2, or a change of regime, SDF grid or face mode)",
                         who, kWarmSkip, n_stages - 1, kWarmSkip, ends[c]);
    // the chaining run's table: cold stages ic .. n-1, then the warm slice 2 .. n-1
    std::vector<LossParams> tab(lps.begin() + ic, lps.end());
    const int wbegin = (int)tab.size();
    for (int k = kWarmSkip; k < n_stages; ++k) tab.push_back(wlps[k]);
    SeqChain q;
    q.cold = make_int2(0, wbegin);
    q.warm = make_int2(wbegin, (int)tab.size());
    q.reinit_loss = s->reinit_loss;
    q.park = c > 0 ? 1 : 0;
    q.keep_pose = n_vp2 == 0 ? 1 : 0;
    SeqState& ss = seq_state(ctx);
    rc = ensure_stream_state(ctx, resident_before ? NS : 0);
    if (!rc && !(rc = dev_grow(ctx, ss.off, (size_t)NS + 1)) && !(rc = dev_grow(ctx, ss.cur, (size_t)NS)) &&
        !(rc = dev_grow(ctx, ss.act, (size_t)NS)))
        rc = dev_grow(ctx, ss.lane_seq, (size_t)ctx->ws.B);
    if (!rc && any_dense) rc = ensure_lane_rows(ctx, gt_xyz != nullptr);
    if (rc) return rc;
    const Regime rg_chain = stage_regime(ctx, lps[ic], H, false);
    if (tw && rg_chain == kResident) {                                // a weight row per frame, as the closure indexes them
        if ((rc = dev_grow(ctx, ss.tw, (size_t)F * kParams))) return rc;
        Row86 r;
        for (int i = 0; i < kParams; ++i) r.v[i] = tw[i];
        MVS_LAUNCH(ctx, KID_MISC, st, fill_rows_kernel<<<(F * kParams + 255) / 256, 256, 0, st>>>(ss.tw.p, r, F));
    } else if (tw && (rc = temporal_slot_rows(ctx, tw, st))) {         // dense: per lane
        return rc;
    }
    q.off = ss.off.p;
    q.cur = ss.cur.p;
    q.act = ss.act.p;
    stream_call_begin(ctx);
    MVS_CUDA_OK(ctx, cudaMemcpyAsync(ss.off.p, off.data(), off.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    std::vector<int> cur(off.begin(), off.end() - 1), act, frames;   // each sequence's pending cold frame, -1: done
    while (!rc) {
        act.clear();
        frames.clear();
        for (int k = 0; k < NS; ++k)
            if (cur[k] >= 0) { act.push_back(k); frames.push_back(cur[k]); }
        if (act.empty()) break;
        const int n = (int)act.size();
        MVS_CUDA_OK(ctx, cudaMemcpyAsync(ss.cur.p, cur.data(), (size_t)NS * sizeof(int), cudaMemcpyHostToDevice, st));
        MVS_CUDA_OK(ctx, cudaMemcpyAsync(ss.act.p, act.data(), (size_t)n * sizeof(int), cudaMemcpyHostToDevice, st));
        if (c > 0) {
            // the pending frames through the runs before c, as a frame stream of their packed rows
            mvs_frame_stream fs;
            const int* prig;
            if ((rc = gather_frames(ctx, in, s->params, frames, false, &fs, &prig, st))) break;
            for (int i = 0, g = 0; g < c && !rc; i = ends[g++])
                rc = run_stream_group(ctx, &fs, prig, stage_regime(ctx, lps[i], H, false), &lps[i], ends[g] - i, opt_cfg, stats, st);
            if (rc) break;
            scatter_frames(ctx, F, s->params, nullptr, fs, st);
        }
        q.n_act = n;
        if ((rc = run_seq_chain(ctx, s, in, rg_chain, tab, q, opt_cfg, stats, st, tw != nullptr))) break;
        MVS_CUDA_OK(ctx, cudaMemcpyAsync(cur.data(), ss.cur.p, (size_t)NS * sizeof(int), cudaMemcpyDeviceToHost, st));
        MVS_CUDA_OK(ctx, cudaStreamSynchronize(st));
    }
    stream_call_end(ctx, lps[n_stages - 1]);
    return rc;
}

// The temporal weight of mvs_fit_seq_temporal / mvs_fit_seq_stream_temporal (who: the entry point): NULL, or 86 finite entries
// >= 0 with n_stages > 2, outside exec mode 1 and with mvs_set_anchor off.  *on: some entry is non-zero (all zero: the term
// is off, and the call is the one it extends).
static int check_temporal_weight(mvs_ctx* ctx, const char* who, const float* w, int n_stages, bool* on) {
    *on = false;
    if (!w) return MVS_OK;
    for (int i = 0; i < kParams; ++i) {
        if (!(w[i] >= 0.f) || !isfinite(w[i]))
            return set_error(ctx, MVS_ERR_INVALID, "%s: temporal weight %d is %g (want finite and >= 0)", who, i, (double)w[i]);
        *on |= w[i] != 0.f;
    }
    if (n_stages <= kWarmSkip)
        return set_error(ctx, MVS_ERR_INVALID, "%s: the temporal term is on the warm frames' stages %d .. n-1, %d stages given", who,
                         kWarmSkip, n_stages);
    if (ctx->exec_mode == 1)
        return set_error(ctx, MVS_ERR_UNSUPPORTED, "%s: warm-started frames are not implemented in the batched reference chain "
                                                   "(exec mode 1)", who);
    if (ctx->anchor_enabled)
        return set_error(ctx, MVS_ERR_UNSUPPORTED, "%s: the temporal term uses the anchor rows; switch mvs_set_anchor off first", who);
    return MVS_OK;
}

// Per sequence (one warp): the mean of the shared entries (betas, and scale with share_scale) over the frames whose rows are
// all finite, accumulated in double in frame order, into rows[q] (zeros elsewhere); ok[q] = 0 when no row is finite.  Once the
// shared entries of a sequence's rows are equal (after a sweep), the mean reproduces them bit for bit.
__global__ void shape_consensus_kernel(const float* __restrict__ params, const int* __restrict__ off, int share_scale,
                                       float* __restrict__ rows, int* __restrict__ ok) {
    const int q = blockIdx.x, lane = threadIdx.x;
    const int e = lane < kOffOrient ? lane : (lane == kOffOrient && share_scale) ? kOffScale : -1;
    double acc = 0.0;
    int n = 0;
    for (int f = off[q]; f < off[q + 1]; ++f) {
        const float* x = params + (size_t)f * kParams;
        bool fin = true;
        for (int i = lane; i < kParams; i += 32) fin = fin && isfinite(x[i]);
        if (!__all_sync(0xffffffffu, fin)) continue;
        ++n;
        if (e >= 0) acc += (double)x[e];
    }
    float* r = rows + (size_t)q * kParams;
    for (int i = lane; i < kParams; i += 32) r[i] = 0.f;
    __syncwarp();
    if (e >= 0 && n > 0) r[e] = (float)(acc / (double)n);
    if (lane == 0) ok[q] = n > 0 ? 1 : 0;
}

// The shared entries of every frame of a sequence with a finite row: its sequence's row
__global__ void shape_write_kernel(float* __restrict__ params, const int* __restrict__ item_of, const float* __restrict__ rows,
                                   const int* __restrict__ ok, int F, int share_scale) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= F || !ok[item_of[f]]) return;
    const float* r = rows + (size_t)item_of[f] * kParams;
    float* x = params + (size_t)f * kParams;
    for (int i = kOffBetas; i < kOffOrient; ++i) x[i] = r[i];
    if (share_scale) x[kOffScale] = r[kOffScale];
}

// The small problems of mvs_fit_shared_shape (a sequence's shape) and mvs_refine_cameras (a view's extrinsics), solved by one
// driver (DESIGN.md section 4).  Problem p's x is sstream->rows[p]; it owns the work items [beg[p], beg[p+1]) (device copy:
// sstream->off, with sstream->item_of), and each item's closure kernel writes the item's part row: its loss, then the gradient
// entries ent.e[0 .. ent.n) of its problem.
struct PartEntries {
    int n, e[kPartCols - 1];
};
struct ProblemSet {
    std::vector<int> beg;               // [P+1] host
    std::vector<int> on;                // [P] 0: the problem is not solved and its row stays (a sequence without a finite row)
    PartEntries ent;
    bool vp2 = false;                   // the pose entries of x hold a latent code (lbfgs_advance's pose length)
};
// The closure kernel of one chunk: the part rows of the chunk's work items
using ChunkClosure = std::function<int(const ProblemChunk&, const LbfgsState&)>;

// Per problem of a chunk (one warp, block j = slot j): lane k adds column k of the part rows of the problem's work items in
// double, in item order; column 0 goes to the slot's loss_eval, column 1 + k to entry ent.e[k] of its g_eval (zeros elsewhere).
// The order depends on the problem's items only.  Problems that have finished are skipped.
__global__ void __launch_bounds__(32)
problem_reduce_kernel(LbfgsState L, ProblemChunk c, PartEntries ent) {
    const int j = blockIdx.x, lane = threadIdx.x, p = c.base + j;
    if (L.sc[j].phase == PH_DONE) return;
    double acc = 0.0;
    if (lane <= ent.n)
        for (int i = c.beg[p]; i < c.beg[p + 1]; ++i) acc += (double)c.part[(size_t)i * kPartCols + lane];
    int e = -1;
#pragma unroll
    for (int k = 0; k < kPartCols - 1; ++k)
        if (lane == k + 1 && k < ent.n) e = ent.e[k];
    float* g = L.g_eval + (size_t)j * kParams;
    for (int i = lane; i < kParams; i += 32) g[i] = 0.f;
    __syncwarp();
    if (lane == 0) L.loss_eval[j] = (float)acc;
    else if (e >= 0) g[e] = (float)acc;
}

// The scratch of ps (rows for P problems and B slots of padding, each slot's final value, a part row per work item) and its
// beg / item_of on the device
static int problem_scratch(mvs_ctx* ctx, const ProblemSet& ps, cudaStream_t st) {
    SeqState& h = seq_state(ctx);
    const int P = (int)ps.beg.size() - 1, items = ps.beg[P], B = ctx->ws.B;
    std::vector<int> item_of((size_t)items);
    for (int p = 0; p < P; ++p)
        for (int i = ps.beg[p]; i < ps.beg[p + 1]; ++i) item_of[i] = p;
    int rc;
    if ((rc = dev_grow(ctx, h.off, (size_t)P + 1)) || (rc = dev_grow(ctx, h.item_of, (size_t)std::max(items, 1))) ||
        (rc = dev_grow(ctx, h.part, (size_t)std::max(items, 1) * kPartCols)) ||
        (rc = dev_grow(ctx, h.rows, ((size_t)P + B) * kParams)) || (rc = dev_grow(ctx, h.seq_final, (size_t)B)))
        return rc;
    MVS_CUDA_OK(ctx, cudaMemcpyAsync(h.off.p, ps.beg.data(), ps.beg.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    MVS_CUDA_OK(ctx, cudaMemcpyAsync(h.item_of.p, item_of.data(), (size_t)items * sizeof(int), cudaMemcpyHostToDevice, st));
    MVS_CUDA_OK(ctx, cudaStreamSynchronize(st));
    return MVS_OK;
}

// Chunk *c of ps: problems base .. base + n - 1, the context's B at most, in slots 0 .. n - 1, each from its row with a fresh
// optimiser unless it is off; the other slots have no stage and leave the active list
static int chunk_start(mvs_ctx* ctx, const ProblemSet& ps, int base, ProblemChunk* c, cudaStream_t st) {
    LbfgsState& S = *ctx->lbfgs;
    Workspace& w = ctx->ws;
    SeqState& h = *ctx->sstream;
    const int B = w.B, n = std::min(B, (int)ps.beg.size() - 1 - base);
    *c = ProblemChunk{h.off.p, h.item_of.p, h.part.p, base, n, ps.beg[base], ps.beg[base + n] - ps.beg[base]};
    std::vector<int> rng((size_t)B * 2, 0);
    bool some_inactive = false;
    for (int j = 0; j < B; ++j) {
        const bool on = j < n && ps.on[base + j];
        rng[2 * j + 1] = on ? 1 : 0;
        some_inactive |= !on;
    }
    if (int rc = upload_stage_rng(ctx, rng, st)) return rc;
    MVS_LAUNCH(ctx, KID_MISC, st, iota2_kernel<<<(B + 255) / 256, 256, 0, st>>>(w.fidx, B, w.na));
    MVS_LAUNCH(ctx, KID_MISC, st, lbfgs_init_kernel<<<B, 32, 0, st>>>(S, h.rows.p + (size_t)base * kParams, B, 1, 1, ctx->stage_rng));
    if (some_inactive) MVS_LAUNCH(ctx, KID_LBFGS_COMPACT, st, lbfgs_compact_kernel<<<1, 1024, 0, st>>>(S, B, w.fidx, w.na));
    return MVS_OK;
}

// One evaluation of chunk c: the closure's part rows, then their sums per problem into the slots' loss_eval / g_eval
static int eval_chunk(mvs_ctx* ctx, const ProblemSet& ps, const ProblemChunk& c, const ChunkClosure& closure, cudaStream_t st) {
    const LbfgsState& S = *ctx->lbfgs;
    if (int rc = closure(c, S)) return rc;
    MVS_LAUNCH(ctx, KID_MISC, st, problem_reduce_kernel<<<c.n, 32, 0, st>>>(S, c, ps.ent));
    MVS_CUDA_OK(ctx, cudaGetLastError());
    return MVS_OK;
}

// Every problem of ps that is on, from its row, the context's B at a time, run as run_fitting runs a frame's stage (the batched
// chain's lbfgs_init / advance / compact with the chunk's evaluation as the closure); final [P] (device, or NULL): run_fitting's
// value of each problem
static int solve_problems(mvs_ctx* ctx, const ProblemSet& ps, const ChunkClosure& closure, const LossParams& lp,
                          const mvs_lbfgs_config* c, float* final, mvs_lbfgs_stats* stats, cudaStream_t st) {
    SeqState& h = *ctx->sstream;
    for (int base = 0; base < (int)ps.beg.size() - 1; base += ctx->ws.B) {
        LbfgsCfg cfg;
        ProblemChunk ch;
        int rc = begin_run(ctx, c, false, &lp, 1, &cfg, st);
        if (!rc) rc = chunk_start(ctx, ps, base, &ch, st);
        if (rc) return rc;
        const std::function<int()> eval = [&]() { return eval_chunk(ctx, ps, ch, closure, st); };
        if ((rc = run_batched(ctx, h.rows.p + (size_t)base * kParams, cfg, ps.vp2, st, eval))) return rc;
        if ((rc = end_run(ctx, kBatched, h.seq_final.p, nullptr, stats, st))) return rc;
        if (final)
            MVS_CUDA_OK(ctx, cudaMemcpyAsync(final + base, h.seq_final.p, (size_t)ch.n * sizeof(float), cudaMemcpyDeviceToDevice, st));
    }
    return MVS_OK;
}

// The debug closures: every problem of ps evaluated once at rows [P][86] (device): loss [P] and grad [P][86] (device) receive
// what the optimiser sees as loss_eval / g_eval.  Uses the context's optimiser state (history size 100 when there is none).
// Synchronises.
static int eval_problems(mvs_ctx* ctx, const ProblemSet& ps, const ChunkClosure& closure, const float* rows, float* loss,
                         float* grad, cudaStream_t st) {
    const int P = (int)ps.beg.size() - 1, B = ctx->ws.B;
    int rc = ensure_state(ctx, ctx->lbfgs ? ctx->lbfgs->H : 100);
    if (rc) return rc;
    MVS_CUDA_OK(ctx, cudaMemcpyAsync(ctx->sstream->rows.p, rows, (size_t)P * kParams * sizeof(float), cudaMemcpyDeviceToDevice, st));
    for (int base = 0; base < P && !rc; base += B) {
        ProblemChunk ch;
        if ((rc = chunk_start(ctx, ps, base, &ch, st)) || (rc = eval_chunk(ctx, ps, ch, closure, st))) break;
        const LbfgsState& S = *ctx->lbfgs;
        MVS_CUDA_OK(ctx, cudaMemcpyAsync(loss + base, S.loss_eval, (size_t)ch.n * sizeof(float), cudaMemcpyDeviceToDevice, st));
        MVS_CUDA_OK(ctx, cudaMemcpyAsync(grad + (size_t)base * kParams, S.g_eval, (size_t)ch.n * kParams * sizeof(float),
                                         cudaMemcpyDeviceToDevice, st));
    }
    MVS_LAUNCH(ctx, KID_MISC, st, iota2_kernel<<<(B + 255) / 256, 256, 0, st>>>(ctx->ws.fidx, B, ctx->ws.na));
    MVS_CUDA_OK(ctx, cudaStreamSynchronize(st));
    MVS_CUDA_OK(ctx, cudaGetLastError());
    return rc;
}

// The body step of an alternating call (who: the entry point called): `frames` (ascending) of the call's frames `in` as one
// frame stream of their packed rows through run_stream under the one stage cfg; their rows and final losses go back to params
// and final_loss (may be NULL)
static int refit_bodies(mvs_ctx* ctx, const char* who, const FrameInputs& in, float* params, float* final_loss,
                        const std::vector<int>& frames, const mvs_loss_config* cfg, const mvs_lbfgs_config* c,
                        mvs_lbfgs_stats* stats, cudaStream_t st) {
    if (frames.empty()) return MVS_OK;
    mvs_frame_stream fs;
    const int* prig;
    int rc = gather_frames(ctx, in, params, frames, true, &fs, &prig, st);
    if (!rc) rc = run_stream(ctx, who, &fs, prig, 1, cfg, c, stats, st);
    if (rc) return rc;
    scatter_frames(ctx, in.n, params, final_loss, fs, st);
    MVS_CUDA_OK(ctx, cudaStreamSynchronize(st));
    MVS_CUDA_OK(ctx, cudaGetLastError());
    return MVS_OK;
}

// What mvs_fit_shared_shape and mvs_debug_shape_closure share once check_seq_stream has passed: the checks of the stage, its
// LossParams (3-D term as the call says), the sequences as problems (a work item per frame, the shared entries as variables)
// with their scratch, and the shape closure's arguments a
static int shape_prepare(mvs_ctx* ctx, const char* who, const mvs_sequence_stream* s, const float* gt_xyz, const float* conf3d,
                         const int* rig, const mvs_loss_config* stage, int H, LossParams* lp, ProblemSet* ps, ShapeArgs* a,
                         cudaStream_t st) {
    if (!stage) return set_error(ctx, MVS_ERR_INVALID, "%s: NULL argument", who);
    if (stage->frozen_mask & 1u)
        return set_error(ctx, MVS_ERR_INVALID, "%s: the stage freezes betas (fix_shape): the shape is given, there is nothing to "
                                               "share", who);
    if (stage->interpenetration)
        return set_error(ctx, MVS_ERR_UNSUPPORTED, "%s: the shape closure is the frame-resident closure, which has no "
                                                   "interpenetration (SDF) term", who);
    int rc = make_loss_params(ctx, stage, lp);
    if (rc) return rc;
    lp->j3d_on = gt_xyz ? 1 : 0;
    if (stage_regime(ctx, *lp, H, false) != kResident)
        return set_error(ctx, MVS_ERR_UNSUPPORTED, "%s: the stage would not run in the frame-resident kernels (exec mode 1, "
                                                   "history_size > 100, or a model they do not take)", who);
    const int NS = s->n_sequences;
    *a = ShapeArgs{FrameInputs{s->seq_offsets[NS], s->gt_uv, s->conf, s->joint_weights, gt_xyz, conf3d, rig}, s->params,
                   (stage->frozen_mask >> 4 & 1u) ? 0 : 1};
    *ps = ProblemSet{};
    ps->beg.assign(s->seq_offsets, s->seq_offsets + NS + 1);
    ps->on.assign((size_t)NS, 1);
    ps->ent.n = kOffOrient + a->share_scale;                         // betas, then scale
    for (int e = 0; e < kOffOrient; ++e) ps->ent.e[e] = kOffBetas + e;
    ps->ent.e[kOffOrient] = kOffScale;
    ps->vp2 = lp->use_vposer == 2;
    if ((rc = dev_grow(ctx, seq_state(ctx).ok, (size_t)NS))) return rc;
    return problem_scratch(ctx, *ps, st);
}

// Refuses a call (who: the entry point called) before the context has model, cameras and batch, and the keypoints (kp) and the
// loss config (loss) where the call reads them
static int check_ready(mvs_ctx* ctx, const char* who, bool kp = false, bool loss = false) {
    if (!ctx) return set_error(nullptr, MVS_ERR_INVALID, "ctx is NULL");
    if (!(ctx->have_model && ctx->have_cams && ctx->ws.B > 0) || (kp && !ctx->have_kp) || (loss && !ctx->have_loss))
        return set_error(ctx, MVS_ERR_INVALID, "%s: %s must be set first", who,
                         loss ? "model, cameras, batch, keypoints and loss config"
                         : kp ? "model, cameras, batch and keypoints" : "model, cameras and batch");
    return MVS_OK;
}

// The preamble of the batch entry points: check_ready, the arguments (args_ok: none is NULL or empty) and the slots' rigs; then
// the device and zeroed stats
static int begin_batch_call(mvs_ctx* ctx, const char* who, bool kp, bool loss, bool args_ok, mvs_lbfgs_stats* stats) {
    if (int rc = check_ready(ctx, who, kp, loss)) return rc;
    if (!args_ok) return set_error(ctx, MVS_ERR_INVALID, "%s: NULL / empty argument", who);
    if (int rc = batch_rigs(ctx, who)) return rc;
    MVS_CUDA_OK(ctx, cudaSetDevice(ctx->device));
    if (stats) memset(stats, 0, sizeof(*stats));
    return MVS_OK;
}

// The alternating calls (mvs_fit_shared_shape, mvs_refine_cameras; who: the one called): what they check of their sweeps
// (check_sweeps), and how they start once every check has passed (start_sweeps: both stats zeroed, the F final losses NaN, as
// the frames without a finite row keep them)
static int check_sweeps(mvs_ctx* ctx, const char* who, const mvs_lbfgs_config* opt_cfg, int n_sweeps) {
    if (!opt_cfg) return set_error(ctx, MVS_ERR_INVALID, "%s: NULL argument", who);
    if (n_sweeps < 1) return set_error(ctx, MVS_ERR_INVALID, "%s: n_sweeps must be >= 1 (got %d)", who, n_sweeps);
    return MVS_OK;
}
static int start_sweeps(mvs_ctx* ctx, int F, float* final_loss, mvs_lbfgs_stats* a, mvs_lbfgs_stats* b, cudaStream_t st) {
    if (a) memset(a, 0, sizeof(*a));
    if (b) memset(b, 0, sizeof(*b));
    if (final_loss) MVS_CUDA_OK(ctx, cudaMemsetAsync(final_loss, 0xff, (size_t)F * sizeof(float), st));
    return MVS_OK;
}

// What every stream call checks last (who: the entry point called; F frames): the anchor term off, and a rig per frame when
// the context has several, its indices checked on the device
static int check_stream_rigs(mvs_ctx* ctx, const char* who, const int* rig, int F, cudaStream_t st) {
    if (ctx->anchor_enabled)
        return set_error(ctx, MVS_ERR_UNSUPPORTED, "%s: the anchor term is per batch (sequence smoothness); switch it off "
                                                   "(mvs_set_anchor enable = 0) to fit a stream", who);
    if (!rig && ctx->rigs.size() > 1)
        return set_error(ctx, MVS_ERR_INVALID, "%s: the context has %d camera rigs: give each frame's rig", who, (int)ctx->rigs.size());
    MVS_CUDA_OK(ctx, cudaSetDevice(ctx->device));
    return rig ? check_frame_rigs(ctx, who, rig, F, st) : MVS_OK;
}

// The checks of a sequence stream s and its gt_xyz, conf3d and rig (who: the entry point called)
static int check_seq_stream(mvs_ctx* ctx, const char* who, const mvs_sequence_stream* s, const float* gt_xyz, const float* conf3d,
                            const int* rig, cudaStream_t st) {
    if (int rc = check_ready(ctx, who)) return rc;
    if (!s) return set_error(ctx, MVS_ERR_INVALID, "%s: NULL argument", who);
    if (s->n_sequences < 1 || !s->seq_offsets)
        return set_error(ctx, MVS_ERR_INVALID, "%s: n_sequences must be >= 1 (got %d) with seq_offsets", who, s->n_sequences);
    if (!s->params || !s->gt_uv || !s->conf || !s->joint_weights)
        return set_error(ctx, MVS_ERR_INVALID, "%s: params, gt_uv, conf and joint_weights are required", who);
    if (s->seq_offsets[0] != 0) return set_error(ctx, MVS_ERR_INVALID, "%s: seq_offsets[0] must be 0", who);
    for (int k = 0; k < s->n_sequences; ++k)
        if (s->seq_offsets[k + 1] <= s->seq_offsets[k])
            return set_error(ctx, MVS_ERR_INVALID, "%s: seq_offsets must ascend strictly (sequence %d is empty or negative)", who, k);
    if (!gt_xyz != !conf3d) return set_error(ctx, MVS_ERR_INVALID, "%s: gt_xyz and conf3d go together", who);
    return check_stream_rigs(ctx, who, rig, s->seq_offsets[s->n_sequences], st);
}

// mvs_fit, mvs_fit_seq and mvs_fit_seq_temporal (who: the entry point called): warm_host NULL: every frame is cold;
// temporal_w_host NULL or all zero: no temporal term, and prev_dev is not read
static int fit_batch(mvs_ctx* ctx, const char* who, float* params_dev, int n_stages, const mvs_loss_config* stage_cfgs,
                     const mvs_lbfgs_config* opt_cfg, const unsigned char* warm_host, const float* prev_dev,
                     const float* temporal_w_host, float* final_loss_dev, mvs_lbfgs_stats* stats, void* stream) {
    const cudaStream_t st = (cudaStream_t)stream;
    bool on = false;
    int rc = begin_batch_call(ctx, who, true, false, params_dev && n_stages > 0 && stage_cfgs && opt_cfg, stats);
    if (!rc) rc = check_temporal_weight(ctx, who, temporal_w_host, n_stages, &on);
    if (!rc && on && !prev_dev) rc = set_error(ctx, MVS_ERR_INVALID, "%s: NULL / empty argument", who);
    if (!rc && on) rc = temporal_slot_rows(ctx, temporal_w_host, st);
    if (rc) return rc;
    if (on)
        MVS_CUDA_OK(ctx, cudaMemcpyAsync(ctx->ws.anchor, prev_dev, (size_t)ctx->ws.B * kParams * sizeof(float),
                                         cudaMemcpyDeviceToDevice, st));
    return run_fit(ctx, who, params_dev, n_stages, stage_cfgs, opt_cfg, final_loss_dev, stats, st, warm_host, on);
}

// mvs_fit_stream and mvs_fit_stream_rigs (who: the entry point called)
static int fit_stream(mvs_ctx* ctx, const char* who, const mvs_frame_stream* s, const int* rig, int n_stages,
                      const mvs_loss_config* stage_cfgs, const mvs_lbfgs_config* opt_cfg, mvs_lbfgs_stats* stats, void* stream) {
    const cudaStream_t st = (cudaStream_t)stream;
    if (int rc = check_ready(ctx, who)) return rc;
    if (!s || n_stages <= 0 || !stage_cfgs || !opt_cfg) return set_error(ctx, MVS_ERR_INVALID, "%s: NULL / empty argument", who);
    if (s->n_frames < 1) return set_error(ctx, MVS_ERR_INVALID, "%s: n_frames must be >= 1 (got %d)", who, s->n_frames);
    if (!s->params || !s->gt_uv || !s->conf || !s->joint_weights)
        return set_error(ctx, MVS_ERR_INVALID, "%s: params, gt_uv, conf and joint_weights are required", who);
    if (s->gt_xyz && !s->conf3d) return set_error(ctx, MVS_ERR_INVALID, "%s: gt_xyz needs conf3d", who);
    if (int rc = check_stream_rigs(ctx, who, rig, s->n_frames, st)) return rc;
    if (stats) memset(stats, 0, sizeof(*stats));
    return run_stream(ctx, who, s, rig, n_stages, stage_cfgs, opt_cfg, stats, st);
}

// The mvs_fit_seq_stream entry points (who: the one called)
static int fit_seq_stream(mvs_ctx* ctx, const char* who, const mvs_sequence_stream* s, const float* gt_xyz, const float* conf3d,
                          const int* rig, const float* temporal_w_host, int n_stages, const mvs_loss_config* stage_cfgs,
                          const mvs_lbfgs_config* opt_cfg, mvs_lbfgs_stats* stats, void* stream) {
    const cudaStream_t st = (cudaStream_t)stream;
    bool on = false;
    if (int rc = check_seq_stream(ctx, who, s, gt_xyz, conf3d, rig, st)) return rc;
    if (!stage_cfgs || !opt_cfg) return set_error(ctx, MVS_ERR_INVALID, "%s: NULL argument", who);
    if (n_stages <= kWarmSkip)
        return set_error(ctx, MVS_ERR_INVALID, "%s: warm-started frames skip the first %d stages, %d given", who, kWarmSkip, n_stages);
    if (int rc = check_temporal_weight(ctx, who, temporal_w_host, n_stages, &on)) return rc;
    if (stats) memset(stats, 0, sizeof(*stats));
    return run_seq_stream(ctx, who, s, gt_xyz, conf3d, rig, n_stages, stage_cfgs, opt_cfg, stats, st, on ? temporal_w_host : nullptr);
}

// The view problems of a mvs_refine_cameras call: the frames with a finite row, ascending (body), grouped by rig in call
// order (frames), and one problem per view 1 .. V_r - 1 of every rig with such frames, a work item per frame of its rig (ps)
struct CameraPlan {
    std::vector<int> body, frames;
    std::vector<CameraProblem> prob;
    ProblemSet ps;
};

// What mvs_refine_cameras and mvs_debug_camera_closure check before anything changes (who: the entry point called), and the
// stage's LossParams (3-D term as the call says)
static int camera_check(mvs_ctx* ctx, const char* who, const mvs_frame_stream* s, const int* rig, const mvs_loss_config* stage,
                        int H, LossParams* lp, cudaStream_t st) {
    if (int rc = check_ready(ctx, who)) return rc;
    if (!s || !stage) return set_error(ctx, MVS_ERR_INVALID, "%s: NULL argument", who);
    if (s->n_frames < 1) return set_error(ctx, MVS_ERR_INVALID, "%s: n_frames must be >= 1 (got %d)", who, s->n_frames);
    if (!s->params || !s->gt_uv || !s->conf || !s->joint_weights)
        return set_error(ctx, MVS_ERR_INVALID, "%s: params, gt_uv, conf and joint_weights are required", who);
    if (!s->gt_xyz != !s->conf3d) return set_error(ctx, MVS_ERR_INVALID, "%s: gt_xyz and conf3d go together", who);
    if (ctx->exec_mode == 1 || H > 100 || !resident_supported(ctx))
        return set_error(ctx, MVS_ERR_UNSUPPORTED, "%s: the held keypoints come from the frame-resident closure, and the body step "
                                                   "is a frame stream (exec mode 1, history_size > 100, or a model the "
                                                   "frame-resident kernels do not take)", who);
    std::vector<LossParams> lps;
    std::vector<int> ends;
    int rc = stage_table(ctx, who, 1, stage, s->gt_xyz ? 1 : 0, &lps);
    if (!rc) rc = stream_runs(ctx, who, lps, H, kMaxStages, &ends);
    if (!rc) rc = check_stream_rigs(ctx, who, rig, s->n_frames, st);
    if (rc) return rc;
    *lp = lps[0];
    return MVS_OK;
}

// The call's plan (finite rows and rigs read back once) and its scratch on the device
static int camera_plan(mvs_ctx* ctx, const mvs_frame_stream* s, const int* rig, CameraPlan* plan, cudaStream_t st) {
    const int F = s->n_frames, nr = (int)ctx->rigs.size();
    SeqState& h = seq_state(ctx);
    int rc;
    if ((rc = dev_grow(ctx, h.fin, (size_t)F)) || (rc = launch_row_finite(ctx, s->params, F, h.fin.p, st))) return rc;
    std::vector<int> fin((size_t)F), rg((size_t)F, 0);
    MVS_CUDA_OK(ctx, cudaMemcpyAsync(fin.data(), h.fin.p, (size_t)F * sizeof(int), cudaMemcpyDeviceToHost, st));
    if (rig) MVS_CUDA_OK(ctx, cudaMemcpyAsync(rg.data(), rig, (size_t)F * sizeof(int), cudaMemcpyDeviceToHost, st));
    MVS_CUDA_OK(ctx, cudaStreamSynchronize(st));
    *plan = CameraPlan{};
    std::vector<std::vector<int>> of((size_t)nr);
    for (int f = 0; f < F; ++f)
        if (fin[f]) { plan->body.push_back(f); of[rg[f]].push_back(f); }
    ProblemSet& ps = plan->ps;
    ps.beg.assign(1, 0);
    for (int r = 0; r < nr; ++r) {
        const int fbeg = (int)plan->frames.size(), nf = (int)of[r].size();
        plan->frames.insert(plan->frames.end(), of[r].begin(), of[r].end());
        if (nf == 0) continue;
        for (int v = 1; v < ctx->rigs[r].num_views; ++v) {
            plan->prob.push_back(CameraProblem{r, v, fbeg});
            ps.beg.push_back(ps.beg.back() + nf);
        }
    }
    const size_t P = plan->prob.size(), n = plan->body.size();
    ps.on.assign(P, 1);
    ps.ent = PartEntries{6, {kOffOrient, kOffOrient + 1, kOffOrient + 2, kOffTransl, kOffTransl + 1, kOffTransl + 2}};
    if ((rc = dev_grow(ctx, h.body, std::max<size_t>(n, 1))) || (rc = dev_grow(ctx, h.held, (size_t)F * ctx->m.K * 3)) ||
        (rc = dev_grow(ctx, h.cam_frames, std::max<size_t>(n, 1))) || (rc = dev_grow(ctx, h.prob, std::max<size_t>(P, 1))) ||
        (rc = dev_grow(ctx, h.cr, std::max<size_t>(P, 1))))
        return rc;
    MVS_CUDA_OK(ctx, cudaMemcpyAsync(h.body.p, plan->body.data(), n * sizeof(int), cudaMemcpyHostToDevice, st));
    MVS_CUDA_OK(ctx, cudaMemcpyAsync(h.cam_frames.p, plan->frames.data(), n * sizeof(int), cudaMemcpyHostToDevice, st));
    MVS_CUDA_OK(ctx, cudaMemcpyAsync(h.prob.p, plan->prob.data(), P * sizeof(CameraProblem), cudaMemcpyHostToDevice, st));
    return problem_scratch(ctx, ps, st);
}

// Each problem's calibrated camera, from the context's rig table as it stands (host copy): view 1 moves on the sphere about view
// 0's centre through its own centre, with a basis computed in double
static int camera_refs(mvs_ctx* ctx, const CameraPlan& plan, cudaStream_t st) {
    std::vector<CamRefine> cr(plan.prob.size());
    auto centre = [](const CamF& c, double* C) {                   // -R^T t
        for (int i = 0; i < 3; ++i) C[i] = -((double)c.R[i] * c.t[0] + (double)c.R[3 + i] * c.t[1] + (double)c.R[6 + i] * c.t[2]);
    };
    for (size_t p = 0; p < cr.size(); ++p) {
        const Rig& rg = ctx->rigs[plan.prob[p].rig];
        const CamF& cam = rg.cam[plan.prob[p].view];
        CamRefine& c = cr[p];
        memset(&c, 0, sizeof(c));
        memcpy(c.R0, cam.R, sizeof(c.R0));
        memcpy(c.t0, cam.t, sizeof(c.t0));
        if (plan.prob[p].view != 1) continue;
        c.sphere = 1;
        double C0[3], C1[3], d[3], r = 0.0;
        centre(rg.cam[0], C0);
        centre(cam, C1);
        for (int i = 0; i < 3; ++i) { d[i] = C1[i] - C0[i]; r += d[i] * d[i]; }
        r = sqrt(r);
        if (!(r > 0.0)) continue;                                  // coincident centres: view 1 only rotates
        for (int i = 0; i < 3; ++i) d[i] /= r;
        const int k = fabs(d[0]) <= fabs(d[1]) && fabs(d[0]) <= fabs(d[2]) ? 0 : fabs(d[1]) <= fabs(d[2]) ? 1 : 2;
        double a[3] = {0.0, 0.0, 0.0}, e1[3], e2[3];
        a[k] = 1.0;                                                // the axis least aligned with d
        e1[0] = d[1] * a[2] - d[2] * a[1]; e1[1] = d[2] * a[0] - d[0] * a[2]; e1[2] = d[0] * a[1] - d[1] * a[0];
        const double l = sqrt(e1[0] * e1[0] + e1[1] * e1[1] + e1[2] * e1[2]);
        for (int i = 0; i < 3; ++i) e1[i] /= l;
        e2[0] = d[1] * e1[2] - d[2] * e1[1]; e2[1] = d[2] * e1[0] - d[0] * e1[2]; e2[2] = d[0] * e1[1] - d[1] * e1[0];
        for (int i = 0; i < 3; ++i) {
            c.E[2 * i] = (float)(r * e1[i]);
            c.E[2 * i + 1] = (float)(r * e2[i]);
            c.n[i] = (float)(r * d[i]);
        }
    }
    if (!cr.empty())
        MVS_CUDA_OK(ctx, cudaMemcpyAsync(ctx->sstream->cr.p, cr.data(), cr.size() * sizeof(CamRefine), cudaMemcpyHostToDevice, st));
    return MVS_OK;
}

static CameraArgs camera_args(mvs_ctx* ctx, const FrameInputs& in) {
    SeqState& h = *ctx->sstream;
    return CameraArgs{in, h.held.p, h.cr.p, h.prob.p, h.cam_frames.p, ctx->rigs_dev.p, ctx->m.K};
}

// The camera step: every view problem from a zero update (solve_problems with the camera closure); then the solved cameras into
// the table and its host copy
static int solve_cameras(mvs_ctx* ctx, const CameraPlan& plan, const ChunkClosure& closure, const LossParams& lp,
                         const mvs_lbfgs_config* c, mvs_lbfgs_stats* stats, cudaStream_t st) {
    const int P = (int)plan.prob.size();
    if (P == 0) return MVS_OK;
    SeqState& h = *ctx->sstream;
    MVS_CUDA_OK(ctx, cudaMemsetAsync(h.rows.p, 0, (size_t)P * kParams * sizeof(float), st));
    if (int rc = solve_problems(ctx, plan.ps, closure, lp, c, nullptr, stats, st)) return rc;
    if (int rc = launch_camera_write(ctx, h.cr.p, h.prob.p, P, h.rows.p, st)) return rc;
    MVS_CUDA_OK(ctx, cudaMemcpyAsync(ctx->rigs.data(), ctx->rigs_dev.p, ctx->rigs.size() * sizeof(Rig), cudaMemcpyDeviceToHost, st));
    MVS_CUDA_OK(ctx, cudaStreamSynchronize(st));
    return MVS_OK;
}

// mvs_refine_cameras (DESIGN.md section 4)
static int refine_cameras(mvs_ctx* ctx, const mvs_frame_stream* s, const int* rig, const mvs_loss_config* stage,
                          const mvs_lbfgs_config* opt_cfg, int n_sweeps, float* R_host, float* t_host, mvs_lbfgs_stats* camera_stats,
                          mvs_lbfgs_stats* pose_stats, cudaStream_t st) {
    static const char* who = "mvs_refine_cameras";
    LossParams lp;
    int rc = check_ready(ctx, who);
    if (!rc) rc = check_sweeps(ctx, who, opt_cfg, n_sweeps);
    if (!rc) rc = camera_check(ctx, who, s, rig, stage, history_size(opt_cfg), &lp, st);
    if (rc) return rc;
    const FrameInputs in{s->n_frames, s->gt_uv, s->conf, s->joint_weights, s->gt_xyz, s->conf3d, rig};
    if ((rc = start_sweeps(ctx, in.n, s->final_loss, camera_stats, pose_stats, st))) return rc;
    CameraPlan plan;
    if ((rc = camera_plan(ctx, s, rig, &plan, st))) return rc;
    SeqState& h = *ctx->sstream;
    const CameraArgs a = camera_args(ctx, in);
    const ChunkClosure closure = [&](const ProblemChunk& c, const LbfgsState& S) { return launch_camera_closure(ctx, a, c, lp, S, st); };
    stream_call_begin(ctx);
    for (int sweep = 0; sweep < n_sweeps && !rc; ++sweep) {
        if ((rc = launch_camera_joints(ctx, in, s->params, h.body.p, (int)plan.body.size(), lp, h.held.p, st)) ||
            (rc = camera_refs(ctx, plan, st)) || (rc = solve_cameras(ctx, plan, closure, lp, opt_cfg, camera_stats, st)))
            break;
        rc = refit_bodies(ctx, who, in, s->params, s->final_loss, plan.body, stage, opt_cfg, pose_stats, st);
    }
    stream_call_end(ctx, lp);
    if (rc) return rc;
    const int V = ctx->vmax;
    for (size_t r = 0; r < ctx->rigs.size(); ++r)
        for (int v = 0; v < V; ++v) {
            if (R_host) memcpy(R_host + (r * V + v) * 9, ctx->rigs[r].cam[v].R, 9 * sizeof(float));
            if (t_host) memcpy(t_host + (r * V + v) * 3, ctx->rigs[r].cam[v].t, 3 * sizeof(float));
        }
    return MVS_OK;
}

void release_fit_state(mvs_ctx* ctx) {
    release(ctx->lbfgs);
    release(ctx->fstream);
    delete ctx->sstream;
    ctx->lbfgs = nullptr;
    ctx->fstream = nullptr;
    ctx->sstream = nullptr;
}

}  // namespace mvs

using namespace mvs;

extern "C" {

int mvs_lbfgs_run(mvs_ctx* ctx, float* params_dev, float* final_loss_dev, const mvs_lbfgs_config* cfg,
                  mvs_lbfgs_stats* stats, void* stream) {
    if (int rc = begin_batch_call(ctx, "mvs_lbfgs_run", true, true, params_dev && cfg, stats)) return rc;
    return run_stage(ctx, params_dev, final_loss_dev, cfg, stats, (cudaStream_t)stream, RunOpts{});
}

int mvs_lbfgs_step(mvs_ctx* ctx, float* params_dev, float* loss_dev, float* last_grad_dev, const mvs_lbfgs_config* cfg,
                   int reset, mvs_lbfgs_stats* stats, void* stream) {
    if (int rc = begin_batch_call(ctx, "mvs_lbfgs_step", true, true, params_dev && cfg, stats)) return rc;
    if (!reset && !ctx->lbfgs) return set_error(ctx, MVS_ERR_INVALID, "mvs_lbfgs_step: reset=0 before any step");
    RunOpts o;
    o.step = true;
    o.reset = reset != 0;
    o.last_grad = last_grad_dev;
    return run_stage(ctx, params_dev, loss_dev, cfg, stats, (cudaStream_t)stream, o);
}

int mvs_fit_seq_temporal(mvs_ctx* ctx, float* params_dev, int n_stages, const mvs_loss_config* stage_cfgs,
                         const mvs_lbfgs_config* opt_cfg, const unsigned char* warm_host, const float* prev_dev,
                         const float* temporal_w_host, float* final_loss_dev, mvs_lbfgs_stats* stats, void* stream) {
    return fit_batch(ctx, "mvs_fit_seq_temporal", params_dev, n_stages, stage_cfgs, opt_cfg, warm_host, prev_dev, temporal_w_host,
                     final_loss_dev, stats, stream);
}

int mvs_fit_seq(mvs_ctx* ctx, float* params_dev, int n_stages, const mvs_loss_config* stage_cfgs, const mvs_lbfgs_config* opt_cfg,
                const unsigned char* warm_host, float* final_loss_dev, mvs_lbfgs_stats* stats, void* stream) {
    return fit_batch(ctx, "mvs_fit_seq", params_dev, n_stages, stage_cfgs, opt_cfg, warm_host, nullptr, nullptr, final_loss_dev,
                     stats, stream);
}

int mvs_fit(mvs_ctx* ctx, float* params_dev, int n_stages, const mvs_loss_config* stage_cfgs, const mvs_lbfgs_config* opt_cfg,
            float* final_loss_dev, mvs_lbfgs_stats* stats, void* stream) {
    return fit_batch(ctx, "mvs_fit", params_dev, n_stages, stage_cfgs, opt_cfg, nullptr, nullptr, nullptr, final_loss_dev, stats,
                     stream);
}

int mvs_fit_stream_rigs(mvs_ctx* ctx, const mvs_frame_stream* s, const int* rig_dev, int n_stages, const mvs_loss_config* stage_cfgs,
                        const mvs_lbfgs_config* opt_cfg, mvs_lbfgs_stats* stats, void* stream) {
    return fit_stream(ctx, "mvs_fit_stream_rigs", s, rig_dev, n_stages, stage_cfgs, opt_cfg, stats, stream);
}

int mvs_fit_stream(mvs_ctx* ctx, const mvs_frame_stream* s, int n_stages, const mvs_loss_config* stage_cfgs,
                   const mvs_lbfgs_config* opt_cfg, mvs_lbfgs_stats* stats, void* stream) {
    return fit_stream(ctx, "mvs_fit_stream", s, nullptr, n_stages, stage_cfgs, opt_cfg, stats, stream);
}

int mvs_fit_seq_stream_temporal(mvs_ctx* ctx, const mvs_sequence_stream* s, const float* gt_xyz, const float* conf3d,
                                const int* rig_dev, const float* temporal_w_host, int n_stages, const mvs_loss_config* stage_cfgs,
                                const mvs_lbfgs_config* opt_cfg, mvs_lbfgs_stats* stats, void* stream) {
    return fit_seq_stream(ctx, "mvs_fit_seq_stream_temporal", s, gt_xyz, conf3d, rig_dev, temporal_w_host, n_stages, stage_cfgs,
                          opt_cfg, stats, stream);
}

int mvs_fit_seq_stream_rigs(mvs_ctx* ctx, const mvs_sequence_stream* s, const float* gt_xyz, const float* conf3d, const int* rig_dev,
                            int n_stages, const mvs_loss_config* stage_cfgs, const mvs_lbfgs_config* opt_cfg, mvs_lbfgs_stats* stats,
                            void* stream) {
    return fit_seq_stream(ctx, "mvs_fit_seq_stream_rigs", s, gt_xyz, conf3d, rig_dev, nullptr, n_stages, stage_cfgs, opt_cfg, stats,
                          stream);
}

int mvs_fit_seq_stream3d(mvs_ctx* ctx, const mvs_sequence_stream* s, const float* gt_xyz, const float* conf3d, int n_stages,
                         const mvs_loss_config* stage_cfgs, const mvs_lbfgs_config* opt_cfg, mvs_lbfgs_stats* stats, void* stream) {
    return fit_seq_stream(ctx, "mvs_fit_seq_stream3d", s, gt_xyz, conf3d, nullptr, nullptr, n_stages, stage_cfgs, opt_cfg, stats,
                          stream);
}

int mvs_fit_seq_stream(mvs_ctx* ctx, const mvs_sequence_stream* s, int n_stages, const mvs_loss_config* stage_cfgs,
                       const mvs_lbfgs_config* opt_cfg, mvs_lbfgs_stats* stats, void* stream) {
    return fit_seq_stream(ctx, "mvs_fit_seq_stream", s, nullptr, nullptr, nullptr, nullptr, n_stages, stage_cfgs, opt_cfg, stats,
                          stream);
}

int mvs_fit_shared_shape(mvs_ctx* ctx, const mvs_sequence_stream* s, const float* gt_xyz, const float* conf3d, const int* rig_dev,
                         const mvs_loss_config* stage, const mvs_lbfgs_config* opt_cfg, int n_sweeps, float* seq_loss_dev,
                         mvs_lbfgs_stats* shape_stats, mvs_lbfgs_stats* pose_stats, void* stream) {
    static const char* who = "mvs_fit_shared_shape";
    const cudaStream_t st = (cudaStream_t)stream;
    LossParams lp;
    ProblemSet ps;
    ShapeArgs a;
    int rc = check_seq_stream(ctx, who, s, gt_xyz, conf3d, rig_dev, st);
    if (!rc) rc = check_sweeps(ctx, who, opt_cfg, n_sweeps);
    if (!rc) rc = shape_prepare(ctx, who, s, gt_xyz, conf3d, rig_dev, stage, history_size(opt_cfg), &lp, &ps, &a, st);
    if (!rc) rc = start_sweeps(ctx, a.in.n, s->final_loss, shape_stats, pose_stats, st);
    if (rc) return rc;
    const int NS = s->n_sequences, F = a.in.n;
    SeqState& h = *ctx->sstream;
    mvs_loss_config pose_cfg = *stage;                                   // the pose step: the shared entries held
    pose_cfg.frozen_mask |= 1u | (a.share_scale ? 16u : 0u);
    const ChunkClosure closure = [&](const ProblemChunk& c, const LbfgsState& S) { return launch_shape_closure(ctx, a, c, lp, S, st); };
    std::vector<int> frames;
    for (int sweep = 0; sweep < n_sweeps && !rc; ++sweep) {
        MVS_LAUNCH(ctx, KID_MISC, st, shape_consensus_kernel<<<NS, 32, 0, st>>>(s->params, h.off.p, a.share_scale, h.rows.p, h.ok.p));
        MVS_CUDA_OK(ctx, cudaMemcpyAsync(ps.on.data(), h.ok.p, (size_t)NS * sizeof(int), cudaMemcpyDeviceToHost, st));
        MVS_CUDA_OK(ctx, cudaStreamSynchronize(st));
        if ((rc = solve_problems(ctx, ps, closure, lp, opt_cfg, seq_loss_dev, shape_stats, st))) break;
        MVS_LAUNCH(ctx, KID_MISC, st, shape_write_kernel<<<(F + 127) / 128, 128, 0, st>>>(s->params, h.item_of.p, h.rows.p, h.ok.p, F,
                                                                                        a.share_scale));
        frames.clear();
        for (int q = 0; q < NS; ++q)
            if (ps.on[q])
                for (int f = ps.beg[q]; f < ps.beg[q + 1]; ++f) frames.push_back(f);
        rc = refit_bodies(ctx, who, a.in, s->params, s->final_loss, frames, &pose_cfg, opt_cfg, pose_stats, st);
    }
    return rc;
}

int mvs_refine_cameras(mvs_ctx* ctx, const mvs_frame_stream* s, const int* rig_dev, const mvs_loss_config* stage,
                       const mvs_lbfgs_config* opt_cfg, int n_sweeps, float* R_host, float* t_host, mvs_lbfgs_stats* camera_stats,
                       mvs_lbfgs_stats* pose_stats, void* stream) {
    return refine_cameras(ctx, s, rig_dev, stage, opt_cfg, n_sweeps, R_host, t_host, camera_stats, pose_stats, (cudaStream_t)stream);
}

int mvs_fit_host(mvs_ctx* ctx, float* params_host, const float* gt_uv_host, const float* conf_host,
                 const float* joint_weights_host, int n_stages, const mvs_loss_config* stage_cfgs,
                 const mvs_lbfgs_config* opt_cfg, float* final_loss_host, mvs_lbfgs_stats* stats, void* stream) {
    static const char* who = "mvs_fit_host";
    int rc = begin_batch_call(ctx, who, false, false, params_host && gt_uv_host && conf_host && joint_weights_host && n_stages > 0 &&
                              stage_cfgs && opt_cfg, stats);
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    const int B = ctx->ws.B;
    if ((rc = mvs_set_keypoints(ctx, gt_uv_host, conf_host, joint_weights_host, 0, stream))) return rc;
    const int H = history_size(opt_cfg);
    if (H > 128) return set_error(ctx, MVS_ERR_INVALID, "%s: history_size must be <= 128", who);
    if ((rc = ensure_state(ctx, H))) return rc;
    LbfgsState& S = *ctx->lbfgs;
    float* x = S.x_fit;                              // [B][86] device copy of the parameters
    MVS_CUDA_OK(ctx, cudaMemcpyAsync(x, params_host, (size_t)B * kParams * sizeof(float), cudaMemcpyHostToDevice, st));
    if ((rc = run_fit(ctx, who, x, n_stages, stage_cfgs, opt_cfg, S.final_fit, stats, st))) return rc;
    MVS_CUDA_OK(ctx, cudaMemcpyAsync(params_host, x, (size_t)B * kParams * sizeof(float), cudaMemcpyDeviceToHost, st));
    if (final_loss_host)
        MVS_CUDA_OK(ctx, cudaMemcpyAsync(final_loss_host, S.final_fit, (size_t)B * sizeof(float), cudaMemcpyDeviceToHost, st));
    MVS_CUDA_OK(ctx, cudaStreamSynchronize(st));
    return MVS_OK;
}

// Testing aids, not part of the ABI (tests/test_gpu_lbfgs_transitions.py): they let a test drive the optimiser's state machine
// from the host, one transition at a time, and compare every transition with a float64 restatement.
//
// mvs_debug_lbfgs_layout: sizeof(FrameScalars) and the byte offset of each of its fields, in declaration order (arrays: the
// offset of their first element), so that a host mirror of the struct cannot drift from it.  Needs no context and no device.
extern "C" int mvs_debug_lbfgs_layout(int* out) {
#define MVS_OFF(f) (int)offsetof(FrameScalars, f)
    const int v[] = {(int)sizeof(FrameScalars),
                     MVS_OFF(phase), MVS_OFF(outer_n), MVS_OFF(state_n_iter), MVS_OFF(n_iter), MVS_OFF(current_evals),
                     MVS_OFF(ls_iter), MVS_OFF(ls_evals), MVS_OFF(ls_first), MVS_OFF(low), MVS_OFF(high), MVS_OFF(done),
                     MVS_OFF(insuf), MVS_OFF(have_prev), MVS_OFF(hist_len), MVS_OFF(hist_head), MVS_OFF(nan_flag),
                     MVS_OFF(pushed_slot), MVS_OFF(stage), MVS_OFF(stage_end), MVS_OFF(nan_acc),
                     MVS_OFF(t), MVS_OFF(H_diag), MVS_OFF(gtd0), MVS_OFF(t_prev), MVS_OFF(gtd_prev), MVS_OFF(d_norm),
                     MVS_OFF(bt), MVS_OFF(bgtd), MVS_OFF(bf),
                     MVS_OFF(loss), MVS_OFF(prev_loss), MVS_OFF(orig_loss), MVS_OFF(f_prev), MVS_OFF(mon_prev_loss),
                     MVS_OFF(final_loss), MVS_OFF(iters), MVS_OFF(evals)};
#undef MVS_OFF
    const int n = (int)(sizeof(v) / sizeof(v[0]));
    if (out)
        for (int i = 0; i < n; ++i) out[i] = v[i];
    return n;
}

// mvs_debug_lbfgs_state: copies the context's optimiser state of all B frames (history size H) to (write == 0) or from
// (write != 0) host buffers; null pointers are skipped.  sc [B] FrameScalars; x [B][86] (the parameters that
// mvs_debug_lbfgs_advance updates); g, d, prev_g, x_init, g_prev [B][86]; bg [B][2][86]; the ring hist_s, hist_y [B][H][86]
// and ro [B][H]; gram [B][16][8][8]; x_eval, g_eval [B][86]; loss_eval [B].  A write first allocates the state for H
// (ensure_state); a read needs the state to exist with history size H.  Synchronises the device first.
extern "C" int mvs_debug_lbfgs_state(mvs_ctx* ctx, int write, int H, void* sc, float* x, float* g, float* d, float* prev_g,
                                     float* x_init, float* g_prev, float* bg, float* hist_s, float* hist_y, float* ro,
                                     float* gram, float* x_eval, float* g_eval, float* loss_eval) {
    if (!ctx) return set_error(nullptr, MVS_ERR_INVALID, "ctx is NULL");
    if (ctx->ws.B <= 0) return set_error(ctx, MVS_ERR_INVALID, "mvs_debug_lbfgs_state: set the batch first");
    if (H < 1 || H > 128) return set_error(ctx, MVS_ERR_INVALID, "mvs_debug_lbfgs_state: history size %d", H);
    MVS_CUDA_OK(ctx, cudaSetDevice(ctx->device));
    MVS_CUDA_OK(ctx, cudaDeviceSynchronize());
    if (write) {
        if (int rc = ensure_state(ctx, H)) return rc;
    } else if (!ctx->lbfgs || ctx->lbfgs->H != H) {
        return set_error(ctx, MVS_ERR_INVALID, "mvs_debug_lbfgs_state: no optimiser state with history size %d", H);
    }
    const LbfgsState& S = *ctx->lbfgs;
    const size_t B = (size_t)S.B, V = B * kParams * sizeof(float), R = V * (size_t)H;
    struct { void* host; void* dev; size_t bytes; } cp[] = {
        {sc, S.sc, B * sizeof(FrameScalars)}, {x, S.x_fit, V}, {g, S.g, V}, {d, S.d, V}, {prev_g, S.prev_g, V},
        {x_init, S.x_init, V}, {g_prev, S.g_prev, V}, {bg, S.bg, 2 * V}, {hist_s, S.hist_s, R}, {hist_y, S.hist_y, R},
        {ro, S.ro, B * H * sizeof(float)}, {gram, S.gram, B * kGramFloats * sizeof(float)}, {x_eval, S.x_eval, V},
        {g_eval, S.g_eval, V}, {loss_eval, S.loss_eval, B * sizeof(float)}};
    for (auto& c : cp)
        if (c.host)
            MVS_CUDA_OK(ctx, write ? cudaMemcpy(c.dev, c.host, c.bytes, cudaMemcpyHostToDevice)
                                   : cudaMemcpy(c.host, c.dev, c.bytes, cudaMemcpyDeviceToHost));
    return MVS_OK;
}

// mvs_debug_lbfgs_advance: one launch of the production lbfgs_advance_kernel over every frame of the context that is not
// PH_DONE (the active list of lbfgs_compact_kernel), on the context's state, with the LbfgsCfg that begin_run builds from cfg
// and the given step_mode and pose_len (69: body_pose, 32: pose_embedding).  The parameters it updates are the state's x
// (mvs_debug_lbfgs_state).  Synchronises before it returns.
extern "C" int mvs_debug_lbfgs_advance(mvs_ctx* ctx, const mvs_lbfgs_config* c, int step_mode, int pose_len) {
    if (!ctx) return set_error(nullptr, MVS_ERR_INVALID, "ctx is NULL");
    if (!c || ctx->ws.B <= 0) return set_error(ctx, MVS_ERR_INVALID, "mvs_debug_lbfgs_advance: NULL config or no batch");
    MVS_CUDA_OK(ctx, cudaSetDevice(ctx->device));
    const cudaStream_t st = 0;
    LbfgsCfg cfg;
    if (int rc = begin_run(ctx, c, step_mode != 0, &ctx->loss, 1, &cfg, st)) return rc;
    cfg.step_mode = step_mode;
    LbfgsState& S = *ctx->lbfgs;
    Workspace& w = ctx->ws;
    const int B = w.B;
    MVS_LAUNCH(ctx, KID_MISC, st, iota2_kernel<<<(B + 255) / 256, 256, 0, st>>>(w.fidx, B, w.na));
    MVS_LAUNCH(ctx, KID_LBFGS_COMPACT, st, lbfgs_compact_kernel<<<1, 1024, 0, st>>>(S, B, w.fidx, w.na));
    MVS_LAUNCH(ctx, KID_LBFGS_ADVANCE, st, lbfgs_advance_kernel<<<B, 32, 0, st>>>(S, cfg, S.x_fit, w.fidx, w.na, pose_len));
    MVS_LAUNCH(ctx, KID_MISC, st, iota2_kernel<<<(B + 255) / 256, 256, 0, st>>>(w.fidx, B, w.na));
    MVS_CUDA_OK(ctx, cudaStreamSynchronize(st));
    MVS_CUDA_OK(ctx, cudaGetLastError());
    return MVS_OK;
}

// mvs_debug_shape_closure (tests/test_gpu_shared_shape.py): the shape closure of mvs_fit_shared_shape evaluated once, with the
// same arguments, at the shared rows rows_dev [S][86] (device; the shared entries are read): loss_dev [S] and grad_dev [S][86]
// (device) receive what the optimiser sees as loss_eval / g_eval of each sequence's problem.  Uses the context's optimiser state
// (history size 100 when there is none).  Synchronises.
extern "C" int mvs_debug_shape_closure(mvs_ctx* ctx, const mvs_sequence_stream* s, const float* gt_xyz, const float* conf3d,
                                       const int* rig_dev, const mvs_loss_config* stage, const float* rows_dev, float* loss_dev,
                                       float* grad_dev, void* stream) {
    static const char* who = "mvs_debug_shape_closure";
    const cudaStream_t st = (cudaStream_t)stream;
    LossParams lp;
    ProblemSet ps;
    ShapeArgs a;
    int rc = check_seq_stream(ctx, who, s, gt_xyz, conf3d, rig_dev, st);
    if (!rc && (!rows_dev || !loss_dev || !grad_dev)) rc = set_error(ctx, MVS_ERR_INVALID, "%s: NULL argument", who);
    if (!rc) rc = shape_prepare(ctx, who, s, gt_xyz, conf3d, rig_dev, stage, 100, &lp, &ps, &a, st);
    if (rc) return rc;
    const ChunkClosure closure = [&](const ProblemChunk& c, const LbfgsState& S) { return launch_shape_closure(ctx, a, c, lp, S, st); };
    return eval_problems(ctx, ps, closure, rows_dev, loss_dev, grad_dev, st);
}

// mvs_debug_camera_closure (tests/test_gpu_camera_refine.py): the camera closure of mvs_refine_cameras evaluated once, with the
// same arguments, the context's rig table as the calibration and the keypoints of s->params held.  *n_prob receives the number
// P of view problems and prob_host [P][2] (may be NULL) their (rig, view), in the order of the rows.  With rows_dev [P][86]
// (device; entries 10..12 and 82..84 are read) loss_dev [P] and grad_dev [P][86] (device) receive what the optimiser sees as
// loss_eval / g_eval of each problem; rows_dev NULL: only the problems are reported.  Uses the context's optimiser state
// (history size 100 when there is none).  Synchronises.
extern "C" int mvs_debug_camera_closure(mvs_ctx* ctx, const mvs_frame_stream* s, const int* rig_dev, const mvs_loss_config* stage,
                                        const float* rows_dev, float* loss_dev, float* grad_dev, int* prob_host, int* n_prob,
                                        void* stream) {
    static const char* who = "mvs_debug_camera_closure";
    const cudaStream_t st = (cudaStream_t)stream;
    LossParams lp;
    int rc = camera_check(ctx, who, s, rig_dev, stage, 100, &lp, st);
    if (!rc && (!n_prob || (rows_dev && (!loss_dev || !grad_dev)))) rc = set_error(ctx, MVS_ERR_INVALID, "%s: NULL argument", who);
    CameraPlan plan;
    if (!rc) rc = camera_plan(ctx, s, rig_dev, &plan, st);
    if (rc) return rc;
    const int P = (int)plan.prob.size();
    *n_prob = P;
    for (int p = 0; p < P && prob_host; ++p) { prob_host[2 * p] = plan.prob[p].rig; prob_host[2 * p + 1] = plan.prob[p].view; }
    if (!rows_dev || P == 0) return MVS_OK;
    const CameraArgs a = camera_args(ctx, FrameInputs{s->n_frames, s->gt_uv, s->conf, s->joint_weights, s->gt_xyz, s->conf3d, rig_dev});
    if ((rc = launch_camera_joints(ctx, a.in, s->params, ctx->sstream->body.p, (int)plan.body.size(), lp, ctx->sstream->held.p, st)) ||
        (rc = camera_refs(ctx, plan, st)))
        return rc;
    const ChunkClosure closure = [&](const ProblemChunk& c, const LbfgsState& S) { return launch_camera_closure(ctx, a, c, lp, S, st); };
    return eval_problems(ctx, plan.ps, closure, rows_dev, loss_dev, grad_dev, st);
}

}  // extern "C"
