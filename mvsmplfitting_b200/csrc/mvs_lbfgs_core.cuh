// L-BFGS / strong-Wolfe per-frame state machine shared by the batched kernel (mvs_lbfgs.cu) and the
// frame-resident kernel (mvs_resident.cu).  See mvs_lbfgs.cu for the reference line mapping.
#pragma once
#include "mvs_internal.cuh"

namespace mvs {

constexpr int kMaxStages = 16;
constexpr int kGramBlocks = 16;          // history ring slots / 8 (H <= 128)
constexpr int kGramFloats = kGramBlocks * 64;

enum Phase { PH_STEP_ENTRY = 0, PH_LS_BRACKET = 1, PH_LS_ZOOM = 2, PH_DONE = 3 };

struct FrameScalars {
    int phase, outer_n, state_n_iter, n_iter, current_evals;
    int ls_iter, ls_evals, ls_first, low, high, done, insuf, have_prev;
    int hist_len, hist_head, nan_flag;
    int pushed_slot;                 // ring slot written by the last advance call (-1: none)
    int stage;                       // index into the stage table of a multi-stage run (frames change stage on their own)
    int stage_end;                   // one past this frame's last entry of the table (warm-started frames own a different slice)
    int nan_acc;                     // NaN / Inf stops of the stages this frame already left
    float t, H_diag, gtd0, t_prev, gtd_prev, d_norm;
    float bt[2], bgtd[2], bf[2];
    float loss, prev_loss, orig_loss, f_prev, mon_prev_loss, final_loss;
    long long iters, evals;
};

// A frame starting on its slice rng = [first, end) of the stage table, with a fresh optimiser; an empty slice: the frame has
// no stage in this run and is done at once (its parameters stay)
__device__ __forceinline__ FrameScalars fresh_frame_scalars(int2 rng) {
    FrameScalars s;
    memset(&s, 0, sizeof(s));
    s.phase = rng.x < rng.y ? PH_STEP_ENTRY : PH_DONE;
    s.H_diag = 1.f;
    s.final_loss = __int_as_float(0x7fc00000);
    s.stage = rng.x; s.stage_end = rng.y;
    return s;
}

// A frame that finished stage k of a multi-stage run starts stage k + 1 at once, with a fresh optimiser (the reference
// builds one optimiser per stage, fitting.py / fit_single_frame) and the parameters it has: frames are independent
// problems, so nothing makes a fast frame wait for the slowest one at a stage boundary.
__device__ __forceinline__ void next_stage_scalars(FrameScalars& s) {
    FrameScalars n = fresh_frame_scalars(make_int2(s.stage + 1, s.stage_end));
    n.iters = s.iters; n.evals = s.evals; n.nan_acc = s.nan_acc + s.nan_flag;
    s = n;
}

// A retiring frame's iterations, evaluations and NaN / Inf stops, added to totals[0 .. 2]
__device__ __forceinline__ void add_frame_totals(long long* totals, const FrameScalars& s) {
    atomicAdd((unsigned long long*)&totals[0], (unsigned long long)s.iters);
    atomicAdd((unsigned long long*)&totals[1], (unsigned long long)s.evals);
    atomicAdd((unsigned long long*)&totals[2], (unsigned long long)(s.nan_flag + s.nan_acc));
}

struct LbfgsState {
    int B = 0, H = 0;
    float *g = nullptr, *d = nullptr, *prev_g = nullptr, *x_init = nullptr, *g_prev = nullptr, *bg = nullptr;
    float *hist_y = nullptr, *hist_s = nullptr, *ro = nullptr;
    float* gram = nullptr;           // [B][kGramFloats] s_i . y_j of pairs in the same 8-slot block of the history ring
    float *x_eval = nullptr, *loss_eval = nullptr, *g_eval = nullptr;
    FrameScalars* sc = nullptr;
    long long* totals = nullptr;     // [4] iters, evals, nan frames, real rounds
    float *x_fit = nullptr, *final_fit = nullptr;   // mvs_fit_host staging
    int* na_host = nullptr;          // pinned
    cudaEvent_t na_event[2] = {nullptr, nullptr};   // host side: active-count readback of the two chunks in flight
    LossParams* lp_tab = nullptr;    // [kMaxStages] loss parameters of the stages of the current run (device)
    LossParams* lp_tab_host = nullptr;   // pinned staging copy
};

struct LbfgsCfg {
    int max_outer, max_iter, max_eval, history, max_ls;
    int step_mode;                   // 1: exactly one LBFGS.step() per call (the outer run_fitting loop is the caller's)
    float lr, tol_grad, tol_change;
    double ftol, gtol;
};

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
// each lane owns elements lane, lane+32, lane+64 (< 86) of every 86-vector
#define VL(c, i) _Pragma("unroll") for (int c = 0; c < 3; ++c) for (int i = lane + 32 * c; i < kParams; i = kParams)
#define VLOOP(i) VL(_c, i)

__device__ __forceinline__ float vdot(const float* a, const float* b, int lane) {
    float p = 0.f;
    VLOOP(i) p = fmaf(a[i], b[i], p);
    return warp_sum(p);
}
__device__ __forceinline__ float vabsmax(const float* a, int lane) {
    float p = 0.f;
    VLOOP(i) p = fmaxf(p, fabsf(a[i]));
    return warp_max(p);
}

// Hard bound on one frame's closure evaluations in one stage (never reached by a terminating line search; a guard against
// hanging the GPU): every outer step costs at most 1 + max_eval + max_iter evaluations
__host__ __device__ __forceinline__ long long stage_eval_cap(const LbfgsCfg& cfg) {
    return (long long)cfg.max_outer * (cfg.max_eval + cfg.max_iter + 2) + 8;
}

// After an optimiser step of one warp: a frame that is done and has another stage in its slice moves on to it, its next
// evaluation at the parameters it has (x_eval <- x)
__device__ __forceinline__ void advance_stage_if_done(FrameScalars& s, float* x_eval, const float* x, int lane) {
    if (s.phase == PH_DONE && s.stage + 1 < s.stage_end) {
        next_stage_scalars(s);
        VLOOP(i) x_eval[i] = x[i];
        __syncwarp();
    }
}

// lbfgs_ls.py:11-36.  Python's min(max(pos, lo), hi) keeps `pos` when a comparison with NaN fails.
static __device__ __forceinline__ float cubic_interpolate(float x1, float f1, float g1, float x2, float f2, float g2, bool has_bounds,
                                   float lo, float hi) {
    if (!has_bounds) { if (x1 <= x2) { lo = x1; hi = x2; } else { lo = x2; hi = x1; } }
    const float num = (float)(3.0 * ((double)f1 - (double)f2));
    const float d1 = (g1 + g2) - num / (x1 - x2);
    const float d2sq = d1 * d1 - g1 * g2;
    if (d2sq >= 0.f) {
        const float d2 = sqrtf(d2sq);
        float pos;
        if (x1 <= x2) pos = x2 - (x2 - x1) * ((g2 + d2 - d1) / (g2 - g1 + 2.f * d2));
        else pos = x1 - (x1 - x2) * ((g1 + d2 - d1) / (g1 - g2 + 2.f * d2));
        float r = pos;
        if (lo > r) r = lo;
        if (hi < r) r = hi;
        return r;
    }
    return (lo + hi) / 2.f;
}


struct LbfgsPtrs {
    float *x, *g, *d, *prev_g, *x_init, *g_prev, *bg0, *bg1, *hy, *hs, *ro, *al, *x_eval;
    const float* g_new;
    int H;
    float* gram;        // [kGramFloats] block Gram entries (shared or global)
    float* scratch;     // [96] shared-memory scratch of the two-loop recursion (q vector + 8 coefficients)
};

// 8 groups of 4 lanes: group u takes one history pair, its lanes split the 86 elements (i = sub + 4 e)
__device__ __forceinline__ float group_dot(const float* a, const float* b, int sub) {
    float p0 = 0.f, p1 = 0.f;
#pragma unroll
    for (int e = 0; e < 22; e += 2) {
        const int i0 = sub + 4 * e, i1 = sub + 4 * (e + 1);
        if (i0 < kParams) p0 = fmaf(a[i0], b[i0], p0);
        if (i1 < kParams) p1 = fmaf(a[i1], b[i1], p1);
    }
    float p = p0 + p1;
    p += __shfl_xor_sync(0xffffffffu, p, 1);
    p += __shfl_xor_sync(0xffffffffu, p, 2);
    return p;
}

// One warp walks ONE frame's optimiser from "closure result (f_new, g_new) available" to its next closure
// request (x_eval written, s.phase says what is pending) or to PH_DONE.  Pointers may be global or shared.
// pose_len: entries of the pose slot that belong to the optimised tensor -- 69 (body_pose) or 32 (pose_embedding, use_vposer = 2);
// only run_fitting's gtol test looks at tensors one by one.
__device__ __forceinline__ void lbfgs_advance_core(FrameScalars& s, const LbfgsPtrs& P, const float f_new,
                                                   const LbfgsCfg& cfg, const int lane, const int pose_len = kOffTransl - kOffPose) {
    float* const x = P.x; float* const g = P.g; float* const d = P.d; float* const prev_g = P.prev_g;
    float* const x_init = P.x_init; float* const g_prev = P.g_prev; float* const bg0 = P.bg0; float* const bg1 = P.bg1;
    float* const hy = P.hy; float* const hs = P.hs; float* const ro = P.ro; float* const al = P.al;
    float* const x_eval = P.x_eval; const float* const g_new = P.g_new;
    const float c1 = 1e-4f, c2 = 0.9f;
    s.pushed_slot = -1;
    s.evals++;
    enum { L_STEP_ENTRY, L_LS_BRACKET, L_LS_ZOOM, L_ITER_BEGIN, L_ZOOM_INIT, L_ZOOM_HEAD, L_LS_FINISH, L_STEP_END,
           L_REQ_LS, L_FINISH, L_EXIT };
    int label = s.phase == PH_STEP_ENTRY ? L_STEP_ENTRY : (s.phase == PH_LS_BRACKET ? L_LS_BRACKET : L_LS_ZOOM);
    float gtd_new = 0.f;

    while (label != L_EXIT) {
        switch (label) {
        case L_STEP_ENTRY: {                                   // lbfgs_ls.py:279-290
            s.orig_loss = f_new;
            s.loss = f_new;
            s.current_evals = 1;
            VLOOP(i) g[i] = g_new[i];
            __syncwarp();
            if (vabsmax(g, lane) <= cfg.tol_grad) { label = L_STEP_END; break; }
            s.n_iter = 0;
            label = L_ITER_BEGIN;
            break;
        }
        case L_ITER_BEGIN: {                                   // lbfgs_ls.py:304-379
            s.n_iter++;
            s.state_n_iter++;
            s.iters++;
            if (s.state_n_iter == 1) {
                VLOOP(i) d[i] = -g[i];
                s.hist_len = 0; s.hist_head = 0;
                s.H_diag = 1.f;
            } else {
                // y = g - prev_g ; s = d * t
                float py = 0.f, pyy = 0.f;
                const int slot_new = (s.hist_head + s.hist_len) % P.H;
                float yv[3] = {0.f, 0.f, 0.f}, sv[3] = {0.f, 0.f, 0.f};
                VL(c, i) {
                    yv[c] = g[i] - prev_g[i];
                    sv[c] = d[i] * s.t;
                    py = fmaf(yv[c], sv[c], py);
                    pyy = fmaf(yv[c], yv[c], pyy);
                }
                const float ys = warp_sum(py), yy = warp_sum(pyy);
                if (ys > 1e-10f) {
                    int w = slot_new;
                    if (s.hist_len == P.H) { w = s.hist_head; s.hist_head = (s.hist_head + 1) % P.H; }   // drop the oldest
                    else s.hist_len++;
                    VL(c, i) { hy[(size_t)w * kParams + i] = yv[c]; hs[(size_t)w * kParams + i] = sv[c]; }
                    if (lane == 0) ro[w] = 1.f / ys;
                    s.pushed_slot = w;
                    s.H_diag = ys / yy;
                }
                __syncwarp();
                // Two-loop recursion, eight pairs at a time.  The textbook loop is a strictly serial chain of
                // (86-dot, warp reduction, axpy) per history pair: ~300 cycles x 2 x 100 pairs = 30 us for a full
                // history, the longest phase of a straggler's round.  Within a block of 8 consecutive ring slots the
                // products s_i . y_j are kept (updated when a pair is pushed), so the eight dots against the CURRENT
                // vector can be taken at once (8 groups of 4 lanes), the eight coefficients follow from an 8-step
                // scalar recurrence   a_u = ro_u (s_u.q - sum_{v<u} a_v s_u.y_v),   and the eight axpys are applied
                // together.  Same mathematics, different rounding; everything stays frame-local and deterministic.
#ifdef MVS_TL_MARK
                const long long tl_t0 = clock64();
#endif
                const int gq = lane >> 2, sub = lane & 3;
                float* const gram = P.gram;
                float* const qb = P.scratch;                     // [88] q / r vector
                float* const cb = P.scratch + 88;                // [8] coefficients of the current block
                if (s.pushed_slot >= 0) {                        // Gram row and column of the new pair
                    const int wp = s.pushed_slot, bw = wp >> 3, j = (bw << 3) + gq;
                    const bool live = j < P.H && (s.hist_len == P.H || j < s.hist_len);
                    const int jj = live ? j : wp;                // idle groups recompute the diagonal (and drop it)
                    const float g1 = group_dot(hs + (size_t)wp * kParams, hy + (size_t)jj * kParams, sub);
                    const float g2 = group_dot(hs + (size_t)jj * kParams, hy + (size_t)wp * kParams, sub);
                    if (live && sub == 0) { gram[bw * 64 + (wp & 7) * 8 + gq] = g1; gram[bw * 64 + gq * 8 + (wp & 7)] = g2; }
                    __syncwarp();
                }
                VLOOP(i) qb[i] = -g[i];
                __syncwarp();
                const int hl = s.hist_len;
                for (int k = hl - 1; k >= 0;) {                  // newest -> oldest
                    const int w_hi = (s.hist_head + k) % P.H;
                    const int cnt = min(k + 1, (w_hi & 7) + 1);
                    const bool on = gq < cnt;
                    const int wu = on ? w_hi - gq : w_hi;
                    float acc = group_dot(hs + (size_t)wu * kParams, qb, sub);
                    const float rou = ro[wu];
                    const float* grow = gram + (w_hi >> 3) * 64 + (wu & 7) * 8;      // s_wu . y_*
                    float a_mine = 0.f;
                    for (int v = 0; v < cnt; ++v) {
                        const float av = __shfl_sync(0xffffffffu, rou * acc, 4 * v);
                        if (gq == v) a_mine = av;
                        else if (on && gq > v) acc = fmaf(-av, grow[(w_hi - v) & 7], acc);
                    }
                    if (on && sub == 0) { al[k - gq] = a_mine; cb[gq] = a_mine; }
                    __syncwarp();
                    VLOOP(i) {
                        float qi = qb[i];
                        for (int v = 0; v < cnt; ++v) qi = fmaf(-cb[v], hy[(size_t)(w_hi - v) * kParams + i], qi);
                        qb[i] = qi;
                    }
                    __syncwarp();
                    k -= cnt;
                }
                VLOOP(i) qb[i] *= s.H_diag;
                __syncwarp();
                for (int k = 0; k < hl;) {                       // oldest -> newest
                    const int w_lo = (s.hist_head + k) % P.H;
                    const int cnt = min(min(hl - k, 8 - (w_lo & 7)), P.H - w_lo);
                    const bool on = gq < cnt;
                    const int wu = on ? w_lo + gq : w_lo;
                    float acc = group_dot(hy + (size_t)wu * kParams, qb, sub);
                    const float rou = ro[wu];
                    const float alu = on ? al[k + gq] : 0.f;
                    const float* gcol = gram + (w_lo >> 3) * 64 + (wu & 7);          // s_* . y_wu
                    float c_mine = 0.f;
                    for (int v = 0; v < cnt; ++v) {
                        const float cv = __shfl_sync(0xffffffffu, alu - rou * acc, 4 * v);
                        if (gq == v) c_mine = cv;
                        else if (on && gq > v) acc = fmaf(cv, gcol[((w_lo + v) & 7) * 8], acc);
                    }
                    if (on && sub == 0) cb[gq] = c_mine;
                    __syncwarp();
                    VLOOP(i) {
                        float qi = qb[i];
                        for (int v = 0; v < cnt; ++v) qi = fmaf(cb[v], hs[(size_t)(w_lo + v) * kParams + i], qi);
                        qb[i] = qi;
                    }
                    __syncwarp();
                    k += cnt;
                }
                float q[3] = {0.f, 0.f, 0.f};
                VL(c, i) q[c] = qb[i];
#ifdef MVS_TL_MARK
                if (lane == 0) MVS_TL_MARK(clock64() - tl_t0, hl);
#endif
                VL(c, i) d[i] = q[c];
            }
            VLOOP(i) prev_g[i] = g[i];
            s.prev_loss = s.loss;
            __syncwarp();
            if (s.state_n_iter == 1) {
                float p = 0.f;
                VLOOP(i) p += fabsf(g[i]);
                const float inv = 1.f / warp_sum(p);
                s.t = (inv < 1.f ? inv : 1.f) * cfg.lr;        // min(1., 1./|g|_1) * lr
            } else {
                s.t = cfg.lr;
            }
            const float gtd = vdot(g, d, lane);
            if (gtd > -cfg.tol_change) { label = L_STEP_END; break; }
            // ---- _strong_Wolfe prologue (lbfgs_ls.py:42-52)
            VLOOP(i) { x_init[i] = x[i]; g_prev[i] = g[i]; }
            s.d_norm = vabsmax(d, lane);
            s.gtd0 = gtd;
            s.t_prev = 0.f; s.f_prev = s.loss; s.gtd_prev = gtd;
            s.ls_iter = 0; s.ls_evals = 0; s.ls_first = 1; s.done = 0; s.insuf = 0;
            s.phase = PH_LS_BRACKET;
            label = L_REQ_LS;
            break;
        }
        case L_LS_BRACKET: {                                   // lbfgs_ls.py:53-101
            s.ls_evals++;
            gtd_new = vdot(g_new, d, lane);
            if (!s.ls_first) {
                s.ls_iter++;
                if (s.ls_iter == cfg.max_ls) {                 // lbfgs_ls.py:97-101
                    s.bt[0] = 0.f; s.bt[1] = s.t; s.bf[0] = s.loss; s.bf[1] = f_new;
                    s.bgtd[0] = s.gtd0; s.bgtd[1] = gtd_new;
                    VLOOP(i) { bg0[i] = g[i]; bg1[i] = g_new[i]; }
                    label = L_ZOOM_INIT;
                    break;
                }
            }
            s.ls_first = 0;
            const float armijo = s.loss + (c1 * s.t) * s.gtd0;
            if (f_new > armijo || (s.ls_iter > 1 && f_new >= s.f_prev)) {
                s.bt[0] = s.t_prev; s.bt[1] = s.t; s.bf[0] = s.f_prev; s.bf[1] = f_new;
                s.bgtd[0] = s.gtd_prev; s.bgtd[1] = gtd_new;
                VLOOP(i) { bg0[i] = g_prev[i]; bg1[i] = g_new[i]; }
                label = L_ZOOM_INIT;
                break;
            }
            if (fabsf(gtd_new) <= -c2 * s.gtd0) {
                s.bt[0] = s.t; s.bt[1] = s.t; s.bf[0] = f_new; s.bf[1] = f_new; s.bgtd[0] = gtd_new; s.bgtd[1] = gtd_new;
                VLOOP(i) bg0[i] = g_new[i];
                s.done = 1; s.low = 0; s.high = 1;
                label = L_LS_FINISH;
                break;
            }
            if (gtd_new >= 0.f) {
                s.bt[0] = s.t_prev; s.bt[1] = s.t; s.bf[0] = s.f_prev; s.bf[1] = f_new;
                s.bgtd[0] = s.gtd_prev; s.bgtd[1] = gtd_new;
                VLOOP(i) { bg0[i] = g_prev[i]; bg1[i] = g_new[i]; }
                label = L_ZOOM_INIT;
                break;
            }
            {   // interpolate (lbfgs_ls.py:82-95)
                const float min_step = s.t + 0.01f * (s.t - s.t_prev);
                const float max_step = s.t * 10.f;
                const float tmp = s.t;
                s.t = cubic_interpolate(s.t_prev, s.f_prev, s.gtd_prev, s.t, f_new, gtd_new, true, min_step, max_step);
                s.t_prev = tmp; s.f_prev = f_new; s.gtd_prev = gtd_new;
                VLOOP(i) g_prev[i] = g_new[i];
                label = L_REQ_LS;
            }
            break;
        }
        case L_ZOOM_INIT: {                                    // lbfgs_ls.py:106-108
            s.insuf = 0;
            if (s.bf[0] <= s.bf[1]) { s.low = 0; s.high = 1; } else { s.low = 1; s.high = 0; }
            s.phase = PH_LS_ZOOM;
            label = L_ZOOM_HEAD;
            break;
        }
        case L_ZOOM_HEAD: {                                    // lbfgs_ls.py:109-129
            if (s.done || s.ls_iter >= cfg.max_iter) { label = L_LS_FINISH; break; }
            float t = cubic_interpolate(s.bt[0], s.bf[0], s.bgtd[0], s.bt[1], s.bf[1], s.bgtd[1], false, 0.f, 0.f);
            const float bmax = (s.bt[1] > s.bt[0]) ? s.bt[1] : s.bt[0];
            const float bmin = (s.bt[1] < s.bt[0]) ? s.bt[1] : s.bt[0];
            const float eps = 0.1f * (bmax - bmin);
            const float da = bmax - t, db = t - bmin;
            if (((db < da) ? db : da) < eps) {
                if (s.insuf || t >= bmax || t <= bmin) {
                    t = (fabsf(t - bmax) < fabsf(t - bmin)) ? bmax - eps : bmin + eps;
                    s.insuf = 0;
                } else {
                    s.insuf = 1;
                }
            } else {
                s.insuf = 0;
            }
            s.t = t;
            label = L_REQ_LS;
            break;
        }
        case L_LS_ZOOM: {                                      // lbfgs_ls.py:131-161
            s.ls_evals++;
            gtd_new = vdot(g_new, d, lane);
            s.ls_iter++;
            const float armijo = s.loss + (c1 * s.t) * s.gtd0;
            float* bgl = s.low ? bg1 : bg0;
            float* bgh = s.high ? bg1 : bg0;
            if (f_new > armijo || f_new >= s.bf[s.low]) {
                s.bt[s.high] = s.t; s.bf[s.high] = f_new; s.bgtd[s.high] = gtd_new;
                VLOOP(i) bgh[i] = g_new[i];
                if (s.bf[0] <= s.bf[1]) { s.low = 0; s.high = 1; } else { s.low = 1; s.high = 0; }
            } else {
                if (fabsf(gtd_new) <= -c2 * s.gtd0) {
                    s.done = 1;
                } else if (gtd_new * (s.bt[s.high] - s.bt[s.low]) >= 0.f) {
                    s.bt[s.high] = s.bt[s.low]; s.bf[s.high] = s.bf[s.low]; s.bgtd[s.high] = s.bgtd[s.low];
                    VLOOP(i) bgh[i] = bgl[i];
                }
                s.bt[s.low] = s.t; s.bf[s.low] = f_new; s.bgtd[s.low] = gtd_new;
                VLOOP(i) bgl[i] = g_new[i];
            }
            __syncwarp();
            // the reference's step() calls _strong_Wolfe without tolerance_change (lbfgs_ls.py:393-397), so the bracket
            // width is always tested against its default 1e-9, whatever tolerance_change the optimiser was given
            if (fabsf(s.bt[1] - s.bt[0]) * s.d_norm < 1e-9f) { label = L_LS_FINISH; break; }
            label = L_ZOOM_HEAD;
            break;
        }
        case L_LS_FINISH: {                                    // lbfgs_ls.py:163-167, 399-434
            const float* bgl = s.low ? bg1 : bg0;
            // A line search that ends on a non-finite point (a trial step far enough out that the closure overflows, or a
            // NaN step length from the cubic interpolation of such values) would write NaN into the parameters, and the
            // monitor's NaN guard (fitting.py:101-107) would then stop the frame with NaN parameters.  Instead the
            // parameters, loss and gradient stay at the line search's start and the step ends: the next monitor check
            // sees no progress and the stage finishes with the last finite iterate.  Deliberate departure from
            // lbfgs_ls.py, which only differs where the reference itself would produce a non-finite result.
            bool finite = isfinite(s.bt[s.low]) && isfinite(s.bf[s.low]);
            VLOOP(i) if (!isfinite(bgl[i]) || !isfinite(fmaf(s.bt[s.low], d[i], x_init[i]))) finite = false;
            if (!__all_sync(0xffffffffu, finite)) {
                s.t = 0.f;
                s.current_evals += s.ls_evals;
                label = L_STEP_END;
                break;
            }
            s.t = s.bt[s.low];
            s.loss = s.bf[s.low];
            VLOOP(i) { g[i] = bgl[i]; x[i] = fmaf(s.t, d[i], x_init[i]); }
            __syncwarp();
            const bool opt_cond = vabsmax(g, lane) <= cfg.tol_grad;
            s.current_evals += s.ls_evals;
            float p = 0.f;
            VLOOP(i) p = fmaxf(p, fabsf(d[i] * s.t));
            const float step_max = warp_max(p);
            if (s.n_iter == cfg.max_iter || s.current_evals >= cfg.max_eval || opt_cond || step_max <= cfg.tol_change ||
                fabs((double)s.loss - (double)s.prev_loss) < (double)cfg.tol_change) {
                label = L_STEP_END;
                break;
            }
            label = L_ITER_BEGIN;
            break;
        }
        case L_STEP_END: {                                     // fitting.py:99-140
            const float ret = s.orig_loss;
            if (cfg.step_mode) {                               // step() returns the loss at entry (lbfgs_ls.py:445)
                s.final_loss = ret;
                s.phase = PH_DONE;
                label = L_EXIT;
                break;
            }
            if (isnan(ret) || isinf(ret)) { s.nan_flag = 1; label = L_FINISH; break; }
            if (s.outer_n > 0 && s.have_prev && cfg.ftol > 0.0) {
                const double pl = (double)s.mon_prev_loss, cl = (double)ret;
                const double den = fmax(fmax(fabs(pl), fabs(cl)), 1.0);
                if ((pl - cl) / den <= cfg.ftol) { label = L_FINISH; break; }
            }
            {   // all(abs(max(grad_tensor)) < gtol) on the grads left by the LAST closure call (fitting.py:115-117)
                const int seg_a[5] = {kOffBetas, kOffOrient, kOffPose, kOffTransl, kOffScale};
                const int seg_e[5] = {kOffOrient, kOffPose, kOffPose + pose_len, kOffScale, kParams};
                bool all_small = true;
                for (int sg = 0; sg < 5; ++sg) {
                    float m = -3.0e38f;
                    VLOOP(i) if (i >= seg_a[sg] && i < seg_e[sg]) m = fmaxf(m, g_new[i]);
                    m = warp_max(m);
                    if (!(fabs((double)m) < cfg.gtol)) all_small = false;
                }
                if (all_small) { label = L_FINISH; break; }
            }
            s.mon_prev_loss = ret;
            s.have_prev = 1;
            s.outer_n++;
            if (s.outer_n >= cfg.max_outer) { label = L_FINISH; break; }
            VLOOP(i) x_eval[i] = x[i];
            s.phase = PH_STEP_ENTRY;
            label = L_EXIT;
            break;
        }
        case L_REQ_LS: {                                       // lbfgs_ls.py:249-254: x + t*d, evaluated by the next round
            VLOOP(i) x_eval[i] = fmaf(s.t, d[i], x_init[i]);
            label = L_EXIT;
            break;
        }
        case L_FINISH: {
            s.final_loss = s.have_prev ? s.mon_prev_loss : __int_as_float(0x7fc00000);
            s.phase = PH_DONE;
            label = L_EXIT;
            break;
        }
        default: label = L_EXIT; break;
        }
    }
    __syncwarp();
}

}  // namespace mvs
