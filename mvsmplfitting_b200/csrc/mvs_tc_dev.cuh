// Device-side building blocks of the tensor-core vertex forward (mvs_tc.cu): mbarrier / TMA / wgmma wrappers, tile
// constants, and the one vertex routine every skinning variant calls (so that a frame gets the same bits whichever
// kernel evaluated it).
#pragma once
#include <cuda.h>
#include "mvs_internal.cuh"

namespace mvs {

constexpr int kTcBM = 128;            // frames per CTA: two consumer warpgroups of 64 rows (wgmma M = 64)
constexpr int kTcWgM = 64;            // frames per consumer warpgroup
constexpr int kTcBN = kTileC;         // 96 columns = 32 vertices (wgmma N)
constexpr int kTcBK = 32;             // floats per 128-byte swizzle row
constexpr int kTcKCh = kFeatPad / kTcBK;   // 7 K chunks
constexpr int kTcStages = 2;             // ring stages of (A lo chunk | B hi chunk | B lo chunk)
constexpr int kTcABytes = kTcBM * kTcBK * 4;   // 16 KB
constexpr int kTcBBytes = kTcBN * kTcBK * 4;   // 12 KB
constexpr int kTcThreads = 384;       // warpgroup 0: TMA producer; warpgroups 1, 2: wgmma + epilogue, 64 frames each
constexpr int kTcStageBytes = kTcABytes + 2 * kTcBBytes;     // 40 KB
constexpr int kTcEpiCols = 32;                                 // pose-offset columns per TMA store of the epilogue
constexpr int kTcEpiBytes = kTcEpiCols * kTcBM * 4;            // 16 KB: one 8 KB staging tile [column][64 frames] per warpgroup
constexpr size_t kTcSmem = 1024 /*align slack*/ + (size_t)kTcKCh * kTcABytes + (size_t)kTcStages * kTcStageBytes + kTcEpiBytes + 256;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// bounded spin: a protocol bug must not hang the GPU -- after ~2 s the kernel raises the error flag and carries on
__device__ __forceinline__ bool mbar_wait(uint64_t* bar, uint32_t parity, int* err_flag) {
    uint32_t done = 0;
    for (long long it = 0; it < (1ll << 26); ++it) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done) : "r"(smem_u32(bar)), "r"(parity) : "memory");
        if (done) return true;
        if ((it & 8191) == 8191 && err_flag && *reinterpret_cast<volatile int*>(err_flag) != 0) return false;
    }
    if (err_flag) atomicExch(err_flag, 1);
    return false;
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}
// shared -> global tile store (bulk async group of the issuing thread); the tensor map clips the box at the tensor's bounds
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, const void* src, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
                 ::"l"(map), "r"(smem_u32(src)), "r"(c0), "r"(c1) : "memory");
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
// wgmma shared-memory matrix descriptor: K-major, 128-byte swizzle, rows of 128 B packed 8 per 1024 B
// (start >> 4, LBO = 1 (unused for swizzled K-major), SBO = 1024 B, layout type 1 = SWIZZLE_128B)
__device__ __forceinline__ uint64_t wgmma_desc_k_sw128(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
    d |= (uint64_t)1 << 16;
    d |= (uint64_t)(1024 >> 4) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// D[64 x 96] (+)= A[64 x 8] . B[96 x 8]^T, tf32 inputs (both K-major in shared memory), fp32 accumulators in registers:
// with w = t / 32 and l = t % 32 for thread t of the warpgroup, d[4 i + 2 h + j] = D[16 w + l / 4 + 8 h][8 i + 2 (l % 4) + j]
__device__ __forceinline__ void wgmma_m64n96k8_tf32(float* d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %50, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n96k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
        "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}, "
        "%48, %49, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
          "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
          "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),
          "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),
          "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
        : "l"(adesc), "l"(bdesc), "r"(accumulate)
        : "memory");
}

// One vertex of one frame: v_posed = template + shapedirs.betas + pose offset, then linear blend skinning
// (lbs.py:179,203,207-220).  skin_kernel (lane = frame) and skin_small_kernel (lane = vertex) both call this with every
// operation spelled out, so the two produce the same bits: a frame's result must not depend on which of the two
// kernels its batch size selected.  A(j, a12) loads the 12 entries (row-major 3x4) of joint j's transform for this frame.
template <class AFn>
__device__ __forceinline__ void skin_vertex(const float* __restrict__ st /* [3][11]: shapedirs row | template */,
                                            const float* beta, const float* poff, const int* __restrict__ ell_j,
                                            const float* __restrict__ ell_w, int KW, size_t n, AFn A, float* vp, float* vv) {
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        float a = st[11 * c + kBetas];
#pragma unroll
        for (int l = 0; l < kBetas; ++l) a = fmaf(st[11 * c + l], beta[l], a);
        vp[c] = __fadd_rn(a, poff[c]);
    }
    float T[12];
#pragma unroll
    for (int c = 0; c < 12; ++c) T[c] = 0.f;
    // padding entries have weight 0 and a valid joint: fma(0, a, T) == T exactly, so no branch (and no dependent
    // load behind it) is needed
#pragma unroll 4
    for (int e = 0; e < KW; ++e) {
        const float w = ell_w[n * KW + e];
        float a12[12];
        A(ell_j[n * KW + e], a12);
#pragma unroll
        for (int c = 0; c < 12; ++c) T[c] = fmaf(w, a12[c], T[c]);
    }
#pragma unroll
    for (int r = 0; r < 3; ++r)
        vv[r] = __fadd_rn(fmaf(T[4 * r + 2], vp[2], fmaf(T[4 * r + 1], vp[1], __fmul_rn(T[4 * r], vp[0]))), T[4 * r + 3]);
}

// ------------------------------------------------------------------------------------------------ skinning
// v_posed = v_template + shapedirs.betas (fp32) + pose offsets (tensor cores), then linear blend skinning
// (lbs.py:179,203,207-220).  CTA = 32 frames x 64 vertices; lane = frame.  The 32 frames' skinning transforms
// (288 floats each) sit in shared memory frame-fastest, so the 48 reads per (frame, vertex) are conflict-free LDS
// instead of global loads; outputs are transposed through shared memory into coalesced row stores.  Also emits the
// per-chunk bounding-box partial of every frame for the SDF kernels.
constexpr int kSkinV = 64;
constexpr int kSkinThreads = 256;
constexpr int kSkinOutLd = 3 * kSkinV + 1;     // 193
constexpr int kSkinEllMax = 8;                 // skinning weights per vertex staged in shared memory (SMPL: 4)
constexpr size_t kSkinSmem =
    (size_t)(kSkinFloats * 32 + kBetas * 32 + 2 * 32 * kSkinOutLd + 8 * 32 * 6 * 2 + kSkinV * 33 + 2 * kSkinV * kSkinEllMax) * sizeof(float);
constexpr size_t kSkinSmemNoVp = kSkinSmem - (size_t)32 * kSkinOutLd * sizeof(float);     // v_posed not stored

// v_posed of one vertex coordinate exactly as skin_vertex computes it (consumers that need a handful of v_posed values
// recompute them instead of reading a [B][N][3] array the skinning kernels would have to write every round)
__device__ __forceinline__ float vposed_of(const float* __restrict__ st11 /* shapedirs row (10) | template */, const float* beta,
                                           const float poff) {
    float a = st11[kBetas];
#pragma unroll
    for (int l = 0; l < kBetas; ++l) a = fmaf(st11[l], beta[l], a);
    return __fadd_rn(a, poff);
}

// Arguments of the skinning bodies.  poffT / Phi / At / verts / bboxp are rewritten every round by other CTAs of the
// persistent dense-round kernel, so they are plain pointers (no __restrict__ / read-only path); the model constants may
// use the read-only path.  vposed == nullptr: v_posed is not stored (the few consumers recompute it, vposed_of).
struct SkinArgs {
    const float* poffT; const float* ST; const float* Phi; const float* At; int ldA;
    const int* ell_j; const float* ell_w; int KW; int N;
    float* vposed; float* verts; float* bboxp;
};

// skin_kernel's CTA (vbx, vby) of a virtual grid (nchunks, frame groups); `sk` = kSkinSmem bytes of shared memory.
// All kSkinThreads threads must call.
__device__ __forceinline__ void skin_body(float* sk, const SkinArgs& ar, const int na, const int cta_slots, const int vbx, const int vby) {
    const float* poffT = ar.poffT; const float* __restrict__ ST = ar.ST; const float* Phi = ar.Phi; const float* At = ar.At;
    const int ldA = ar.ldA, KW = ar.KW, N = ar.N;
    const int* __restrict__ ell_j = ar.ell_j; const float* __restrict__ ell_w = ar.ell_w;
    float* vposed = ar.vposed; float* verts = ar.verts; float* bboxp = ar.bboxp;
    float* As = sk;                                   // [24 joints][32 lanes][12]
    float* Bs = As + kSkinFloats * 32;                // [10][32]
    float* Ovp = Bs + kBetas * 32;                    // [32][193] (only when v_posed is stored)
    float* Ov = vposed ? Ovp + 32 * kSkinOutLd : Ovp; // [32][193]
    float* Bb = Ov + 32 * kSkinOutLd;                 // [8 warps][32 lanes][6] values, then [..][6] indices
    float* Sts = Bb + 8 * 32 * 6 * 2;                 // [64][33] shapedirs rows | template of this CTA's vertices
    float* Ews = Sts + kSkinV * 33;                   // [64][KW] skinning weights of the chunk
    int* Ejs = reinterpret_cast<int*>(Ews + kSkinV * kSkinEllMax);   // [64][KW] their joints
    const bool ell_smem = KW <= kSkinEllMax;
    const int f0 = vby * 32;
    if (f0 >= na) return;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int slotc = min(f0 + lane, na - 1);
    // chunks per CTA from the number of ACTIVE frame groups: one chunk each while the active CTAs fit in one wave
    // (latency at the tail of a stage), several once they do not (the 36 KB of transforms are then loaded once)
    const int nchunks = (N + kSkinV - 1) / kSkinV;
    const int per_cta = (nchunks * ((na + 31) / 32) + cta_slots - 1) / cta_slots;
    const int nx = (nchunks + per_cta - 1) / per_cta;
    if (vbx >= nx) return;
    // the 32 frames' transforms and shape coefficients are loaded once and reused for every vertex chunk of this CTA
    // layout [joint][lane][12]: a lane's 3x4 transform is three conflict-free LDS.128 (lane stride 48 B)
    for (int e = tid; e < kSkinFloats * 32; e += kSkinThreads) {
        const int jc = e >> 5, ln = e & 31;
        As[((jc / 12) * 32 + ln) * 12 + jc % 12] = At[(size_t)jc * ldA + min(f0 + ln, na - 1)];
    }
    for (int e = tid; e < kBetas * 32; e += kSkinThreads)
        Bs[e] = Phi[(size_t)min(f0 + (e & 31), na - 1) * kFeatPad + kPoseBasis + (e >> 5)];
    constexpr int kVw = kSkinV / 8;                                       // vertices per warp and chunk
    float beta[kBetas];
    bool have_beta = false;
    for (int ch = vbx; ch < nchunks; ch += nx) {
        const int v0 = ch * kSkinV;
        // pose offsets of this warp's vertices: 24 independent coalesced loads in flight before anything waits
        float pf[kVw][3];
#pragma unroll
        for (int i = 0; i < kVw; ++i) {
            const int n = v0 + warp * kVw + i;
#pragma unroll
            for (int c = 0; c < 3; ++c) pf[i][c] = n < N ? poffT[(size_t)(3 * n + c) * ldA + slotc] : 0.f;
        }
        __syncthreads();                                                  // previous chunk's staging buffers are free
        for (int e = tid; e < kSkinV * 33; e += kSkinThreads) Sts[e] = (v0 * 33 + e < N * 33) ? ST[(size_t)v0 * 33 + e] : 0.f;
        if (ell_smem)
            for (int e = tid; e < kSkinV * KW; e += kSkinThreads) {
                const bool in = (size_t)v0 * KW + e < (size_t)N * KW;
                Ews[e] = in ? ell_w[(size_t)v0 * KW + e] : 0.f;
                Ejs[e] = in ? ell_j[(size_t)v0 * KW + e] : 0;
            }
        __syncthreads();
        if (!have_beta) {
#pragma unroll
            for (int l = 0; l < kBetas; ++l) beta[l] = Bs[l * 32 + lane];
            have_beta = true;
        }
        float blo[3] = {3e38f, 3e38f, 3e38f}, bhi[3] = {-3e38f, -3e38f, -3e38f};
        int bilo[3] = {0, 0, 0}, bihi[3] = {0, 0, 0};
#pragma unroll
        for (int i = 0; i < kVw; ++i) {
            const int li = warp * kVw + i;
            const int n = v0 + li;
            if (n < N) {
                float vp[3], vvv[3];
                skin_vertex(Sts + li * 33, beta, pf[i], ell_smem ? Ejs : ell_j, ell_smem ? Ews : ell_w, KW,
                            ell_smem ? (size_t)li : (size_t)n,
                            [&](int j, float* a12) {
                                const float4* q = reinterpret_cast<const float4*>(As + (j * 32 + lane) * 12);
                                const float4 q0 = q[0], q1 = q[1], q2 = q[2];
                                a12[0] = q0.x; a12[1] = q0.y; a12[2] = q0.z; a12[3] = q0.w; a12[4] = q1.x; a12[5] = q1.y;
                                a12[6] = q1.z; a12[7] = q1.w; a12[8] = q2.x; a12[9] = q2.y; a12[10] = q2.z; a12[11] = q2.w;
                            }, vp, vvv);
#pragma unroll
                for (int r = 0; r < 3; ++r) {
                    const float vv = vvv[r];
                    if (vposed) Ovp[lane * kSkinOutLd + 3 * li + r] = vp[r];
                    Ov[lane * kSkinOutLd + 3 * li + r] = vv;
                    if (vv < blo[r]) { blo[r] = vv; bilo[r] = n; }       // strict: ties keep the lowest vertex index
                    if (vv > bhi[r]) { bhi[r] = vv; bihi[r] = n; }
                }
            }
        }
        int* Bi = reinterpret_cast<int*>(Bb + 8 * 32 * 6);
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            Bb[(warp * 32 + lane) * 6 + r] = blo[r]; Bb[(warp * 32 + lane) * 6 + 3 + r] = bhi[r];
            Bi[(warp * 32 + lane) * 6 + r] = bilo[r]; Bi[(warp * 32 + lane) * 6 + 3 + r] = bihi[r];
        }
        __syncthreads();
        const int ncol = 3 * min(kSkinV, N - v0);                         // contiguous floats of this chunk per frame
        for (int fl = warp; fl < 32; fl += 8) {                           // a warp stores one frame's row segment at a time
            const int slot = f0 + fl;
            if (slot >= na) break;
            const size_t off = ((size_t)slot * N + v0) * 3;
            for (int col = lane; col < ncol; col += 32) {
                if (vposed) vposed[off + col] = Ovp[fl * kSkinOutLd + col];
                verts[off + col] = Ov[fl * kSkinOutLd + col];
            }
        }
        if (bboxp && warp == 0 && f0 + lane < na) {       // fold the 8 warps' vertex groups (ascending vertex index)
            float lo[3], hi[3];
            int ilo[3], ihi[3];
#pragma unroll
            for (int r = 0; r < 3; ++r) { lo[r] = Bb[lane * 6 + r]; hi[r] = Bb[lane * 6 + 3 + r]; ilo[r] = Bi[lane * 6 + r]; ihi[r] = Bi[lane * 6 + 3 + r]; }
            for (int w2 = 1; w2 < 8; ++w2)
#pragma unroll
                for (int r = 0; r < 3; ++r) {
                    const float l2 = Bb[(w2 * 32 + lane) * 6 + r], h2 = Bb[(w2 * 32 + lane) * 6 + 3 + r];
                    if (l2 < lo[r]) { lo[r] = l2; ilo[r] = Bi[(w2 * 32 + lane) * 6 + r]; }
                    if (h2 > hi[r]) { hi[r] = h2; ihi[r] = Bi[(w2 * 32 + lane) * 6 + 3 + r]; }
                }
            float* bp = bboxp + ((size_t)(f0 + lane) * nchunks + ch) * 12;
#pragma unroll
            for (int r = 0; r < 3; ++r) { bp[r] = lo[r]; bp[3 + r] = hi[r]; bp[6 + r] = __int_as_float(ilo[r]); bp[9 + r] = __int_as_float(ihi[r]); }
        }
    }
    __syncthreads();
}

// The same for a handful of frames (the straggler tail of a fit): with lane = frame almost every lane of skin_kernel
// idles and its fixed costs (36 KB of transforms per CTA, staging, three barriers per chunk) are pure latency.  Here
// lane = vertex, a CTA owns one 64-vertex chunk (= one box partial) and loops over the <= kSkinSmallMax frames.
constexpr int kSkinSmallMax = 8;
constexpr int kSkinSmallThreads = 64;
static_assert(kSkinSmallThreads == kSkinV, "one thread per vertex of a box chunk");

struct SkinSmallSmem {
    float As[kSkinSmallMax][kSkinFloats];
    float Bs[kSkinSmallMax][kBetas];
    float s_b[kSkinSmallMax][6];
    int s_i[kSkinSmallMax][6];
};

// skin_small_kernel's CTA for one 64-vertex chunk, executed by the kSkinSmallThreads threads t = 0..63 of a thread group
// that synchronises on named barrier `bar` (0 with a 64-thread CTA = __syncthreads).
__device__ __forceinline__ void skin_small_body(SkinSmallSmem& sm, const SkinArgs& ar, int na_in, const int chunk, const int nchunks,
                                                const int t, const int bar) {
    const float* poffT = ar.poffT; const float* __restrict__ ST = ar.ST; const float* Phi = ar.Phi; const float* At = ar.At;
    const int ldA = ar.ldA, KW = ar.KW, N = ar.N;
    const int* __restrict__ ell_j = ar.ell_j; const float* __restrict__ ell_w = ar.ell_w;
    float* vposed = ar.vposed; float* verts = ar.verts; float* bboxp = ar.bboxp;
    auto& As = sm.As; auto& Bs = sm.Bs; auto& s_b = sm.s_b; auto& s_i = sm.s_i;
    const int na = min(na_in, kSkinSmallMax);
    if (na <= 0) return;
    const int lane = t & 31, warp = t >> 5;
    const int n = chunk * kSkinSmallThreads + t;
    for (int e = t; e < na * kSkinFloats; e += kSkinSmallThreads) As[e / kSkinFloats][e % kSkinFloats] = At[(size_t)(e % kSkinFloats) * ldA + e / kSkinFloats];
    for (int e = t; e < na * kBetas; e += kSkinSmallThreads) Bs[e / kBetas][e % kBetas] = Phi[(size_t)(e / kBetas) * kFeatPad + kPoseBasis + e % kBetas];
    float st[33];
    if (n < N) {
#pragma unroll
        for (int q = 0; q < 33; ++q) st[q] = ST[(size_t)n * 33 + q];
    }
    asm volatile("bar.sync %0, %1;" ::"r"(bar), "r"(kSkinSmallThreads) : "memory");
    for (int f = 0; f < na; ++f) {
        float lo[3] = {3e38f, 3e38f, 3e38f}, hi[3] = {-3e38f, -3e38f, -3e38f};
        int ilo[3] = {0x7fffffff, 0x7fffffff, 0x7fffffff}, ihi[3] = {0x7fffffff, 0x7fffffff, 0x7fffffff};
        if (n < N) {
            float poff[3], vp[3], vv[3];
#pragma unroll
            for (int c = 0; c < 3; ++c) poff[c] = poffT[(size_t)(3 * n + c) * ldA + f];
            skin_vertex(st, Bs[f], poff, ell_j, ell_w, KW, (size_t)n,
                        [&](int j, float* a12) {
#pragma unroll
                            for (int c = 0; c < 12; ++c) a12[c] = As[f][j * 12 + c];
                        }, vp, vv);
            const size_t off = ((size_t)f * N + n) * 3;
#pragma unroll
            for (int r = 0; r < 3; ++r) {
                if (vposed) vposed[off + r] = vp[r];
                verts[off + r] = vv[r];
                lo[r] = vv[r]; hi[r] = vv[r]; ilo[r] = n; ihi[r] = n;
            }
        }
        if (bboxp) {               // box of the chunk: extreme value, ties -> lowest vertex index (as skin_kernel)
#pragma unroll
            for (int r = 0; r < 3; ++r) { warp_argmin(lo[r], ilo[r]); warp_argmax(hi[r], ihi[r]); }
            if (warp == 1 && lane == 0) {
#pragma unroll
                for (int r = 0; r < 3; ++r) { s_b[f][r] = lo[r]; s_b[f][3 + r] = hi[r]; s_i[f][r] = ilo[r]; s_i[f][3 + r] = ihi[r]; }
            }
            asm volatile("bar.sync %0, %1;" ::"r"(bar), "r"(kSkinSmallThreads) : "memory");
            if (warp == 0 && lane == 0) {
                float* bp = bboxp + ((size_t)f * nchunks + chunk) * 12;
#pragma unroll
                for (int r = 0; r < 3; ++r) {
                    const float l2 = s_b[f][r], h2 = s_b[f][3 + r];
                    const int il2 = s_i[f][r], ih2 = s_i[f][3 + r];
                    if (l2 < lo[r] || (l2 == lo[r] && il2 < ilo[r])) { lo[r] = l2; ilo[r] = il2; }
                    if (h2 > hi[r] || (h2 == hi[r] && ih2 < ihi[r])) { hi[r] = h2; ihi[r] = ih2; }
                    bp[r] = lo[r]; bp[3 + r] = hi[r]; bp[6 + r] = __int_as_float(ilo[r]); bp[9 + r] = __int_as_float(ihi[r]);
                }
            }
        }
    }
}

}  // namespace mvs
