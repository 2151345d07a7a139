// Device-side building blocks of the tensor-core kernels (mvs_tc.cu): mbarrier / TMA / wgmma wrappers, tile constants, the
// TMA / wgmma ring both contractions share, and the one vertex routine every skinning variant calls (so that a frame gets
// the same bits whichever kernel evaluated it).
#pragma once
#include <cuda.h>
#include "mvs_internal.cuh"

namespace mvs {

// Tiles of posedirs_gemm_tc_kernel.  The contraction runs transposed, poffT = Qk[:, :207] . Phi^T: the 3N posedirs rows
// are the wgmma M side (64 rows per consumer warpgroup, 128 per CTA tile) and the active frames the N side, so the
// accumulator fragment is already [coordinate][frame], the layout of poffT.
constexpr int kTcRows = 128;          // posedirs rows per CTA tile: two consumer warpgroups of 64 rows (wgmma M = 64)
constexpr int kTcWgRows = 64;         // posedirs rows per consumer warpgroup
constexpr int kTcCols = 128;          // frames per column tile (largest wgmma N instance used); larger batches run several
constexpr int kTcBK = 32;             // floats per 128-byte swizzle row
constexpr int kTcKCh = kFeatPad / kTcBK;   // 7 K chunks
constexpr int kTcPBytes = kTcRows * kTcBK * 4;     // 16 KB fp32 posedirs per stage (split into TF32 hi | lo on chip)
constexpr int kTcThreads = 288;       // warpgroups 0, 1: convert + wgmma + store, 64 rows each; warp 8: TMA producer
// frame columns of one launch (wgmma N): the active-frame bound rounded up to 8, 16, 32, 64 or 128
__host__ __device__ constexpr int tc_cols_for(int nb) { return nb <= 8 ? 8 : nb <= 16 ? 16 : nb <= 32 ? 32 : nb <= 64 ? 64 : 128; }
__host__ __device__ constexpr int tc_fbytes(int nf) { return nf * kTcBK * 4; }            // one feature chunk (hi or lo): nf rows of 128 B
// ring stage: posedirs chunk | feature hi chunk | feature lo chunk
__host__ __device__ constexpr int tc_stage_bytes(int nf) { return kTcPBytes + 2 * tc_fbytes(nf); }

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// arrive if `pred`, as a predicated instruction rather than a branch (no divergent path between in-flight wgmma groups)
__device__ __forceinline__ void mbar_arrive_if(uint64_t* bar, bool pred) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %1, 0;\n\t@p mbarrier.arrive.shared::cta.b64 _, [%0];\n\t}"
                 ::"r"(smem_u32(bar)), "r"((uint32_t)pred) : "memory");
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
__device__ __forceinline__ void wgmma_wait1() { asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory"); }
// D[64 x N] (+)= A[64 x 8] . B[N x 8]^T, tf32: A from registers, B K-major in shared memory, fp32 accumulators in registers.
// For thread t of the warpgroup with w = t / 32, l = t % 32, g = l / 4, q = l % 4:
//   a[0] = A[16 w + g][q], a[1] = A[16 w + g + 8][q], a[2] = A[16 w + g][q + 4], a[3] = A[16 w + g + 8][q + 4]
//   d[4 i + 2 h + j] = D[16 w + g + 8 h][8 i + 2 q + j]
template <int N> struct WgmmaTf32Rs;
template <> struct WgmmaTf32Rs<8> {
    static __device__ __forceinline__ void mma(float* d, const uint32_t* a, uint64_t bdesc, uint32_t accumulate) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "setp.ne.b32 p, %9, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n8k8.f32.tf32.tf32 "
            "{%0, %1, %2, %3}, "
            "{%4, %5, %6, %7}, %8, p, 1, 1;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
            : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate)
            : "memory");
    }
};
template <> struct WgmmaTf32Rs<16> {
    static __device__ __forceinline__ void mma(float* d, const uint32_t* a, uint64_t bdesc, uint32_t accumulate) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "setp.ne.b32 p, %13, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 "
            "{%0, %1, %2, %3, %4, %5, %6, %7}, "
            "{%8, %9, %10, %11}, %12, p, 1, 1;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
            : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate)
            : "memory");
    }
};
template <> struct WgmmaTf32Rs<32> {
    static __device__ __forceinline__ void mma(float* d, const uint32_t* a, uint64_t bdesc, uint32_t accumulate) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "setp.ne.b32 p, %21, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
            "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
            "{%16, %17, %18, %19}, %20, p, 1, 1;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
              "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
            : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate)
            : "memory");
    }
};
template <> struct WgmmaTf32Rs<64> {
    static __device__ __forceinline__ void mma(float* d, const uint32_t* a, uint64_t bdesc, uint32_t accumulate) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "setp.ne.b32 p, %37, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
            "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
            "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
            "{%32, %33, %34, %35}, %36, p, 1, 1;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
              "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
              "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
              "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
            : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate)
            : "memory");
    }
};
template <> struct WgmmaTf32Rs<128> {
    static __device__ __forceinline__ void mma(float* d, const uint32_t* a, uint64_t bdesc, uint32_t accumulate) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "setp.ne.b32 p, %69, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
            "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
            "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
            "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
            "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
            "{%64, %65, %66, %67}, %68, p, 1, 1;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
              "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
              "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
              "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
              "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
              "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
              "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
              "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
            : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate)
            : "memory");
    }
};

// ------------------------------------------------------------------------------------------------ the TMA / wgmma ring
// Both tensor-core kernels stream their operands through kRingStages stages of kStageBytes, 1024-byte aligned (the period
// of the 128-byte swizzle), with a `full` and an `empty` mbarrier per stage.  One producer thread waits until a stage is
// empty, arms `full` with the stage's byte count and issues its TMA boxes (ring_produce).  Each consumer warpgroup waits
// until the stage is full (Ring::wait_full), runs its k8 steps on it (A split into TF32 hi + lo, hi.Bhi, hi.Blo, lo.Bhi as
// one wgmma group, one group kept in flight by wait_group 1) and hands it back with one predicated arrival on `empty` once
// every group that read it has retired: after the next stage's first group, or after wait_group 0 at the end.
constexpr int kRingStages = 4;
__host__ __device__ constexpr size_t ring_smem(int stage_bytes) { return 1024 /*align slack*/ + (size_t)kRingStages * stage_bytes + 256 /*barriers*/; }

struct RingPos {                      // a thread's stage and the parity of its pass; next() moves on, returns the stage left
    int stage = 0;
    uint32_t phase = 0;
    __device__ __forceinline__ int next() { const int s = stage; if (++stage == kRingStages) { stage = 0; phase ^= 1; } return s; }
};

template <uint32_t kStageBytes>
struct Ring {
    unsigned char* base;              // stage s at base + s * kStageBytes
    uint64_t* full;                   // [kRingStages] completed by the producer's expect_tx and the TMA bytes
    uint64_t* empty;                  // [kRingStages] one arrival per consumer warpgroup
    __device__ __forceinline__ unsigned char* stage(int s) const { return base + (size_t)s * kStageBytes; }
    // consumer: wait for stage p to be full.  A timeout raises the error flag (the host reports it) and the warpgroup carries
    // on: leaving the loop would be a divergent exit with a wgmma group in flight, which makes ptxas serialise every group
    __device__ __forceinline__ void wait_full(const RingPos& p, int* err_flag) const { mbar_wait(&full[p.stage], p.phase, err_flag); }
};

// By the whole CTA: the ring in the dynamic shared memory (ring_smem bytes), its barriers set for `consumers` warpgroups.
template <uint32_t kStageBytes>
__device__ __forceinline__ Ring<kStageBytes> ring_setup(unsigned char* smem_raw, uint32_t consumers) {
    Ring<kStageBytes> r;
    r.base = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    r.full = reinterpret_cast<uint64_t*>(r.stage(kRingStages));
    r.empty = r.full + kRingStages;
    if (threadIdx.x == 0) {
        for (int s = 0; s < kRingStages; ++s) { mbar_init(&r.full[s], 1); mbar_init(&r.empty[s], consumers); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    return r;
}

// The producer (one thread): ring steps (item, chunk), item in [item_begin, item_end), chunk in [0, kChunks).  issue(item,
// chunk, dst, bar) issues the step's TMA boxes into the stage at dst, completing on bar.  Returns once a wait timed out.
template <int kChunks, uint32_t kStageBytes, class Issue>
__device__ __forceinline__ void ring_produce(const Ring<kStageBytes>& r, int item_begin, int item_end, int* err_flag, Issue issue) {
    RingPos p;
    for (int item = item_begin; item < item_end; ++item)
        for (int chunk = 0; chunk < kChunks; ++chunk) {
            if (!mbar_wait(&r.empty[p.stage], p.phase ^ 1, err_flag)) return;
            mbar_expect_tx(&r.full[p.stage], kStageBytes);
            issue(item, chunk, r.stage(p.stage), &r.full[p.stage]);
            p.next();
        }
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

// Arguments of the skinning kernels (mvs_tc.cu).  verts and bboxp are read back within skin_small_kernel's launch by the CTA
// that computes a frame's SDF set-up (sdf_frame_setup), so they are plain pointers.  sdf: read by skin_small_kernel only, set
// at <= kSkinSetupMax frames (otherwise sdf_setup_kernel computes the set-ups).  vposed == nullptr: v_posed is not stored
// (the few consumers recompute it, vposed_of).
struct SkinArgs {
    const float* poffT; const float* ST; const float* Phi; const float* At; int ldA;
    const int* ell_j; const float* ell_w; int KW; int N;
    float* vposed; float* verts; float* bboxp;
    SdfSetupArgs sdf;
};

// ------------------------------------------------------------------------------------------------ per-frame SDF set-up
// One warp computes frame `slot`'s SdfFrameSetup from the frame's nbox chunk boxes and skinned vertices, with the
// expressions sdf_fused used to evaluate in every CTA: the box (ties -> lowest vertex index), triangle 0 in box coordinates
// (fitting.py:362-363), the cone of planes it spans from the corner (-1,-1,-1), the plane of the triangle, the vertex-level
// pads and the chunk-cull verdicts.  Called by sdf_setup_kernel (mvs_tc.cu: one warp per slot, after the skinning kernel)
// and at the end of skin_small_kernel at <= 4 frames (sdf_setup_frames).  The chunk boxes and vertices were written by other
// CTAs, in skin_small_kernel of the same launch, so they are read through L2 (__ldcg).  Resets the frame's arrival counter
// for the next round (sdf_setup_kernel finds it at 0 and leaves it there).
static __device__ __noinline__ void sdf_frame_setup(const SdfSetupArgs sa, const float* bboxp, const float* verts, const int N,
                                             const int nbox, const int slot, const int lane) {
    const float tr[3] = {sa.slot_tr[4 * slot], sa.slot_tr[4 * slot + 1], sa.slot_tr[4 * slot + 2]};
    const float* vf = verts + (size_t)slot * N * 3;
    float traw[9];
    {
        const int fid[3] = {sa.f0, sa.f1, sa.f2};
#pragma unroll
        for (int q = 0; q < 9; ++q) traw[q] = __ldcg(vf + 3 * fid[q / 3] + q % 3);
    }
    // ---- bounding box: each lane folds its chunks in ascending order, the warp folds the lanes.  Chunks are loaded
    //      kSetupCh per lane at a time, all loads in flight; the first group's boxes stay in registers for the verdicts.
    constexpr int kSetupCh = 4;
    float lo[3] = {3e38f, 3e38f, 3e38f}, hi[3] = {-3e38f, -3e38f, -3e38f};
    int ilo[3] = {0x7fffffff, 0x7fffffff, 0x7fffffff}, ihi[3] = {0x7fffffff, 0x7fffffff, 0x7fffffff};
    float cb[kSetupCh][6];                             // pre-transl lo | hi of chunks lane + 32 i
#pragma unroll 1
    for (int g0 = 0; g0 < nbox; g0 += 32 * kSetupCh) {
        float bv[kSetupCh][12];
#pragma unroll
        for (int i = 0; i < kSetupCh; ++i) {
            const int tl = g0 + 32 * i + lane;
            const float* bp = bboxp + ((size_t)slot * nbox + min(tl, nbox - 1)) * 12;
#pragma unroll
            for (int e = 0; e < 12; ++e) bv[i][e] = __ldcg(bp + e);
        }
#pragma unroll
        for (int i = 0; i < kSetupCh; ++i) {
            if (g0 + 32 * i + lane >= nbox) break;
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const float l2 = bv[i][c], h2 = bv[i][3 + c];
                const int il2 = __float_as_int(bv[i][6 + c]), ih2 = __float_as_int(bv[i][9 + c]);
                if (l2 < lo[c] || (l2 == lo[c] && il2 < ilo[c])) { lo[c] = l2; ilo[c] = il2; }
                if (h2 > hi[c] || (h2 == hi[c] && ih2 < ihi[c])) { hi[c] = h2; ihi[c] = ih2; }
            }
        }
        if (g0 == 0) {
#pragma unroll
            for (int i = 0; i < kSetupCh; ++i)
#pragma unroll
                for (int e = 0; e < 6; ++e) cb[i][e] = bv[i][e];
        }
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) { warp_argmin(lo[c], ilo[c]); warp_argmax(hi[c], ihi[c]); }
    FrameBox fb;
    {
        float ext = -1.f;
        fb.cmax = 0;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            // the partials are on pre-transl vertices; fl(v + tr) is monotone in v, so min/max and their
            // arg-indices commute with the translation (body_models_scale.py:403)
            const float lc = lo[c] + tr[c], hc = hi[c] + tr[c];
            fb.centre[c] = (lc + hc) / 2.f;
            fb.ilo[c] = ilo[c]; fb.ihi[c] = ihi[c];
            const float e = hc - lc;
            if (e > ext) { ext = e; fb.cmax = c; }
        }
        fb.scale = 0.6f * ext;
        fb.pad = 0.f;
    }
    // triangle 0 in box coordinates and the cone it spans from the corner (-1,-1,-1)
    float tri[9], cn[3][3], cm[3];
#pragma unroll
    for (int q = 0; q < 9; ++q) tri[q] = ((traw[q] + tr[q % 3]) - fb.centre[q % 3]) / fb.scale;
#pragma unroll
    for (int q = 0; q < 3; ++q) {
        const float* a = &tri[3 * q];
        const float* bb = &tri[3 * ((q + 1) % 3)];
        const float ea[3] = {a[0] + 1.f, a[1] + 1.f, a[2] + 1.f}, eb[3] = {bb[0] + 1.f, bb[1] + 1.f, bb[2] + 1.f};
        cn[q][0] = ea[1] * eb[2] - ea[2] * eb[1]; cn[q][1] = ea[2] * eb[0] - ea[0] * eb[2]; cn[q][2] = ea[0] * eb[1] - ea[1] * eb[0];
        cm[q] = 3.5e-4f * sqrtf(cn[q][0] * cn[q][0] + cn[q][1] * cn[q][1] + cn[q][2] * cn[q][2]);
    }
    // plane of triangle 0 in the same shifted coordinates (w = centre + 1, the corner is the origin): the ray from a
    // voxel centre to the corner can only cross the triangle if the two lie on opposite sides of this plane, i.e.
    // <pn, w> - pd has the sign of pd.  Voxels between the corner and the triangle pass the cone test but fail this one.
    float pn[3], pd, pm;
    {
        const float e1[3] = {tri[3] - tri[0], tri[4] - tri[1], tri[5] - tri[2]}, e2[3] = {tri[6] - tri[0], tri[7] - tri[1], tri[8] - tri[2]};
        pn[0] = e1[1] * e2[2] - e1[2] * e2[1]; pn[1] = e1[2] * e2[0] - e1[0] * e2[2]; pn[2] = e1[0] * e2[1] - e1[1] * e2[0];
        pd = pn[0] * (tri[0] + 1.f) + pn[1] * (tri[1] + 1.f) + pn[2] * (tri[2] + 1.f);
        pm = 2e-3f * sqrtf(pn[0] * pn[0] + pn[1] * pn[1] + pn[2] * pn[2]);      // conservative: |w| <= 2 sqrt 3, fp32 rounding
    }
    // vertex-level early-out: the 8 voxel centres a vertex at `loc` can touch lie within +-vhalf of (loc + 1) G/(G-1) on
    // every axis, so each plane function varies by at most vhalf * |n|_1 over them
    const int G = sa.G;
    const float vhalf = 2.02f / (float)(G - 1) + 1e-5f;
    float vpad[3];
#pragma unroll
    for (int q = 0; q < 3; ++q) vpad[q] = vhalf * (fabsf(cn[q][0]) + fabsf(cn[q][1]) + fabsf(cn[q][2]));
    const float vpadp = vhalf * (fabsf(pn[0]) + fabsf(pn[1]) + fabsf(pn[2]));
    SdfFrameSetup* rec = sa.rec + slot;
    // Chunk-level cull: the voxel centres a vertex at `loc` can touch lie within (loc + 1) G/(G-1) +- 2/(G-1) (+1
    // shifted); if the whole box of a 64-vertex chunk is on the negative side of one cone plane and on the positive side
    // of another, no vertex of the chunk can see a voxel with phi != 0: value and gradient are exactly zero.
    const bool cull = sa.cull && nbox <= 32 * kSdfSkipWords;
    unsigned live_lo = 0u, live_hi = 0u;               // bit b of the pair: block b has a chunk that is not culled
#pragma unroll 1
    for (int k = 0; k < kSdfSkipWords; ++k) {
        const int chunk = 32 * k + lane;
        bool skip = false;
        if (cull && chunk < nbox) {
            float bx[6];
            if (k < kSetupCh) {
#pragma unroll
                for (int e = 0; e < 6; ++e) bx[e] = cb[0][e];
#pragma unroll
                for (int i = 1; i < kSetupCh; ++i)
                    if (k == i)
#pragma unroll
                        for (int e = 0; e < 6; ++e) bx[e] = cb[i][e];
            } else {
                const float* bp = bboxp + ((size_t)slot * nbox + chunk) * 12;
#pragma unroll
                for (int e = 0; e < 6; ++e) bx[e] = __ldcg(bp + e);
            }
            const float gs = (float)G / (float)(G - 1), pad = 2.02f / (float)(G - 1) + 1e-5f;
            float wlo[3], whi[3];
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const float l_lo = ((bx[c] + tr[c]) - fb.centre[c]) / fb.scale;
                const float l_hi = ((bx[3 + c] + tr[c]) - fb.centre[c]) / fb.scale;
                wlo[c] = (l_lo + 1.f) * gs - pad; whi[c] = (l_hi + 1.f) * gs + pad;
            }
            bool all_neg = false, all_pos = false;
#pragma unroll
            for (int q = 0; q < 3; ++q) {
                float smin = 0.f, smax = 0.f;
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    const float a = cn[q][c] * wlo[c], b2 = cn[q][c] * whi[c];
                    smin += fminf(a, b2); smax += fmaxf(a, b2);
                }
                all_neg = all_neg || (smax < -cm[q]);
                all_pos = all_pos || (smin > cm[q]);
            }
            skip = all_neg && all_pos;
        }
        const unsigned bits = __ballot_sync(0xffffffffu, skip);
        if (lane == 0) rec->skip[k] = bits;
        // the word's 32 chunks are blocks 8k..8k+7: a block is live when one of its chunks below nbox is not culled
        unsigned live = __ballot_sync(0xffffffffu, chunk < nbox && !skip);
        live |= live >> 1;
        live |= live >> 2;
        unsigned b8 = 0u;
#pragma unroll
        for (int j = 0; j < 8; ++j) b8 |= ((live >> (4 * j)) & 1u) << j;
        if (k < 4) live_lo |= b8 << (8 * k);
        else live_hi |= b8 << (8 * (k - 4));
    }
    if (lane == 0) {
        rec->fb = fb;
#pragma unroll
        for (int q = 0; q < 9; ++q) rec->tri[q] = tri[q];
#pragma unroll
        for (int q = 0; q < 3; ++q) {
            rec->cn[q][0] = cn[q][0]; rec->cn[q][1] = cn[q][1]; rec->cn[q][2] = cn[q][2];
            rec->cm[q] = cm[q]; rec->pn[q] = pn[q]; rec->vpad[q] = vpad[q];
        }
        rec->pd = pd; rec->pm = pm; rec->vpadp = vpadp;
        rec->live_blocks[0] = cull ? live_lo : ~0u;
        rec->live_blocks[1] = cull ? live_hi : ~0u;
        sa.boxout[slot] = fb;
        sa.arrive[slot] = 0;
    }
}

// Arrival protocol of skin_small_kernel (SDF term on, at most kSkinSetupMax frames; with more frames the skinning kernels
// write only the chunk boxes and vertices, and sdf_setup_kernel computes every frame's set-up in the next launch, one warp
// per frame).
// Every CTA has written its chunk boxes and vertices; each thread
// fences its own writes (__threadfence: visible device-wide before anything it does later), the CTA barrier orders all of
// them before the one atomicAdd per frame that adds the CTA's chunk count to the frame's counter.  Exactly one CTA sees its
// add complete the frame's nbox: every other CTA's fence-then-add precedes it in the counter's modification order, so
// after its own fence that CTA reads every chunk box and vertex of the frame (through L2).  It computes the set-up and
// puts the counter back to 0; nothing else touches the counter before the next round's skinning launch.
// `mine`: frames whose set-up this CTA computes (bit i = frame base + i), from the caller's adds; `nwarps` warps share them.
__device__ __forceinline__ void sdf_setup_frames(const SdfSetupArgs& sa, const float* bboxp, const float* verts, const int N,
                                                 const int nbox, const int base, unsigned mine, const int warp, const int lane,
                                                 const int nwarps) {
    if (!mine) return;
    __threadfence();
    for (int k = 0; mine; mine &= mine - 1, ++k)
        if (k % nwarps == warp) sdf_frame_setup(sa, bboxp, verts, N, nbox, base + __ffs(mine) - 1, lane);
}

}  // namespace mvs
