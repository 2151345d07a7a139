// Dense vertex forward on the Hopper tensor cores (sm_90a: wgmma + TMA + mbarrier).
//
//   pose_offsets[b, 3n+c] = sum_k  pose_feature[b,k] * posedirs[k, 3n+c]        (lbs.py:192-195)
//
// is the one dense contraction of the path: M = frames in flight, N = 20670, K = 207.  It is skinny in M
// (<= a few hundred frames), so it is bound by streaming the 17 MB of posedirs from L2/HBM once per 128-frame
// tile, not by tensor throughput; the kernel is therefore organised around keeping the A operand (the frames'
// pose features, 112 KB; only the live 8-row groups are fetched when few frames are active) RESIDENT in shared memory
// for the CTA's whole life while posedirs tiles stream through a TMA ring:
//
//   warpgroup 0      TMA producer (one thread): A once (7 boxes 128x32, or 8-row boxes), then B boxes 96x32 through
//                    a 2-stage mbarrier ring
//   warpgroups 1, 2  wgmma.m64n96k8.f32.tf32 on 64 frames each, fp32 accumulators in registers; each warpgroup
//                    releases a ring stage once its MMAs on it have retired, then stores its 64 x 96 tile of pose
//                    offsets TRANSPOSED (frame fastest) through shared memory and the TMA store engine.  A warpgroup
//                    whose 64 frames are all inactive exits at once.
//
// The rest of the vertex forward (template + shape blend shapes in fp32, linear blend skinning, box partials) is
// skin_kernel / skin_small_kernel below.
//
// Precision: error-compensated "3xTF32".  Both operands are split into two TF32 numbers (x = hi + lo, lo = TF32(x - hi)) and
// the tensor cores accumulate hi*hi + lo*hi + hi*lo in fp32 (the dropped lo*lo term is 2^-22 of a product), i.e. the pose
// offsets come out with fp32-class accuracy.  Plain TF32 leaves 1e-6 absolute on a vertex: harmless for the joints, but
// the SDF samples are voxel-sized distances, so it is a 1e-5 .. 1e-4 relative error of the interpenetration term and
// pushes its gradient past the 1e-4 parity bar.  The path is bound by operand streaming, so the 3x MMA count is free;
// the price is operand traffic (B hi + B lo, and the A lo chunks stream through the ring).
// The template and the shape blend shapes are NOT sent through the tensor cores.
#include <cuda.h>
#include <cudaTypedefs.h>

#include <algorithm>
#include "mvs_internal.cuh"
#include "mvs_tc_dev.cuh"

namespace mvs {

#ifdef MVS_PHASE_DBG
__device__ long long g_tc_clk[32];      // clock64 stamps of CTA (0,0): see scripts/phase_times.py
#define TC_MARK(i) do { if (blockIdx.x == 0 && blockIdx.y == 0) g_tc_clk[i] = clock64(); } while (0)
#else
#define TC_MARK(i) do {} while (0)
#endif

__global__ void __launch_bounds__(kTcThreads, 1)
posedirs_gemm_tc_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_a8,
                        const __grid_constant__ CUtensorMap map_b, const __grid_constant__ CUtensorMap map_o, int ldA, int ncols,
                        const int* __restrict__ na_ptr, int cta_slots, int ntiles, float* __restrict__ poffT,
                        int* __restrict__ err_flag) {
    pdl_wait();
    extern __shared__ unsigned char smem_raw[];
    unsigned char* base = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    unsigned char* sA = base;                                        // A hi: 7 x [128 rows][128 B], 1024-aligned, resident
    unsigned char* sR = sA + (size_t)kTcKCh * kTcABytes;             // ring: kTcStages x (A lo chunk 16 KB | B hi chunk 12 KB | B lo chunk 12 KB)
    float* sO = reinterpret_cast<float*>(sR + (size_t)kTcStages * kTcStageBytes);       // epilogue staging: 2 x [32 columns][64 frames]
    uint64_t* bars = reinterpret_cast<uint64_t*>(sR + (size_t)kTcStages * kTcStageBytes + kTcEpiBytes);
    uint64_t* a_full = bars;                      // [1]
    uint64_t* b_full = bars + 1;                  // [stages]
    uint64_t* b_empty = b_full + kTcStages;       // [stages]

    const int na = *na_ptr;
    const int m0 = blockIdx.y * kTcBM;
    if (m0 >= na) return;
    // the launch provides cta_slots CTAs per M tile of the FULL batch; with fewer active M tiles the survivors
    // spread the vertex tiles over all of them (the tail of a stage runs one M tile on every SM)
    const int active_m = (na + kTcBM - 1) / kTcBM;
    const int ctas_n = max(1, min((int)gridDim.x, cta_slots / active_m));
    if ((int)blockIdx.x >= ctas_n) return;
    const int tiles_per_cta = (ntiles + ctas_n - 1) / ctas_n;
    const int tile_begin = blockIdx.x * tiles_per_cta;
    const int tile_end = min(tile_begin + tiles_per_cta, ntiles);
    if (tile_begin >= tile_end) return;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int live_rows = min(kTcBM, na - m0);
    const int live_wgs = (live_rows + kTcWgM - 1) / kTcWgM;          // consumer warpgroups with at least one active frame
    if (threadIdx.x == 0) TC_MARK(0);

    if (threadIdx.x == 0) {
        mbar_init(a_full, 1);
        for (int s = 0; s < kTcStages; ++s) { mbar_init(&b_full[s], 1); mbar_init(&b_empty[s], live_wgs); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (threadIdx.x == 0) TC_MARK(1);

    if (warp < 4) {
        if (warp == 0 && lane == 0) {
            // ---------------- TMA producer
            // A operand.  Every CTA of the M tile reads it, so with one CTA per SM the 112 KB tile costs as much L2
            // traffic as posedirs itself; at the tail of a fit only a few of its 128 rows are live, and those are fetched
            // as 8-row boxes (one swizzle atom each: same shared-memory image).  Rows that are not loaded hold whatever
            // was there: their accumulator rows are never stored.
            // lo parts: rows ldA.. of the A array, rows ncols.. of the posedirs array (same tensor maps, row offset)
            const bool small = live_rows <= 32;
            const int groups = (live_rows + 7) / 8;
            if (small) {
                mbar_expect_tx(a_full, kTcKCh * groups * 8 * kTcBK * 4);
                for (int kc = 0; kc < kTcKCh; ++kc)
                    for (int gq = 0; gq < groups; ++gq)
                        tma_load_2d(sA + (size_t)kc * kTcABytes + (size_t)gq * 1024, &map_a8, kc * kTcBK, m0 + 8 * gq, a_full);
            } else {
                mbar_expect_tx(a_full, kTcKCh * kTcABytes);
                for (int kc = 0; kc < kTcKCh; ++kc) tma_load_2d(sA + (size_t)kc * kTcABytes, &map_a, kc * kTcBK, m0, a_full);
            }
            const uint32_t stage_bytes = (small ? groups * 8 * kTcBK * 4 : kTcABytes) + 2 * kTcBBytes;
            int stage = 0; uint32_t phase = 0;
            for (int tile = tile_begin; tile < tile_end; ++tile) {
                for (int kc = 0; kc < kTcKCh; ++kc) {
                    if (!mbar_wait(&b_empty[stage], phase ^ 1, err_flag)) return;
                    unsigned char* sAl = sR + (size_t)stage * kTcStageBytes;
                    unsigned char* sBh = sAl + kTcABytes;
                    unsigned char* sBl = sBh + kTcBBytes;
                    mbar_expect_tx(&b_full[stage], stage_bytes);
                    if (small) {
                        for (int gq = 0; gq < groups; ++gq) tma_load_2d(sAl + (size_t)gq * 1024, &map_a8, kc * kTcBK, ldA + m0 + 8 * gq, &b_full[stage]);
                    } else {
                        tma_load_2d(sAl, &map_a, kc * kTcBK, ldA + m0, &b_full[stage]);
                    }
                    tma_load_2d(sBh, &map_b, kc * kTcBK, tile * kTcBN, &b_full[stage]);
                    tma_load_2d(sBl, &map_b, kc * kTcBK, ncols + tile * kTcBN, &b_full[stage]);
                    if (++stage == kTcStages) { stage = 0; phase ^= 1; }
                }
            }
        }
        return;
    }

    // ---------------- consumer warpgroup g: frames m0 + 64 g .. m0 + 64 g + 63
    const int g = warp / 4 - 1;
    if (g >= live_wgs) return;
    const int wt = threadIdx.x - 128 * (g + 1);                       // thread of the warpgroup
    const uint32_t a_row_off = (uint32_t)(g * kTcWgM * kTcBK * 4);    // 64 rows of 128 B = 8 swizzle atoms
    float* sOw = sO + (size_t)g * kTcEpiCols * kTcWgM;
    const int row = 16 * (wt >> 5) + ((wt & 31) >> 2);                // accumulator rows row, row + 8
    const int colq = 2 * (wt & 3);                                    // accumulator columns 8 i + colq (+ 1)
    float acc[kTcBN / 2];
#pragma unroll
    for (int i = 0; i < kTcBN / 2; ++i) acc[i] = 0.f;
    if (!mbar_wait(a_full, 0, err_flag)) return;
    if (wt == 0) TC_MARK(2);
    int stage = 0; uint32_t phase = 0;
    for (int tile = tile_begin; tile < tile_end; ++tile) {
        for (int kc = 0; kc < kTcKCh; ++kc) {
            if (!mbar_wait(&b_full[stage], phase, err_flag)) return;
            const uint32_t ah = smem_u32(sA + (size_t)kc * kTcABytes) + a_row_off;
            const uint32_t al = smem_u32(sR + (size_t)stage * kTcStageBytes) + a_row_off;
            const uint32_t bh = smem_u32(sR + (size_t)stage * kTcStageBytes) + kTcABytes, bl = bh + kTcBBytes;
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < kTcBK / 8; ++k) {                  // hi*hi, then the two correction products
                wgmma_m64n96k8_tf32(acc, wgmma_desc_k_sw128(ah + k * 32), wgmma_desc_k_sw128(bh + k * 32), (kc | k) ? 1u : 0u);
                wgmma_m64n96k8_tf32(acc, wgmma_desc_k_sw128(al + k * 32), wgmma_desc_k_sw128(bh + k * 32), 1u);
                wgmma_m64n96k8_tf32(acc, wgmma_desc_k_sw128(ah + k * 32), wgmma_desc_k_sw128(bl + k * 32), 1u);
            }
            wgmma_commit();
            wgmma_wait0();
            if (wt == 0) mbar_arrive(&b_empty[stage]);              // this warpgroup's MMAs on the stage have retired
            if (++stage == kTcStages) { stage = 0; phase ^= 1; }
        }
        if (wt == 0) TC_MARK(3 + (tile - tile_begin));
        // The tile leaves through shared memory and the TMA store engine, 32 columns ([column][frame] rows of 256 B) at a
        // time: the warpgroup fills its staging tile, one thread issues the bulk tensor store, which clips the box at the
        // array bounds (last vertex tile, frame padding).  Rows of slots that are not active hold whatever the accumulator
        // held: nobody reads them.
        const int c0 = tile * kTcBN;
#pragma unroll
        for (int ch = 0; ch < kTcBN / kTcEpiCols; ++ch) {          // unrolled: acc[] stays in registers
            if (c0 + ch * kTcEpiCols >= ncols) break;
            if (wt == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");   // staging tile free again
            asm volatile("bar.sync %0, 128;" ::"r"(1 + g) : "memory");
#pragma unroll
            for (int i = 0; i < kTcEpiCols / 8; ++i)
#pragma unroll
                for (int h = 0; h < 2; ++h)
#pragma unroll
                    for (int j = 0; j < 2; ++j)
                        sOw[(8 * i + colq + j) * kTcWgM + row + 8 * h] = acc[4 * (ch * kTcEpiCols / 8 + i) + 2 * h + j];
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            asm volatile("bar.sync %0, 128;" ::"r"(1 + g) : "memory");
            if (wt == 0) tma_store_2d(&map_o, sOw, m0 + g * kTcWgM, c0 + ch * kTcEpiCols);
        }
    }
    if (wt == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");         // all stores of this warpgroup have landed
    if (threadIdx.x == 128) TC_MARK(20);
}

__global__ void __launch_bounds__(kSkinThreads)
skin_kernel(SkinArgs ar, const int* __restrict__ na_ptr, int cta_slots) {
    pdl_wait();
    extern __shared__ __align__(16) float sk[];
    skin_body(sk, ar, *na_ptr, cta_slots, (int)blockIdx.x, (int)blockIdx.y);
}

__global__ void __launch_bounds__(kSkinSmallThreads)
skin_small_kernel(SkinArgs ar, const int* __restrict__ na_ptr) {
    __shared__ SkinSmallSmem sm;
    pdl_wait();
    skin_small_body(sm, ar, *na_ptr, (int)blockIdx.x, (int)gridDim.x, (int)threadIdx.x, 0);
}

// ------------------------------------------------------------------------------------------------ host side
struct TcState {
    CUtensorMap map_a, map_a8, map_b, map_o;
    float* Qtc = nullptr;       // [2][3N][224] posedirs rows split into TF32 hi | lo parts (columns >= 207 zero)
    float* poffT = nullptr;     // [3N][ldA] pose offsets, frame fastest (output of the tensor-core contraction)
    int* err = nullptr;
    bool ready = false;
};

static float round_tf32(float x) {                      // cvt.rna.tf32.f32: nearest, ties away from zero
    uint32_t u;
    memcpy(&u, &x, 4);
    if ((u & 0x7F800000u) == 0x7F800000u) return x;
    u = (u + 0x1000u) & 0xFFFFE000u;
    float r;
    memcpy(&r, &u, 4);
    return r;
}

static int encode_map(mvs_ctx* ctx, CUtensorMap* map, const float* ptr, uint64_t rows, uint32_t box_rows) {
    static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
    if (!fn) {
        cudaDriverEntryPointQueryResult q;
        void* p = nullptr;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || !p)
            return set_error(ctx, MVS_ERR_CUDA, "cuTensorMapEncodeTiled is not available from the driver");
        fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(p);
    }
    cuuint64_t dims[2] = {(cuuint64_t)kFeatPad, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)kFeatPad * sizeof(float)};
    cuuint32_t box[2] = {(cuuint32_t)kTcBK, box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(ptr), dims, strides, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return set_error(ctx, MVS_ERR_CUDA, "cuTensorMapEncodeTiled failed (%d)", (int)r);
    return MVS_OK;
}

// output of the contraction: poffT [ncols][ldA] fp32, frame fastest; box = 64 frames x kTcEpiCols columns, no swizzle
static int encode_out_map(mvs_ctx* ctx, CUtensorMap* map, float* ptr, uint64_t ldA, uint64_t ncols) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || !p)
        return set_error(ctx, MVS_ERR_CUDA, "cuTensorMapEncodeTiled is not available from the driver");
    auto fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(p);
    cuuint64_t dims[2] = {(cuuint64_t)ldA, (cuuint64_t)ncols};
    cuuint64_t strides[1] = {(cuuint64_t)ldA * sizeof(float)};
    cuuint32_t box[2] = {(cuuint32_t)kTcWgM, (cuuint32_t)kTcEpiCols};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, ptr, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return set_error(ctx, MVS_ERR_CUDA, "cuTensorMapEncodeTiled (output) failed (%d)", (int)r);
    return MVS_OK;
}

// posedirs copy for the tensor path (called from mvs_set_model with the host Qk rows)
int tc_upload_model(mvs_ctx* ctx, const float* Qk_host) {
    TcState* T = new TcState();
    ctx->tc = T;
    const size_t n = (size_t)3 * ctx->m.N * kFeatPad;
    std::vector<float> q(2 * n);                 // hi rows, then lo rows: posedirs = hi + lo, both TF32 (hi - x is exact in fp32)
    for (size_t i = 0; i < n; ++i) {
        const bool pose = (i % kFeatPad) < (size_t)kPoseBasis;
        const float hi = pose ? round_tf32(Qk_host[i]) : 0.f;
        q[i] = hi;
        q[n + i] = pose ? round_tf32(Qk_host[i] - hi) : 0.f;
    }
    int rc = dev_upload(ctx, &T->Qtc, q.data(), 2 * n);
    if (rc) return rc;
    if ((rc = dev_alloc(ctx, &T->err, 1))) return rc;
    MVS_CUDA_OK(ctx, cudaMemset(T->err, 0, sizeof(int)));
    return MVS_OK;
}

bool tc_available(const mvs_ctx* ctx) {
    return ctx->exec_mode != 1 && ctx->tc != nullptr && ctx->ws.PhiTc != nullptr;
}

int tc_prepare(mvs_ctx* ctx) {
    TcState* T = static_cast<TcState*>(ctx->tc);
    Workspace& w = ctx->ws;
    const DevModel& m = ctx->m;
    if (!T) return set_error(ctx, MVS_ERR_INVALID, "tensor-core path not initialised (mvs_set_model)");
    if (!T->ready) {
        int rc;
        if ((rc = encode_map(ctx, &T->map_a, w.PhiTc, (uint64_t)2 * w.ldA, kTcBM))) return rc;       // hi rows, then lo rows
        if ((rc = encode_map(ctx, &T->map_a8, w.PhiTc, (uint64_t)2 * w.ldA, 8))) return rc;
        if ((rc = encode_map(ctx, &T->map_b, T->Qtc, (uint64_t)2 * 3 * m.N, kTcBN))) return rc;
        if ((rc = dev_alloc(ctx, &T->poffT, (size_t)3 * m.N * w.ldA))) return rc;
        if ((rc = encode_out_map(ctx, &T->map_o, T->poffT, (uint64_t)w.ldA, (uint64_t)3 * m.N))) return rc;
        MVS_CUDA_OK(ctx, cudaFuncSetAttribute(posedirs_gemm_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kTcSmem));
        MVS_CUDA_OK(ctx, cudaFuncSetAttribute(skin_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSkinSmem));
        T->ready = true;
    }
    return MVS_OK;
}

float* tc_poffT(mvs_ctx* ctx) {
    TcState* T = static_cast<TcState*>(ctx->tc);
    if (!T || tc_prepare(ctx) != MVS_OK) return nullptr;
    return T->poffT;
}

const void* tc_maps(mvs_ctx* ctx) {            // [map_a, map_a8, map_b] (CUtensorMap x 3) for the persistent dense-round kernel
    TcState* T = static_cast<TcState*>(ctx->tc);
    if (!T || tc_prepare(ctx) != MVS_OK) return nullptr;
    return &T->map_a;
}
int* tc_err_flag(mvs_ctx* ctx) { TcState* T = static_cast<TcState*>(ctx->tc); return T ? T->err : nullptr; }

int launch_vertex_fwd_tc(mvs_ctx* ctx, cudaStream_t st, bool need_vposed) {
    TcState* T = static_cast<TcState*>(ctx->tc);
    Workspace& w = ctx->ws;
    const DevModel& m = ctx->m;
    { const int rc = tc_prepare(ctx); if (rc) return rc; }
    const int ntiles = (m.N + kTileV - 1) / kTileV;
    const int nb = w.na_bound > 0 ? w.na_bound : w.B;             // upper bound of the active-frame count
    const int mtiles = (nb + kTcBM - 1) / kTcBM;
    dim3 grid(std::min(ctx->sm_count, ntiles), mtiles);          // surplus CTAs exit: the kernel splits the tiles from *na
    MVS_LAUNCH(ctx, KID_VERTEX_FWD_TC, st,
               MVS_CUDA_OK(ctx, launch_pdl(posedirs_gemm_tc_kernel, grid, dim3(kTcThreads), kTcSmem, st, T->map_a, T->map_a8, T->map_b, T->map_o, w.ldA,
                                           3 * m.N, (const int*)w.na, ctx->sm_count, ntiles, T->poffT, T->err)));
    const int nchunks = (m.N + kSkinV - 1) / kSkinV, fgroups = (nb + 31) / 32;
    const SkinArgs sa{T->poffT, m.ST, w.Phi, w.At, w.ldA, m.ell_j, m.ell_w, m.KW, m.N, need_vposed ? w.vposed : nullptr, w.verts, w.bboxp};
    if (nb <= kSkinSmallMax) {                          // straggler tail: lane = vertex, one chunk per CTA
        MVS_LAUNCH(ctx, KID_SKIN, st,
                   MVS_CUDA_OK(ctx, launch_pdl(skin_small_kernel, dim3(nchunks), dim3(kSkinSmallThreads), 0, st, sa, (const int*)w.na)));
    } else {
        // each CTA keeps its 32 frames' transforms in shared memory and walks 1..3 chunks (sized from *na in the kernel)
        dim3 g2(nchunks, fgroups);                      // surplus CTAs exit
        MVS_LAUNCH(ctx, KID_SKIN, st,
                   MVS_CUDA_OK(ctx, launch_pdl(skin_kernel, g2, dim3(kSkinThreads), kSkinSmem, st, sa, (const int*)w.na, 2 * ctx->sm_count)));
    }
    MVS_CUDA_OK(ctx, cudaGetLastError());
    return MVS_OK;
}

int tc_check_error(mvs_ctx* ctx) {          // host-side check after a synchronisation point
    TcState* T = static_cast<TcState*>(ctx->tc);
    if (!T || !T->ready) return MVS_OK;
    int e = 0;
    MVS_CUDA_OK(ctx, cudaMemcpy(&e, T->err, sizeof(int), cudaMemcpyDeviceToHost));
    if (e) return set_error(ctx, MVS_ERR_CUDA, "vertex_fwd_tc_kernel: mbarrier wait timed out (pipeline protocol error)");
    return MVS_OK;
}

}  // namespace mvs

#ifdef MVS_PHASE_DBG
extern "C" int mvs_debug_tc_clocks(long long* out, int n) {       // debug builds only; not part of the ABI
    long long h[32];
    if (cudaMemcpyFromSymbol(h, mvs::g_tc_clk, sizeof(h)) != cudaSuccess) return -1;
    for (int i = 0; i < n && i < 32; ++i) out[i] = h[i];
    return 0;
}
#endif
