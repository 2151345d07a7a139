// Dense vertex forward on the Hopper tensor cores (sm_90a: wgmma + TMA + mbarrier).
//
//   pose_offsets[b, 3n+c] = sum_k  pose_feature[b,k] * posedirs[k, 3n+c]        (lbs.py:192-195)
//
// is the one dense contraction of the path: 20670 posedirs rows x K = 207 against the frames in flight (a few hundred at
// most, usually a few dozen, one to three at the tail of a stage).  It is bound by streaming the 18.5 MB of fp32 posedirs,
// not by tensor throughput, so the kernel is organised to read posedirs exactly once per launch at any active count up to
// one column tile, and to keep enough of it in flight to approach HBM bandwidth:
//
//   transposed product   poffT[3N][frames] = Qk[:, :207] . Phi^T: posedirs rows are the wgmma M side (64 per warpgroup),
//                        the active frames the N side (8 .. 128, the instance is chosen from the host's bound of the
//                        active count; batches above 128 run column tiles of 128 frames as a second grid dimension).  The
//                        accumulator fragment is [coordinate][frame], the layout of poffT, and is stored straight from
//                        registers.
//   warp 8               TMA producer (one thread): per (row tile, k chunk) the fp32 posedirs box 128 x 32 (straight from
//                        the model's Qk rows) and the frames' feature hi and lo boxes, through a 4-stage mbarrier ring.
//   warpgroups 0, 1      64 posedirs rows each: load the fp32 A fragment from shared memory, split it into TF32 hi and lo
//                        in registers, issue wgmma.m64nNk8 with A from registers and B (features) from shared memory; one
//                        wgmma group stays in flight while the next chunk is split, and a ring stage is released once the
//                        group that read it has retired.  CTAs are persistent over a contiguous range of row tiles.
//
// The rest of the vertex forward (template + shape blend shapes in fp32, linear blend skinning, box partials) is
// skin_kernel / skin_small_kernel below.
//
// Precision: error-compensated "3xTF32".  Both operands are split into two TF32 numbers (x = hi + lo, lo = TF32(x - hi)) and
// the tensor cores accumulate hi*hi + lo*hi + hi*lo in fp32 (the dropped lo*lo term is 2^-22 of a product), i.e. the pose
// offsets come out with fp32-class accuracy.  Plain TF32 leaves 1e-6 absolute on a vertex: harmless for the joints, but
// the SDF samples are voxel-sized distances, so it is a 1e-5 .. 1e-4 relative error of the interpenetration term and
// pushes its gradient past the 1e-4 parity bar.  The features are split by the kernels that compute them (PhiTc); posedirs
// is split on chip, so only one fp32 copy of it exists and streams.  Per k8 step the products are issued in the order
// F_hi.P_hi, F_lo.P_hi, F_hi.P_lo, each an exact product of two TF32 numbers accumulated in fp32.
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

template <int NF>
__global__ void __launch_bounds__(kTcThreads, 1)
posedirs_gemm_tc_kernel(const __grid_constant__ CUtensorMap map_p, const __grid_constant__ CUtensorMap map_f, int ldA, int nrows,
                        const int* __restrict__ na_ptr, int cta_slots, int ntiles, float* __restrict__ poffT,
                        int* __restrict__ err_flag) {
    constexpr uint32_t kFBytes = tc_fbytes(NF), kStageBytes = tc_stage_bytes(NF);
    pdl_wait();
    extern __shared__ unsigned char smem_raw[];
    unsigned char* sR = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    // ring: kTcStages x (posedirs fp32 [128 rows][128 B] | features hi [NF rows][128 B] | features lo), all 1024-aligned
    uint64_t* full = reinterpret_cast<uint64_t*>(sR + (size_t)kTcStages * kStageBytes);      // [stages]
    uint64_t* empty = full + kTcStages;                                                      // [stages]

    const int na = *na_ptr;
    const int f0 = blockIdx.y * kTcCols;                              // this CTA's column tile of frames
    if (f0 >= na) return;
    // the launch provides cta_slots CTAs per column tile of the bound; with fewer active column tiles the survivors
    // spread the row tiles over all of them
    const int active_c = (na + kTcCols - 1) / kTcCols;
    const int ctas = max(1, min((int)gridDim.x, cta_slots / active_c));
    if ((int)blockIdx.x >= ctas) return;
    const int tiles_per_cta = (ntiles + ctas - 1) / ctas;
    const int tile_begin = blockIdx.x * tiles_per_cta;
    const int tile_end = min(tile_begin + tiles_per_cta, ntiles);
    if (tile_begin >= tile_end) return;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) TC_MARK(0);

    if (threadIdx.x == 0) {
        for (int s = 0; s < kTcStages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 2); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (threadIdx.x == 0) TC_MARK(1);

    if (warp == 8) {
        if (lane == 0) {
            // ---------------- TMA producer.  Rows past 3N (last row tile) are zero-filled by the tensor map; feature rows
            // past the active frames hold stale slots, which only feed accumulator columns that are never stored.
            // lo parts of the features: rows ldA.. of PhiTc (same tensor map, row offset)
            int stage = 0; uint32_t phase = 0;
            for (int tile = tile_begin; tile < tile_end; ++tile) {
                for (int kc = 0; kc < kTcKCh; ++kc) {
                    if (!mbar_wait(&empty[stage], phase ^ 1, err_flag)) return;
                    unsigned char* sP = sR + (size_t)stage * kStageBytes;
                    mbar_expect_tx(&full[stage], kStageBytes);
                    tma_load_2d(sP, &map_p, kc * kTcBK, tile * kTcRows, &full[stage]);
                    tma_load_2d(sP + kTcPBytes, &map_f, kc * kTcBK, f0, &full[stage]);
                    tma_load_2d(sP + kTcPBytes + kFBytes, &map_f, kc * kTcBK, ldA + f0, &full[stage]);
                    if (++stage == kTcStages) { stage = 0; phase ^= 1; }
                }
            }
        }
        return;
    }

    // ---------------- consumer warpgroup g: posedirs rows 64 g .. 64 g + 63 of each row tile
    const int g = warp >> 2;
    const int wt = threadIdx.x & 127;                                  // thread of the warpgroup
    const int q = lane & 3;
    const int frow = kTcWgRows * g + 16 * (wt >> 5) + (lane >> 2);    // A fragment / accumulator rows frow, frow + 8
    const int xr = (lane >> 2) & 7;                                   // 128-byte swizzle phase of those rows
    float acc[NF / 2];
#pragma unroll
    for (int i = 0; i < NF / 2; ++i) acc[i] = 0.f;
    int stage = 0; uint32_t phase = 0;
    for (int tile = tile_begin; tile < tile_end; ++tile) {
        int held = 0;                                                 // ring stage read by the wgmma group in flight
#pragma unroll
        for (int kc = 0; kc < kTcKCh; ++kc) {
            // a timeout raises the error flag (the host reports it) and the warpgroup carries on: leaving the loop here
            // would be a divergent exit with a wgmma group in flight, which makes ptxas serialise every group
            mbar_wait(&full[stage], phase, err_flag);
            if (kc == 0 && tile == tile_begin && wt == 0) TC_MARK(2);
            const unsigned char* sP = sR + (size_t)stage * kStageBytes;
            const uint32_t bh = smem_u32(sP + kTcPBytes), bl = bh + kFBytes;
#pragma unroll
            for (int k = 0; k < kTcBK / 8; ++k) {
                // A fragment of the k8 step, split x = hi + lo (tf32_split: round to nearest, ties away, as the host-side
                // split of the earlier pre-split copy did); columns k >= 207 hold shape blend shapes and the template in
                // Qk and enter as zero
                uint32_t ahi[4], alo[4];
#pragma unroll
                for (int v = 0; v < 4; ++v) {
                    const int r = frow + 8 * (v & 1), c16 = 2 * k + (v >> 1);        // row, logical 16-byte column group
                    float x = *reinterpret_cast<const float*>(sP + r * 128 + ((c16 ^ xr) << 4) + 4 * q);
                    if (kc * kTcBK + 4 * c16 + q >= kPoseBasis) x = 0.f;
                    float hi, lo;
                    tf32_split(x, hi, lo);
                    ahi[v] = __float_as_uint(hi);
                    alo[v] = __float_as_uint(lo);
                }
                wgmma_fence();                                            // hi*hi, then the two correction products
                WgmmaTf32Rs<NF>::mma(acc, ahi, wgmma_desc_k_sw128(bh + k * 32), (kc | k) ? 1u : 0u);
                WgmmaTf32Rs<NF>::mma(acc, ahi, wgmma_desc_k_sw128(bl + k * 32), 1u);
                WgmmaTf32Rs<NF>::mma(acc, alo, wgmma_desc_k_sw128(bh + k * 32), 1u);
                wgmma_commit();
                // one group in flight while the next fragment is split; once the first group of this chunk is issued,
                // every group of the previous chunk has retired and its ring stage goes back to the producer
                wgmma_wait1();
                if (k == 0 && kc > 0) mbar_arrive_if(&empty[held], wt == 0);
            }
            held = stage;
            if (++stage == kTcStages) { stage = 0; phase ^= 1; }
        }
        wgmma_wait0();
        mbar_arrive_if(&empty[held], wt == 0);
        if (wt == 0) TC_MARK(3 + (tile - tile_begin));
        // d[4 i + 2 h + j] = poffT[row tile + frow + 8 h][f0 + 8 i + 2 q + j]: 32-byte row segments per quad.  Slots past
        // the active count are not stored (ldA is a multiple of 64, so a pair that starts below na stays inside the row).
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int row = tile * kTcRows + frow + 8 * h;
            if (row >= nrows) continue;
            float* dst = poffT + (size_t)row * ldA + f0 + 2 * q;
#pragma unroll
            for (int i = 0; i < NF / 8; ++i)
                if (f0 + 8 * i + 2 * q < na) *reinterpret_cast<float2*>(dst + 8 * i) = make_float2(acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1]);
        }
    }
    if (threadIdx.x == 0) TC_MARK(20);
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
constexpr int kTcInstances[] = {8, 16, 32, 64, 128};       // wgmma N instances of posedirs_gemm_tc_kernel
constexpr int kTcNumInst = 5;

struct TcState {
    CUtensorMap map_p;              // fp32 posedirs: the model's Qk rows [3N][224], box 128 rows x 32
    CUtensorMap map_f[kTcNumInst];  // PhiTc [2][ldA][224] (hi rows, then lo rows), box kTcInstances[i] rows x 32
    float* poffT = nullptr;         // [3N][ldA] pose offsets, frame fastest (output of the tensor-core contraction)
    int* err = nullptr;
    bool ready = false;
};

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

// state of the tensor path (called from mvs_set_model once the Qk rows are on the device: the kernel reads them directly)
int tc_upload_model(mvs_ctx* ctx) {
    TcState* T = new TcState();
    ctx->tc = T;
    int rc;
    if ((rc = dev_alloc(ctx, &T->err, 1))) return rc;
    MVS_CUDA_OK(ctx, cudaMemset(T->err, 0, sizeof(int)));
    return MVS_OK;
}

bool tc_available(const mvs_ctx* ctx) {
    return ctx->exec_mode != 1 && ctx->tc != nullptr && ctx->ws.PhiTc != nullptr;
}

template <int NF>
static int tc_set_smem(mvs_ctx* ctx) {
    MVS_CUDA_OK(ctx, cudaFuncSetAttribute(posedirs_gemm_tc_kernel<NF>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tc_smem(NF)));
    return MVS_OK;
}

int tc_prepare(mvs_ctx* ctx) {
    TcState* T = static_cast<TcState*>(ctx->tc);
    Workspace& w = ctx->ws;
    const DevModel& m = ctx->m;
    if (!T) return set_error(ctx, MVS_ERR_INVALID, "tensor-core path not initialised (mvs_set_model)");
    if (!T->ready) {
        int rc;
        if ((rc = encode_map(ctx, &T->map_p, m.Qk, (uint64_t)3 * m.N, kTcRows))) return rc;
        for (int i = 0; i < kTcNumInst; ++i)                                                       // hi rows, then lo rows
            if ((rc = encode_map(ctx, &T->map_f[i], w.PhiTc, (uint64_t)2 * w.ldA, kTcInstances[i]))) return rc;
        if ((rc = dev_alloc(ctx, &T->poffT, (size_t)3 * m.N * w.ldA))) return rc;
        if ((rc = tc_set_smem<8>(ctx)) || (rc = tc_set_smem<16>(ctx)) || (rc = tc_set_smem<32>(ctx)) || (rc = tc_set_smem<64>(ctx)) ||
            (rc = tc_set_smem<128>(ctx)))
            return rc;
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

int* tc_err_flag(mvs_ctx* ctx) { TcState* T = static_cast<TcState*>(ctx->tc); return T ? T->err : nullptr; }

template <int NF>
static cudaError_t launch_gemm(mvs_ctx* ctx, const TcState* T, int inst, dim3 grid, cudaStream_t st, int ntiles) {
    const Workspace& w = ctx->ws;
    return launch_pdl(posedirs_gemm_tc_kernel<NF>, grid, dim3(kTcThreads), tc_smem(NF), st, T->map_p, T->map_f[inst], w.ldA,
                      3 * ctx->m.N, (const int*)w.na, ctx->sm_count, ntiles, T->poffT, T->err);
}

int launch_vertex_fwd_tc(mvs_ctx* ctx, cudaStream_t st, bool need_vposed, bool sdf_setup) {
    TcState* T = static_cast<TcState*>(ctx->tc);
    Workspace& w = ctx->ws;
    const DevModel& m = ctx->m;
    { const int rc = tc_prepare(ctx); if (rc) return rc; }
    SdfSetupArgs sd{};
    if (sdf_setup) {                                    // the skinning kernel also computes each frame's SDF set-up
        const int rc = ensure_sdf_setup_ws(ctx, st);
        if (rc) return rc;
        sd = make_sdf_setup_args(ctx);
    }
    const int nb = w.na_bound > 0 ? w.na_bound : w.B;             // upper bound of the active-frame count
    const int ntiles = (3 * m.N + kTcRows - 1) / kTcRows;
    const int nf = tc_cols_for(nb);
    dim3 grid(std::min(ctx->sm_count, ntiles), (nb + kTcCols - 1) / kTcCols);   // surplus CTAs exit: the kernel splits the tiles from *na
    MVS_LAUNCH(ctx, KID_VERTEX_FWD_TC, st,
               MVS_CUDA_OK(ctx, nf == 8    ? launch_gemm<8>(ctx, T, 0, grid, st, ntiles)
                                : nf == 16 ? launch_gemm<16>(ctx, T, 1, grid, st, ntiles)
                                : nf == 32 ? launch_gemm<32>(ctx, T, 2, grid, st, ntiles)
                                : nf == 64 ? launch_gemm<64>(ctx, T, 3, grid, st, ntiles)
                                           : launch_gemm<128>(ctx, T, 4, grid, st, ntiles)));
    const int nchunks = (m.N + kSkinV - 1) / kSkinV, fgroups = (nb + 31) / 32;
    const SkinArgs sa{T->poffT, m.ST, w.Phi, w.At, w.ldA, m.ell_j, m.ell_w, m.KW, m.N, need_vposed ? w.vposed : nullptr, w.verts, w.bboxp, sd};
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
