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
//   ring                 the TMA / wgmma ring of mvs_tc_dev.cuh.  Warp 8 is its producer: per (row tile, k chunk) the fp32
//                        posedirs box 128 x 32 (straight from the model's Qk rows) and the frames' feature hi and lo boxes.
//   warpgroups 0, 1      its consumers, 64 posedirs rows each: A (posedirs) gathered from the swizzled box, B (features) from
//                        shared memory.  CTAs are persistent over a contiguous range of row tiles.
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
#include <type_traits>
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

    const Ring<kStageBytes> ring = ring_setup<kStageBytes>(smem_raw, kTcRows / kTcWgRows);
    if (threadIdx.x == 0) TC_MARK(1);

    if (warp == 8) {
        // ---------------- TMA producer.  Rows past 3N (last row tile) are zero-filled by the tensor map; feature rows past
        // the active frames hold stale slots, which only feed accumulator columns that are never stored.  lo parts of the
        // features: rows ldA.. of PhiTc (same tensor map, row offset)
        if (lane == 0)
            ring_produce<kTcKCh>(ring, tile_begin, tile_end, err_flag, [&](int tile, int kc, unsigned char* sP, uint64_t* bar) {
                tma_load_2d(sP, &map_p, kc * kTcBK, tile * kTcRows, bar);
                tma_load_2d(sP + kTcPBytes, &map_f, kc * kTcBK, f0, bar);
                tma_load_2d(sP + kTcPBytes + kFBytes, &map_f, kc * kTcBK, ldA + f0, bar);
            });
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
    RingPos pos;
    for (int tile = tile_begin; tile < tile_end; ++tile) {
        int held = 0;                                                 // ring stage read by the wgmma group in flight
#pragma unroll
        for (int kc = 0; kc < kTcKCh; ++kc) {
            ring.wait_full(pos, err_flag);
            if (kc == 0 && tile == tile_begin && wt == 0) TC_MARK(2);
            // (spelled out: through Ring::stage, ptxas allocates the unrolled k8 steps' registers differently)
            const unsigned char* sP = ring.base + (size_t)pos.stage * kStageBytes;
            const uint32_t bh = smem_u32(sP + kTcPBytes), bl = bh + kFBytes;
#pragma unroll
            for (int k = 0; k < kTcBK / 8; ++k) {
                // A fragment of the k8 step; columns k >= 207 hold shape blend shapes and the template in Qk and enter as zero
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
                wgmma_wait1();
                if (k == 0 && kc > 0) mbar_arrive_if(&ring.empty[held], wt == 0);
            }
            held = pos.next();
        }
        wgmma_wait0();
        mbar_arrive_if(&ring.empty[held], wt == 0);
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

// The blend-shape adjoint of mvs_forward_vjp on the tensor cores:
//
//   dPhi[b][k] = sum_r dVp[b][r] Qk[r][k]        r over the 3N posedirs rows (K = 20670), k over the 224 feature columns
//
// run as dPhi^T = Qk^T . dVp^T: the features are the wgmma M side (four consumer warpgroups of 64 features, 256 >= 224), the
// frames the N side (8 .. 64 per column tile), the posedirs rows the reduction.  Split-K: CTA (s, c) sums the rows of strip s
// (a contiguous range of 32-row chunks) for column tile c and writes its partial into the feature columns of
// part[s][slot][288 ..] -- the per-strip layout frame_bwd_kernel reduces, in strip order, next to the skinning partials
// vertex_bwd_kernel<true> wrote.  No atomics: the sum has a fixed order, so a call gives the same bits every time.
//   ring                 the TMA / wgmma ring of mvs_tc_dev.cuh.  Warp 16 is its producer: per 32-row chunk the seven 32 x 32
//                        boxes of Qk (fp32, the model's rows) and the frames' dVp hi and lo boxes (vertex_bwd_kernel<true>).
//   warpgroups 0 .. 3    its consumers: A (Qk^T: feature x row) gathered from the swizzled boxes, B (dVp) from shared memory.
constexpr int kTbRows = 32;                                 // posedirs rows per ring stage (the reduction chunk)
constexpr int kTbBoxes = kFeatPad / 32;                     // 7 boxes of 32 features per row chunk
constexpr int kTbQBytes = kTbBoxes * kTbRows * 128;         // 28 KB of Qk per stage
constexpr int kTbWg = 4;                                    // consumer warpgroups
constexpr int kTbThreads = 128 * kTbWg + 32;                // + the producer warp
constexpr int kTbCols = 64;                                 // largest frame column tile (wgmma N)
__host__ __device__ constexpr int tb_stage_bytes(int nf) { return kTbQBytes + 2 * tc_fbytes(nf); }   // Qk boxes | dVp hi | lo
__host__ __device__ constexpr int tb_dvp_ld(int N) { return (3 * N + 3) / 4 * 4; }       // 16-byte rows for the tensor map

template <int NF>
__global__ void __launch_bounds__(kTbThreads, 1)
vertex_bwd_tc_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_d, int ldA,
                     const int* __restrict__ na_ptr, int nchunks, float* __restrict__ part, int* __restrict__ err_flag) {
    constexpr uint32_t kFBytes = tc_fbytes(NF), kStageBytes = tb_stage_bytes(NF);
    extern __shared__ unsigned char smem_raw[];
    const int na = *na_ptr;
    const int f0 = blockIdx.y * NF;
    if (f0 >= na) return;
    const int strip = blockIdx.x;
    const int per = (nchunks + gridDim.x - 1) / gridDim.x;
    const int c_begin = min(strip * per, nchunks), c_end = min(c_begin + per, nchunks);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const Ring<kStageBytes> ring = ring_setup<kStageBytes>(smem_raw, kTbWg);
    if (warp == 4 * kTbWg) {
        if (lane == 0)                 // TMA producer; rows past 3N (last chunk) are zero-filled by both tensor maps
            ring_produce<1>(ring, c_begin, c_end, err_flag, [&](int kc, int, unsigned char* sP, uint64_t* bar) {
                for (int bx = 0; bx < kTbBoxes; ++bx) tma_load_2d(sP + bx * kTbRows * 128, &map_q, 32 * bx, kc * kTbRows, bar);
                tma_load_2d(sP + kTbQBytes, &map_d, kc * kTbRows, f0, bar);
                tma_load_2d(sP + kTbQBytes + kFBytes, &map_d, kc * kTbRows, ldA + f0, bar);
            });
        return;
    }
    // consumer warpgroup g: features 64 g + 16 w + lr (+ 8), w = warp of the warpgroup, lr = lane / 4; rows q, q + 4 of each k8
    const int g = warp >> 2, wt = threadIdx.x & 127, w = wt >> 5, q = lane & 3, lr = lane >> 2;
    const int fa = 64 * g + 16 * w + lr;                      // feature of a[0], a[2]; a[1], a[3] have fa + 8 (same box)
    const bool fvalid = fa < kFeatPad;                        // warpgroup 3's upper half is past the 224 columns
    const int box = min(fa >> 5, kTbBoxes - 1), ca = fa & 31;
    float acc[NF / 2];
#pragma unroll
    for (int i = 0; i < NF / 2; ++i) acc[i] = 0.f;
    RingPos pos;
    int held = -1;                                            // ring stage read by the wgmma group in flight
    for (int kc = c_begin; kc < c_end; ++kc) {
        ring.wait_full(pos, err_flag);
        const unsigned char* sS = ring.stage(pos.stage);
        const unsigned char* sQ = sS + box * kTbRows * 128;
        const uint32_t bh = smem_u32(sS + kTbQBytes), bl = bh + kFBytes;
#pragma unroll
        for (int k = 0; k < kTbRows / 8; ++k) {
            uint32_t ahi[4], alo[4];
#pragma unroll
            for (int v = 0; v < 4; ++v) {
                const int r = 8 * k + q + 4 * (v >> 1), c = ca + 8 * (v & 1);     // row of the chunk, column of the box
                float x = *reinterpret_cast<const float*>(sQ + r * 128 + ((((c >> 2) ^ (r & 7))) << 4) + 4 * (c & 3));
                if (!fvalid) x = 0.f;
                float hi, lo;
                tf32_split(x, hi, lo);
                ahi[v] = __float_as_uint(hi);
                alo[v] = __float_as_uint(lo);
            }
            wgmma_fence();
            WgmmaTf32Rs<NF>::mma(acc, ahi, wgmma_desc_k_sw128(bh + k * 32), 1u);
            WgmmaTf32Rs<NF>::mma(acc, ahi, wgmma_desc_k_sw128(bl + k * 32), 1u);
            WgmmaTf32Rs<NF>::mma(acc, alo, wgmma_desc_k_sw128(bh + k * 32), 1u);
            wgmma_commit();
            wgmma_wait1();                                    // the previous chunk's groups have retired: its stage is free
            if (k == 0 && held >= 0) mbar_arrive_if(&ring.empty[held], wt == 0);
        }
        held = pos.next();
    }
    wgmma_wait0();
    // d[4 i + 2 h + j] = dPhi^T[feature fa + 8 h][frame f0 + 8 i + 2 q + j]
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int f = fa + 8 * h;
        if (f >= kFeatPad) continue;
#pragma unroll
        for (int i = 0; i < NF / 8; ++i)
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                const int slot = f0 + 8 * i + 2 * q + j;
                if (slot < na) part[((size_t)strip * ldA + slot) * kPartFloats + kSkinFloats + f] = acc[4 * i + 2 * h + j];
            }
    }
}

// grid (nchunks, frame groups of 32); kSkinSmem bytes of dynamic shared memory
__global__ void __launch_bounds__(kSkinThreads)
skin_kernel(SkinArgs ar, const int* __restrict__ na_ptr, int cta_slots) {
    pdl_wait();
    extern __shared__ __align__(16) float sk[];
    const int na = *na_ptr;
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
    const int f0 = blockIdx.y * 32;
    if (f0 >= na) return;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int slotc = min(f0 + lane, na - 1);
    // chunks per CTA from the number of ACTIVE frame groups: one chunk each while the active CTAs fit in one wave
    // (latency at the tail of a stage), several once they do not (the 36 KB of transforms are then loaded once)
    const int nchunks = (N + kSkinV - 1) / kSkinV;
    const int per_cta = (nchunks * ((na + 31) / 32) + cta_slots - 1) / cta_slots;
    const int nx = (nchunks + per_cta - 1) / per_cta;
    if ((int)blockIdx.x >= nx) return;
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
    for (int ch = blockIdx.x; ch < nchunks; ch += nx) {
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
    // (SDF term on: the frames' set-ups are sdf_setup_kernel's, the next launch)
}

// The same for a handful of frames (the straggler tail of a fit): with lane = frame almost every lane of skin_kernel
// idles and its fixed costs (36 KB of transforms per CTA, staging, three barriers per chunk) are pure latency.  Here
// lane = vertex, a CTA owns one 64-vertex chunk (= one box partial) and loops over the <= kSkinSmallMax frames.  With the
// SDF term on and at most kSkinSetupMax frames it also computes the frames' set-ups at its end (sdf_setup_frames), so the
// smallest rounds keep the four launches the dispatch tests fix (tests/test_gpu_dispatch.py runs 4 frames; DESIGN.md
// section 5); its 2 warps take ceil(na / 2) set-ups each, one after the other.  Above that
// sdf_setup_kernel computes them, one set-up deep plus a dependent launch: at 8 frames a round takes 127 us instead of 137
// (H100, scripts/round_times.py; DESIGN.md section 5 has the sizes below).
constexpr int kSkinSmallMax = 8;
constexpr int kSkinSetupMax = 4;
constexpr int kSkinSmallThreads = 64;
static_assert(kSkinSmallThreads == kSkinV, "one thread per vertex of a box chunk");

struct SkinSmallSmem {
    float As[kSkinSmallMax][kSkinFloats];
    float Bs[kSkinSmallMax][kBetas];
    float s_b[kSkinSmallMax][6];
    int s_i[kSkinSmallMax][6];
    unsigned mine;                         // frames whose SDF set-up this CTA computes
};

// one CTA per 64-vertex chunk, thread t = vertex of the chunk
__global__ void __launch_bounds__(kSkinSmallThreads)
skin_small_kernel(SkinArgs ar, const int* __restrict__ na_ptr) {
    __shared__ SkinSmallSmem sm;
    pdl_wait();
    const int t = threadIdx.x, chunk = blockIdx.x, nchunks = gridDim.x;
    const float* poffT = ar.poffT; const float* __restrict__ ST = ar.ST; const float* Phi = ar.Phi; const float* At = ar.At;
    const int ldA = ar.ldA, KW = ar.KW, N = ar.N;
    const int* __restrict__ ell_j = ar.ell_j; const float* __restrict__ ell_w = ar.ell_w;
    float* vposed = ar.vposed; float* verts = ar.verts; float* bboxp = ar.bboxp;
    auto& As = sm.As; auto& Bs = sm.Bs; auto& s_b = sm.s_b; auto& s_i = sm.s_i;
    const int na = min(*na_ptr, kSkinSmallMax);
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
    __syncthreads();
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
            __syncthreads();
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
    if (ar.sdf.rec != nullptr) {                          // per-frame SDF set-up by the last CTA of each frame (sdf_setup_frames)
        __threadfence();
        __syncthreads();
        if (warp == 0) {
            const bool last = lane < na && atomicAdd(ar.sdf.arrive + lane, 1) + 1 == nchunks;   // one chunk per CTA
            const unsigned m = __ballot_sync(0xffffffffu, last);
            if (lane == 0) sm.mine = m;
        }
        __syncthreads();
        sdf_setup_frames(ar.sdf, bboxp, verts, N, nchunks, 0, sm.mine, warp, lane, kSkinSmallThreads / 32);
    }
}

// The per-frame SDF set-up after the skinning kernel (SDF term on, more than kSkinSetupMax frames): one warp per active
// slot calls sdf_frame_setup on the chunk boxes and vertices the previous launch wrote.  In skin_kernel the CTA that
// completed a frame's chunks computed it, usually the same CTA for all 32 frames of a group, so its 8 warps ran 4 set-ups
// each, one after the other, at the end of the launch.  Here every frame's set-up runs in parallel with the others.
constexpr int kSetupWarps = 4;                             // frames per CTA
__global__ void __launch_bounds__(32 * kSetupWarps)
sdf_setup_kernel(const SdfSetupArgs sa, const float* bboxp, const float* verts, const int N, const int nbox,
                 const int* __restrict__ na_ptr) {
    pdl_wait();                                            // every thread: sdf_fused's wait then also covers the skinning
    const int slot = blockIdx.x * kSetupWarps + (threadIdx.x >> 5);
    if (slot >= *na_ptr) return;                           // whole warps: the set-up uses warp-wide reductions
    sdf_frame_setup(sa, bboxp, verts, N, nbox, slot, threadIdx.x & 31);
}

// ------------------------------------------------------------------------------------------------ host side
constexpr int kTcInstances[] = {8, 16, 32, 64, 128};       // wgmma N instances (frames per column tile); the VJP has the first 4
constexpr int kTcNumInst = 5, kTbNumInst = 4;
static_assert(kTcInstances[kTcNumInst - 1] == kTcCols && kTcInstances[kTbNumInst - 1] == kTbCols, "instances up to the column tiles");

// f(std::integral_constant<int, kTcInstances[I]>(), I) for the instance equal to nf; the kernel templates are instantiated
// for the instances up to kMax only.  Returns f's error, cudaErrorInvalidValue if no instance matches.
template <int kMax, int I = 0, class F>
static cudaError_t with_instance(int nf, F f) {
    if constexpr (I == kTcNumInst || kTcInstances[I] > kMax) return cudaErrorInvalidValue;
    else return nf == kTcInstances[I] ? f(std::integral_constant<int, kTcInstances[I]>(), I) : with_instance<kMax, I + 1>(nf, f);
}

struct TcState {
    CUtensorMap map_p;              // fp32 posedirs: the model's Qk rows [3N][224], box 128 rows x 32
    CUtensorMap map_f[kTcNumInst];  // PhiTc [2][ldA][224] (hi rows, then lo rows), box kTcInstances[i] rows x 32
    float* poffT = nullptr;         // [3N][ldA] pose offsets, frame fastest (output of the tensor-core contraction)
    int* err = nullptr;
    // mvs_forward_vjp (vertex_bwd_tc_kernel), set up on first use
    CUtensorMap map_q;              // the model's Qk rows [3N][224], box 32 rows x 32
    CUtensorMap map_d[kTbNumInst];  // dvp [2][ldA][3N] (row stride ldR), box kTcInstances[i] rows x 32
    float* dvp = nullptr;           // [2][ldA][ldR] d v_posed split into TF32 hi | lo (vertex_bwd_kernel<true>)
};

// 2-D fp32 tensor map [rows][cols] (row stride ld floats), box box_rows x 32 floats, 128-byte swizzle
static int encode_map(mvs_ctx* ctx, CUtensorMap* map, const float* ptr, uint64_t rows, uint32_t box_rows,
                      uint64_t cols = kFeatPad, uint64_t ld = kFeatPad) {
    static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
    if (!fn) {
        cudaDriverEntryPointQueryResult q;
        void* p = nullptr;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || !p)
            return set_error(ctx, MVS_ERR_CUDA, "cuTensorMapEncodeTiled is not available from the driver");
        fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(p);
    }
    cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)ld * sizeof(float)};
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
    int* err = nullptr;
    if (int rc = dev_alloc(ctx, &err, 1)) return rc;
    MVS_CUDA_OK(ctx, cudaMemset(err, 0, sizeof(int)));
    ctx->tc = new TcState();
    ctx->tc->err = err;
    return MVS_OK;
}

void release_tc_state(mvs_ctx* ctx) {
    delete ctx->tc;
    ctx->tc = nullptr;
}

// kernel attributes and the tensor maps over the model's Qk rows and the batch's PhiTc
int tc_set_attributes(mvs_ctx* ctx) {
    TcState* T = ctx->tc;
    const Workspace& w = ctx->ws;
    int rc;
    if ((rc = encode_map(ctx, &T->map_p, ctx->m.Qk, (uint64_t)3 * ctx->m.N, kTcRows))) return rc;
    for (int i = 0; i < kTcNumInst; ++i)                                                           // hi rows, then lo rows
        if ((rc = encode_map(ctx, &T->map_f[i], w.PhiTc, (uint64_t)2 * w.ldA, kTcInstances[i]))) return rc;
    constexpr cudaFuncAttribute kSmem = cudaFuncAttributeMaxDynamicSharedMemorySize;
    for (int nf : kTcInstances)
        MVS_CUDA_OK(ctx, with_instance<kTcCols>(nf, [&](auto n, int) {
                        cudaError_t e = cudaFuncSetAttribute(posedirs_gemm_tc_kernel<n>, kSmem, (int)ring_smem(tc_stage_bytes(n)));
                        if constexpr (n <= kTbCols)
                            if (e == cudaSuccess) e = cudaFuncSetAttribute(vertex_bwd_tc_kernel<n>, kSmem, (int)ring_smem(tb_stage_bytes(n)));
                        return e;
                    }));
    MVS_CUDA_OK(ctx, cudaFuncSetAttribute(skin_kernel, kSmem, (int)kSkinSmem));
    return MVS_OK;
}

int tc_vjp_buffer(mvs_ctx* ctx, float** dvp, int* ldR) {
    TcState* T = ctx->tc;
    const Workspace& w = ctx->ws;
    const int N = ctx->m.N, ld = tb_dvp_ld(N);
    if (!T->dvp) {                                      // allocated on first use: only mvs_forward_vjp needs it
        float* p = nullptr;
        if (int rc = dev_alloc(ctx, &p, (size_t)2 * w.ldA * ld)) return rc;
        int rc;
        if ((rc = encode_map(ctx, &T->map_q, ctx->m.Qk, (uint64_t)3 * N, kTbRows))) return rc;
        for (int i = 0; i < kTbNumInst; ++i)
            if ((rc = encode_map(ctx, &T->map_d[i], p, (uint64_t)2 * w.ldA, kTcInstances[i], (uint64_t)3 * N, ld))) return rc;
        T->dvp = p;
    }
    *dvp = T->dvp;
    *ldR = ld;
    return MVS_OK;
}

int launch_vertex_bwd_tc(mvs_ctx* ctx, int nstrips, cudaStream_t st) {
    const TcState* T = ctx->tc;
    const Workspace& w = ctx->ws;
    const int nchunks = (3 * ctx->m.N + kTbRows - 1) / kTbRows;
    const int nf = std::min(tc_cols_for(w.B), kTbCols);
    const dim3 grid(nstrips, (w.B + nf - 1) / nf);
    MVS_LAUNCH(ctx, KID_VERTEX_BWD, st, MVS_CUDA_OK(ctx, with_instance<kTbCols>(nf, [&](auto n, int i) {
                   vertex_bwd_tc_kernel<n><<<grid, kTbThreads, ring_smem(tb_stage_bytes(n)), st>>>(T->map_q, T->map_d[i], w.ldA, w.na,
                                                                                              nchunks, w.part, T->err);
                   return cudaSuccess;
               })));
    MVS_CUDA_OK(ctx, cudaGetLastError());
    return MVS_OK;
}

float* tc_poffT(mvs_ctx* ctx) { return ctx->tc->poffT; }

int launch_vertex_fwd_tc(mvs_ctx* ctx, cudaStream_t st, bool need_vposed, bool sdf_setup) {
    TcState* T = ctx->tc;
    Workspace& w = ctx->ws;
    const DevModel& m = ctx->m;
    if (!T->poffT) {                                    // allocated on first use: sparse-regime contexts never need it
        const int rc = dev_alloc(ctx, &T->poffT, (size_t)3 * m.N * w.ldA);
        if (rc) return rc;
    }
    const int nb = w.na_bound > 0 ? w.na_bound : w.B;             // upper bound of the active-frame count
    // each frame's SDF set-up: skin_small_kernel's tail at <= kSkinSetupMax frames, else sdf_setup_kernel after the skinning
    const bool setup_in_skin = sdf_setup && nb <= kSkinSetupMax;
    SdfSetupArgs sd{};
    if (sdf_setup) {
        const int rc = ensure_sdf_setup_ws(ctx, st);
        if (rc) return rc;
        sd = make_sdf_setup_args(ctx);
    }
    const int ntiles = (3 * m.N + kTcRows - 1) / kTcRows;
    const int nf = tc_cols_for(nb);
    dim3 grid(std::min(ctx->sm_count, ntiles), (nb + kTcCols - 1) / kTcCols);   // surplus CTAs exit: the kernel splits the tiles from *na
    MVS_LAUNCH(ctx, KID_VERTEX_FWD_TC, st, MVS_CUDA_OK(ctx, with_instance<kTcCols>(nf, [&](auto n, int i) {
                   return launch_pdl(posedirs_gemm_tc_kernel<n>, grid, dim3(kTcThreads), ring_smem(tc_stage_bytes(n)), st, T->map_p,
                                     T->map_f[i], w.ldA, 3 * m.N, (const int*)w.na, ctx->sm_count, ntiles, T->poffT, T->err);
               })));
    const int nchunks = (m.N + kSkinV - 1) / kSkinV, fgroups = (nb + 31) / 32;
    const SkinArgs sa{T->poffT, m.ST, w.Phi, w.At, w.ldA, m.ell_j, m.ell_w, m.KW, m.N, need_vposed ? w.vposed : nullptr, w.verts, w.bboxp,
                      setup_in_skin ? sd : SdfSetupArgs{}};
    if (nb <= kSkinSmallMax) {                          // straggler tail: lane = vertex, one chunk per CTA
        MVS_LAUNCH(ctx, KID_SKIN, st,
                   MVS_CUDA_OK(ctx, launch_pdl(skin_small_kernel, dim3(nchunks), dim3(kSkinSmallThreads), 0, st, sa, (const int*)w.na)));
    } else {
        // each CTA keeps its 32 frames' transforms in shared memory and walks 1..3 chunks (sized from *na in the kernel)
        dim3 g2(nchunks, fgroups);                      // surplus CTAs exit
        MVS_LAUNCH(ctx, KID_SKIN, st,
                   MVS_CUDA_OK(ctx, launch_pdl(skin_kernel, g2, dim3(kSkinThreads), kSkinSmem, st, sa, (const int*)w.na, 2 * ctx->sm_count)));
    }
    if (sdf_setup && !setup_in_skin)
        MVS_LAUNCH(ctx, KID_SDF_SETUP, st,
                   MVS_CUDA_OK(ctx, launch_pdl(sdf_setup_kernel, dim3((nb + kSetupWarps - 1) / kSetupWarps), dim3(32 * kSetupWarps), 0, st,
                                               sd, (const float*)w.bboxp, (const float*)w.verts, m.N, nchunks, (const int*)w.na)));
    MVS_CUDA_OK(ctx, cudaGetLastError());
    return MVS_OK;
}

int tc_check_error(mvs_ctx* ctx) {          // host-side check after a synchronisation point
    TcState* T = ctx->tc;
    if (!T->poffT) return MVS_OK;                  // no tensor-core kernel has run
    int e = 0;
    MVS_CUDA_OK(ctx, cudaMemcpy(&e, T->err, sizeof(int), cudaMemcpyDeviceToHost));
    if (e) return set_error(ctx, MVS_ERR_CUDA, "tensor-core pipeline: an mbarrier wait of the TMA / wgmma ring timed out (protocol error)");
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
