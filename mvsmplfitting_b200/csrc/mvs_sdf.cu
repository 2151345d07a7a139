// SDF interpenetration term.  Replaces (reference):
//   sdf/sdf/csrc/sdf_cuda_kernel.cu:242-335  brute-force voxel SDF kernel (+ sdf_cuda.cpp:14-28 binding)
//   code/utils/fitting.py:352-393            bounding box, normalisation, grid_sample, squared weighted sum
//
// Three entry points:
//   sdf_grid_launch    the reference's op: phi[B,G,G,G] for normalised vertices (kept for callers that want the
//                      grid; triangles staged through shared memory instead of re-read per voxel)
//   launch_sdf_terms   the term for the batched reference chain (bbox / sample / finalize kernels): phi is never
//                      materialised.  The loss only reads phi at the <= 8 voxels around each vertex, and phi(voxel)
//                      is a pure function of the voxel index, so those voxels are evaluated on the fly while
//                      sampling.  That removes the 128^3 x 4 B = 8.4 MB grid write + gather per frame (2.1 GB per
//                      256-frame closure) and G^3 / (8 N) = 38x of the voxel work, with identical sampled values.
//   launch_sdf_fused   the dense regime's kernel: the same sampling, preceded by conservative geometric tests
//                      (chunk / cell / voxel against the cone and the plane of triangle 0), followed by the adjoint
//                      of the few vertices that see a non-zero value, all in one launch (see sdf_fused_kernel)
//
// Reference quirks reproduced (SURVEY A12): voxel centres use dx = 2/(G-1) while grid_sample assumes 2/G;
// the fitting code passes faces as [1,F,3] so the kernel loops over ONE triangle (sdf_all_faces = 0);
// gradients flow through the sample coordinates and through the bounding-box centre / scale, not through phi.
#include <cstdlib>
#include "mvs_internal.cuh"
// -DMVS_PHASE_DBG (scripts/sdf_phase_times.py): thread 0 of every sdf_fused CTA that runs to the end stamps clock64() at
// entry (0), after pdl_wait (1), after the box fold and its barrier (2), once the cone/plane set-up and the chunk-cull
// verdicts are ready (3), after sampling and its barrier (4) and after the block reduction and adjoint (5).  The intervals
// 1..5 are summed over CTAs into g_sdf_clk[1..5] and maxed into [9..13]; [16] counts the CTAs, [17] sums the CTAs'
// entry->end globaltimer nanoseconds (the cycles/ns ratio gives the SM clock of the run).
#ifdef MVS_PHASE_DBG
namespace mvs {
__device__ unsigned long long g_sdf_clk[32];
__device__ __forceinline__ void sdf_mark(int i) {
    if (threadIdx.x != 0) return;
    __shared__ long long s_clk[6];
    __shared__ unsigned long long s_ns0;
    const long long c = clock64();
    s_clk[i] = c;
    if (i == 0) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(s_ns0));
    if (i == 5) {
        unsigned long long ns;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(ns));
        for (int k = 1; k <= 5; ++k) {
            const unsigned long long d = (unsigned long long)(s_clk[k] - s_clk[k - 1]);
            atomicAdd(&g_sdf_clk[k], d);
            atomicMax(&g_sdf_clk[8 + k], d);
        }
        atomicAdd(&g_sdf_clk[16], 1ull);
        atomicAdd(&g_sdf_clk[17], ns - s_ns0);
        atomicAdd(&g_sdf_clk[18], (unsigned long long)(s_clk[5] - s_clk[0]));
    }
}
}  // namespace mvs
#define SDF_MARK(i) mvs::sdf_mark(i)
#endif
#include "mvs_sdf_dev.cuh"

namespace mvs {

// ---------------------------------------------------------------------------------- the reference op: full grid
constexpr int kSdfThreads = 512;
constexpr int kTriChunk = 256;

__global__ void __launch_bounds__(kSdfThreads)
sdf_grid_kernel(float* __restrict__ phi, const int* __restrict__ faces, const float* __restrict__ verts, int batch,
                int num_faces, int num_verts, int G) {
    __shared__ float tri[kTriChunk * 9];
    const long long tid = (long long)blockIdx.x * kSdfThreads + threadIdx.x;
    const long long G3 = (long long)G * G * G;
    // a block never straddles two batch items when G^3 % 512 == 0 (the reference case); otherwise fall back
    // to per-thread batch ids with the block's first item used for the staged triangles
    const int bn0 = (int)(((long long)blockIdx.x * kSdfThreads) / G3);
    const int i = (int)(tid % G), j = (int)((tid / G) % G), k = (int)((tid / ((long long)G * G)) % G);
    const int bn = (int)(tid / G3);
    float c[3];
    voxel_centre(i, j, k, G, c);
    int hits = 0;
    float min_d = 1000.f;
    const bool uniform = (((long long)(blockIdx.x + 1) * kSdfThreads - 1) / G3) == bn0;
    for (int f0 = 0; f0 < num_faces; f0 += kTriChunk) {
        const int nf = min(kTriChunk, num_faces - f0);
        __syncthreads();
        for (int e = threadIdx.x; e < nf * 9; e += kSdfThreads) {
            const int f = e / 9, r = e % 9;
            tri[e] = verts[((size_t)bn0 * num_verts + faces[3 * (f0 + f) + r / 3]) * 3 + r % 3];
        }
        __syncthreads();
        if (bn < batch) {
            for (int f = 0; f < nf; ++f) {
                float a[3], b[3], cc[3];
                if (uniform) {
#pragma unroll
                    for (int r = 0; r < 3; ++r) { a[r] = tri[9 * f + r]; b[r] = tri[9 * f + 3 + r]; cc[r] = tri[9 * f + 6 + r]; }
                } else {
                    const float* vb = verts + (size_t)bn * num_verts * 3;
#pragma unroll
                    for (int r = 0; r < 3; ++r) {
                        a[r] = vb[3 * faces[3 * (f0 + f)] + r]; b[r] = vb[3 * faces[3 * (f0 + f) + 1] + r];
                        cc[r] = vb[3 * faces[3 * (f0 + f) + 2] + r];
                    }
                }
                const float dd = triangle_distance(c, a, b, cc);
                if (dd < min_d) min_d = dd;
                if (ray_hits(c, a, b, cc)) ++hits;
            }
        }
    }
    if (bn < batch) phi[tid] = (hits % 2 == 0) ? 0.f : min_d;        // sdf_cuda_kernel.cu:291-299
}

int sdf_grid_launch(mvs_ctx* ctx, float* phi, const int* faces, int num_faces, const float* verts, int batch,
                    int n_verts, int G, cudaStream_t st) {
    const long long total = (long long)batch * G * G * G;
    const long long blocks = total / kSdfThreads;                    // integer division as in the reference (:316-317)
    if (blocks > 0) {
        MVS_LAUNCH(ctx, KID_SDF_GRID, st,
                   sdf_grid_kernel<<<(unsigned)blocks, kSdfThreads, 0, st>>>(phi, faces, verts, batch, num_faces, n_verts, G));
    }
    MVS_CUDA_OK(ctx, cudaGetLastError());
    return MVS_OK;
}

// ---------------------------------------------------------------------------------- fused term for the closure
constexpr int kBoxThreads = 256;
__global__ void __launch_bounds__(kBoxThreads)
sdf_bbox_kernel(const float* __restrict__ verts, const float* __restrict__ x, const int* __restrict__ fidx,
                const int* __restrict__ na_ptr, int N, FrameBox* __restrict__ box) {
    const int slot = blockIdx.x;
    if (slot >= *na_ptr) return;
    const int b = fidx[slot], t = threadIdx.x;
    const float* tr = x + (size_t)b * kParams + kOffTransl;
    const float* vf = verts + (size_t)slot * N * 3;
    float lo[3] = {3e38f, 3e38f, 3e38f}, hi[3] = {-3e38f, -3e38f, -3e38f};
    int ilo[3] = {0, 0, 0}, ihi[3] = {0, 0, 0};
    for (int n = t; n < N; n += kBoxThreads) {
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const float v = vf[3 * n + c] + tr[c];                    // vertices += transl (body_models_scale.py:403)
            if (v < lo[c]) { lo[c] = v; ilo[c] = n; }
            if (v > hi[c]) { hi[c] = v; ihi[c] = n; }
        }
    }
    __shared__ float s_lo[3][kBoxThreads], s_hi[3][kBoxThreads];
    __shared__ int s_ilo[3][kBoxThreads], s_ihi[3][kBoxThreads];
#pragma unroll
    for (int c = 0; c < 3; ++c) { s_lo[c][t] = lo[c]; s_hi[c][t] = hi[c]; s_ilo[c][t] = ilo[c]; s_ihi[c][t] = ihi[c]; }
    __syncthreads();
    for (int o = kBoxThreads / 2; o > 0; o >>= 1) {
        if (t < o) {
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                // ties -> lowest vertex index (first occurrence, like torch.min / torch.max on CPU)
                const float l2 = s_lo[c][t + o]; const int il2 = s_ilo[c][t + o];
                if (l2 < s_lo[c][t] || (l2 == s_lo[c][t] && il2 < s_ilo[c][t])) { s_lo[c][t] = l2; s_ilo[c][t] = il2; }
                const float h2 = s_hi[c][t + o]; const int ih2 = s_ihi[c][t + o];
                if (h2 > s_hi[c][t] || (h2 == s_hi[c][t] && ih2 < s_ihi[c][t])) { s_hi[c][t] = h2; s_ihi[c][t] = ih2; }
            }
        }
        __syncthreads();
    }
    if (t == 0) {
        FrameBox fb;
        float ext = -1.f;
        fb.cmax = 0;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            fb.centre[c] = (s_lo[c][0] + s_hi[c][0]) / 2.f;          // boxes.mean(dim=1)  (fitting.py:357)
            fb.ilo[c] = s_ilo[c][0]; fb.ihi[c] = s_ihi[c][0];
            const float e = s_hi[c][0] - s_lo[c][0];
            if (e > ext) { ext = e; fb.cmax = c; }
        }
        fb.scale = 0.6f * ext;                                        // (1 + 0.2) * 0.5 * max extent (fitting.py:358-359)
        fb.pad = 0.f;
        box[slot] = fb;
    }
}

// phi at voxel (i,j,k) for this frame; tri0 = the normalised triangle(s)
__device__ float voxel_phi_frame(int i, int j, int k, int G, int num_faces, const int* __restrict__ faces,
                                 const float* __restrict__ vf, const float* tr, const FrameBox& fb, const float* tri0) {
    float c[3];
    voxel_centre(i, j, k, G, c);
    if (num_faces == 1) {
        if (!ray_hits(c, tri0, tri0 + 3, tri0 + 6)) return 0.f;
        return triangle_distance(c, tri0, tri0 + 3, tri0 + 6);
    }
    int hits = 0;
    float min_d = 1000.f;
    for (int f = 0; f < num_faces; ++f) {
        float p[9];
#pragma unroll
        for (int r = 0; r < 9; ++r)
            p[r] = ((vf[3 * faces[3 * f + r / 3] + r % 3] + tr[r % 3]) - fb.centre[r % 3]) / fb.scale;
        const float dd = triangle_distance(c, p, p + 3, p + 6);
        if (dd < min_d) min_d = dd;
        if (ray_hits(c, p, p + 3, p + 6)) ++hits;
    }
    return (hits % 2 == 0) ? 0.f : min_d;
}

constexpr int kSampleThreads = 128;
// per vertex: value = trilinear sample of phi at the vertex' normalised position, gcoord = d value / d local
__global__ void __launch_bounds__(kSampleThreads)
sdf_sample_kernel(const float* __restrict__ verts, const float* __restrict__ x, const int* __restrict__ fidx,
                  const int* __restrict__ na_ptr, int N, const int* __restrict__ faces, int num_faces, int G,
                  const FrameBox* __restrict__ box, float* __restrict__ gcoord, float* __restrict__ part, int nblk) {
    const int slot = blockIdx.y;
    if (slot >= *na_ptr) return;
    const int b = fidx[slot], t = threadIdx.x;
    const int n = blockIdx.x * kSampleThreads + t;
    const FrameBox fb = box[slot];
    const float* vf = verts + (size_t)slot * N * 3;
    const float tr[3] = {x[(size_t)b * kParams + kOffTransl], x[(size_t)b * kParams + kOffTransl + 1],
                         x[(size_t)b * kParams + kOffTransl + 2]};
    __shared__ float tri0[9];
    if (t < 9) tri0[t] = ((vf[3 * faces[t / 3] + t % 3] + tr[t % 3]) - fb.centre[t % 3]) / fb.scale;   // fitting.py:362-363
    __syncthreads();
    float val = 0.f, gc[3] = {0.f, 0.f, 0.f}, gdotl = 0.f;
    if (n < N) {
        float loc[3], ix[3], w1[3];
        int i0[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            loc[c] = ((vf[3 * n + c] + tr[c]) - fb.centre[c]) / fb.scale;                              // fitting.py:376-377
            ix[c] = ((loc[c] + 1.f) * G - 1.f) / 2.f;                   // grid_sample, align_corners=False
            const float fl = floorf(ix[c]);
            i0[c] = (int)fl;
            w1[c] = ix[c] - fl;
        }
        float dix[3] = {0.f, 0.f, 0.f};
#pragma unroll
        for (int corner = 0; corner < 8; ++corner) {
            const int ox = corner & 1, oy = (corner >> 1) & 1, oz = corner >> 2;
            const int ii = i0[0] + ox, jj = i0[1] + oy, kk = i0[2] + oz;
            if (ii < 0 || ii >= G || jj < 0 || jj >= G || kk < 0 || kk >= G) continue;   // zeros padding
            const float p = voxel_phi_frame(ii, jj, kk, G, num_faces, faces, vf, tr, fb, tri0);
            if (p == 0.f) continue;
            const float wx = ox ? w1[0] : 1.f - w1[0], wy = oy ? w1[1] : 1.f - w1[1], wz = oz ? w1[2] : 1.f - w1[2];
            val += p * wx * wy * wz;
            dix[0] += p * (ox ? 1.f : -1.f) * wy * wz;
            dix[1] += p * wx * (oy ? 1.f : -1.f) * wz;
            dix[2] += p * wx * wy * (oz ? 1.f : -1.f);
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) { gc[c] = dix[c] * (0.5f * G); gdotl += gc[c] * loc[c]; }
        float* go = gcoord + ((size_t)slot * N + n) * 3;
        go[0] = gc[0]; go[1] = gc[1]; go[2] = gc[2];
    }
    // block partials: [val, sum gcoord (3), sum gcoord . local]
    __shared__ float red[5][kSampleThreads];
    red[0][t] = val; red[1][t] = gc[0]; red[2][t] = gc[1]; red[3][t] = gc[2]; red[4][t] = gdotl;
    __syncthreads();
    for (int o = kSampleThreads / 2; o > 0; o >>= 1) {
        if (t < o) {
#pragma unroll
            for (int q = 0; q < 5; ++q) red[q][t] += red[q][t + o];
        }
        __syncthreads();
    }
    if (t < 5) part[((size_t)slot * nblk + blockIdx.x) * 5 + t] = red[t][0];
}

// d loss / d vertex of the penetration term (dense), and the loss itself
__global__ void __launch_bounds__(kSampleThreads)
sdf_finalize_kernel(const int* __restrict__ na_ptr, int N, const FrameBox* __restrict__ box,
                    const float* __restrict__ gcoord, const float* __restrict__ part, int nblk, float coll_w,
                    float* __restrict__ dv, int dv_stride, int dv_offset, float* __restrict__ pen_loss) {
    const int slot = blockIdx.y;
    if (slot >= *na_ptr) return;
    const int t = threadIdx.x, n = blockIdx.x * kSampleThreads + t;
    __shared__ float tot[5];
    if (t < 5) {
        float a = 0.f;
        for (int k = 0; k < nblk; ++k) a += part[((size_t)slot * nblk + k) * 5 + t];
        tot[t] = a;
    }
    __syncthreads();
    const FrameBox fb = box[slot];
    const float wsum = coll_w * tot[0];                               // coll_loss_weight * cur_loss.sum() / 1
    if (blockIdx.x == 0 && t == 0) pen_loss[slot] = wsum * wsum;      // fitting.py:391-392
    if (n >= N) return;
    const float cg = 2.f * wsum * coll_w;                             // d pen / d (sum of samples)
    const float inv_s = 1.f / fb.scale;
    const float* g = gcoord + ((size_t)slot * N + n) * 3;
    float d[3] = {cg * g[0] * inv_s, cg * g[1] * inv_s, cg * g[2] * inv_s};
    // through the box centre (mean of min and max vertex) and the scale (0.6 x largest extent)
    const float dscale = -cg * tot[4] * inv_s;                        // local = (v - c)/s  ->  d local/d s = -local/s
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float dcentre = -cg * tot[1 + c] * inv_s;
        if (n == fb.ilo[c]) d[c] += 0.5f * dcentre;
        if (n == fb.ihi[c]) d[c] += 0.5f * dcentre;
        if (c == fb.cmax) {
            if (n == fb.ihi[c]) d[c] += 0.6f * dscale;
            if (n == fb.ilo[c]) d[c] -= 0.6f * dscale;
        }
    }
    float* o = dv + ((size_t)slot * dv_stride + dv_offset + n) * 3;
    o[0] = d[0]; o[1] = d[1]; o[2] = d[2];
}

// ------------------------------------------------------------------------------------------------ all-faces bins (N3)
// One CTA per active frame builds the frame's candidate structures of mvs_sdf_bins.cuh: triangle corners in box coordinates,
// the cell lists (counting sort over kBinCells in shared memory) and the ray-bin lists (the same over kBinRays).  The order of
// the triangles inside a list is whatever the atomics produce: minimum and parity do not depend on it.
constexpr int kBinsThreads = 1024;
constexpr size_t kBinsSmem = (size_t)kBinCells * sizeof(int) + 64 * sizeof(float);

struct SdfBinsArgs {
    const float* verts; const float* slot_tr; const SdfFrameSetup* setup; const int* faces; int N, F;
    float* tri; int* cell_ptr; unsigned short* cell_idx; int* ray_ptr; unsigned short* ray_idx; float* meta;
};

// exclusive scan of hist[0 .. n) in place (n a multiple of 1024, <= kBinCells), all kBinsThreads threads; returns the total
__device__ __forceinline__ int block_exclusive_scan(int* hist, int n, int* wtot) {
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const int per_warp = n / 32;                               // 32 warps
    const int base = warp * per_warp;
    int carry = 0;
    for (int i = 0; i < per_warp; i += 32) {
        const int v = hist[base + i + lane];
        int incl = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int u = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += u; }
        hist[base + i + lane] = carry + incl - v;
        carry += __shfl_sync(0xffffffffu, incl, 31);
    }
    if (lane == 0) wtot[warp] = carry;
    __syncthreads();
    if (warp == 0) {
        const int v = wtot[lane];
        int incl = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int u = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += u; }
        wtot[lane] = incl - v;
        if (lane == 31) wtot[32] = incl;
    }
    __syncthreads();
    const int off = wtot[warp];
    for (int i = 0; i < per_warp; i += 32) hist[base + i + lane] += off;
    __syncthreads();
    return wtot[32];
}

__global__ void __launch_bounds__(kBinsThreads, 1)
sdf_bins_kernel(SdfBinsArgs a, const int* __restrict__ na_ptr) {
    pdl_wait();
    extern __shared__ __align__(16) unsigned char bins_smem[];
    int* hist = reinterpret_cast<int*>(bins_smem);
    float* sf = reinterpret_cast<float*>(bins_smem + (size_t)kBinCells * sizeof(int));      // 64 floats of scratch
    __shared__ int wtot[33];
    const int slot = blockIdx.x;
    if (slot >= *na_ptr) return;
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const float* vf = a.verts + (size_t)slot * a.N * 3;
    const float tr[3] = {a.slot_tr[4 * slot], a.slot_tr[4 * slot + 1], a.slot_tr[4 * slot + 2]};
    // ---- frame box: the set-up sdf_setup_kernel (or skin_small_kernel) computed for this frame (the box sdf_fused uses)
    const FrameBox& fbx = a.setup[slot].fb;
    const float centre[3] = {fbx.centre[0], fbx.centre[1], fbx.centre[2]}, scale = fbx.scale;
    float* wb = reinterpret_cast<float*>(hist);                // [32][4] scratch of the projected-box fold
    // ---- triangle corners in box coordinates (the brute force's operands, same expression) + bounding box of the projected mesh
    float* tri = a.tri + (size_t)slot * a.F * 9;
    float smn[2] = {3e38f, 3e38f}, smx[2] = {-3e38f, -3e38f};
    for (int f = t; f < a.F; f += kBinsThreads) {
        float p[9];
#pragma unroll
        for (int r = 0; r < 9; ++r) p[r] = ((vf[3 * a.faces[3 * f + r / 3] + r % 3] + tr[r % 3]) - centre[r % 3]) / scale;
#pragma unroll
        for (int r = 0; r < 9; ++r) tri[9 * f + r] = p[r];
        float bmn[2], bmx[2];
        tri_proj_box(p, bmn, bmx);
#pragma unroll
        for (int q = 0; q < 2; ++q) { smn[q] = fminf(smn[q], bmn[q]); smx[q] = fmaxf(smx[q], bmx[q]); }
    }
#pragma unroll
    for (int q = 0; q < 2; ++q)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            smn[q] = fminf(smn[q], __shfl_xor_sync(0xffffffffu, smn[q], o));
            smx[q] = fmaxf(smx[q], __shfl_xor_sync(0xffffffffu, smx[q], o));
        }
    if (lane == 0) { wb[warp * 4] = smn[0]; wb[warp * 4 + 1] = smn[1]; wb[warp * 4 + 2] = smx[0]; wb[warp * 4 + 3] = smx[1]; }
    __syncthreads();
    if (t == 0) {
        float mn[2] = {wb[0], wb[1]}, mx[2] = {wb[2], wb[3]};
        for (int w = 1; w < kBinsThreads / 32; ++w) {
            mn[0] = fminf(mn[0], wb[w * 4]); mn[1] = fminf(mn[1], wb[w * 4 + 1]);
            mx[0] = fmaxf(mx[0], wb[w * 4 + 2]); mx[1] = fmaxf(mx[1], wb[w * 4 + 3]);
        }
        ray_bin_frame(mn, mx, &sf[0], &sf[2]);
    }
    __syncthreads();
    const float s_lo[2] = {sf[0], sf[1]}, s_scale[2] = {sf[2], sf[3]};
    __syncthreads();
    // ---- cell lists
    for (int i = t; i < kBinCells; i += kBinsThreads) hist[i] = 0;
    __syncthreads();
    for (int f = t; f < a.F; f += kBinsThreads) {
        int cl[3], ch[3];
        tri_cell_range(tri + 9 * f, cl, ch);
        for (int x = cl[0]; x <= ch[0]; ++x) for (int y = cl[1]; y <= ch[1]; ++y) for (int z = cl[2]; z <= ch[2]; ++z)
            atomicAdd(&hist[(x * kBinC + y) * kBinC + z], 1);
    }
    __syncthreads();
    const int tot_d = block_exclusive_scan(hist, kBinCells, wtot);
    int* cptr = a.cell_ptr + (size_t)slot * (kBinCells + 1);
    for (int i = t; i < kBinCells; i += kBinsThreads) cptr[i] = hist[i];
    if (t == 0) cptr[kBinCells] = tot_d;
    __syncthreads();
    if (tot_d <= kBinCapD) {
        unsigned short* cidx = a.cell_idx + (size_t)slot * kBinCapD;
        for (int f = t; f < a.F; f += kBinsThreads) {
            int cl[3], ch[3];
            tri_cell_range(tri + 9 * f, cl, ch);
            for (int x = cl[0]; x <= ch[0]; ++x) for (int y = cl[1]; y <= ch[1]; ++y) for (int z = cl[2]; z <= ch[2]; ++z)
                cidx[atomicAdd(&hist[(x * kBinC + y) * kBinC + z], 1)] = (unsigned short)f;
        }
    }
    __syncthreads();
    // ---- ray-bin lists
    for (int i = t; i < kBinRays; i += kBinsThreads) hist[i] = 0;
    __syncthreads();
    for (int f = t; f < a.F; f += kBinsThreads) {
        float bmn[2], bmx[2];
        int rl[2], rh[2];
        tri_proj_box(tri + 9 * f, bmn, bmx);
        tri_ray_range(bmn, bmx, s_lo, s_scale, rl, rh);
        for (int x = rl[0]; x <= rh[0]; ++x) for (int y = rl[1]; y <= rh[1]; ++y) atomicAdd(&hist[x * kBinR + y], 1);
    }
    __syncthreads();
    const int tot_r = block_exclusive_scan(hist, kBinRays, wtot);
    int* rptr = a.ray_ptr + (size_t)slot * (kBinRays + 1);
    for (int i = t; i < kBinRays; i += kBinsThreads) rptr[i] = hist[i];
    if (t == 0) rptr[kBinRays] = tot_r;
    __syncthreads();
    if (tot_r <= kBinCapR) {
        unsigned short* ridx = a.ray_idx + (size_t)slot * kBinCapR;
        for (int f = t; f < a.F; f += kBinsThreads) {
            float bmn[2], bmx[2];
            int rl[2], rh[2];
            tri_proj_box(tri + 9 * f, bmn, bmx);
            tri_ray_range(bmn, bmx, s_lo, s_scale, rl, rh);
            for (int x = rl[0]; x <= rh[0]; ++x) for (int y = rl[1]; y <= rh[1]; ++y)
                ridx[atomicAdd(&hist[x * kBinR + y], 1)] = (unsigned short)f;
        }
    }
    if (t == 0) {
        float* mt = a.meta + 8 * (size_t)slot;
        mt[0] = s_lo[0]; mt[1] = s_lo[1]; mt[2] = s_scale[0]; mt[3] = s_scale[1];
        mt[4] = (tot_d > kBinCapD || tot_r > kBinCapR) ? 1.f : 0.f;      // overflow: sdf_fused falls back to the brute force for this frame
        mt[5] = (float)tot_d; mt[6] = (float)tot_r; mt[7] = 0.f;
    }
}

static int ensure_sdf_bins_ws(mvs_ctx* ctx) {
    Workspace& w = ctx->ws;
    if (w.bins_tri) return MVS_OK;
    if (ctx->m.F > 65535) return set_error(ctx, MVS_ERR_UNSUPPORTED, "accelerated all-faces SDF: more than 65535 faces");
    const size_t B = (size_t)w.B;
    int rc;
    if ((rc = dev_alloc(ctx, &w.bins_tri, B * ctx->m.F * 9))) return rc;
    if ((rc = dev_alloc(ctx, &w.bins_cell_ptr, B * (kBinCells + 1)))) return rc;
    if ((rc = dev_alloc(ctx, &w.bins_cell_idx, B * kBinCapD))) return rc;
    if ((rc = dev_alloc(ctx, &w.bins_ray_ptr, B * (kBinRays + 1)))) return rc;
    if ((rc = dev_alloc(ctx, &w.bins_ray_idx, B * kBinCapR))) return rc;
    if ((rc = dev_alloc(ctx, &w.bins_meta, B * 8))) return rc;
    return MVS_OK;
}

int sdf_set_attributes(mvs_ctx* ctx) {
    MVS_CUDA_OK(ctx, cudaFuncSetAttribute(sdf_bins_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kBinsSmem));
    return MVS_OK;
}

int ensure_sdf_fused_ws(mvs_ctx* ctx) {
    Workspace& w = ctx->ws;
    const int B = w.B, N = ctx->m.N;
    const int nblocks = (N + kSdfFThreads - 1) / kSdfFThreads;
    int rc;
    if (!w.sdf_gcoord && (rc = dev_alloc(ctx, &w.sdf_gcoord, (size_t)B * N * 3))) return rc;
    if (!w.sdf_parts5) {
        if ((rc = dev_alloc(ctx, &w.sdf_parts5, (size_t)B * nblocks * 5))) return rc;
        if ((rc = dev_alloc(ctx, &w.sdf_part, (size_t)B * nblocks * kPartFloats))) return rc;
        if ((rc = dev_alloc(ctx, &w.sdf_pflag, (size_t)B * nblocks))) return rc;
    }
    if (!w.sdf_box && (rc = dev_alloc(ctx, &w.sdf_box, (size_t)B))) return rc;
    return MVS_OK;
}

int ensure_sdf_setup_ws(mvs_ctx* ctx, cudaStream_t st) {
    Workspace& w = ctx->ws;
    int rc;
    if ((rc = ensure_sdf_fused_ws(ctx))) return rc;
    if (!w.sdf_setup) {
        if ((rc = dev_alloc(ctx, &w.sdf_setup, (size_t)w.B))) return rc;
        if ((rc = dev_alloc(ctx, &w.sdf_arrive, (size_t)w.B))) return rc;
        MVS_CUDA_OK(ctx, cudaMemsetAsync(w.sdf_arrive, 0, (size_t)w.B * sizeof(int), st));
    }
    return MVS_OK;
}

SdfSetupArgs make_sdf_setup_args(mvs_ctx* ctx) {
    Workspace& w = ctx->ws;
    const DevModel& m = ctx->m;
    SdfSetupArgs a;
    a.rec = w.sdf_setup; a.boxout = w.sdf_box;
    a.arrive = w.sdf_arrive; a.slot_tr = w.slot_tr;
    a.f0 = m.tri0[0]; a.f1 = m.tri0[1]; a.f2 = m.tri0[2]; a.G = ctx->loss.sdf_grid;
    a.cull = ctx->loss.sdf_all_faces ? (m.F == 1) : 1;        // the cone/plane tests hold for a single face (num_faces == 1)
    return a;
}

SdfFusedArgs make_sdf_fused_args(mvs_ctx* ctx) {
    Workspace& w = ctx->ws;
    const DevModel& m = ctx->m;
    const LossParams& lp = ctx->loss;
    SdfFusedArgs a;
    a.verts = w.verts; a.poffT = tc_poffT(ctx); a.Phi = w.Phi; a.ST = m.ST; a.slot_tr = w.slot_tr;
    a.N = m.N; a.nbox = (m.N + 63) / 64; a.setup = w.sdf_setup; a.faces = m.faces;
    a.num_faces = lp.sdf_all_faces ? m.F : 1; a.G = lp.sdf_grid;
    a.At = w.At; a.ldA = w.ldA; a.ell_j = m.ell_j; a.ell_w = m.ell_w; a.KW = m.KW; a.Wd = m.Wd; a.Qk = m.Qk;
    a.parts5 = w.sdf_parts5; a.part = w.sdf_part; a.pflag = w.sdf_pflag;
    a.gcoord = w.sdf_gcoord;
    // sdf_all_faces: 0 as written (triangle 0), 1 all faces over candidate lists (accelerated), 2 all faces by brute force
    const bool binned = lp.sdf_all_faces == 1 && w.bins_tri != nullptr;
    a.bins.tri = binned ? w.bins_tri : nullptr; a.bins.cell_ptr = w.bins_cell_ptr; a.bins.cell_idx = w.bins_cell_idx;
    a.bins.ray_ptr = w.bins_ray_ptr; a.bins.ray_idx = w.bins_ray_idx; a.bins.meta = w.bins_meta; a.bins.F = m.F;
    {   // A/B knob (experiments only): MVS_SDF_BLOCK_SKIP=0 runs every CTA as if each of its blocks had a live chunk
        static const int block_skip = getenv("MVS_SDF_BLOCK_SKIP") ? atoi(getenv("MVS_SDF_BLOCK_SKIP")) : 1;
        a.block_skip = block_skip != 0;
    }
    return a;
}

int launch_sdf_fused(mvs_ctx* ctx, cudaStream_t st) {
    Workspace& w = ctx->ws;
    const DevModel& m = ctx->m;
    const int B = w.B, N = m.N;
    const int nb = w.na_bound > 0 ? w.na_bound : B;    // host-side upper bound of the active-frame count
    const int nblocks = (N + kSdfFThreads - 1) / kSdfFThreads;
    // 256-vertex blocks per CTA (1 at the tail, 2 in the bulk; see sdf_passes_for)
    int passes = sdf_passes_for(nb, nblocks, 3 * ctx->sm_count);
    {   // tuning knob (experiments only): MVS_SDF_PASSES=n forces n blocks per CTA
        static const int forced = getenv("MVS_SDF_PASSES") ? atoi(getenv("MVS_SDF_PASSES")) : 0;
        if (forced >= 1 && forced <= kSdfMaxPasses) passes = forced;
    }
    const int nparts = (nblocks + passes - 1) / passes;
    int rc = ensure_sdf_fused_ws(ctx);
    if (rc) return rc;
    dim3 g(nparts, nb);
    if (ctx->loss.sdf_all_faces == 1) {                  // accelerated all-faces mode: this round's candidate lists first
        if ((rc = ensure_sdf_bins_ws(ctx))) return rc;
        SdfBinsArgs ba;
        ba.verts = w.verts; ba.slot_tr = w.slot_tr; ba.setup = w.sdf_setup; ba.faces = m.faces;
        ba.N = N; ba.F = m.F;
        ba.tri = w.bins_tri; ba.cell_ptr = w.bins_cell_ptr; ba.cell_idx = w.bins_cell_idx; ba.ray_ptr = w.bins_ray_ptr;
        ba.ray_idx = w.bins_ray_idx; ba.meta = w.bins_meta;
        MVS_LAUNCH(ctx, KID_SDF_BBOX, st,
                   MVS_CUDA_OK(ctx, launch_pdl(sdf_bins_kernel, dim3(nb), dim3(kBinsThreads), kBinsSmem, st, ba, (const int*)w.na)));
    }
    const SdfFusedArgs sa = make_sdf_fused_args(ctx);
    if (ctx->loss.sdf_all_faces)
        MVS_LAUNCH(ctx, KID_SDF_FRAME, st,
                   MVS_CUDA_OK(ctx, launch_pdl(sdf_fused_kernel<true>, g, dim3(kSdfFThreads), 0, st, sa, (const int*)w.na, passes)));
    else
        MVS_LAUNCH(ctx, KID_SDF_FRAME, st,
                   MVS_CUDA_OK(ctx, launch_pdl(sdf_fused_kernel<false>, g, dim3(kSdfFThreads), 0, st, sa, (const int*)w.na, passes)));
    MVS_CUDA_OK(ctx, cudaGetLastError());
    return MVS_OK;
}

int launch_sdf_terms(mvs_ctx* ctx, const float* x_dev, cudaStream_t st) {
    Workspace& w = ctx->ws;
    const DevModel& m = ctx->m;
    const LossParams& lp = ctx->loss;
    const int B = w.B, N = m.N;
    const int nblk = (N + kSampleThreads - 1) / kSampleThreads;
    if (!w.sdf_frame) {
        int rc;
        if ((rc = dev_alloc(ctx, &w.sdf_frame, (size_t)B))) return rc;
        if (!w.sdf_gcoord && (rc = dev_alloc(ctx, &w.sdf_gcoord, (size_t)B * N * 3))) return rc;
        if ((rc = dev_alloc(ctx, &w.sdf_valpart, (size_t)B * nblk * 5))) return rc;
    }
    FrameBox* box = w.sdf_frame;
    MVS_LAUNCH(ctx, KID_SDF_BBOX, st, sdf_bbox_kernel<<<B, kBoxThreads, 0, st>>>(w.verts, x_dev, w.fidx, w.na, N, box));
    dim3 g(nblk, B);
    MVS_LAUNCH(ctx, KID_SDF_SAMPLE, st,
               sdf_sample_kernel<<<g, kSampleThreads, 0, st>>>(w.verts, x_dev, w.fidx, w.na, N, m.faces,
                                                               lp.sdf_all_faces ? m.F : 1, lp.sdf_grid, box, w.sdf_gcoord,
                                                               w.sdf_valpart, nblk));
    MVS_LAUNCH(ctx, KID_SDF_FINALIZE, st,
               sdf_finalize_kernel<<<g, kSampleThreads, 0, st>>>(w.na, N, box, w.sdf_gcoord, w.sdf_valpart, nblk,
                                                                 lp.coll_loss_weight, w.dv, m.nsup + N, m.nsup, w.pen_loss));
    MVS_CUDA_OK(ctx, cudaGetLastError());
    return MVS_OK;
}

}  // namespace mvs

// Testing aid, not part of the ABI (tests/test_gpu_sdf_setup.py): copies the dense-regime SDF state of the last round to host
// buffers (null pointers are skipped): the chunk boxes [B][nbox][12], the slot translations [B][4], the FrameBox of every
// slot as frame_step reads it [B][12 words], the per-block sums [B][nblocks][5] and flags [B][nblocks], and the arrival
// counters [B].  Synchronises the device first.
extern "C" int mvs_debug_sdf_state(mvs_ctx* ctx, float* bboxp, float* slot_tr, void* box, float* parts5, int* pflag, int* arrive) {
    const mvs::Workspace& w = ctx->ws;
    const size_t B = (size_t)w.B, N = (size_t)ctx->m.N, nbox = (N + 63) / 64, nblocks = (N + mvs::kSdfFThreads - 1) / mvs::kSdfFThreads;
    if (cudaDeviceSynchronize() != cudaSuccess) return -1;
    if (!w.sdf_setup || !w.sdf_box || !w.sdf_parts5) return -2;
    struct { void* dst; const void* src; size_t bytes; } cp[] = {
        {bboxp, w.bboxp, B * nbox * 12 * sizeof(float)}, {slot_tr, w.slot_tr, B * 4 * sizeof(float)},
        {box, w.sdf_box, B * sizeof(mvs::FrameBox)}, {parts5, w.sdf_parts5, B * nblocks * 5 * sizeof(float)},
        {pflag, w.sdf_pflag, B * nblocks * sizeof(int)}, {arrive, w.sdf_arrive, B * sizeof(int)}};
    for (auto& c : cp)
        if (c.dst && cudaMemcpy(c.dst, c.src, c.bytes, cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
    return 0;
}

// Testing aid, not part of the ABI (tests/test_gpu_sdf_setup_kernel.py): copies the SdfFrameSetup record of every slot
// [B][208 B] as the last dense round left it.  Synchronises the device first.
extern "C" int mvs_debug_sdf_setup(mvs_ctx* ctx, void* rec) {
    const mvs::Workspace& w = ctx->ws;
    if (cudaDeviceSynchronize() != cudaSuccess) return -1;
    if (!w.sdf_setup) return -2;
    return cudaMemcpy(rec, w.sdf_setup, (size_t)w.B * sizeof(mvs::SdfFrameSetup), cudaMemcpyDeviceToHost) == cudaSuccess ? 0 : -1;
}

// Testing aid, not part of the ABI (tests/test_gpu_sdf_block_mask.py): copies sdf_fused's per-block adjoint partials
// [B][nblocks][kPartFloats] as the last dense round left them (only the rows of flagged blocks are written each round).
// part == nullptr: returns kPartFloats.  Synchronises the device first.
extern "C" int mvs_debug_sdf_part(mvs_ctx* ctx, float* part) {
    const mvs::Workspace& w = ctx->ws;
    if (!part) return mvs::kPartFloats;
    const size_t B = (size_t)w.B, nblocks = ((size_t)ctx->m.N + mvs::kSdfFThreads - 1) / mvs::kSdfFThreads;
    if (cudaDeviceSynchronize() != cudaSuccess) return -1;
    if (!w.sdf_part) return -2;
    return cudaMemcpy(part, w.sdf_part, B * nblocks * mvs::kPartFloats * sizeof(float), cudaMemcpyDeviceToHost) == cudaSuccess ? 0 : -1;
}

#ifdef MVS_PHASE_DBG
extern "C" int mvs_debug_sdf_clocks(unsigned long long* out, int n, int reset) {   // debug builds only; not part of the ABI
    unsigned long long h[32];
    if (cudaMemcpyFromSymbol(h, mvs::g_sdf_clk, sizeof(h)) != cudaSuccess) return -1;
    for (int i = 0; i < n && i < 32; ++i) out[i] = h[i];
    if (reset) {
        for (int i = 0; i < 32; ++i) h[i] = 0;
        if (cudaMemcpyToSymbol(mvs::g_sdf_clk, h, sizeof(h)) != cudaSuccess) return -1;
    }
    return 0;
}
#endif
