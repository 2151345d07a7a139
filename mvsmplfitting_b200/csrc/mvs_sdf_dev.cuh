// Device side of the dense regime's SDF term (mvs_sdf.cu): the reference's geometric primitives and sdf_fused_kernel, the
// fused sampling + sparse adjoint.
#pragma once
#include "mvs_internal.cuh"
#include "mvs_tc_dev.cuh"
#include "mvs_sdf_geom.cuh"
#include "mvs_sdf_bins.cuh"

// A translation unit may define SDF_MARK(i) before including this file (clock instrumentation of sdf_fused_kernel, see
// scripts/sdf_phase_times.py); default: nothing.
#ifndef SDF_MARK
#define SDF_MARK(i) do {} while (0)
#endif

namespace mvs {

// ---------------------------------------------------------------------------------- dense regime, v4: fused adjoint
// sdf_fused_kernel: P CTAs per frame, 1 to kSdfMaxPasses blocks of 256 vertices each.  Per CTA: load the frame's set-up record
// (box, triangle 0, cone / plane, chunk-cull verdicts; written once per frame by sdf_setup_kernel or skin_small_kernel), sample phi at the <= 8 voxels around each vertex, compact the vertices with a non-zero sample gradient
// (deterministic order: warp, pass, lane) and -- because with the as-written semantics that list holds a handful of
// vertices -- run the adjoint of the vertex stage for exactly those vertices right here:
//     d v_posed = T_3x3^T g,   dA_j += W[n,j] [g (x) v_posed | g],   dPhi += d v_posed . Qk[rows of n]
// with g = d value / d local (UNIT scale; the frame factor cg/scale is linear and applied by frame_step once the
// frame's total is known).
constexpr int kSdfFThreads = 256;
constexpr int kSdfFChunk = 128;                              // list entries per adjoint pass

// device-side entry of the candidate-list evaluation: kept out of line so that the (default) as-written path of sdf_fused_kernel
// keeps its register budget
__device__ __noinline__ float phi_binned_dev(const float* c, const SdfBinsView* v) { return phi_binned(c, *v, nullptr); }

// kAll = false: the as-written kernel (triangle 0 only) carries none of the all-faces code
template <bool kAll>
__device__ __forceinline__ float voxel_phi_at(const float* c, int num_faces, const int* __restrict__ faces,
                                              const float* __restrict__ vf, const float* tr, const FrameBox& fb,
                                              const float* tri0, const SdfBinsView* bins) {
    if (!kAll || num_faces == 1) {
        if (!ray_hits(c, tri0, tri0 + 3, tri0 + 6)) return 0.f;
        return triangle_distance(c, tri0, tri0 + 3, tri0 + 6);
    }
    if (bins) return phi_binned_dev(c, bins);          // all faces over candidate lists (mvs_sdf_bins.cuh): identical bits
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

// per-slot bin structures of the accelerated all-faces mode (null pointers: brute force)
struct SdfBinsDev {
    const float* tri; const int* cell_ptr; const unsigned short* cell_idx; const int* ray_ptr; const unsigned short* ray_idx;
    const float* meta;                     // [B][8]: s_lo[2], s_scale[2], overflow flag, -, -, -
    int F;
};

// Shared-memory working set of sdf_fused_kernel
struct SdfFusedSmem {
    float ctab[256];
    float s_red[kSdfMaxPasses][8][5];
    int s_wcnt[kSdfMaxPasses][8], s_woff[kSdfMaxPasses][9];
    unsigned s_mask[kSdfMaxPasses][8];
    int seg_n[kSdfFThreads];               // one block's vertices with a non-zero sample gradient
    float seg_g[kSdfFThreads * 3];
    float sA[kSkinFloats];
    float s_beta[kBetas];
    int c_n[kSdfFChunk];
    float c_dv[kSdfFChunk * 3], c_vp[kSdfFChunk * 3], c_dvp[kSdfFChunk * 3];
    float s_dphi[8][kFeatPad];
};

// verts / poffT / Phi / slot_tr / setup / At are rewritten every round by the preceding kernels: plain pointers.  v_posed
// of the (few) listed vertices is recomputed from the pose offsets (vposed_of).
struct SdfFusedArgs {
    const float* verts; const float* poffT; const float* Phi; const float* ST; const float* slot_tr;
    int N, nbox; const SdfFrameSetup* setup; const int* faces; int num_faces, G;
    const float* At; int ldA; const int* ell_j; const float* ell_w; int KW; const float* Wd; const float* Qk;
    float* parts5; float* part; int* pflag; float* gcoord;
    SdfBinsDev bins;
    int block_skip;                        // 0: ignore the record's live-block mask (MVS_SDF_BLOCK_SKIP=0, experiments only)
};

// kAll = false: the reference call as written (the kernel sees triangle 0), the default and the benchmark's mode; kAll = true: the
// intended all-faces field, over candidate lists or by brute force.  Grid (block groups, slots): CTA (pidx, slot) takes
// `passes` blocks of 256 vertices of the frame in `slot`.
template <bool kAll>
__global__ void __launch_bounds__(kSdfFThreads, 3)
sdf_fused_kernel(SdfFusedArgs ar, const int* __restrict__ na_ptr, int passes) {
    SDF_MARK(0);
    pdl_wait();
    SDF_MARK(1);
    __shared__ SdfFusedSmem sm;
    const int na = *na_ptr, slot = blockIdx.y, pidx = blockIdx.x;
    const float* verts = ar.verts; const float* slot_tr = ar.slot_tr;
    const int N = ar.N, nbox = ar.nbox, num_faces = ar.num_faces, G = ar.G, ldA = ar.ldA, KW = ar.KW;
    const int* __restrict__ faces = ar.faces; const float* At = ar.At;
    const int* __restrict__ ell_j = ar.ell_j; const float* __restrict__ ell_w = ar.ell_w;
    const float* __restrict__ Wd = ar.Wd; const float* __restrict__ Qk = ar.Qk;
    float* parts5 = ar.parts5; float* part = ar.part; int* pflag = ar.pflag; float* gcoord = ar.gcoord;
    auto& ctab = sm.ctab; auto& s_red = sm.s_red; auto& s_wcnt = sm.s_wcnt;
    auto& s_woff = sm.s_woff; auto& s_mask = sm.s_mask; auto& seg_n = sm.seg_n; auto& seg_g = sm.seg_g; auto& sA = sm.sA;
    auto& c_n = sm.c_n; auto& c_dv = sm.c_dv; auto& c_vp = sm.c_vp; auto& c_dvp = sm.c_dvp; auto& s_dphi = sm.s_dphi;
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    if (slot >= na) return;
    if (pidx * passes * kSdfFThreads >= N) return;
    // ---- prologue: the frame's set-up (box, triangle 0, cone / plane, chunk-cull verdicts; computed once per frame before
    //      this launch, sdf_frame_setup) with its live-block mask, and its translation, all addressed by the slot alone:
    //      one round trip; then the first vertices of the chunks the cull leaves
    const SdfFrameSetup* rec = ar.setup + slot;
    const float* vf = verts + (size_t)slot * N * 3;
    const float4 tr4 = *reinterpret_cast<const float4*>(slot_tr + 4 * slot);
    const FrameBox fb = rec->fb;
    float cn[3][3], cm[3], pn[3], vpad[3];
#pragma unroll
    for (int q = 0; q < 3; ++q) {
        cn[q][0] = rec->cn[q][0]; cn[q][1] = rec->cn[q][1]; cn[q][2] = rec->cn[q][2];
        cm[q] = rec->cm[q]; pn[q] = rec->pn[q]; vpad[q] = rec->vpad[q];
    }
    const float pd = rec->pd, pm = rec->pm, vpadp = rec->vpadp;
    const float* tri = rec->tri;                       // triangle 0 in box coordinates: read only by the (rare) exact voxel tests
    const uint2 lb = *reinterpret_cast<const uint2*>(rec->live_blocks);
    // Chunk-level cull (sdf_frame_setup): lane p of a warp reads the verdict of the warp's 64-vertex chunk in pass p; a
    // ballot gives every lane all of them (bit p: pass p).  A culled chunk's value and gradient are exactly zero: its warps
    // skip loads, divisions, corners.
    unsigned skipm;
    {
        const int chunk = ((pidx * passes + lane) * kSdfFThreads + warp * 32) / 64;
        const unsigned word = rec->skip[min(chunk >> 5, kSdfSkipWords - 1)];
        const bool my_skip = lane < passes && chunk < nbox && chunk < 32 * kSdfSkipWords && ((word >> (chunk & 31)) & 1u);
        skipm = __ballot_sync(0xffffffffu, my_skip);
    }
    const int nblocks = (N + kSdfFThreads - 1) / kSdfFThreads;
    if (!kAll && ar.block_skip) {
        // Block-level cull: a CTA none of whose blocks has a chunk that is not culled writes what the sampling below would
        // (five +0 sums and flag 0 per block) and retires before its first vertex load and its first barrier.
        const int b0 = pidx * passes;
        const unsigned long long live = ((unsigned long long)lb.y << 32) | lb.x;
        if (b0 < 64 && ((live >> b0) & ((1ull << passes) - 1ull)) == 0ull) {
            if (t < 5 * passes) {
                const int blk = b0 + t / 5;
                if (blk < nblocks) parts5[((size_t)slot * nblocks + blk) * 5 + t % 5] = 0.f;
            } else if (t >= 128 && t < 128 + passes) {
                const int blk = b0 + t - 128;
                if (blk < nblocks) pflag[(size_t)slot * nblocks + blk] = 0;
            }
            return;
        }
    }
    float vcur[3] = {0.f, 0.f, 0.f};                   // this pass' vertex; the next one is fetched a pass ahead
    {
        const int n0 = pidx * passes * kSdfFThreads + t;
        // a culled chunk's vertices are never read
        if (n0 < N && !(skipm & 1u)) { vcur[0] = vf[3 * n0]; vcur[1] = vf[3 * n0 + 1]; vcur[2] = vf[3 * n0 + 2]; }
    }
    if (t < G && t < 256) ctab[t] = (float)(-1 + (t + 0.5) * (double)(float)(2. / (G - 1)));   // voxel_centre, tabulated
    const float tr[3] = {tr4.x, tr4.y, tr4.z};
    const float vgs = (float)G / (float)(G - 1);
    __syncthreads();
    SDF_MARK(2);
    SDF_MARK(3);
    // ---- sampling: block (pidx * passes + pass) of 256 vertices per pass, one vertex per thread and pass.  Sums,
    //      vertex lists and adjoint partials are emitted PER BLOCK, so the arithmetic of a frame does not depend on
    //      how many blocks this launch gave to one CTA (i.e. not on how many other frames are still active): frames
    //      stay bit-for-bit independent problems.  All passes are sampled before the first barrier.
    // accelerated all-faces mode: this frame's candidate lists (built by sdf_bins_kernel just before this launch)
    SdfBinsView bview;
    const SdfBinsView* bvp = nullptr;
    if (kAll && num_faces > 1 && ar.bins.tri != nullptr) {
        const float* mt = ar.bins.meta + 8 * (size_t)slot;
        if (mt[4] == 0.f) {                                 // no list overflow for this frame
            bview.tri = ar.bins.tri + (size_t)slot * ar.bins.F * 9;
            bview.cell_ptr = ar.bins.cell_ptr + (size_t)slot * (kBinCells + 1);
            bview.cell_idx = ar.bins.cell_idx + (size_t)slot * kBinCapD;
            bview.ray_ptr = ar.bins.ray_ptr + (size_t)slot * (kBinRays + 1);
            bview.ray_idx = ar.bins.ray_idx + (size_t)slot * kBinCapR;
            bview.s_lo[0] = mt[0]; bview.s_lo[1] = mt[1]; bview.s_scale[0] = mt[2]; bview.s_scale[1] = mt[3];
            bvp = &bview;
        }
    }
    const bool cull = (num_faces == 1);
    const bool tab = (G <= 256);
#pragma unroll 1
    for (int pass = 0; pass < passes; ++pass) {
        const int blk = pidx * passes + pass;
        if (blk >= nblocks) { if (lane == 0) s_wcnt[pass][warp] = 0; continue; }
        const int n = blk * kSdfFThreads + t;
        const float vme[3] = {vcur[0], vcur[1], vcur[2]};
        if (pass + 1 < passes && n + kSdfFThreads < N && !((skipm >> (pass + 1)) & 1u)) {
            vcur[0] = vf[3 * (n + kSdfFThreads)]; vcur[1] = vf[3 * (n + kSdfFThreads) + 1]; vcur[2] = vf[3 * (n + kSdfFThreads) + 2];
        }
        float acc[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
        float gcv[3] = {0.f, 0.f, 0.f};
        const bool skip = (skipm >> pass) & 1u;
        // all faces over candidate lists: the warp evaluates its 32 vertices' voxels ONE AT A TIME, the lanes sharing out the
        // candidates (phi_binned_warp); every lane then goes on with its own eight values exactly as in the other modes
        float pc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        bool have_pc = false;
        if constexpr (kAll) {
            if (bvp != nullptr) {
                const bool act = n < N && !skip;
                int j0[3] = {0, 0, 0};
                float ccx[2] = {0.f, 0.f}, ccy[2] = {0.f, 0.f}, ccz[2] = {0.f, 0.f};
                if (act) {
#pragma unroll
                    for (int c = 0; c < 3; ++c) {
                        const float lc = ((vme[c] + tr[c]) - fb.centre[c]) / fb.scale;
                        j0[c] = (int)floorf(((lc + 1.f) * G - 1.f) / 2.f);
                    }
#pragma unroll
                    for (int o = 0; o < 2; ++o) {
                        const int ii = min(max(j0[0] + o, 0), G - 1), jj = min(max(j0[1] + o, 0), G - 1), kk = min(max(j0[2] + o, 0), G - 1);
                        if (tab) { ccx[o] = ctab[ii]; ccy[o] = ctab[jj]; ccz[o] = ctab[kk]; }
                        else { float c3[3]; voxel_centre(ii, jj, kk, G, c3); ccx[o] = c3[0]; ccy[o] = c3[1]; ccz[o] = c3[2]; }
                    }
                }
                const unsigned actm = __ballot_sync(0xffffffffu, act);
                for (int src = 0; src < 32; ++src) {
                    if (!((actm >> src) & 1u)) continue;
                    const int b0 = __shfl_sync(0xffffffffu, j0[0], src), b1 = __shfl_sync(0xffffffffu, j0[1], src),
                              b2 = __shfl_sync(0xffffffffu, j0[2], src);
                    float bx[2], by[2], bz[2];
#pragma unroll
                    for (int o = 0; o < 2; ++o) {
                        bx[o] = __shfl_sync(0xffffffffu, ccx[o], src); by[o] = __shfl_sync(0xffffffffu, ccy[o], src);
                        bz[o] = __shfl_sync(0xffffffffu, ccz[o], src);
                    }
#pragma unroll
                    for (int corner = 0; corner < 8; ++corner) {
                        const int ox = corner & 1, oy = (corner >> 1) & 1, oz = corner >> 2;
                        const int ii = b0 + ox, jj = b1 + oy, kk = b2 + oz;
                        if (ii < 0 || ii >= G || jj < 0 || jj >= G || kk < 0 || kk >= G) continue;
                        const float cc[3] = {bx[ox], by[oy], bz[oz]};
                        const float p = phi_binned_warp(cc, bvp);
                        if (lane == src) pc[corner] = p;
                    }
                }
                have_pc = true;
            }
        }
        if (n < N && !skip) {
            float loc[3], w1[3];
            int i0[3];
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                loc[c] = ((vme[c] + tr[c]) - fb.centre[c]) / fb.scale;
                const float ix = ((loc[c] + 1.f) * G - 1.f) / 2.f;
                const float fl = floorf(ix);
                i0[c] = (int)fl;
                w1[c] = ix - fl;
            }
            bool vout = false;                             // no voxel this vertex touches can have phi != 0
            if (cull) {
                const float wc[3] = {(loc[0] + 1.f) * vgs, (loc[1] + 1.f) * vgs, (loc[2] + 1.f) * vgs};
                bool any_neg = false, any_pos = false;
#pragma unroll
                for (int q = 0; q < 3; ++q) {
                    const float sq = cn[q][0] * wc[0] + cn[q][1] * wc[1] + cn[q][2] * wc[2];
                    any_neg = any_neg || (sq + vpad[q] < -cm[q]);
                    any_pos = any_pos || (sq - vpad[q] > cm[q]);
                }
                const float sp = pn[0] * wc[0] + pn[1] * wc[1] + pn[2] * wc[2] - pd;
                vout = (any_neg && any_pos) || (pd > pm && sp + vpadp < -pm) || (pd < -pm && sp - vpadp > pm);
            }
            float val = 0.f, dix[3] = {0.f, 0.f, 0.f};
            if (!vout) {
                // voxel centres of the 2 x 2 x 2 cell and, per cone plane, the per-axis parts of <centre + 1, normal>:
                // a corner's three plane distances are then two adds each
                float cx[2], cy[2], cz[2], px[3][2], py[3][2], pz[3][2];
#pragma unroll
                for (int o = 0; o < 2; ++o) {
                    const int ii = min(max(i0[0] + o, 0), G - 1), jj = min(max(i0[1] + o, 0), G - 1), kk = min(max(i0[2] + o, 0), G - 1);
                    if (tab) { cx[o] = ctab[ii]; cy[o] = ctab[jj]; cz[o] = ctab[kk]; }
                    else { float c3[3]; voxel_centre(ii, jj, kk, G, c3); cx[o] = c3[0]; cy[o] = c3[1]; cz[o] = c3[2]; }
#pragma unroll
                    for (int q = 0; q < 3; ++q) {
                        px[q][o] = (cx[o] + 1.f) * cn[q][0]; py[q][o] = (cy[o] + 1.f) * cn[q][1]; pz[q][o] = (cz[o] + 1.f) * cn[q][2];
                    }
                }
                // whole-cell test first: the extreme plane distances over the 8 corners are sums of per-axis extremes; if
                // one plane has every corner outside (negative) and another every corner on its positive side, no corner
                // can be inside the cone -- true for almost every vertex -- and the corner loop is skipped
                float qx[2], qy[2], qz[2];
#pragma unroll
                for (int o = 0; o < 2; ++o) { qx[o] = (cx[o] + 1.f) * pn[0]; qy[o] = (cy[o] + 1.f) * pn[1]; qz[o] = (cz[o] + 1.f) * pn[2]; }
                bool cell_out = false;
                if (cull) {
                    // plane side of the whole cell
                    const float smaxp = fmaxf(qx[0], qx[1]) + fmaxf(qy[0], qy[1]) + fmaxf(qz[0], qz[1]) - pd;
                    const float sminp = fminf(qx[0], qx[1]) + fminf(qy[0], qy[1]) + fminf(qz[0], qz[1]) - pd;
                    if ((pd > pm && smaxp < -pm) || (pd < -pm && sminp > pm)) cell_out = true;
                    bool any_neg = false, any_pos = false;
#pragma unroll
                    for (int q = 0; q < 3; ++q) {
                        const float smax = fmaxf(px[q][0], px[q][1]) + fmaxf(py[q][0], py[q][1]) + fmaxf(pz[q][0], pz[q][1]);
                        const float smin = fminf(px[q][0], px[q][1]) + fminf(py[q][0], py[q][1]) + fminf(pz[q][0], pz[q][1]);
                        any_neg = any_neg || (smax < -cm[q]);
                        any_pos = any_pos || (smin > cm[q]);
                    }
                    cell_out = cell_out || (any_neg && any_pos);
                }
#pragma unroll
                for (int corner = 0; corner < 8; ++corner) {
                    if (cell_out) break;
                    const int ox = corner & 1, oy = (corner >> 1) & 1, oz = corner >> 2;
                    const int ii = i0[0] + ox, jj = i0[1] + oy, kk = i0[2] + oz;
                    if (ii < 0 || ii >= G || jj < 0 || jj >= G || kk < 0 || kk >= G) continue;
                    if (cull) {
                        // phi != 0 needs the ray from the voxel centre to (-1,-1,-1) to cross triangle 0, i.e. the centre
                        // inside the cone the triangle spans from that corner: on the same side of its three planes.
                        // Conservative margin (|centre + 1| <= 2 sqrt 3): only voxels safely outside are skipped, every
                        // other one is decided exactly by ray_hits.
                        const float s1 = px[0][ox] + py[0][oy] + pz[0][oz];
                        const float s2 = px[1][ox] + py[1][oy] + pz[1][oz];
                        const float s3 = px[2][ox] + py[2][oy] + pz[2][oz];
                        const bool neg = (s1 < -cm[0]) || (s2 < -cm[1]) || (s3 < -cm[2]);
                        const bool pos = (s1 > cm[0]) || (s2 > cm[1]) || (s3 > cm[2]);
                        if (neg && pos) continue;
                        const float sp = qx[ox] + qy[oy] + qz[oz] - pd;
                        if ((pd > pm && sp < -pm) || (pd < -pm && sp > pm)) continue;      // corner side of the triangle plane
                    }
                    const float cc[3] = {cx[ox], cy[oy], cz[oz]};
                    const float p = (kAll && have_pc) ? pc[corner] : voxel_phi_at<kAll>(cc, num_faces, faces, vf, tr, fb, tri, bvp);
                    if (p == 0.f) continue;
                    const float wx = ox ? w1[0] : 1.f - w1[0], wy = oy ? w1[1] : 1.f - w1[1], wz = oz ? w1[2] : 1.f - w1[2];
                    val += p * wx * wy * wz;
                    dix[0] += p * (ox ? 1.f : -1.f) * wy * wz;
                    dix[1] += p * wx * (oy ? 1.f : -1.f) * wz;
                    dix[2] += p * wx * wy * (oz ? 1.f : -1.f);
                }
            }
            float gdl = 0.f;
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                gcv[c] = dix[c] * (0.5f * G);
                acc[1 + c] = gcv[c]; gdl += gcv[c] * loc[c];
            }
            acc[0] = val;
            acc[4] = gdl;
        }
        const bool nz = (gcv[0] != 0.f) || (gcv[1] != 0.f) || (gcv[2] != 0.f);
        const unsigned nzm = __ballot_sync(0xffffffffu, nz);
        if (nz) {                                          // rare: parked in global scratch until the adjoint phase
            float* gp = gcoord + ((size_t)slot * N + n) * 3;
            gp[0] = gcv[0]; gp[1] = gcv[1]; gp[2] = gcv[2];
        }
        // almost every warp is outside the cone: all-zero contributions need no shuffle tree (adding zeros is exact)
        if (__ballot_sync(0xffffffffu, acc[0] != 0.f || nz)) {
#pragma unroll
            for (int q = 0; q < 5; ++q) {
                float a = acc[q];
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
                if (lane == 0) s_red[pass][warp][q] = a;
            }
        } else if (lane < 5) {
            s_red[pass][warp][lane] = 0.f;
        }
        if (lane == 0) { s_wcnt[pass][warp] = __popc(nzm); s_mask[pass][warp] = nzm; }
    }
    __syncthreads();
    SDF_MARK(4);
    if (t < 5 * passes) {
        const int pass = t / 5, q = t % 5, blk = pidx * passes + pass;
        if (blk < nblocks) {
            float a = 0.f;
            for (int w2 = 0; w2 < 8; ++w2) a += s_red[pass][w2][q];
            parts5[((size_t)slot * nblocks + blk) * 5 + q] = a;
        }
    } else if (t >= 128 && t < 128 + passes) {
        const int pass = t - 128, blk = pidx * passes + pass;
        int o = 0;
        if (blk < nblocks) {
            for (int w2 = 0; w2 < 8; ++w2) { s_woff[pass][w2] = o; o += s_wcnt[pass][w2]; }
            pflag[(size_t)slot * nblocks + blk] = o > 0 ? 1 : 0;
        }
        s_woff[pass][8] = o;
    }
    __syncthreads();
    // ---- adjoint of the vertex stage for the listed vertices of each block (unit frame factor); rare
    bool have_A = false;
#pragma unroll 1
    for (int pass = 0; pass < passes; ++pass) {
        const int blk = pidx * passes + pass;
        const int total = s_woff[pass][8];
        if (total == 0) continue;
        __syncthreads();                                   // the previous block's adjoint is done with seg_* / c_*
        const unsigned nzm = s_mask[pass][warp];
        if (nzm & (1u << lane)) {                          // ascending vertex order: (warp, lane)
            const int pos = s_woff[pass][warp] + __popc(nzm & ((1u << lane) - 1u));
            seg_n[pos] = blk * kSdfFThreads + t;
            const float* gp = gcoord + ((size_t)slot * N + blk * kSdfFThreads + t) * 3;       // written by this thread
            seg_g[3 * pos] = gp[0]; seg_g[3 * pos + 1] = gp[1]; seg_g[3 * pos + 2] = gp[2];
        }
        if (!have_A) {
            for (int e = t; e < kSkinFloats; e += kSdfFThreads) sA[e] = At[(size_t)e * ldA + slot];
            if (t < kBetas) sm.s_beta[t] = ar.Phi[(size_t)slot * kFeatPad + kPoseBasis + t];
            have_A = true;
        }
        float accA0 = 0.f, accA1 = 0.f;
        float accP[7] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};    // d Phi[lane + 32 i], this warp's share of the columns
        for (int e0 = 0; e0 < total; e0 += kSdfFChunk) {
            const int cnt = min(kSdfFChunk, total - e0);
            __syncthreads();
            if (t < cnt) {
                const int src = e0 + t;
                const int nn = seg_n[src];
                c_n[t] = nn;
                const float d0 = seg_g[3 * src], d1 = seg_g[3 * src + 1], d2 = seg_g[3 * src + 2];
                float Gm[9];
#pragma unroll
                for (int c = 0; c < 9; ++c) Gm[c] = 0.f;
                for (int e = 0; e < KW; ++e) {
                    const float w = ell_w[(size_t)nn * KW + e];
                    if (w != 0.f) {
                        const float* Aj = &sA[12 * ell_j[(size_t)nn * KW + e]];
#pragma unroll
                        for (int r = 0; r < 3; ++r)
#pragma unroll
                            for (int c = 0; c < 3; ++c) Gm[3 * r + c] = fmaf(w, Aj[4 * r + c], Gm[3 * r + c]);
                    }
                }
                c_dv[3 * t] = d0; c_dv[3 * t + 1] = d1; c_dv[3 * t + 2] = d2;
                c_dvp[3 * t] = Gm[0] * d0 + Gm[3] * d1 + Gm[6] * d2;
                c_dvp[3 * t + 1] = Gm[1] * d0 + Gm[4] * d1 + Gm[7] * d2;
                c_dvp[3 * t + 2] = Gm[2] * d0 + Gm[5] * d1 + Gm[8] * d2;
#pragma unroll
                for (int c = 0; c < 3; ++c)      // v_posed, bit for bit what skin_vertex computed
                    c_vp[3 * t + c] = vposed_of(ar.ST + (size_t)nn * 33 + 11 * c, sm.s_beta, ar.poffT[(size_t)(3 * nn + c) * ldA + slot]);
            }
            __syncthreads();
            {   // dA: thread t owns entry t (and 256 + t for t < 32)
                const int j0 = t / 12, r0 = (t % 12) / 4, cc0 = t % 4;
                const int e1 = t + kSdfFThreads, j1 = e1 / 12, r1 = (e1 % 12) / 4, cc1 = e1 % 4;
                const bool two = t < kSkinFloats - kSdfFThreads;
#pragma unroll 4
                for (int i = 0; i < cnt; ++i) {
                    const float* wrow = Wd + (size_t)c_n[i] * kJoints;
                    const float w0 = __ldg(wrow + j0);
                    const float w1v = two ? __ldg(wrow + j1) : 0.f;
                    if (w0 != 0.f) {
                        const float wd = w0 * c_dv[3 * i + r0];
                        accA0 = (cc0 < 3) ? fmaf(wd, c_vp[3 * i + cc0], accA0) : accA0 + wd;
                    }
                    if (w1v != 0.f) {
                        const float wd = w1v * c_dv[3 * i + r1];
                        accA1 = (cc1 < 3) ? fmaf(wd, c_vp[3 * i + cc1], accA1) : accA1 + wd;
                    }
                }
            }
            // d Phi: a warp takes every 8th column and reads its whole Qk row (7 coalesced loads per lane, two columns
            // = 14 independent loads in flight); the eight warps' shares are folded in a fixed order below
            for (int col = warp; col < 3 * cnt; col += 16) {
                const int colb = col + 8;
                const bool hb = colb < 3 * cnt;
                const float* ra = Qk + (size_t)(3 * c_n[col / 3] + col % 3) * kFeatPad + lane;
                const float* rb = Qk + (size_t)(3 * c_n[(hb ? colb : col) / 3] + (hb ? colb : col) % 3) * kFeatPad + lane;
                float qa[7], qb[7];
#pragma unroll
                for (int i = 0; i < 7; ++i) { qa[i] = __ldg(ra + 32 * i); qb[i] = __ldg(rb + 32 * i); }
                const float da = c_dvp[col], db = hb ? c_dvp[colb] : 0.f;
#pragma unroll
                for (int i = 0; i < 7; ++i) { accP[i] = fmaf(da, qa[i], accP[i]); accP[i] = fmaf(db, qb[i], accP[i]); }
            }
        }
#pragma unroll
        for (int i = 0; i < 7; ++i) s_dphi[warp][lane + 32 * i] = accP[i];
        __syncthreads();
        float* o = part + ((size_t)slot * nblocks + blk) * kPartFloats;
        o[t] = accA0;
        if (t < kSkinFloats - kSdfFThreads) o[kSdfFThreads + t] = accA1;
        if (t < kFeatPad) {
            float a = 0.f;
#pragma unroll
            for (int w2 = 0; w2 < 8; ++w2) a += s_dphi[w2][t];
            o[kSkinFloats + t] = a;
        }
    }
    __syncthreads();
    SDF_MARK(5);
}

int ensure_sdf_fused_ws(mvs_ctx* ctx);                 // mvs_sdf.cu: allocates the dense-regime SDF scratch
SdfFusedArgs make_sdf_fused_args(mvs_ctx* ctx);         // mvs_sdf.cu (needs the tensor-core path's pose offsets: tc_poffT)

}  // namespace mvs
