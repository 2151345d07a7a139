// mvs_render: a batched rasteriser for fitted meshes (DESIGN.md section 4d).  One work item is one (frame, view) pair.  Per chunk
// of frames:
//   render_normals    per (frame, vertex): the sum of the cross products of the faces around the vertex, gathered in ascending
//                     face order from the model's vertex -> face CSR (no atomics: deterministic)
//   render_vertices   per (item, vertex / keypoint): pixel position and camera depth through the view (project_fwd, with the
//                     rig's lens distortion)
//   render_bin<count> per (item, face): the screen tiles its clamped box touches, counted; then an exclusive scan of the counts
//   render_bin<fill>  the same tiles, each gets the face in its list (order within a list is free: see below)
//   render_raster     one CTA per (item, tile): every pixel keeps the smallest (depth bits << 32 | face) of the triangles covering
//                     its sample, so visibility does not depend on the order of a tile's list; then shading, background, markers
// Every launch is timed under KID_MISC.
#include <algorithm>

#include "mvs_internal.cuh"
#include "mvs_render_dev.cuh"

namespace mvs {

namespace {

constexpr int kRasterThreads = kRenderTile * kRenderTile;
constexpr int kScanThreads = 1024;
constexpr size_t kRenderChunkBytes = size_t(256) << 20;      // scratch of one chunk of frames (vertices, keypoints, tile counts)
constexpr long long kRenderListEntries = 1LL << 28;          // tile-list entries (1 GiB) above which a chunk of frames is split

struct RenderArgs {
    const float* verts;               // [n][N][3]
    const float* kps;                 // [n][K][3] or NULL
    RigSet rigs;                      // rig of frame f0 + f: rigs.of[f0 + f]
    const unsigned char* bg;
    unsigned char* img;
    int* face;
    float* depth;
    const int* faces;
    const int* vf_ptr;
    const int* vf_idx;
    float4* nrm;
    float4* sv;
    float4* sk;
    int* cnt;
    long long* off;
    int* list;
    int N, F, K, Vmax, W, H, TX, T, f0;
    float base[3], ambient, radius;
    unsigned char mc[3];
};

__device__ __forceinline__ void load_vec3(const float* p, float* q) { q[0] = __ldg(p); q[1] = __ldg(p + 1); q[2] = __ldg(p + 2); }

__global__ void render_normals_kernel(RenderArgs a) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x, f = blockIdx.y;
    if (i >= a.N) return;
    const float* V = a.verts + (size_t)(a.f0 + f) * a.N * 3;
    float s[3] = {0.f, 0.f, 0.f};
    for (int e = __ldg(a.vf_ptr + i), e1 = __ldg(a.vf_ptr + i + 1); e < e1; ++e) {
        const int* t = a.faces + 3 * __ldg(a.vf_idx + e);
        float p0[3], p1[3], p2[3];
        load_vec3(V + 3 * __ldg(t), p0);
        load_vec3(V + 3 * __ldg(t + 1), p1);
        load_vec3(V + 3 * __ldg(t + 2), p2);
        const float b[3] = {p1[0] - p0[0], p1[1] - p0[1], p1[2] - p0[2]}, c[3] = {p2[0] - p0[0], p2[1] - p0[1], p2[2] - p0[2]};
        s[0] += b[1] * c[2] - b[2] * c[1];
        s[1] += b[2] * c[0] - b[0] * c[2];
        s[2] += b[0] * c[1] - b[1] * c[0];
    }
    a.nrm[(size_t)f * a.N + i] = make_float4(s[0], s[1], s[2], 0.f);
}

__global__ void render_vertices_kernel(RenderArgs a) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x, item = blockIdx.y;
    const int f = item / a.Vmax, v = item % a.Vmax, g = a.f0 + f;
    const FrameRig fr = frame_rig(a.rigs, g);
    if (v >= fr.num_views || i >= a.N + a.K) return;
    const CamF cam = rig_camera(fr, v);
    float q[3], x[3], uv[2];
    if (i < a.N) load_vec3(a.verts + ((size_t)g * a.N + i) * 3, q);
    else load_vec3(a.kps + ((size_t)g * a.K + i - a.N) * 3, q);
    project_fwd(cam, q, x, uv, fr.dist ? fr.dist + v : nullptr);
    const float4 o = make_float4(uv[0], uv[1], x[2], 0.f);
    if (i < a.N) a.sv[(size_t)item * a.N + i] = o;
    else a.sk[(size_t)item * a.K + i - a.N] = o;
}

__device__ __forceinline__ RVert screen_vertex(const RenderArgs& a, int item, int vid) {
    const float4 p = a.sv[(size_t)item * a.N + vid];
    return RVert{p.x, p.y, p.z, 0.f};
}

// kFill = false: count each face in the tiles its box touches; true: write it into their lists (a.cnt zeroed: the cursors)
template <bool kFill> __global__ void render_bin_kernel(RenderArgs a) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x, item = blockIdx.y;
    if (t >= a.F) return;
    const int v = item % a.Vmax;
    if (v >= frame_rig(a.rigs, a.f0 + item / a.Vmax).num_views) return;
    const int* fv = a.faces + 3 * t;
    int x0, x1, y0, y1;
    if (!render_tri_box(screen_vertex(a, item, __ldg(fv)), screen_vertex(a, item, __ldg(fv + 1)), screen_vertex(a, item, __ldg(fv + 2)),
                        a.W, a.H, &x0, &x1, &y0, &y1))
        return;
    const size_t base = (size_t)item * a.T;
    for (int ty = y0 / kRenderTile; ty <= y1 / kRenderTile; ++ty)
        for (int tx = x0 / kRenderTile; tx <= x1 / kRenderTile; ++tx) {
            const size_t tile = base + (size_t)ty * a.TX + tx;
            const int slot = atomicAdd(a.cnt + tile, 1);
            if (kFill) a.list[a.off[tile] + slot] = t;
        }
}

// exclusive scan of cnt [M] into off [M + 1]: block-local inclusive scans (off[i + 1]) and block totals, the totals' exclusive
// scan by one block, then each block's offset added
__device__ __forceinline__ long long block_inclusive_scan(long long x, long long* warp_tot) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const long long y = __shfl_up_sync(0xffffffffu, x, d);
        if (lane >= d) x += y;
    }
    if (lane == 31) warp_tot[w] = x;
    __syncthreads();
    if (w == 0) {
        long long s = warp_tot[lane];
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const long long y = __shfl_up_sync(0xffffffffu, s, d);
            if (lane >= d) s += y;
        }
        warp_tot[lane] = s;
    }
    __syncthreads();
    return x + (w ? warp_tot[w - 1] : 0);
}

__global__ void __launch_bounds__(kScanThreads) render_scan_local_kernel(const int* cnt, long long M, long long* off, long long* part) {
    __shared__ long long wt[32];
    const long long i = (long long)blockIdx.x * kScanThreads + threadIdx.x;
    const long long s = block_inclusive_scan(i < M ? cnt[i] : 0, wt);
    if (i < M) off[i + 1] = s;
    if (threadIdx.x == kScanThreads - 1) part[blockIdx.x] = s;
    if (i == 0) off[0] = 0;
}

__global__ void __launch_bounds__(kScanThreads) render_scan_parts_kernel(long long* part, int nb) {
    __shared__ long long wt[32];
    __shared__ long long carry;
    if (threadIdx.x == 0) carry = 0;
    for (int b0 = 0; b0 < nb; b0 += kScanThreads) {
        const int i = b0 + threadIdx.x;
        const long long x = i < nb ? part[i] : 0;
        __syncthreads();
        const long long s = block_inclusive_scan(x, wt);
        const long long c = carry;
        if (i < nb) part[i] = c + s - x;             // exclusive
        __syncthreads();
        if (threadIdx.x == kScanThreads - 1) carry = c + s;
        __syncthreads();
    }
}

__global__ void __launch_bounds__(kScanThreads) render_scan_add_kernel(long long* off, long long M, const long long* part) {
    const long long i = (long long)blockIdx.x * kScanThreads + threadIdx.x;
    if (i < M) off[i + 1] += part[blockIdx.x];
}

__global__ void __launch_bounds__(kRasterThreads) render_raster_kernel(RenderArgs a) {
    __shared__ RTri tri[kRasterThreads];
    __shared__ RVert kp[kMaxKeypoints];
    const long long blk = blockIdx.x;
    const int item = (int)(blk / a.T), tile = (int)(blk % a.T);
    const int f = item / a.Vmax, v = item % a.Vmax, g = a.f0 + f;
    const FrameRig fr = frame_rig(a.rigs, g);
    if (v >= fr.num_views) return;                      // the whole CTA
    const int x = (tile % a.TX) * kRenderTile + (threadIdx.x % kRenderTile);
    const int y = (tile / a.TX) * kRenderTile + (threadIdx.x / kRenderTile);
    const bool in = x < a.W && y < a.H;
    const float px = (float)x, py = (float)y;
    const int K = a.radius > 0.f ? a.K : 0;
    if (threadIdx.x < K) {
        const float4 k = a.sk[(size_t)item * a.K + threadIdx.x];
        kp[threadIdx.x] = RVert{k.x, k.y, k.z, 0.f};
    }
    unsigned long long best = ~0ull;
    float bl[3] = {0.f, 0.f, 0.f};
    const long long beg = a.off[blk], end = a.off[blk + 1];
    for (long long b0 = beg; b0 < end; b0 += kRasterThreads) {
        __syncthreads();
        if (b0 + threadIdx.x < end) {
            const int fc = a.list[b0 + threadIdx.x];
            const int id[3] = {__ldg(a.faces + 3 * fc), __ldg(a.faces + 3 * fc + 1), __ldg(a.faces + 3 * fc + 2)};
            const RVert p[3] = {screen_vertex(a, item, id[0]), screen_vertex(a, item, id[1]), screen_vertex(a, item, id[2])};
            RTri t;
            if (!render_tri_setup(p, id, fc, a.W, a.H, t)) t.face = -1;
            tri[threadIdx.x] = t;
        }
        __syncthreads();
        const int nb = (int)min((long long)kRasterThreads, end - b0);
        if (!in) continue;
        for (int j = 0; j < nb; ++j) {
            const RTri& t = tri[j];
            if (t.face < 0 || px < t.x0 || px > t.x1 || py < t.y0 || py > t.y1) continue;
            double w[3];
            if (!render_cover(t, px, py, w)) continue;
            float lam[3];
            const float z = render_depth(t, w, lam);
            const unsigned long long key = render_key(z, t.face);
            if (key < best) { best = key; bl[0] = lam[0]; bl[1] = lam[1]; bl[2] = lam[2]; }
        }
    }
    __syncthreads();
    if (!in) return;
    const size_t pix = (((size_t)g * a.Vmax + v) * a.H + y) * a.W + x;
    const int face = best == ~0ull ? -1 : (int)(unsigned)(best & 0xffffffffu);
    if (a.face) a.face[pix] = face;
    if (a.depth) a.depth[pix] = face < 0 ? __int_as_float(0x7f800000) : __uint_as_float((unsigned)(best >> 32));
    if (!a.img) return;
    unsigned char rgb[3];
    if (face >= 0) {
        const CamF cam = rig_camera(fr, v);
        float z[3], p[3][3], n[3][3];
        for (int k = 0; k < 3; ++k) {
            const int vid = __ldg(a.faces + 3 * face + k);
            float q[3];
            load_vec3(a.verts + ((size_t)g * a.N + vid) * 3, q);
            mat3_vec(cam.R, q, p[k]);                   // camera-space position R q + t
            for (int c = 0; c < 3; ++c) p[k][c] += cam.t[c];
            z[k] = screen_vertex(a, item, vid).z;
            const float4 s = a.nrm[(size_t)f * a.N + vid];
            const float sv[3] = {s.x, s.y, s.z};
            render_normal(cam.R, sv, n[k]);
        }
        const float I = render_intensity(bl, z, p, n, a.ambient);
        for (int c = 0; c < 3; ++c) rgb[c] = render_channel(a.base[c], I);
    } else {
        for (int c = 0; c < 3; ++c) rgb[c] = a.bg ? a.bg[pix * 3 + c] : (unsigned char)0;
    }
    for (int k = 0; k < K; ++k)
        if (render_marker(kp[k], px, py, a.radius)) {
            rgb[0] = a.mc[0]; rgb[1] = a.mc[1]; rgb[2] = a.mc[2];
            break;
        }
    for (int c = 0; c < 3; ++c) a.img[pix * 3 + c] = rgb[c];
}

}  // namespace

int render_launch(mvs_ctx* ctx, int n, const float* verts, const float* keypoints, const int* rig, const unsigned char* background,
                  unsigned char* image, int* face, float* depth, const mvs_render_config& cfg, cudaStream_t st) {
    const DevModel& m = ctx->m;
    RenderScratch& S = ctx->render;
    RenderArgs a{};
    a.verts = verts; a.kps = keypoints; a.rigs = RigSet{ctx->rigs_dev.p, rig};
    a.bg = background; a.img = image; a.face = face; a.depth = depth;
    a.faces = m.faces; a.vf_ptr = m.vf_ptr; a.vf_idx = m.vf_idx;
    a.N = m.N; a.F = m.F; a.K = keypoints ? m.K : 0; a.Vmax = ctx->vmax; a.W = cfg.width; a.H = cfg.height;
    a.TX = (cfg.width + kRenderTile - 1) / kRenderTile;
    a.T = a.TX * ((cfg.height + kRenderTile - 1) / kRenderTile);
    for (int c = 0; c < 3; ++c) { a.base[c] = cfg.base_color[c]; a.mc[c] = cfg.marker_color[c]; }
    a.ambient = cfg.ambient; a.radius = cfg.marker_radius;
    // frames per chunk: the chunk's scratch under kRenderChunkBytes (at least one frame), items within a grid's y extent
    const size_t per_frame = (size_t)m.N * 16 + (size_t)a.Vmax * ((size_t)(m.N + m.K) * 16 + (size_t)a.T * 12);
    int nc = (int)std::max<size_t>(1, std::min<size_t>({(size_t)n, kRenderChunkBytes / per_frame, (size_t)(65535 / a.Vmax)}));
    int rc;
    if ((rc = dev_grow(ctx, S.nrm, (size_t)nc * m.N)) || (rc = dev_grow(ctx, S.sv, (size_t)nc * a.Vmax * m.N)) ||
        (rc = dev_grow(ctx, S.sk, (size_t)nc * a.Vmax * m.K)) || (rc = dev_grow(ctx, S.cnt, (size_t)nc * a.Vmax * a.T)) ||
        (rc = dev_grow(ctx, S.off, (size_t)nc * a.Vmax * a.T + 1)) ||
        (rc = dev_grow(ctx, S.part, ((size_t)nc * a.Vmax * a.T + kScanThreads - 1) / kScanThreads)))
        return rc;
    a.nrm = S.nrm.p; a.sv = S.sv.p; a.sk = S.sk.p; a.cnt = S.cnt.p; a.off = S.off.p;
    for (int f0 = 0; f0 < n;) {
        const int fn = std::min(nc, n - f0), items = fn * a.Vmax;
        const long long M = (long long)items * a.T;
        const int nb = (int)((M + kScanThreads - 1) / kScanThreads);
        a.f0 = f0;
        MVS_LAUNCH(ctx, KID_MISC, st, render_normals_kernel<<<dim3((m.N + 255) / 256, fn), 256, 0, st>>>(a));
        MVS_LAUNCH(ctx, KID_MISC, st, render_vertices_kernel<<<dim3((m.N + a.K + 255) / 256, items), 256, 0, st>>>(a));
        MVS_CUDA_OK(ctx, cudaMemsetAsync(a.cnt, 0, (size_t)M * sizeof(int), st));
        MVS_LAUNCH(ctx, KID_MISC, st, render_bin_kernel<false><<<dim3((m.F + 255) / 256, items), 256, 0, st>>>(a));
        MVS_LAUNCH(ctx, KID_MISC, st, render_scan_local_kernel<<<nb, kScanThreads, 0, st>>>(a.cnt, M, a.off, S.part.p));
        MVS_LAUNCH(ctx, KID_MISC, st, render_scan_parts_kernel<<<1, kScanThreads, 0, st>>>(S.part.p, nb));
        MVS_LAUNCH(ctx, KID_MISC, st, render_scan_add_kernel<<<nb, kScanThreads, 0, st>>>(a.off, M, S.part.p));
        long long total = 0;
        MVS_CUDA_OK(ctx, cudaMemcpyAsync(&total, a.off + M, sizeof(long long), cudaMemcpyDeviceToHost, st));
        MVS_CUDA_OK(ctx, cudaStreamSynchronize(st));
        // Faces close to the near plane can have boxes that span the image, so a chunk's lists may be far longer than its body
        // coverage suggests: then the chunk is redone in halves (every frame's bits are its own, so the split changes none).
        // One frame alone may still need up to faces x tiles entries per view.
        if (total > kRenderListEntries && fn > 1) {
            nc = fn / 2;
            continue;
        }
        if ((rc = dev_grow(ctx, S.list, (size_t)std::max(total, 1LL)))) return rc;
        a.list = S.list.p;
        MVS_CUDA_OK(ctx, cudaMemsetAsync(a.cnt, 0, (size_t)M * sizeof(int), st));
        MVS_LAUNCH(ctx, KID_MISC, st, render_bin_kernel<true><<<dim3((m.F + 255) / 256, items), 256, 0, st>>>(a));
        MVS_LAUNCH(ctx, KID_MISC, st, render_raster_kernel<<<(unsigned)M, kRasterThreads, 0, st>>>(a));
        f0 += fn;
    }
    MVS_CUDA_OK(ctx, cudaGetLastError());
    return MVS_OK;
}

}  // namespace mvs
