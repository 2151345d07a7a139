// Host build of the rasteriser's per-pixel routines (mvsmplfitting_b200/csrc/mvs_render_dev.cuh): one view drawn by brute force
// (every triangle over its sample box) with the same set-up, coverage, depth key, shading and marker functions the raster kernel
// calls.  Built by tests/test_render_oracle.py.
#include <limits>
#include <vector>

#include "../../mvsmplfitting_b200/csrc/mvs_render_dev.cuh"

using namespace mvs;

extern "C" void render_view_host(int N, int F, const float* sv, const int* faces, int W, int H, const float* pcam, const float* nsum,
                                 const float* R, int K, const float* kp, const float* base, float ambient, float radius,
                                 const unsigned char* mc, const unsigned char* bg, unsigned char* img, int* face, float* depth) {
    std::vector<unsigned long long> best((size_t)W * H, ~0ull);
    std::vector<float> lam((size_t)W * H * 3, 0.f);
    const RVert* p = reinterpret_cast<const RVert*>(sv);
    for (int t = 0; t < F; ++t) {
        const int id[3] = {faces[3 * t], faces[3 * t + 1], faces[3 * t + 2]};
        const RVert q[3] = {p[id[0]], p[id[1]], p[id[2]]};
        RTri tri;
        if (!render_tri_setup(q, id, t, W, H, tri)) continue;
        for (int y = (int)tri.y0; y <= (int)tri.y1; ++y)
            for (int x = (int)tri.x0; x <= (int)tri.x1; ++x) {
                double w[3];
                if (!render_cover(tri, (float)x, (float)y, w)) continue;
                float l[3];
                const float z = render_depth(tri, w, l);
                const unsigned long long key = render_key(z, t);
                const size_t i = (size_t)y * W + x;
                if (key < best[i]) {
                    best[i] = key;
                    for (int k = 0; k < 3; ++k) lam[3 * i + k] = l[k];
                }
            }
    }
    const RVert* kv = reinterpret_cast<const RVert*>(kp);
    for (int y = 0; y < H; ++y)
        for (int x = 0; x < W; ++x) {
            const size_t i = (size_t)y * W + x;
            const int f = best[i] == ~0ull ? -1 : (int)(unsigned)(best[i] & 0xffffffffu);
            face[i] = f;
            const unsigned u = (unsigned)(best[i] >> 32);
            float d;
            memcpy(&d, &u, sizeof(d));
            depth[i] = f < 0 ? std::numeric_limits<float>::infinity() : d;
            unsigned char rgb[3];
            if (f >= 0) {
                float z[3], pp[3][3], n[3][3];
                for (int k = 0; k < 3; ++k) {
                    const int v = faces[3 * f + k];
                    z[k] = p[v].z;
                    for (int c = 0; c < 3; ++c) pp[k][c] = pcam[3 * v + c];
                    render_normal(R, nsum + 3 * v, n[k]);
                }
                const float I = render_intensity(&lam[3 * i], z, pp, n, ambient);
                for (int c = 0; c < 3; ++c) rgb[c] = render_channel(base[c], I);
            } else {
                for (int c = 0; c < 3; ++c) rgb[c] = bg ? bg[3 * i + c] : 0;
            }
            for (int k = 0; radius > 0.f && k < K; ++k)
                if (render_marker(kv[k], (float)x, (float)y, radius)) {
                    for (int c = 0; c < 3; ++c) rgb[c] = mc[c];
                    break;
                }
            for (int c = 0; c < 3; ++c) img[3 * i + c] = rgb[c];
        }
    (void)N;
}

// Coverage of every sample by the triangles faces [F,3] over screen vertices sv [N,4] (u, v, z, pad): count[H,W] the triangles
// whose render_tri_setup / render_cover accept the sample, face[H,W] the last of them (-1: none)
extern "C" void render_count_host(int F, const float* sv, const int* faces, int W, int H, int* count, int* face) {
    const RVert* p = reinterpret_cast<const RVert*>(sv);
    for (int i = 0; i < W * H; ++i) { count[i] = 0; face[i] = -1; }
    for (int t = 0; t < F; ++t) {
        const int id[3] = {faces[3 * t], faces[3 * t + 1], faces[3 * t + 2]};
        const RVert q[3] = {p[id[0]], p[id[1]], p[id[2]]};
        RTri tri;
        if (!render_tri_setup(q, id, t, W, H, tri)) continue;
        for (int y = (int)tri.y0; y <= (int)tri.y1; ++y)
            for (int x = (int)tri.x0; x <= (int)tri.x1; ++x) {
                double w[3];
                if (!render_cover(tri, (float)x, (float)y, w)) continue;
                ++count[(size_t)y * W + x];
                face[(size_t)y * W + x] = t;
            }
    }
}
