// Per-pixel arithmetic of the mesh rasteriser (mvs_render.cu, DESIGN.md section 4d).  Every function is MVS_HD, so the kernels and
// the host build of tests/hostsim/render_hostsim.cpp run the same expressions.
//
// Conventions:
//   * pixel (column x, row y) is sampled at (u, v) = (x, y), OpenCV's convention;
//   * edge k of a triangle is the one opposite its vertex k;
//   * an edge is evaluated with its endpoints in ascending vertex-id order, in double, without contraction, so the two triangles
//     that share it compute the same value and see each sample on opposite sides (watertight); a sample exactly on it belongs to
//     the triangle whose interior lies below the edge (image y down), whatever the edge's slope, or to its right when the edge is
//     vertical.  That is the same as moving every sample down by an infinitesimal step and right by a much smaller one, so among
//     the faces around a vertex or along an edge exactly one owns the sample.
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>

#include "mvs_math.cuh"

namespace mvs {

constexpr int kRenderTile = 16;              // screen tile edge (px): one raster CTA of 256 threads per tile
constexpr float kRenderNear = 1e-3f;         // a triangle with a vertex at camera depth <= this is not drawn

// a vertex on one view's screen: pixel position and camera depth
struct alignas(16) RVert { float u, v, z, pad; };

// what the raster loop needs of one triangle: each edge's canonical endpoints, the sign that makes the edge function positive
// inside, which edges own the samples on them, the vertex depths, the covered sample box
struct RTri {
    float ax[3], ay[3], bx[3], by[3];
    float s[3];
    float z[3];
    float x0, x1, y0, y1;
    int own;
    int face;
};

MVS_HD double render_mul(double a, double b) {
#ifdef __CUDA_ARCH__
    return __dmul_rn(a, b);
#else
    return a * b;
#endif
}

// canonical edge function of the edge a -> b at sample (px, py)
MVS_HD double render_edge(float ax, float ay, float bx, float by, double px, double py) {
    const double l = render_mul((double)bx - (double)ax, py - (double)ay);
    const double r = render_mul((double)by - (double)ay, px - (double)ax);
    return l - r;
}

// The samples a triangle may cover, clamped to the image: columns [*x0, *x1], rows [*y0, *y1].  false: not drawn (a vertex at or
// before the near plane or not finite, or no sample of the image inside its bounding box).
MVS_HD bool render_tri_box(const RVert& p0, const RVert& p1, const RVert& p2, int W, int H, int* x0, int* x1, int* y0, int* y1) {
    if (!(p0.z > kRenderNear && p1.z > kRenderNear && p2.z > kRenderNear)) return false;
    const float lx = fminf(p0.u, fminf(p1.u, p2.u)), hx = fmaxf(p0.u, fmaxf(p1.u, p2.u));
    const float ly = fminf(p0.v, fminf(p1.v, p2.v)), hy = fmaxf(p0.v, fmaxf(p1.v, p2.v));
    if (!(isfinite(lx) && isfinite(hx) && isfinite(ly) && isfinite(hy))) return false;
    const float cx0 = ceilf(fmaxf(lx, 0.f)), cx1 = floorf(fminf(hx, (float)(W - 1)));
    const float cy0 = ceilf(fmaxf(ly, 0.f)), cy1 = floorf(fminf(hy, (float)(H - 1)));
    if (!(cx0 <= cx1 && cy0 <= cy1)) return false;
    *x0 = (int)cx0; *x1 = (int)cx1; *y0 = (int)cy0; *y1 = (int)cy1;
    return true;
}

// Set-up of face `face` with vertex ids id[3] and screen vertices p[3].  false: the triangle covers no sample (near plane, not
// finite, no sample in its box, or zero area).
MVS_HD bool render_tri_setup(const RVert* p, const int* id, int face, int W, int H, RTri& t) {
    int x0, x1, y0, y1;
    if (!render_tri_box(p[0], p[1], p[2], W, H, &x0, &x1, &y0, &y1)) return false;
    float sig[3];
    for (int k = 0; k < 3; ++k) {
        const int jj = (k + 1) % 3, ll = (k + 2) % 3;   // edge k in winding order: 1 -> 2, 2 -> 0, 0 -> 1
        if (id[jj] == id[ll]) return false;
        const int a = id[jj] < id[ll] ? jj : ll, b = a == jj ? ll : jj;
        sig[k] = a == jj ? 1.f : -1.f;
        t.ax[k] = p[a].u; t.ay[k] = p[a].v; t.bx[k] = p[b].u; t.by[k] = p[b].v;
    }
    // orientation: the directed edge 0 -> 1 (edge 2) at vertex 2
    const double o = (double)sig[2] * render_edge(t.ax[2], t.ay[2], t.bx[2], t.by[2], (double)p[2].u, (double)p[2].v);
    if (!(o != 0.0)) return false;
    const float sa = o > 0.0 ? 1.f : -1.f;
    t.own = 0;
    for (int k = 0; k < 3; ++k) {
        t.s[k] = sig[k] * sa;
        const float gy = t.s[k] * (t.bx[k] - t.ax[k]), gx = -t.s[k] * (t.by[k] - t.ay[k]);   // inward normal of the edge
        if (gy > 0.f || (gy == 0.f && gx > 0.f)) t.own |= 1 << k;
        t.z[k] = p[k].z;
    }
    t.x0 = (float)x0; t.x1 = (float)x1; t.y0 = (float)y0; t.y1 = (float)y1;
    t.face = face;
    return true;
}

// Coverage of sample (px, py): true when it is inside or on an owned edge; w[k] >= 0 are the edge functions (barycentric weights
// up to their sum).
MVS_HD bool render_cover(const RTri& t, float px, float py, double* w) {
    for (int k = 0; k < 3; ++k) {
        w[k] = (double)t.s[k] * render_edge(t.ax[k], t.ay[k], t.bx[k], t.by[k], (double)px, (double)py);
        if (w[k] < 0.0 || (w[k] == 0.0 && !(t.own >> k & 1))) return false;
    }
    return w[0] + w[1] + w[2] > 0.0;
}

// perspective-correct depth z = 1 / sum_i lam_i / z_i and the screen barycentrics lam
MVS_HD float render_depth(const RTri& t, const double* w, float* lam) {
    const double sw = w[0] + w[1] + w[2];
    double iz = 0.0;
    for (int k = 0; k < 3; ++k) {
        const double l = w[k] / sw;
        lam[k] = (float)l;
        iz += l / (double)t.z[k];
    }
    return (float)(1.0 / iz);
}

// visibility key: the smallest wins; depth > 0, so its bits order as the floats do, and ties go to the lower face
MVS_HD unsigned long long render_key(float z, int face) {
    unsigned u;
    memcpy(&u, &z, sizeof(u));
    return (unsigned long long)u << 32 | (unsigned)face;
}

// Headlight intensity at a covered sample: perspective-correct weights w_i ~ lam_i / z_i of the camera-space vertex positions
// p[i] and normals n[i]; n = normalize(sum w_i n_i), l = -p / |p| at p = sum w_i p_i, I = ambient + (1 - ambient) max(0, n.l)
MVS_HD float render_intensity(const float* lam, const float* z, const float (*p)[3], const float (*n)[3], float ambient) {
    float w[3], sw = 0.f;
    for (int k = 0; k < 3; ++k) { w[k] = lam[k] / z[k]; sw += w[k]; }
    float N[3], P[3];
    for (int c = 0; c < 3; ++c) {
        N[c] = (w[0] * n[0][c] + w[1] * n[1][c] + w[2] * n[2][c]) / sw;
        P[c] = (w[0] * p[0][c] + w[1] * p[1][c] + w[2] * p[2][c]) / sw;
    }
    const float nl = sqrtf(N[0] * N[0] + N[1] * N[1] + N[2] * N[2]), pl = sqrtf(P[0] * P[0] + P[1] * P[1] + P[2] * P[2]);
    float d = 0.f;
    if (nl > 0.f && pl > 0.f) d = -(N[0] * P[0] + N[1] * P[1] + N[2] * P[2]) / (nl * pl);
    return ambient + (1.f - ambient) * fmaxf(0.f, d);
}

// one channel of a shaded pixel: min(255, floor(255 base I + 1/2))
MVS_HD unsigned char render_channel(float base, float I) {
    const float v = floorf(255.f * base * I + 0.5f);
    return v >= 255.f ? (unsigned char)255 : (unsigned char)v;
}

// a keypoint's marker disc covers sample (px, py): the keypoint is in front of the camera and within r of the sample
MVS_HD bool render_marker(const RVert& k, float px, float py, float r) {
    if (!(k.z > kRenderNear)) return false;
    const float dx = px - k.u, dy = py - k.v;
    return dx * dx + dy * dy <= r * r;
}

// camera-space vertex normal from the (unnormalised) sum of its faces' cross products in world space: R normalize(s), 0 when s = 0
MVS_HD void render_normal(const float* R, const float* s, float* n) {
    const float l = sqrtf(s[0] * s[0] + s[1] * s[1] + s[2] * s[2]);
    if (!(l > 0.f)) { n[0] = n[1] = n[2] = 0.f; return; }
    const float u[3] = {s[0] / l, s[1] / l, s[2] / l};
    mat3_vec(R, u, n);
}

}  // namespace mvs
