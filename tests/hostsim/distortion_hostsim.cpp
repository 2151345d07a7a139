// Host build of the lens-distortion blocks of mvs_math.cuh (project_fwd / project_bwd with coefficients) and mvs_init.cuh
// (undistort_px), in float and double (tests/test_hostsim_distortion.py).  dist == NULL: the pinhole projection.
#include <cstring>

#include "../../mvsmplfitting_b200/csrc/mvs_init.cuh"

using namespace mvs;

static CamF make_cam(const float* R, const float* t, const float* f, const float* c) {
    CamF cam;
    std::memcpy(cam.R, R, sizeof(cam.R));
    std::memcpy(cam.t, t, sizeof(cam.t));
    std::memcpy(cam.f, f, sizeof(cam.f));
    std::memcpy(cam.c, c, sizeof(cam.c));
    return cam;
}

static Dist make_dist(const float* d) { return Dist{d[0], d[1], d[2], d[3], d[4], {0.f, 0.f, 0.f}}; }

// n points q [n][3] -> x [n][3], uv [n][2]
template <class T> static void fwd(const float* R, const float* t, const float* f, const float* c, const float* d, int n, const T* q,
                                   T* x, T* uv) {
    const CamF cam = make_cam(R, t, f, c);
    const Dist dk = d ? make_dist(d) : Dist{};
    for (int i = 0; i < n; ++i) project_fwd(cam, q + 3 * i, x + 3 * i, uv + 2 * i, d ? &dk : nullptr);
}

// n points: dq [n][3] = (d uv / d q)^T duv at the camera-space points x [n][3]
template <class T> static void bwd(const float* R, const float* t, const float* f, const float* c, const float* d, int n, const T* x,
                                   const T* duv, T* dq) {
    const CamF cam = make_cam(R, t, f, c);
    const Dist dk = d ? make_dist(d) : Dist{};
    for (int i = 0; i < n; ++i) {
        dq[3 * i] = dq[3 * i + 1] = dq[3 * i + 2] = T(0);
        project_bwd(cam, x + 3 * i, duv + 2 * i, dq + 3 * i, d ? &dk : nullptr);
    }
}

template <class T> static void undist(const float* f, const float* c, const float* d, int n, const T* uv, T* out) {
    CamF cam;
    std::memset(&cam, 0, sizeof(cam));
    std::memcpy(cam.f, f, sizeof(cam.f));
    std::memcpy(cam.c, c, sizeof(cam.c));
    const Dist dk = make_dist(d);
    for (int i = 0; i < n; ++i) undistort_px<T>(cam, dk, uv[2 * i], uv[2 * i + 1], out + 2 * i, out + 2 * i + 1);
}

extern "C" {
void dist_fwd_f(const float* R, const float* t, const float* f, const float* c, const float* d, int n, const float* q, float* x,
                float* uv) { fwd(R, t, f, c, d, n, q, x, uv); }
void dist_fwd_d(const float* R, const float* t, const float* f, const float* c, const float* d, int n, const double* q, double* x,
                double* uv) { fwd(R, t, f, c, d, n, q, x, uv); }
void dist_bwd_f(const float* R, const float* t, const float* f, const float* c, const float* d, int n, const float* x,
                const float* duv, float* dq) { bwd(R, t, f, c, d, n, x, duv, dq); }
void dist_bwd_d(const float* R, const float* t, const float* f, const float* c, const float* d, int n, const double* x,
                const double* duv, double* dq) { bwd(R, t, f, c, d, n, x, duv, dq); }
void undist_f(const float* f, const float* c, const float* d, int n, const float* uv, float* out) { undist(f, c, d, n, uv, out); }
void undist_d(const float* f, const float* c, const float* d, int n, const double* uv, double* out) { undist(f, c, d, n, uv, out); }
}
