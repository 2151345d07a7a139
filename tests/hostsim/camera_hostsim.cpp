// Host build of the camera-refinement block of mvs_math.cuh (cam_from_delta and its adjoint), in float and double
// (tests/test_hostsim_camera.py).
#include <cstring>

#include "../../mvsmplfitting_b200/csrc/mvs_math.cuh"

using namespace mvs;

static CamRefine make(const float* R0, const float* t0, const float* E, const float* n, int sphere) {
    CamRefine c;
    std::memset(&c, 0, sizeof(c));
    std::memcpy(c.R0, R0, sizeof(c.R0));
    std::memcpy(c.t0, t0, sizeof(c.t0));
    if (sphere) {
        std::memcpy(c.E, E, sizeof(c.E));
        std::memcpy(c.n, n, sizeof(c.n));
    }
    c.sphere = sphere;
    return c;
}

template <class T> static void fwd(const float* R0, const float* t0, const float* E, const float* n, int sphere, const T* w,
                                   const T* c, T* R, T* t) {
    CamDeltaState<T> S;
    cam_from_delta(make(R0, t0, E, n, sphere), w, c, R, t, S);
}

template <class T> static void bwd(const float* R0, const float* t0, const float* E, const float* n, int sphere, const T* w,
                                   const T* c, const T* dR, const T* dt, T* gw, T* gc) {
    const CamRefine cr = make(R0, t0, E, n, sphere);
    CamDeltaState<T> S;
    T R[9], t[3];
    cam_from_delta(cr, w, c, R, t, S);
    cam_from_delta_bwd(cr, w, c, S, dR, dt, gw, gc);
}

extern "C" {
void cam_fwd_f(const float* R0, const float* t0, const float* E, const float* n, int sphere, const float* w, const float* c,
               float* R, float* t) { fwd(R0, t0, E, n, sphere, w, c, R, t); }
void cam_fwd_d(const float* R0, const float* t0, const float* E, const float* n, int sphere, const double* w, const double* c,
               double* R, double* t) { fwd(R0, t0, E, n, sphere, w, c, R, t); }
void cam_bwd_f(const float* R0, const float* t0, const float* E, const float* n, int sphere, const float* w, const float* c,
               const float* dR, const float* dt, float* gw, float* gc) { bwd(R0, t0, E, n, sphere, w, c, dR, dt, gw, gc); }
void cam_bwd_d(const float* R0, const float* t0, const float* E, const float* n, int sphere, const double* w, const double* c,
               const double* dR, const double* dt, double* gw, double* gc) { bwd(R0, t0, E, n, sphere, w, c, dR, dt, gw, gc); }
}
