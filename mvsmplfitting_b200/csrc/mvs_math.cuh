// Scalar building blocks of the multi-view SMPL fitting closure and their
// hand-derived adjoints.  Every function is __host__ __device__ so the CUDA kernels
// and the CPU host-simulation test (tests/hostsim) execute the SAME arithmetic.
//
// Conventions (they follow the reference, cited as file:line of /root/reference/code):
//   * 3x3 matrices are row-major float[9]; a rigid transform is [Gam | g] (3x3 + 3).
//   * Rodrigues uses angle = ||r + 1e-8|| (epsilon added to every component) and the
//     direction r / angle without epsilon                      (smplx/lbs.py:284-285)
//   * the root rotation block is multiplied by `scale`          (smplx/lbs.py:348)
#pragma once
#include <math.h>

#if defined(__CUDACC__)
#define MVS_HD __host__ __device__ __forceinline__
#define MVS_DIST_FN __host__ __device__ __noinline__
#else
#define MVS_HD inline
#define MVS_DIST_FN inline
#endif

namespace mvs {

constexpr int kJoints = 24;
constexpr int kBetas = 10;
constexpr int kPoseBasis = 207;              // 23 * 9
constexpr int kFeat = kPoseBasis + kBetas + 1;  // [pose_feature | betas | 1] = 218
constexpr int kFeatPad = 224;                // padded K of the blend-shape contraction
constexpr int kParams = 86;                  // betas10 | global_orient3 | body_pose69 | transl3 | scale1
constexpr int kOffBetas = 0, kOffOrient = 10, kOffPose = 13, kOffTransl = 82, kOffScale = 85;
constexpr int kMaxKeypoints = 32;
constexpr int kMaxViews = 16;

MVS_HD float mvs_sin(float x) { return sinf(x); }
MVS_HD float mvs_cos(float x) { return cosf(x); }
MVS_HD float mvs_sqrt(float x) { return sqrtf(x); }
MVS_HD float mvs_exp(float x) { return expf(x); }
MVS_HD double mvs_sin(double x) { return sin(x); }
MVS_HD double mvs_cos(double x) { return cos(x); }
MVS_HD double mvs_sqrt(double x) { return sqrt(x); }
MVS_HD double mvs_exp(double x) { return exp(x); }

// ---------------------------------------------------------------- small linear algebra
template <class T> MVS_HD void mat3_mul(const T* A, const T* B, T* C) {       // C = A B
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c)
            C[3 * r + c] = A[3 * r] * B[c] + A[3 * r + 1] * B[3 + c] + A[3 * r + 2] * B[6 + c];
}
template <class T> MVS_HD void mat3_mul_nt(const T* A, const T* B, T* C) {    // C = A B^T
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c)
            C[3 * r + c] = A[3 * r] * B[3 * c] + A[3 * r + 1] * B[3 * c + 1] + A[3 * r + 2] * B[3 * c + 2];
}
template <class T> MVS_HD void mat3_mul_tn(const T* A, const T* B, T* C) {    // C = A^T B
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c)
            C[3 * r + c] = A[r] * B[c] + A[3 + r] * B[3 + c] + A[6 + r] * B[6 + c];
}
template <class T> MVS_HD void mat3_vec(const T* A, const T* x, T* y) {       // y = A x
#pragma unroll
    for (int r = 0; r < 3; ++r) y[r] = A[3 * r] * x[0] + A[3 * r + 1] * x[1] + A[3 * r + 2] * x[2];
}
template <class T> MVS_HD void mat3_tvec(const T* A, const T* x, T* y) {      // y = A^T x
#pragma unroll
    for (int r = 0; r < 3; ++r) y[r] = A[r] * x[0] + A[3 + r] * x[1] + A[6 + r] * x[2];
}

// ---------------------------------------------------------------- VPoser rotation head (model/VPoser.py)
// One joint of VPoser.decode(z, 'aa') after the last linear layer: the 6 outputs o[0..5] -> continuous rotation
// representation -> rotation matrix (ContinousRotReprDecoder, VPoser.py:161-174) -> quaternion
// (rotation_matrix_to_quaternion, VPoser.py:29-98, on the TRANSPOSED matrix, four branches, eps 1e-6) -> axis-angle
// (quaternion_to_angle_axis, VPoser.py:101-156).  view(-1, 3, 2): a1 = (o0, o2, o4), a2 = (o1, o3, o5).
MVS_HD float mvs_atan2(float y, float x) { return atan2f(y, x); }
MVS_HD double mvs_atan2(double y, double x) { return atan2(y, x); }

template <class T> struct Cont6dState {      // intermediates shared by the forward pass and its adjoint
    T a1[3], a2[3], n1, b1[3], d, u[3], n2, b2[3], b3[3];
    int branch;                               // which of the four quaternion formulas was selected
    T qs[4], tsel, q[4], sin2, sn, k, tt;
};

template <class T> MVS_HD void cont6d_to_aa_fwd(const T* o, T* aa, Cont6dState<T>& S) {
#pragma unroll
    for (int i = 0; i < 3; ++i) { S.a1[i] = o[2 * i]; S.a2[i] = o[2 * i + 1]; }
    const T l1 = mvs_sqrt(S.a1[0] * S.a1[0] + S.a1[1] * S.a1[1] + S.a1[2] * S.a1[2]);
    S.n1 = l1 > T(1e-12) ? l1 : T(1e-12);                     // F.normalize: x / max(|x|, eps)
#pragma unroll
    for (int i = 0; i < 3; ++i) S.b1[i] = S.a1[i] / S.n1;
    S.d = S.b1[0] * S.a2[0] + S.b1[1] * S.a2[1] + S.b1[2] * S.a2[2];
#pragma unroll
    for (int i = 0; i < 3; ++i) S.u[i] = S.a2[i] - S.d * S.b1[i];
    const T l2 = mvs_sqrt(S.u[0] * S.u[0] + S.u[1] * S.u[1] + S.u[2] * S.u[2]);
    S.n2 = l2 > T(1e-12) ? l2 : T(1e-12);
#pragma unroll
    for (int i = 0; i < 3; ++i) S.b2[i] = S.u[i] / S.n2;
    S.b3[0] = S.b1[1] * S.b2[2] - S.b1[2] * S.b2[1];
    S.b3[1] = S.b1[2] * S.b2[0] - S.b1[0] * S.b2[2];
    S.b3[2] = S.b1[0] * S.b2[1] - S.b1[1] * S.b2[0];
    // R = [b1 b2 b3] (columns); the quaternion routine works on rt = R^T, whose ROWS are b1, b2, b3
    const T* r0 = S.b1; const T* r1 = S.b2; const T* r2 = S.b3;
    const T m00 = r0[0], m11 = r1[1], m22 = r2[2];
    const bool d2 = m22 < T(1e-6), d0_d1 = m00 > m11, d0_nd1 = m00 < -m11;
    if (d2 && d0_d1) {
        S.branch = 0; S.tsel = T(1) + m00 - m11 - m22;
        S.qs[0] = r1[2] - r2[1]; S.qs[1] = S.tsel; S.qs[2] = r0[1] + r1[0]; S.qs[3] = r2[0] + r0[2];
    } else if (d2) {
        S.branch = 1; S.tsel = T(1) - m00 + m11 - m22;
        S.qs[0] = r2[0] - r0[2]; S.qs[1] = r0[1] + r1[0]; S.qs[2] = S.tsel; S.qs[3] = r1[2] + r2[1];
    } else if (d0_nd1) {
        S.branch = 2; S.tsel = T(1) - m00 - m11 + m22;
        S.qs[0] = r0[1] - r1[0]; S.qs[1] = r2[0] + r0[2]; S.qs[2] = r1[2] + r2[1]; S.qs[3] = S.tsel;
    } else {
        S.branch = 3; S.tsel = T(1) + m00 + m11 + m22;
        S.qs[0] = S.tsel; S.qs[1] = r1[2] - r2[1]; S.qs[2] = r2[0] - r0[2]; S.qs[3] = r0[1] - r1[0];
    }
    const T isq = T(0.5) / mvs_sqrt(S.tsel);
#pragma unroll
    for (int i = 0; i < 4; ++i) S.q[i] = S.qs[i] * isq;
    S.sin2 = S.q[1] * S.q[1] + S.q[2] * S.q[2] + S.q[3] * S.q[3];
    S.sn = mvs_sqrt(S.sin2);
    const T cs = S.q[0];
    S.tt = T(2) * (cs < T(0) ? mvs_atan2(-S.sn, -cs) : mvs_atan2(S.sn, cs));
    S.k = S.sin2 > T(0) ? S.tt / S.sn : T(2);
    aa[0] = S.q[1] * S.k; aa[1] = S.q[2] * S.k; aa[2] = S.q[3] * S.k;
}

// d_o[0..5] = (d aa / d o)^T d_aa for the state left by cont6d_to_aa_fwd (branch selections are locally constant)
template <class T> MVS_HD void cont6d_to_aa_bwd(const Cont6dState<T>& S, const T* daa, T* d_o) {
    T dq[4] = {T(0), daa[0] * S.k, daa[1] * S.k, daa[2] * S.k};
    if (S.sin2 > T(0)) {
        const T dk = daa[0] * S.q[1] + daa[1] * S.q[2] + daa[2] * S.q[3];
        const T dtt = dk / S.sn;
        T dsn = -dk * S.tt / S.sin2;
        const T cs = S.q[0], r2 = S.sin2 + cs * cs;
        dsn += T(2) * dtt * cs / r2;                          // tt = 2 atan2(+-sn, +-cs): same partials in both branches
        dq[0] += -T(2) * dtt * S.sn / r2;
        const T dsin2 = dsn / (T(2) * S.sn);
        dq[1] += T(2) * S.q[1] * dsin2; dq[2] += T(2) * S.q[2] * dsin2; dq[3] += T(2) * S.q[3] * dsin2;
    }
    // q = 0.5 qs / sqrt(t)
    const T isq = T(0.5) / mvs_sqrt(S.tsel);
    T dqs[4];
    T dt = T(0);
#pragma unroll
    for (int i = 0; i < 4; ++i) { dqs[i] = dq[i] * isq; dt += dq[i] * S.q[i]; }
    dt = -T(0.5) * dt / S.tsel;
    T dr0[3] = {T(0), T(0), T(0)}, dr1[3] = {T(0), T(0), T(0)}, dr2[3] = {T(0), T(0), T(0)};   // d rows of rt = d b1, b2, b3
    if (S.branch == 0) {
        dt += dqs[1];
        dr1[2] += dqs[0]; dr2[1] -= dqs[0]; dr0[1] += dqs[2]; dr1[0] += dqs[2]; dr2[0] += dqs[3]; dr0[2] += dqs[3];
        dr0[0] += dt; dr1[1] -= dt; dr2[2] -= dt;
    } else if (S.branch == 1) {
        dt += dqs[2];
        dr2[0] += dqs[0]; dr0[2] -= dqs[0]; dr0[1] += dqs[1]; dr1[0] += dqs[1]; dr1[2] += dqs[3]; dr2[1] += dqs[3];
        dr0[0] -= dt; dr1[1] += dt; dr2[2] -= dt;
    } else if (S.branch == 2) {
        dt += dqs[3];
        dr0[1] += dqs[0]; dr1[0] -= dqs[0]; dr2[0] += dqs[1]; dr0[2] += dqs[1]; dr1[2] += dqs[2]; dr2[1] += dqs[2];
        dr0[0] -= dt; dr1[1] -= dt; dr2[2] += dt;
    } else {
        dt += dqs[0];
        dr1[2] += dqs[1]; dr2[1] -= dqs[1]; dr2[0] += dqs[2]; dr0[2] -= dqs[2]; dr0[1] += dqs[3]; dr1[0] -= dqs[3];
        dr0[0] += dt; dr1[1] += dt; dr2[2] += dt;
    }
    T db1[3] = {dr0[0], dr0[1], dr0[2]}, db2[3] = {dr1[0], dr1[1], dr1[2]};
    const T* db3 = dr2;
    // b3 = b1 x b2
    db1[0] += S.b2[1] * db3[2] - S.b2[2] * db3[1]; db1[1] += S.b2[2] * db3[0] - S.b2[0] * db3[2]; db1[2] += S.b2[0] * db3[1] - S.b2[1] * db3[0];
    db2[0] += db3[1] * S.b1[2] - db3[2] * S.b1[1]; db2[1] += db3[2] * S.b1[0] - db3[0] * S.b1[2]; db2[2] += db3[0] * S.b1[1] - db3[1] * S.b1[0];
    // b2 = u / n2
    T du[3];
    {
        const T pb = S.b2[0] * db2[0] + S.b2[1] * db2[1] + S.b2[2] * db2[2];
        const bool live = S.n2 > T(1e-12);
#pragma unroll
        for (int i = 0; i < 3; ++i) du[i] = live ? (db2[i] - S.b2[i] * pb) / S.n2 : db2[i] / S.n2;
    }
    // u = a2 - d b1,  d = b1 . a2
    T da2[3] = {du[0], du[1], du[2]};
    const T dd = -(du[0] * S.b1[0] + du[1] * S.b1[1] + du[2] * S.b1[2]);
#pragma unroll
    for (int i = 0; i < 3; ++i) { db1[i] += -S.d * du[i] + dd * S.a2[i]; da2[i] += dd * S.b1[i]; }
    // b1 = a1 / n1
    T da1[3];
    {
        const T pb = S.b1[0] * db1[0] + S.b1[1] * db1[1] + S.b1[2] * db1[2];
        const bool live = S.n1 > T(1e-12);
#pragma unroll
        for (int i = 0; i < 3; ++i) da1[i] = live ? (db1[i] - S.b1[i] * pb) / S.n1 : db1[i] / S.n1;
    }
#pragma unroll
    for (int i = 0; i < 3; ++i) { d_o[2 * i] = da1[i]; d_o[2 * i + 1] = da2[i]; }
}

// ---------------------------------------------------------------- Rodrigues (lbs.py:269-300)
template <class T> MVS_HD void rodrigues_fwd(const T* r, T* R) {
    const T e = T(1e-8);
    const T ax = r[0] + e, ay = r[1] + e, az = r[2] + e;
    const T a = mvs_sqrt(ax * ax + ay * ay + az * az);
    const T x = r[0] / a, y = r[1] / a, z = r[2] / a;
    const T s = mvs_sin(a), c1 = T(1) - mvs_cos(a);
    // K = [0 -z y; z 0 -x; -y x 0],  K^2 = k k^T - |k|^2 I  (|k| != 1 exactly because of the shift)
    const T xx = x * x, yy = y * y, zz = z * z;
    R[0] = T(1) + c1 * (-zz - yy);  R[1] = -s * z + c1 * (x * y);  R[2] = s * y + c1 * (x * z);
    R[3] = s * z + c1 * (x * y);    R[4] = T(1) + c1 * (-zz - xx); R[5] = -s * x + c1 * (y * z);
    R[6] = -s * y + c1 * (x * z);   R[7] = s * x + c1 * (y * z);   R[8] = T(1) + c1 * (-yy - xx);
}

// dr += (dR/dr)^T dR   for the expression above
template <class T> MVS_HD void rodrigues_bwd(const T* r, const T* dR, T* dr) {
    const T e = T(1e-8);
    const T ax = r[0] + e, ay = r[1] + e, az = r[2] + e;
    const T a = mvs_sqrt(ax * ax + ay * ay + az * az);
    const T inv_a = T(1) / a;
    const T x = r[0] * inv_a, y = r[1] * inv_a, z = r[2] * inv_a;
    const T s = mvs_sin(a), c = mvs_cos(a), c1 = T(1) - c;
    const T K[9] = {T(0), -z, y, z, T(0), -x, -y, x, T(0)};
    const T xx = x * x, yy = y * y, zz = z * z;
    const T K2[9] = {-zz - yy, x * y, x * z, x * y, -zz - xx, y * z, x * z, y * z, -yy - xx};
    T ds = T(0), dc1 = T(0);
#pragma unroll
    for (int i = 0; i < 9; ++i) { ds += dR[i] * K[i]; dc1 += dR[i] * K2[i]; }
    // gradient w.r.t. the entries of K:  s * dR  +  c1 * (dR K^T + K^T dR)   (Y = K K)
    T t1[9], t2[9], dK[9];
    mat3_mul_nt(dR, K, t1);
    mat3_mul_tn(K, dR, t2);
#pragma unroll
    for (int i = 0; i < 9; ++i) dK[i] = s * dR[i] + c1 * (t1[i] + t2[i]);
    const T dk[3] = {dK[7] - dK[5], dK[2] - dK[6], dK[3] - dK[1]};
    // a enters through sin/cos and through k = r / a
    const T da = ds * c + dc1 * s - (dk[0] * r[0] + dk[1] * r[1] + dk[2] * r[2]) * inv_a * inv_a;
    dr[0] += dk[0] * inv_a + da * ax * inv_a;
    dr[1] += dk[1] * inv_a + da * ay * inv_a;
    dr[2] += dk[2] * inv_a + da * az * inv_a;
}

// ---------------------------------------------------------------- kinematic chain (lbs.py:316-370)
// forward for one non-root joint:  [Gam|g] = [Gp|gp] * [R|rel]
template <class T> MVS_HD void chain_step_fwd(const T* Gp, const T* gp, const T* R, const T* rel, T* Gam, T* g) {
    mat3_mul(Gp, R, Gam);
    T t[3];
    mat3_vec(Gp, rel, t);
    g[0] = t[0] + gp[0]; g[1] = t[1] + gp[1]; g[2] = t[2] + gp[2];
}
// skinning transform A = [Gam | g - Gam J]   (lbs.py:365-368), 12 floats row-major 3x4
template <class T> MVS_HD void make_skin_transform(const T* Gam, const T* g, const T* J, T* A) {
    T t[3];
    mat3_vec(Gam, J, t);
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        A[4 * r] = Gam[3 * r]; A[4 * r + 1] = Gam[3 * r + 1]; A[4 * r + 2] = Gam[3 * r + 2];
        A[4 * r + 3] = g[r] - t[r];
    }
}
// adjoint of make_skin_transform: accumulates into dGam, dg, dJ
template <class T> MVS_HD void skin_transform_bwd(const T* dA, const T* Gam, const T* J, T* dGam, T* dg, T* dJ) {
    const T dt[3] = {dA[3], dA[7], dA[11]};
#pragma unroll
    for (int r = 0; r < 3; ++r) {
#pragma unroll
        for (int c = 0; c < 3; ++c) dGam[3 * r + c] += dA[4 * r + c] - dt[r] * J[c];
        dg[r] += dt[r];
    }
    T t[3];
    mat3_tvec(Gam, dt, t);
    dJ[0] -= t[0]; dJ[1] -= t[1]; dJ[2] -= t[2];
}
// adjoint of chain_step_fwd: given dGam, dg of the child accumulate into the parent's
// dGp, dgp and produce dR (overwritten) and drel (overwritten)
template <class T> MVS_HD void chain_step_bwd(const T* dGam, const T* dg, const T* Gp, const T* R, const T* rel,
                                              T* dGp, T* dgp, T* dR, T* drel) {
    T t[9];
    mat3_mul_nt(dGam, R, t);                      // dGp += dGam R^T + dg rel^T
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) dGp[3 * r + c] += t[3 * r + c] + dg[r] * rel[c];
    mat3_mul_tn(Gp, dGam, dR);                    // dR = Gp^T dGam
    mat3_tvec(Gp, dg, drel);                      // drel = Gp^T dg
    dgp[0] += dg[0]; dgp[1] += dg[1]; dgp[2] += dg[2];
}

// ---------------------------------------------------------------- camera + robust residual
struct CamF { float R[9]; float t[3]; float f[2]; float c[2]; };

// A view's lens distortion (mvs_set_camera_rigs_dist): OpenCV's projectPoints coefficients (k1, k2, p1, p2, k3), two float4
// per view.  Applied to the normalised coordinates (x', y') = (x/z, y/z):
//   r2 = x'^2 + y'^2,  a = 1 + k1 r2 + k2 r2^2 + k3 r2^3
//   x'' = x' a + 2 p1 x'y' + p2 (r2 + 2 x'^2),   y'' = y' a + p1 (r2 + 2 y'^2) + 2 p2 x'y',   uv = f (x'', y'') + c
// No clamp (as OpenCV): the map is only monotone, and a fit only meaningful, inside the calibrated field of view.
struct alignas(16) Dist { float k1, k2, p1, p2, k3, pad[3]; };

// (x', y') -> (x'', y'') and, with J != NULL, the Jacobian J = d(x'', y'')/d(x', y') row-major (it is symmetric: J[1] = J[2])
template <class T> MVS_HD void distort_norm(const Dist& d, T xn, T yn, T* xd, T* yd, T* J = nullptr) {
    const T k1 = T(d.k1), k2 = T(d.k2), k3 = T(d.k3), p1 = T(d.p1), p2 = T(d.p2);
    const T r2 = xn * xn + yn * yn, xy = xn * yn;
    const T a = T(1) + r2 * (k1 + r2 * (k2 + r2 * k3));
    *xd = xn * a + T(2) * p1 * xy + p2 * (r2 + T(2) * xn * xn);
    *yd = yn * a + p1 * (r2 + T(2) * yn * yn) + T(2) * p2 * xy;
    if (J) {
        const T da = k1 + r2 * (T(2) * k2 + T(3) * k3 * r2);        // d a / d r2
        J[0] = a + T(2) * xn * xn * da + T(2) * p1 * yn + T(6) * p2 * xn;
        J[1] = T(2) * xy * da + T(2) * p1 * xn + T(2) * p2 * yn;
        J[2] = J[1];
        J[3] = a + T(2) * yn * yn * da + T(6) * p1 * yn + T(2) * p2 * xn;
    }
}

// The distorted halves of project_fwd / project_bwd_x, kept out of line on the device: the pinhole path of the kernels that
// call them keeps its own register allocation, and the distorted path pays a call.
template <class T> struct Pair { T a, b; };
template <class T> MVS_DIST_FN Pair<T> distort_px(const Dist* d, T x0, T x1, T x2) {
    Pair<T> o;
    distort_norm(*d, x0 / x2, x1 / x2, &o.a, &o.b);
    return o;
}
// (J^T g) / z: the adjoint of (x0, x1) through the divide's numerators, g = d loss / d(x'', y'')
template <class T> MVS_DIST_FN Pair<T> distort_px_adjoint(const Dist* d, T x0, T x1, T x2, T g0, T g1) {
    T xd, yd, J[4];
    distort_norm(*d, x0 / x2, x1 / x2, &xd, &yd, J);
    const T iz = T(1) / x2;
    return Pair<T>{(J[0] * g0 + J[2] * g1) * iz, (J[1] * g0 + J[3] * g1) * iz};
}

// camera.py:93-117 : x = R q + t ; uv = f * x.xy / x.z + c        (no clamp)
// dist != NULL: uv = f * distort(x.xy / x.z) + c.  dist == NULL evaluates exactly the pinhole expressions.
template <class T, class C> MVS_HD void project_fwd(const C& cam, const T* q, T* x, T* uv, const Dist* dist = nullptr) {
    const T R0 = cam.R[0], R1 = cam.R[1], R2 = cam.R[2], R3 = cam.R[3], R4 = cam.R[4], R5 = cam.R[5],
            R6 = cam.R[6], R7 = cam.R[7], R8 = cam.R[8];
    x[0] = R0 * q[0] + R1 * q[1] + R2 * q[2] + T(cam.t[0]);
    x[1] = R3 * q[0] + R4 * q[1] + R5 * q[2] + T(cam.t[1]);
    x[2] = R6 * q[0] + R7 * q[1] + R8 * q[2] + T(cam.t[2]);
    if (dist) {
        const Pair<T> d = distort_px(dist, x[0], x[1], x[2]);
        uv[0] = d.a * T(cam.f[0]) + T(cam.c[0]);
        uv[1] = d.b * T(cam.f[1]) + T(cam.c[1]);
        return;
    }
    uv[0] = (x[0] / x[2]) * T(cam.f[0]) + T(cam.c[0]);
    uv[1] = (x[1] / x[2]) * T(cam.f[1]) + T(cam.c[1]);
}
// dx = the camera-space adjoint of the projection: duv through f, the distortion's Jacobian (transposed) when dist != NULL,
// and the perspective divide
template <class T, class C> MVS_HD void project_bwd_x(const C& cam, const T* x, const T* duv, T* dx, const Dist* dist = nullptr) {
    const T iz = T(1) / x[2];
    if (dist) {
        const Pair<T> d = distort_px_adjoint(dist, x[0], x[1], x[2], duv[0] * T(cam.f[0]), duv[1] * T(cam.f[1]));
        dx[0] = d.a;
        dx[1] = d.b;
    } else {
        dx[0] = duv[0] * T(cam.f[0]) * iz;
        dx[1] = duv[1] * T(cam.f[1]) * iz;
    }
    dx[2] = -(dx[0] * x[0] + dx[1] * x[1]) * iz;
}
// dq += R^T dx, with dx the adjoint of the projection (project_bwd_x)
template <class T, class C> MVS_HD void project_bwd(const C& cam, const T* x, const T* duv, T* dq, const Dist* dist = nullptr) {
    T dx[3];
    project_bwd_x(cam, x, duv, dx, dist);
    const T dx0 = dx[0], dx1 = dx[1], dx2 = dx[2];
    dq[0] += T(cam.R[0]) * dx0 + T(cam.R[3]) * dx1 + T(cam.R[6]) * dx2;
    dq[1] += T(cam.R[1]) * dx0 + T(cam.R[4]) * dx1 + T(cam.R[7]) * dx2;
    dq[2] += T(cam.R[2]) * dx0 + T(cam.R[5]) * dx1 + T(cam.R[8]) * dx2;
}

// ---------------------------------------------------------------- camera refinement (mvs_refine_cameras, DESIGN.md section 4)
// A refined view's camera from its update (w, c):  R = Rod(w) R0,  t = Rod(w) (t0 - R0 dC),  i.e.  x_cam = Rod(w) (R0 (q - dC) + t0).
// Rod(w) = I + D,  D = A K + B K^2,  K = [w]x,  A = sin th / th,  B = (1 - cos th) / th^2,  th = |w|  (series below th^2 = 0.1),
// so D = 0 exactly at w = 0 (rodrigues_fwd's +1e-8 shift is not).  dC is the camera-centre update: c itself for a free view; for
// the view that keeps its distance r to view 0 (sphere), dC = (E u - n (s - 1)) / s with u = (c0, c1), s = sqrt(1 + |u|^2),
// E = r [e1 e2] and n = r d (d: unit vector from view 0's centre to this one's, e1, e2 orthonormal and normal to it): the new
// centre is view 0's + r (d + e1 u0 + e2 u1) / s.  Every entry adds its increment to the calibrated one, and an increment that
// is zero keeps the calibrated bits (a -0 entry stays -0): at w = c = 0 the camera IS (R0, t0).
struct CamRefine {
    float R0[9], t0[3];
    float E[6];                       // [3][2] row-major (sphere only)
    float n[3];                       // (sphere only)
    int sphere;
};

template <class T> struct CamDeltaState { T K[9], K2[9], D[9], p[3], a[3], A, B, dA, dB, s, nu, m; };

// A, B and their derivatives with respect to th2 = th^2
template <class T> MVS_HD void rotvec_coeffs(T th2, T* A, T* B, T* dA, T* dB) {
    if (th2 < T(0.1)) {
        *A = T(1) + th2 * (T(-1) / T(6) + th2 * (T(1) / T(120) + th2 * (T(-1) / T(5040))));
        *B = T(0.5) + th2 * (T(-1) / T(24) + th2 * (T(1) / T(720) + th2 * (T(-1) / T(40320))));
        *dA = T(-1) / T(6) + th2 * (T(1) / T(60) + th2 * (T(-1) / T(1680) + th2 * (T(1) / T(90720))));
        *dB = T(-1) / T(24) + th2 * (T(1) / T(360) + th2 * (T(-1) / T(13440) + th2 * (T(1) / T(907200))));
    } else {
        const T th = mvs_sqrt(th2), s = mvs_sin(th), c = mvs_cos(th);
        *A = s / th;
        *B = (T(1) - c) / th2;
        *dA = (th * c - s) / (T(2) * th2 * th);
        *dB = (th * s - T(2) * (T(1) - c)) / (T(2) * th2 * th2);
    }
}

template <class T> MVS_HD T add_increment(float base, T inc) { return inc == T(0) ? T(base) : T(base) + inc; }

template <class T> MVS_HD void cam_from_delta(const CamRefine& cr, const T* w, const T* c, T* R, T* t, CamDeltaState<T>& S) {
    const T th2 = w[0] * w[0] + w[1] * w[1] + w[2] * w[2];
    rotvec_coeffs(th2, &S.A, &S.B, &S.dA, &S.dB);
    const T K[9] = {T(0), -w[2], w[1], w[2], T(0), -w[0], -w[1], w[0], T(0)};
#pragma unroll
    for (int i = 0; i < 9; ++i) S.K[i] = K[i];
    mat3_mul(S.K, S.K, S.K2);
#pragma unroll
    for (int i = 0; i < 9; ++i) S.D[i] = S.A * S.K[i] + S.B * S.K2[i];
    T dC[3];
    if (cr.sphere) {
        S.nu = c[0] * c[0] + c[1] * c[1];
        S.s = mvs_sqrt(T(1) + S.nu);
        S.m = S.nu / (S.s + T(1));                                     // s - 1 without the cancellation
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            S.a[i] = T(cr.E[2 * i]) * c[0] + T(cr.E[2 * i + 1]) * c[1] - T(cr.n[i]) * S.m;
            dC[i] = S.a[i] / S.s;
        }
    } else {
        dC[0] = c[0]; dC[1] = c[1]; dC[2] = c[2];
    }
    T R0[9], wv[3], Dp[3], RD[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) R0[i] = T(cr.R0[i]);
    mat3_mul(S.D, R0, RD);
#pragma unroll
    for (int i = 0; i < 9; ++i) R[i] = add_increment(cr.R0[i], RD[i]);
    mat3_vec(R0, dC, wv);
#pragma unroll
    for (int i = 0; i < 3; ++i) S.p[i] = T(cr.t0[i]) - wv[i];
    mat3_vec(S.D, S.p, Dp);
#pragma unroll
    for (int i = 0; i < 3; ++i) t[i] = add_increment(cr.t0[i], Dp[i] - wv[i]);
}

// (gw, gc) = the adjoint of cam_from_delta for the camera's adjoint (dR, dt); gc[2] = 0 for a sphere view
template <class T> MVS_HD void cam_from_delta_bwd(const CamRefine& cr, const T* w, const T* c, const CamDeltaState<T>& S,
                                                  const T* dR, const T* dt, T* gw, T* gc) {
    T R0[9], dD[9], t1[9], t2[9], dp[3], dwv[3], ddC[3];
#pragma unroll
    for (int i = 0; i < 9; ++i) R0[i] = T(cr.R0[i]);
    mat3_mul_nt(dR, R0, dD);                                           // R = R0 + D R0
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int k = 0; k < 3; ++k) dD[3 * r + k] += dt[r] * S.p[k];   // t = t0 - R0 dC + D p
    mat3_tvec(S.D, dt, dp);
#pragma unroll
    for (int i = 0; i < 3; ++i) dwv[i] = -dt[i] - dp[i];
    mat3_tvec(R0, dwv, ddC);
    // D = A K + B K K
    T dA = T(0), dB = T(0);
#pragma unroll
    for (int i = 0; i < 9; ++i) { dA += dD[i] * S.K[i]; dB += dD[i] * S.K2[i]; }
    mat3_mul_nt(dD, S.K, t1);
    mat3_mul_tn(S.K, dD, t2);
    T dK[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) dK[i] = S.A * dD[i] + S.B * (t1[i] + t2[i]);
    const T dth2 = dA * S.dA + dB * S.dB;
    gw[0] = dK[7] - dK[5] + T(2) * w[0] * dth2;
    gw[1] = dK[2] - dK[6] + T(2) * w[1] * dth2;
    gw[2] = dK[3] - dK[1] + T(2) * w[2] * dth2;
    if (cr.sphere) {
        // dC = a / s,  a = E u - n m,  m = nu / (s + 1),  s = sqrt(1 + nu),  nu = |u|^2
        T da[3], ds = T(0), dm = T(0);
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            da[i] = ddC[i] / S.s;
            ds -= ddC[i] * S.a[i] / (S.s * S.s);
            dm -= T(cr.n[i]) * da[i];
        }
        const T sp1 = S.s + T(1);
        T dnu = dm / sp1;
        ds -= dm * S.nu / (sp1 * sp1);
        dnu += ds / (T(2) * S.s);
        gc[0] = T(cr.E[0]) * da[0] + T(cr.E[2]) * da[1] + T(cr.E[4]) * da[2] + T(2) * c[0] * dnu;
        gc[1] = T(cr.E[1]) * da[0] + T(cr.E[3]) * da[1] + T(cr.E[5]) * da[2] + T(2) * c[1] * dnu;
        gc[2] = T(0);
    } else {
        gc[0] = ddC[0]; gc[1] = ddC[1]; gc[2] = ddC[2];
    }
}

// GMoF (utils/utils.py:427-438): rho^2 e^2 / (e^2 + rho^2) ; returns value, *dval = d/de
template <class T> MVS_HD T gmof(T e, T rho2, T* dval) {
    const T sq = e * e, den = sq + rho2;
    *dval = T(2) * rho2 * rho2 * e / (den * den);
    return rho2 * (sq / den);
}

}  // namespace mvs
