// Scalar building blocks of the per-frame initial guess (SURVEY §8f row N2): triangulation of the keypoints from V
// views, similarity alignment of the model's rest joints to them, rotation matrix -> axis-angle.
// __host__ __device__ like mvs_math.cuh: tests/hostsim runs the same arithmetic on the CPU.
//
// Reference (file:line of /root/reference/code):
//   * triangulation            utils/recompute3D.py:24-61  (as written, incl. the float32 rounding of AtA at :52)
//   * similarity alignment     utils/umeyama.py:18-109     -> by default the PUBLISHED algorithm (Umeyama, PAMI 1991,
//                              eq. 38-43) that file says it restates.  Its own full-rank branch multiplies by the
//                              transpose of numpy's V^H (:67); that product depends on the sign convention of the LAPACK
//                              build.  umeyama_fit(as_written = true) evaluates the file's expression with a fixed sign
//                              convention.  See oracle/init_oracle.py.
//   * single-view depth guess  utils/init_guess.py:54-78
//   * matrix -> axis-angle     cv2.Rodrigues as called at utils/init_guess.py:86
//   * torso joints, scale      utils/init_guess.py:80-93
#pragma once
#include "mvs_math.cuh"

namespace mvs {

MVS_HD float mvs_acos(float x) { return acosf(x); }
MVS_HD double mvs_acos(double x) { return acos(x); }
MVS_HD float mvs_abs(float x) { return fabsf(x); }
MVS_HD double mvs_abs(double x) { return fabs(x); }

// One view's contribution to the normal equations of "the point closest to all viewing rays" (recompute3D.py:42-50):
//   n = normalize(K^-1 (u, v, 1)),  P = R^T (I - n n^T),  AtA += w P R,  Atb += -w P t,  w = conf + 1e-6
// AtA is accumulated row-major in M[9], Atb in b[3].
template <class T, class C> MVS_HD void ray_normal_eq(const C& cam, T u, T v, T conf, T* M, T* b) {
    T n[3] = {(u - T(cam.c[0])) / T(cam.f[0]), (v - T(cam.c[1])) / T(cam.f[1]), T(1)};
    const T inv = T(1) / mvs_sqrt(n[0] * n[0] + n[1] * n[1] + n[2] * n[2]);
    n[0] *= inv; n[1] *= inv; n[2] *= inv;
    const T w = conf + T(1e-6);
    T Q[9];                                           // I - n n^T
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) Q[3 * i + j] = (i == j ? T(1) : T(0)) - n[i] * n[j];
    T P[9];                                           // R^T Q
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j)
            P[3 * i + j] = T(cam.R[i]) * Q[j] + T(cam.R[3 + i]) * Q[3 + j] + T(cam.R[6 + i]) * Q[6 + j];
#pragma unroll
    for (int i = 0; i < 3; ++i) {
#pragma unroll
        for (int j = 0; j < 3; ++j)
            M[3 * i + j] += w * (P[3 * i] * T(cam.R[j]) + P[3 * i + 1] * T(cam.R[3 + j]) + P[3 * i + 2] * T(cam.R[6 + j]));
        b[i] -= w * (P[3 * i] * T(cam.t[0]) + P[3 * i + 1] * T(cam.t[1]) + P[3 * i + 2] * T(cam.t[2]));
    }
}

// A detection (u, v) of a view with lens distortion d, taken to the ideal (pinhole) pixel that project_fwd without distortion
// would give: invert (x', y') -> (x'', y'') (mvs_math.cuh distort_norm) by kUndistortSteps Newton steps from (x'', y'') with the
// 2x2 Jacobian.  A fixed count, no convergence test: every thread runs the same steps (deterministic).  Converges inside the
// monotone region of the map (the calibrated field of view).
constexpr int kUndistortSteps = 10;
template <class T, class C> MVS_HD void undistort_px(const C& cam, const Dist& d, T u, T v, T* uu, T* vu) {
    const T fx = T(cam.f[0]), fy = T(cam.f[1]), cx = T(cam.c[0]), cy = T(cam.c[1]);
    const T xd = (u - cx) / fx, yd = (v - cy) / fy;
    T xn = xd, yn = yd;
    for (int it = 0; it < kUndistortSteps; ++it) {
        T ex, ey, J[4];
        distort_norm(d, xn, yn, &ex, &ey, J);
        ex -= xd; ey -= yd;
        const T det = J[0] * J[3] - J[1] * J[2];
        xn -= (J[3] * ex - J[1] * ey) / det;
        yn -= (J[0] * ey - J[2] * ex) / det;
    }
    *uu = xn * fx + cx;
    *vu = yn * fy + cy;
}

// x = M^-1 b for a 3x3 system, Gaussian elimination with partial pivoting (what np.linalg.solve / LAPACK gesv does)
template <class T> MVS_HD void solve3(const T* M, const T* b, T* x) {
    T a[3][4] = {{M[0], M[1], M[2], b[0]}, {M[3], M[4], M[5], b[1]}, {M[6], M[7], M[8], b[2]}};
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        int p = c;
#pragma unroll
        for (int r = c + 1; r < 3; ++r)
            if (mvs_abs(a[r][c]) > mvs_abs(a[p][c])) p = r;
        if (p != c) {
#pragma unroll
            for (int k = 0; k < 4; ++k) { const T tmp = a[c][k]; a[c][k] = a[p][k]; a[p][k] = tmp; }
        }
#pragma unroll
        for (int r = c + 1; r < 3; ++r) {
            const T f = a[r][c] / a[c][c];
#pragma unroll
            for (int k = c; k < 4; ++k) a[r][k] -= f * a[c][k];
        }
    }
    x[2] = a[2][3] / a[2][2];
    x[1] = (a[1][3] - a[1][2] * x[2]) / a[1][1];
    x[0] = (a[0][3] - a[0][1] * x[1] - a[0][2] * x[2]) / a[0][0];
}

// recompute3D.py:24-61 for ONE keypoint: (u, v) of view w at uv[w * stride_uv + {0, 1}], its confidence at
// conf[w * stride_conf].  CS: anything with .num_views and .cam[w] (R, t, f, c).  X[3] = world point.
// dist [num_views] or NULL (no distortion): a detection with non-zero confidence is undistorted first (undistort_px); one with
// confidence 0 is used as it stands (its weight is 1e-6, and a zero row far outside the field may have no preimage).
template <class T, class CS> MVS_HD void triangulate_point(const CS& cams, const float* uv, const float* conf,
                                                           long stride_uv, long stride_conf, T* X, const Dist* dist = nullptr) {
    T M[9] = {T(0), T(0), T(0), T(0), T(0), T(0), T(0), T(0), T(0)}, b[3] = {T(0), T(0), T(0)};
    for (int w = 0; w < cams.num_views; ++w) {
        T u = T(uv[w * stride_uv]), v = T(uv[w * stride_uv + 1]);
        const float cf = conf[w * stride_conf];
        if (dist && cf != 0.f) undistort_px<T>(cams.cam[w], dist[w], u, v, &u, &v);
        ray_normal_eq<T>(cams.cam[w], u, v, T(cf), M, b);
    }
#pragma unroll
    for (int k = 0; k < 9; ++k) M[k] = T(float(M[k]));        // AtA.astype(np.float32), recompute3D.py:52
    solve3<T>(M, b, X);
}

// Eigen-decomposition of a symmetric 3x3 matrix S (row-major) by cyclic Jacobi rotations: S = V diag(lam) V^T,
// V row-major with the eigenvectors as COLUMNS, det(V) = +1, lam sorted in decreasing order.
template <class T> MVS_HD void jacobi_eig3(const T* S, T* lam, T* V) {
    T a[3][3] = {{S[0], S[1], S[2]}, {S[1], S[4], S[5]}, {S[2], S[5], S[8]}};
    T v[3][3] = {{T(1), T(0), T(0)}, {T(0), T(1), T(0)}, {T(0), T(0), T(1)}};
    for (int sweep = 0; sweep < 12; ++sweep) {
        const T off = mvs_abs(a[0][1]) + mvs_abs(a[0][2]) + mvs_abs(a[1][2]);
        const T diag = mvs_abs(a[0][0]) + mvs_abs(a[1][1]) + mvs_abs(a[2][2]);
        if (off <= T(1e-30) + T(1e-17) * diag) break;
#pragma unroll
        for (int pq = 0; pq < 3; ++pq) {
            const int p = pq == 2 ? 1 : 0, q = pq == 0 ? 1 : 2;
            const T apq = a[p][q];
            if (apq == T(0)) continue;
            const T theta = (a[q][q] - a[p][p]) / (T(2) * apq);
            const T t = (theta >= T(0) ? T(1) : T(-1)) / (mvs_abs(theta) + mvs_sqrt(theta * theta + T(1)));
            const T c = T(1) / mvs_sqrt(t * t + T(1)), s = t * c;
#pragma unroll
            for (int k = 0; k < 3; ++k) {                      // A <- A J
                const T akp = a[k][p], akq = a[k][q];
                a[k][p] = c * akp - s * akq; a[k][q] = s * akp + c * akq;
            }
#pragma unroll
            for (int k = 0; k < 3; ++k) {                      // A <- J^T A
                const T apk = a[p][k], aqk = a[q][k];
                a[p][k] = c * apk - s * aqk; a[q][k] = s * apk + c * aqk;
            }
#pragma unroll
            for (int k = 0; k < 3; ++k) {                      // V <- V J
                const T vkp = v[k][p], vkq = v[k][q];
                v[k][p] = c * vkp - s * vkq; v[k][q] = s * vkp + c * vkq;
            }
        }
    }
    int o[3] = {0, 1, 2};                                      // sort (3 elements): decreasing eigenvalue
    T l[3] = {a[0][0], a[1][1], a[2][2]};
#pragma unroll
    for (int pass = 0; pass < 2; ++pass)
#pragma unroll
        for (int i = 0; i < 2; ++i)
            if (l[o[i]] < l[o[i + 1]]) { const int tmp = o[i]; o[i] = o[i + 1]; o[i + 1] = tmp; }
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        lam[k] = l[o[k]];
#pragma unroll
        for (int i = 0; i < 3; ++i) V[3 * i + k] = v[i][o[k]];
    }
    // a column permutation may have turned V into a reflection: keep det(V) = +1 by negating the last column
    const T det = V[0] * (V[4] * V[8] - V[5] * V[7]) - V[1] * (V[3] * V[8] - V[5] * V[6]) + V[2] * (V[3] * V[7] - V[4] * V[6]);
    if (det < T(0)) { V[2] = -V[2]; V[5] = -V[5]; V[8] = -V[8]; }
}

// Umeyama 1991: least-squares similarity  dst ~ scale * R src + t  over n <= 17 point pairs (src, dst: [n][3]).
// A = dst_c^T src_c / n = U diag(sig) V^T;  R = U diag(1, 1, d) V^T with d = sign(det A)  (eq. 39-40; the rank-2
// rule of eq. 43 gives the same R because only u0, u1 and u0 x u1 enter);  scale = (sig0 + sig1 + d sig2) / var(src)
// (eq. 41-42).  The right singular vectors come from the Jacobi eigen-decomposition of A^T A, u0, u1 from A v / sig
// (re-orthonormalised), so nothing is divided by the smallest singular value (torso points are nearly coplanar).
// Returns false (outputs untouched) if the points are degenerate (rank(A) < 2), umeyama.py:61-62.
//
// as_written = true evaluates what code/utils/umeyama.py computes instead (the `umeyama_as_written` switch of
// mvs_init_config, like sdf_all_faces = 0 for the SDF term):
//   * full rank: rot = U diag(d) (V^H)^T (umeyama.py:67 transposes the V^H numpy.linalg.svd returned).  That product is NOT
//     invariant under the sign freedom of singular pairs (u_i, v_i) -> (-u_i, -v_i), so the file's output depends on the
//     LAPACK build behind numpy; here the pairs are fixed by "the largest-magnitude component of v_i is positive" (the
//     convention oracle/init_oracle.py: svd_sign_normalised applies to numpy's factors).  Rank 2: U V^H as published (:61-66);
//   * the two-candidate patch (:77-107): the rotation with its first two columns negated replaces it when that lowers
//     |scale * rot * src + t - dst|, and -- `rot` being a view of T -- the returned translation is ALWAYS computed from
//     the negated one (:100).
template <class T> MVS_HD bool umeyama_fit(const T* src, const T* dst, int n, bool estimate_scale, T* R, T* t, T* scale,
                                           bool as_written = false) {
    T sm[3] = {T(0), T(0), T(0)}, dm[3] = {T(0), T(0), T(0)};
    for (int i = 0; i < n; ++i)
#pragma unroll
        for (int k = 0; k < 3; ++k) { sm[k] += src[3 * i + k]; dm[k] += dst[3 * i + k]; }
    const T invn = T(1) / T(n);
#pragma unroll
    for (int k = 0; k < 3; ++k) { sm[k] *= invn; dm[k] *= invn; }
    T A[9] = {T(0), T(0), T(0), T(0), T(0), T(0), T(0), T(0), T(0)};
    T var = T(0);
    for (int i = 0; i < n; ++i) {
        T s[3], d[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) { s[k] = src[3 * i + k] - sm[k]; d[k] = dst[3 * i + k] - dm[k]; }
        var += s[0] * s[0] + s[1] * s[1] + s[2] * s[2];
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int c = 0; c < 3; ++c) A[3 * r + c] += d[r] * s[c];
    }
#pragma unroll
    for (int k = 0; k < 9; ++k) A[k] *= invn;
    var *= invn;
    T S[9];                                                    // A^T A
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) S[3 * r + c] = A[r] * A[c] + A[3 + r] * A[3 + c] + A[6 + r] * A[6 + c];
    T lam[3], V[9];
    jacobi_eig3(S, lam, V);
    const T sig0 = mvs_sqrt(lam[0] > T(0) ? lam[0] : T(0)), sig1 = mvs_sqrt(lam[1] > T(0) ? lam[1] : T(0));
    const T sig2 = mvs_sqrt(lam[2] > T(0) ? lam[2] : T(0));
    // numpy matrix_rank tolerance: sig_max * max(M, N) * eps  (umeyama.py:60)
    const T eps = sizeof(T) == 8 ? T(2.220446049250313e-16) : T(1.1920929e-7);
    if (!(sig1 > sig0 * T(3) * eps)) return false;
    T u0[3], u1[3], u2[3];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        u0[r] = (A[3 * r] * V[0] + A[3 * r + 1] * V[3] + A[3 * r + 2] * V[6]) / sig0;
        u1[r] = (A[3 * r] * V[1] + A[3 * r + 1] * V[4] + A[3 * r + 2] * V[7]) / sig1;
    }
    T nrm = T(1) / mvs_sqrt(u0[0] * u0[0] + u0[1] * u0[1] + u0[2] * u0[2]);
#pragma unroll
    for (int r = 0; r < 3; ++r) u0[r] *= nrm;
    const T dot = u0[0] * u1[0] + u0[1] * u1[1] + u0[2] * u1[2];
#pragma unroll
    for (int r = 0; r < 3; ++r) u1[r] -= dot * u0[r];
    nrm = T(1) / mvs_sqrt(u1[0] * u1[0] + u1[1] * u1[1] + u1[2] * u1[2]);
#pragma unroll
    for (int r = 0; r < 3; ++r) u1[r] *= nrm;
    u2[0] = u0[1] * u1[2] - u0[2] * u1[1];
    u2[1] = u0[2] * u1[0] - u0[0] * u1[2];
    u2[2] = u0[0] * u1[1] - u0[1] * u1[0];
    // det(V) = +1, so d * (true u2) = u0 x u1: R = u0 v0^T + u1 v1^T + (u0 x u1) v2^T is a proper rotation
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) R[3 * r + c] = u0[r] * V[3 * c] + u1[r] * V[3 * c + 1] + u2[r] * V[3 * c + 2];
    const T detA = A[0] * (A[4] * A[8] - A[5] * A[7]) - A[1] * (A[3] * A[8] - A[5] * A[6]) + A[2] * (A[3] * A[7] - A[4] * A[6]);
    const T sc = estimate_scale ? (sig0 + sig1 + (detA < T(0) ? -sig2 : sig2)) / var : T(1);
    if (as_written) {
        if (sig2 > sig0 * T(3) * eps) {                        // full rank (numpy matrix_rank, umeyama.py:60,67)
            T f[3];
#pragma unroll
            for (int i = 0; i < 3; ++i) {
                const T a0 = mvs_abs(V[i]), a1 = mvs_abs(V[3 + i]), a2 = mvs_abs(V[6 + i]);
                const T big = (a0 >= a1 && a0 >= a2) ? V[i] : (a1 >= a2 ? V[3 + i] : V[6 + i]);
                f[i] = big < T(0) ? T(-1) : T(1);
            }
            // pairs (f_i u_i, f_i v_i); true u2 = d det(V') (u0' x u1'), so diag(d) leaves f2 (u0 x u1) in the third term;
            // entry (i, c) of the untransposed factor is component i of v_c'
#pragma unroll
            for (int r = 0; r < 3; ++r)
#pragma unroll
                for (int c = 0; c < 3; ++c)
                    R[3 * r + c] = f[c] * (f[0] * u0[r] * V[c] + f[1] * u1[r] * V[3 + c] + f[2] * u2[r] * V[6 + c]);
        }
        T loss[2];
#pragma unroll
        for (int cand = 0; cand < 2; ++cand) {
            const T sg = cand ? T(-1) : T(1);
            T acc = T(0);
            for (int i = 0; i < n; ++i)
#pragma unroll
                for (int r = 0; r < 3; ++r) {
                    const T e = sc * (sg * R[3 * r] * (src[3 * i] - sm[0]) + sg * R[3 * r + 1] * (src[3 * i + 1] - sm[1]) +
                                      R[3 * r + 2] * (src[3 * i + 2] - sm[2])) + dm[r] - dst[3 * i + r];
                    acc += e * e;
                }
            loss[cand] = acc;
        }
#pragma unroll
        for (int r = 0; r < 3; ++r)                            // translation: from the negated candidate, whichever wins
            t[r] = dm[r] - sc * (-R[3 * r] * sm[0] - R[3 * r + 1] * sm[1] + R[3 * r + 2] * sm[2]);
        if (loss[0] > loss[1]) {
#pragma unroll
            for (int r = 0; r < 3; ++r) { R[3 * r] = -R[3 * r]; R[3 * r + 1] = -R[3 * r + 1]; }
        }
        *scale = sc;
        return true;
    }
#pragma unroll
    for (int r = 0; r < 3; ++r) t[r] = dm[r] - sc * (R[3 * r] * sm[0] + R[3 * r + 1] * sm[1] + R[3 * r + 2] * sm[2]);
    *scale = sc;
    return true;
}

// Single-view depth guess (init_guess.py:54-78, as written): the rest joints pushed along the camera's optical axis by
//   est_d = fx * (mean 3-D torso height) / (2-D torso height),
// torso heights: |j5 - j11| and |j6 - j12| in 3-D (rest joints; camera rotation leaves the norms alone), and in 2-D the
// L-shoulder -- L-hip difference taken TWICE (:66 repeats torso2d[0] - torso2d[2]) over the detection rows (u, v, conf),
// i.e. the confidence difference is part of the norm.  joints3d = E^-1 (E j + est_d e_z) = j + est_d * R^T e_z.
// dist != NULL: the view's distortion; the two detections with non-zero confidence are undistorted first (undistort_px).
template <class T, class C> MVS_HD T single_view_depth(const C& cam, const T* rest, const float* uv, const float* conf,
                                                       const Dist* dist = nullptr) {
    T p5[2] = {T(uv[10]), T(uv[11])}, p11[2] = {T(uv[22]), T(uv[23])};
    if (dist && conf[5] != 0.f) undistort_px<T>(cam, *dist, p5[0], p5[1], &p5[0], &p5[1]);
    if (dist && conf[11] != 0.f) undistort_px<T>(cam, *dist, p11[0], p11[1], &p11[0], &p11[1]);
    const T h3 = (mvs_sqrt((rest[15] - rest[33]) * (rest[15] - rest[33]) + (rest[16] - rest[34]) * (rest[16] - rest[34]) +
                           (rest[17] - rest[35]) * (rest[17] - rest[35])) +
                  mvs_sqrt((rest[18] - rest[36]) * (rest[18] - rest[36]) + (rest[19] - rest[37]) * (rest[19] - rest[37]) +
                           (rest[20] - rest[38]) * (rest[20] - rest[38]))) * T(0.5);
    const T du = p5[0] - p11[0], dv = p5[1] - p11[1], dc = T(conf[5]) - T(conf[11]);
    const T h2 = mvs_sqrt(du * du + dv * dv + dc * dc);
    return T(cam.f[0]) * (h3 / h2);
}

// cv2.Rodrigues, 3x3 rotation -> rotation vector (OpenCV calib3d cvRodrigues2, matrix branch; the input is already
// orthonormal here, so its SVD re-orthonormalisation is the identity)
template <class T> MVS_HD void rotmat_to_aa(const T* R, T* r) {
    T v[3] = {R[7] - R[5], R[2] - R[6], R[3] - R[1]};
    const T s = mvs_sqrt((v[0] * v[0] + v[1] * v[1] + v[2] * v[2]) * T(0.25));
    T c = (R[0] + R[4] + R[8] - T(1)) * T(0.5);
    c = c > T(1) ? T(1) : (c < T(-1) ? T(-1) : c);
    const T theta = mvs_acos(c);
    if (s < T(1e-5)) {
        if (c > T(0)) { r[0] = r[1] = r[2] = T(0); return; }
        T t0 = (R[0] + T(1)) * T(0.5), t1 = (R[4] + T(1)) * T(0.5), t2 = (R[8] + T(1)) * T(0.5);
        T rx = mvs_sqrt(t0 > T(0) ? t0 : T(0));
        T ry = mvs_sqrt(t1 > T(0) ? t1 : T(0)) * (R[1] < T(0) ? T(-1) : T(1));
        T rz = mvs_sqrt(t2 > T(0) ? t2 : T(0)) * (R[2] < T(0) ? T(-1) : T(1));
        if (mvs_abs(rx) < mvs_abs(ry) && mvs_abs(rx) < mvs_abs(rz) && ((R[5] > T(0)) != (ry * rz > T(0)))) rz = -rz;
        const T k = theta / mvs_sqrt(rx * rx + ry * ry + rz * rz);
        r[0] = rx * k; r[1] = ry * k; r[2] = rz * k;
        return;
    }
    const T k = theta / (T(2) * s);
    r[0] = v[0] * k; r[1] = v[1] * k; r[2] = v[2] * k;
}

}  // namespace mvs
