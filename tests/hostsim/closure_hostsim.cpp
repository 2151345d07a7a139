// TEST INFRASTRUCTURE -- serial host execution of the SAME scalar building blocks the CUDA
// kernels use (mvsmplfitting_b200/csrc/mvs_math.cuh), wired together in the same data flow
// (Phi.Qk contraction, ELL skinning, sparse keypoints, strip-free adjoint).  It lets the CPU
// test-suite check the hand-derived gradient against the oracle's autograd in float and double
// without a GPU.  It is not shipped and not a fallback: the product library never links it.
#include <stdlib.h>
#include <string.h>
#include <vector>

#include "../../mvsmplfitting_b200/csrc/mvs_math.cuh"
#include "../../mvsmplfitting_b200/csrc/mvs_init.cuh"
#include "../../mvsmplfitting_b200/csrc/mvs_sdf_bins.cuh"
#include <vector>

using namespace mvs;

template <class T> struct HostModel {
    int N, K, V;
    std::vector<T> Q;        // [3N][218]
    std::vector<T> Jt, JS;   // [72], [720]
    int parents[24];
    std::vector<T> W;        // [N][24]
    std::vector<int> kp_ptr, kp_v, kp_chain;
    std::vector<T> kp_w;
    CamF cam[kMaxViews];
};

struct HostLoss {
    double data_weight, body_pose_weight, shape_weight, bending_prior_weight, rho;
    int body_prior, use_conf, fix_shape, M;
};

template <class T>
static void run(const HostModel<T>& m, const HostLoss& lp, const double* gmm_means, const double* gmm_prec,
                const double* gmm_lognllw, const double* x86, const double* gt_uv, const double* conf,
                const double* jw, double* loss_out, double* grad_out, double* joints_out, double* verts_out) {
    const int N = m.N, K = m.K, V = m.V;
    T x[kParams];
    for (int i = 0; i < kParams; ++i) x[i] = (T)x86[i];
    // ---- pose forward
    T R[24][9], J[24][3], Gam[24][9], g[24][3], A[24][12];
    for (int j = 0; j < 24; ++j) rodrigues_fwd(&x[kOffOrient + 3 * j], R[j]);
    for (int jc = 0; jc < 72; ++jc) {
        T a = m.Jt[jc];
        for (int l = 0; l < kBetas; ++l) a += m.JS[jc * kBetas + l] * x[l];
        J[jc / 3][jc % 3] = a;
    }
    const T sc = x[kOffScale];
    for (int i = 0; i < 9; ++i) Gam[0][i] = sc * R[0][i];
    for (int c = 0; c < 3; ++c) g[0][c] = J[0][c];
    for (int j = 1; j < 24; ++j) {
        const int p = m.parents[j];
        T rel[3] = {J[j][0] - J[p][0], J[j][1] - J[p][1], J[j][2] - J[p][2]};
        chain_step_fwd(Gam[p], g[p], R[j], rel, Gam[j], g[j]);
    }
    for (int j = 0; j < 24; ++j) make_skin_transform(Gam[j], g[j], J[j], A[j]);
    std::vector<T> Phi(kFeat);
    for (int k = 0; k < kPoseBasis; ++k) Phi[k] = R[1 + k / 9][k % 9] - (((k % 9) % 4 == 0) ? T(1) : T(0));
    for (int l = 0; l < kBetas; ++l) Phi[kPoseBasis + l] = x[l];
    Phi[kFeat - 1] = T(1);
    // ---- vertices
    std::vector<T> vp((size_t)N * 3), v((size_t)N * 3);
    for (int col = 0; col < 3 * N; ++col) {
        T a = 0;
        const T* q = &m.Q[(size_t)col * kFeat];
        for (int k = 0; k < kFeat; ++k) a += Phi[k] * q[k];
        vp[col] = a;
    }
    for (int n = 0; n < N; ++n) {
        T Tm[12] = {0};
        for (int j = 0; j < 24; ++j) {
            const T w = m.W[(size_t)n * 24 + j];
            if (w != T(0)) for (int c = 0; c < 12; ++c) Tm[c] += w * A[j][c];
        }
        for (int r = 0; r < 3; ++r)
            v[3 * n + r] = Tm[4 * r] * vp[3 * n] + Tm[4 * r + 1] * vp[3 * n + 1] + Tm[4 * r + 2] * vp[3 * n + 2] + Tm[4 * r + 3];
    }
    if (verts_out) for (int i = 0; i < 3 * N; ++i) verts_out[i] = (double)(v[i] + x[kOffTransl + i % 3]);
    // ---- keypoints, projection, data term
    std::vector<T> q((size_t)K * 3), dq((size_t)K * 3, T(0));
    for (int k = 0; k < K; ++k) {
        T a[3] = {0, 0, 0};
        for (int e = m.kp_ptr[k]; e < m.kp_ptr[k + 1]; ++e)
            for (int c = 0; c < 3; ++c) a[c] += m.kp_w[e] * v[3 * m.kp_v[e] + c];
        if (m.kp_chain[k] >= 0) for (int c = 0; c < 3; ++c) a[c] += g[m.kp_chain[k]][c];
        for (int c = 0; c < 3; ++c) { q[3 * k + c] = a[c] + x[kOffTransl + c]; if (joints_out) joints_out[3 * k + c] = (double)q[3 * k + c]; }
    }
    const T rho2 = (T)(lp.rho * lp.rho), dw2 = (T)(lp.data_weight * lp.data_weight);
    T data = 0;
    for (int vv = 0; vv < V; ++vv) {
        T s = 0;
        for (int k = 0; k < K; ++k) {
            T xc[3], uv[2];
            project_fwd(m.cam[vv], &q[3 * k], xc, uv);
            T w = (T)jw[k];
            if (lp.use_conf) w *= (T)conf[vv * K + k];
            const T w2 = w * w;
            T d0, d1;
            const T g0 = gmof((T)gt_uv[(vv * K + k) * 2] - uv[0], rho2, &d0);
            const T g1 = gmof((T)gt_uv[(vv * K + k) * 2 + 1] - uv[1], rho2, &d1);
            s += w2 * g0 + w2 * g1;
            const T duv[2] = {-(w2 * d0) * dw2, -(w2 * d1) * dw2};
            project_bwd(m.cam[vv], xc, duv, &dq[3 * k]);
        }
        data += s * dw2;
    }
    // ---- adjoint
    T grad[kParams] = {0};
    std::vector<T> dv((size_t)N * 3, T(0));
    T dgch[24][3] = {{0}};
    for (int k = 0; k < K; ++k) {
        for (int c = 0; c < 3; ++c) grad[kOffTransl + c] += dq[3 * k + c];
        for (int e = m.kp_ptr[k]; e < m.kp_ptr[k + 1]; ++e)
            for (int c = 0; c < 3; ++c) dv[3 * m.kp_v[e] + c] += m.kp_w[e] * dq[3 * k + c];
        if (m.kp_chain[k] >= 0) for (int c = 0; c < 3; ++c) dgch[m.kp_chain[k]][c] += dq[3 * k + c];
    }
    T dA[24][12] = {{0}};
    std::vector<T> dPhi(kFeat, T(0));
    for (int n = 0; n < N; ++n) {
        const T d[3] = {dv[3 * n], dv[3 * n + 1], dv[3 * n + 2]};
        if (d[0] == T(0) && d[1] == T(0) && d[2] == T(0)) continue;
        T G[9] = {0};
        for (int j = 0; j < 24; ++j) {
            const T w = m.W[(size_t)n * 24 + j];
            if (w == T(0)) continue;
            for (int r = 0; r < 3; ++r) {
                for (int c = 0; c < 3; ++c) { G[3 * r + c] += w * A[j][4 * r + c]; dA[j][4 * r + c] += w * d[r] * vp[3 * n + c]; }
                dA[j][4 * r + 3] += w * d[r];
            }
        }
        T dvp[3];
        mat3_tvec(G, d, dvp);
        for (int c = 0; c < 3; ++c) {
            const T* qq = &m.Q[(size_t)(3 * n + c) * kFeat];
            for (int k = 0; k < kFeat; ++k) dPhi[k] += dvp[c] * qq[k];
        }
    }
    T dGam[24][9] = {{0}}, dg[24][3], dJ[24][3] = {{0}}, dR[24][9] = {{0}};
    for (int j = 0; j < 24; ++j) for (int c = 0; c < 3; ++c) dg[j][c] = dgch[j][c];
    for (int j = 0; j < 24; ++j) skin_transform_bwd(dA[j], Gam[j], J[j], dGam[j], dg[j], dJ[j]);
    for (int j = 23; j >= 1; --j) {
        const int p = m.parents[j];
        T rel[3] = {J[j][0] - J[p][0], J[j][1] - J[p][1], J[j][2] - J[p][2]}, drel[3];
        chain_step_bwd(dGam[j], dg[j], Gam[p], R[j], rel, dGam[p], dg[p], dR[j], drel);
        for (int c = 0; c < 3; ++c) { dJ[j][c] += drel[c]; dJ[p][c] -= drel[c]; }
    }
    T ds = 0;
    for (int i = 0; i < 9; ++i) { dR[0][i] = sc * dGam[0][i]; ds += dGam[0][i] * R[0][i]; }
    for (int c = 0; c < 3; ++c) dJ[0][c] += dg[0][c];
    grad[kOffScale] = ds;
    for (int k = 0; k < kPoseBasis; ++k) dR[1 + k / 9][k % 9] += dPhi[k];
    for (int j = 0; j < 24; ++j) rodrigues_bwd(&x[kOffOrient + 3 * j], dR[j], &grad[kOffOrient + 3 * j]);
    for (int l = 0; l < kBetas; ++l) {
        T a = dPhi[kPoseBasis + l];
        for (int jc = 0; jc < 72; ++jc) a += m.JS[jc * kBetas + l] * dJ[jc / 3][jc % 3];
        grad[l] = a;
    }
    // ---- priors (fitting.py:327-350)
    const T bpw = (T)lp.body_pose_weight, bpw2 = bpw * bpw;
    const T* th = &x[kOffPose];
    T pprior = 0, gs = bpw2;
    std::vector<T> ybest(69, T(0));
    if (lp.body_prior == 1) {
        T best = (T)3e38;
        for (int mm = 0; mm < lp.M; ++mm) {
            T diff[69], y[69], qd = 0;
            for (int i = 0; i < 69; ++i) diff[i] = th[i] - (T)gmm_means[mm * 69 + i];
            for (int i = 0; i < 69; ++i) {
                T a = 0;
                for (int j = 0; j < 69; ++j) a += (T)gmm_prec[((size_t)mm * 69 + j) * 69 + i] * diff[j];
                y[i] = a; qd += a * diff[i];
            }
            const T ll = T(0.5) * qd - (T)gmm_lognllw[mm];
            if (ll < best) { best = ll; for (int i = 0; i < 69; ++i) ybest[i] = y[i]; }
        }
        pprior = best * bpw2;
    } else if (lp.body_prior == 0) {
        T a = 0;
        for (int i = 0; i < 69; ++i) { a += th[i] * th[i]; ybest[i] = T(2) * th[i]; }
        pprior = a * bpw2;
    }
    if (pprior > T(5e4)) { pprior = 0; gs = 0; }
    T a2 = 0;
    for (int i = 0; i < 69; ++i) a2 += th[i] * th[i];
    const T w4 = (bpw * T(4)) * (bpw * T(4));
    for (int i = 0; i < 69; ++i) grad[kOffPose + i] += T(2) * th[i] * w4 + gs * ybest[i];
    T shape = 0;
    if (!lp.fix_shape) {
        const T sw2 = (T)(lp.shape_weight * lp.shape_weight);
        for (int l = 0; l < kBetas; ++l) { shape += x[l] * x[l]; grad[l] += T(2) * x[l] * sw2; }
        shape *= sw2;
    }
    const int idx[4] = {52, 55, 9, 12};
    const T sg[4] = {1, -1, -1, -1};
    T angle = 0, ev[4];
    for (int i = 0; i < 4; ++i) { const T e = mvs_exp(th[idx[i]] * sg[i]); ev[i] = e * e; angle += ev[i]; }
    angle *= (T)lp.bending_prior_weight;
    T ga = (T)lp.bending_prior_weight;
    if (angle > T(1e4)) { angle = 0; ga = 0; }
    for (int i = 0; i < 4; ++i) grad[kOffPose + idx[i]] += T(2) * sg[i] * ev[i] * ga;
    *loss_out = (double)(data + (pprior + a2 * w4) + shape + angle);
    for (int i = 0; i < kParams; ++i) grad_out[i] = (double)grad[i];
}

template <class T>
static void build(HostModel<T>& m, int N, const double* v_template, const double* shapedirs, const double* posedirs,
                  const double* J_regressor, const int* parents, const double* W, int K, const int* kp_ptr,
                  const int* kp_v, const double* kp_w, const int* kp_chain, int V, const double* cR, const double* ct,
                  const double* cf, const double* cc) {
    m.N = N; m.K = K; m.V = V;
    m.Q.assign((size_t)3 * N * kFeat, T(0));
    for (int col = 0; col < 3 * N; ++col) {
        for (int k = 0; k < kPoseBasis; ++k) m.Q[(size_t)col * kFeat + k] = (T)posedirs[(size_t)k * 3 * N + col];
        for (int l = 0; l < kBetas; ++l) m.Q[(size_t)col * kFeat + kPoseBasis + l] = (T)shapedirs[(size_t)col * kBetas + l];
        m.Q[(size_t)col * kFeat + kFeat - 1] = (T)v_template[col];
    }
    m.Jt.assign(72, T(0)); m.JS.assign(720, T(0));
    for (int j = 0; j < 24; ++j)
        for (int c = 0; c < 3; ++c) {
            double a = 0, al[kBetas] = {0};
            for (int n = 0; n < N; ++n) {
                const double w = J_regressor[(size_t)j * N + n];
                if (w == 0) continue;
                a += w * v_template[3 * n + c];
                for (int l = 0; l < kBetas; ++l) al[l] += w * shapedirs[((size_t)3 * n + c) * kBetas + l];
            }
            m.Jt[3 * j + c] = (T)a;
            for (int l = 0; l < kBetas; ++l) m.JS[(3 * j + c) * kBetas + l] = (T)al[l];
        }
    memcpy(m.parents, parents, sizeof(int) * 24);
    m.W.resize((size_t)N * 24);
    for (size_t i = 0; i < (size_t)N * 24; ++i) m.W[i] = (T)W[i];
    m.kp_ptr.assign(kp_ptr, kp_ptr + K + 1);
    m.kp_v.assign(kp_v, kp_v + kp_ptr[K]);
    m.kp_chain.assign(kp_chain, kp_chain + K);
    m.kp_w.resize(kp_ptr[K]);
    for (int e = 0; e < kp_ptr[K]; ++e) m.kp_w[e] = (T)kp_w[e];
    for (int v = 0; v < V; ++v) {
        for (int i = 0; i < 9; ++i) m.cam[v].R[i] = (float)cR[9 * v + i];
        for (int i = 0; i < 3; ++i) m.cam[v].t[i] = (float)ct[3 * v + i];
        for (int i = 0; i < 2; ++i) { m.cam[v].f[i] = (float)cf[2 * v + i]; m.cam[v].c[i] = (float)cc[2 * v + i]; }
    }
}

extern "C" {
struct Handle { HostModel<float> f; HostModel<double> d; };

void* hostsim_create(int N, const double* v_template, const double* shapedirs, const double* posedirs,
                     const double* J_regressor, const int* parents, const double* W, int K, const int* kp_ptr,
                     const int* kp_v, const double* kp_w, const int* kp_chain, int V, const double* cR,
                     const double* ct, const double* cf, const double* cc) {
    Handle* h = new Handle();
    build(h->f, N, v_template, shapedirs, posedirs, J_regressor, parents, W, K, kp_ptr, kp_v, kp_w, kp_chain, V, cR, ct, cf, cc);
    build(h->d, N, v_template, shapedirs, posedirs, J_regressor, parents, W, K, kp_ptr, kp_v, kp_w, kp_chain, V, cR, ct, cf, cc);
    return h;
}
void hostsim_destroy(void* h) { delete (Handle*)h; }
void hostsim_eval(void* hv, int use_double, const HostLoss* lp, const double* gmm_means, const double* gmm_prec,
                  const double* gmm_lognllw, const double* x86, const double* gt_uv, const double* conf, const double* jw,
                  double* loss, double* grad, double* joints, double* verts) {
    Handle* h = (Handle*)hv;
    if (use_double) run(h->d, *lp, gmm_means, gmm_prec, gmm_lognllw, x86, gt_uv, conf, jw, loss, grad, joints, verts);
    else run(h->f, *lp, gmm_means, gmm_prec, gmm_lognllw, x86, gt_uv, conf, jw, loss, grad, joints, verts);
}
// cont6d_to_aa_fwd / _bwd of mvs_math.cuh on n six-vectors: aa[n][3], d_o[n][6] = (d aa/d o)^T daa, branch[n]
void hostsim_cont6d(int n, int use_double, const double* o6, const double* daa, double* aa, double* d_o, int* branch) {
    for (int i = 0; i < n; ++i) {
        if (use_double) {
            mvs::Cont6dState<double> S; double a[3], g[6];
            mvs::cont6d_to_aa_fwd<double>(o6 + 6 * i, a, S);
            mvs::cont6d_to_aa_bwd<double>(S, daa + 3 * i, g);
            for (int k = 0; k < 3; ++k) aa[3 * i + k] = a[k];
            for (int k = 0; k < 6; ++k) d_o[6 * i + k] = g[k];
            branch[i] = S.branch;
        } else {
            mvs::Cont6dState<float> S; float o[6], d[3], a[3], g[6];
            for (int k = 0; k < 6; ++k) o[k] = (float)o6[6 * i + k];
            for (int k = 0; k < 3; ++k) d[k] = (float)daa[3 * i + k];
            mvs::cont6d_to_aa_fwd<float>(o, a, S);
            mvs::cont6d_to_aa_bwd<float>(S, d, g);
            for (int k = 0; k < 3; ++k) aa[3 * i + k] = a[k];
            for (int k = 0; k < 6; ++k) d_o[6 * i + k] = g[k];
            branch[i] = S.branch;
        }
    }
}
// mvs_init.cuh on the host.  cams: R [V,9], t [V,3], f [V,2], c [V,2]; uv [V,K,2], conf [V,K] -> X [K,3]
struct HostCamSet { int num_views; CamF cam[kMaxViews]; };
void hostsim_triangulate(int V, int K, const double* cR, const double* ct, const double* cf, const double* cc,
                         const float* uv, const float* conf, int use_double, double* X) {
    HostCamSet cs; cs.num_views = V;
    for (int v = 0; v < V; ++v) {
        for (int i = 0; i < 9; ++i) cs.cam[v].R[i] = (float)cR[9 * v + i];
        for (int i = 0; i < 3; ++i) cs.cam[v].t[i] = (float)ct[3 * v + i];
        for (int i = 0; i < 2; ++i) { cs.cam[v].f[i] = (float)cf[2 * v + i]; cs.cam[v].c[i] = (float)cc[2 * v + i]; }
    }
    for (int k = 0; k < K; ++k) {
        if (use_double) {
            triangulate_point<double>(cs, uv + 2 * k, conf + k, 2L * K, (long)K, X + 3 * k);
        } else {
            float x[3];
            triangulate_point<float>(cs, uv + 2 * k, conf + k, 2L * K, (long)K, x);
            for (int i = 0; i < 3; ++i) X[3 * k + i] = x[i];
        }
    }
}
// returns 1 if a transform was found.  src, dst [n,3]; R [9] row-major, t [3], scale [1], aa [3] = rotmat_to_aa(R)
int hostsim_umeyama(int n, const double* src, const double* dst, int estimate_scale, int use_double, double* R, double* t,
                    double* scale, double* aa, int as_written) {
    if (use_double) {
        if (!umeyama_fit<double>(src, dst, n, estimate_scale != 0, R, t, scale, as_written != 0)) return 0;
        rotmat_to_aa<double>(R, aa);
        return 1;
    }
    float s[51], d[51], Rf[9], tf[3], sf, af[3];
    for (int i = 0; i < 3 * n; ++i) { s[i] = (float)src[i]; d[i] = (float)dst[i]; }
    if (!umeyama_fit<float>(s, d, n, estimate_scale != 0, Rf, tf, &sf, as_written != 0)) return 0;
    rotmat_to_aa<float>(Rf, af);
    for (int i = 0; i < 9; ++i) R[i] = Rf[i];
    for (int i = 0; i < 3; ++i) { t[i] = tf[i]; aa[i] = af[i]; }
    *scale = sf;
    return 1;
}
// init_guess.py:54-78 on the host: cam (R [9], t [3], f [2], c [2]), rest [K,3], uv [K,2], conf [K] -> joints3d [K,3]
void hostsim_single_view(int K, const double* cR, const double* ct, const double* cf, const double* cc, const double* rest,
                         const float* uv, const float* conf, double* X) {
    CamF cam;
    for (int i = 0; i < 9; ++i) cam.R[i] = (float)cR[i];
    for (int i = 0; i < 3; ++i) cam.t[i] = (float)ct[i];
    for (int i = 0; i < 2; ++i) { cam.f[i] = (float)cf[i]; cam.c[i] = (float)cc[i]; }
    const double d = single_view_depth<double>(cam, rest, uv, conf);
    for (int k = 0; k < K; ++k)
        for (int c = 0; c < 3; ++c) X[3 * k + c] = rest[3 * k + c] + d * (double)cam.R[6 + c];
}
void hostsim_rotmat_to_aa(int n, const double* R, double* aa) {
    for (int i = 0; i < n; ++i) rotmat_to_aa<double>(R + 9 * i, aa + 3 * i);
}

// mvs_sdf_bins.cuh on the host: the frame's bin structures built serially (what sdf_bins_kernel does with a counting sort),
// then phi at the listed voxels over the candidate lists AND by brute force over all F triangles with the same primitives.
// tri [F][9] box coordinates; vox [n] flat voxel ids (i + G (j + G k)); out_b / out_f [n]; evals [2] totals; returns 0, or 1 / 2
// if a list capacity would overflow.
int hostsim_sdf_bins(int F, const float* tri, int G, long n, const long* vox, float* out_b, float* out_f, long* evals) {
    std::vector<int> cell_cnt(kBinCells + 1, 0), ray_cnt(kBinRays + 1, 0);
    float mn[2] = {3e38f, 3e38f}, mx[2] = {-3e38f, -3e38f};
    for (int f = 0; f < F; ++f) {
        float a[2], b[2];
        tri_proj_box(tri + 9 * f, a, b);
        for (int q = 0; q < 2; ++q) { mn[q] = fminf(mn[q], a[q]); mx[q] = fmaxf(mx[q], b[q]); }
    }
    SdfBinsView v;
    ray_bin_frame(mn, mx, v.s_lo, v.s_scale);
    for (int f = 0; f < F; ++f) {
        int lo[3], hi[3];
        tri_cell_range(tri + 9 * f, lo, hi);
        for (int x = lo[0]; x <= hi[0]; ++x) for (int y = lo[1]; y <= hi[1]; ++y) for (int z = lo[2]; z <= hi[2]; ++z)
            cell_cnt[(x * kBinC + y) * kBinC + z + 1]++;
        float a[2], b[2];
        int rl[2], rh[2];
        tri_proj_box(tri + 9 * f, a, b);
        tri_ray_range(a, b, v.s_lo, v.s_scale, rl, rh);
        for (int x = rl[0]; x <= rh[0]; ++x) for (int y = rl[1]; y <= rh[1]; ++y) ray_cnt[x * kBinR + y + 1]++;
    }
    for (int i = 0; i < kBinCells; ++i) cell_cnt[i + 1] += cell_cnt[i];
    for (int i = 0; i < kBinRays; ++i) ray_cnt[i + 1] += ray_cnt[i];
    evals[0] = evals[1] = 0; evals[2] = cell_cnt[kBinCells]; evals[3] = ray_cnt[kBinRays];
    if (cell_cnt[kBinCells] > kBinCapD) return 1;
    if (ray_cnt[kBinRays] > kBinCapR) return 2;
    std::vector<unsigned short> cell_idx(cell_cnt[kBinCells] + 1), ray_idx(ray_cnt[kBinRays] + 1);
    std::vector<int> cc(cell_cnt.begin(), cell_cnt.end()), rc(ray_cnt.begin(), ray_cnt.end());
    for (int f = F - 1; f >= 0; --f) {               // any order inside a bin: min and parity do not depend on it
        int lo[3], hi[3];
        tri_cell_range(tri + 9 * f, lo, hi);
        for (int x = lo[0]; x <= hi[0]; ++x) for (int y = lo[1]; y <= hi[1]; ++y) for (int z = lo[2]; z <= hi[2]; ++z)
            cell_idx[cc[(x * kBinC + y) * kBinC + z]++] = (unsigned short)f;
        float a[2], b[2];
        int rl[2], rh[2];
        tri_proj_box(tri + 9 * f, a, b);
        tri_ray_range(a, b, v.s_lo, v.s_scale, rl, rh);
        for (int x = rl[0]; x <= rh[0]; ++x) for (int y = rl[1]; y <= rh[1]; ++y) ray_idx[rc[x * kBinR + y]++] = (unsigned short)f;
    }
    v.tri = tri; v.cell_ptr = cell_cnt.data(); v.cell_idx = cell_idx.data(); v.ray_ptr = ray_cnt.data(); v.ray_idx = ray_idx.data();
    for (long q = 0; q < n; ++q) {
        const long id = vox[q];
        float c[3];
        voxel_centre((int)(id % G), (int)((id / G) % G), (int)(id / ((long)G * G)), G, c);
        int ev[2] = {0, 0};
        out_b[q] = phi_binned(c, v, ev);
        evals[0] += ev[0]; evals[1] += ev[1];
        if (out_f) {
            int hits = 0;
            float min_d = 1000.f;
            for (int f = 0; f < F; ++f) {
                const float* p = tri + 9 * f;
                const float dd = triangle_distance(c, p, p + 3, p + 6);
                if (dd < min_d) min_d = dd;
                if (ray_hits(c, p, p + 3, p + 6)) ++hits;
            }
            out_f[q] = (hits % 2 == 0) ? 0.f : min_d;
        }
    }
    return 0;
}
}
