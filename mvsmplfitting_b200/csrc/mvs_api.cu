// C ABI of libmvsmpl.so (see include/mvsmpl.h): context lifetime, one-time uploads with the
// host-side pre-contractions, workspace allocation, and the thin entry points that enqueue the
// kernels of mvs_closure.cu / mvs_lbfgs.cu / mvs_sdf.cu on the caller's stream.
#include <algorithm>
#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include "mvs_internal.cuh"

static std::string g_last_error;

namespace mvs {

int set_error(mvs_ctx* ctx, int code, const char* fmt, ...) {
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    g_last_error = buf;
    if (ctx) ctx->err = buf;
    return code;
}

template <class T> int dev_alloc(mvs_ctx* ctx, T** p, size_t count) {
    void* d = nullptr;
    MVS_CUDA_OK(ctx, cudaMalloc(&d, std::max<size_t>(count, 1) * sizeof(T)));
    ctx->allocs.push_back(d);
    *p = static_cast<T*>(d);
    return MVS_OK;
}
template <class T> int dev_upload(mvs_ctx* ctx, T** p, const T* host, size_t count) {
    int rc = dev_alloc(ctx, p, count);
    if (rc) return rc;
    if (count) MVS_CUDA_OK(ctx, cudaMemcpy(*p, host, count * sizeof(T), cudaMemcpyHostToDevice));
    return MVS_OK;
}
template int dev_alloc<unsigned short>(mvs_ctx*, unsigned short**, size_t);
template int dev_alloc<float>(mvs_ctx*, float**, size_t);
template int dev_alloc<int>(mvs_ctx*, int**, size_t);
template int dev_alloc<double>(mvs_ctx*, double**, size_t);
template int dev_alloc<unsigned char>(mvs_ctx*, unsigned char**, size_t);
template int dev_upload<float>(mvs_ctx*, float**, const float*, size_t);
template int dev_upload<int>(mvs_ctx*, int**, const int*, size_t);

void prof_mark(mvs_ctx* ctx, int kid, cudaStream_t st) {
    Profiler& P = ctx->prof;
    if (P.used[kid] == P.ev[kid].size()) {
        cudaEvent_t e;
        if (cudaEventCreate(&e) != cudaSuccess) return;
        P.ev[kid].push_back(e);
    }
    cudaEventRecord(P.ev[kid][P.used[kid]++], st);
}

__global__ void iota_kernel(int* p, int n, int* na) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = i;
    if (i == 0) *na = n;
}

}  // namespace mvs

using namespace mvs;

#define MVS_REQUIRE(ctx, cond, ...) \
    do { if (!(cond)) return set_error(ctx, MVS_ERR_INVALID, __VA_ARGS__); } while (0)

namespace mvs {
int make_loss_params(mvs_ctx* ctx, const mvs_loss_config* c, LossParams* out) {
    MVS_REQUIRE(ctx, c, "mvs_set_loss_config: NULL config");
    MVS_REQUIRE(ctx, c->body_prior >= 0 && c->body_prior <= 2, "mvs_set_loss_config: bad body_prior");
    MVS_REQUIRE(ctx, c->body_prior != MVS_PRIOR_GMM || c->use_vposer || ctx->m.M > 0,
                "mvs_set_loss_config: GMM prior selected but mvs_set_gmm_prior was not called");
    MVS_REQUIRE(ctx, !c->interpenetration || ctx->m.faces, "mvs_set_loss_config: interpenetration needs faces");
    MVS_REQUIRE(ctx, c->use_vposer >= 0 && c->use_vposer <= 2, "mvs_set_loss_config: use_vposer must be 0, 1 or 2");
    MVS_REQUIRE(ctx, c->use_vposer != 2 || ctx->m.vp_w1, "mvs_set_loss_config: use_vposer = 2 needs mvs_set_vposer");
    LossParams l{};
    l.data_weight = c->data_weight; l.body_pose_weight = c->body_pose_weight; l.shape_weight = c->shape_weight;
    l.bending_prior_weight = c->bending_prior_weight; l.coll_loss_weight = c->coll_loss_weight; l.rho = c->rho;
    l.body_prior = c->body_prior; l.use_joints_conf = c->use_joints_conf; l.use_vposer = c->use_vposer;
    l.fix_shape = c->fix_shape; l.interpenetration = c->interpenetration;
    l.sdf_grid = c->sdf_grid > 0 ? c->sdf_grid : 128; l.sdf_all_faces = c->sdf_all_faces;
    l.frozen_mask = c->frozen_mask; l.num_gaussians = ctx->m.M;
    l.anchor_on = ctx->anchor_enabled ? 1 : 0;
    *out = l;
    return MVS_OK;
}
}  // namespace mvs

extern "C" {

int mvs_version(void) { return 200; }

#ifndef MVS_BUILD_ID
#define MVS_BUILD_ID "unknown"
#endif
static const char kBuildIdTag[] = "MVS_BUILD_ID=" MVS_BUILD_ID;      // the tag makes the id findable in the file (build.py)
const char* mvs_build_id(void) { return kBuildIdTag + 13; }

const char* mvs_last_error(const mvs_ctx* ctx) { return ctx ? ctx->err.c_str() : g_last_error.c_str(); }

long long mvs_launch_count(const mvs_ctx* ctx) { return ctx ? ctx->launches : 0; }

int mvs_create(int device, mvs_ctx** out) {
    if (!out) return set_error(nullptr, MVS_ERR_INVALID, "mvs_create: out is NULL");
    *out = nullptr;
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0)
        return set_error(nullptr, MVS_ERR_NO_DEVICE,
                         "mvs_create: no CUDA device (%s); libmvsmpl has no CPU fallback",
                         e != cudaSuccess ? cudaGetErrorString(e) : "device count is 0");
    if (device < 0 || device >= count) return set_error(nullptr, MVS_ERR_INVALID, "mvs_create: bad device %d", device);
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) != cudaSuccess || prop.major != 9 || prop.minor != 0)
        return set_error(nullptr, MVS_ERR_NO_DEVICE, "mvs_create: device %d is sm_%d%d; this library is built for sm_90a only",
                         device, prop.major, prop.minor);
    if (cudaSetDevice(device) != cudaSuccess) return set_error(nullptr, MVS_ERR_CUDA, "cudaSetDevice failed");
    mvs_ctx* ctx = new mvs_ctx();
    ctx->device = device;
    ctx->sm_count = prop.multiProcessorCount;
    *out = ctx;
    return MVS_OK;
}

static const char* kKernelNames[KID_COUNT] = {
    "frame_fwd", "vertex_fwd", "sdf_bbox", "sdf_sample", "sdf_finalize", "keypoint_loss", "vertex_bwd", "frame_bwd",
    "lbfgs_advance", "lbfgs_compact", "sdf_grid", "misc", "closure_resident", "lbfgs_resident", "sdf_fused", "frame_step", "posedirs_gemm_tc", "skin"};

const char* mvs_kernel_name(int k) { return (k >= 0 && k < KID_COUNT) ? kKernelNames[k] : ""; }

int mvs_set_exec_mode(mvs_ctx* ctx, int mode) {
    if (!ctx) return set_error(nullptr, MVS_ERR_INVALID, "ctx is NULL");
    MVS_REQUIRE(ctx, mode >= 0 && mode <= 3, "mvs_set_exec_mode: mode must be 0, 1, 2 or 3");
    ctx->exec_mode = mode;
    return MVS_OK;
}

int mvs_profile(mvs_ctx* ctx, unsigned mask) {
    if (!ctx) return set_error(nullptr, MVS_ERR_INVALID, "ctx is NULL");
    MVS_CUDA_OK(ctx, cudaSetDevice(ctx->device));
    MVS_CUDA_OK(ctx, cudaDeviceSynchronize());
    ctx->prof.mask = mask;
    for (int k = 0; k < KID_COUNT; ++k) ctx->prof.used[k] = 0;
    return MVS_OK;
}

int mvs_profile_read(mvs_ctx* ctx, double* ms, long long* launches) {
    if (!ctx) return set_error(nullptr, MVS_ERR_INVALID, "ctx is NULL");
    MVS_REQUIRE(ctx, ms && launches, "mvs_profile_read: NULL output");
    MVS_CUDA_OK(ctx, cudaSetDevice(ctx->device));
    MVS_CUDA_OK(ctx, cudaDeviceSynchronize());
    for (int k = 0; k < KID_COUNT; ++k) {
        double acc = 0.0;
        const size_t n = ctx->prof.used[k] / 2;
        for (size_t i = 0; i < n; ++i) {
            float e = 0.f;
            if (cudaEventElapsedTime(&e, ctx->prof.ev[k][2 * i], ctx->prof.ev[k][2 * i + 1]) == cudaSuccess) acc += e;
        }
        ms[k] = acc;
        launches[k] = (long long)n;
        ctx->prof.used[k] = 0;
    }
    return MVS_OK;
}

void mvs_destroy(mvs_ctx* ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    cudaDeviceSynchronize();
    for (int k = 0; k < KID_COUNT; ++k)
        for (cudaEvent_t e : ctx->prof.ev[k]) cudaEventDestroy(e);
    for (void* p : ctx->allocs) cudaFree(p);
    delete ctx;
}

int mvs_set_model(mvs_ctx* ctx, const mvs_model_desc* d) {
    if (!ctx) return set_error(nullptr, MVS_ERR_INVALID, "ctx is NULL");
    MVS_REQUIRE(ctx, d && d->v_template && d->shapedirs && d->posedirs && d->J_regressor && d->parents && d->lbs_weights,
                "mvs_set_model: missing array");
    MVS_REQUIRE(ctx, !ctx->have_model, "mvs_set_model: model already set (create a new context)");
    MVS_REQUIRE(ctx, d->n_verts > 0 && d->n_keypoints > 0 && d->n_keypoints <= kMaxKeypoints, "mvs_set_model: bad sizes");
    MVS_REQUIRE(ctx, d->parents[0] < 0, "mvs_set_model: parents[0] must be -1");
    for (int j = 1; j < kJoints; ++j)
        MVS_REQUIRE(ctx, d->parents[j] >= 0 && d->parents[j] < j, "mvs_set_model: parents must satisfy 0 <= parents[j] < j");
    MVS_CUDA_OK(ctx, cudaSetDevice(ctx->device));
    const int N = d->n_verts;
    DevModel& m = ctx->m;
    m.N = N;
    m.F = d->faces ? d->n_faces : 0;
    for (int j = 0; j < kJoints; ++j) ctx->parents.p[j] = d->parents[j];

    // Qk rows: [posedirs column | shapedirs row | v_template | pad]
    {
        std::vector<float> Q((size_t)3 * N * kFeatPad, 0.f);
        for (int col = 0; col < 3 * N; ++col) {
            float* row = &Q[(size_t)col * kFeatPad];
            for (int k = 0; k < kPoseBasis; ++k) row[k] = d->posedirs[(size_t)k * 3 * N + col];
            for (int l = 0; l < kBetas; ++l) row[kPoseBasis + l] = d->shapedirs[(size_t)col * kBetas + l];
            row[kFeat - 1] = d->v_template[col];
        }
        int rc = dev_upload(ctx, &m.Qk, Q.data(), Q.size());
        if (rc) return rc;
        if ((rc = tc_upload_model(ctx, Q.data()))) return rc;
        std::vector<float> stv((size_t)N * 33);
        for (int n = 0; n < N; ++n)
            for (int c = 0; c < 3; ++c) {
                for (int l = 0; l < kBetas; ++l) stv[(size_t)n * 33 + 11 * c + l] = d->shapedirs[((size_t)3 * n + c) * kBetas + l];
                stv[(size_t)n * 33 + 11 * c + kBetas] = d->v_template[3 * n + c];
            }
        if ((rc = dev_upload(ctx, &m.ST, stv.data(), stv.size()))) return rc;
    }
    // rest joints pre-contracted through the shape blend shapes (fp64)
    {
        std::vector<float> Jt(kJoints * 3), JS(kJoints * 3 * kBetas);
        for (int j = 0; j < kJoints; ++j)
            for (int c = 0; c < 3; ++c) {
                double a = 0.0;
                double al[kBetas] = {0};
                for (int n = 0; n < N; ++n) {
                    const double w = d->J_regressor[(size_t)j * N + n];
                    if (w == 0.0) continue;
                    a += w * (double)d->v_template[3 * n + c];
                    for (int l = 0; l < kBetas; ++l) al[l] += w * (double)d->shapedirs[((size_t)3 * n + c) * kBetas + l];
                }
                Jt[3 * j + c] = (float)a;
                for (int l = 0; l < kBetas; ++l) JS[(3 * j + c) * kBetas + l] = (float)al[l];
            }
        int rc = dev_upload(ctx, &m.Jt, Jt.data(), Jt.size());
        if (rc) return rc;
        rc = dev_upload(ctx, &m.JS, JS.data(), JS.size());
        if (rc) return rc;
    }
    // skinning weights: ELL + dense
    {
        int KW = 1;
        for (int n = 0; n < N; ++n) {
            int c = 0;
            for (int j = 0; j < kJoints; ++j) c += d->lbs_weights[(size_t)n * kJoints + j] != 0.f;
            KW = std::max(KW, c);
        }
        m.KW = KW;
        std::vector<int> ej((size_t)N * KW, 0);
        std::vector<float> ew((size_t)N * KW, 0.f);
        for (int n = 0; n < N; ++n) {
            int c = 0;
            for (int j = 0; j < kJoints; ++j) {
                const float w = d->lbs_weights[(size_t)n * kJoints + j];
                if (w != 0.f) { ej[(size_t)n * KW + c] = j; ew[(size_t)n * KW + c] = w; ++c; }
            }
        }
        int rc = dev_upload(ctx, &m.ell_j, ej.data(), ej.size());
        if (rc) return rc;
        rc = dev_upload(ctx, &m.ell_w, ew.data(), ew.size());
        if (rc) return rc;
        rc = dev_upload(ctx, &m.Wd, d->lbs_weights, (size_t)N * kJoints);
        if (rc) return rc;
    }
    if (d->faces && d->n_faces > 0) {
        for (int c = 0; c < 3; ++c) m.tri0[c] = d->faces[c];
        int rc = dev_upload(ctx, &m.faces, d->faces, (size_t)d->n_faces * 3);
        if (rc) return rc;
    }
    // keypoint definition
    {
        const int K = d->n_keypoints;
        const int n_src = (d->n_reg > 0 ? d->n_reg : kJoints) + d->n_extra;
        MVS_REQUIRE(ctx, d->joint_map, "mvs_set_model: joint_map is NULL");
        MVS_REQUIRE(ctx, d->n_reg == 0 || d->joint_regressor, "mvs_set_model: joint_regressor is NULL");
        std::vector<int> ptr(K + 1, 0), vidx, chain(K, -1);
        std::vector<float> wts;
        for (int k = 0; k < K; ++k) {
            const int src = d->joint_map[k];
            MVS_REQUIRE(ctx, src >= 0 && src < n_src, "mvs_set_model: joint_map[%d]=%d out of range", k, src);
            const int n_first = d->n_reg > 0 ? d->n_reg : kJoints;
            if (src < n_first) {
                if (d->n_reg > 0) {
                    for (int n = 0; n < N; ++n) {
                        const float w = d->joint_regressor[(size_t)src * N + n];
                        if (w != 0.f) { vidx.push_back(n); wts.push_back(w); }
                    }
                } else {
                    chain[k] = src;
                }
            } else {
                const int v = d->extra_vertex_ids[src - n_first];
                MVS_REQUIRE(ctx, v >= 0 && v < N, "mvs_set_model: extra vertex id out of range");
                vidx.push_back(v);
                wts.push_back(1.f);
            }
            ptr[k + 1] = (int)vidx.size();
        }
        std::vector<int> sup(vidx);
        std::sort(sup.begin(), sup.end());
        sup.erase(std::unique(sup.begin(), sup.end()), sup.end());
        const int nsup = (int)sup.size();
        std::vector<int> spos(vidx.size());
        for (size_t e = 0; e < vidx.size(); ++e) spos[e] = (int)(std::lower_bound(sup.begin(), sup.end(), vidx[e]) - sup.begin());
        std::vector<int> sptr(nsup + 1, 0), sk;
        std::vector<float> swt;
        for (int i = 0; i < nsup; ++i) {
            for (int k = 0; k < K; ++k)
                for (int e = ptr[k]; e < ptr[k + 1]; ++e)
                    if (vidx[e] == sup[i]) { sk.push_back(k); swt.push_back(wts[e]); }
            sptr[i + 1] = (int)sk.size();
        }
        m.K = K; m.nsup = nsup; m.n_kp_entries = (int)vidx.size();
        int rc;
        if ((rc = dev_upload(ctx, &m.kp_ptr, ptr.data(), ptr.size()))) return rc;
        if ((rc = dev_upload(ctx, &m.kp_vidx, vidx.data(), vidx.size()))) return rc;
        if ((rc = dev_upload(ctx, &m.kp_spos, spos.data(), spos.size()))) return rc;
        if ((rc = dev_upload(ctx, &m.kp_w, wts.data(), wts.size()))) return rc;
        if ((rc = dev_upload(ctx, &m.kp_chain, chain.data(), chain.size()))) return rc;
        if ((rc = dev_upload(ctx, &m.sup, sup.data(), sup.size()))) return rc;
        // per joint: which support vertices it skins (adjoint dA_j without atomics in the frame-resident kernel)
        {
            std::vector<int> jp(kJoints + 1, 0), ji;
            std::vector<float> jw;
            for (int j = 0; j < kJoints; ++j) {
                for (int i = 0; i < nsup; ++i) {
                    const float w = d->lbs_weights[(size_t)sup[i] * kJoints + j];
                    if (w != 0.f) { ji.push_back(i); jw.push_back(w); }
                }
                jp[j + 1] = (int)ji.size();
            }
            if ((rc = dev_upload(ctx, &m.supj_ptr, jp.data(), jp.size()))) return rc;
            if ((rc = dev_upload(ctx, &m.supj_i, ji.data(), ji.size()))) return rc;
            if ((rc = dev_upload(ctx, &m.supj_w, jw.data(), jw.size()))) return rc;
        }
        std::vector<int> comb(sup);
        for (int n = 0; n < N; ++n) comb.push_back(n);
        if ((rc = dev_upload(ctx, &m.sup_then_all, comb.data(), comb.size()))) return rc;
        if ((rc = dev_upload(ctx, &m.sup_ptr, sptr.data(), sptr.size()))) return rc;
        if ((rc = dev_upload(ctx, &m.sup_k, sk.data(), sk.size()))) return rc;
        if ((rc = dev_upload(ctx, &m.sup_w, swt.data(), swt.size()))) return rc;
    }
    ctx->have_model = true;
    return MVS_OK;
}

int mvs_set_gmm_prior(mvs_ctx* ctx, int M, const float* means, const float* precisions, const float* nll_weights) {
    if (!ctx) return set_error(nullptr, MVS_ERR_INVALID, "ctx is NULL");
    MVS_REQUIRE(ctx, M > 0 && M <= 64 && means && precisions && nll_weights, "mvs_set_gmm_prior: bad arguments");
    MVS_CUDA_OK(ctx, cudaSetDevice(ctx->device));
    const int D = 69;
    // x^T P x == x^T sym(P) x, and the gradient of the quadratic form is sym(P) x: store the symmetric part
    std::vector<float> P((size_t)M * D * D), lw(M);
    for (int m = 0; m < M; ++m) {
        for (int i = 0; i < D; ++i)
            for (int j = 0; j < D; ++j)
                P[((size_t)m * D + i) * D + j] = (float)(0.5 * ((double)precisions[((size_t)m * D + i) * D + j] +
                                                                (double)precisions[((size_t)m * D + j) * D + i]));
        lw[m] = logf(nll_weights[m]);                       // prior.py:189 takes torch.log of the fp32 buffer
    }
    DevModel& dm = ctx->m;
    dm.M = M;
    int rc;
    if ((rc = dev_upload(ctx, &dm.gmm_means, means, (size_t)M * D))) return rc;
    if ((rc = dev_upload(ctx, &dm.gmm_prec, P.data(), P.size()))) return rc;
    if ((rc = dev_upload(ctx, &dm.gmm_lognllw, lw.data(), lw.size()))) return rc;
    return MVS_OK;
}

int mvs_set_vposer(mvs_ctx* ctx, const float* fc1_w, const float* fc1_b, const float* fc2_w, const float* fc2_b,
                   const float* out_w, const float* out_b) {
    if (!ctx) return set_error(nullptr, MVS_ERR_INVALID, "ctx is NULL");
    MVS_REQUIRE(ctx, fc1_w && fc1_b && fc2_w && fc2_b && out_w && out_b, "mvs_set_vposer: NULL array");
    MVS_CUDA_OK(ctx, cudaSetDevice(ctx->device));
    DevModel& m = ctx->m;
    constexpr int H = 512, Z = 32, O = 138;
    auto up = [&](float** plain, float** transposed, const float* w, int no, int ni) -> int {
        std::vector<float> t((size_t)no * ni);
        for (int o = 0; o < no; ++o)
            for (int i = 0; i < ni; ++i) t[(size_t)i * no + o] = w[(size_t)o * ni + i];
        int rc = dev_upload(ctx, plain, w, (size_t)no * ni);
        if (rc) return rc;
        return dev_upload(ctx, transposed, t.data(), t.size());
    };
    int rc;
    if ((rc = up(&m.vp_w1, &m.vp_w1t, fc1_w, H, Z))) return rc;
    if ((rc = up(&m.vp_w2, &m.vp_w2t, fc2_w, H, H))) return rc;
    if ((rc = up(&m.vp_w3, &m.vp_w3t, out_w, O, H))) return rc;
    if ((rc = dev_upload(ctx, &m.vp_b1, fc1_b, H))) return rc;
    if ((rc = dev_upload(ctx, &m.vp_b2, fc2_b, H))) return rc;
    if ((rc = dev_upload(ctx, &m.vp_b3, out_b, O))) return rc;
    return MVS_OK;
}

int mvs_set_cameras(mvs_ctx* ctx, int V, const float* R, const float* t, const float* f, const float* c) {
    if (!ctx) return set_error(nullptr, MVS_ERR_INVALID, "ctx is NULL");
    MVS_REQUIRE(ctx, V > 0 && V <= kMaxViews && R && t && f && c, "mvs_set_cameras: need 1..%d views", kMaxViews);
    ctx->cams.num_views = V;
    for (int v = 0; v < V; ++v) {
        memcpy(ctx->cams.cam[v].R, R + 9 * v, 9 * sizeof(float));
        memcpy(ctx->cams.cam[v].t, t + 3 * v, 3 * sizeof(float));
        memcpy(ctx->cams.cam[v].f, f + 2 * v, 2 * sizeof(float));
        memcpy(ctx->cams.cam[v].c, c + 2 * v, 2 * sizeof(float));
    }
    ctx->have_cams = true;
    ctx->have_kp = false;                                   // keypoints are per view: must be set again
    return MVS_OK;
}

int mvs_set_batch(mvs_ctx* ctx, int B) {
    if (!ctx) return set_error(nullptr, MVS_ERR_INVALID, "ctx is NULL");
    MVS_REQUIRE(ctx, ctx->have_model, "mvs_set_batch: set the model first");
    MVS_REQUIRE(ctx, B > 0 && B <= (1 << 20), "mvs_set_batch: bad batch %d", B);
    MVS_REQUIRE(ctx, ctx->ws.B == 0, "mvs_set_batch: batch already set (create a new context)");
    MVS_CUDA_OK(ctx, cudaSetDevice(ctx->device));
    Workspace& w = ctx->ws;
    const DevModel& m = ctx->m;
    w.B = B;
    w.na_bound = B;
    w.ldA = (B + kTileF - 1) / kTileF * kTileF;
    const int ftiles = w.ldA / kTileF;
    w.nstrips_max = std::min((m.N + kTileV - 1) / kTileV, (ctx->sm_count + ftiles - 1) / ftiles + 1);
    int rc;
    if ((rc = dev_alloc(ctx, &w.fidx, B))) return rc;
    if ((rc = dev_alloc(ctx, &w.na, 1))) return rc;
    if ((rc = dev_alloc(ctx, &w.Phi, (size_t)w.ldA * kFeatPad))) return rc;
    if ((rc = dev_alloc(ctx, &w.PhiTc, (size_t)2 * w.ldA * kFeatPad))) return rc;
    if ((rc = dev_alloc(ctx, &w.bboxp, (size_t)B * ((m.N + 63) / 64) * 12))) return rc;
    if ((rc = dev_alloc(ctx, &w.At, (size_t)kSkinFloats * w.ldA))) return rc;
    if ((rc = dev_alloc(ctx, &w.gchain, (size_t)B * kJoints * 3))) return rc;
    if ((rc = dev_alloc(ctx, &w.slot_tr, (size_t)B * 4))) return rc;
    if ((rc = dev_alloc(ctx, &w.vposed, (size_t)B * m.N * 3))) return rc;
    if ((rc = dev_alloc(ctx, &w.verts, (size_t)B * m.N * 3))) return rc;
    if ((rc = dev_alloc(ctx, &w.dv, (size_t)B * (m.nsup + m.N) * 3))) return rc;
    if ((rc = dev_alloc(ctx, &w.part, (size_t)w.nstrips_max * w.ldA * kPartFloats))) return rc;
    if ((rc = dev_alloc(ctx, &w.data_loss, B))) return rc;
    if ((rc = dev_alloc(ctx, &w.pen_loss, B))) return rc;
    if ((rc = dev_alloc(ctx, &w.dtransl, (size_t)B * 3))) return rc;
    if ((rc = dev_alloc(ctx, &w.dgchain, (size_t)B * kJoints * 3))) return rc;
    if ((rc = dev_alloc(ctx, &w.loss_scratch, B))) return rc;
    if ((rc = dev_alloc(ctx, &w.grad_scratch, (size_t)B * kParams))) return rc;
    MVS_CUDA_OK(ctx, cudaMemset(w.At, 0, (size_t)kSkinFloats * w.ldA * sizeof(float)));
    MVS_CUDA_OK(ctx, cudaMemset(w.Phi, 0, (size_t)w.ldA * kFeatPad * sizeof(float)));
    MVS_CUDA_OK(ctx, cudaMemset(w.PhiTc, 0, (size_t)2 * w.ldA * kFeatPad * sizeof(float)));
    MVS_LAUNCH(ctx, KID_MISC, 0, iota_kernel<<<(B + 255) / 256, 256>>>(w.fidx, B, w.na));
    MVS_CUDA_OK(ctx, cudaDeviceSynchronize());
    return MVS_OK;
}

int mvs_set_keypoints(mvs_ctx* ctx, const float* gt_uv, const float* conf, const float* joint_weights, int on_device,
                      void* stream) {
    if (!ctx) return set_error(nullptr, MVS_ERR_INVALID, "ctx is NULL");
    MVS_REQUIRE(ctx, ctx->ws.B > 0 && ctx->have_cams, "mvs_set_keypoints: set cameras and batch first");
    MVS_REQUIRE(ctx, gt_uv && conf && joint_weights, "mvs_set_keypoints: NULL array");
    MVS_CUDA_OK(ctx, cudaSetDevice(ctx->device));
    Workspace& w = ctx->ws;
    const size_t n = (size_t)ctx->cams.num_views * w.B * ctx->m.K;
    int rc;
    if (!w.gt_uv || !ctx->have_kp) {
        if ((rc = dev_alloc(ctx, &w.gt_uv, n * 2))) return rc;
        if ((rc = dev_alloc(ctx, &w.conf, n))) return rc;
        if (!w.joint_w && (rc = dev_alloc(ctx, &w.joint_w, kMaxKeypoints))) return rc;
    }
    cudaStream_t st = (cudaStream_t)stream;
    const cudaMemcpyKind kind = on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
    MVS_CUDA_OK(ctx, cudaMemcpyAsync(w.gt_uv, gt_uv, n * 2 * sizeof(float), kind, st));
    MVS_CUDA_OK(ctx, cudaMemcpyAsync(w.conf, conf, n * sizeof(float), kind, st));
    MVS_CUDA_OK(ctx, cudaMemcpyAsync(w.joint_w, joint_weights, ctx->m.K * sizeof(float), kind, st));
    if (!on_device) MVS_CUDA_OK(ctx, cudaStreamSynchronize(st));
    ctx->have_kp = true;
    return MVS_OK;
}

int mvs_set_loss_config(mvs_ctx* ctx, const mvs_loss_config* c) {
    if (!ctx) return set_error(nullptr, MVS_ERR_INVALID, "ctx is NULL");
    LossParams l;
    const int rc = make_loss_params(ctx, c, &l);
    if (rc) return rc;
    ctx->loss = l;
    ctx->have_loss = true;
    return MVS_OK;
}

int mvs_set_anchor(mvs_ctx* ctx, const float* anchor_dev, const float* weight_dev, int enable, void* stream) {
    if (!ctx) return set_error(nullptr, MVS_ERR_INVALID, "ctx is NULL");
    MVS_REQUIRE(ctx, ctx->ws.B > 0, "mvs_set_anchor: set the batch first");
    MVS_CUDA_OK(ctx, cudaSetDevice(ctx->device));
    Workspace& w = ctx->ws;
    if (!enable) { ctx->loss.anchor_on = 0; ctx->anchor_enabled = false; return MVS_OK; }
    MVS_REQUIRE(ctx, anchor_dev && weight_dev, "mvs_set_anchor: NULL array");
    int rc;
    if (!w.anchor) {
        if ((rc = dev_alloc(ctx, &w.anchor, (size_t)w.B * kParams))) return rc;
        if ((rc = dev_alloc(ctx, &w.anchor_w, (size_t)w.B * kParams))) return rc;
    }
    cudaStream_t st = (cudaStream_t)stream;
    MVS_CUDA_OK(ctx, cudaMemcpyAsync(w.anchor, anchor_dev, (size_t)w.B * kParams * sizeof(float), cudaMemcpyDeviceToDevice, st));
    MVS_CUDA_OK(ctx, cudaMemcpyAsync(w.anchor_w, weight_dev, (size_t)w.B * kParams * sizeof(float), cudaMemcpyDeviceToDevice, st));
    ctx->loss.anchor_on = 1;
    ctx->anchor_enabled = true;
    return MVS_OK;
}

int mvs_closure(mvs_ctx* ctx, const float* params_dev, float* loss_dev, float* grad_dev, float* joints_dev,
                float* proj_dev, float* verts_dev, void* stream) {
    if (!ctx) return set_error(nullptr, MVS_ERR_INVALID, "ctx is NULL");
    MVS_REQUIRE(ctx, ctx->have_model && ctx->have_cams && ctx->have_kp && ctx->have_loss && ctx->ws.B > 0,
                "mvs_closure: model, cameras, batch, keypoints and loss config must be set first");
    MVS_REQUIRE(ctx, params_dev, "mvs_closure: params_dev is NULL");
    MVS_CUDA_OK(ctx, cudaSetDevice(ctx->device));
    return launch_closure(ctx, params_dev, loss_dev, grad_dev, joints_dev, proj_dev, verts_dev, (cudaStream_t)stream);
}

int mvs_forward(mvs_ctx* ctx, const float* params_dev, float* joints_dev, float* verts_dev, void* stream) {
    if (!ctx) return set_error(nullptr, MVS_ERR_INVALID, "ctx is NULL");
    MVS_REQUIRE(ctx, ctx->have_model && ctx->ws.B > 0, "mvs_forward: model and batch must be set first");
    MVS_REQUIRE(ctx, params_dev, "mvs_forward: params_dev is NULL");
    MVS_CUDA_OK(ctx, cudaSetDevice(ctx->device));
    return launch_closure(ctx, params_dev, nullptr, nullptr, joints_dev, nullptr, verts_dev, (cudaStream_t)stream, true);
}

int mvs_vposer_decode(mvs_ctx* ctx, const float* params_dev, float* body_pose_dev, void* stream) {
    if (!ctx) return set_error(nullptr, MVS_ERR_INVALID, "ctx is NULL");
    MVS_REQUIRE(ctx, ctx->have_model && ctx->ws.B > 0 && ctx->m.vp_w1, "mvs_vposer_decode: model, batch and mvs_set_vposer first");
    MVS_REQUIRE(ctx, params_dev && body_pose_dev, "mvs_vposer_decode: NULL argument");
    MVS_CUDA_OK(ctx, cudaSetDevice(ctx->device));
    return launch_vposer_decode(ctx, params_dev, body_pose_dev, (cudaStream_t)stream);
}

int mvs_sdf_grid(mvs_ctx* ctx, float* phi_dev, const int* faces_dev, int num_faces, const float* verts_dev, int batch,
                 int n_verts, int grid_size, void* stream) {
    if (!ctx) return set_error(nullptr, MVS_ERR_INVALID, "ctx is NULL");
    MVS_REQUIRE(ctx, phi_dev && faces_dev && verts_dev && num_faces > 0 && batch > 0 && grid_size > 1,
                "mvs_sdf_grid: bad arguments");
    MVS_CUDA_OK(ctx, cudaSetDevice(ctx->device));
    return sdf_grid_launch(ctx, phi_dev, faces_dev, num_faces, verts_dev, batch, n_verts, grid_size, (cudaStream_t)stream);
}

}  // extern "C"
