// C ABI of libmvsmpl.so (see include/mvsmpl.h): context lifetime, one-time uploads with the
// host-side pre-contractions, workspace allocation, and the thin entry points that enqueue the
// kernels of mvs_closure.cu / mvs_lbfgs.cu / mvs_sdf.cu on the caller's stream.
#include <algorithm>
#include <mutex>
#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "mvs_internal.cuh"
#include "mvs_lbfgs_core.cuh"

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
void dev_free(mvs_ctx* ctx, void* p) {
    if (!p) return;
    ctx->allocs.erase(std::find(ctx->allocs.begin(), ctx->allocs.end(), p));
    cudaFree(p);
}
template int dev_alloc<unsigned short>(mvs_ctx*, unsigned short**, size_t);
template int dev_alloc<float>(mvs_ctx*, float**, size_t);
template int dev_alloc<int>(mvs_ctx*, int**, size_t);
template int dev_alloc<double>(mvs_ctx*, double**, size_t);
template int dev_alloc<unsigned char>(mvs_ctx*, unsigned char**, size_t);
template int dev_alloc<int2>(mvs_ctx*, int2**, size_t);
template int dev_alloc<float4>(mvs_ctx*, float4**, size_t);
template int dev_alloc<FrameBox>(mvs_ctx*, FrameBox**, size_t);
template int dev_alloc<SdfFrameSetup>(mvs_ctx*, SdfFrameSetup**, size_t);
template int dev_alloc<long long>(mvs_ctx*, long long**, size_t);
template int dev_alloc<Rig>(mvs_ctx*, Rig**, size_t);
template int dev_alloc<CamRefine>(mvs_ctx*, CamRefine**, size_t);
template int dev_alloc<CameraProblem>(mvs_ctx*, CameraProblem**, size_t);
template int dev_alloc<LossParams>(mvs_ctx*, LossParams**, size_t);
template int dev_alloc<FrameScalars>(mvs_ctx*, FrameScalars**, size_t);

// ----------------------------------------------------------------------------- model constants shared between contexts
// Every context of the process that uploads the same constants to the same device (mvs_set_model, mvs_set_gmm_prior,
// mvs_set_vposer) reads ONE device copy of them.  Several batches in flight, each on its own context, then stream one posedirs
// table through L2 instead of one each (DESIGN.md section 5), and a context costs ~20 MB less device memory.  An entry is
// keyed by its device and the exact bytes of its arrays, kept on the host and compared in full, so two different models never
// alias.  It counts the contexts that hold it; the last one out frees it (mvs_destroy).  Sharing is sound because nothing
// writes into these arrays after the upload (the const pointers of DevModel).  MVS_SHARE_MODEL=0 in the environment gives
// every context its own copy (A/B measurements of one build).
struct ConstArray {
    const void** dev;                 // where the device pointer goes
    const void* host;
    size_t bytes;
};
template <class T> static ConstArray const_array(const T*& dev, const T* host, size_t count) {
    return ConstArray{reinterpret_cast<const void**>(&dev), host, count * sizeof(T)};
}

struct SharedConsts {
    int device = 0;
    int refs = 0;
    std::vector<size_t> sizes;        // bytes of each array
    std::vector<char> bytes;          // their contents back to back (shared entries only: the key)
    std::vector<void*> dev;
};

static std::mutex g_consts_mu;
static std::vector<SharedConsts*> g_consts;   // the shared entries of every device

static bool same_consts(const SharedConsts* e, int device, const std::vector<ConstArray>& a) {
    if (e->device != device || e->sizes.size() != a.size()) return false;
    for (size_t i = 0; i < a.size(); ++i)
        if (e->sizes[i] != a[i].bytes) return false;
    size_t off = 0;
    for (const ConstArray& x : a) {
        if (x.bytes && memcmp(e->bytes.data() + off, x.host, x.bytes) != 0) return false;
        off += x.bytes;
    }
    return true;
}

static void free_consts(SharedConsts* e) {
    for (void* p : e->dev) cudaFree(p);
    delete e;
}

// Points *a[i].dev at a device copy of a[i].host for every i: the shared copy of an entry with the same bytes on ctx's device,
// else a new upload (inserted into the store unless MVS_SHARE_MODEL=0).  The context holds the entry until mvs_destroy.
static int upload_consts(mvs_ctx* ctx, const std::vector<ConstArray>& a) {
    static const bool share = !(getenv("MVS_SHARE_MODEL") && strcmp(getenv("MVS_SHARE_MODEL"), "0") == 0);
    std::lock_guard<std::mutex> lock(g_consts_mu);
    SharedConsts* e = nullptr;
    if (share)
        for (SharedConsts* s : g_consts)
            if (same_consts(s, ctx->device, a)) { e = s; break; }
    if (!e) {
        e = new SharedConsts();
        e->device = ctx->device;
        for (const ConstArray& x : a) {
            void* d = nullptr;
            cudaError_t err = cudaMalloc(&d, std::max<size_t>(x.bytes, 1));
            if (err == cudaSuccess) {
                e->dev.push_back(d);
                if (x.bytes) err = cudaMemcpy(d, x.host, x.bytes, cudaMemcpyHostToDevice);
            }
            if (err != cudaSuccess) {
                free_consts(e);
                return set_error(ctx, MVS_ERR_CUDA, "uploading the model constants failed: %s", cudaGetErrorString(err));
            }
            e->sizes.push_back(x.bytes);
        }
        if (share) {
            for (const ConstArray& x : a)
                e->bytes.insert(e->bytes.end(), (const char*)x.host, (const char*)x.host + x.bytes);
            g_consts.push_back(e);
        }
    }
    ++e->refs;
    ctx->consts.push_back(e);
    for (size_t i = 0; i < a.size(); ++i) *a[i].dev = e->dev[i];
    return MVS_OK;
}

// mvs_destroy: drops the context's entries; the last holder of an entry frees its arrays
static void release_consts(mvs_ctx* ctx) {
    std::lock_guard<std::mutex> lock(g_consts_mu);
    for (SharedConsts* e : ctx->consts) {
        if (--e->refs) continue;
        g_consts.erase(std::remove(g_consts.begin(), g_consts.end(), e), g_consts.end());
        free_consts(e);
    }
    ctx->consts.clear();
}

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
    l.j3d_on = ctx->j3d_enabled ? 1 : 0;
    *out = l;
    return MVS_OK;
}

int ensure_keypoint_ws(mvs_ctx* ctx) {
    Workspace& w = ctx->ws;
    const int V = ctx->vmax;
    if (w.gt_uv && w.kp_views == V) return MVS_OK;
    const size_t n = (size_t)V * w.B * ctx->m.K;
    int rc;
    if ((rc = dev_alloc(ctx, &w.gt_uv, n * 2))) return rc;
    if ((rc = dev_alloc(ctx, &w.conf, n))) return rc;
    if (!w.joint_w && (rc = dev_alloc(ctx, &w.joint_w, kMaxKeypoints))) return rc;
    w.kp_views = V;
    return MVS_OK;
}

int batch_rigs(mvs_ctx* ctx, const char* who) {
    if (ctx->rigs.size() > 1 && !ctx->slot_rigs)
        return set_error(ctx, MVS_ERR_INVALID, "%s: the context has %d camera rigs and no per-slot rigs were given since the last "
                                               "mvs_set_batch, mvs_set_camera_rigs or stream call (mvs_set_frame_rigs)",
                         who, (int)ctx->rigs.size());
    return MVS_OK;
}

__global__ void rig_check_kernel(const int* __restrict__ rig, int n, int n_rigs, int* __restrict__ first_bad) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && (unsigned)rig[i] >= (unsigned)n_rigs) atomicMin(first_bad, i);
}

int check_frame_rigs(mvs_ctx* ctx, const char* who, const int* rig_dev, int n, cudaStream_t st) {
    int rc;
    if (!ctx->rig_bad && (rc = dev_alloc(ctx, &ctx->rig_bad, 1))) return rc;
    MVS_CUDA_OK(ctx, cudaMemsetAsync(ctx->rig_bad, 0x7f, sizeof(int), st));         // 0x7f7f7f7f: no bad frame
    MVS_LAUNCH(ctx, KID_MISC, st, rig_check_kernel<<<(n + 255) / 256, 256, 0, st>>>(rig_dev, n, (int)ctx->rigs.size(), ctx->rig_bad));
    int bad = 0;
    MVS_CUDA_OK(ctx, cudaMemcpyAsync(&bad, ctx->rig_bad, sizeof(int), cudaMemcpyDeviceToHost, st));
    MVS_CUDA_OK(ctx, cudaStreamSynchronize(st));
    if (bad < n) {
        int r = 0;
        MVS_CUDA_OK(ctx, cudaMemcpy(&r, rig_dev + bad, sizeof(int), cudaMemcpyDeviceToHost));
        return set_error(ctx, MVS_ERR_INVALID, "%s: frame %d names rig %d, the context has %d", who, bad, r, (int)ctx->rigs.size());
    }
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
    "lbfgs_advance", "lbfgs_compact", "sdf_grid", "misc", "closure_resident", "lbfgs_resident", "sdf_fused", "frame_step", "posedirs_gemm_tc", "skin",
    "sdf_setup"};

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
    release_fit_state(ctx);
    release_tc_state(ctx);
    for (void* p : ctx->allocs) cudaFree(p);
    release_consts(ctx);
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
    {   // level schedule of the tree (ctx->chain is zero-initialised)
        ChainSched& cs = ctx->chain;
        int depth[kJoints];
        depth[0] = 0;
        int maxd = 0;
        for (int j = 1; j < kJoints; ++j) { depth[j] = depth[d->parents[j]] + 1; if (depth[j] > maxd) maxd = depth[j]; }
        cs.nlev = maxd + 1;
        int o = 0;
        for (int L = 0; L <= maxd; ++L) {
            cs.lev_ptr[L] = (unsigned char)o;
            for (int j = 0; j < kJoints; ++j) if (depth[j] == L) cs.lev_j[o++] = (unsigned char)j;
        }
        for (int L = maxd + 1; L <= kJoints; ++L) cs.lev_ptr[L] = (unsigned char)o;
        o = 0;
        for (int p = 0; p < kJoints; ++p) {
            cs.ch_ptr[p] = (unsigned char)o;
            for (int j = kJoints - 1; j >= 1; --j) if (d->parents[j] == p) cs.ch_j[o++] = (unsigned char)j;
        }
        cs.ch_ptr[kJoints] = (unsigned char)o;
    }

    // Qk rows: [posedirs column | shapedirs row | v_template | pad]
    std::vector<float> Q((size_t)3 * N * kFeatPad, 0.f);
    for (int col = 0; col < 3 * N; ++col) {
        float* row = &Q[(size_t)col * kFeatPad];
        for (int k = 0; k < kPoseBasis; ++k) row[k] = d->posedirs[(size_t)k * 3 * N + col];
        for (int l = 0; l < kBetas; ++l) row[kPoseBasis + l] = d->shapedirs[(size_t)col * kBetas + l];
        row[kFeat - 1] = d->v_template[col];
    }
    std::vector<float> stv((size_t)N * 33);
    for (int n = 0; n < N; ++n)
        for (int c = 0; c < 3; ++c) {
            for (int l = 0; l < kBetas; ++l) stv[(size_t)n * 33 + 11 * c + l] = d->shapedirs[((size_t)3 * n + c) * kBetas + l];
            stv[(size_t)n * 33 + 11 * c + kBetas] = d->v_template[3 * n + c];
        }
    // rest joints pre-contracted through the shape blend shapes (fp64)
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
    // skinning weights: ELL + dense
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
    if (d->faces && d->n_faces > 0)
        for (int c = 0; c < 3; ++c) m.tri0[c] = d->faces[c];
    // keypoint definition
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
    // per joint: which support vertices it skins (adjoint dA_j without atomics in the frame-resident kernel)
    std::vector<int> jp(kJoints + 1, 0), ji;
    std::vector<float> jw;
    for (int j = 0; j < kJoints; ++j) {
        for (int i = 0; i < nsup; ++i) {
            const float w = d->lbs_weights[(size_t)sup[i] * kJoints + j];
            if (w != 0.f) { ji.push_back(i); jw.push_back(w); }
        }
        jp[j + 1] = (int)ji.size();
    }
    std::vector<int> comb(sup);
    for (int n = 0; n < N; ++n) comb.push_back(n);
    // the scalars above (N, F, KW, K, nsup, n_kp_entries, tri0) follow from these arrays' sizes and contents, so a context
    // that finds them in the store has the same scalars as the one that uploaded them
    std::vector<ConstArray> arrays = {
        const_array(m.Qk, Q.data(), Q.size()), const_array(m.ST, stv.data(), stv.size()),
        const_array(m.Jt, Jt.data(), Jt.size()), const_array(m.JS, JS.data(), JS.size()),
        const_array(m.ell_j, ej.data(), ej.size()), const_array(m.ell_w, ew.data(), ew.size()),
        const_array(m.Wd, d->lbs_weights, (size_t)N * kJoints),
        const_array(m.kp_ptr, ptr.data(), ptr.size()), const_array(m.kp_vidx, vidx.data(), vidx.size()),
        const_array(m.kp_spos, spos.data(), spos.size()), const_array(m.kp_w, wts.data(), wts.size()),
        const_array(m.kp_chain, chain.data(), chain.size()), const_array(m.sup, sup.data(), sup.size()),
        const_array(m.supj_ptr, jp.data(), jp.size()), const_array(m.supj_i, ji.data(), ji.size()),
        const_array(m.supj_w, jw.data(), jw.size()), const_array(m.sup_then_all, comb.data(), comb.size()),
        const_array(m.sup_ptr, sptr.data(), sptr.size()), const_array(m.sup_k, sk.data(), sk.size()),
        const_array(m.sup_w, swt.data(), swt.size())};
    // vertex -> face CSR (faces in ascending order) for the renderer's vertex normals (mvs_render); only for faces whose vertex
    // ids are all in range, without which mvs_render refuses the model
    std::vector<int> vfp(N + 1, 0), vfi;
    bool faces_ok = d->faces && d->n_faces > 0;
    for (int e = 0; faces_ok && e < 3 * d->n_faces; ++e) faces_ok = d->faces[e] >= 0 && d->faces[e] < N;
    if (d->faces && d->n_faces > 0) arrays.push_back(const_array(m.faces, d->faces, (size_t)d->n_faces * 3));
    if (faces_ok) {
        for (int e = 0; e < 3 * d->n_faces; ++e) ++vfp[d->faces[e] + 1];
        for (int n = 0; n < N; ++n) vfp[n + 1] += vfp[n];
        vfi.resize(vfp[N]);
        std::vector<int> cur(vfp.begin(), vfp.end() - 1);
        for (int e = 0; e < 3 * d->n_faces; ++e) vfi[cur[d->faces[e]]++] = e / 3;
        arrays.push_back(const_array(m.vf_ptr, vfp.data(), vfp.size()));
        arrays.push_back(const_array(m.vf_idx, vfi.data(), vfi.size()));
    }
    int rc;
    if ((rc = upload_consts(ctx, arrays)) || (rc = tc_upload_model(ctx))) return rc;
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
    return upload_consts(ctx, {const_array(dm.gmm_means, means, (size_t)M * D), const_array(dm.gmm_prec, P.data(), P.size()),
                               const_array(dm.gmm_lognllw, lw.data(), lw.size())});
}

int mvs_set_vposer(mvs_ctx* ctx, const float* fc1_w, const float* fc1_b, const float* fc2_w, const float* fc2_b,
                   const float* out_w, const float* out_b) {
    if (!ctx) return set_error(nullptr, MVS_ERR_INVALID, "ctx is NULL");
    MVS_REQUIRE(ctx, fc1_w && fc1_b && fc2_w && fc2_b && out_w && out_b, "mvs_set_vposer: NULL array");
    MVS_CUDA_OK(ctx, cudaSetDevice(ctx->device));
    DevModel& m = ctx->m;
    constexpr int H = 512, Z = 32, O = 138;
    auto transpose = [](const float* w, int no, int ni) {
        std::vector<float> t((size_t)no * ni);
        for (int o = 0; o < no; ++o)
            for (int i = 0; i < ni; ++i) t[(size_t)i * no + o] = w[(size_t)o * ni + i];
        return t;
    };
    const std::vector<float> w1t = transpose(fc1_w, H, Z), w2t = transpose(fc2_w, H, H), w3t = transpose(out_w, O, H);
    return upload_consts(ctx, {const_array(m.vp_w1, fc1_w, (size_t)H * Z), const_array(m.vp_w1t, w1t.data(), w1t.size()),
                               const_array(m.vp_w2, fc2_w, (size_t)H * H), const_array(m.vp_w2t, w2t.data(), w2t.size()),
                               const_array(m.vp_w3, out_w, (size_t)O * H), const_array(m.vp_w3t, w3t.data(), w3t.size()),
                               const_array(m.vp_b1, fc1_b, H), const_array(m.vp_b2, fc2_b, H), const_array(m.vp_b3, out_b, O)});
}

int mvs_set_camera_rigs_dist(mvs_ctx* ctx, int n_rigs, const int* num_views, const float* R, const float* t, const float* f,
                             const float* c, const float* dist, const float* data_weight_scale) {
    if (!ctx) return set_error(nullptr, MVS_ERR_INVALID, "ctx is NULL");
    MVS_REQUIRE(ctx, n_rigs > 0 && num_views && R && t && f && c, "mvs_set_camera_rigs: need n_rigs >= 1 and the camera arrays");
    int vmax = 0;
    for (int r = 0; r < n_rigs; ++r) {
        MVS_REQUIRE(ctx, num_views[r] > 0 && num_views[r] <= kMaxViews, "mvs_set_camera_rigs: rig %d has %d views (1..%d)", r,
                    num_views[r], kMaxViews);
        MVS_REQUIRE(ctx, !data_weight_scale || (isfinite(data_weight_scale[r]) && data_weight_scale[r] > 0.f),
                    "mvs_set_camera_rigs: rig %d has data_weight_scale %g (want a finite positive scale)", r,
                    data_weight_scale ? data_weight_scale[r] : 1.f);
        vmax = std::max(vmax, num_views[r]);
    }
    if (dist)
        for (int r = 0; r < n_rigs; ++r)
            for (int v = 0; v < num_views[r]; ++v)
                for (int k = 0; k < 5; ++k)
                    MVS_REQUIRE(ctx, isfinite(dist[((size_t)r * vmax + v) * 5 + k]),
                                "mvs_set_camera_rigs_dist: rig %d view %d has distortion coefficient %d = %g (want finite)", r, v, k,
                                dist[((size_t)r * vmax + v) * 5 + k]);
    MVS_CUDA_OK(ctx, cudaSetDevice(ctx->device));
    std::vector<Rig> rigs((size_t)n_rigs);
    for (int r = 0; r < n_rigs; ++r) {
        Rig& g = rigs[r];
        memset(&g, 0, sizeof(g));
        g.num_views = num_views[r];
        g.dw_scale = data_weight_scale ? data_weight_scale[r] : 1.f;
        for (int v = 0; v < g.num_views; ++v) {
            const size_t i = (size_t)r * vmax + v;           // host arrays padded to vmax views
            memcpy(g.cam[v].R, R + 9 * i, 9 * sizeof(float));
            memcpy(g.cam[v].t, t + 3 * i, 3 * sizeof(float));
            memcpy(g.cam[v].f, f + 2 * i, 2 * sizeof(float));
            memcpy(g.cam[v].c, c + 2 * i, 2 * sizeof(float));
            if (!dist) continue;
            const float* d = dist + 5 * i;
            g.dist[v] = Dist{d[0], d[1], d[2], d[3], d[4], {0.f, 0.f, 0.f}};
            for (int k = 0; k < 5; ++k) g.distorted |= d[k] != 0.f;  // all zero: the pinhole instructions, bit for bit
        }
    }
    // no kernel may still read the table it replaces
    MVS_CUDA_OK(ctx, cudaDeviceSynchronize());
    if (int rc = dev_grow(ctx, ctx->rigs_dev, (size_t)n_rigs)) return rc;
    MVS_CUDA_OK(ctx, cudaMemcpy(ctx->rigs_dev.p, rigs.data(), (size_t)n_rigs * sizeof(Rig), cudaMemcpyHostToDevice));
    ctx->rigs = std::move(rigs);
    ctx->vmax = vmax;
    ctx->have_cams = true;
    ctx->have_kp = false;                                   // keypoints are per view: must be set again
    ctx->slot_rigs = nullptr;                               // so are the slots' rigs
    return MVS_OK;
}

int mvs_set_camera_rigs(mvs_ctx* ctx, int n_rigs, const int* num_views, const float* R, const float* t, const float* f,
                        const float* c, const float* data_weight_scale) {
    return mvs_set_camera_rigs_dist(ctx, n_rigs, num_views, R, t, f, c, nullptr, data_weight_scale);
}

int mvs_set_cameras(mvs_ctx* ctx, int V, const float* R, const float* t, const float* f, const float* c) {
    if (!ctx) return set_error(nullptr, MVS_ERR_INVALID, "ctx is NULL");
    MVS_REQUIRE(ctx, V > 0 && V <= kMaxViews && R && t && f && c, "mvs_set_cameras: need 1..%d views", kMaxViews);
    return mvs_set_camera_rigs(ctx, 1, &V, R, t, f, c, nullptr);
}

int mvs_set_frame_rigs(mvs_ctx* ctx, const int* rig_host) {
    if (!ctx) return set_error(nullptr, MVS_ERR_INVALID, "ctx is NULL");
    MVS_REQUIRE(ctx, ctx->ws.B > 0 && ctx->have_cams, "mvs_set_frame_rigs: set cameras and batch first");
    MVS_REQUIRE(ctx, rig_host, "mvs_set_frame_rigs: NULL array");
    const int B = ctx->ws.B, n = (int)ctx->rigs.size();
    for (int b = 0; b < B; ++b)
        MVS_REQUIRE(ctx, rig_host[b] >= 0 && rig_host[b] < n, "mvs_set_frame_rigs: slot %d names rig %d, the context has %d", b,
                    rig_host[b], n);
    MVS_CUDA_OK(ctx, cudaSetDevice(ctx->device));
    MVS_CUDA_OK(ctx, cudaDeviceSynchronize());              // no kernel may still read the rows it replaces
    MVS_CUDA_OK(ctx, cudaMemcpy(ctx->ws.slot_rig, rig_host, (size_t)B * sizeof(int), cudaMemcpyHostToDevice));
    ctx->slot_rig_host.assign(rig_host, rig_host + B);
    ctx->slot_rigs = ctx->ws.slot_rig;
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
    if ((rc = dev_alloc(ctx, &w.slot_rig, B))) return rc;
    ctx->slot_rigs = nullptr;
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
    if ((rc = closure_set_attributes(ctx)) || (rc = resident_set_attributes(ctx)) || (rc = tc_set_attributes(ctx)) ||
        (rc = sdf_set_attributes(ctx)))
        return rc;
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
    const size_t n = (size_t)ctx->vmax * w.B * ctx->m.K;
    const int rc = ensure_keypoint_ws(ctx);
    if (rc) return rc;
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

int mvs_set_joints3d(mvs_ctx* ctx, const float* gt_xyz, const float* conf, int enable, int on_device, void* stream) {
    if (!ctx) return set_error(nullptr, MVS_ERR_INVALID, "ctx is NULL");
    MVS_REQUIRE(ctx, ctx->have_model && ctx->ws.B > 0, "mvs_set_joints3d: set the model and the batch first");
    if (!enable) { ctx->loss.j3d_on = 0; ctx->j3d_enabled = false; return MVS_OK; }
    MVS_REQUIRE(ctx, gt_xyz && conf, "mvs_set_joints3d: NULL array");
    MVS_CUDA_OK(ctx, cudaSetDevice(ctx->device));
    Workspace& w = ctx->ws;
    const size_t n = (size_t)w.B * ctx->m.K;
    int rc;
    if (!w.j3d_xyz) {
        if ((rc = dev_alloc(ctx, &w.j3d_xyz, n * 3))) return rc;
        if ((rc = dev_alloc(ctx, &w.j3d_conf, n))) return rc;
    }
    cudaStream_t st = (cudaStream_t)stream;
    const cudaMemcpyKind kind = on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
    MVS_CUDA_OK(ctx, cudaMemcpyAsync(w.j3d_xyz, gt_xyz, n * 3 * sizeof(float), kind, st));
    MVS_CUDA_OK(ctx, cudaMemcpyAsync(w.j3d_conf, conf, n * sizeof(float), kind, st));
    if (!on_device) MVS_CUDA_OK(ctx, cudaStreamSynchronize(st));
    ctx->loss.j3d_on = 1;
    ctx->j3d_enabled = true;
    return MVS_OK;
}

int mvs_closure(mvs_ctx* ctx, const float* params_dev, float* loss_dev, float* grad_dev, float* joints_dev,
                float* proj_dev, float* verts_dev, void* stream) {
    if (!ctx) return set_error(nullptr, MVS_ERR_INVALID, "ctx is NULL");
    MVS_REQUIRE(ctx, ctx->have_model && ctx->have_cams && ctx->have_kp && ctx->have_loss && ctx->ws.B > 0,
                "mvs_closure: model, cameras, batch, keypoints and loss config must be set first");
    MVS_REQUIRE(ctx, params_dev, "mvs_closure: params_dev is NULL");
    if (int rc = batch_rigs(ctx, "mvs_closure")) return rc;
    MVS_CUDA_OK(ctx, cudaSetDevice(ctx->device));
    return evaluate_closure(ctx, params_dev, loss_dev, grad_dev, joints_dev, proj_dev, verts_dev, (cudaStream_t)stream);
}

int mvs_forward(mvs_ctx* ctx, const float* params_dev, float* joints_dev, float* verts_dev, void* stream) {
    if (!ctx) return set_error(nullptr, MVS_ERR_INVALID, "ctx is NULL");
    MVS_REQUIRE(ctx, ctx->have_model && ctx->ws.B > 0, "mvs_forward: model and batch must be set first");
    MVS_REQUIRE(ctx, params_dev, "mvs_forward: params_dev is NULL");
    MVS_CUDA_OK(ctx, cudaSetDevice(ctx->device));
    return launch_closure(ctx, params_dev, nullptr, nullptr, joints_dev, nullptr, verts_dev, (cudaStream_t)stream, true);
}

int mvs_forward_vjp(mvs_ctx* ctx, const float* params_dev, const float* djoints_dev, const float* dverts_dev,
                    float* dparams_dev, void* stream) {
    if (!ctx) return set_error(nullptr, MVS_ERR_INVALID, "ctx is NULL");
    MVS_REQUIRE(ctx, ctx->have_model && ctx->ws.B > 0, "mvs_forward_vjp: model and batch must be set first");
    MVS_REQUIRE(ctx, params_dev && dparams_dev, "mvs_forward_vjp: params_dev and dparams_dev are required");
    MVS_REQUIRE(ctx, djoints_dev || dverts_dev, "mvs_forward_vjp: give djoints_dev, dverts_dev or both");
    MVS_CUDA_OK(ctx, cudaSetDevice(ctx->device));
    return launch_forward_vjp(ctx, params_dev, djoints_dev, dverts_dev, dparams_dev, (cudaStream_t)stream);
}

int mvs_vposer_decode(mvs_ctx* ctx, const float* params_dev, float* body_pose_dev, void* stream) {
    if (!ctx) return set_error(nullptr, MVS_ERR_INVALID, "ctx is NULL");
    MVS_REQUIRE(ctx, ctx->have_model && ctx->ws.B > 0 && ctx->m.vp_w1, "mvs_vposer_decode: model, batch and mvs_set_vposer first");
    MVS_REQUIRE(ctx, params_dev && body_pose_dev, "mvs_vposer_decode: NULL argument");
    MVS_CUDA_OK(ctx, cudaSetDevice(ctx->device));
    return launch_vposer_decode(ctx, params_dev, body_pose_dev, (cudaStream_t)stream);
}

int mvs_render(mvs_ctx* ctx, int n_frames, const float* verts_dev, const float* keypoints_dev, const int* rig_dev,
               const unsigned char* background_dev, unsigned char* image_dev, int* face_dev, float* depth_dev,
               const mvs_render_config* cfg, void* stream) {
    if (!ctx) return set_error(nullptr, MVS_ERR_INVALID, "ctx is NULL");
    MVS_REQUIRE(ctx, ctx->have_model && ctx->m.F > 0 && ctx->m.faces, "mvs_render: needs a model with faces (mvs_set_model)");
    MVS_REQUIRE(ctx, ctx->m.vf_ptr, "mvs_render: the model's faces name vertices out of range");
    MVS_REQUIRE(ctx, ctx->have_cams, "mvs_render: set the cameras first");
    MVS_REQUIRE(ctx, n_frames >= 1, "mvs_render: n_frames = %d (want >= 1)", n_frames);
    MVS_REQUIRE(ctx, verts_dev, "mvs_render: verts_dev is NULL");
    MVS_REQUIRE(ctx, image_dev || face_dev || depth_dev, "mvs_render: every output is NULL");
    MVS_REQUIRE(ctx, cfg, "mvs_render: NULL config");
    MVS_REQUIRE(ctx, cfg->width >= 1 && cfg->width <= 8192 && cfg->height >= 1 && cfg->height <= 8192,
                "mvs_render: image size %d x %d (want 1 .. 8192 each)", cfg->width, cfg->height);
    for (int c = 0; c < 3; ++c)
        MVS_REQUIRE(ctx, isfinite(cfg->base_color[c]) && cfg->base_color[c] >= 0.f && cfg->base_color[c] <= 1.f,
                    "mvs_render: base_color[%d] = %g (want [0, 1])", c, cfg->base_color[c]);
    MVS_REQUIRE(ctx, isfinite(cfg->ambient) && cfg->ambient >= 0.f && cfg->ambient <= 1.f, "mvs_render: ambient = %g (want [0, 1])",
                cfg->ambient);
    MVS_REQUIRE(ctx, isfinite(cfg->marker_radius) && cfg->marker_radius >= 0.f, "mvs_render: marker_radius = %g (want finite, >= 0)",
                cfg->marker_radius);
    MVS_REQUIRE(ctx, rig_dev || ctx->rigs.size() == 1,
                "mvs_render: the context has %d camera rigs and no per-frame rigs were given", (int)ctx->rigs.size());
    MVS_CUDA_OK(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = (cudaStream_t)stream;
    if (rig_dev)
        if (int rc = check_frame_rigs(ctx, "mvs_render", rig_dev, n_frames, st)) return rc;
    return render_launch(ctx, n_frames, verts_dev, keypoints_dev, rig_dev, background_dev, image_dev, face_dev, depth_dev, *cfg, st);
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
