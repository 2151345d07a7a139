// Internal types of libmvsmpl.so (not part of the ABI).
#pragma once
#include <utility>
#include <cuda_runtime.h>
#include <stdint.h>
#include <string>
#include <vector>

#include "../../include/mvsmpl.h"
#include "mvs_math.cuh"

namespace mvs {

// ----------------------------------------------------------------------------- tiling constants
constexpr int kTileF = 64;     // frames per CTA tile of the vertex kernels
constexpr int kTileV = 32;     // vertices per CTA tile
constexpr int kTileC = 3 * kTileV;
constexpr int kGemmKC = 16;    // K chunk of the forward blend-shape contraction
constexpr int kVertThreads = 256;
constexpr int kFrameThreads = 128;
constexpr int kSkinFloats = kJoints * 12;           // 288 = 24 x (3x4)
constexpr int kPartFloats = kSkinFloats + kFeatPad; // per (strip, frame) partial of the vertex backward

struct Parents { int p[kJoints]; };

struct CamSet {
    int num_views;
    CamF cam[kMaxViews];
};

// Everything a kernel needs to know about the loss (passed by value)
struct LossParams {
    float data_weight, body_pose_weight, shape_weight, bending_prior_weight, coll_loss_weight, rho;
    int body_prior, use_joints_conf, use_vposer, fix_shape, interpenetration, sdf_grid, sdf_all_faces;
    unsigned frozen_mask;
    int num_gaussians;
    int anchor_on;
};

// Model constants resident in HBM.  Layouts chosen for the kernels, not the reference's:
//   Qk  [3N][224]   row (3n+c) = [posedirs[:,3n+c] (207) | shapedirs[n,c,:] (10) | v_template[n,c] | 0-pad]
//                   so that v_posed = Phi . Qk^T with Phi = [pose_feature | betas | 1]  (one contraction
//                   replaces lbs.py:179 + :194-203); K-contiguous = "K-major B operand" for UMMA/TMA.
//   Jt [24][3], JS [24][3][10]  pre-contracted rest-joint regressor: J = Jt + JS.betas  (lbs.py:183 folded
//                   through lbs.py:179; computed in fp64 at upload)
//   ell_j/ell_w [N][KW]  skinning weights in ELL form (KW = max non-zeros per vertex, 4 for SMPL)
//   Wd  [N][24]     dense skinning weights (vertex backward)
struct DevModel {
    int N = 0, F = 0, KW = 0;
    float* Qk = nullptr;
    float* Jt = nullptr;
    float* JS = nullptr;
    int* parents = nullptr;
    int* ell_j = nullptr;
    float* ell_w = nullptr;
    float* Wd = nullptr;
    float* ST = nullptr;      // [N][3][11] shapedirs row | template, fp32 (skinning kernel of the tensor-core path)
    int* faces = nullptr;
    int tri0[3] = {0, 0, 0};          // vertex ids of face 0 (the triangle the as-written SDF term sees)
    // keypoints: k-th keypoint = sum_e kp_w[e] * v[kp_vidx[e]]  (+ posed chain joint kp_chain[k] if >= 0) + transl
    int K = 0, n_kp_entries = 0, nsup = 0;
    int* kp_ptr = nullptr;    // [K+1]
    int* kp_vidx = nullptr;   // vertex id
    int* kp_spos = nullptr;   // position of that vertex in the support list
    float* kp_w = nullptr;
    int* kp_chain = nullptr;  // [K]
    int* sup = nullptr;       // [nsup] sorted unique vertex ids touched by any keypoint
    int* sup_then_all = nullptr;  // [nsup + N] the support list followed by 0..N-1 (backward list with the SDF term)
    int* sup_ptr = nullptr;   // [nsup+1] transposed structure: support vertex -> (keypoint, weight)
    int* sup_k = nullptr;
    float* sup_w = nullptr;
    int* supj_ptr = nullptr;  // [25] per joint: support vertices it skins (frame-resident adjoint)
    int* supj_i = nullptr;
    float* supj_w = nullptr;
    // GMM prior
    int M = 0;
    float* gmm_means = nullptr;     // [M][69]
    float* gmm_prec = nullptr;      // [M][69][69] symmetrised
    float* gmm_lognllw = nullptr;   // [M]  log(nll_weights)
    // VPoser decoder (mvs_set_vposer): [out][in] as uploaded and the transposes [in][out] (coalesced mat-vec both ways)
    float *vp_w1 = nullptr, *vp_w2 = nullptr, *vp_w3 = nullptr, *vp_w1t = nullptr, *vp_w2t = nullptr, *vp_w3t = nullptr;
    float *vp_b1 = nullptr, *vp_b2 = nullptr, *vp_b3 = nullptr;
};

// Per-batch workspace (slot-indexed: slot = position in the active-frame list)
struct Workspace {
    int B = 0, ldA = 0;               // ldA = B rounded up to kTileF
    int na_bound = 0;                 // host-side upper bound of *na (grids of the dense-regime rounds are sized by it;
                                      // equals B outside mvs_lbfgs_run / while the active list is full)
    int nstrips_max = 0;
    int* fidx = nullptr;              // [B] active list: slot -> frame
    int* na = nullptr;                // [1] number of active slots
    float* Phi = nullptr;             // [ldA][224]
    float* PhiTc = nullptr;           // [2][ldA][224] pose feature split into TF32 hi | lo parts (A operand of the tensor-core contraction)
    float* At = nullptr;              // [288][ldA]   skinning transforms, frame fastest
    float* gchain = nullptr;          // [B][24][3]   posed chain joints (model_type 'smpl')
    float* pose_cache = nullptr;      // [B][864] per FRAME: R | J | Gam | g | A of the pending trial point (frame_step -> frame_step)
    int* pose_valid = nullptr;        // [B]
    float* slot_tr = nullptr;         // [B][4] translation of the frame in each slot (dense-regime kernels index by slot only)
    float* vposed = nullptr;          // [B][nvmax][3]
    float* verts = nullptr;           // [B][nvmax][3]  (pre-transl)
    float* dv = nullptr;              // [B][nsup + N][3]
    float* part = nullptr;            // [nstrips_max][ldA][kPartFloats]
    float* data_loss = nullptr;       // [B]
    float* pen_loss = nullptr;        // [B]
    float* dtransl = nullptr;         // [B][3]
    float* dgchain = nullptr;         // [B][24][3]
    float* gt_uv = nullptr;           // [V][B][K][2]
    float* conf = nullptr;            // [V][B][K]
    float* joint_w = nullptr;         // [K]
    float* loss_scratch = nullptr;    // [B] when the caller passes no loss pointer
    float* grad_scratch = nullptr;    // [B][86]
    float* anchor = nullptr;          // [B][86] quadratic anchor (sequence mode)
    float* anchor_w = nullptr;        // [B][86]
    // SDF scratch
    float* bbox_part = nullptr;       // [B][nbt][6]
    float* sdf_frame = nullptr;       // [B][16]  centre(3) scale(1) argmin/argmax ids etc.
    float* sdf_gcoord = nullptr;      // [B][N][3]
    float* sdf_valpart = nullptr;     // [B][nbt]
    float* bboxp = nullptr;           // [B][nchunks][12] per-chunk bbox partials written by the skinning kernel
    // dense regime (sdf_fused_kernel -> frame_step_kernel), P = 256-vertex blocks per frame
    float* sdf_parts5 = nullptr;      // [B][P][5] per 256-vertex block: value, d value/d local (3), <d value/d local, local>
    float* sdf_part = nullptr;        // [B][P][512] unit-factor partial adjoints (288 skin | 224 feature)
    int* sdf_pflag = nullptr;         // [B][P] 1 iff the block has vertices with a non-zero sample gradient
    unsigned char* sdf_box = nullptr; // [B] FrameBox
    // accelerated all-faces SDF (mvs_sdf_bins.cuh): per slot triangle corners, cell lists, ray-bin lists, meta (s_lo, s_scale, overflow)
    float* bins_tri = nullptr; int* bins_cell_ptr = nullptr; unsigned short* bins_cell_idx = nullptr;
    int* bins_ray_ptr = nullptr; unsigned short* bins_ray_idx = nullptr; float* bins_meta = nullptr;
};

struct FrameBox {                     // bounding box of one frame's mesh (fitting.py:352-359)
    float centre[3];
    float scale;
    int ilo[3], ihi[3];
    int cmax;                         // coordinate with the largest extent
    float pad;
};

// sdf_fused_kernel gives a CTA 1 or 2 blocks of 256 vertices (results are emitted per block and do not depend on it).
// Measured on the benchmark (us per launch, ~150 active frames): 1 block 40.0, 2 blocks 37.7, 3: 40.7, 4: 42, 8: 54,
// 16: 76 -- the few expensive blocks near the cone must not pile up in one CTA, and small CTAs balance better than the
// shorter prologue of large ones saves.
constexpr int kSdfMaxPasses = 8;
__host__ __device__ inline int sdf_passes_for(int na, int nblocks, int cta_slots) {
    return (long long)na * nblocks > 2LL * cta_slots ? 2 : 1;
}

enum KernelId {
    KID_FRAME_FWD = 0, KID_VERTEX_FWD, KID_SDF_BBOX, KID_SDF_SAMPLE, KID_SDF_FINALIZE, KID_KEYPOINT, KID_VERTEX_BWD,
    KID_FRAME_BWD, KID_LBFGS_ADVANCE, KID_LBFGS_COMPACT, KID_SDF_GRID, KID_MISC, KID_RESIDENT_CLOSURE, KID_RESIDENT_LBFGS,
    KID_SDF_FRAME, KID_FRAME_STEP, KID_VERTEX_FWD_TC, KID_SKIN, KID_COUNT
};
static_assert(KID_COUNT == MVS_NUM_KERNEL_IDS, "kernel id table out of sync with mvsmpl.h");

struct Profiler {
    unsigned mask = 0;
    std::vector<cudaEvent_t> ev[KID_COUNT];     // start/stop pairs
    size_t used[KID_COUNT] = {0};
};

}  // namespace mvs

struct mvs_ctx {
    int device = 0;
    int sm_count = 0;
    std::string err;
    long long launches = 0;
    mvs::DevModel m;
    mvs::CamSet cams{};
    mvs::LossParams loss{};
    mvs::Workspace ws;
    mvs::Parents parents{};
    bool attr_done = false, attr_done_res = false, attr_done_step = false;
    int attr_res_lbfgs_smem = 0;
    bool anchor_enabled = false;
    int exec_mode = 0;               // 0 auto (frame-resident kernels where they apply), 1 batched kernels only
    bool have_model = false, have_cams = false, have_kp = false, have_loss = false;
    std::vector<void*> allocs;       // everything cudaMalloc'ed, freed in mvs_destroy
    void* lbfgs = nullptr;           // optimiser state (mvs_lbfgs.cu)
    mvs::Profiler prof;
    void* tc = nullptr;              // tensor-core path state (mvs_tc.cu)
    float* rest_joints = nullptr;    // [K,3] keypoints of the rest pose at scale rest_scale (mvs_init.cu), computed once
    float rest_scale = -1.f;
    int* stage_rng = nullptr;        // [B][2] per-frame slice of the stage table (mvs_fit_seq), device
};

namespace mvs {
int set_error(mvs_ctx* ctx, int code, const char* fmt, ...);
#define MVS_CUDA_OK(ctx, expr)                                                              \
    do {                                                                                    \
        cudaError_t _e = (expr);                                                            \
        if (_e != cudaSuccess)                                                              \
            return mvs::set_error(ctx, MVS_ERR_CUDA, "%s failed: %s (%s:%d)", #expr,        \
                                  cudaGetErrorString(_e), __FILE__, __LINE__);              \
    } while (0)

void prof_mark(mvs_ctx* ctx, int kid, cudaStream_t st);   // records one event of a start/stop pair when enabled
// every kernel launch of the library goes through this macro: launch counter + optional event timing
#define MVS_LAUNCH(ctx, kid, st, ...)                                     \
    do {                                                                  \
        if ((ctx)->prof.mask >> (kid) & 1u) mvs::prof_mark(ctx, kid, st); \
        __VA_ARGS__;                                                      \
        if ((ctx)->prof.mask >> (kid) & 1u) mvs::prof_mark(ctx, kid, st); \
        (ctx)->launches++;                                                \
    } while (0)

// Programmatic dependent launch (sm_90+): the kernel may be scheduled while its predecessor in the stream is still
// draining; it must execute pdl_wait() before touching anything the predecessor wrote (here: first statement).  The
// dense-regime rounds are chains of short dependent kernels, so this takes the launch latency of every link off the
// critical path.  Expands to a plain launch when the attribute is not supported.
// pdl_wait(): predecessor complete and its writes visible; then let OUR successor be scheduled as soon as all of our
// CTAs have started (its CTAs park in their own pdl_wait, prologue done, until this grid has drained).
__device__ __forceinline__ void pdl_wait() {
    asm volatile("griddepcontrol.wait;" ::: "memory");
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}
template <class... KArgs, class... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}

// v = hi + lo with hi = TF32(v) (round to nearest, ties away) and lo = TF32(v - hi); v - hi is exact in fp32.  The tensor-core
// contraction multiplies hi*hi + lo*hi + hi*lo (error-compensated "3xTF32"): the dropped lo*lo term is 2^-22 of a product.
__device__ __forceinline__ void tf32_split(float v, float& hi, float& lo) {
    unsigned u;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(v));
    hi = __uint_as_float(u);
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(v - hi));
    lo = __uint_as_float(u);
}

// Warp-wide extreme of a float with the arg-index of its first occurrence ("ties -> lowest vertex index", like
// torch.min / max on CPU) in two redux.sync instructions: floats are mapped to unsigned keys of the same order
// (-0 is folded into +0 first, so equal floats have equal keys).
__device__ __forceinline__ unsigned float_order_key(float f) {
    const unsigned u = __float_as_uint(f + 0.0f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float float_from_order_key(unsigned k) {
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}
__device__ __forceinline__ void warp_argmin(float& v, int& idx) {
    const unsigned k = float_order_key(v);
    const unsigned kmin = __reduce_min_sync(0xffffffffu, k);
    idx = (int)__reduce_min_sync(0xffffffffu, k == kmin ? (unsigned)idx : 0x7fffffffu);
    v = float_from_order_key(kmin);
}
__device__ __forceinline__ void warp_argmax(float& v, int& idx) {
    const unsigned k = float_order_key(v);
    const unsigned kmax = __reduce_max_sync(0xffffffffu, k);
    idx = (int)__reduce_min_sync(0xffffffffu, k == kmax ? (unsigned)idx : 0x7fffffffu);
    v = float_from_order_key(kmax);
}

template <class T> int dev_alloc(mvs_ctx* ctx, T** p, size_t count);
template <class T> int dev_upload(mvs_ctx* ctx, T** p, const T* host, size_t count);

// closure launcher (mvs_closure.cu): evaluates all active slots.  x_dev [B][86].
int launch_closure(mvs_ctx* ctx, const float* x_dev, float* loss_dev, float* grad_dev, float* joints_dev,
                   float* proj_dev, float* verts_dev, cudaStream_t st, bool geometry_only = false);
int launch_sdf_terms(mvs_ctx* ctx, const float* x_dev, cudaStream_t st);   // mvs_sdf.cu
// mvs_resident.cu: frame-resident (one CTA per frame) closure and whole-stage optimiser for the sparse regime
bool resident_closure_available(const mvs_ctx* ctx);
int launch_vposer_decode(mvs_ctx* ctx, const float* x_dev, float* body_pose_dev, cudaStream_t st);
int launch_closure_resident(mvs_ctx* ctx, const float* x_dev, float* loss_dev, float* grad_dev, float* joints_dev,
                            float* proj_dev, cudaStream_t st);
bool resident_lbfgs_available(const mvs_ctx* ctx, int history);
int launch_lbfgs_resident(mvs_ctx* ctx, float* params_dev, const void* lbfgs_cfg, int history, const void* lp_tab_dev,
                          const void* lp_tab_host, int nstages, void* frame_scalars_out, float* last_grad_dev, cudaStream_t st,
                          const void* stage_rng_dev = nullptr);
// dense regime (SDF term): per round  posedirs_gemm_tc -> skin -> sdf_fused -> frame_step
bool hybrid_available(const mvs_ctx* ctx);
int launch_vertex_fwd_dense(mvs_ctx* ctx, cudaStream_t st, bool allow_tc = true, bool need_vposed = true);                                   // mvs_closure.cu
int launch_frame_fwd(mvs_ctx* ctx, const float* x_dev, cudaStream_t st);                      // mvs_closure.cu
int launch_sdf_fused(mvs_ctx* ctx, cudaStream_t st);   // mvs_sdf.cu
// mvs_tc.cu: wgmma / TMA dense vertex forward
int tc_upload_model(mvs_ctx* ctx, const float* Qk_host);
bool tc_available(const mvs_ctx* ctx);
int launch_vertex_fwd_tc(mvs_ctx* ctx, cudaStream_t st, bool need_vposed = true);
int tc_check_error(mvs_ctx* ctx);
float* tc_poffT(mvs_ctx* ctx);                 // [3N][ldA] pose offsets of the tensor-core contraction (allocated on first use)
int tc_prepare(mvs_ctx* ctx);                  // tensor maps + pose-offset buffer (idempotent)
int launch_frame_step(mvs_ctx* ctx, float* params_dev, const void* lbfgs_state, const void* lbfgs_cfg, int nstages,
                      cudaStream_t st);
int frame_step_begin_run(mvs_ctx* ctx, cudaStream_t st);                 // mvs_resident.cu
int launch_frame_fwd_dense(mvs_ctx* ctx, const float* x_dev, const void* lbfgs_state, int nstages, cudaStream_t st);   // mvs_resident.cu
bool resident_lbfgs_available_for(const mvs_ctx* ctx, const LossParams& lp, int history);
bool hybrid_available_for(const mvs_ctx* ctx, const LossParams& lp);
int dense_regime_closure(mvs_ctx* ctx, const float* x_dev, float* loss_dev, float* grad_dev, cudaStream_t st);   // mvs_lbfgs.cu
int make_loss_params(mvs_ctx* ctx, const mvs_loss_config* c, LossParams* out);      // mvs_api.cu: validation + conversion
int sdf_grid_launch(mvs_ctx* ctx, float* phi, const int* faces, int num_faces, const float* verts, int batch,
                    int n_verts, int G, cudaStream_t st);
}  // namespace mvs
