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

// Depth-level schedule of the kinematic tree: joints of one level only depend on the level above (forward) / below
// (adjoint), so a level is processed by parallel lane groups and the 23-step serial chain becomes <= 9 level steps
// for SMPL.  Children are listed in DESCENDING index order: gathering them in that order reproduces the summation
// order of the plain "for j = 23 .. 1" reverse sweep bit for bit.
struct ChainSched {
    int nlev;
    unsigned char lev_ptr[kJoints + 1], lev_j[kJoints];
    unsigned char ch_ptr[kJoints + 1], ch_j[kJoints];
};

// One camera rig of the context's table (mvs_set_camera_rigs): its views, their number and the scale of every stage's
// data_weight for the frames that name it.  Lives in device memory; kernels reach it through frame_rig() only.
struct __align__(16) Rig {
    CamF cam[kMaxViews];
    int num_views;
    float dw_scale;
    int pad[2];
};
static_assert(sizeof(CamF) == 64 && sizeof(Rig) % 16 == 0, "rig layout (float4 loads of a camera)");

// Where a kernel finds each frame's rig: the context's table and the rig index of every row it indexes frames by (frame of
// a stream, slot of a batch or lane of a dense run); of == NULL: every row has rig 0 (a table of one rig).
struct RigSet {
    const Rig* rig;
    const int* of;
};

// What a kernel reads of a frame's rig: the rig's cameras (device memory), view count and data-weight scale
struct FrameRig {
    const CamF* cam;
    int num_views;
    float dw_scale;
};
#ifdef __CUDACC__
__device__ __forceinline__ FrameRig frame_rig(const RigSet& rs, int row) {
    const Rig* r = rs.rig + (rs.of ? __ldg(rs.of + row) : 0);
    return FrameRig{r->cam, __ldg(&r->num_views), __ldg(&r->dw_scale)};
}
// camera v of a frame's rig, into registers (four 16-byte loads)
__device__ __forceinline__ CamF rig_camera(const FrameRig& fr, int v) {
    const float4* p = reinterpret_cast<const float4*>(fr.cam + v);
    CamF c;
    float4* d = reinterpret_cast<float4*>(&c);
#pragma unroll
    for (int i = 0; i < 4; ++i) d[i] = __ldg(p + i);
    return c;
}
#endif

// Everything a kernel needs to know about the loss (passed by value)
struct LossParams {
    float data_weight, body_pose_weight, shape_weight, bending_prior_weight, coll_loss_weight, rho;
    int body_prior, use_joints_conf, use_vposer, fix_shape, interpenetration, sdf_grid, sdf_all_faces;
    unsigned frozen_mask;
    int num_gaussians;
    int anchor_on;
    int j3d_on;                       // 3-D joint term (mvs_set_joints3d)
};

inline bool sdf_term_on(const LossParams& lp) { return lp.interpenetration && lp.coll_loss_weight > 0.f; }

// execution regime of an optimiser run (DESIGN.md section 4)
enum Regime { kResident, kDense, kBatched };

// Model constants resident in HBM.  Layouts chosen for the kernels, not the reference's:
//   Qk  [3N][224]   row (3n+c) = [posedirs[:,3n+c] (207) | shapedirs[n,c,:] (10) | v_template[n,c] | 0-pad]
//                   so that v_posed = Phi . Qk^T with Phi = [pose_feature | betas | 1]  (one contraction
//                   replaces lbs.py:179 + :194-203); K-contiguous = "K-major B operand" for UMMA/TMA.
//   Jt [24][3], JS [24][3][10]  pre-contracted rest-joint regressor: J = Jt + JS.betas  (lbs.py:183 folded
//                   through lbs.py:179; computed in fp64 at upload)
//   ell_j/ell_w [N][KW]  skinning weights in ELL form (KW = max non-zeros per vertex, 4 for SMPL)
//   Wd  [N][24]     dense skinning weights (vertex backward)
// Read-only after upload: every array here may be shared with other contexts that uploaded the same bytes (upload_consts in
// mvs_api.cu), so no kernel or host path writes through these pointers; they are const so that the compiler holds to it.
// The per-call pointers that ride along with them (ResidentModel's anchor / 3-D targets) are swapped, never written through.
struct DevModel {
    int N = 0, F = 0, KW = 0;
    const float* Qk = nullptr;
    const float* Jt = nullptr;
    const float* JS = nullptr;
    const int* parents = nullptr;
    const int* ell_j = nullptr;
    const float* ell_w = nullptr;
    const float* Wd = nullptr;
    const float* ST = nullptr;  // [N][3][11] shapedirs row | template, fp32 (skinning kernel of the tensor-core path)
    const int* faces = nullptr;
    int tri0[3] = {0, 0, 0};          // vertex ids of face 0 (the triangle the as-written SDF term sees)
    // keypoints: k-th keypoint = sum_e kp_w[e] * v[kp_vidx[e]]  (+ posed chain joint kp_chain[k] if >= 0) + transl
    int K = 0, n_kp_entries = 0, nsup = 0;
    const int* kp_ptr = nullptr;    // [K+1]
    const int* kp_vidx = nullptr;   // vertex id
    const int* kp_spos = nullptr;   // position of that vertex in the support list
    const float* kp_w = nullptr;
    const int* kp_chain = nullptr;  // [K]
    const int* sup = nullptr;       // [nsup] sorted unique vertex ids touched by any keypoint
    const int* sup_then_all = nullptr;  // [nsup + N] the support list followed by 0..N-1 (backward list with the SDF term)
    const int* sup_ptr = nullptr;   // [nsup+1] transposed structure: support vertex -> (keypoint, weight)
    const int* sup_k = nullptr;
    const float* sup_w = nullptr;
    const int* supj_ptr = nullptr;  // [25] per joint: support vertices it skins (frame-resident adjoint)
    const int* supj_i = nullptr;
    const float* supj_w = nullptr;
    // GMM prior
    int M = 0;
    const float* gmm_means = nullptr;     // [M][69]
    const float* gmm_prec = nullptr;      // [M][69][69] symmetrised
    const float* gmm_lognllw = nullptr;   // [M]  log(nll_weights)
    // VPoser decoder (mvs_set_vposer): [out][in] as uploaded and the transposes [in][out] (coalesced mat-vec both ways)
    const float *vp_w1 = nullptr, *vp_w2 = nullptr, *vp_w3 = nullptr, *vp_w1t = nullptr, *vp_w2t = nullptr, *vp_w3t = nullptr;
    const float *vp_b1 = nullptr, *vp_b2 = nullptr, *vp_b3 = nullptr;
};

struct FrameBox;
struct SdfFrameSetup;
// optimiser state and configuration (mvs_lbfgs_core.cuh), tensor-core path state (mvs_tc.cu)
struct LbfgsState;
struct LbfgsCfg;
struct FrameScalars;
struct TcState;
struct StreamState;                   // mvs_fit_stream scratch (mvs_lbfgs.cu)
struct SeqState;                      // mvs_fit_seq_stream, mvs_fit_shared_shape and mvs_refine_cameras scratch (mvs_lbfgs.cu)
struct SharedConsts;                  // model constants shared by the contexts that uploaded the same bytes (mvs_api.cu)

// A device array of the context that only grows (dev_grow): cap elements at p
template <class T> struct DevBuf {
    T* p = nullptr;
    size_t cap = 0;
};

// The frames a frame-resident run fits when they are not the context's batch (mvs_fit_stream): n frames, every array with
// row stride n (gt_uv [V][n][K][2], conf [V][n][K], j3d_xyz [n][K][3], j3d_conf [n][K]; the 3-D pair may be NULL; rig [n]
// or NULL: every frame has rig 0)
struct FrameInputs {
    int n;
    const float *gt_uv, *conf, *joint_w, *j3d_xyz, *j3d_conf;
    const int* rig;
};

// One chunk of a set of small problems solved by the batched chain's L-BFGS (DESIGN.md section 4): problems base .. base + n - 1
// in the optimiser's slots 0 .. n - 1, whose work items are i0 .. i0 + ni - 1.  Problem p owns the work items [beg[p], beg[p+1])
// and item i belongs to problem item_of[i].  Each work item writes its row of part: its loss, then its problem's gradient
// entries of the call (at most kPartCols - 1, the same for every item); the driver adds the rows per problem.
constexpr int kPartCols = 12;
struct ProblemChunk {
    const int* beg;                   // [P+1]
    const int* item_of;               // [items]
    float* part;                      // [items][kPartCols]
    int base, n, i0, ni;
};

// The shape step of mvs_fit_shared_shape (DESIGN.md section 4): a problem per sequence, a work item per frame (in.n = F: the
// row stride of every input)
struct ShapeArgs {
    FrameInputs in;
    const float* params;              // [F][86] the frames' rows (poses held)
    int share_scale;                  // 1: scale (entry 85) is shared, 0: it stays per frame
};

// One view problem of mvs_refine_cameras: view `view` of rig `rig`, whose frames are frames[fbeg ..) of the call's rig-grouped
// frame list (the frames with that rig and a finite row, in call order), one work item each
struct CameraProblem {
    int rig, view, fbeg;
};

// The camera step of mvs_refine_cameras (DESIGN.md section 4).  A problem's variables are the entries kOffOrient .. +2 (rotation
// update) and kOffTransl .. +2 (centre update) of its slot's row; its closure is the 2-D data term of its view over its frames
// at the held keypoints q.
struct CameraArgs {
    FrameInputs in;                   // the call's frames (in.n = F: the row stride of gt_uv / conf)
    const float* q;                   // [F][K][3] held keypoints (with translation)
    const CamRefine* cr;              // [P] each problem's calibrated camera and centre map
    const CameraProblem* prob;        // [P]
    const int* frames;                // the rig-grouped frame list
    const Rig* rigs;                  // the context's rig table (intrinsics and data-weight scale)
    int K;
};

// The chaining run of mvs_fit_seq_stream (DESIGN.md section 4): a finished frame hands its slot (a CTA of the frame-resident
// kernel, a lane of the dense rounds) to its successor in the same sequence.  Frames of sequence s are [off[s], off[s+1]).
struct SeqChain {
    int n_act = 0;                    // sequences of this pass
    const int* act = nullptr;         // [n_act] their indices, ascending
    int* cur = nullptr;               // [S] in: each sequence's first frame of the pass (cold); out: its parked frame, -1 = done
    const int* off = nullptr;         // [S+1]
    int2 cold{0, 0}, warm{0, 0};      // slices of the run's stage table for cold and warm-started frames
    float reinit_loss = 0.f;          // a successor is warm iff its predecessor's final loss <= reinit_loss
    int park = 0;                     // 1: a cold successor leaves the run (it has earlier runs to pass first)
    int keep_pose = 0;                // 1: a warm frame keeps its own body-pose slot (axis-angle stages; fix_params)
    float* final_loss = nullptr;      // [F] or NULL
    long long* totals = nullptr;      // [4] iters, evals, NaN stops, largest evaluations of one CTA (frame-resident kernel)
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
    int kp_views = 0;                 // V of the allocated gt_uv / conf (the rig table's largest view count)
    int* slot_rig = nullptr;          // [B] rig of each slot (mvs_set_frame_rigs) or of each lane's frame (dense stream runs)
    float* gt_uv = nullptr;           // [V][B][K][2]
    float* conf = nullptr;            // [V][B][K]
    float* joint_w = nullptr;         // [K]
    float* loss_scratch = nullptr;    // [B] when the caller passes no loss pointer
    float* grad_scratch = nullptr;    // [B][86]
    float* anchor = nullptr;          // [B][86] quadratic anchor (sequence mode)
    float* anchor_w = nullptr;        // [B][86]
    float* j3d_xyz = nullptr;         // [B][K][3] 3-D joint targets (mvs_set_joints3d)
    float* j3d_conf = nullptr;        // [B][K]
    // SDF scratch
    FrameBox* sdf_frame = nullptr;    // [B] frame boxes of the batched chain's SDF term (launch_sdf_terms)
    float* sdf_gcoord = nullptr;      // [B][N][3]
    float* sdf_valpart = nullptr;     // [B][nbt]
    float* bboxp = nullptr;           // [B][nchunks][12] per-chunk bbox partials written by the skinning kernel
    // dense regime (sdf_fused_kernel -> frame_step_kernel), P = 256-vertex blocks per frame
    float* sdf_parts5 = nullptr;      // [B][P][5] per 256-vertex block: value, d value/d local (3), <d value/d local, local>
    float* sdf_part = nullptr;        // [B][P][512] unit-factor partial adjoints (288 skin | 224 feature)
    int* sdf_pflag = nullptr;         // [B][P] 1 iff the block has vertices with a non-zero sample gradient
    FrameBox* sdf_box = nullptr;      // [B] frame boxes of the dense rounds, written with the set-up, read by frame_step
    SdfFrameSetup* sdf_setup = nullptr;   // [B] by sdf_setup_kernel (at <= 4 frames by skin_small_kernel's last CTA of a frame)
    int* sdf_arrive = nullptr;        // [B] skin_small_kernel: chunk boxes of a frame written so far this round (0 between rounds)
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

// What sdf_fused needs of a frame before it touches a vertex: the frame box, triangle 0 in box coordinates, the cone it
// spans from the corner (-1,-1,-1) and the triangle's plane with their margins, the vertex-level pads, and the chunk-cull
// verdict of every 64-vertex chunk.  Computed once per frame and round (sdf_frame_setup in mvs_tc_dev.cuh), by sdf_setup_kernel
// after the skinning kernel or by skin_small_kernel's tail (<= 4 frames), instead of by every sdf_fused CTA.
constexpr int kSdfSkipWords = 8;      // chunk-cull bits for up to 256 chunks (16384 vertices); larger meshes are not culled
struct __align__(16) SdfFrameSetup {
    FrameBox fb;
    float tri[9];
    float cn[3][3], cm[3];
    float pn[3], pd, pm;
    float vpad[3], vpadp;
    float unused[2];
    unsigned skip[kSdfSkipWords];     // bit (c & 31) of word c / 32: no vertex of chunk c can see phi != 0
};
static_assert(sizeof(SdfFrameSetup) == 208, "SdfFrameSetup layout");

// Per-launch arguments of the set-up; rec == nullptr: skin_small_kernel does not compute it (SDF term off)
struct SdfSetupArgs {
    SdfFrameSetup* rec; FrameBox* boxout; int* arrive; const float* slot_tr;
    int f0, f1, f2, G, cull;          // triangle 0, grid size, cone/plane culls on (as-written semantics: one face)
};

// sdf_fused_kernel gives a CTA 1 or 2 blocks of 256 vertices (results are emitted per block and do not depend on it).
// Measured on the benchmark (us per launch, ~150 active frames): 1 block 40.0, 2 blocks 37.7, 3: 40.7, 4: 42, 8: 54,
// 16: 76 -- the few expensive blocks near the cone must not pile up in one CTA, and small CTAs balance better than the
// shorter prologue of large ones saves.  Re-measured once the prologue became a single load of the skinning kernel's set-up
// record (H100, one dense round, us per launch at 256 / 64 / 8 / 1 active frames): 1 block 65.5 / 28.8 / 15.8 / 17.0,
// 2: 54.2 / 30.1 / 19.6 / 20.2, 4: 54.8 / 29.8 / 22.6 / 21.9, 8: 52.7 / 28.9 / 25.4 / 24.5.  No setting beats this rule by
// more than the spread of a single sample (~3 %), so it stays.
constexpr int kSdfMaxPasses = 8;
__host__ __device__ inline int sdf_passes_for(int na, int nblocks, int cta_slots) {
    return (long long)na * nblocks > 2LL * cta_slots ? 2 : 1;
}

enum KernelId {
    KID_FRAME_FWD = 0, KID_VERTEX_FWD, KID_SDF_BBOX, KID_SDF_SAMPLE, KID_SDF_FINALIZE, KID_KEYPOINT, KID_VERTEX_BWD,
    KID_FRAME_BWD, KID_LBFGS_ADVANCE, KID_LBFGS_COMPACT, KID_SDF_GRID, KID_MISC, KID_RESIDENT_CLOSURE, KID_RESIDENT_LBFGS,
    KID_SDF_FRAME, KID_FRAME_STEP, KID_VERTEX_FWD_TC, KID_SKIN, KID_SDF_SETUP, KID_COUNT
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
    // camera rigs (mvs_set_camera_rigs; mvs_set_cameras is a table of one): host copy and device table
    std::vector<mvs::Rig> rigs;
    mvs::DevBuf<mvs::Rig> rigs_dev;
    int vmax = 0;                    // largest view count of the table: the view rows of every detection array
    std::vector<int> slot_rig_host;  // [B] per-slot rigs of mvs_set_frame_rigs
    const int* slot_rigs = nullptr;  // per-slot rigs the batch entry points read (ws.slot_rig), NULL: none given (rig 0)
    int* rig_bad = nullptr;          // [1] first frame of a stream whose rig index is out of range (check_frame_rigs)
    mvs::LossParams loss{};
    mvs::Workspace ws;
    mvs::Parents parents{};
    mvs::ChainSched chain{};         // level schedule of parents
    bool anchor_enabled = false;
    bool j3d_enabled = false;
    int exec_mode = 0;               // mvs_set_exec_mode: 0 auto, 1 batched chain only, 2 stage barriers, 3 dense-round closures
    bool have_model = false, have_cams = false, have_kp = false, have_loss = false;
    std::vector<void*> allocs;       // everything cudaMalloc'ed, freed in mvs_destroy (dev_alloc / dev_free)
    std::vector<mvs::SharedConsts*> consts;   // the entries holding ctx->m's arrays, dropped by mvs_destroy (upload_consts)
    // The state objects below are set only once complete, and released by mvs_destroy (release_fit_state, release_tc_state)
    mvs::LbfgsState* lbfgs = nullptr;    // optimiser state (mvs_lbfgs.cu)
    mvs::Profiler prof;
    mvs::TcState* tc = nullptr;          // tensor-core path state (mvs_tc.cu)
    float* rest_joints = nullptr;    // [K,3] keypoints of the rest pose at scale rest_scale (mvs_init.cu), computed once
    float rest_scale = -1.f;
    int2* stage_rng = nullptr;       // [B] per-frame slice of the stage table (mvs_fit_seq), device
    mvs::StreamState* fstream = nullptr;  // frame-stream scratch (mvs_fit_stream), created on first use
    mvs::SeqState* sstream = nullptr;     // sequence-stream, shared-shape and camera-refinement scratch, created on first use
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
void dev_free(mvs_ctx* ctx, void* p);          // a dev_alloc'ed array (NULL: nothing)
// Room for n elements in b: a larger array replaces a smaller one (its contents are lost).  b.cap counts only what is
// allocated: after a failed allocation b is empty.
template <class T> int dev_grow(mvs_ctx* ctx, DevBuf<T>& b, size_t n) {
    if (b.cap >= n) return MVS_OK;
    dev_free(ctx, b.p);
    b = DevBuf<T>{};
    if (int rc = dev_alloc(ctx, &b.p, n)) return rc;
    b.cap = n;
    return MVS_OK;
}

// mvs_lbfgs.cu: mvs_closure through the frame-resident closure, a dense round or the batched chain
int evaluate_closure(mvs_ctx* ctx, const float* x_dev, float* loss_dev, float* grad_dev, float* joints_dev, float* proj_dev,
                     float* verts_dev, cudaStream_t st);
// dynamic shared memory limits of each unit's kernels (largest launch), set by mvs_set_batch
int closure_set_attributes(mvs_ctx* ctx);
int resident_set_attributes(mvs_ctx* ctx);
int tc_set_attributes(mvs_ctx* ctx);           // also encodes the tensor maps over Qk and PhiTc
int sdf_set_attributes(mvs_ctx* ctx);
// batched chain (mvs_closure.cu): evaluates all active slots.  x_dev [B][86].
int launch_closure(mvs_ctx* ctx, const float* x_dev, float* loss_dev, float* grad_dev, float* joints_dev,
                   float* proj_dev, float* verts_dev, cudaStream_t st, bool geometry_only = false);
int launch_sdf_terms(mvs_ctx* ctx, const float* x_dev, cudaStream_t st);   // mvs_sdf.cu
// mvs_forward_vjp (mvs_closure.cu): dparams [B][86] from params x_dev and the cotangents djoints [B][K][3] / dverts [B][N][3]
int launch_forward_vjp(mvs_ctx* ctx, const float* x_dev, const float* djoints, const float* dverts, float* dparams,
                       cudaStream_t st);
// mvs_resident.cu: frame-resident (one CTA per frame) closure and whole-stage optimiser for the sparse regime
bool resident_supported(const mvs_ctx* ctx);   // the model fits the frame-resident kernels
int launch_vposer_decode(mvs_ctx* ctx, const float* x_dev, float* body_pose_dev, cudaStream_t st);
int launch_closure_resident(mvs_ctx* ctx, const float* x_dev, float* loss_dev, float* grad_dev, float* joints_dev,
                            float* proj_dev, cudaStream_t st);
// The frame-resident optimiser over the nstages stages of the run's table (ctx->lbfgs->lp_tab, as begin_run filled it): one
// CTA per frame of frames, rows params_dev [frames.n][86]; each frame's scalars to frame_scalars_out [frames.n]
int launch_lbfgs_resident(mvs_ctx* ctx, float* params_dev, const LbfgsCfg& cfg, int nstages, const FrameInputs& frames,
                          FrameScalars* frame_scalars_out, float* last_grad_dev, const int2* stage_rng_dev, cudaStream_t st);
// the chaining run of mvs_fit_seq_stream in the frame-resident regime: one CTA per sequence of q.act.  temporal_w [F][86]
// (mvs_fit_seq_stream_temporal; NULL: term off) are the anchor weights of the warm stages, whose anchor row is the
// predecessor's fitted row of params_dev
int launch_lbfgs_resident_seq(mvs_ctx* ctx, float* params_dev, const LbfgsCfg& cfg, int nstages, const FrameInputs& frames,
                              const SeqChain& q, cudaStream_t st, const float* temporal_w = nullptr);
// the shape closure of mvs_fit_shared_shape: the part rows of chunk c's frames (loss, betas, scale); frames whose problem is
// done are skipped
int launch_shape_closure(mvs_ctx* ctx, const ShapeArgs& a, const ProblemChunk& c, const LossParams& lp, const LbfgsState& L,
                         cudaStream_t st);
// mvs_refine_cameras (mvs_resident.cu): the keypoints q [F][K][3] (with translation) of frames[0 .. n), the rows of params [F][86],
// from resident_closure's joints output under lp (in: the call's frames, for the rigs)
int launch_camera_joints(mvs_ctx* ctx, const FrameInputs& in, const float* params, const int* frames, int n, const LossParams& lp,
                         float* q, cudaStream_t st);
// mvs_camera.cu: the camera closure of one chunk of view problems: the part rows of its work items (loss, rotation gradient [3],
// centre gradient [3]); items whose problem is done are skipped
int launch_camera_closure(mvs_ctx* ctx, const CameraArgs& a, const ProblemChunk& c, const LossParams& lp, const LbfgsState& L,
                          cudaStream_t st);
// mvs_camera.cu: the cameras of problems 0 .. P-1 at their rows x [P][86] into the device rig table
int launch_camera_write(mvs_ctx* ctx, const CamRefine* cr, const CameraProblem* prob, int P, const float* x, cudaStream_t st);
// mvs_camera.cu: fin[f] = 1 iff row f of params [F][86] is all finite
int launch_row_finite(mvs_ctx* ctx, const float* params, int F, int* fin, cudaStream_t st);
// dense regime (SDF term): per round  posedirs_gemm_tc -> skin -> sdf_setup -> sdf_fused -> frame_step (skin_small in place of
// skin at <= 8 frames; at <= 4 frames skin_small computes the set-ups itself and sdf_setup is not launched)
int launch_frame_fwd(mvs_ctx* ctx, const float* x_dev, cudaStream_t st);                      // mvs_closure.cu
int launch_sdf_fused(mvs_ctx* ctx, cudaStream_t st);   // mvs_sdf.cu
int ensure_sdf_setup_ws(mvs_ctx* ctx, cudaStream_t st);   // mvs_sdf.cu: set-up records, arrival counters (zeroed on st), boxes
SdfSetupArgs make_sdf_setup_args(mvs_ctx* ctx);          // mvs_sdf.cu
// mvs_tc.cu: wgmma / TMA dense vertex forward
int tc_upload_model(mvs_ctx* ctx);                 // after m.Qk is on the device
int launch_vertex_fwd_tc(mvs_ctx* ctx, cudaStream_t st, bool need_vposed, bool sdf_setup);
int tc_check_error(mvs_ctx* ctx);
// the d v_posed operand of vertex_bwd_tc_kernel, [2][ldA][ldR] (TF32 hi rows, then lo rows), allocated on first use
int tc_vjp_buffer(mvs_ctx* ctx, float** dvp, int* ldR);
// d Phi of mvs_forward_vjp on the tensor cores: the feature columns of the nstrips per-strip partials (w.part) from the
// d v_posed rows vertex_bwd_kernel<true> wrote
int launch_vertex_bwd_tc(mvs_ctx* ctx, int nstrips, cudaStream_t st);
float* tc_poffT(mvs_ctx* ctx);                 // [3N][ldA] pose offsets of the tensor-core contraction (written by launch_vertex_fwd_tc)
int launch_frame_step(mvs_ctx* ctx, float* params_dev, const LbfgsState& L, const LbfgsCfg& cfg, int nstages, cudaStream_t st);
int frame_step_begin_run(mvs_ctx* ctx, cudaStream_t st);                 // mvs_resident.cu
int launch_frame_fwd_dense(mvs_ctx* ctx, const float* x_dev, const LbfgsState& L, int nstages, cudaStream_t st);   // mvs_resident.cu
int make_loss_params(mvs_ctx* ctx, const mvs_loss_config* c, LossParams* out);      // mvs_api.cu: validation + conversion
int ensure_keypoint_ws(mvs_ctx* ctx);          // mvs_api.cu: gt_uv / conf for the rigs' largest view count, joint weights
// mvs_api.cu: the rigs of the batch's slots (ctx->slot_rigs); MVS_ERR_INVALID when the table has several rigs and no per-slot
// rigs were given
int batch_rigs(mvs_ctx* ctx, const char* who);
inline RigSet slot_rig_set(const mvs_ctx* ctx) { return RigSet{ctx->rigs_dev.p, ctx->slot_rigs}; }
// mvs_api.cu: every entry of rig_dev [n] names a rig of the table; MVS_ERR_INVALID naming the first frame that does not.
// Synchronises st.
int check_frame_rigs(mvs_ctx* ctx, const char* who, const int* rig_dev, int n, cudaStream_t st);
void release_fit_state(mvs_ctx* ctx);          // mvs_lbfgs.cu: the optimiser state and the stream scratch (mvs_destroy)
void release_tc_state(mvs_ctx* ctx);           // mvs_tc.cu (mvs_destroy)
int sdf_grid_launch(mvs_ctx* ctx, float* phi, const int* faces, int num_faces, const float* verts, int batch,
                    int n_verts, int G, cudaStream_t st);
}  // namespace mvs
