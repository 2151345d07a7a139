/* mvsmpl.h -- C ABI of libmvsmpl.so, the H100-native (sm_90a) replacement of the
 * multi-view SMPL fitting hot path of boycehbz/MvSMPLfitting.
 *
 * Plain C, no torch / C++ types.  Every entry point returns 0 on success and a
 * negative mvs_status on failure; mvs_last_error() gives the message.  Device
 * pointers are BORROWED (the caller, normally PyTorch, owns them and keeps them
 * alive until the stream has run); host pointers are copied before the call
 * returns.  All work is enqueued on the caller-supplied cudaStream_t (passed as
 * void*; 0 = legacy default stream) and no entry point synchronises unless its
 * comment says so.  One context per device; a context is not thread-safe,
 * distinct contexts are independent.
 *
 * Each entry point names the reference interface it replaces (paths relative to
 * the reference repository root).
 */
#ifndef MVSMPL_H_
#define MVSMPL_H_

#ifdef __cplusplus
extern "C" {
#endif

#define MVS_NUM_PARAMS 86      /* betas10 | global_orient3 | body_pose69 | transl3 | scale1 :
                                  flat order of LBFGS._gather_flat_grad (code/optimizers/lbfgs_ls.py:221-231)
                                  over SMPL's parameter registration order (code/smplx/body_models_scale.py:213-268) */
#define MVS_NUM_JOINTS 24
#define MVS_NUM_BETAS 10
#define MVS_NUM_POSE_BASIS 207
#define MVS_VPOSER_LATENT 32

typedef struct mvs_ctx mvs_ctx;

typedef enum {
    MVS_OK = 0,
    MVS_ERR_INVALID = -1,      /* bad argument / call order */
    MVS_ERR_CUDA = -2,         /* CUDA runtime error */
    MVS_ERR_NO_DEVICE = -3,    /* no usable sm_90 device: there is NO CPU fallback */
    MVS_ERR_UNSUPPORTED = -4
} mvs_status;

/* ---- lifetime -------------------------------------------------------------------- */
int mvs_version(void);
const char* mvs_build_id(void);    /* hash of the sources this library was compiled from (mvsmplfitting_b200/build.py: source_hash) */
int mvs_create(int device, mvs_ctx** out);
void mvs_destroy(mvs_ctx* ctx);
const char* mvs_last_error(const mvs_ctx* ctx);          /* ctx may be NULL (creation errors) */
long long mvs_launch_count(const mvs_ctx* ctx);          /* kernels launched by this context so far */

/* ---- model: replaces SMPL.__init__ buffers (code/smplx/body_models_scale.py:270-305),
 *      VertexJointSelector (code/smplx/vertex_joint_selector.py:38-77) and JointMapper
 *      (code/utils/utils.py:411-424).  All pointers are HOST pointers. ---------------- */
typedef struct {
    int n_verts;                   /* 6890 */
    int n_faces;                   /* 13776 (0 if faces == NULL) */
    const float* v_template;       /* [n_verts,3] */
    const float* shapedirs;        /* [n_verts,3,10] */
    const float* posedirs;         /* [207, 3*n_verts]  (the reference's registered layout) */
    const float* J_regressor;      /* [24, n_verts] */
    const int* parents;            /* [24], parents[0] = -1 */
    const float* lbs_weights;      /* [n_verts,24] */
    const int* faces;              /* [n_faces,3] or NULL */
    int n_keypoints;               /* 17 */
    int n_reg;                     /* rows of joint_regressor: 14 ('smpllsp') or 0 ('smpl': the 24 posed chain joints) */
    const float* joint_regressor;  /* [n_reg, n_verts] dense, or NULL when n_reg == 0 */
    int n_extra;                   /* 5 face vertices appended after the regressed / chain joints */
    const int* extra_vertex_ids;   /* [n_extra] */
    const int* joint_map;          /* [n_keypoints] indices into cat(joints, extra vertices) */
} mvs_model_desc;
int mvs_set_model(mvs_ctx* ctx, const mvs_model_desc* desc);

/* MaxMixturePrior buffers (code/prior.py:142-160): means [M,69], precisions [M,69,69], nll_weights [M] (host) */
int mvs_set_gmm_prior(mvs_ctx* ctx, int num_gaussians, const float* means, const float* precisions,
                      const float* nll_weights);

/* VPoser decoder weights (code/model/VPoser.py:190-197: bodyprior_dec_fc1 [512,32], bodyprior_dec_fc2 [512,512],
 * bodyprior_dec_out [138,512] and their biases; host arrays, row-major [out,in] as torch.nn.Linear stores them).
 * With them a loss configuration may set use_vposer = 2: the pose is VPoser.decode(z, 'aa') (VPoser.py:218-232 and
 * fitting.py:121-123) evaluated ON THE DEVICE inside the closure, z = the first 32 entries of the body_pose slot of the
 * 86-vector (entries 32..68 of the slot are ignored and get zero gradient), the body prior is |z|^2 * body_pose_weight^2
 * (fitting.py:327-329).  Implemented in the frame-resident closure / optimiser and in the dense (SDF) rounds, which
 * mvs_lbfgs_step uses as well; not in the batched reference chain (exec mode 1, closures that ask for vertices). */
int mvs_set_vposer(mvs_ctx* ctx, const float* fc1_w, const float* fc1_b, const float* fc2_w, const float* fc2_b,
                   const float* out_w, const float* out_b);

/* vposer.decode(pose_embedding, output_type='aa') on its own (what save_results does with the fitted latent code before it
 * writes a result, code/utils/utils.py:741-743): params_dev [B,86] with the latent code in the first 32 entries of the
 * body_pose slot -> body_pose_dev [B,69] axis-angle.  Needs mvs_set_vposer. */
int mvs_vposer_decode(mvs_ctx* ctx, const float* params_dev, float* body_pose_dev, void* stream);

/* PerspectiveCamera list (code/camera.py:41-117, built in code/init.py:108-131): host arrays
 * R [V,3,3], t [V,3], f [V,2] (focal x,y), c [V,2].  The same as mvs_set_camera_rigs with one rig of scale 1. */
int mvs_set_cameras(mvs_ctx* ctx, int num_views, const float* R, const float* t, const float* f, const float* c);

/* ---- camera rigs: the frames of one context may come from different camera setups (the reference runs one camera file per
 *      run, code/init.py cam_param).  A rig is num_views[r] <= 16 views plus a data-weight scale s_r.  A frame with rig r is
 *      evaluated exactly as in a context whose only cameras are rig r's and whose stage configurations have
 *      data_weight = fl32(data_weight * s_r): s_r scales the data weight of the 2-D term and of the 3-D joint term (e.g. the
 *      reference's 500 / H for rigs of different image heights).  A scale of 1 is exact.
 *      Host arrays padded to Vmax = max num_views: R [n_rigs,Vmax,3,3], t [n_rigs,Vmax,3], f and c [n_rigs,Vmax,2] (rows
 *      v >= num_views[r] are not read); data_weight_scale [n_rigs] (finite, > 0) or NULL = all 1.  Replaces the previous rigs
 *      or cameras (waits for the device first); keypoints and per-slot rigs must be set again.  Every detection array of the
 *      context has Vmax view rows; rows v >= V_r of a frame with rig r are never read, and closure projections of those rows
 *      are left untouched. */
int mvs_set_camera_rigs(mvs_ctx* ctx, int n_rigs, const int* num_views, const float* R, const float* t, const float* f,
                        const float* c, const float* data_weight_scale);

/* ---- mvs_set_camera_rigs with lens distortion: dist [n_rigs,Vmax,5] (host) holds each view's OpenCV projectPoints coefficients
 *      (k1, k2, p1, p2, k3); rows v >= num_views[r] are not read.  With x' = x/z, y' = y/z, r2 = x'^2 + y'^2 and
 *      a = 1 + k1 r2 + k2 r2^2 + k3 r2^3 every projection is
 *          u = fx (x' a + 2 p1 x'y' + p2 (r2 + 2 x'^2)) + cx,   v = fy (y' a + p1 (r2 + 2 y'^2) + 2 p2 x'y') + cy
 *      with no clamp: fits are only meaningful inside the calibrated field of view, where this map is monotone.  It serves the
 *      2-D term of every closure and fitting driver, mvs_init_guess (which undistorts each detection with non-zero confidence
 *      before it triangulates or takes the one-view depth guess) and mvs_refine_cameras (the coefficients are held, like f and
 *      c, and the refined table keeps them).  A rig whose coefficients are all zero is evaluated exactly as without them.
 *      Otherwise the same as mvs_set_camera_rigs (same validation, waits for the device, keypoints and per-slot rigs must be
 *      set again); MVS_ERR_INVALID naming the rig and view if a coefficient is not finite.  mvs_set_camera_rigs is this call
 *      with dist = NULL. */
int mvs_set_camera_rigs_dist(mvs_ctx* ctx, int n_rigs, const int* num_views, const float* R, const float* t, const float* f,
                             const float* c, const float* dist, const float* data_weight_scale);

/* The rig of every slot of the batch: rig_host [B] (HOST ints in [0, n_rigs)), validated and copied before return (waits for
 *      the device first).  Read by mvs_closure, mvs_lbfgs_run, mvs_lbfgs_step, mvs_fit, mvs_fit_seq, mvs_fit_host and
 *      mvs_init_guess.  With more than one rig, those entry points return MVS_ERR_INVALID unless per-slot rigs were given
 *      since the last mvs_set_batch, mvs_set_camera_rigs / mvs_set_cameras or stream call; with one rig every slot has rig 0
 *      unless told otherwise. */
int mvs_set_frame_rigs(mvs_ctx* ctx, const int* rig_host);

/* frames in flight (the reference is fixed to 1: code/utils/non_linear_solver.py:56); allocates workspace */
int mvs_set_batch(mvs_ctx* ctx, int num_frames);

/* 2-D detections: gt_uv [V,B,K,2], conf [V,B,K], joint_weights [K] (V = the rigs' largest view count)
 * (code/utils/non_linear_solver.py:77-101).  on_device != 0: device pointers (copied D2D on `stream`),
 * else host pointers (copied before return). */
int mvs_set_keypoints(mvs_ctx* ctx, const float* gt_uv, const float* conf, const float* joint_weights,
                      int on_device, void* stream);

/* ---- loss: SMPLifyLoss weights + flags (code/utils/fitting.py:208-280, reset_loss_weights :270-280) */
typedef enum { MVS_PRIOR_L2 = 0, MVS_PRIOR_GMM = 1, MVS_PRIOR_NONE = 2 } mvs_body_prior;
typedef struct {
    float data_weight;             /* 500 / image height (non_linear_solver.py:148-150) */
    float body_pose_weight;
    float shape_weight;
    float bending_prior_weight;    /* 3.17 * body_pose_weight (non_linear_solver.py:178-179) */
    float coll_loss_weight;
    float rho;                     /* GMoF rho (utils.py:427-438) */
    int body_prior;                /* mvs_body_prior */
    int use_joints_conf;
    int use_vposer;                /* 1: body_pose comes decoded from the caller, body-pose prior terms are the caller's
                                      (|z|^2), angle guard disabled; 2: decoded on the device (mvs_set_vposer) */
    int fix_shape;                 /* no shape prior (fitting.py:340) */
    int interpenetration;          /* SDF term on (needs faces) */
    int sdf_grid;                  /* 128 in the reference call (fitting.py:367-368) */
    int sdf_all_faces;             /* 0 = as written (the kernel sees num_faces == 1: triangle 0 only, fitting.py:367);
                                      1 = intended semantics, all faces, evaluated over per-frame candidate lists (uniform cell
                                          grid for the distance, central projection from the ray target for the parity;
                                          bit-identical to 2, ~100x fewer primitive evaluations; SURVEY N3);
                                      2 = all faces by brute force (the cross-check of 1).  The batched reference chain
                                          (exec mode 1, closures that ask for vertices) always uses the brute force. */
    unsigned frozen_mask;          /* bit i set -> parameter tensor i (betas, orient, pose, transl, scale) has
                                      requires_grad=False: its gradient is forced to 0 (init_guess.py:190-212) */
} mvs_loss_config;
int mvs_set_loss_config(mvs_ctx* ctx, const mvs_loss_config* cfg);

/* ---- per-frame quadratic anchor (NOT in the reference; used by the jointly regularised sequence mode, see
 *      DESIGN.md section 6): adds  sum_i weight[b,i] * (x[b,i] - anchor[b,i])^2  to frame b's loss, and its gradient.
 *      anchor_dev and weight_dev are [B,86] device pointers, copied; enable = 0 switches the term off. */
int mvs_set_anchor(mvs_ctx* ctx, const float* anchor_dev, const float* weight_dev, int enable, void* stream);

/* ---- 3-D joint supervision: SMPLifyLoss(use_3d=True) (code/utils/fitting.py:318-324, targets from
 *      code/utils/non_linear_solver.py:86-99): adds  data_weight^2 * sum_k conf[b,k]^2 * sum_c GMoF_rho(gt_xyz[b,k,c] - q[b,k,c])
 *      to frame b's loss, q = the keypoints the 2-D term projects, with the stage's rho and data_weight; joint_weights and
 *      use_joints_conf do not apply to it.  The confidences are taken as given (the reference zeroes hips 11 and 12 unless
 *      use_hip is set; that is the caller's).  gt_xyz [B,K,3], conf [B,K]; on_device != 0: device pointers (copied D2D on
 *      `stream`), else host pointers (copied before return).  enable = 0 switches the term off (the arrays are not read).
 *      Needs the model and mvs_set_batch first: a context's batch size is fixed once set, so the targets always have its
 *      B rows, and nothing from another batch size can be read.  Every later mvs_set_loss_config / mvs_fit stage sees the
 *      term; mvs_init_guess aligns to the targets instead of the triangulated keypoints while it is on (init_guess.py:85-86). */
int mvs_set_joints3d(mvs_ctx* ctx, const float* gt_xyz, const float* conf, int enable, int on_device, void* stream);

/* ---- closure: replaces fitting_func() (code/utils/fitting.py:162-203) = SMPL.forward + SMPLifyLoss.forward
 *      + backward, for all B frames at once.  params_dev [B,86]; outputs (device, any may be NULL):
 *      loss_dev [B], grad_dev [B,86], joints_dev [B,K,3], proj_dev [V,B,K,2], verts_dev [B,n_verts,3].
 *      Requesting verts (or interpenetration) selects the dense 6890-vertex path. */
int mvs_closure(mvs_ctx* ctx, const float* params_dev, float* loss_dev, float* grad_dev, float* joints_dev,
                float* proj_dev, float* verts_dev, void* stream);

/* ---- geometry only: replaces SMPL.forward (code/smplx/body_models_scale.py:327-412) when it is called outside
 *      the closure (result export, visualisation): joints_dev [B,K,3] and / or verts_dev [B,n_verts,3].
 *      Needs only the model and the batch size.  The body_pose slot is read as axis-angle whatever the loss configuration
 *      says: decode latent codes first (mvs_vposer_decode). */
int mvs_forward(mvs_ctx* ctx, const float* params_dev, float* joints_dev, float* verts_dev, void* stream);

/* ---- vector-Jacobian product of mvs_forward (the autograd backward of SMPL.forward, body_models_scale.py:327-412 +
 *      lbs.py:135-222, outside the closure): given params_dev [B,86] and cotangents of its outputs -- djoints_dev [B,K,3]
 *      and / or dverts_dev [B,n_verts,3] (device, either may be NULL, not both) -- writes dparams_dev [B,86] =
 *      d<dj,joints> + d<dv,verts> with respect to every entry (betas, global_orient, body_pose as axis-angle, transl, scale).
 *      Needs only the model and the batch size, like mvs_forward; recomputes what it needs from params_dev (nothing is kept
 *      from an earlier mvs_forward).  It is the model's Jacobian and nothing else: the frozen mask, the loss configuration,
 *      the anchor, keypoints, 3-D targets, cameras and rigs are neither read nor changed, and neither is the optimiser state
 *      mvs_lbfgs_step keeps between calls.  Workspace it borrows, which every entry point writes before it reads: the forward
 *      arrays of the batch (pose features, skinning transforms, chain joints, v_posed, vertices; what mvs_forward writes)
 *      and the closure's backward scratch (per-vertex cotangents, per-strip partials, translation and chain-joint
 *      cotangents); with dverts_dev, the d v_posed operand of the tensor-core contraction, grow-only and its own.
 *      With dverts_dev the adjoint runs over all vertices (the blend-shape contraction on the tensor cores; exec mode 1:
 *      SIMT); joints only, over the <= 86 vertices the keypoints read.  Deterministic: the same call gives the same bits.
 *      Asynchronous on `stream`.  MVS_ERR_INVALID: ctx, params_dev or dparams_dev NULL, both cotangents NULL, no model or
 *      batch. */
int mvs_forward_vjp(mvs_ctx* ctx, const float* params_dev, const float* djoints_dev, const float* dverts_dev,
                    float* dparams_dev, void* stream);

/* ---- optimiser: replaces LBFGS.step + _strong_Wolfe (code/optimizers/lbfgs_ls.py:39-445) driven by
 *      FittingMonitor.run_fitting (code/utils/fitting.py:71-142), one independent problem per frame,
 *      entirely on the device. */
typedef struct {
    int max_outer;                 /* FittingMonitor.maxiters (30) */
    int max_iter;                  /* LBFGS max_iter (30) */
    int max_eval;                  /* LBFGS max_eval (max_iter*5/4 = 37); <=0 -> derived */
    int history_size;              /* 100 */
    float lr;                      /* 1.0 */
    float tolerance_grad;          /* 1e-5 */
    float tolerance_change;        /* 1e-9 */
    float ftol;                    /* FittingMonitor ftol */
    float gtol;                    /* FittingMonitor gtol */
} mvs_lbfgs_config;
typedef struct {
    long long frame_iterations;    /* sum over frames of L-BFGS iterations (lbfgs_ls.py:304-434 loop bodies) */
    long long frame_evals;         /* sum over frames of closure evaluations */
    int rounds;                    /* batched closure launches */
    int frames_nan;                /* frames stopped by the NaN/Inf guard (fitting.py:101-107) */
    long long dense_frame_evals;   /* of frame_evals: those evaluated by dense (SDF) rounds */
    int dense_rounds;              /* of rounds: dense rounds (gemm -> skin -> sdf_setup -> sdf_fused -> frame_step each) */
    int reserved;
} mvs_lbfgs_stats;
/* params_dev [B,86] in/out; final_loss_dev [B] or NULL (run_fitting's return value per frame).
 * Synchronises `stream` before returning (stats are read back). */
int mvs_lbfgs_run(mvs_ctx* ctx, float* params_dev, float* final_loss_dev, const mvs_lbfgs_config* cfg,
                  mvs_lbfgs_stats* stats, void* stream);

/* Exactly one LBFGS.step(closure) for every frame (code/optimizers/lbfgs_ls.py:256-445), for callers that keep
 * their own outer loop (the reference's FittingMonitor.run_fitting calls optimizer.step once per outer
 * iteration).  The optimiser state persists inside the context between calls; reset != 0 starts a fresh
 * optimiser (a new stage builds a new one: code/utils/non_linear_solver.py:172).  loss_dev [B] receives what
 * step() returns (the loss at entry), last_grad_dev [B,86] (may be NULL) what p.grad holds afterwards (the
 * gradients of the last closure call).  Synchronises. */
int mvs_lbfgs_step(mvs_ctx* ctx, float* params_dev, float* loss_dev, float* last_grad_dev, const mvs_lbfgs_config* cfg,
                   int reset, mvs_lbfgs_stats* stats, void* stream);

/* ---- all stages of one fit, device buffers: what code/utils/non_linear_solver.py:109-203 does per frame (for every
 *      stage: new loss weights, new optimiser, run_fitting) for all B frames at once.  Consecutive stages that run in
 *      the same execution regime are merged into one run in which every frame moves to its next stage as soon as ITS
 *      current stage stops -- frames are independent problems, so the per-frame schedule is the reference's, but no
 *      frame waits at a stage boundary for the slowest one.  params_dev [B,86] is updated in place, final_loss_dev [B]
 *      (may be NULL) receives each frame's last-stage result of run_fitting.  Leaves the last stage's loss
 *      configuration set.  Synchronises. */
int mvs_fit(mvs_ctx* ctx, float* params_dev, int n_stages, const mvs_loss_config* stage_cfgs, const mvs_lbfgs_config* opt_cfg,
            float* final_loss_dev, mvs_lbfgs_stats* stats, void* stream);

/* ---- mvs_fit for video sequences (is_seq, code/main.py:76-79 + code/utils/non_linear_solver.py:157-162): warm_host [B]
 *      (HOST bytes, may be NULL = mvs_fit) marks the frames that continue a sequence -- their params_dev rows hold the previous
 *      frame's result as load_init leaves it (code/utils/init_guess.py:137-166 + fix_params) -- and that therefore skip the
 *      first two stages and run the third with 0.15 x its body_pose_weight; the other frames run every stage.  Frames of
 *      one call are independent, so a batch is e.g. frame t of S sequences, some of them at their first frame.  Needs
 *      n_stages > 2 when any frame is warm; not implemented in the batched reference chain (exec mode 1). */
int mvs_fit_seq(mvs_ctx* ctx, float* params_dev, int n_stages, const mvs_loss_config* stage_cfgs,
                const mvs_lbfgs_config* opt_cfg, const unsigned char* warm_host, float* final_loss_dev,
                mvs_lbfgs_stats* stats, void* stream);

/* ---- mvs_fit_seq with a causal temporal term (NOT in the reference: smoother video fits).  temporal_w_host [86] (HOST floats,
 *      finite, >= 0, the same for every frame) adds  sum_i w[i] * (x[b,i] - prev[b,i])^2  to the loss of every stage a WARM
 *      frame b runs (stages 2 .. n-1; the weight is not scaled by the stage, the 0.15 damping of stage 2 or a rig's data-weight
 *      scale); cold frames never carry it.  prev_dev [B,86] (device) holds each warm frame's predecessor's FITTED row as
 *      mvs_fit_seq returned it (before load_init / fix_params: without VPoser the anchor keeps the fitted body pose while the
 *      start point has the hip seed; with use_vposer = 2 the latent code is anchored); rows of cold frames are not read.
 *      A warm frame gets exactly what mvs_fit gives it alone on its slice of the stages after
 *      mvs_set_anchor(row = prev[b], weight = w).  temporal_w_host NULL or all zero: mvs_fit_seq, bit for bit.
 *      Refused: MVS_ERR_INVALID for a weight entry that is negative or not finite and for n_stages <= 2; MVS_ERR_UNSUPPORTED in
 *      exec mode 1 and while mvs_set_anchor is on.  Afterwards the anchor term is off, as it had to be before the call (the
 *      context's anchor rows and weights are overwritten); otherwise the context is as after mvs_fit_seq.  Synchronises. */
int mvs_fit_seq_temporal(mvs_ctx* ctx, float* params_dev, int n_stages, const mvs_loss_config* stage_cfgs,
                         const mvs_lbfgs_config* opt_cfg, const unsigned char* warm_host, const float* prev_dev,
                         const float* temporal_w_host, float* final_loss_dev, mvs_lbfgs_stats* stats, void* stream);

/* ---- mvs_fit over a stream of F frames, F of any size relative to the context's batch B.  Every frame gets exactly what
 *      mvs_fit gives it in a batch of any size, bit for bit: the same parameters, final loss and iteration / evaluation
 *      counts.  Stages are grouped into runs as mvs_fit groups them; each run covers all F frames before the next starts
 *      (one barrier per run for the whole stream).  A frame-resident run is one launch over the F frames.  A dense (SDF) run
 *      keeps B frames in flight, one per slot: whenever a frame finishes, its slot takes the next frame of the stream at the
 *      next compaction of the active list (every 8 rounds), so the tail of one batch overlaps the start of the next.
 *      All arrays are device pointers.  stats sums over frames equal those of mvs_fit over the same frames; rounds and
 *      dense_rounds are the rounds the stream ran.  Refused (MVS_ERR_UNSUPPORTED): stages that would run in the batched
 *      reference chain (exec mode 1, history_size > 100 without the SDF term, a model the frame-resident / dense kernels do
 *      not take) and the anchor term (mvs_set_anchor: it is per batch).  MVS_ERR_INVALID: NULL or empty arguments,
 *      n_frames < 1, gt_xyz without conf3d.
 *      Context state afterwards: the dense runs overwrite the slots' keypoint and 3-D target rows, so after the call the
 *      context behaves as if no keypoints and no 3-D targets had been uploaded: entry points that need keypoints return
 *      MVS_ERR_INVALID until mvs_set_keypoints is called again, and the 3-D term is off until mvs_set_joints3d enables it
 *      again.  The stream never reads the context's own keypoints or 3-D targets.  Leaves the last stage's loss
 *      configuration set (3-D term off).  Synchronises. */
typedef struct {
    int n_frames;                  /* F >= 1 */
    float* params;                 /* [F,86] in/out: start point in, fitted parameters out */
    const float* gt_uv;            /* [V,F,K,2] */
    const float* conf;             /* [V,F,K] */
    const float* joint_weights;    /* [K] */
    const float* gt_xyz;           /* [F,K,3]: the 3-D joint term is on for this call iff non-NULL */
    const float* conf3d;           /* [F,K], required with gt_xyz */
    float* final_loss;             /* [F] or NULL */
} mvs_frame_stream;
int mvs_fit_stream(mvs_ctx* ctx, const mvs_frame_stream* s, int n_stages, const mvs_loss_config* stage_cfgs,
                   const mvs_lbfgs_config* opt_cfg, mvs_lbfgs_stats* stats, void* stream);

/* ---- mvs_fit_stream with a rig per frame (mvs_set_camera_rigs): rig_dev [F] (device ints) names each frame's rig; every frame
 *      gets the bits mvs_fit gives it in a context whose only cameras are its rig's.  The indices are checked on the device
 *      before any fitting work: one out of [0, n_rigs) returns MVS_ERR_INVALID naming the first such frame.  rig_dev = NULL:
 *      every frame has rig 0, allowed with one rig only (MVS_ERR_INVALID otherwise); mvs_fit_stream is this call with NULL.
 *      Context state afterwards as after mvs_fit_stream, and no per-slot rigs either (the lanes' rig rows were overwritten
 *      with the keypoints): mvs_set_frame_rigs again before a batch entry point of a context with several rigs.
 *      Synchronises. */
int mvs_fit_stream_rigs(mvs_ctx* ctx, const mvs_frame_stream* s, const int* rig_dev, int n_stages,
                        const mvs_loss_config* stage_cfgs, const mvs_lbfgs_config* opt_cfg, mvs_lbfgs_stats* stats,
                        void* stream);

/* ---- mvs_fit_seq over S video sequences of any number and length through the context's B slots (is_seq, code/main.py:76-79).
 *      Sequence s owns frames [seq_offsets[s], seq_offsets[s+1]) of the F-frame arrays, in time order.  Every frame gets
 *      exactly the parameters and final loss that mvs_fit_seq gives it when frame t of every sequence is fitted as one batch
 *      of S (mvsmplfitting_b200.seqio.fit_sequences with a batch of S):
 *        cold frame: the first frame of a sequence, or one whose predecessor's final loss is not <= reinit_loss (NaN is not).
 *          It starts from its own params row -- the caller's cold start point, mvs_init_guess -- and runs every stage.
 *        warm frame: starts from the predecessor's fitted row (load_init, code/utils/init_guess.py:137-166) with its own
 *          params row's body-pose slot [13,82) (fix_params puts the pose back to the hip seed) unless the stages optimise a
 *          latent code (use_vposer = 2: the whole row is carried), and runs stages 2 .. n-1 with stage 2's body_pose_weight
 *          x 0.15 (code/utils/non_linear_solver.py:157-162).
 *      Stages are grouped into runs as mvs_fit_seq groups them; stages 2 .. n-1 must form one run, the chaining run, in which
 *      a finished frame hands its slot to its successor on the device (frame-resident: one CTA per sequence walks its frames
 *      in one launch; dense: a lane takes the successor at the next compaction of the active list).  The runs before it take
 *      cold frames as a frame stream (mvs_fit_stream); a sequence whose next frame is cold parks it until the next pass of
 *      those runs.  All arrays except seq_offsets are device pointers.
 *      stats: frame_iterations, frame_evals, frames_nan and dense_frame_evals are sums over the F frames; rounds and
 *      dense_rounds count the rounds the call ran.  A frame-resident chaining run counts, per pass, the largest number of
 *      closure evaluations one sequence's frames needed in it (the critical path of its launch) as rounds.
 *      Refused (MVS_ERR_UNSUPPORTED): stages in the batched reference chain, the anchor term, stages 2 .. n-1 that do not
 *      form one run (exec mode 2 with n_stages > 3, a change of regime, SDF grid or face mode between them).
 *      MVS_ERR_INVALID: NULL or empty arguments, n_stages <= 2, seq_offsets not starting at 0 or not strictly ascending,
 *      stages that mix use_vposer 2 with axis-angle poses.
 *      Context state afterwards as after mvs_fit_stream: no keypoints, 3-D term off, the last stage's loss configuration set.
 *      The call never reads the context's own keypoints or 3-D targets; mvs_fit_seq_stream3d adds the 3-D joint term.
 *      Synchronises. */
typedef struct {
    int n_sequences;               /* S >= 1 */
    const int* seq_offsets;        /* HOST [S+1]: 0 = off[0] < off[1] < ... < off[S] = F (no empty sequence) */
    float* params;                 /* [F,86] in: every frame's cold start point; out: fitted parameters */
    const float* gt_uv;            /* [V,F,K,2] */
    const float* conf;             /* [V,F,K] */
    const float* joint_weights;    /* [K] */
    float* final_loss;             /* [F] or NULL */
    float reinit_loss;             /* 5000 in the reference (code/utils/init_guess.py:142) */
} mvs_sequence_stream;
int mvs_fit_seq_stream(mvs_ctx* ctx, const mvs_sequence_stream* s, int n_stages, const mvs_loss_config* stage_cfgs,
                       const mvs_lbfgs_config* opt_cfg, mvs_lbfgs_stats* stats, void* stream);

/* ---- mvs_fit_seq_stream with the 3-D joint term (SMPLifyLoss use_3d, code/utils/fitting.py:318-324): gt_xyz [F,K,3] and
 *      conf3d [F,K] (device pointers) are every frame's 3-D targets and confidences, rows in the order of the frames of s.
 *      The term is on in every stage of every frame, cold and warm; a frame without annotations takes zero rows (confidence 0
 *      gives, bit for bit, the result with the term off).  The bit-for-bit contract includes the term: every frame gets the
 *      parameters and final loss that mvs_fit_seq gives it in a batch of S after mvs_set_joints3d with frame t's rows of the
 *      S sequences.  Both pointers NULL: mvs_fit_seq_stream (which is this call with two NULLs).  Exactly one NULL:
 *      MVS_ERR_INVALID.  Refusals and context state afterwards as mvs_fit_seq_stream.  Synchronises. */
int mvs_fit_seq_stream3d(mvs_ctx* ctx, const mvs_sequence_stream* s, const float* gt_xyz, const float* conf3d, int n_stages,
                         const mvs_loss_config* stage_cfgs, const mvs_lbfgs_config* opt_cfg, mvs_lbfgs_stats* stats,
                         void* stream);

/* ---- mvs_fit_seq_stream3d with a rig per frame: rig_dev [F] (device ints, rows in the order of the frames of s) names each
 *      frame's rig; the frames of one sequence may change rig.  Every frame gets the bits mvs_fit_seq gives it in a batch of S
 *      (frame t of every sequence) with mvs_set_frame_rigs naming each slot's rig; a warm frame starts from its predecessor's
 *      result whatever rig either has.  Checked on the device first: an index out of [0, n_rigs) returns MVS_ERR_INVALID
 *      naming the first such frame.  rig_dev = NULL: every frame has rig 0, one rig only; mvs_fit_seq_stream3d and
 *      mvs_fit_seq_stream are this call with NULL.  Context state afterwards as after mvs_fit_stream_rigs.  Synchronises. */
int mvs_fit_seq_stream_rigs(mvs_ctx* ctx, const mvs_sequence_stream* s, const float* gt_xyz, const float* conf3d,
                            const int* rig_dev, int n_stages, const mvs_loss_config* stage_cfgs,
                            const mvs_lbfgs_config* opt_cfg, mvs_lbfgs_stats* stats, void* stream);

/* ---- mvs_fit_seq_stream_rigs with the causal temporal term of mvs_fit_seq_temporal: temporal_w_host [86] (HOST floats, finite,
 *      >= 0).  Every warm frame's stages 2 .. n-1 carry  sum_i w[i] * (x_i - x^_i)^2, x^ = its predecessor's fitted row, which
 *      the device hands over with the slot (never passed in): the frame-resident chaining run anchors to the row it has just
 *      written to params, a dense lane copies the fitted row into its anchor row before the successor's start point replaces
 *      it.  Every frame gets exactly the parameters and final loss that mvs_fit_seq_temporal gives it in a batch of S
 *      (seqio.fit_sequences with a batch of S and the same weight), in both chaining regimes, with rigs and the 3-D term.
 *      temporal_w_host NULL or all zero: mvs_fit_seq_stream_rigs, bit for bit (which is this call with NULL).  Refusals as
 *      mvs_fit_seq_temporal adds them to those of mvs_fit_seq_stream_rigs; context state afterwards as after
 *      mvs_fit_seq_stream_rigs, anchor term off.  Synchronises. */
int mvs_fit_seq_stream_temporal(mvs_ctx* ctx, const mvs_sequence_stream* s, const float* gt_xyz, const float* conf3d,
                                const int* rig_dev, const float* temporal_w_host, int n_stages,
                                const mvs_loss_config* stage_cfgs, const mvs_lbfgs_config* opt_cfg, mvs_lbfgs_stats* stats,
                                void* stream);

/* ---- one body shape per video sequence (NOT in the reference, whose only tool is fix_shape with a hand-typed shape): for
 *      sequence q of s and the one stage configuration `stage` (normally the schedule's last), minimises
 *        E_q = sum_{t in q} L(x_t with betas <- beta, scale <- s)
 *      over beta, s and the other entries of every frame's row x_t, L = what mvs_closure returns for that row under `stage`
 *      (2-D term, priors with each frame's own shape prior, the 3-D term with gt_xyz, the rig's data-weight scale).  scale
 *      is shared unless `stage` freezes it (frozen_mask bit 4, fix_scale): a frozen scale stays at each row's own value.
 *      Block-coordinate descent, n_sweeps >= 1 times:
 *        consensus: beta (, s) = the mean over the sequence's frames whose rows are all finite (double, frame order); a
 *          sequence without a finite row is skipped: its rows are left as they are, its losses are NaN;
 *        shape step: one L-BFGS problem per sequence over its shared entries with the poses held (the 86-vector state machine
 *          of mvs_fit's frames, with run_fitting's NaN / ftol / gtol rules and opt_cfg), the context's B sequences at a time;
 *          its closure adds the frames' mvs_closure losses and shared gradient entries in double, in frame order;
 *        pose step: the shared entries written into every row of the sequence, then every frame runs `stage` from its row with
 *          betas (and a shared scale) frozen: exactly mvs_fit_stream's bits for that row.
 *      s->params [F,86] holds the fitted rows on entry and the result on exit (s->reinit_loss is not read); s->final_loss [F]
 *      (may be NULL) receives each frame's pose-step result of the last sweep; seq_loss_dev [S] (device, may be NULL) each
 *      sequence's run_fitting value of its last shape step.  gt_xyz, conf3d and rig_dev as in mvs_fit_seq_stream_rigs.
 *      shape_stats counts the sequence problems' iterations and evaluations, pose_stats what mvs_fit_stream reports (both
 *      summed over the sweeps).  Refused: MVS_ERR_INVALID for NULL or empty arguments, n_sweeps < 1, bad seq_offsets, exactly
 *      one of gt_xyz / conf3d, betas frozen in `stage` (frozen_mask bit 0: the shape is given) and a rig index out of range
 *      (checked on the device); MVS_ERR_UNSUPPORTED for stage.interpenetration (the shape closure has no SDF term), the anchor
 *      term, and what mvs_fit_stream refuses (exec mode 1, history_size > 100).  Context state afterwards as after
 *      mvs_fit_stream.  Synchronises. */
int mvs_fit_shared_shape(mvs_ctx* ctx, const mvs_sequence_stream* s, const float* gt_xyz, const float* conf3d,
                         const int* rig_dev, const mvs_loss_config* stage, const mvs_lbfgs_config* opt_cfg,
                         int n_sweeps, float* seq_loss_dev, mvs_lbfgs_stats* shape_stats,
                         mvs_lbfgs_stats* pose_stats, void* stream);

/* ---- refine the camera rigs' extrinsics from fitted bodies (NOT in the reference, whose calibration is fixed): for the frames
 *      of s and the one stage configuration `stage` (normally the schedule's last), minimises  sum_f L(x_f; cameras of rig(f))
 *      (L = what mvs_closure returns for row x_f under `stage`) by block-coordinate descent, n_sweeps >= 1 times:
 *        held keypoints: each frame's keypoints (the points the 2-D term projects) from its row;
 *        camera step: one L-BFGS problem per view v >= 1 of every rig r with frames in the call (the 86-vector state machine of
 *          mvs_fit's frames, with run_fitting's NaN / ftol / gtol rules and opt_cfg), the context's B at a time.  Its loss is
 *          view v's 2-D data term of mvs_closure, summed over the frames with rig r at their held keypoints (in double, in
 *          call order).  Variables: a rotation update w and a camera-centre update, R = Rod(w) R0 and
 *          x_cam = Rod(w) (R0 (q - dC) + t0), exactly (R0, t0) at 0.  View 0 is held; view 1 keeps its distance to view 0
 *          (its centre moves on that sphere: 2 centre variables); views 2 .. V_r - 1 have 3.  The solved cameras replace the
 *          calibrated ones in the context's rig table;
 *        body step: every frame runs `stage` from its row against the refined table: exactly mvs_fit_stream_rigs's bits.
 *      A frame whose row is not all finite takes no part: its row is kept and its final loss is NaN.  Intrinsics, distortion and
 *      the data-weight scales are not refined; a view without a confident detection in the call and a rig of one view keep
 *      their cameras bit for bit.
 *      s->params [F,86] holds the fitted rows on entry and the result on exit; s->final_loss [F] (may be NULL) receives each
 *      frame's body-step result of the last sweep; s->gt_xyz / conf3d switch the 3-D term of the body step on.  rig_dev as in
 *      mvs_fit_stream_rigs.  R_host [n_rigs,Vmax,3,3] and t_host [n_rigs,Vmax,3] (HOST, each may be NULL) receive the refined
 *      table (rows v >= V_r are zero).  camera_stats counts the view problems' iterations and evaluations, pose_stats what
 *      mvs_fit_stream reports (both summed over the sweeps).  SDF stages are taken (the body step runs them as mvs_fit_stream).
 *      Refused: MVS_ERR_INVALID for NULL or empty arguments, n_sweeps < 1, exactly one of gt_xyz / conf3d, several rigs
 *      without rig_dev and a rig index out of range (checked on the device); MVS_ERR_UNSUPPORTED for the anchor term, exec
 *      mode 1, history_size > 100 and what mvs_fit_stream refuses.  Nothing is changed by a refused call.
 *      Context state afterwards as after mvs_fit_stream (no keypoints, 3-D term off, no per-slot rigs), and the rig table
 *      holds the refined extrinsics (f, c and the scales unchanged).  Synchronises. */
int mvs_refine_cameras(mvs_ctx* ctx, const mvs_frame_stream* s, const int* rig_dev, const mvs_loss_config* stage,
                       const mvs_lbfgs_config* opt_cfg, int n_sweeps, float* R_host, float* t_host,
                       mvs_lbfgs_stats* camera_stats, mvs_lbfgs_stats* pose_stats, void* stream);

/* ---- host-buffer entry point (what a caller without device memory uses): copies keypoints and
 *      parameters host->device, runs `n_stages` optimisation stages (one mvs_loss_config each, the weight
 *      schedule of code/utils/non_linear_solver.py:109-203), copies parameters and losses back.
 *      Stages are scheduled as in mvs_fit.  All pointers are HOST pointers; synchronises. */
int mvs_fit_host(mvs_ctx* ctx, float* params_host, const float* gt_uv_host, const float* conf_host,
                 const float* joint_weights_host, int n_stages, const mvs_loss_config* stage_cfgs,
                 const mvs_lbfgs_config* opt_cfg, float* final_loss_host, mvs_lbfgs_stats* stats, void* stream);

/* ---- initial guess for all frames of the batch (code/utils/init_guess.py:18-107 + fix_params :190-212, which
 *      main.py:76-82 runs per frame in numpy before the solver): triangulates the K keypoints from the V >= 2 views
 *      (code/utils/recompute3D.py:24-61, as written; with ONE view the rest joints are pushed along the optical axis by the
 *      depth guess of init_guess.py:54-78 instead, as written), aligns the model's rest joints (zero pose, zero shape,
 *      scale = fixed_scale) to them with a similarity transform (code/utils/umeyama.py:18 -> the published
 *      algorithm, Umeyama PAMI 1991; the file's own transposed-V variant depends on the LAPACK build's sign
 *      convention, see oracle/init_oracle.py) and writes the parameter block the solver starts from:
 *      betas 0, global_orient = axis-angle of R (cv2.Rodrigues, init_guess.py:86), body_pose 0 except the first six
 *      entries = hip_seed (fix_params; the reference uses 1.0; ignored when the loss config has use_vposer = 2, where
 *      the pose slots hold the latent code, which is zeroed as init_guess.py:96-98 does), transl = t, scale = s or
 *      fixed_scale.  Frames whose detections are degenerate (rank < 2) get the translation of the centroids only.
 *      With the 3-D joint term on (mvs_set_joints3d) the alignment target is the 3-D annotations instead of the triangulated
 *      or depth-guessed keypoints (init_guess.py:85-86), and one view needs no keypoints 5, 6, 11, 12 unless use_torso is set.
 *      params_dev [B,86] is overwritten; joints3d_dev [B,K,3] receives the alignment target (may be NULL).
 *      Uses the keypoints and cameras already uploaded; asynchronous on `stream`.  The rest joints are computed once per
 *      context and fixed_scale (seed + the 3-kernel geometry chain) and cached: a call is one launch afterwards.
 *      The warm start of sequences (load_init, init_guess.py:137-166) is a parameter copy done by mvs_fit_seq_stream on the
 *      device; with mvs_fit_seq the caller passes the previous result as the frame's params row and marks it warm. */
typedef struct {
    int estimate_scale;            /* not setting['fix_scale'] (init_guess.py:24) */
    float fixed_scale;             /* setting['fixed_scale'] or 1 (init_guess.py:25) */
    int use_torso;                 /* align on keypoints 5, 6, 11, 12 only (main.py:77 passes True) */
    float hip_seed;                /* fix_params init_guess.py:198-201: 1.0 in the reference */
    int umeyama_as_written;        /* 0: the published Umeyama algorithm (default).  1: what code/utils/umeyama.py computes: its
                                      full-rank branch multiplies by the transpose of numpy's V^H (:67) -- a product that depends
                                      on the sign convention of the LAPACK build; evaluated here with "largest-magnitude
                                      component of every right singular vector positive" -- plus its two-candidate patch and
                                      the translation taken from the negated candidate (:77-107).  Like sdf_all_faces = 0, the
                                      switch exists for parity with the file, not because the result is a better fit. */
} mvs_init_config;
int mvs_init_guess(mvs_ctx* ctx, float* params_dev, float* joints3d_dev, const mvs_init_config* cfg, void* stream);

/* ---- SDF grid: replaces the pybind op sdf.csrc.sdf(phi, faces, vertices) (sdf/sdf/csrc/sdf_cuda.cpp:14-28,
 *      kernel sdf_cuda_kernel.cu:242-335).  phi_dev [B,G,G,G] (written), faces_dev int32 [*,3],
 *      verts_dev [B,n_verts,3] normalised to [-1,1].  num_faces is what the kernel loops over
 *      (the reference call passes 1, see SURVEY A12). */
int mvs_sdf_grid(mvs_ctx* ctx, float* phi_dev, const int* faces_dev, int num_faces, const float* verts_dev,
                 int batch, int n_verts, int grid_size, void* stream);

/* ---- render fitted meshes into every view's image (what the reference's save_images option draws with pyrender and cv2,
 *      code/utils/utils.py:574-712, 866-882), see DESIGN.md section 4d.  For every frame f < n_frames with rig r and every view
 *      v < V_r: the mesh verts_dev [n,N,3] (e.g. what mvs_forward writes) projected through view v (with its lens distortion),
 *      rasterised with a depth buffer (pixel (x, y) sampled at (u, v) = (x, y); watertight edges, top-left fill rule, both
 *      windings; a triangle with a vertex at camera depth <= 1e-3 is not drawn), shaded by a headlight plus ambient light and
 *      drawn opaque over the background, with a filled disc of marker_radius px in marker_color around every keypoint of
 *      keypoints_dev [n,K,3] (NULL: no markers) in front of the camera.
 *      rig_dev [n] (device ints) names each frame's rig; NULL: rig 0, allowed only with a table of one rig.
 *      background_dev [n,Vmax,H,W,3] uint8 (NULL: black).  Outputs, each [n,Vmax,H,W(,3)] and each may be NULL but not all:
 *      image_dev (uint8), face_dev (int32, -1 = background), depth_dev (float, +inf = background).  Rows v >= V_r are not
 *      written.  A shaded channel is min(255, floor(255 base_color[c] I + 1/2)), I = ambient + (1 - ambient) max(0, n.l) with
 *      the interpolated camera-space normal n and l the unit vector from the surface point to the camera.  Deterministic: a
 *      frame gets the same bits alone and in a call of any size.  Needs mvs_set_model with faces and cameras; uses no batch,
 *      keypoints, loss configuration or optimiser state and changes none.  Refused (MVS_ERR_INVALID, nothing written): no
 *      faces or cameras, n_frames < 1, verts_dev NULL, all outputs NULL, a size or config value out of range or not finite,
 *      several rigs without rig_dev, a rig index out of range (naming the frame).  Enqueued on `stream`; synchronises it once
 *      per chunk of frames to size the screen tiles' triangle lists (and once for the rig check when rig_dev is given). */
typedef struct {
    int width, height;               /* every view's image size, 1 .. 8192 */
    float base_color[3];             /* in the images' channel order, [0, 1] */
    float ambient;                   /* [0, 1] */
    float marker_radius;             /* px, >= 0; 0 = no markers */
    unsigned char marker_color[3];
} mvs_render_config;
int mvs_render(mvs_ctx* ctx, int n_frames, const float* verts_dev, const float* keypoints_dev, const int* rig_dev,
               const unsigned char* background_dev, unsigned char* image_dev, int* face_dev, float* depth_dev,
               const mvs_render_config* cfg, void* stream);

/* Execution mode: 0 (default) = frame-resident kernels wherever they apply (sparse regime: no vertices requested,
 * no SDF term): one CTA per frame runs the closure -- and in mvs_lbfgs_run / mvs_fit_host the frame's whole
 * L-BFGS stage -- out of shared memory;  1 = always the batched multi-kernel path (used by tests to cross-check);
 * 2 = like 0, but mvs_fit / mvs_fit_host keep a barrier between stages (one run per stage, as mvs_lbfgs_run);
 * 3 = like 0, and mvs_closure with the SDF term on (loss and gradient only) runs ONE evaluation through the dense-regime
 *     kernels the optimiser uses for SDF stages instead of the batched reference chain (parity tests; synchronises).
 *     Mode 3 affects mvs_closure only: the optimiser entry points (mvs_lbfgs_run, mvs_lbfgs_step, mvs_fit*) run as in 0. */
int mvs_set_exec_mode(mvs_ctx* ctx, int mode);

/* ---- measurement support (bench.py): per-kernel device time with CUDA events recorded on the launching
 *      stream around every launch whose kernel id bit is set in `mask` (0 = off, the default).
 *      mvs_profile_read synchronises the device, adds up the elapsed times since the last mvs_profile call
 *      and writes, for kernel id k < MVS_NUM_KERNEL_IDS, ms[k] and launches[k]. */
#define MVS_NUM_KERNEL_IDS 19
int mvs_profile(mvs_ctx* ctx, unsigned mask);
int mvs_profile_read(mvs_ctx* ctx, double* ms, long long* launches);
const char* mvs_kernel_name(int kernel_id);

#ifdef __cplusplus
}
#endif
#endif /* MVSMPL_H_ */
