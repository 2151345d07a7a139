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
 * R [V,3,3], t [V,3], f [V,2] (focal x,y), c [V,2] */
int mvs_set_cameras(mvs_ctx* ctx, int num_views, const float* R, const float* t, const float* f, const float* c);

/* frames in flight (the reference is fixed to 1: code/utils/non_linear_solver.py:56); allocates workspace */
int mvs_set_batch(mvs_ctx* ctx, int num_frames);

/* 2-D detections: gt_uv [V,B,K,2], conf [V,B,K], joint_weights [K]
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
    int dense_rounds;              /* of rounds: dense rounds (gemm -> skin -> sdf_fused -> frame_step each) */
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
 *      params_dev [B,86] is overwritten; joints3d_dev [B,K,3] receives the triangulated keypoints (may be NULL).
 *      Uses the keypoints and cameras already uploaded; asynchronous on `stream`.  The rest joints are computed once per
 *      context and fixed_scale (seed + the 3-kernel geometry chain) and cached: a call is one launch afterwards.
 *      The warm start of sequences (load_init, init_guess.py:137-166) is a parameter copy and has no entry point: pass the
 *      previous result as params to mvs_fit with skip_stages (below). */
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

/* Execution mode: 0 (default) = frame-resident kernels wherever they apply (sparse regime: no vertices requested,
 * no SDF term): one CTA per frame runs the closure -- and in mvs_lbfgs_run / mvs_fit_host the frame's whole
 * L-BFGS stage -- out of shared memory;  1 = always the batched multi-kernel path (used by tests to cross-check);
 * 2 = like 0, but mvs_fit / mvs_fit_host keep a barrier between stages (one run per stage, as mvs_lbfgs_run);
 * 3 = like 0, and mvs_closure with the SDF term on (loss and gradient only) runs ONE evaluation through the dense-regime
 *     kernels the optimiser uses for SDF stages instead of the batched reference chain (parity tests; synchronises). */
int mvs_set_exec_mode(mvs_ctx* ctx, int mode);

/* ---- measurement support (bench.py): per-kernel device time with CUDA events recorded on the launching
 *      stream around every launch whose kernel id bit is set in `mask` (0 = off, the default).
 *      mvs_profile_read synchronises the device, adds up the elapsed times since the last mvs_profile call
 *      and writes, for kernel id k < MVS_NUM_KERNEL_IDS, ms[k] and launches[k]. */
#define MVS_NUM_KERNEL_IDS 18
int mvs_profile(mvs_ctx* ctx, unsigned mask);
int mvs_profile_read(mvs_ctx* ctx, double* ms, long long* launches);
const char* mvs_kernel_name(int kernel_id);

#ifdef __cplusplus
}
#endif
#endif /* MVSMPL_H_ */
