/*
 * caliscope_b200 -- C ABI of the H100 bundle-adjustment engine.
 *
 * Drop-in boundary for the bundle-adjustment hot path of mprib/caliscope.  The
 * reference has no FFI; its seam is the Python call
 *     scipy.optimize.least_squares(joint_residuals, x0, args=(...), jac=joint_jacobian, ...)
 * at /root/reference/src/caliscope/core/capture_volume.py:387-411 (inside
 * CaptureVolume.optimize, :322-444).  The entry points below are what a ctypes
 * binding behind that seam calls; INTEGRATION.md shows the stub.
 *
 * Conventions: plain pointers and sizes, fp64, row-major, no exceptions cross the
 * ABI.  Every function returns 0 on success or a negative CB_E_* code;
 * cb_ba_error_string() gives the text, cb_ba_last_error() the detail (CUDA error
 * string) of the most recent failure on the calling thread.
 *
 * Parameter vector layout == BundleParameterization.pack
 * (/root/reference/src/caliscope/core/bundle_parameterization.py:127-149):
 *   x = [block_0 | ... | block_{n_cams-1} | X_0 | X_1 | ...],
 *   block_i = [rvec(3), tvec(3)] (+ [s, k1, k2] iff cam_flags[i] & CB_CAM_FREE_INTRINSICS),
 *   X_j = xyz of world point j.
 */
#ifndef CALISCOPE_B200_H
#define CALISCOPE_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CB_BA_ABI_VERSION 3

/* cam_flags bits (CameraBlock.free_intrinsics / .fisheye, bundle_parameterization.py:36-51) */
#define CB_CAM_FREE_INTRINSICS 1
#define CB_CAM_FISHEYE 2

/* loss ids: scipy.optimize.least_squares(loss=...) as forwarded by capture_volume.py:405 */
#define CB_LOSS_LINEAR 0
#define CB_LOSS_SOFT_L1 1
#define CB_LOSS_HUBER 2
#define CB_LOSS_CAUCHY 3
#define CB_LOSS_ARCTAN 4

/* error codes */
#define CB_OK 0
#define CB_E_INVALID (-1)      /* bad argument (null pointer, index out of range, ...) */
#define CB_E_CUDA (-2)         /* CUDA runtime failure; see cb_ba_last_error() */
#define CB_E_NO_DEVICE (-3)    /* no usable CUDA device */
#define CB_E_UNSUPPORTED (-4)  /* feature not implemented by this build */
#define CB_E_CALLBACK (-5)     /* the all-reduce callback reported failure */
#define CB_E_NOMEM (-6)

typedef struct CbBaProblem CbBaProblem; /* opaque, device resident */

/*
 * Problem description == the args tuple CaptureVolume.optimize hands to scipy
 * (capture_volume.py:390-399) plus BundleParameterization.blocks flattened.
 *   cam_const[i*9 + 0..8] = fx_initial, fy_initial, cx, cy, c4..c8 where
 *     Brown-Conrady: (c4..c8) = (k1_initial, k2_initial, p1, p2, k3)
 *     fisheye      : (c4..c7) = (k1, k2, k3, k4), c8 unused
 *   obs_cam  = camera_indices          (capture_volume.py:353-355; int16 there, int32 here)
 *   obs_pt   = image_to_world_indices  (capture_volume.py:358)
 *   obs_xy   = image_coords            (capture_volume.py:357), n_obs x 2
 * obs_* may be host pointers (obs_on_device = 0; copied inside the call) or device
 * pointers on `device` (obs_on_device = 1).  Inputs are never modified.
 */
typedef struct {
  int32_t n_cams;
  int32_t n_pts;
  int64_t n_obs;
  const int32_t* cam_flags; /* host, n_cams */
  const double* cam_const;  /* host, n_cams*9 */
  const int32_t* obs_cam;
  const int32_t* obs_pt;
  const double* obs_xy;
  int32_t obs_on_device;
  int32_t obs_cam_bits; /* 0 or 32: obs_cam is int32; 16: obs_cam is int16 (what capture_volume.py:353-355 builds) and is
                           widened on the device -- halves that upload and saves the caller a conversion pass */
  /* Optional (NULL: the engine decides).  Internal camera order, host, n_cams entries: cam_order[slot] = camera index.
   * Only the layout of the reduced camera system depends on it (cameras that see the same points should be neighbours,
   * so that whole 96-column tile pairs of the Schur product are empty); no input or output of the ABI is reordered.
   * Every rank of a sharded solve MUST pass the same order (caliscope_b200.distributed does). */
  const int32_t* cam_order;
  /* Rigid-distance constraint rows (reprojection.py:112-117 and :207-226): groups_a / groups_b are n_constraints x 4
   * world-point row indices, distances and weights n_constraints doubles -- the arrays
   * CaptureVolume._build_constraint_arrays produces (capture_volume.py:446-516) with
   * weights = (pixel_sigma / f_median) / sigma (:377-381).  Host pointers, copied; ignored when n_constraints == 0.
   * Under observation sharding every point a row touches must belong to the same rank (shard by connected component
   * of the constraint graph). */
  int64_t n_constraints;
  const int32_t* groups_a;
  const int32_t* groups_b;
  const double* distances;
  const double* weights;
} CbBaProblemDesc;

/*
 * Sum-all-reduce hook for observation sharding (one process per GPU).  Called on
 * the host thread inside cb_ba_solve with a DEVICE buffer of n doubles that must be
 * summed element-wise across ranks in place, ordered after all work already queued
 * on `stream` and before any work queued afterwards (torch.distributed.all_reduce on
 * the current stream satisfies this).  Return 0 on success.
 */
typedef int (*CbAllReduceSum)(void* user, double* device_buf, int64_t n, void* stream);

/* least_squares keyword arguments the reference passes (capture_volume.py:403-410)
 * plus scipy's defaults for the ones it leaves out (xtol = gtol = 1e-8). */
typedef struct {
  double ftol;
  double xtol;
  double gtol;
  int64_t max_nfev; /* <= 0: scipy's default 100 * n */
  int32_t loss;     /* CB_LOSS_* */
  double f_scale;
  int32_t verbose;     /* 0 silent, 1 summary, 2 per-iteration table on stderr */
  int32_t use_bounds;  /* 1: s in [0.5,2], k1 in [-1,1], k2 in [-2,2] (bundle_parameterization.py:151-164) */
  double lambda0;      /* initial LM damping; <= 0: 1e-4 */
  double pcg_tol;      /* relative PCG tolerance for the reduced camera system; <= 0: 1e-6 */
  int32_t pcg_max_iter; /* <= 0: 4 * n_camera_params */
  CbAllReduceSum allreduce; /* NULL: single GPU (unless nccl_comm is set) */
  void* allreduce_user;
  void* nccl_comm;          /* ncclComm_t from cb_nccl_comm_create: the engine calls ncclAllReduce itself on the solve stream */
  void* peer_group;         /* CbPeerGroup* from cb_peer_create/_connect: all-reduce over NVLink peer memory, fused into
                               the Schur finalize kernel (takes precedence over nccl_comm / allreduce) */
  int32_t rank;       /* informational (verbose output only on rank 0) */
  int32_t world_size; /* 1 if allreduce is NULL */
  int32_t time_kernels; /* diagnostic: launch every trial directly with CUDA events around the point pass and the Schur
                           product (CbBaResult.rj_ms / syrk_ms); 0 (default): the trials are replayed from CUDA graphs
                           (see used_graph), where events cannot be read back */
  int32_t pad_;
} CbBaOptions;

/* mirrors scipy.optimize.OptimizeResult fields the reference reads
 * (capture_volume.py:413-433): status, nfev, cost; plus njev/nit/optimality. */
typedef struct {
  int32_t status; /* scipy codes: 0 max_nfev, 1 gtol, 2 ftol, 3 xtol, 4 ftol&xtol */
  int64_t nfev;
  int64_t njev;
  int64_t nit;       /* LM iterations (linearisations solved) */
  double cost;       /* 0.5 * sum rho(f^2), scipy's definition */
  double initial_cost;
  double optimality; /* inf-norm of the gradient at the solution */
  double lambda_final;
  int64_t pcg_iterations; /* total PCG iterations over the solve */
  int64_t kernel_launches;
  double solve_ms; /* device time of the LM loop (CUDA events on the solve stream) */
  double rj_ms;    /* total device time spent in the residual+Jacobian (point pass) kernel, CUDA events around each launch */
  int64_t rj_launches;
  double syrk_ms;  /* total device time spent in the Schur product kernel */
  int64_t syrk_launches;
  int64_t trials_queued; /* LM trials handed to the device (the last one runs predicated-off) */
  int32_t used_graph;    /* how the trials ran: 2 device loop, one WHILE-conditional graph per solve (one GPU); 1 one CUDA
                            graph per trial (sharded over nccl_comm or peer_group); 0 launched directly (allreduce callback,
                            time_kernels, or a graph that could not be built) */
  int32_t pad_;
} CbBaResult;

int cb_ba_abi_version(void);
const char* cb_ba_error_string(int code);
const char* cb_ba_last_error(void);
void cb_ba_default_options(CbBaOptions* opt);

/* Upload + index build (sort by camera / by point, chunk and pair tables, constraint components). */
int cb_ba_problem_create(const CbBaProblemDesc* desc, int device, void* stream, CbBaProblem** out);
/* The same problem with some parameters held at their values in x0 (DESIGN.md section 4.12): every solve is the solve of
 * the problem over the free parameters alone (scipy's least_squares on the free subvector), and the fixed entries of the
 * returned x are bit-identical to x0.  cb_ba_problem_create is this call with both lists empty.
 *   fixed_cam_params (host): n_fixed_cam_params indices into x's camera section, caller layout (as cb_ba_covariance's
 *                    `fixed`).  A fixed camera parameter's rows and columns of the reduced system S are unit vectors and
 *                    its entry of b is 0; observations still contribute to the camera's free parameters.
 *   fixed_pts (host): n_fixed_pts point indices.  A fixed point is a known 3-D point: its observations contribute to the
 *                    cost and the camera blocks, it has no Schur term, no step and no place in the gradient norm.
 * CB_E_INVALID for an index out of range or repeated, or when no free parameter is left; CB_E_UNSUPPORTED for a fixed point
 * in a rigid-distance constraint row.  All of these are refused before any device work.  cb_ba_cull's filtered problem
 * keeps both sets; cb_ba_covariance treats the fixed camera parameters as part of its `fixed` and the fixed points as
 * constants; a sharded cb_ba_solve (allreduce, nccl_comm or peer_group) on such a problem fails with CB_E_UNSUPPORTED. */
int cb_ba_problem_create_fixed(const CbBaProblemDesc* desc, int32_t n_fixed_cam_params, const int32_t* fixed_cam_params,
                               int32_t n_fixed_pts, const int32_t* fixed_pts, int device, void* stream,
                               CbBaProblem** out);
/* Gaussian priors on chosen cameras and points (DESIGN.md section 4.13).  Each adds a quadratic term to the objective,
 * whatever the loss:
 *   F(x) = 1/2 sum rho(r_i^2) + 1/2 sum_c (x_c - m_c)^T L_c (x_c - m_c) + 1/2 sum_j (X_j - m_j)^T L_j (X_j - m_j),
 * i.e. scipy's least_squares on the residuals extended by rows W (x - m) with W^T W = L that the loss leaves linear.  L
 * is symmetric positive semi-definite (a singular L is a partial prior) and in the objective's units: reprojection rows
 * are pixels / fx_initial, so a covariance Sigma under pixel noise sigma gives L = (sigma / fx)^2 Sigma^-1.  Host pointers,
 * copied at creation:
 *   cams: n_cams camera indices (caller numbering); cam_mean n_cams x 9: the camera's slice of x (6 or 9 values, the rest
 *         ignored); cam_info n_cams x 9 x 9, row-major, zero outside the 6 x 6 block of a 6-parameter camera.
 *   pts: n_pts point indices; pt_mean n_pts x 3; pt_info n_pts x 3 x 3, row-major. */
typedef struct {
  int32_t n_cams;
  const int32_t* cams;
  const double* cam_mean;
  const double* cam_info;
  int32_t n_pts;
  const int32_t* pts;
  const double* pt_mean;
  const double* pt_info;
} CbBaPriors;

/* cb_ba_problem_create_fixed with Gaussian priors (priors may be NULL: cb_ba_problem_create_fixed is this call with
 * priors = NULL).  A solve minimises F above over the free parameters; a fixed entry of a camera with a prior stays x0's,
 * and the prior still pulls the camera's free entries through the off-diagonal of L.  Refused before any device work:
 * CB_E_INVALID for an index out of range or repeated within its list, a non-finite mean or information entry, an L that
 * is not symmetric to 1e-12 relative or has an eigenvalue below -1e-12 of its largest, non-zero information outside a
 * 6-parameter camera's 6 x 6 block, or a point that is both fixed and has a prior; CB_E_UNSUPPORTED for a point prior on
 * a point of a rigid-distance constraint row.  A sharded cb_ba_solve on a problem with priors fails with
 * CB_E_UNSUPPORTED.  cb_ba_cull's filtered problem keeps the priors; cb_ba_normal_equations returns S, b, U, gc, V, gp
 * and the cost with them; the cost, initial_cost and optimality of a solve include them; cb_ba_covariance inverts the
 * reduced system with them and counts sum rank(L) more rows in m. */
int cb_ba_problem_create_priors(const CbBaProblemDesc* desc, int32_t n_fixed_cam_params, const int32_t* fixed_cam_params,
                                int32_t n_fixed_pts, const int32_t* fixed_pts, const CbBaPriors* priors, int device,
                                void* stream, CbBaProblem** out);
int cb_ba_problem_destroy(CbBaProblem* p);
int64_t cb_ba_problem_n_params(const CbBaProblem* p);
/* Facts about how the engine laid the problem out (measurement / diagnostics): what = 0: 1 if the Schur product walks
 * compacted row lists (sparse visibility), 1: floating-point operations one Schur-product launch issues, 2: 1 if the reduced
 * system is solved directly (<= 96 camera parameters), 3: CTAs of the Schur product, 4 / 5 / 6: see cb_ba_covariance,
 * 7: lanes per point in the point kernels (8, or 32 when points average more than 96 rows), 8: 1 if some (camera, point)
 * pair has repeated rows, 9: 1 if the point kernels stage the camera table in shared memory, 10: reduced solve (0 direct,
 * 1 PCG with the slab streamed from L2, 2 PCG with the slab in registers), 11: CTAs of the PCG cluster, 12: matrix
 * columns per lane of the register PCG (0 otherwise), 13: 1 if the internal camera order is not the caller's numbering,
 * 14-17: host microseconds the last cb_ba_solve spent on the bounds, the start state, the upload of x, and the LM loop
 * with the download of x up to its one synchronisation.  -1 for an unknown key. */
double cb_ba_problem_stat(const CbBaProblem* p, int what);

/* Constraint rows at x, n_c = CbBaProblemDesc.n_constraints: r_out (n_c) == the tail of joint_residuals; dir_out (n_c x 3,
 * nullable) = weight * unit vector between the two endpoint means: the Jacobian entry of a group-a (group-b) member is
 * +(-) dir / 4, repeats summed. */
int cb_ba_constraint_rows(CbBaProblem* p, const double* x, double* r_out, double* dir_out, void* stream);

/* Replaces least_squares(joint_residuals, x0, jac=joint_jacobian, method="trf", ...)
 * (capture_volume.py:387-411).  x_inout: host, n_params doubles, overwritten with result.x (after a failure: see
 * cb_ba_solve_from). */
int cb_ba_solve(CbBaProblem* p, const CbBaOptions* opt, double* x_inout, CbBaResult* result, void* stream);
/* The same solve from x0 into x_out (host, n_params doubles each; they may be the same array), so that a caller who
 * keeps x0 needs no copy of it.  x_out is written only by a solve that ran to its end (its content is unspecified after
 * a failure reported by the device or by a peer rank). */
int cb_ba_solve_from(CbBaProblem* p, const CbBaOptions* opt, const double* x0, double* x_out, CbBaResult* result,
                     void* stream);

/* == joint_residuals (reprojection.py:75-119), reprojection rows only: r_out host, 2*n_obs,
 * interleaved (x, y) / fx_initial in the caller's observation order. */
int cb_ba_residuals(CbBaProblem* p, const double* x, double* r_out, void* stream);

/* Dense blocks of joint_jacobian (reprojection.py:171-205) in the caller's observation order:
 * Jc host n_obs*2*9 (columns rvec3, tvec3, s, k1, k2; zeros where a block is locked),
 * Jp host n_obs*2*3; both already divided by fx_initial. */
int cb_ba_jacobian_blocks(CbBaProblem* p, const double* x, double* Jc, double* Jp, void* stream);

/* == reprojection_errors (reprojection.py:35-72): pixel errors with the intrinsics in x. err_xy host n_obs*2. */
int cb_ba_reproj_errors_px(CbBaProblem* p, const double* x, double* err_xy, void* stream);

/* Test/diagnostic access to one damped linearisation (all host outputs, any may be NULL):
 * U n_cams*P*P, gc n_cams*P, V n_pts*9, gp n_pts*3, S (n_cams*P)^2, b n_cams*P,
 * dc n_cams*P (PCG solution of S dc = -b), dp n_pts*3 (back-substituted), with P = cb_ba_cam_stride().  On a problem
 * with fixed parameters S, b, dc and dp are those the solve uses: fixed camera parameters have unit rows and columns of
 * S before the damping, zero b and zero dc; fixed points have zero dp. */
int cb_ba_cam_stride(const CbBaProblem* p);
int cb_ba_normal_equations(CbBaProblem* p, const double* x, double lambda, int32_t loss, double f_scale,
                           double* cost, double* U, double* gc, double* V, double* gp, double* S, double* b,
                           double* dc, double* dp, void* stream);

/* Covariance of the parameters at x (normally a solution), DESIGN.md section 4.6.  With J the engine's residual Jacobian
 * (pixels / fx_initial, then the constraint rows, then the rows W (x - m) of any priors) after the robust row rescaling
 * at x:
 *   Sigma = s2 * (J_F^T J_F)^-1,  F = parameters neither fixed nor masked,
 * through the Schur complement at lambda = 0 with the pseudo-inverse of every 3x3 point block V_j (a point seen by one
 * camera has rank(V_j) = 2, an unobserved point 0: their null directions are not parameters of F).
 *   fixed: n_fixed indices into x's camera section (caller layout), the gauge (caliscope_b200.uncertainty.default_gauge);
 *          their rows and columns of cam_cov are 0.  The problem's own fixed camera parameters (cb_ba_problem_create_fixed)
 *          join them; its fixed points are constants: pt_cov zero, pt_rank -2, and 3 parameters each fewer in the rank.
 *   masked: every parameter of a camera without observations; NaN rows and columns of cam_cov.
 *   variance_factor > 0: s2 as given (e.g. (pixel_sigma / fx)^2); <= 0: s2 = 2 cost / dof with dof = m - rank,
 *          m = 2 n_obs + n_c (+ sum rank(L) over the problem's priors, cb_ba_problem_create_priors),
 *          rank = n_params - |fixed| - |masked| - sum_j (3 - rank V_j) over unconstrained points.
 *   cam_cov (nullable): n_camera_params^2, caller layout.  pt_cov (nullable): n_pts*9, NaN for points with a rank
 *          deficient V_j and for points of rigid-constraint components.  pt_rank (nullable): n_pts, rank of V_j, -1 for
 *          component points.  s2_out / dof_out nullable.
 * Fails with CB_E_INVALID when the gauge-fixed reduced system S_F is not positive definite (a Cholesky pivot at or below
 * CB_COV_PIVOT_RTOL times the parameter's diagonal of S_F; cb_ba_last_error() names the camera and parameter), or when a
 * constraint component's block is not positive definite at lambda = 0.  The problem must hold every observation: a
 * per-rank shard of a sharded problem holds only part of the information.  cb_ba_problem_stat(p, 4 / 5 / 6) give the
 * last call's milliseconds (CUDA events) in linearisation + Schur product, dense inverse, and point marginals. */
#define CB_COV_PIVOT_RTOL 1e-10
int cb_ba_covariance(CbBaProblem* p, const double* x, int32_t loss, double f_scale, int32_t n_fixed, const int32_t* fixed,
                     double variance_factor, double* cam_cov, double* pt_cov, double* s2_out, int64_t* dof_out,
                     int32_t* pt_rank, void* stream);

/* Per-camera order statistics of the pixel error norm for the percentile filter
 * (capture_volume.py:709-753): for camera c with n_c observations, lo[c] / hi[c] are the
 * floor / ceil order statistics of rank (n_c - 1) * q / 100 (numpy's linear interpolation
 * nodes), count[c] = n_c; err host n_obs (euclidean error per observation, caller order). */
int cb_ba_error_order_stats(CbBaProblem* p, const double* x, double q_percent, double* err, double* lo,
                            double* hi, int64_t* count, void* stream);

/* Overall and per-camera (nullable, n_cams) RMS pixel error, reduced on the device
 * (ReprojectionReport.overall_rmse / by_camera, capture_volume.py:197-202). */
int cb_ba_rmse_px(CbBaProblem* p, const double* x, double* overall, double* per_camera, void* stream);

/* Device-side observation cull == _filter_by_reprojection_thresholds (capture_volume.py:607-646) at array level:
 * keep error <= thresholds[camera] (host, n_cams), restore lowest-error observations up to min_per_camera, compact
 * the observation list on the device and build the filtered problem (same cameras and point numbering) from it.
 * keep_mask: host, n_obs bytes in the caller's observation order, or NULL.  *out must be destroyed by the caller.
 * min_per_camera = 0 applies the thresholds only (sharded solves: the floor is a global property and is folded into the
 * thresholds by the caller, caliscope_b200/distributed.global_cull_thresholds). */
int cb_ba_cull(CbBaProblem* p, const double* x, const double* thresholds, int32_t min_per_camera, CbBaProblem** out,
               int64_t* n_kept, uint8_t* keep_mask, void* stream);

/* Diagnostic: mean milliseconds of one PCG-kernel launch forced to run exactly max_iter iterations on the
 * system left by the last cb_ba_normal_equations call.  CB_E_UNSUPPORTED on problems of at most 96 camera parameters,
 * which are solved directly (small_rig_step_kernel), not by PCG. */
int cb_ba_debug_pcg_time(CbBaProblem* p, int max_iter, int reps, double* ms_per_launch, void* stream);

/* Measured fp64 throughput of the device (TFLOP/s): `mma.sync.m8n8k4.f64` (DMMA, the tensor path the Schur product
 * runs on) and plain DFMA register chains, 8 warps per SM, a few milliseconds each.  The roofline denominator for the
 * Schur product; there is no driver-measured fp64 figure in MEASURED_PEAKS.json. */
int cb_debug_fp64_peak(int device, double* dmma_tflops, double* dfma_tflops);

/* ---- the step in front of bundle adjustment (SURVEY.md §8(f) rank 3) ------------------------------------------- */

/* == CameraData.undistort_points (reference cameras/camera_array.py:135-174): cv2.undistortPoints (5 fixed-point
 * iterations) / cv2.fisheye.undistortPoints (Newton on theta) on float32 copies of the points, float32 results,
 * here for the observations of all cameras in one launch.
 *   cam_fisheye[n_cams]; cam_k[n_cams][5] = fx,fy,cx,cy,skew; cam_dist[n_cams][12] = k1 k2 p1 p2 k3 k4 k5 k6 s1..s4
 *   (zero-padded; fisheye: k1..k4); obs_cam[n] camera row per point (NULL with a single camera);
 *   to_pixels: 0 = normalised image plane (P = I), 1 = pixels (P = K).
 *   on_device: xy_in / obs_cam / xy_out are device pointers.
 * Pinhole results are bit-exact with OpenCV; fisheye within one float32 ulp (device tan).  Edges as OpenCV:
 *   a fisheye point whose Newton iteration does not converge or flips theta's sign is (-1e6, -1e6) in both outputs;
 *   NaN / inf input: pinhole (NaN, NaN); fisheye normalised: a NaN theta_d is clamped to -pi/2 and iterated, so the
 *   finite coordinate keeps a value (e.g. (NaN, 100) -> (NaN, y)); any non-finite result in pixel output is (NaN, NaN). */
int cb_undistort_points(int32_t n_cams, const int32_t* cam_fisheye, const double* cam_k, const double* cam_dist,
                        int64_t n, const int32_t* obs_cam, const double* xy_in, int on_device, int to_pixels,
                        double* xy_out, int device, void* stream);

typedef struct CbTriStats {
  double group_ms;  /* upload + radix sort + group boundaries */
  double dlt_ms;    /* the DLT kernel alone (CUDA events on the launch stream) */
  double total_ms;
  int32_t kernel_launches;
  int32_t pad_;
} CbTriStats;

/* == triangulate_image_points (reference core/point_data.py:122-229).  Observations with equal obs_key (a
 * non-negative 63-bit packing of (sync_index, object_id, keypoint_id) made by the caller) form one group; every
 * group gets the DLT point of its rows  [x*P2 - P0 ; y*P2 - P1]  (smallest right singular vector, via the 4x4 normal
 * matrix), groups in ascending key order.  proj = host [n_cams][3][4] normalised projection matrices.
 * Outputs (host, room for max_groups): xyz[g][3] (NaN when the group has < 2 rows), count[g], rep_row[g] = caller
 * row of the group's first observation, camset_sig[g][2] = order-independent 128-bit signature of the group's
 * camera multiset (lets the host mirror reproduce the reference's by-camera-set output order). */
int cb_triangulate_dlt(int32_t n_cams, const double* proj, int64_t n_obs, const int32_t* obs_cam,
                       const int64_t* obs_key, const double* obs_xy, int obs_on_device, int32_t max_groups,
                       int32_t* n_groups_out, double* xyz_out, int32_t* count_out, int32_t* rep_row_out,
                       uint64_t* camset_sig_out, CbTriStats* stats, int device, void* stream);

/* cb_undistort_points (normalised output) + cb_triangulate_dlt in one call: obs_px are raw pixels, the undistorted
 * coordinates stay in HBM between the two kernels (what ImagePoints.triangulate does, point_data.py:416-559). */
int cb_undistort_triangulate(int32_t n_cams, const int32_t* cam_fisheye, const double* cam_k, const double* cam_dist,
                             const double* proj, int64_t n_obs, const int32_t* obs_cam, const int64_t* obs_key,
                             const double* obs_px, int obs_on_device, int32_t max_groups, int32_t* n_groups_out,
                             double* xyz_out, int32_t* count_out, int32_t* rep_row_out, uint64_t* camset_sig_out,
                             CbTriStats* stats, int device, void* stream);

typedef struct CbTriRefineStats {
  double group_ms;   /* upload + undistortion + radix sort + group boundaries */
  double dlt_ms;     /* the DLT start */
  double refine_ms;  /* the Levenberg-Marquardt kernel */
  double cov_ms;     /* the covariance kernel (0 without cov_out) */
  double total_ms;
  int32_t kernel_launches;
  int32_t pad_;
} CbTriRefineStats;

/* Triangulation with calibrated cameras to the reprojection optimum, with a first-order covariance per point
 * (DESIGN.md section 4.7).  Groups as cb_triangulate_dlt (equal obs_key, ascending key order).  The cameras are given in
 * the bundle-adjustment layout: cam_flags / cam_const as CbBaProblemDesc, cam_x = the camera section of x
 * (n_camera_params = sum of 6 or 9 per camera).  obs_px are raw pixels (float64, read at full precision).
 * Per group with >= 2 rows: the DLT point of cb_undistort_triangulate (projection matrices and lens tables derived from
 * cam_x) starts a Levenberg-Marquardt minimisation of sum_i |pi(X; c_i) - u_i|^2 in pixels (lambda0 = 1e-3, accept on a
 * lower cost with lambda / 10, else lambda * 10; stop when |dX| <= xtol (|X| + xtol) or after max_iter steps).
 *   cov = pixel_sigma^2 H^-1 + H^-1 G cam_cov G^T H^-1,  H = sum J_X^T J_X,  G = sum J_X^T J_c  (pixels; J_X, J_c the
 *   derivatives of the projection by the point and the camera parameters).  cam_cov (nullable: the first term alone) is
 *   the n_camera_params^2 camera covariance in x's camera layout (BAProblem.covariance's cameras).  It assumes the
 *   triangulated observations are independent of those the calibration used, and is relative to cam_cov's gauge.
 * Outputs (host, room for max_groups): xyz[g][3], cov[g][9] (nullable: no covariance stage), rmse_px[g] (reprojection
 * RMSE over the group's rows), count[g], rep_row[g] (as cb_triangulate_dlt) and status[g], first match wins:
 *   1 fewer than 2 rows (xyz, cov, rmse NaN);  2 H not positive definite at the start or at the solution (a Cholesky
 *   pivot <= 1e-12 times H's largest diagonal entry: parallel rays, or every row from one camera; xyz = the DLT point,
 *   rmse there, cov NaN);  3 max_iter reached;  4 behind a camera at the solution (some row with Xc.z <= 0);  0 none.
 * No atomics: repeated calls return bit-identical outputs. */
int cb_triangulate_refine(int32_t n_cams, const int32_t* cam_flags, const double* cam_const, const double* cam_x,
                          const double* cam_cov, int64_t n_obs, const int32_t* obs_cam, const int64_t* obs_key,
                          const double* obs_px, int obs_on_device, double pixel_sigma, int32_t max_iter, double xtol,
                          int32_t max_groups, int32_t* n_groups_out, double* xyz_out, double* cov_out,
                          double* rmse_px_out, int32_t* count_out, int32_t* rep_row_out, int32_t* status_out,
                          CbTriRefineStats* stats, int device, void* stream);

typedef struct CbTriRobustStats {
  double group_ms;      /* upload + undistortion + radix sort + group boundaries */
  double consensus_ms;  /* the consensus kernel and the compaction of the consensus rows */
  double refine_ms;     /* the Levenberg-Marquardt kernel on the consensus rows */
  double cov_ms;        /* the covariance kernel (0 without cov_out) */
  double total_ms;
  int32_t kernel_launches;
  int32_t pad_;
} CbTriRobustStats;

/* cb_triangulate_refine on each group's consensus rows, chosen by view-pair consensus (DESIGN.md section 4.8).  Inputs
 * as cb_triangulate_refine, plus threshold_px tau (finite, > 0), min_inliers (>= 2) and max_pairs (>= 1).  Inside a
 * group of k rows (key-sorted, caller order within a key, positions 0..k-1):
 *   candidate pairs: the pairs i < j ranked lexicographically, rank(i,j) = i k - i (i + 1) / 2 + (j - i - 1),
 *     T = k (k - 1) / 2; every rank when T <= max_pairs, else the ranks floor(m T / max_pairs), m = 0..max_pairs-1 (exact
 *     64-bit integers; no random sampling).
 *   hypothesis of a pair: none when both rows come from one camera; else the DLT point of the two rows (the normal
 *     matrix of cb_undistort_triangulate on float32-rounded undistorted coordinates, smallest eigenvector,
 *     de-homogenised); none when it is not finite or has Xc.z <= 0 in either of the pair's cameras.
 *   score (MSAC): sum over all k rows of min(e_r^2, tau^2), e_r = |pi(X; c_r) - u_r| in raw pixels with the engine's
 *     projection; a row with Xc.z <= 0 or a non-finite e_r adds tau^2.  The lowest score wins, the lowest rank on a tie.
 *   consensus set: the rows with Xc.z > 0 and e_r <= tau at the winner.
 * The refinement and covariance of cb_triangulate_refine then run on the consensus rows alone, started from the winning
 * hypothesis; rmse_px is over the consensus rows.  There is one consensus round: rows are not re-classified at the
 * refined point.  In a two-view group an error along the epipolar line cannot be seen.
 * Outputs (host, room for max_groups): xyz, cov (nullable), rmse_px, count (all rows of the group), n_inliers, rep_row
 * and status per group; inlier[n_obs] (1 = the caller row is in its group's consensus set).  status, first match wins:
 *   1 fewer than 2 rows;  5 no consensus: no valid hypothesis, or fewer than min_inliers consensus rows (xyz, cov, rmse
 *   NaN, n_inliers 0, no row inlier; a group whose rows all come from one camera is 5);  2, 3, 4 as cb_triangulate_refine
 *   (for 2, xyz = the hypothesis);  0 none.
 * No atomics: repeated calls return bit-identical outputs. */
int cb_triangulate_robust(int32_t n_cams, const int32_t* cam_flags, const double* cam_const, const double* cam_x,
                          const double* cam_cov, int64_t n_obs, const int32_t* obs_cam, const int64_t* obs_key,
                          const double* obs_px, int obs_on_device, double threshold_px, int32_t min_inliers,
                          int32_t max_pairs, double pixel_sigma, int32_t max_iter, double xtol, int32_t max_groups,
                          int32_t* n_groups_out, double* xyz_out, double* cov_out, double* rmse_px_out,
                          int32_t* count_out, int32_t* n_inliers_out, int32_t* rep_row_out, int32_t* status_out,
                          uint8_t* inlier_out, CbTriRobustStats* stats, int device, void* stream);

typedef struct CbResectStats {
  double group_ms;      /* upload + undistortion + radix sort + group boundaries */
  double consensus_ms;  /* hypotheses, MSAC scoring, selection and the compaction of the consensus rows */
  double refine_ms;     /* the Levenberg-Marquardt kernel on the consensus rows */
  double cov_ms;        /* the point sort and the covariance kernel (0 without cov_out) */
  double total_ms;
  int32_t kernel_launches;
  int32_t pad_;
} CbResectStats;

/* Robust resection: the pose of a camera from 2-D detections of points whose 3-D positions are known (DESIGN.md
 * section 4.9).  Cameras in the bundle-adjustment layout as cb_triangulate_refine; pts_xyz[n_pts][3] and pts_cov
 * (nullable) [n_pts][3][3] are host arrays; obs_pt[n_obs] indexes them.  Observations (raw pixels) are host arrays or,
 * with obs_on_device, device pointers (obs_cam, obs_key, obs_pt, obs_px).  A group is the rows of one obs_key: one pose
 * of one camera (key = camera, or (camera, frame)), k rows key-sorted and in caller order within a key, positions 0..k-1.
 *   1. rows from more than one camera: status 6.  2. k < 4: status 1.
 *   3. a row whose point is not finite is unusable: it scores tau^2, is in no sample's solution set, never an inlier.
 *   4. candidate samples, T = C(k, 3): every triple i < j < l in lexicographic order when T <= max_samples; else sample
 *      m = 0..max_samples-1 draws positions splitmix64(m 2^32 + t) mod k, t = 0, 1, ... (exact unsigned 64-bit;
 *      splitmix64(x) = the standard finaliser of x + 0x9e3779b97f4a7c15), keeps the first three distinct, sorted, and
 *      gives up after 16 draws.  No random state.
 *   5. hypotheses of a sample of three usable rows: the Lambda Twist P3P solutions (Persson & Nordberg, ECCV 2018; up
 *      to 4, in the solver's order) on the bearings of the float32-rounded undistorted normalised coordinates; a
 *      solution that is not finite or puts one of its three points at Xc.z <= 0 is none.  With use_prior the pose of
 *      the group's camera in cam_x is one more hypothesis, ranked before every sample.
 *   6. score (MSAC): sum over all k rows of min(e_r^2, tau^2), e_r = |pi(X_r; R, t, intrinsics) - u_r| in raw pixels with
 *      the engine's projection and the hypothesis's R; a row with Xc.z <= 0, a non-finite e_r or an unusable point adds
 *      tau^2.  The lowest score wins, ties to the lowest (prior, sample m, solution index).
 *   7. consensus set: the usable rows with Xc.z > 0 and e_r^2 <= tau^2 at the winner.  No hypothesis, or fewer than
 *      min_inliers such rows: status 5 (pose, cov, rmse NaN, n_inliers 0, no row inlier).
 *   8. Levenberg-Marquardt over q = (r, t) on the consensus rows (intrinsics fixed), from the winner's R as a rotation
 *      vector with theta in [0, pi] (cv2.Rodrigues): H = sum J^T J, g = sum J^T r (pixels, J = d pi / d q); solve
 *      (H + lambda diag H) d = -g, lambda0 = 1e-3; accept when the cost drops (lambda / 10) else lambda * 10; q += d;
 *      stop when |d| <= xtol (|q| + xtol) or after max_iter steps.
 *   9. cov = pixel_sigma^2 H^-1 + H^-1 M H^-1, M = sum_p G_p Sigma_p G_p^T, G_p = sum over the consensus rows of point p
 *      of J_q^T J_X (6 x 3, pixels), Sigma_p = pts_cov[p] (without pts_cov the first term alone; a NaN Sigma_p in the
 *      consensus set makes cov NaN).  It assumes the points are independent of each other and of the group's own
 *      observations and uses only each point's marginal: triangulate them without the resected camera's rows.
 *  10. status, first match wins: 6;  1;  5;  2 H not positive definite at the start or at the solution (a Cholesky
 *      pivot <= 1e-12 of the Jacobi-scaled D^-1/2 H D^-1/2; pose = the hypothesis, cov NaN);  3 max_iter reached;  4 a
 *      consensus row has Xc.z <= 0 at q*;  0 none.
 * Arguments: threshold_px tau finite > 0, min_inliers >= 4, 1 <= max_samples <= 4096, max_iter >= 1, finite
 * pixel_sigma >= 0 and xtol >= 0; obs_pt in [0, n_pts).
 * Outputs per group in ascending key order (host, room for max_groups): cam (the camera slot), pose[6] = (r, t) in x's
 * camera layout, cov[36] (nullable), rmse_px over the consensus rows, count, n_inliers, rep_row, status; inlier[n_obs]
 * (caller order).  No floating-point atomics: repeated calls return bit-identical outputs. */
int cb_resect_robust(int32_t n_cams, const int32_t* cam_flags, const double* cam_const, const double* cam_x,
                     int32_t n_pts, const double* pts_xyz, const double* pts_cov, int64_t n_obs, const int32_t* obs_cam,
                     const int64_t* obs_key, const int32_t* obs_pt, const double* obs_px, int obs_on_device,
                     double threshold_px, int32_t min_inliers, int32_t max_samples, int32_t use_prior,
                     double pixel_sigma, int32_t max_iter, double xtol, int32_t max_groups, int32_t* n_groups_out,
                     int32_t* cam_out, double* pose_out, double* cov_out, double* rmse_px_out, int32_t* count_out,
                     int32_t* n_inliers_out, int32_t* rep_row_out, int32_t* status_out, uint8_t* inlier_out,
                     CbResectStats* stats, int device, void* stream);

typedef struct CbRigidStats {
  double group_ms;      /* upload + validation + undistortion + radix sort + group boundaries */
  double points_ms;     /* the (group, point) sort, the point consensus, the qualified points and the prior lookup */
  double consensus_ms;  /* Horn hypotheses, MSAC scoring, selection and the compaction of the consensus rows */
  double refine_ms;     /* the Levenberg-Marquardt kernel on the consensus rows */
  double cov_ms;        /* the camera sort, the camera-term and covariance kernels (0 without cov_out) */
  double total_ms;
  int32_t kernel_launches;
  int32_t pad_;
} CbRigidStats;

/* Robust pose of a rigid body seen by a calibrated rig (DESIGN.md section 4.14): X_w = R(r) M + t for the body's own
 * model points M.  Cameras in the bundle-adjustment layout as cb_triangulate_refine, cam_cov (nullable) the
 * n_camera_params^2 camera covariance (BAProblem.covariance's cameras).  model_xyz[n_model][3] is a host array in the
 * body's frame; obs_pt[n_obs] (the model point of a row) indexes it.  Observations (raw pixels) are host arrays or, with
 * obs_on_device, device pointers (obs_cam, obs_key, obs_pt, obs_px).  A group is the rows of one obs_key: one body at
 * one moment (key = frame, or (body, frame); several bodies share the model table through disjoint point ranges), k rows
 * key-sorted and in caller order within a key.  Optional priors: prior_key[n_prior] (strictly ascending) and
 * prior_pose[n_prior][6] (finite), host arrays; a group's prior is the entry of its key.
 *   1. k < 4: status 1.  A row whose model point is not finite is unusable: it scores tau^2 and is never an inlier.
 *   2. point hypotheses: each model point p with rows in the group gets cb_triangulate_robust's consensus on those rows
 *      (the same tau, min_inliers 2, max_pairs): the DLT point of the best view pair, or none (a point whose rows all
 *      come from one camera, or whose views do not agree; its rows still take part in scoring and refinement).  The
 *      qualified points are the points with a point hypothesis, positions 0..n_q-1 in ascending model index.
 *   3. samples, T = C(n_q, 3): every triple in lexicographic order when T <= max_samples, else cb_resect_robust's
 *      splitmix64 draw.
 *   4. pose hypothesis of a sample: Horn's closed-form absolute orientation (JOSA A 4(4), 1987) without scale of the
 *      three model points against their point hypotheses: q the eigenvector of the largest eigenvalue of Horn's 4 x 4 N,
 *      R = R(q), t = mean(X) - R mean(M).  None when the model triangle is degenerate,
 *      |(M_j - M_i) x (M_l - M_i)| <= 1e-9 |M_j - M_i| |M_l - M_i|, or R or t is not finite.  The group's prior, if it
 *      has one, is slot 0; sample m is slot 1 + m.
 *   3-4 with gp3p_samples > 0 (1..4096), in a group with k >= 4 rows and n_q < 3 (every other group as above):
 *      samples of three row positions 0..k-1, every triple in lexicographic order when C(k, 3) <= gp3p_samples, else
 *      section 4.9's splitmix64 draw of gp3p_samples.  A sample gives no hypothesis when two of its rows share a model
 *      point, a row is unusable (model point not finite, or undistorted coordinate not finite or the fisheye failure
 *      sentinel), the model triangle is degenerate or the rays are parallel; else oracle/gp3p.py's gp3p on the rows'
 *      camera centres c_i = -R_i^T t_i, unit rays d_i = R_i^T (x_i, y_i, 1) / |.| of the undistorted normalised
 *      coordinates and model points: the real roots of the octic in the first depth, each back-substituted, polished by
 *      Newton on the three distance equations and posed by Horn.  Hypothesis c of sample m is slot 1 + 8 m + c.
 *      Constants: rays parallel when det(sum (I - d_i d_i^T)) <= 1e-12; Delta_j >= -1e-8 (1 + p_j^2) clamped to 0,
 *      below it no hypothesis; roots with |u_1| <= 1e9; at most 3 Newton steps.
 *   5. score (MSAC): sum over all k rows of min(e_r^2, tau^2), e_r = |pi(R M_r + t; c_r) - u_r| in raw pixels with the
 *      engine's projection and the row's own camera; a row behind its camera, with a non-finite error or an unusable
 *      point adds tau^2.  The lowest score wins, the lowest slot on a tie.
 *   6. consensus set: the usable rows in front of their camera with e_r^2 <= tau^2 at the winner.  No hypothesis, or
 *      fewer than min_inliers such rows: status 5 (pose, cov, rmse NaN, n_inliers 0, no row inlier).  One round.
 *   7. Levenberg-Marquardt over q = (r, t) on the consensus rows from the winner's R as a rotation vector with theta in
 *      [0, pi]: cb_resect_robust's loop (lambda0 1e-3, / 10, * 10, |d| <= xtol (|q| + xtol), max_iter) with
 *      J_q = J_X [d(R(r) M)/dr | I] per row.
 *   8. cov = pixel_sigma^2 H^-1 + H^-1 G cam_cov G^T H^-1, G = sum over the consensus rows of J_q^T J_c (6 x
 *      n_camera_params, pixels); without cam_cov the first term alone.  It assumes the body's observations are
 *      independent of those that calibrated the rig, and takes the model as exact.
 *   9. status, first match wins: 1;  5;  2 H not positive definite at the start or at the solution (a Cholesky pivot
 *      <= 1e-12 of the Jacobi-scaled D^-1/2 H D^-1/2, e.g. every consensus row on one marker; pose = the hypothesis, cov
 *      NaN);  3 max_iter reached;  4 a consensus row is behind its camera at q*;  0 none.
 * Arguments: threshold_px tau finite > 0, min_inliers >= 4, max_pairs >= 1, 1 <= max_samples <= 4096, max_iter >= 1,
 * finite pixel_sigma >= 0 and xtol >= 0; obs_pt in [0, n_model).
 * Outputs per group in ascending key order (host, room for max_groups): pose[6] = (r, t), cov[36] (nullable), rmse_px
 * over the consensus rows, count, n_inliers, n_points (qualified points), rep_row, status; inlier[n_obs] (caller
 * order).  No floating-point atomics: repeated calls return bit-identical outputs. */
int cb_rigid_pose_robust(int32_t n_cams, const int32_t* cam_flags, const double* cam_const, const double* cam_x,
                         const double* cam_cov, int32_t n_model, const double* model_xyz, int64_t n_obs,
                         const int32_t* obs_cam, const int64_t* obs_key, const int32_t* obs_pt, const double* obs_px,
                         int obs_on_device, double threshold_px, int32_t min_inliers, int32_t max_pairs,
                         int32_t max_samples, int32_t n_prior, const int64_t* prior_key, const double* prior_pose,
                         double pixel_sigma, int32_t max_iter, double xtol, int32_t max_groups, int32_t* n_groups_out,
                         double* pose_out, double* cov_out, double* rmse_px_out, int32_t* count_out,
                         int32_t* n_inliers_out, int32_t* n_points_out, int32_t* rep_row_out, int32_t* status_out,
                         uint8_t* inlier_out, CbRigidStats* stats, int device, void* stream);

/* cb_rigid_pose_robust with gP3P hypotheses (steps 3-4 with gp3p_samples above): gp3p_samples 0 is
 * cb_rigid_pose_robust itself, 1..4096 the most gP3P samples a group draws, anything else CB_E_INVALID.  Groups with
 * three or more qualified points give the outputs of gp3p_samples = 0 bit for bit.
 *   9 in a group that gP3P reaches, with status 6 added: a group whose consensus winner is a gP3P hypothesis (slot >= 1
 *      in a group with n_q < 3) and whose consensus rows hold fewer than four distinct model points is ambiguous,
 *      status 6: refinement runs as for status 0, pose and rmse are reported, cov is NaN.  First match wins: 1, 5, 6,
 *      2, 3, 4, 0.  Two triangulated markers leave the body free to turn about their axis; a third marker seen by one
 *      camera lies on a circle about that axis, which its ray can meet twice, and both poses fit every row.  A group
 *      won by its prior (slot 0) keeps step 9's statuses: the prior chooses the branch. */
int cb_rigid_pose_robust_gp3p(int32_t n_cams, const int32_t* cam_flags, const double* cam_const, const double* cam_x,
                              const double* cam_cov, int32_t n_model, const double* model_xyz, int64_t n_obs,
                              const int32_t* obs_cam, const int64_t* obs_key, const int32_t* obs_pt,
                              const double* obs_px, int obs_on_device, double threshold_px, int32_t min_inliers,
                              int32_t max_pairs, int32_t max_samples, int32_t gp3p_samples, int32_t n_prior,
                              const int64_t* prior_key, const double* prior_pose, double pixel_sigma, int32_t max_iter,
                              double xtol, int32_t max_groups, int32_t* n_groups_out, double* pose_out,
                              double* cov_out, double* rmse_px_out, int32_t* count_out, int32_t* n_inliers_out,
                              int32_t* n_points_out, int32_t* rep_row_out, int32_t* status_out, uint8_t* inlier_out,
                              CbRigidStats* stats, int device, void* stream);

typedef struct CbRigidModelStats {
  double group_ms;  /* upload + validation + grouping by key, the frame table and the per-body frame lists */
  double solve_ms;  /* the Levenberg-Marquardt cluster kernel */
  double cov_ms;    /* the covariance cluster kernel (status 2 / 4, rmse, cov) */
  double total_ms;
  int32_t kernel_launches;
  int32_t pad_;
} CbRigidModelStats;

/* Refinement of rigid-body marker layouts from tracked frames (DESIGN.md section 4.15): one Levenberg-Marquardt per body
 * over its layout and every frame pose, with the frames eliminated, and the layout's covariance.  Cameras in the
 * bundle-adjustment layout as cb_triangulate_refine, cam_cov (nullable) the n_camera_params^2 camera covariance
 * (BAProblem.covariance's cameras).  model_xyz[n_model][3] (host) is the start layout M0;
 * body_start[n_bodies + 1] (host, ascending from 0 to n_model): model points body_start[b] .. body_start[b+1]-1 are body
 * b, with 3 <= K <= 32 markers.  Observations (raw pixels) are host arrays or, with obs_on_device, device pointers
 * (obs_cam, obs_key, obs_pt, obs_px); rows with equal obs_key are one frame of one body (all its rows in one body's
 * range).  start_key[n_start] (strictly ascending) and start_pose[n_start][6] (finite) are the start pose (r, t) per key,
 * host arrays; X_w = R(r_f) M_k + t_f.
 *   1. frames: a frame is used when it has a start pose, at least 4 rows and at least 3 distinct markers among them;
 *      otherwise its status is 1 and its rows take no part.  A body's status is 1 when it has no used frame, or when
 *      one of its markers has no row in a used frame; its layout is then the start, its cov NaN and its frames' poses
 *      the start.
 *   2. residuals over body b's rows in used frames: the projection of R(r_f) M_k + t_f with the row's own camera (the
 *      engine's projection), minus the raw pixel, in pixels.
 *   3. gauge: inner constraints on the start layout, sum_k (M_k - M0_k) = 0 and
 *      sum_k (M0_k - mean M0) x (M_k - M0_k) = 0: steps dM lie in null(C^T), C (3K x 6) = [I_3 | [M0_k - mean M0]x] per
 *      marker.  The result keeps the start's centroid and has no net rotation against it.
 *   4. step: H_MM + lam diag(H_MM) and H_ff + lam diag(H_ff) per frame; the frames eliminated into
 *      S_lam = H_MM,lam - sum_f H_Mf H_ff,lam^-1 H_fM; dM = -N (N^T S_lam N)^-1 N^T b for an orthonormal basis N of
 *      null(C^T); each frame's step by back-substitution.  lambda0 1e-3, / 10 on a lower cost, * 10 otherwise; stop
 *      when |d| <= xtol (|x| + xtol), d and x over the layout and every frame pose of the body; max_iter steps at most;
 *      a damped block that is not positive definite is a rejected step.
 *   5. covariance at the solution (lam = 0), P = N (N^T S N)^-1 N^T, (3K)^2 per body:
 *      cov = pixel_sigma^2 P + P G Sigma_c G^T P, G = sum_f (G_M,f - H_Mf H_ff^-1 G_f) the Schur-reduced cross term to
 *      the camera parameters, G_.,f = sum over the frame's rows of J_.^T J_c in pixels; without cam_cov the first term
 *      alone.  Cross-body correlation through the cameras is not given.
 *   6. status per body, first match wins: 1;  2 N^T S N not positive definite at the start or at the solution (a
 *      Cholesky pivot <= 1e-12 of its Jacobi scaling; layout and poses are the start, cov and rmse NaN);  3 max_iter
 *      reached;  4 a row behind its camera at the solution;  0 none.
 * Arguments: finite pixel_sigma >= 0 and xtol >= 0, max_iter >= 1, obs_cam in [0, n_cams), obs_key >= 0, obs_pt in
 * [0, n_model); CB_E_INVALID otherwise, and for a frame whose rows span two bodies.  cam_cov is read only with cov_out.
 * Outputs: model_out[n_model][3]; cov_out (nullable) the per-body (3K)^2 blocks end to end in body order; per body
 * status, iterations, rmse_px (over its rows in used frames), n_frames (used frames), n_rows; per frame in ascending key
 * order (room for max_frames): key, pose[6], rmse_px (NaN for a frame that takes no part), count (every row of the key),
 * status (1 for a frame that takes no part or whose body has status 1, else its body's status).  No floating-point
 * atomics: repeated calls return bit-identical outputs. */
int cb_rigid_model_refine(int32_t n_cams, const int32_t* cam_flags, const double* cam_const, const double* cam_x,
                          const double* cam_cov, int32_t n_model, const double* model_xyz, int32_t n_bodies, const int32_t* body_start,
                          int64_t n_obs, const int32_t* obs_cam, const int64_t* obs_key, const int32_t* obs_pt,
                          const double* obs_px, int obs_on_device, int32_t n_start, const int64_t* start_key,
                          const double* start_pose, double pixel_sigma, int32_t max_iter, double xtol,
                          int32_t max_frames, int32_t* n_frames_out, double* model_out, double* cov_out,
                          int32_t* status_out, int32_t* iterations_out, double* rmse_px_out, int32_t* body_frames_out,
                          int32_t* body_rows_out, int64_t* key_out, double* pose_out, double* frame_rmse_px_out,
                          int32_t* count_out, int32_t* frame_status_out, CbRigidModelStats* stats, int device,
                          void* stream);

typedef struct CbRelPoseStats {
  double group_ms;      /* upload + undistortion + grouping by key, the correspondence slots and their sort by pair */
  double consensus_ms;  /* five-point hypotheses, MSAC scoring, selection and the compaction of the consensus sets */
  double refine_ms;     /* the Levenberg-Marquardt kernel on the consensus sets */
  double cov_ms;        /* the covariance kernel (0 without cov_out) */
  double total_ms;
  int32_t kernel_launches;
  int32_t pad_;
} CbRelPoseStats;

/* Robust relative pose of every camera pair from 2-D correspondences alone (DESIGN.md section 4.11).  Cameras in the
 * bundle-adjustment layout as cb_triangulate_refine; only the intrinsics are read (s, k1, k2 of a free-intrinsics
 * block), the extrinsics are ignored.  Observations (raw pixels) are host arrays or, with obs_on_device, device
 * pointers (obs_cam, obs_key, obs_px); rows with equal obs_key (int64 >= 0) are one world point.  Pixels are undistorted
 * as cv2.undistortPoints does (float32 rounding); a row whose coordinates are not finite, or a fisheye row at OpenCV's
 * (-1e6, -1e6) failure sentinel, is unusable.
 *   0. correspondences: rows i < j of one key (key-sorted, caller order within a key) from different cameras are one
 *      correspondence of the pair (a, b), a < b (camera slots), its a-row camera a's.  A pair's correspondences are
 *      ordered by key, then (i, j), k of them at positions 0..k-1 (cb_stereo_rmse's slot order).  Every pair with a
 *      correspondence is reported, in ascending (a, b).  More than 2^31 - 1 row pairs within keys (the slots before
 *      same-camera pairs are dropped; sum over keys of n (n - 1) / 2): CB_E_INVALID.
 *   1. k < min_inliers: status 1.
 *   2. candidate samples, T = C(k, 5): every 5-subset in lexicographic order when T <= max_samples; else sample m draws
 *      splitmix64(m 2^32 + t) mod k, t = 0, 1, ..., keeps the first five distinct, sorted, gives up after 16 draws.
 *   3. hypotheses of a sample of five usable correspondences: Nister's five-point solver on the normalised coordinates
 *      (null space of the 5 x 9 epipolar system, the 10 x 20 cubic constraints, Gauss-Jordan, every real root of the
 *      degree-10 polynomial by Sturm bisection and a Newton polish), up to 10 E.  Each E gives (R1, t), (R1, -t), (R2, t),
 *      (R2, -t), |t| = 1; the first that puts the five points at positive depth in both cameras (least squares of
 *      [R x_a, -x_b] (la, lb)^T = -t, la, lb > 0) is the hypothesis, slot 10 m + c.
 *   4. score (MSAC): sum over all k correspondences of min(e^2, tau^2), e the Sampson distance in undistorted pixels,
 *      e^2 = (x_b^T E x_a)^2 / ((E x_a)_1^2 / fx_b^2 + (E x_a)_2^2 / fy_b^2 + (E^T x_b)_1^2 / fx_a^2 + (E^T x_b)_2^2 / fy_a^2),
 *      E = [t]x R (cv2.sampsonDistance with F = K_b^-T E K_a^-1); an unusable correspondence or a non-finite e adds
 *      tau^2.  The lowest score wins, the lowest slot on a tie.
 *   5. consensus set: the usable correspondences with e^2 <= tau^2 and positive depths at the winner.  No hypothesis or
 *      fewer than min_inliers: status 5 (pose, cov, rmse, parallax NaN; n_inliers 0).
 *   6. Levenberg-Marquardt over q = (r, alpha, beta) on the consensus set: r the winner's R as a rotation vector
 *      (theta in [0, pi]), t = normalize(t0 + alpha u1 + beta u2), u1, u2 columns 1 and 2 of the Householder reflector
 *      taking t0 to -+e3 (fixed at the start); residual the signed Sampson distance (x_b^T E x_a) / sqrt(den) in pixels;
 *      cb_resect_robust's loop (lambda0 1e-3, / 10, * 10, |d| <= xtol (|q| + xtol), max_iter).
 *   7. covariance at q*: the chart re-based at t*, cov5 = pixel_sigma^2 H^-1 over (r, du), returned as the 6 x 6
 *      J cov5 J^T over (r, t) with J = diag(I3, [u1 u2](t*)) (rank 5).
 *   8. status, first match wins: 1;  5;  2 H not positive definite at the start or at the solution (a Cholesky pivot
 *      <= 1e-12 of the Jacobi-scaled H; pose = the hypothesis, cov NaN);  3 max_iter reached;  4 a consensus
 *      correspondence has a non-positive depth at q*;  0 none.
 * Arguments: threshold_px tau finite > 0, min_inliers >= 5, 1 <= max_samples <= 4096, max_iter >= 1, finite
 * pixel_sigma >= 0 and xtol >= 0; obs_cam in [0, n_cams), obs_key >= 0.
 * Outputs per pair (host, room for max_pairs): cam_a, cam_b, pose[6] = (r, t) with X_b = R X_a + t and |t| = 1,
 * cov[36] (nullable), rmse_px (Sampson, consensus set), parallax_deg (mean angle between R x_a and x_b over the consensus
 * set), count, n_inliers, status.  No floating-point atomics: repeated calls return bit-identical outputs. */
int cb_relative_pose_robust(int32_t n_cams, const int32_t* cam_flags, const double* cam_const, const double* cam_x,
                            int64_t n_obs, const int32_t* obs_cam, const int64_t* obs_key, const double* obs_px,
                            int obs_on_device, double threshold_px, int32_t min_inliers, int32_t max_samples,
                            double pixel_sigma, int32_t max_iter, double xtol, int32_t max_pairs, int32_t* n_pairs_out,
                            int32_t* cam_a_out, int32_t* cam_b_out, double* pose_out, double* cov_out,
                            double* rmse_px_out, double* parallax_deg_out, int32_t* count_out, int32_t* n_inliers_out,
                            int32_t* status_out, CbRelPoseStats* stats, int device, void* stream);

typedef struct CbIntrinsicsStats {
  double group_ms;  /* upload + validation + radix sort + view boundaries */
  double start_ms;  /* view statuses, homographies, Zhang's start, undistortion, IPPE poses */
  double lm_ms;     /* the Levenberg-Marquardt kernel */
  double cov_ms;    /* the covariance kernel */
  double total_ms;
  int32_t iterations;  /* the most LM steps any camera took */
  int32_t kernel_launches;
} CbIntrinsicsStats;

/* Per-camera words of cb_calibrate_intrinsics.  cam_flags is in the CB_CAM_* namespace of every other call:
 * CB_CAM_FISHEYE (a fisheye lens: cv2.fisheye.calibrate is a different model and algorithm) is refused with
 * CB_E_UNSUPPORTED, as is CB_INTR_FIX_ASPECT_RATIO and any bit not named here; CB_CAM_FREE_INTRINSICS is accepted and
 * changes nothing (every parameter not in cam_fixed is free); CB_INTR_USE_GUESS starts the camera from guess[c].
 * cam_fixed (nullable: nothing fixed): bit k (k = 0..8) keeps parameter k of (fx, fy, cx, cy, k1, k2, p1, p2, k3) at its
 * start value; other bits are CB_E_INVALID. */
#define CB_INTR_USE_GUESS 0x100
#define CB_INTR_FIX_ASPECT_RATIO 0x200
#define CB_INTR_FIX_ALL 0x1ff

/* Intrinsic calibration of every camera from planar-board views: pinhole + Brown-Conrady (k1 k2 p1 p2 k3), the model
 * and the optimum of cv2.calibrateCamera, with OpenCV's standard deviations (DESIGN.md section 4.10).
 * Inputs: image_size[n_cams][2] (w, h), cam_flags[n_cams], cam_fixed[n_cams] (nullable), guess (nullable unless a
 * camera sets CB_INTR_USE_GUESS)
 * [n_cams][9]; rows obs_cam, obs_key (int64 >= 0: rows with equal key are one view), obs_obj[n][3] board coordinates,
 * obs_px[n][2] raw pixels (float64, full precision) -- host arrays or, with obs_on_device, device pointers.
 *   1. views, ascending key order, rows in caller order within a key; view status, first match wins: 6 rows from more
 *      than one camera; 1 fewer than min_points rows; 2 non-planar (z spread >= 1e-6, or a non-finite z); 5 degenerate
 *      Harker-O'Leary homography (board points collinear, ...) or a non-finite start pose; else 0.
 *   2. start: the guess, or Zhang's closed form as cv2.initIntrinsicParams2D (no aspect ratio): principal point
 *      ((w-1)/2, (h-1)/2), distortion 0, a = 1/fx^2 and b = 1/fy^2 by least squares from the two constraints of every
 *      view with a homography (camera-major sums in view order); a or b <= 0 or not finite: camera status 2.  Each
 *      view's start pose is cb_pnp_ippe's IPPE on its board points and its pixels undistorted with the start.
 *   3. fixed parameters keep their start value and leave the system (no zero step).
 *   4. Levenberg-Marquardt over the free intrinsics theta and every used view's q = (r, t), residuals in pixels
 *      pi(X; theta, q) - u, unweighted: U, W_v, V_v, g; (H + lambda diag H) d = -g through S = U_lambda - sum_v W_v
 *      V_v,lambda^-1 W_v^T on the free subset, back-substituted per view; lambda0 = 1e-3, a lower cost is accepted with
 *      lambda / 10, else lambda * 10; r += dr additively; stop when |d| <= xtol (|(theta_free, q)| + xtol) or after
 *      max_iter steps (status 4).  A step whose damped system is not positive definite is rejected without the
 *      stopping test.
 *   5. covariance at the solution (lambda = 0): sigma^2 = SSE / (2N - p), N rows, p = free intrinsics + 6 used views;
 *      cov_theta = sigma^2 S^-1 (fixed rows / columns 0); per view cov_q = sigma^2 (V^-1 + V^-1 W^T S^-1 W V^-1).
 *      S not positive definite (a Cholesky pivot <= 1e-12 of the Jacobi-scaled S): status 3, theta the last iterate,
 *      std / cov NaN.
 * A camera with fewer than min_views usable views is status 1.  Camera status, first match wins: 1, 2, 3, 4, else 0.
 * Outputs per camera: params[9] (NaN without a start), std[9], cov[81] (nullable), rms = sqrt(SSE / N) (cv2's return
 * value), sigma^2, used views, rows, iterations, status.  Per view in key order (room for max_views): camera (of its
 * first row), pose[6] = (r, t), std[6], rmse_px (cv2's perViewErrors), count, rep_row (first caller row), status; pose,
 * std and rmse are NaN for a view that was not solved.
 * Arguments: min_points >= 4, min_views >= 2, max_iter >= 1, finite xtol >= 0, image sizes > 0, a guess finite with
 * fx, fy > 0.  No floating-point atomics: repeated calls return bit-identical outputs. */
int cb_calibrate_intrinsics(int32_t n_cams, const int32_t* image_size, const int32_t* cam_flags,
                            const int32_t* cam_fixed, const double* guess,
                            int64_t n_obs, const int32_t* obs_cam, const int64_t* obs_key, const double* obs_obj,
                            const double* obs_px, int obs_on_device, int32_t min_points, int32_t min_views,
                            int32_t max_iter, double xtol, int32_t max_views, int32_t* n_views_out, double* params_out,
                            double* std_out, double* cov_out, double* rms_out, double* sigma2_out,
                            int32_t* used_views_out, int32_t* rows_out, int32_t* iterations_out, int32_t* status_out,
                            int32_t* view_cam_out, double* view_pose_out, double* view_std_out, double* view_rmse_out,
                            int32_t* view_count_out, int32_t* view_rep_out, int32_t* view_status_out,
                            CbIntrinsicsStats* stats, int device, void* stream);

/* Optional NCCL transport owned by the engine (no host callback per all-reduce).  NCCL is resolved at run time from
 * the libnccl the process already has loaded (PyTorch's).  Rank 0 calls cb_nccl_unique_id and distributes the 128
 * bytes (e.g. torch.distributed.broadcast); every rank then calls cb_nccl_comm_create (collective). */
int cb_nccl_unique_id(char id_out[128]);
int cb_nccl_comm_create(const char id[128], int rank, int world_size, int device, void** comm_out);
int cb_nccl_comm_destroy(void* comm);

/* Peer-memory transport (one node, NVLink/NVSwitch, one process per GPU).  Every rank creates its symmetric buffer
 * (capacity_doubles >= (n_cams*P)^2 + 3*n_cams*P + 65 for the problems it will solve, P = 9 with free intrinsics
 * else 6), the 64-byte CUDA IPC handles are exchanged by any means, then every rank connects with all handles in
 * rank order.  During cb_ba_solve the reduced camera system is then summed by schur_finalize_peer_kernel reading
 * the peers' buffers directly; no NCCL call is made.  world_size <= 16.  Destroy only after every rank is done. */
typedef struct CbPeerGroup CbPeerGroup;
int cb_peer_create(int rank, int world_size, int device, int64_t capacity_doubles, CbPeerGroup** out,
                   char handle_out[64]);
int cb_peer_connect(CbPeerGroup* group, const char* handles /* world_size x 64 bytes */);
int cb_peer_destroy(CbPeerGroup* group);

/* Number of kernel launches issued by this library in the calling process so far. */
int64_t cb_ba_launch_count(void);


/* ------------------------------------------------------------------------------------------------------------------
 * Extrinsic bootstrap (what produces bundle adjustment's start vector; SURVEY.md 8(f) rank 1).
 *
 * cb_pnp_ippe == compute_camera_to_object_poses_pnp (reference core/bootstrap_pose/pose_network_builder.py:211-330):
 *   obs_px are raw pixels of camera obs_cam (undistorted on the device with float32 rounding exactly as
 *   CameraData.undistort_points does, cameras/camera_array.py:135-174), obs_obj the object-frame coordinates (n_obs x 3,
 *   NaN z = 0), obs_key >= 0 packs (camera, sync_index, object) -- rows with equal key form one PnP group, groups come
 *   back in ascending key order (== the reference's groupby order when the key is packed camera-major).  Per group:
 *   R (3x3 row-major) and t of the object in the camera frame (cv2.solvePnP(SOLVEPNP_IPPE) + cv2.Rodrigues), the
 *   reprojection RMSE in the normalised plane (:317-318), status (0 ok, 1 fewer than min_points rows, 2 non-planar
 *   target -- the reference switches to SQPNP there, which this build does not implement --, 3 degenerate), row count and
 *   one representative caller row.  All pointers host.
 *
 * cb_stereo_rmse == calculate_stereo_rmse_for_pair for every pair at once (:638-685, with the common observations of
 *   _precompute_common_observations :576-603): pair p = cameras (pair_a[p] < pair_b[p]) with pose pair_Rt[p] = [R (9) | t (3)]
 *   (camera a at the origin).  obs_key >= 0 packs (sync_index, object, keypoint).  Outputs per pair: rmse (NaN when the
 *   pair has fewer than min_common common observations, the reference returns None there) and the number of common
 *   observations.
 * ------------------------------------------------------------------------------------------------------------------ */
int cb_pnp_ippe(int32_t n_cams, const int32_t* cam_fisheye, const double* cam_k, const double* cam_dist, int64_t n_obs,
                const int32_t* obs_cam, const int64_t* obs_key, const double* obs_px, const double* obs_obj,
                int32_t min_points, int32_t max_groups, int32_t* n_groups_out, double* R_out, double* t_out,
                double* rmse_out, int32_t* status_out, int32_t* count_out, int32_t* rep_row_out, CbTriStats* stats,
                int device, void* stream);

int cb_stereo_rmse(int32_t n_cams, const int32_t* cam_fisheye, const double* cam_k, const double* cam_dist,
                   int32_t n_pairs, const int32_t* pair_a, const int32_t* pair_b, const double* pair_Rt, int64_t n_obs,
                   const int32_t* obs_cam, const int64_t* obs_key, const double* obs_px, int32_t min_common,
                   double* rmse_out, int64_t* count_out, CbTriStats* stats, int device, void* stream);

/* cb_relative_pose_network == compute_relative_poses (pose_network_builder.py:484-531) -> reject_outliers (:331-413) ->
 *   aggregate_poses (:533-573, quaternion_average :416-438) for every camera pair in one device pass; the relative poses
 *   never leave the device.
 *   Input: the PnP poses (camera <- object) of the cameras the array does not ignore, sorted by (sync_index, object_id,
 *   camera id): group g has camera id cam_id[g], position cam_pos[g] in the reference's camera dict, pose R[9g..], t[3g..]
 *   (NaN poses allowed: cv2's degenerate groups); frame_start[f] .. frame_start[f+1] are the groups of one (sync_index,
 *   object_id).  Every combination (i < j) of a frame's groups is one candidate relative pose; the reference forms it only if
 *   cam_pos[i] < cam_pos[j] (its `combinations(dict order) if a < b` quirk).
 *   rot_mult / tr_mult: IQR multipliers of the rotation-angle / translation-magnitude rules (1.5 in the reference).
 *   Output, camera pairs in ascending (a, b), at most max_pairs: ids, aggregated R (9) and t (3), number of samples kept.
 *   Optional (n_rel = sum over frames of s(s-1)/2, frame-major, np.triu_indices order inside a frame): rel_valid[m] = 1 when
 *   the combination was formed, rel_keep[m] = 1 when it passed the NaN filter and the IQR rule. */
int cb_relative_pose_network(int32_t n_groups, int32_t n_frames, const int32_t* frame_start, const int32_t* cam_id,
                             const int32_t* cam_pos, const double* R, const double* t, double rot_mult, double tr_mult,
                             int32_t max_pairs, int32_t* n_pairs_out, int32_t* pair_a, int32_t* pair_b, double* R_out,
                             double* t_out, int64_t* count_out, int64_t n_rel, uint8_t* rel_valid, uint8_t* rel_keep,
                             CbTriStats* stats, int device, void* stream);


/* Host-side shard selection of a sharded solve (distributed.shard_points): the observations whose point index lies in
 * [pt_lo, pt_hi), in the caller's order, point index made local (pt - pt_lo).  All host threads; no device work.
 * With every output pointer null it only counts (*n_sel_out).  sel_index = positions in the caller's list. */
int cb_shard_select(int64_t n_obs, const int32_t* obs_cam, const int32_t* obs_pt, const double* obs_xy, int32_t pt_lo,
                    int32_t pt_hi, int64_t capacity, int64_t* n_sel_out, int64_t* sel_index, int32_t* cam_out,
                    int32_t* pt_out, double* xy_out, int32_t n_threads);

/* ------------------------------------------------------------------------------------------------------------------
 * Numeric CSV tables at the boundary of the path (SURVEY.md 8(f) rank 4): xy_<TRACKER>.csv / xyz_<TRACKER>.csv as written
 * by ImagePoints.to_csv / WorldPoints.to_csv (reference core/point_data.py:358-373, 662-677 through
 * persistence._safe_write_csv, persistence.py:27-41: `to_csv(index=False, float_format="%.6f")`, temp file + fsync +
 * rename) and read by pd.read_csv.  Byte-identical files, all host cores; no device work.
 *   col_kind[c]: 0 = int64 column, 1 = float64 column (NaN -> empty field).  header: the column names joined by ','.
 *   cb_csv_parse_numeric: out is column-major float64 [n_cols][n_rows] (sizes from cb_csv_scan); col_all_int / col_has_empty
 *   let the caller rebuild pandas' dtypes (int64 iff every field is an integer literal).
 * ------------------------------------------------------------------------------------------------------------------ */
int cb_csv_write_numeric(const char* path, const char* header, int64_t n_rows, int32_t n_cols, const int32_t* col_kind,
                         const void* const* col_data, int32_t n_threads);
int cb_csv_scan(const char* path, int64_t* n_rows, int32_t* n_cols);
int cb_csv_parse_numeric(const char* path, int64_t n_rows, int32_t n_cols, double* out, int32_t* col_all_int,
                         int32_t* col_has_empty, int32_t n_threads);

#ifdef __cplusplus
}
#endif
#endif /* CALISCOPE_B200_H */
