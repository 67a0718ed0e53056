/*
 * gtsam_b200.h — C-ABI of the H100-native Gauss-Newton / Levenberg-Marquardt
 * inner loop (linearize + multifrontal Cholesky solve) that drops in behind
 * GTSAM's LevenbergMarquardtOptimizer / GaussNewtonOptimizer /
 * GaussianFactorGraph::optimize path.
 *
 * Plain C, plain pointers and sizes, opaque handles, int status codes.  No
 * torch, no GTSAM, no C++ types cross this boundary.  All file:line citations
 * are relative to the reference tree (borglab/gtsam @ 0ffe6c93).
 *
 * Conventions (identical to the reference):
 *  - all arithmetic FP64; tangent order for Pose3 is (omega, v), rotation first
 *    (gtsam/geometry/Pose3.cpp:169-208); perturbations are right-multiplied
 *    (gtsam/base/Lie.h:131-160);
 *  - a Pose3 value is 12 doubles: R row-major (9) then t (3);
 *  - variables are addressed by dense ids 0..nvars-1.  The GTSAM-side shim
 *    assigns ids in ascending Key order (the iteration order of
 *    gtsam::Values, gtsam/nonlinear/Values.h:74-79), so "sorted by id" ==
 *    "sorted by Key" (needed to reproduce gtsam/linear/Scatter.cpp:69-72);
 *  - `ordering[k]` is the id of the k-th eliminated variable (the contents of
 *    a gtsam::Ordering, gtsam/inference/Ordering.h:217-236).  It is an INPUT:
 *    COLAMD/METIS/Schur orderings are produced by the caller.
 */
#ifndef GTSAM_B200_H
#define GTSAM_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- status codes (replace the reference's C++ exceptions) --------------- */
enum {
  B200_OK = 0,
  B200_INDETERMINATE = 1,      /* gtsam::IndeterminantLinearSystemException,
                                  gtsam/linear/HessianFactor.cpp:476-483,
                                  gtsam/linear/linearAlgorithms-inst.h:99 */
  B200_UNSUPPORTED_FACTOR = 2, /* factor type outside the hot path          */
  B200_UNSUPPORTED_NOISE = 3,  /* Constrained noise models (need QR)         */
  B200_INVALID_ARGUMENT = 4,   /* std::invalid_argument / ValuesKeyDoesNotExist */
  B200_CUDA_ERROR = 5,
  B200_NCCL_ERROR = 6,
  B200_NO_DEVICE = 7           /* no CUDA device: there is NO CPU fallback   */
};

/* ---- variable (gtsam::Value) types --------------------------------------- */
enum {
  B200_VAR_POSE3 = 0,       /* gtsam::Pose3; storage 12 (R row-major, t); dim 6 */
  B200_VAR_POINT3 = 1,      /* gtsam::Point3; storage 3; dim 3                  */
  B200_VAR_CAM_BUNDLER = 2, /* PinholeCamera<Cal3Bundler>; storage 17 =
                               R(9) t(3) f k1 k2 u0 v0; dim 9 = pose(6)+f,k1,k2
                               (gtsam/geometry/PinholeCamera.h:199-205)         */
  B200_VAR_POSE2 = 3,       /* gtsam::Pose2; storage 3 = x y theta; dim 3, tangent order (x, y, theta);
                               retract / localCoordinates are the first-order chart the reference uses
                               unless GTSAM_SLOW_BUT_CORRECT_EXPMAP (gtsam/geometry/Pose2.cpp:99-122)  */
  B200_NUM_VAR_TYPES = 4
};

/* ---- factor types --------------------------------------------------------- */
enum {
  /* BetweenFactor<Pose3>, gtsam/slam/BetweenFactor.h:111-124.
     keys (p1,p2); meas = measured Pose3 (12); residual dim 6 */
  B200_FACTOR_BETWEEN_POSE3 = 0,
  /* PriorFactor<Pose3>, gtsam/nonlinear/PriorFactor.h:98-102. key; meas 12; dim 6 */
  B200_FACTOR_PRIOR_POSE3 = 1,
  /* PriorFactor<Point3>. key; meas 3; dim 3 */
  B200_FACTOR_PRIOR_POINT3 = 2,
  /* GenericProjectionFactor<Pose3,Point3,Cal3_S2>, gtsam/slam/ProjectionFactor.h:138-166
     (optional group-wide body_P_sensor, throwCheirality=false). keys (pose,point); meas z (2);
     dim 2; per-factor calibration index into desc.cal (5 doubles fx fy s u0 v0) */
  B200_FACTOR_PROJECTION_CAL3S2 = 3,
  /* GeneralSFMFactor<PinholeCamera<Cal3Bundler>,Point3>, gtsam/slam/GeneralSFMFactor.h:127-177.
     keys (camera,point); meas z (2); dim 2 */
  B200_FACTOR_SFM_BUNDLER = 4,
  /* PriorFactor<PinholeCamera<Cal3Bundler>>. key; meas 17; dim 9 */
  B200_FACTOR_PRIOR_CAM_BUNDLER = 5,
  /* BetweenFactor<Pose2> (the EDGE_SE2 lines of a g2o file, BASELINE configs[0]'s factor family),
     gtsam/slam/BetweenFactor.h:111-124 with gtsam/base/Lie.h:63-69 (between) and the Pose2 chart.
     keys (p1,p2); meas = measured Pose2 (x y theta); residual dim 3 */
  B200_FACTOR_BETWEEN_POSE2 = 6,
  /* PriorFactor<Pose2>. key; meas 3; dim 3 */
  B200_FACTOR_PRIOR_POSE2 = 7,
  B200_NUM_FACTOR_TYPES = 8,
  /* internal tags of the groups of a linear problem (b200_linear_create); never valid in a
     b200_factor_group */
  B200_FACTOR_JACOBIAN = 100,
  B200_FACTOR_HESSIAN = 101
};

/* ---- noise models (gtsam/linear/NoiseModel.cpp:83-130,163-238,322-340,646-675) */
enum {
  B200_NOISE_UNIT = 0,      /* no payload                                      */
  B200_NOISE_ISOTROPIC = 1, /* 1 double: sigma                                  */
  B200_NOISE_DIAGONAL = 2,  /* d doubles: sigmas                                */
  B200_NOISE_GAUSSIAN = 3   /* d*d doubles: sqrt information R (upper
                               triangular), row-major; whitened r = R r       */
};

/* m-estimators of noiseModel::Robust (gtsam/linear/LossFunctions.cpp), Block reweighting:
 * after whitening, A and b are scaled by sqrt(w(|b|)) and the factor's error is rho(|r|). */
enum {
  B200_ROBUST_NONE = 0,
  B200_ROBUST_HUBER = 1,   /* LossFunctions.cpp:179-191 */
  B200_ROBUST_CAUCHY = 2,  /* :217-224 */
  B200_ROBUST_TUKEY = 3,   /* :250-267 */
  B200_ROBUST_FAIR = 4     /* :146-155 */
};

/* One homogeneous run of factors (same type, same noise kind).  Factors of a
 * group occupy consecutive positions graph_index0 .. graph_index0+count-1 of
 * the NonlinearFactorGraph (position matters for the symbolic structure:
 * gtsam/inference/VariableIndex-inl.h:27-50 lists factor indices ascending). */
typedef struct b200_factor_group {
  int32_t type;             /* B200_FACTOR_*                                    */
  int32_t noise_kind;       /* B200_NOISE_*                                     */
  int32_t noise_per_factor; /* 0: one shared model for the group, 1: per factor */
  int32_t robust_kind;      /* B200_ROBUST_*: noiseModel::Robust wrapped around the
                               noise above (gtsam/linear/NoiseModel.cpp:708-733); 0 = none */
  int64_t count;
  int64_t graph_index0;     /* -1: append after the previous group              */
  const int64_t* keys;      /* count*arity variable ids                         */
  const double* meas;       /* count*meas_size                                  */
  const double* noise;      /* payload: shared or count*payload_size            */
  const int32_t* cal_index; /* PROJECTION_CAL3S2 only; NULL => calibration 0    */
  const double* body_P_sensor; /* PROJECTION_CAL3S2 only: one Pose3 (12 doubles) shared by
                               the group = GenericProjectionFactor's body_P_sensor
                               (gtsam/slam/ProjectionFactor.h:141-151), or NULL       */
  double robust_param;      /* k (Huber, Cauchy) / c (Tukey, Fair)                     */
  const int64_t* graph_index; /* optional: explicit graph position of every factor of the
                               group (count entries), for factors of one kind that are NOT
                               consecutive in the NonlinearFactorGraph; NULL => graph_index0 + i */
} b200_factor_group;

typedef struct b200_problem_desc {
  int64_t nvars;
  const int32_t* var_type;  /* nvars                                            */
  const double* values;     /* packed per variable in id order (storage sizes)  */
  const int64_t* ordering;  /* nvars: elimination order (variable ids)          */
  int64_t ncal;
  const double* cal;        /* ncal*5 Cal3_S2 (fx fy s u0 v0)                   */
  int64_t ngroups;
  const b200_factor_group* groups;
} b200_problem_desc;

/* LevenbergMarquardtParams subset, gtsam/nonlinear/LevenbergMarquardtParams.h:49-101
 * + NonlinearOptimizerParams.h:35-60. */
typedef struct b200_lm_params {
  int32_t max_iterations;        /* maxIterations (100)                         */
  double relative_error_tol;     /* 1e-5                                        */
  double absolute_error_tol;     /* 1e-5                                        */
  double error_tol;              /* 0                                           */
  double lambda_initial;         /* 1e-5                                        */
  double lambda_factor;          /* 10                                          */
  double lambda_upper_bound;     /* 1e5                                         */
  double lambda_lower_bound;     /* 0                                           */
  double min_model_fidelity;     /* 1e-3                                        */
  int32_t diagonal_damping;      /* false                                       */
  int32_t use_fixed_lambda_factor; /* true                                      */
  double min_diagonal;           /* 1e-6                                        */
  double max_diagonal;           /* 1e32                                        */
} b200_lm_params;

typedef struct b200_lm_state {
  double error;                  /* NonlinearOptimizerState::error              */
  double lambda;
  double current_factor;
  int32_t iterations;
  int32_t total_inner_iterations;
} b200_lm_state;

/* Sizes of the junction tree the symbolic phase built (a11). */
typedef struct b200_symbolic_info {
  int64_t ncliques;
  int64_t nlevels;
  int64_t total_dim;        /* sum of variable dims                             */
  int64_t max_frontal_dim;
  int64_t max_separator_dim;
  int64_t frontal_list_len; /* sum over cliques of #frontal variables           */
  int64_t separator_list_len;
  double factor_flops;      /* sum f^3/3 + f^2 s + f s^2                        */
  int64_t front_bytes;      /* bytes of all frontal matrices (of the supernodes) */
  /* The fields above describe the junction tree exactly as the reference builds it
   * (gtsam/inference/JunctionTree-inst.h:63-151): what b200_get_cliques and
   * b200_get_conditional report.  The device eliminates SUPERNODES: those cliques after
   * relaxed amalgamation (a non-leaf clique is merged into its parent when that adds few
   * explicit zeros; same elimination order, same conditionals up to rounding). */
  int64_t supernodes;
  int64_t supernode_levels;
  int64_t supernode_max_frontal_dim;
  int64_t supernode_max_separator_dim;
  int64_t supernode_frontal_list_len;
  int64_t supernode_separator_list_len;
  double supernode_flops;
} b200_symbolic_info;

typedef struct b200_ctx b200_ctx;
typedef struct b200_problem b200_problem;
typedef struct b200_lm b200_lm;

/* Static layout tables. */
int b200_var_storage(int32_t var_type);   /* doubles of storage */
int b200_var_dim(int32_t var_type);       /* tangent dimension  */
int b200_factor_arity(int32_t factor_type);
int b200_factor_meas_size(int32_t factor_type);
int b200_factor_dim(int32_t factor_type); /* residual rows      */

/* Context = one CUDA device + streams.  One per process in multi-GPU runs.
 * Fails with B200_NO_DEVICE when no GPU is visible (no CPU fallback). */
int b200_ctx_create(int device, b200_ctx** ctx);
int b200_ctx_destroy(b200_ctx* ctx);
const char* b200_last_error_string(void);
/* Number of kernels this library has launched since ctx creation. */
int64_t b200_launch_count(const b200_ctx* ctx);
/* Measured FP64 throughput of this device, TFLOP/s: the tensor path at its widest shape (mma.sync.m16n8k16.f64 on
 * sm_90, the FP64 tensor peak) and the FMA pipe, from registers with every SM full — the roofline denominators of the
 * dense-front kernels (bench.py). */
int b200_measure_fp64_peak(b200_ctx* ctx, double* dmma_tflops, double* dfma_tflops);
/* CUDA stream (cudaStream_t as void*) the library launches on. */
void* b200_ctx_stream(const b200_ctx* ctx);

/* One-time pack + symbolic phase.  Replaces the walk over
 * NonlinearFactorGraph / Values (gtsam/nonlinear/NonlinearFactorGraph.cpp:239-278)
 * and VariableIndex + EliminationTree + JunctionTree construction
 * (gtsam/inference/EliminateableFactorGraph-inst.h:123-146), hoisted out of
 * the per-solve path.  Copies everything; retains no host pointer. */
int b200_problem_create(b200_ctx* ctx, const b200_problem_desc* desc, b200_problem** prob);
int b200_problem_destroy(b200_problem* prob);

/* Values in / out (host buffers, packed like desc.values). */
int b200_set_values(b200_problem* prob, const double* packed_values);
int b200_get_values(b200_problem* prob, double* packed_values);
int64_t b200_values_size(const b200_problem* prob); /* doubles in packed values */
/* Replace the noise model(s) of factor group `group` (index into desc.groups) in place: `noise` is laid out like
 * b200_factor_group::noise for (noise_kind, noise_per_factor); the group's robust loss is kept.  This is what
 * GncOptimizer::makeWeightedGraph (gtsam/nonlinear/GncOptimizer.h:391-411) does to the graph between outer
 * iterations, without a new symbolic phase.  Invalidates the linearization; b200_lm / b200_dl handles created on
 * the problem before the call hold a stale error: create new ones. */
int b200_set_group_noise(b200_problem* prob, int64_t group, int32_t noise_kind, int32_t noise_per_factor, const double* noise);

int64_t b200_delta_size(const b200_problem* prob);  /* total tangent dim        */

/* NonlinearFactorGraph::error(values), gtsam/nonlinear/NonlinearFactorGraph.cpp:170-179 */
int b200_error(b200_problem* prob, double* error);

/* NonlinearFactorGraph::linearize(values): whitened per-factor [A1 A2 b],
 * device-resident (gtsam/nonlinear/NonlinearFactor.cpp:150-182). */
int b200_linearize(b200_problem* prob);
/* Debug/parity: copy a group's Jacobians to host, factor-major; each factor is
 * a column-major d x (n1 + n2 + 1) block [A1 A2 b] like VerticalBlockMatrix. */
int b200_get_jacobians(b200_problem* prob, int64_t group, double* out);

/* Precision of the stored linearization: 0 (default) = FP64, the reference's arithmetic; 1 = the
 * "FP32 linearize + FP64 solve" mode of BASELINE.json configs[4]: residuals and Jacobians are still evaluated in
 * FP64 registers but the whitened [A1 A2 b] blocks are rounded to and kept as floats (half the HBM traffic of
 * linearize and of every pass over the Jacobians); assembly, the multifrontal Cholesky, back-substitution, retract
 * and the nonlinear error stay FP64.  Parity in this mode is the FP32 protocol of SURVEY 8(c): [A|b] rel <= 1e-5,
 * final error rel <= 1e-5.  Call it any time: it invalidates the current linearization.  Not for linear problems. */
int b200_set_jacobian_precision(b200_problem* prob, int fp32);
int b200_get_jacobian_precision(const b200_problem* prob);
/* Kernel-variant switches of one problem, for A/B measurements (every variant computes the same result):
 * "schur_mma" 1 (default) = the BAL point leaves are factored and their per-run Schur complement formed on the FP64
 * tensor path in one kernel, 0 = a per-point factor kernel followed by the FMA-tile Schur kernel; "schur_pb" 4 / 6 = the
 * latter's points per staged batch; "df_minb" 2 / 3 = the dense-front kernel variant; "lin_variant" 0 / 4 =
 * linearize_kernel build of the projection groups (64 / 128 registers); "factor_staged" is accepted and has no effect
 * (kept so that existing callers still succeed).  Unknown key: B200_INVALID_ARGUMENT. */
int b200_set_tuning(b200_problem* prob, const char* key, int64_t value);

/* GaussianFactorGraph::hessianDiagonal(), gtsam/linear/GaussianFactorGraph.cpp:279-287.
 * out: delta_size doubles, variable-id order. */
int b200_hessian_diagonal(b200_problem* prob, double* out);
/* GaussianFactorGraph::gradientAtZero (gtsam/linear/GaussianFactorGraph.cpp:369-378; JacobianFactor.cpp:690-699,
 * HessianFactor.cpp:422-429): -A^T b of the whitened factors, delta_size doubles in dof order.  After b200_linearize
 * on a typed problem; any time on a linear problem. */
int b200_gradient_at_zero(b200_problem* prob, double* out);
/* GaussianFactorGraph::error(x) (gtsam/linear/GaussianFactorGraph.cpp:71-78) at the caller's x (delta_size doubles, dof
 * order): of the graph of a linear problem, or of the current linearization of a typed one. */
int b200_linear_graph_error(b200_problem* prob, const double* x, double* error);

/* Damped multifrontal Cholesky solve of the current linearization:
 * buildDampedSystem (gtsam/nonlinear/internal/LevenbergMarquardtState.h:125-156)
 * + GaussianFactorGraph::optimize (gtsam/linear/GaussianFactorGraph.cpp:316-319)
 * + the two linear.error() calls of tryLambda
 * (gtsam/nonlinear/LevenbergMarquardtOptimizer.cpp:170-171).
 * lambda == 0 => undamped (Gauss-Newton).  Returns B200_INDETERMINATE and the
 * id of a frontal variable of the failing clique in *fail_var. */
int b200_solve(b200_problem* prob, double lambda, int diagonal_damping,
               double min_diagonal, double max_diagonal,
               double* linear_error_zero, double* linear_error_delta,
               int64_t* fail_var);
/* delta of the last solve, delta_size doubles in variable-id order. */
int b200_get_delta(b200_problem* prob, double* out);

/* newValues = values.retract(delta) into scratch + graph.error(newValues)
 * (gtsam/nonlinear/Values.cpp:52-63). */
int b200_try_step(b200_problem* prob, double* new_error);
/* values <- newValues */
int b200_accept_step(b200_problem* prob);

/* Device-side snapshot / restore of the Values (reset between benchmark steps
 * without host traffic) and an explicit stream sync. */
int b200_save_values(b200_problem* prob);
int b200_restore_values(b200_problem* prob);
int b200_synchronize(b200_problem* prob);

/* Built-in phase timers — the counterpart of the reference's gttic/gttoc call
 * tree (gtsam/base/timing.h:245-302): CUDA events on the launching stream
 * around each phase, accumulated in milliseconds. */
int b200_profile_enable(b200_problem* prob, int on);   /* 1: start from zero, 2: resume, 0: pause */
int b200_profile_phase_count(void);
const char* b200_profile_phase_name(int phase);
int b200_profile_get(b200_problem* prob, double* ms, int64_t* calls);

/* Whole optimizers (host control logic a17/a18 unchanged, data on device). */
void b200_lm_params_legacy(b200_lm_params* p); /* LevenbergMarquardtParams::SetLegacyDefaults */
void b200_lm_params_ceres(b200_lm_params* p);  /* ::SetCeresDefaults                          */
int b200_lm_create(b200_problem* prob, const b200_lm_params* params, b200_lm** lm);
int b200_lm_destroy(b200_lm* lm);
/* LevenbergMarquardtOptimizer::iterate(), .cpp:273-308 */
int b200_lm_iterate(b200_lm* lm);
/* NonlinearOptimizer::defaultOptimize(), NonlinearOptimizer.cpp:62-117 */
int b200_lm_optimize(b200_lm* lm);
int b200_lm_get_state(const b200_lm* lm, b200_lm_state* state);
/* Reset state to (current device values, lambda_initial, iteration 0); recomputes error. */
int b200_lm_reset(b200_lm* lm);
/* GaussNewtonOptimizer::iterate(), gtsam/nonlinear/GaussNewtonOptimizer.cpp:44-67 */
int b200_gn_iterate(b200_problem* prob, double* new_error);

/* Marginals::marginalCovariance(key), gtsam/nonlinear/Marginals.cpp:118-154: the covariance of one variable under
 * the Gaussian of the graph linearised at the current values = the (var, var) block of (A^T A)^-1.  out: d x d
 * doubles, column-major, d = tangent dimension of the variable.  The first call after the values changed (or after
 * a damped solve) linearizes and factors the undamped system (B200_INDETERMINATE if that fails); further calls reuse
 * the factor and only walk the clique path from the variable to the root.  Single-GPU only. */
int b200_marginal_covariance(b200_problem* prob, int64_t var, double* out);
/* Marginals::jointMarginalCovariance(keys).fullMatrix(), gtsam/nonlinear/Marginals.cpp:128-190: vars are distinct
 * variable ids in ASCENDING order (the reference returns the blocks in sorted-key order as well); out: D x D doubles,
 * column-major, D = sum of their tangent dimensions (<= 128). */
int b200_joint_marginal_covariance(b200_problem* prob, const int64_t* vars, int64_t nvars, double* out);

/* Powell's dogleg.  b200_dl_iterate = DoglegOptimizer::iterate(),
 * gtsam/nonlinear/DoglegOptimizer.cpp:84-121, with DoglegOptimizerImpl::Iterate in
 * ONE_STEP_PER_ITERATION mode (gtsam/nonlinear/DoglegOptimizerImpl.h:139-258): linearize,
 * multifrontal solve for the Newton point dx_n, steepest-descent point dx_u
 * (GaussianFactorGraph::optimizeGradientSearch, gtsam/linear/GaussianFactorGraph.cpp:381-407),
 * then the trust-region loop on the dogleg point.  delta_initial is DoglegParams::deltaInitial.
 * Single-GPU only: B200_INVALID_ARGUMENT on a context with a communicator. */
typedef struct b200_dl b200_dl;
int b200_dl_create(b200_problem* prob, double delta_initial, b200_dl** out);
int b200_dl_destroy(b200_dl* dl);
int b200_dl_iterate(b200_dl* dl);
/* error = state error, delta = trust region radius, iterations = iterate() calls so far */
int b200_dl_get_state(const b200_dl* dl, double* error, double* delta, int32_t* iterations);

/* ---- GaussianFactorGraph level -----------------------------------------------------------
 * The same multifrontal solve on an ALREADY LINEARIZED graph: what
 * GaussianFactorGraph::optimize(ordering, EliminatePreferCholesky)
 * (gtsam/linear/GaussianFactorGraph.cpp:316-319 -> EliminateableFactorGraph-inst.h:123-146 ->
 * HessianFactor.cpp:516-536 -> linearAlgorithms-inst.h:50-117) does for a graph of JacobianFactors
 * of any arity and any block widths (gtsam/linear/JacobianFactor.h:93-103) and HessianFactors
 * (gtsam/linear/HessianFactor.h:99-110; HessianFactor::updateHessian, HessianFactor.cpp:348-374),
 * i.e. rows a11-a16 of the hot path without a1-a9.  The handle is a b200_problem: b200_solve (lambda = 0, or > 0 for
 * buildDampedSystem's priors), b200_get_delta, b200_hessian_diagonal, b200_get_conditional,
 * b200_symbolic_info_get / b200_get_cliques, b200_marginal_covariance and
 * b200_joint_marginal_covariance work on it; the calls that need Values (b200_error, b200_linearize,
 * b200_try_step, b200_lm_*, b200_gn_iterate, b200_dl_*) return B200_INVALID_ARGUMENT.
 * On a context with a communicator the factors are split by owning subtree exactly like the typed groups
 * (SURVEY 8e): every rank passes the WHOLE description (and whole groups to b200_linear_update*) and keeps its
 * share; b200_get_delta returns the rank's own view (zeros elsewhere), as for a sharded b200_problem. */
#define B200_JACOBIAN_MAX_ARITY 8
/* One run of JacobianFactors with the same shape (rows, arity, block widths). */
typedef struct b200_jacobian_group {
  int32_t rows;             /* rows of [A1 .. Ak b]                                   */
  int32_t arity;            /* k, 1 .. B200_JACOBIAN_MAX_ARITY                         */
  const int32_t* dims;      /* k block widths; must equal var_dim of the keyed variables */
  int64_t count;
  int64_t graph_index0;     /* -1: append after the previous group                     */
  const int64_t* graph_index; /* optional explicit graph positions (count), else NULL  */
  const int64_t* keys;      /* count*arity variable ids, in the factor's key order    */
  const double* Ab;         /* count blocks, each rows x (sum(dims)+1) COLUMN-MAJOR =
                               JacobianFactor::matrixObject() (VerticalBlockMatrix, b last) */
  const double* sigmas;     /* NULL: unit model (or already whitened); else count*rows Diagonal
                               sigmas: row r of [A|b] is divided by sigmas[r]
                               (JacobianFactor::whiten, gtsam/linear/JacobianFactor.cpp:743-757, as updateHessian :563-598 does).
                               Constrained models (sigma == 0) are rejected: B200_UNSUPPORTED_NOISE */
} b200_jacobian_group;

/* One run of HessianFactors (gtsam/linear/HessianFactor.h:99-110) with the same block widths: the
 * quadratic 0.5 (f - 2 x'g + x'G x), stored as the augmented information matrix [G g; g' f]. */
typedef struct b200_hessian_group {
  int32_t arity;            /* k, 1 .. B200_JACOBIAN_MAX_ARITY                         */
  const int32_t* dims;      /* k block widths                                          */
  int64_t count;
  int64_t graph_index0;     /* -1: append after the previous group (Jacobian groups come first) */
  const int64_t* graph_index;
  const int64_t* keys;      /* count*arity variable ids                                */
  const double* info;       /* count blocks, each (N+1) x (N+1) COLUMN-MAJOR, N = sum(dims):
                               HessianFactor::info() (SymmetricBlockMatrix); only the upper
                               triangle is read                                        */
} b200_hessian_group;

typedef struct b200_linear_desc {
  int64_t nvars;
  const int32_t* var_dim;   /* nvars: tangent dimension of every variable (>= 1)       */
  const int64_t* ordering;  /* nvars: elimination order (variable ids)                 */
  int64_t ngroups;
  const b200_jacobian_group* groups;
  int64_t nhgroups;         /* HessianFactor groups (0 / NULL when the graph has none) */
  const b200_hessian_group* hgroups;
} b200_linear_desc;

/* Pack + symbolic phase + upload of the whitened [A|b] blocks (whitening is a kernel). */
int b200_linear_create(b200_ctx* ctx, const b200_linear_desc* desc, b200_problem** prob);
/* New numbers, same structure (the next linearization of the same graph): re-uploads group
 * `group`'s [A|b] (and sigmas, NULL = unit); the symbolic phase and all tables are reused. */
int b200_linear_update(b200_problem* prob, int64_t group, const double* Ab, const double* sigmas);
/* The same for HessianFactor group `hgroup`: new augmented information matrices. */
int b200_linear_update_hessian(b200_problem* prob, int64_t hgroup, const double* info);
/* Host-only symbolic phase of a linear description (CPU tests of a11 on n-ary factors). */
typedef struct b200_symbolic b200_symbolic;
int b200_linear_symbolic_create(const b200_linear_desc* desc, b200_symbolic** out);

/* Symbolic-phase introspection (parity of a11 against the reference's
 * junction tree).  Cliques are numbered in elimination post-order. */
int b200_symbolic_info_get(const b200_problem* prob, b200_symbolic_info* info);
/* frontal_ptr/separator_ptr: ncliques+1; frontal_vars/separator_vars: list
 * lengths from b200_symbolic_info; parent: ncliques (-1 for roots). */
int b200_get_cliques(const b200_problem* prob, int64_t* frontal_ptr, int64_t* frontal_vars,
                     int64_t* separator_ptr, int64_t* separator_vars, int64_t* parent);
/* The supernodes the device eliminates (sizes: the supernode_* fields of b200_symbolic_info). */
int b200_get_supernodes(const b200_problem* prob, int64_t* frontal_ptr, int64_t* frontal_vars,
                        int64_t* separator_ptr, int64_t* separator_vars, int64_t* parent);

/* Host-only symbolic phase (no GPU needed): the same junction tree
 * b200_problem_create builds, for inspection and CPU-side tests of a11. */
int b200_symbolic_create(const b200_problem_desc* desc, b200_symbolic** out);
int b200_symbolic_destroy(b200_symbolic* s);
int b200_symbolic_get_info(const b200_symbolic* s, b200_symbolic_info* info);
int b200_symbolic_get_cliques(const b200_symbolic* s, int64_t* frontal_ptr, int64_t* frontal_vars,
                              int64_t* separator_ptr, int64_t* separator_vars, int64_t* parent);
int b200_symbolic_get_levels(const b200_symbolic* s, int32_t* level); /* ncliques */
int b200_symbolic_get_supernodes(const b200_symbolic* s, int64_t* frontal_ptr, int64_t* frontal_vars,
                                 int64_t* separator_ptr, int64_t* separator_vars, int64_t* parent);
int b200_symbolic_get_clique_supernode(const b200_symbolic* s, int32_t* supernode); /* ncliques: supernode holding each clique */
/* Scatter tables of the assembly (a12): owning SUPERNODE of every factor by graph position (nfactors entries) and the
 * scalar slot, in that supernode's front, of every key of every factor (laid out factor after factor in graph order,
 * each factor's keys in its own key order). */
int b200_symbolic_get_factor_slots(const b200_symbolic* s, int32_t* clique, int32_t* slots);

/* Parity of a14: the conditional [R S d] of clique c after a solve
 * (gtsam/linear/HessianFactor.cpp:459-487), nf x (nf+ns+1) column-major. */
int b200_get_conditional(b200_problem* prob, int64_t clique, double* out);

/* Multi-GPU (SURVEY §8(e)), one process per GPU.  Rank 0 calls b200_nccl_unique_id and
 * ships the 128 bytes to the other ranks (torch.distributed / MPI / a file); every rank then
 * calls b200_ctx_comm_init BEFORE b200_problem_create.  The problem description is the
 * full graph on every rank; the junction tree is cut into a replicated top and subtrees
 * (BAL: the points; nested dissection: the ND branches); each rank keeps the subtrees it owns
 * and their factors.  Per solve there is ONE exchange step:
 * an in-place ncclAllReduce (FP64 sum, NVLink) of the top fronts, plus a 2-double / 2-int
 * all-reduce of the scalars LM branches on.  b200_get_values returns this rank's view
 * (owned leaf variables + the replicated top variables are current). */
/* Sharded problems move only a rank's share of the Values between host and device: view 0 = the variables the rank needs
 * as input (those its factors touch, the frontal variables of its cliques and of the top), view 1 = the variables it owns
 * (its own subtrees; rank 0 reports the top) — the new values of a step are current on their owner.  var_ids (ascending,
 * may be NULL) lists the variables; the packed view is their storage concatenated.  One rank: both views are everything. */
int b200_values_view(const b200_problem* prob, int which, int64_t* nvars, int64_t* ndoubles, int64_t* var_ids);
int b200_set_values_view(b200_problem* prob, const double* packed_input_view);
int b200_get_values_view(b200_problem* prob, double* packed_owned_view);
/* The whole packed Values on every rank (the owned views gathered by one all-reduce); one rank: b200_get_values. */
int b200_get_values_all(b200_problem* prob, double* packed);
int b200_nccl_unique_id(void* out128);
int b200_ctx_comm_init(b200_ctx* ctx, const void* id128, int rank, int world);
int b200_shard_plan(const b200_problem_desc* desc, int world, int32_t* clique_owner, int32_t* factor_owner);

/* The dense frontal storage of the cliques that are
 * shared between ranks (the top of the tree) as one contiguous device buffer,
 * so the caller's communicator (NCCL via torch.distributed) can sum it between
 * "eliminate local subtrees" and "eliminate shared top".  See DESIGN.md. */
int b200_shared_front_buffer(b200_problem* prob, void** device_ptr, int64_t* ndoubles);

#ifdef __cplusplus
}
#endif
#endif /* GTSAM_B200_H */
