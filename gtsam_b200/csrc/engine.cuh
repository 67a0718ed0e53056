// engine.cuh — internal structures shared by the kernels and the C-ABI glue.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <string>
#include <vector>

#include "../../include/gtsam_b200.h"
#include "symbolic.h"

namespace b200 {

void set_error(const std::string& s);

#define B200_CUDA(call)                                                                   \
  do {                                                                                    \
    cudaError_t e_ = (call);                                                              \
    if (e_ != cudaSuccess) {                                                              \
      ::b200::set_error(std::string(#call) + ": " + cudaGetErrorString(e_) + " at " +     \
                        __FILE__ + ":" + std::to_string(__LINE__));                       \
      return B200_CUDA_ERROR;                                                             \
    }                                                                                     \
  } while (0)

// Device-side view of one factor group (passed to kernels by value).
struct GroupView {
  int type, noise_kind, per_factor, noise_size;
  int count;
  int robust_kind;         // B200_ROBUST_*
  double robust_param;
  const int2* keys;        // (key0, key1 or -1)
  const double* meas;      // AoS, MEAS doubles per factor
  const double* noise;     // shared payload or per-factor AoS
  const int* cal_index;    // may be null
  const double* body;      // body_P_sensor (12 doubles) of a projection group, or null
  double* J;               // SoA: J[e * count + f], e = r + c*D (column-major element order); holds floats in the
                           // FP32-storage mode (the kernels' JT template parameter says which)
  const int4* scat;        // (clique, slot0, slot1, unused) per factor
};

// Device-side view of one JacobianFactor group of a linear problem (b200_linear_create): factors of any
// arity and block widths, [A1 .. Ak b] stored like the typed groups (element-major SoA).
struct JacobianView {
  int count, rows, arity, ncols;            // ncols = sum of the block widths + 1
  int col0[B200_JACOBIAN_MAX_ARITY + 2];    // first column of block a; col0[arity] = the rhs column, col0[arity+1] = ncols
  const int* keys;                          // count*arity variable ids
  const int* slots;                         // count*arity scalar slots of the keys in the owning clique's front
  const int* clique;                        // count: owning clique
  double* J;                                // J[e * count + f], e = r + c*rows
};

// Device-side view of the junction tree + frontal arena.
struct TreeView {
  double* arena;           // all fronts, each (nf+ns+1)^2 col-major, upper triangle used
  const int64_t* off;      // per clique offset into arena
  const int* nf;
  const int* ns;
  const int* parent;
  const int* ld;           // leading dimension of the stored block (n, or nf for fused leaves)
  const int64_t* ea_ptr;
  const int* ea_map;
  const int64_t* didx_ptr;
  const int* didx;
};

struct Scalars {           // device scalars fetched once per LM try
  double error;            // graph.error(values)
  double lin_err0;         // linear.error(0)
  double lin_err_delta;    // linear.error(delta)
  double new_error;        // graph.error(newValues)
  int fail_code;           // INT_MAX - (min clique id whose partial Cholesky failed); 0 = none
  int nan_code;            // INT_MAX - (min clique id with NaN in back-substitution); 0 = none
  int df_abort;            // front_df_kernel: a bounded wait timed out and the launch bailed out (internal error)
  int pad;
  double dl_dots[3];       // Dogleg: g.g, g.dx_n, dx_n.dx_n
  double dl_half_Ag2;      // Dogleg: 0.5*|A g|^2
  double dl_scratch;       // second output slot of linerr_kernel when only one is wanted
  double graph_err;        // b200_linear_graph_error: GaussianFactorGraph::error(x)
};

struct LevelPlan {
  int small_begin, small_count;   // range in d_lvl_small (elimination, one warp per clique)
  int bsmall_begin, bsmall_count; // range in d_lvl_bsmall (back-substitution, one warp per clique: at most kSmallMaxN pivots)
  int blarge_begin, blarge_count; // back-substitution of fronts with more than kSmallMaxN pivots (range in d_lvl_blarge)
  int blarge_max_nf;
  int bpoint_begin[2], bpoint_count[2];  // BAL point leaves, DC = 6 / 9 (ranges in d_lvl_bpoint)
};

}  // namespace b200

namespace b200 { struct ncclUniqueIdBlob { char internal[128]; }; }

struct b200_ctx {
  int rank = 0, world = 1;   // one process per GPU; world > 1 after b200_ctx_comm_init
  void* comm = nullptr;      // ncclComm_t
  int device = 0;
  cudaStream_t stream = nullptr;
  int64_t launches = 0;
  int sm_count = 0;
};

struct b200_problem {
  b200_ctx* ctx = nullptr;
  bool linear = false;     // created by b200_linear_create: JacobianFactor groups, no Values
  bool jac_f32 = false;    // whitened Jacobians stored as floats (b200_set_jacobian_precision): "FP32 linearize + FP64 solve"
  b200::Symbolic sym;
  int64_t nvars = 0, nfactors = 0, nval = 0, ndelta = 0;
  std::vector<int> var_type;
  // host copies of group metadata
  struct Group {
    int type, noise_kind, per_factor, noise_size, d, ncols, arity, meas;
    int robust_kind = 0;
    double robust_param = 0;
    int64_t count;
    std::vector<int64_t> pos;          // graph position of every factor of the caller's group
    int2* d_keys = nullptr;
    double* d_meas = nullptr;
    double* d_noise = nullptr;
    int* d_cal = nullptr;
    double* d_body = nullptr;
    double* d_J = nullptr;
    int4* d_scat = nullptr;
    int col0[B200_JACOBIAN_MAX_ARITY + 2] = {0};   // JacobianFactor groups: first column of every block
    int *d_jkeys = nullptr, *d_jslots = nullptr, *d_jclique = nullptr;   // JacobianFactor groups (see JacobianView)
    int64_t n_nonleaf = 0;   // factors NOT owned by a fused leaf clique
    std::vector<int64_t> local_index;  // index in the caller's group of every factor kept on this rank
    int64_t full_count = 0;            // linear groups: the caller's factor count (count = this rank's share)
  };
  std::vector<Group> groups;
  // device state
  double *d_values = nullptr, *d_new_values = nullptr, *d_delta = nullptr, *d_hdiag = nullptr;
  double* d_grad = nullptr;          // b200_gradient_at_zero (allocated on first use)
  int *d_val_off = nullptr, *d_var_type = nullptr, *d_var_dof = nullptr;
  double* d_cal = nullptr;
  double* d_arena = nullptr;
  int64_t* d_off = nullptr;
  int *d_nf = nullptr, *d_ns = nullptr, *d_parent = nullptr, *d_ld = nullptr;
  std::vector<int64_t> h_off;       // final arena offsets (fused leaves store f x n only)
  std::vector<int> h_ld;
  // fused leaf path
  int n_fused = 0, n_runs = 0, leaf_lb_cap = 1, leaf_acc_cap = 0;
  int leaf_run_begin[3] = {0, 0, 0}, leaf_run_end[3] = {0, 0, 0};  // run ranges: generic / point DC=6 / point DC=9
  int schur_pb = 4;                                                 // points per staged batch of leaf_point_schur_kernel
  bool schur_mma = true;                                            // BAL point leaves: factor + per-run Schur complement on the FP64 tensor path in one kernel (leaf_point_fused_mma_kernel)
  int lin_variant = 0;                                              // linearize_kernel variant of the projection groups (b200_set_tuning)
  int leaf_max_w[3] = {1, 1, 1};                                    // widest separator + 1 per kind
  int leaf_pos_begin[3] = {0, 0, 0}, leaf_pos_end[3] = {0, 0, 0};  // the same ranges as positions in d_fused_list
  int *d_fused_list = nullptr, *d_fused_fac_ptr = nullptr, *d_fused_run_ptr = nullptr;
  int2* d_fused_fac = nullptr;
  int2* d_pt_tab = nullptr;         // BAL point leaves: per (list position, factor slot) (factor index, group << 8 | camera slot); -1: no factor
  int64_t* d_pt_off = nullptr;      // ... and the arena offset of the point's conditional
  int64_t top_doubles = 0;          // [0, top_doubles) = fronts of the replicated top (all-reduced when sharded)
  int n_sub_levels = 0;             // levels[0..n_sub_levels) = owned subtrees, the rest = the top
  int64_t arena_doubles = 0, zero_doubles = 0;  // [0, zero_doubles) = non-leaf fronts (memset per solve)
  int64_t *d_ea_ptr = nullptr, *d_didx_ptr = nullptr;
  int *d_ea_map = nullptr, *d_didx = nullptr;
  int64_t* d_diag_index = nullptr;  // per delta scalar: arena index of its diagonal entry
  int *d_lvl_small = nullptr, *d_lvl_bsmall = nullptr, *d_lvl_blarge = nullptr, *d_lvl_bpoint = nullptr;
  std::vector<b200::LevelPlan> levels;
  int *d_bs_flags = nullptr, *d_bs_flag_base = nullptr;  // publish flags of the multi-CTA back-substitution
  int n_bs_flags = 0;
  double* d_lambda = nullptr;       // lambda of the current try (device resident)
  double* h_lambda = nullptr;       // pinned
  cudaGraphExec_t try_graph[2] = {nullptr, nullptr};  // LM try (solve + retract + error), by diagonal flag
  double graph_min_diag[2] = {0, 0}, graph_max_diag[2] = {0, 0};
  bool hdiag_valid = false;         // d_hdiag holds hessianDiagonal of the current linearization
  int64_t try_launches = 0;
  // tile-dataflow elimination of the non-leaf fronts (front_df.cuh): one launch per phase (own subtrees / replicated top)
  int df_level[2] = {-1, -1};       // index in `levels` at which the launch of the phase is issued
  int df_ntasks[2] = {0, 0};
  int4* d_df_tasks[2] = {nullptr, nullptr};
  int *d_df_flag_off = nullptr, *d_df_expect = nullptr;
  int* d_df_sync = nullptr;         // [ctrl of phase 0 (2) | ctrl of phase 1 (2) | done per clique | piece flags]: zeroed per solve
  int64_t df_sync_ints = 0;
  int df_ctrl_ints = 4;
  int df_minb = 3;                  // kernel variant: resident CTAs per SM it is compiled for
  unsigned long long* d_df_trace = nullptr;   // B200_DF_TRACE: 32 globaltimer stamps per tile of phase 0
  // sharded solve, distributed top (DESIGN.md 7): every front of the top of the tree has an OWNER rank; per top level
  // ("stage") the ranks' partial fronts are summed onto their owners (ncclReduce, grouped), the owners factor them
  // (front_df_kernel over their tiles of the stage) and extend-add into their copy of the parent; back-substitution
  // walks the stages downwards, the owners' solutions travel in a packed vector (one small all-reduce per stage)
  double* d_winv = nullptr;         // W = R_kk^-1 of every factored 32 x 32 diagonal block (front_df_kernel), for back-substitution
  int64_t* d_winv_off = nullptr;    // per clique: offset into d_winv (-1: none)
  // values views of a sharded problem (b200_values_view): [0] what this rank needs as input, [1] what it owns
  std::vector<int64_t> view_vars[2];
  int64_t view_doubles[2] = {0, 0};
  int* d_view_idx[2] = {nullptr, nullptr};   // per packed double: its index in the full packed Values
  double* d_view_buf = nullptr;
  double* d_gather_buf = nullptr;            // b200_get_values_all: full-size buffer the owned views are all-reduced in
  bool defer_scalar_reduce = false; // inside an LM try: the scalar all-reduces are merged into one (enqueue_try)
  double* d_red = nullptr;
  bool top_staged = false;
  struct TopFront { int64_t off, count; int owner, clique; };
  std::vector<TopFront> ts_fronts;              // all top fronts, grouped by stage
  std::vector<int> ts_level, ts_begin, ts_task_begin, ts_task_count, ts_x_begin, ts_x_count;   // per stage (ts_begin has nstages + 1 entries)
  int *d_ts_cliques = nullptr, *d_ts_xoff = nullptr, *d_ts_owned = nullptr;
  double* d_topx = nullptr;
  int64_t topx_doubles = 0;
  double* d_partials = nullptr;     // block partial sums
  unsigned* d_counters = nullptr;   // tickets of the last-block reductions
  int partial_cap = 0;
  b200::Scalars* d_scalars = nullptr;
  b200::Scalars* h_scalars = nullptr;  // pinned
  double* h_pinned = nullptr;          // pinned staging for values
  bool linearized = false, solved = false, factored = false;
  bool marg_ready = false;          // the fronts hold the UNDAMPED factor of H at the current values
  double* d_marg_work = nullptr;    // Marginals: one scratch vector per covariance column
  int* d_marg_path = nullptr;
  double* d_marg_out = nullptr;
  double* d_saved_values = nullptr;
  // phase timers
  bool profile = false;
  std::vector<std::pair<cudaEvent_t, cudaEvent_t>> ev_pool;
  std::vector<int> ev_phase;
  size_t ev_used = 0;
  double phase_ms[16] = {0};
  int64_t phase_calls[16] = {0};
  int max_small_n = 0;
};

struct b200_dl {
  b200_problem* prob;
  double delta;        // trust region radius (DoglegState::delta)
  double error;
  int iterations;
  double* d_grad = nullptr;   // gradientAtZero, then scaled in the blend
  double* d_dxn = nullptr;    // Newton point
};

struct b200_lm {
  b200_problem* prob;
  b200_lm_params params;
  b200_lm_state state;
};
