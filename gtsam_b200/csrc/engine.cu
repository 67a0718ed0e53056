// engine.cu — C-ABI of include/gtsam_b200.h: packing, symbolic phase, kernel
// scheduling (level-by-level walk of the junction tree) and the LM / GN host
// control logic.  No CPU fallback anywhere: every numeric step is a kernel.
#include <algorithm>
#include <chrono>
#include <climits>
#include <cmath>
#include <cstdlib>
#include <dlfcn.h>
#include <cstring>
#include <limits>
#include <memory>
#include <thread>

#include "kernels.cuh"

namespace b200 {

static thread_local std::string g_err;

// Host loops of the one-time setup that write disjoint ranges run on a few threads (B200_SETUP_THREADS; 1 = serial).
template <class F>
static void parallel_chunks(int64_t n, F f) {
  int nt = (int)std::min<int64_t>(std::max(1u, std::thread::hardware_concurrency()), 16);
  if (const char* e = getenv("B200_SETUP_THREADS")) nt = std::min(16, std::max(1, atoi(e)));
  nt = (int)std::min<int64_t>(nt, std::max<int64_t>(1, n / 65536));
  if (nt <= 1) { f((int64_t)0, n, 0); return; }
  std::vector<std::thread> pool;
  for (int t = 0; t < nt; t++) pool.emplace_back([=, &f]() { f(n * t / nt, n * (t + 1) / nt, t); });
  for (auto& th : pool) th.join();
}
void set_error(const std::string& s) { g_err = s; }

static const int VAR_STORAGE[B200_NUM_VAR_TYPES] = {12, 3, 17, 3};
static const int VAR_DIM[B200_NUM_VAR_TYPES] = {6, 3, 9, 3};
static const int F_ARITY[B200_NUM_FACTOR_TYPES] = {2, 1, 1, 2, 2, 1, 2, 1};
static const int F_MEAS[B200_NUM_FACTOR_TYPES] = {12, 12, 3, 2, 2, 17, 3, 3};
static const int F_DIM[B200_NUM_FACTOR_TYPES] = {6, 6, 3, 2, 2, 9, 3, 3};
static const int F_VT[B200_NUM_FACTOR_TYPES][2] = {{0, 0}, {0, -1}, {1, -1}, {0, 1}, {2, 1}, {2, -1}, {3, 3}, {3, -1}};

static int noise_payload(int kind, int d) {
  switch (kind) {
    case B200_NOISE_UNIT: return 0;
    case B200_NOISE_ISOTROPIC: return 1;
    case B200_NOISE_DIAGONAL: return d;
    case B200_NOISE_GAUSSIAN: return d * d;
  }
  return -1;
}

template <class T>
static cudaError_t upload(DevPtr<T>& dst, const T* src, size_t n, cudaStream_t st) {
  cudaError_t e = dst.alloc(n);
  if (e == cudaSuccess && n) e = cudaMemcpyAsync(dst, src, n * sizeof(T), cudaMemcpyHostToDevice, st);
  return e;
}
template <class T>
static cudaError_t upload(DevPtr<T>& dst, const std::vector<T>& v, cudaStream_t st) { return upload(dst, v.data(), v.size(), st); }

static GroupView view(const b200_problem::Group& g) {
  GroupView v;
  v.type = g.type; v.noise_kind = g.noise_kind; v.per_factor = g.per_factor; v.noise_size = g.noise_size;
  v.count = (int)g.count; v.robust_kind = g.robust_kind; v.robust_param = g.robust_param; v.keys = g.d_keys; v.meas = g.d_meas; v.noise = g.d_noise; v.cal_index = g.d_cal; v.body = g.d_body;
  v.J = g.d_J; v.scat = g.d_scat;
  return v;
}
static JacobianView jview(const b200_problem::Group& g) {
  JacobianView v;
  v.count = (int)g.count; v.rows = g.d; v.arity = g.arity; v.ncols = g.ncols;
  for (int a = 0; a < B200_JACOBIAN_MAX_ARITY + 2; a++) v.col0[a] = g.col0[a];
  v.keys = g.d_jkeys; v.slots = g.d_jslots; v.clique = g.d_jclique; v.J = g.d_J;
  return v;
}
static TreeView tview(const b200_problem* p) {
  TreeView t;
  t.arena = p->d_arena; t.off = p->d_off; t.nf = p->d_nf; t.ns = p->d_ns; t.parent = p->d_parent; t.ld = p->d_ld;
  t.ea_ptr = p->d_ea_ptr; t.ea_map = p->d_ea_map; t.didx_ptr = p->d_didx_ptr; t.didx = p->d_didx;
  return t;
}
static EvalCtx ectx(const b200_problem* p, const double* values) {
  EvalCtx c;
  c.values = values; c.val_off = p->d_val_off; c.cal = p->d_cal;
  return c;
}

#define DISPATCH_TYPE(T, STMT)                                                                  \
  switch (T) {                                                                                  \
    case B200_FACTOR_BETWEEN_POSE3: { constexpr int TY = B200_FACTOR_BETWEEN_POSE3; STMT; break; }         \
    case B200_FACTOR_PRIOR_POSE3: { constexpr int TY = B200_FACTOR_PRIOR_POSE3; STMT; break; }             \
    case B200_FACTOR_PRIOR_POINT3: { constexpr int TY = B200_FACTOR_PRIOR_POINT3; STMT; break; }           \
    case B200_FACTOR_PROJECTION_CAL3S2: { constexpr int TY = B200_FACTOR_PROJECTION_CAL3S2; STMT; break; } \
    case B200_FACTOR_SFM_BUNDLER: { constexpr int TY = B200_FACTOR_SFM_BUNDLER; STMT; break; }             \
    case B200_FACTOR_PRIOR_CAM_BUNDLER: { constexpr int TY = B200_FACTOR_PRIOR_CAM_BUNDLER; STMT; break; } \
    case B200_FACTOR_BETWEEN_POSE2: { constexpr int TY = B200_FACTOR_BETWEEN_POSE2; STMT; break; }         \
    case B200_FACTOR_PRIOR_POSE2: { constexpr int TY = B200_FACTOR_PRIOR_POSE2; STMT; break; }             \
  }

// storage type of the whitened Jacobians (b200_set_jacobian_precision): JT = float or double inside the statement
#define DISPATCH_JT(P, ...)                                   \
  do {                                                        \
    if ((P)->jac_f32) { typedef float JT; __VA_ARGS__; }      \
    else { typedef double JT; __VA_ARGS__; }                  \
  } while (0)

// ---- built-in phase timers (the reference has gttic/gttoc, gtsam/base/timing.h:245-302):
// CUDA events on the launching stream, resolved at the next host sync. -----------------
enum Phase { PH_LINEARIZE = 0, PH_MEMSET, PH_ASSEMBLE, PH_DAMP, PH_ELIM_SMALL, PH_ELIM_LARGE, PH_BACKSUB,
             PH_LINERR, PH_RETRACT, PH_ERROR, PH_LEAF, PH_ALLREDUCE, PH_LINEARIZE_MINOR, PH_LEAF_SCHUR, PH_TOPX, PH_COUNT };
struct PhaseScope {
  b200_problem* p; int ph; size_t idx; bool on;
  PhaseScope(b200_problem* p_, int ph_) : p(p_), ph(ph_), idx(0), on(p_->profile) {
    if (!on) return;
    if (p->ev_used == p->ev_pool.size()) {
      cudaEvent_t a, b;
      cudaEventCreate(&a); cudaEventCreate(&b);
      p->ev_pool.push_back({a, b});
    }
    idx = p->ev_used++;
    p->ev_phase.resize(p->ev_used);
    p->ev_phase[idx] = ph;
    cudaEventRecord(p->ev_pool[idx].first, p->ctx->stream);
  }
  ~PhaseScope() { if (on) cudaEventRecord(p->ev_pool[idx].second, p->ctx->stream); }
};
static void resolve_profile(b200_problem* p) {  // call after a stream sync
  for (size_t i = 0; i < p->ev_used; i++) {
    float ms = 0;
    if (cudaEventElapsedTime(&ms, p->ev_pool[i].first, p->ev_pool[i].second) == cudaSuccess) {
      p->phase_ms[p->ev_phase[i]] += ms;
      p->phase_calls[p->ev_phase[i]] += 1;
    }
  }
  p->ev_used = 0;
}

// Kernel launch with the programmatic-dependent-launch attribute (see pdl_sync in kernels.cuh).
static const bool g_use_pdl = getenv("B200_NO_PDL") == nullptr;
#ifdef B200_EMULATE
// test-only host emulation build (tests/emu/cuda_emu_full.h): a launch runs the kernel's blocks one after the other
template <typename... KArgs, typename... Args>
static void launch_k(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t, Args&&... args) {
  // ascending blockIdx.x is dependency-safe: backsub_large_kernel's row blocks only wait (flags) on lower block ids
  b200_emu::count_launch((const void*)kernel);   // B200_EMU_TRACE_FILE: which kernels the scenarios reach
  b200_emu::run(grid, block, smem, false, [&]() { kernel(KArgs(args)...); });
}
template <typename... KArgs, typename... Args>
static void launch_plain(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  launch_k(kernel, grid, block, smem, st, std::forward<Args>(args)...);
}
#else
template <typename... KArgs, typename... Args>
static void launch_k(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = g_use_pdl ? 1 : 0;
  cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}
// a plain launch (what kernel<<<grid, block, smem, st>>>(args...) does): no programmatic dependent launch
template <typename... KArgs, typename... Args>
static void launch_plain(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}
#endif

static int allreduce_sum(b200_problem* p, double* buf, size_t n);
static int allreduce_max_int(b200_problem* p, int* buf, size_t n);
static int reduce_top_stage(b200_problem* p, size_t stage);

static int reduce_blocks(int64_t count, int threads, int sm) {
  int64_t b = (count + threads - 1) / threads;
  return (int)std::max<int64_t>(1, std::min<int64_t>(b, (int64_t)sm * 8));
}

// graph.error(values) -> *slot (device double)
static int enqueue_error(b200_problem* p, const double* values, double* slot) {
  cudaStream_t st = p->ctx->stream;
  PhaseScope ps(p, PH_ERROR);
  bool first = true;
  for (auto& g : p->groups) {
    if (!g.count) continue;
    const int nb = reduce_blocks(g.count, 256, p->ctx->sm_count);
    DISPATCH_TYPE(g.type, (launch_k(error_kernel<TY>, dim3(nb), dim3(256), 0, st, view(g), ectx(p, values), p->d_partials, p->d_counters, slot, first ? 0 : 1)));
    p->ctx->launches += 1;
    first = false;
  }
  if (first) B200_CUDA(cudaMemsetAsync(slot, 0, sizeof(double), st));
  B200_CUDA(cudaGetLastError());
  if (p->defer_scalar_reduce) return B200_OK;   // an LM try reduces all its scalars in one all-reduce (enqueue_try)
  return allreduce_sum(p, slot, 1);   // sharded: partial sums over the rank's own factors
}

static int enqueue_linearize(b200_problem* p) {
  if (p->linear) return B200_OK;   // a linear problem is its own linearization (b200_linear_create / b200_linear_update)
  cudaStream_t st = p->ctx->stream;
  for (auto& g : p->groups) {
    if (!g.count) continue;
    // tiny groups (a handful of priors) are pure launch latency: timed apart from the bandwidth kernels
    PhaseScope ps(p, g.count >= 4096 ? PH_LINEARIZE : PH_LINEARIZE_MINOR);
    const int nb = (int)((g.count + 127) / 128);
    const bool proj = g.type == B200_FACTOR_PROJECTION_CAL3S2 || g.type == B200_FACTOR_SFM_BUNDLER;
    if (proj && p->lin_variant == 4) {        // 128-register build of the two projection evaluators (no spills, 4 CTAs per SM)
      if (g.type == B200_FACTOR_PROJECTION_CAL3S2)
        DISPATCH_JT(p, launch_k(linearize_kernel<B200_FACTOR_PROJECTION_CAL3S2, JT, 4>, dim3(nb), dim3(128), 0, st, view(g), ectx(p, p->d_values)));
      else
        DISPATCH_JT(p, launch_k(linearize_kernel<B200_FACTOR_SFM_BUNDLER, JT, 4>, dim3(nb), dim3(128), 0, st, view(g), ectx(p, p->d_values)));
    } else
    DISPATCH_JT(p, DISPATCH_TYPE(g.type, (launch_k(linearize_kernel<TY, JT>, dim3(nb), dim3(128), 0, st, view(g), ectx(p, p->d_values)))));
    p->ctx->launches++;
  }
  B200_CUDA(cudaGetLastError());
  p->linearized = true;
  p->hdiag_valid = false;
  return B200_OK;
}

static int enqueue_hdiag(b200_problem* p) {
  cudaStream_t st = p->ctx->stream;
  B200_CUDA(cudaMemsetAsync(p->d_hdiag, 0, (size_t)p->ndelta * sizeof(double), st));
  for (auto& g : p->groups) {
    if (!g.count) continue;
    const int nb = (int)((g.count + 127) / 128);
    if (g.type == B200_FACTOR_JACOBIAN) launch_k(hdiag_jacobian_kernel, dim3(nb), dim3(128), 0, st, jview(g), (const int*)p->d_var_dof, p->d_hdiag);
    else if (g.type == B200_FACTOR_HESSIAN) launch_k(hdiag_hessian_kernel, dim3(nb), dim3(128), 0, st, jview(g), (const int*)p->d_var_dof, p->d_hdiag);
    else DISPATCH_JT(p, DISPATCH_TYPE(g.type, (launch_k(hdiag_kernel<TY, JT>, dim3(nb), dim3(128), 0, st, view(g), p->d_var_dof, p->d_hdiag))));
    p->ctx->launches++;
  }
  B200_CUDA(cudaGetLastError());
  return allreduce_sum(p, p->d_hdiag, (size_t)p->ndelta);
}

// assemble + damp + eliminate + back-substitute + linear errors; no host sync
// lambda lives in p->d_lambda (written by the caller); `damped` only says whether lambda > 0 may occur
static int enqueue_solve(b200_problem* p, bool damped, int diagonal, double min_diag, double max_diag) {
  cudaStream_t st = p->ctx->stream;
  b200_ctx* ctx = p->ctx;
  const TreeView t = tview(p);
  {
    PhaseScope ps(p, PH_MEMSET);
    if (p->zero_doubles) B200_CUDA(cudaMemsetAsync(p->d_arena, 0, (size_t)p->zero_doubles * sizeof(double), st));
    if (p->df_sync_ints) B200_CUDA(cudaMemsetAsync(p->d_df_sync, 0, (size_t)p->df_sync_ints * sizeof(int), st));
    if (p->topx_doubles && p->d_topx) B200_CUDA(cudaMemsetAsync(p->d_topx, 0, (size_t)p->topx_doubles * sizeof(double), st));
  }
  {
    PhaseScope ps(p, PH_ASSEMBLE);
    for (auto& g : p->groups) {
      if (!g.n_nonleaf) continue;   // every factor of the group is owned by a fused leaf clique
      const int nb = (int)((g.count + 127) / 128);
      if (g.type == B200_FACTOR_JACOBIAN) launch_k(assemble_jacobian_kernel, dim3(nb), dim3(128), 0, st, jview(g), t);
      else if (g.type == B200_FACTOR_HESSIAN) launch_k(assemble_hessian_kernel, dim3(nb), dim3(128), 0, st, jview(g), t);
      else DISPATCH_JT(p, DISPATCH_TYPE(g.type, (launch_k(assemble_kernel<TY, JT>, dim3(nb), dim3(128), 0, st, view(g), t))));
      ctx->launches++;
    }
  }
  if (damped) {
    PhaseScope ps(p, PH_DAMP);
    // hessianDiagonal depends on the linearization only: once per iterate() (b200_lm_iterate computes it right after
    // linearize, as the reference does, LevenbergMarquardtOptimizer.cpp:293-299), not once per lambda try
    if (diagonal && !p->hdiag_valid) { const int rc = enqueue_hdiag(p); if (rc) return rc; p->hdiag_valid = true; }
    launch_k(damp_kernel, dim3((int)((p->ndelta + 255) / 256)), dim3(256), 0, st, p->d_arena, p->d_diag_index, (int)p->ndelta, p->d_lambda,
                                                                diagonal ? p->d_hdiag.get() : nullptr, min_diag, max_diag);
    ctx->launches++;
  }
  if (p->n_fused) {
    PhaseScope ps(p, PH_LEAF);
    GroupTable gt;
    for (size_t gi = 0; gi < p->groups.size(); gi++) gt.g[gi] = view(p->groups[gi]);
    const double* hd = (damped && diagonal) ? p->d_hdiag.get() : nullptr;
    if (p->leaf_run_end[0] > p->leaf_run_begin[0]) {
      const int nr = p->leaf_run_end[0] - p->leaf_run_begin[0], nb = (nr + kWarpsPerBlock - 1) / kWarpsPerBlock;
      const size_t sm = (size_t)kWarpsPerBlock * p->leaf_lb_cap * sizeof(double);
      DISPATCH_JT(p, launch_k(leaf_fused_kernel<JT>, dim3(nb), dim3(kWarpsPerBlock * 32), sm, st, t, gt, p->d_fused_list, p->d_fused_run_ptr + p->leaf_run_begin[0], nr,
                                                           p->d_fused_fac_ptr, p->d_fused_fac, p->d_lambda, hd, min_diag, max_diag,
                                                           p->d_scalars, p->leaf_lb_cap, 0));
      ctx->launches++;
    }
    // BAL points.  schur_mma (default): one CTA per run of points with the same cameras factors the run's points and adds
    // their Schur complement into the parent on the FP64 tensor path, in one kernel
    for (int kd = 1; kd <= 2 && p->schur_mma; kd++) {
      const int nr = p->leaf_run_end[kd] - p->leaf_run_begin[kd];
      if (nr <= 0) continue;
      const int* runs = p->d_fused_run_ptr + p->leaf_run_begin[kd];
      const int dc = kd == 1 ? 6 : 9, maxw = p->leaf_max_w[kd], nt8 = (maxw + 7) / 8;
      const int mmax = std::max(1, (maxw - 1) / dc), sa = (dc < 8 ? 8 : 16) * kSmPA + kSmPadA;
      const size_t jb = p->jac_f32 ? sizeof(float) : sizeof(double);
      // leaf_point_fused_mma_kernel's layout: per warp [R S' d']^T, then per warp [A_c b]^T (two buffers) and A_p (two
      // buffers); the four warps' Schur sums (8 nt8)^2 reuse it at the end
      const size_t sm = std::max((size_t)4 * (3 + 8 * nt8) * kSmKS * sizeof(double) + (size_t)4 * (2 * mmax * sa + 2 * 6 * 32) * jb,
                                 (size_t)64 * nt8 * nt8 * sizeof(double));
      bool done = false;
#define B200_LAUNCH_FUSED(DC_, T_)                                                                                                    \
      if (!done && dc == DC_ && nt8 <= T_) {                                                                                          \
        DISPATCH_JT(p, launch_k(leaf_point_fused_mma_kernel<DC_, T_, JT>, dim3(nr), dim3(128), sm, st, t, gt, (const int*)p->d_fused_list, runs, \
                 (const double*)p->d_lambda, hd, min_diag, max_diag, p->d_scalars, (const int2*)p->d_pt_tab, (const int64_t*)p->d_pt_off)); \
        done = true;                                                                                                                  \
      }
      B200_LAUNCH_FUSED(6, 4) B200_LAUNCH_FUSED(6, 5) B200_LAUNCH_FUSED(6, 7)
      B200_LAUNCH_FUSED(9, 4) B200_LAUNCH_FUSED(9, 5) B200_LAUNCH_FUSED(9, 7) B200_LAUNCH_FUSED(9, 10)
#undef B200_LAUNCH_FUSED
      if (!done) { set_error("leaf_point_fused_mma_kernel: separator wider than the compiled tile counts"); return B200_CUDA_ERROR; }
      ctx->launches++;
    }
    // schur_mma = 0: per-point factorisation (8 lanes per point) ...
    for (int kd = 1; kd <= 2 && !p->schur_mma; kd++) {
      if (p->leaf_run_end[kd] <= p->leaf_run_begin[kd]) continue;
      const int i0 = p->leaf_pos_begin[kd], i1 = p->leaf_pos_end[kd];
      const int nb = (int)(((int64_t)(i1 - i0) * 8 + 127) / 128);
#define B200_LAUNCH_POINT(DC_)                                                                                                        \
      DISPATCH_JT(p, launch_k(leaf_point_factor_kernel<DC_, JT>, dim3(nb), dim3(128), 0, st, t, gt, (const int*)p->d_fused_list, i0, i1, \
               (const int*)p->d_fused_fac_ptr, (const int2*)p->d_fused_fac, (const double*)p->d_lambda, hd, min_diag, max_diag,        \
               p->d_scalars, (const int2*)p->d_pt_tab, (const int64_t*)p->d_pt_off));
      if (kd == 1) { B200_LAUNCH_POINT(6) } else { B200_LAUNCH_POINT(9) }
#undef B200_LAUNCH_POINT
      ctx->launches++;
    }
  }
  if (p->n_fused && !p->schur_mma) {
    // ... then one CTA per run of points with the same cameras for the Schur complement (3x3 FMA tiles)
    PhaseScope ps(p, PH_LEAF_SCHUR);
    GroupTable gt;
    for (size_t gi = 0; gi < p->groups.size(); gi++) gt.g[gi] = view(p->groups[gi]);
    for (int kd = 1; kd <= 2; kd++) {
      const int nr = p->leaf_run_end[kd] - p->leaf_run_begin[kd];
      if (nr <= 0) continue;
      const int* runs = p->d_fused_run_ptr + p->leaf_run_begin[kd];
      // CTA shape from the widest separator of the kind: 3x3 tiles over (s+1)^2 / 2
      const int ntd = (p->leaf_max_w[kd] + 2) / 3, ntiles = ntd * (ntd + 1) / 2;
      const int thr = ntiles <= 96 ? 96 : 128, tpt = (ntiles + thr - 1) / thr;
#define B200_LAUNCH_SCHUR(DC_, T_, P_)                                                                                               \
      if (kd == (DC_ == 6 ? 1 : 2) && tpt == T_ && p->schur_pb == P_)                                                                \
        DISPATCH_JT(p, launch_k(leaf_point_schur_kernel<DC_, T_, P_, JT>, dim3(nr), dim3(thr), 0, st, t, gt, (const int*)p->d_fused_list, runs, \
                 (const int*)p->d_fused_fac_ptr, (const int2*)p->d_fused_fac));
      // (6-dof cameras: at most kPtMaxObs * 6 + 1 = 49 columns = 153 tiles = 2 per thread; 9-dof: 73 columns = 325 tiles = 3)
      if (tpt > (kd == 1 ? 2 : 3)) { set_error("leaf_point_schur_kernel: separator wider than the compiled tile counts"); return B200_CUDA_ERROR; }
      B200_LAUNCH_SCHUR(6, 1, 4) B200_LAUNCH_SCHUR(6, 2, 4)
      B200_LAUNCH_SCHUR(6, 1, 6) B200_LAUNCH_SCHUR(6, 2, 6)
      B200_LAUNCH_SCHUR(9, 1, 4) B200_LAUNCH_SCHUR(9, 2, 4) B200_LAUNCH_SCHUR(9, 3, 4)
      B200_LAUNCH_SCHUR(9, 1, 6) B200_LAUNCH_SCHUR(9, 2, 6) B200_LAUNCH_SCHUR(9, 3, 6)
#undef B200_LAUNCH_SCHUR
      ctx->launches++;
    }
  }
  // ---- elimination, leaves to roots ----
  for (size_t l = 0; l < p->levels.size(); l++) {
    if ((int)l == p->n_sub_levels && ctx->world > 1 && !p->top_staged) {
      // SURVEY §8e: the one exchange step of the solve — every rank has eliminated its own subtrees
      // into its copy of the shared top fronts; sum them (NCCL over NVLink, in place, on-stream)
      PhaseScope ps(p, PH_ALLREDUCE);
      const int rc = allreduce_sum(p, p->d_arena, (size_t)p->top_doubles);
      if (rc) return rc;
    }
    const LevelPlan& L = p->levels[l];
    auto launch_df = [&](int slot, const int4* tasks, int ntasks, bool trace) {
      DfView v;
      v.tasks = tasks; v.ntasks = ntasks;
      v.ctrl = p->d_df_sync + 2 * slot; v.done = p->d_df_sync + p->df_ctrl_ints; v.flags = v.done + p->sym.ncliques;
      v.flag_off = p->d_df_flag_off; v.expect = p->d_df_expect;
      v.trace = trace ? p->d_df_trace.get() : nullptr;
      v.winv = p->d_winv; v.winv_off = p->d_winv_off;
      v.warm_ctas = getenv("B200_DF_NO_WARM") ? 0 : 3 * ctx->sm_count;
      if (p->df_minb == 3) launch_k(front_df_kernel<3>, dim3(ntasks), dim3(kDfThreads), (size_t)kDfSmemBytes, st, t, v, p->d_scalars);
      else launch_k(front_df_kernel<2>, dim3(ntasks), dim3(kDfThreads), (size_t)kDfSmemBytes, st, t, v, p->d_scalars);
      ctx->launches++;
    };
    for (int ph = 0; ph < 2; ph++)
      if ((int)l == p->df_level[ph] && p->df_ntasks[ph] && !(ph == 1 && p->top_staged)) {
        // every remaining non-leaf front of the phase, all levels, as one tile dataflow (front_df.cuh)
        PhaseScope ps(p, PH_ELIM_LARGE);
        launch_df(ph, p->d_df_tasks[ph], p->df_ntasks[ph], ph == 0);
      }
    if (p->top_staged)
      for (size_t s = 0; s < p->ts_level.size(); s++)
        if (p->ts_level[s] == (int)l) {
          {
            // SURVEY 8e, the exchange step, per top level: every rank's partial copy of the level's fronts (the Schur
            // complements of its own subtrees and of the top fronts it owns below) is summed onto the front's owner
            PhaseScope ps(p, PH_ALLREDUCE);
            const int rc = reduce_top_stage(p, s);
            if (rc) return rc;
          }
          if (p->ts_task_count[s]) {
            PhaseScope ps(p, PH_ELIM_LARGE);
            launch_df(2 + (int)s, p->d_df_tasks[1] + p->ts_task_begin[s], p->ts_task_count[s], false);
          }
        }
    if (L.small_count) {
      PhaseScope ps(p, PH_ELIM_SMALL);
      const int nb = (L.small_count + kWarpsPerBlock - 1) / kWarpsPerBlock;
      const size_t smem = (size_t)kWarpsPerBlock * p->max_small_n * p->max_small_n * sizeof(double);
      launch_k(elim_small_kernel, dim3(nb), dim3(kWarpsPerBlock * 32), smem, st, t, p->d_lvl_small + L.small_begin, L.small_count,
                                                               p->max_small_n, p->d_scalars);
      ctx->launches++;
    }
  }
  // ---- back-substitution, roots to leaves ----
  if (p->n_bs_flags) B200_CUDA(cudaMemsetAsync(p->d_bs_flags, 0, (size_t)p->n_bs_flags * sizeof(int), st));
  {
  PhaseScope ps(p, PH_BACKSUB);
  for (int l = (int)p->levels.size() - 1; l >= 0; l--) {
    const LevelPlan& L = p->levels[l];
    if (L.blarge_count) {
      const int nblk = (L.blarge_max_nf + kBsRows - 1) / kBsRows;
      launch_k(backsub_large_kernel, dim3(dim3(nblk, L.blarge_count)), dim3(256), 0, st, t, p->d_lvl_blarge + L.blarge_begin, p->d_delta, p->d_scalars,
                                                                      p->d_bs_flags, p->d_bs_flag_base, L.blarge_begin, 1,
                                                                      (const double*)p->d_winv, (const int64_t*)p->d_winv_off);
      ctx->launches++;
    }
    if (L.bsmall_count) {
      const int nb = (L.bsmall_count + kWarpsPerBlock - 1) / kWarpsPerBlock;
      launch_k(backsub_small_kernel, dim3(nb), dim3(kWarpsPerBlock * 32), 0, st, t, p->d_lvl_bsmall + L.bsmall_begin, L.bsmall_count,
                                                               p->d_delta, p->d_scalars);
      ctx->launches++;
    }
    if (p->top_staged)
      for (size_t s = 0; s < p->ts_level.size(); s++)
        if (p->ts_level[s] == l) {
          // the owners' solutions of this top level -> packed vector -> one small all-reduce (zeros from the others) -> delta everywhere
          PhaseScope px(p, PH_TOPX);    // (inside the back_substitute scope: counted in both)
          const int nfr = p->ts_begin[s + 1] - p->ts_begin[s];
          launch_k(top_x_kernel, dim3(nfr), dim3(128), 0, st, t, (const int*)(p->d_ts_cliques + p->ts_begin[s]), (const int*)(p->d_ts_xoff + p->ts_begin[s]),
                   (const int*)(p->d_ts_owned + p->ts_begin[s]), p->d_delta, p->d_topx, 0);
          const int rc = allreduce_sum(p, p->d_topx + p->ts_x_begin[s], (size_t)p->ts_x_count[s]);
          if (rc) return rc;
          launch_k(top_x_kernel, dim3(nfr), dim3(128), 0, st, t, (const int*)(p->d_ts_cliques + p->ts_begin[s]), (const int*)(p->d_ts_xoff + p->ts_begin[s]),
                   (const int*)(p->d_ts_owned + p->ts_begin[s]), p->d_delta, p->d_topx, 1);
          ctx->launches += 2;
        }
    for (int kd = 0; kd < 2; kd++) {
      if (!L.bpoint_count[kd]) continue;
      const int nb = (int)(((int64_t)L.bpoint_count[kd] * 8 + 127) / 128);
      const int* lst = p->d_lvl_bpoint + L.bpoint_begin[kd];
      if (kd == 0) launch_k(backsub_point_kernel<6>, dim3(nb), dim3(128), 0, st, t, lst, L.bpoint_count[kd], p->d_delta, p->d_scalars);
      else launch_k(backsub_point_kernel<9>, dim3(nb), dim3(128), 0, st, t, lst, L.bpoint_count[kd], p->d_delta, p->d_scalars);
      ctx->launches++;
    }
  }
  }
  // ---- linear errors on the undamped graph ----
  PhaseScope pl(p, PH_LINERR);
  bool first = true;
  for (auto& g : p->groups) {
    if (!g.count) continue;
    const int nb = reduce_blocks(g.count, 256, ctx->sm_count);
    double* p0 = p->d_partials;
    double* p1 = p->d_partials + p->partial_cap / 2;
    if (g.type == B200_FACTOR_JACOBIAN)
      launch_k(linerr_jacobian_kernel, dim3(nb), dim3(256), 0, st, jview(g), (const double*)p->d_delta, (const int*)p->d_var_dof, p0, p1, p->d_counters + 1,
               &p->d_scalars->lin_err0, &p->d_scalars->lin_err_delta, first ? 0 : 1, 1.0);
    else if (g.type == B200_FACTOR_HESSIAN)
      launch_k(linerr_hessian_kernel, dim3(nb), dim3(256), 0, st, jview(g), (const double*)p->d_delta, (const int*)p->d_var_dof, p0, p1, p->d_counters + 1,
               &p->d_scalars->lin_err0, &p->d_scalars->lin_err_delta, first ? 0 : 1, 1.0);
    else
    DISPATCH_JT(p, DISPATCH_TYPE(g.type, (launch_k(linerr_kernel<TY, JT>, dim3(nb), dim3(256), 0, st, view(g), p->d_delta, p->d_var_dof, p0, p1, p->d_counters + 1,
                                                                 &p->d_scalars->lin_err0, &p->d_scalars->lin_err_delta, first ? 0 : 1, 1.0))));
    ctx->launches += 1;
    first = false;
  }
  if (first) B200_CUDA(cudaMemsetAsync(&p->d_scalars->lin_err0, 0, 2 * sizeof(double), st));
  B200_CUDA(cudaGetLastError());
  if (ctx->world > 1 && !p->defer_scalar_reduce) {
    int rc = allreduce_sum(p, &p->d_scalars->lin_err0, 2);          // lin_err0, lin_err_delta are adjacent
    if (rc) return rc;
    rc = allreduce_max_int(p, &p->d_scalars->fail_code, 2);          // every rank takes the same decision
    if (rc) return rc;
  }
  p->solved = true;
  p->factored = true;
  p->marg_ready = !damped;   // an undamped factor of H at the current values: what Marginals needs
  return B200_OK;
}

static int enqueue_try_step(b200_problem* p) {
  cudaStream_t st = p->ctx->stream;
  {
    PhaseScope ps(p, PH_RETRACT);
    launch_k(retract_kernel, dim3((int)((p->nvars + 127) / 128)), dim3(128), 0, st, p->d_values, p->d_delta, p->d_val_off, p->d_var_dof,
                                                                   p->d_var_type, (int)p->nvars, p->d_new_values);
    p->ctx->launches++;
  }
  return enqueue_error(p, p->d_new_values, &p->d_scalars->new_error);
}

static int reset_flags(b200_problem* p) {
  B200_CUDA(cudaMemsetAsync(&p->d_scalars->fail_code, 0, 4 * sizeof(int), p->ctx->stream));   // fail, nan, df_abort, pad
  return B200_OK;
}
static int set_lambda(b200_problem* p, double lambda) {
  *p->h_lambda = lambda;
  B200_CUDA(cudaMemcpyAsync(p->d_lambda, p->h_lambda, sizeof(double), cudaMemcpyHostToDevice, p->ctx->stream));
  return B200_OK;
}
static int fetch_scalars(b200_problem* p) {
  B200_CUDA(cudaMemcpyAsync(p->h_scalars, p->d_scalars, sizeof(Scalars), cudaMemcpyDeviceToHost, p->ctx->stream));
  B200_CUDA(cudaStreamSynchronize(p->ctx->stream));
  if (p->profile) resolve_profile(p);
  return B200_OK;
}
static int solve_status(const b200_problem* p, int64_t* fail_var) {
  const Scalars* s = p->h_scalars;
  if (s->df_abort) { set_error("front_df_kernel: a dependency wait timed out (internal scheduling error)"); return B200_CUDA_ERROR; }
  // a failed factorisation poisons everything below it: report the Cholesky failure first
  const int code = s->fail_code ? s->fail_code : s->nan_code;
  if (code == 0) { if (fail_var) *fail_var = -1; return B200_OK; }
  const int c = INT_MAX - code;
  if (fail_var) *fail_var = p->sym.front_vars[p->sym.front_ptr[c]];
  return B200_INDETERMINATE;
}

// Validation of a problem description + the symbolic phase.  Host only: needs
// no GPU, so it is also exposed through b200_symbolic_create for CPU tests.
struct PackedGroup {
  int type, noise_kind = 0, per_factor = 0, noise_size = 0, d, ncols, arity, meas = 0, robust_kind = 0;
  double robust_param = 0;
  int64_t count;
  std::vector<int64_t> pos;   // graph position of every factor of the group
  int dims[B200_JACOBIAN_MAX_ARITY] = {0};   // block widths (groups of a linear problem)
};
struct Packed {
  std::vector<int> val_off, var_dof, var_dim;
  std::vector<int64_t> fptr, fkeys;   // CSR of the keys of every factor by graph position
  std::vector<PackedGroup> groups;
  int64_t total = 0;
  Symbolic sym;
};
// graph positions of a group (explicit list, or a consecutive run) + overlap / range checks
static int resolve_positions(int64_t count, const int64_t* graph_index, int64_t graph_index0, int64_t total, int64_t* next,
                             std::vector<char>* used, std::vector<int64_t>* pos) {
  if (count < 0) { set_error("negative factor count"); return B200_INVALID_ARGUMENT; }
  if (count > INT_MAX / 2) { set_error("factor group too large"); return B200_INVALID_ARGUMENT; }
  pos->resize(count);
  if (graph_index) {
    for (int64_t i = 0; i < count; i++) (*pos)[i] = graph_index[i];
  } else {
    const int64_t gi0 = graph_index0 < 0 ? *next : graph_index0;
    for (int64_t i = 0; i < count; i++) (*pos)[i] = gi0 + i;
    *next = gi0 + count;
  }
  for (int64_t i = 0; i < count; i++) {
    const int64_t q = (*pos)[i];
    if (q < 0 || q >= total) { set_error("graph position out of range"); return B200_INVALID_ARGUMENT; }
    if ((*used)[q]) { set_error("overlapping graph positions"); return B200_INVALID_ARGUMENT; }
    (*used)[q] = 1;
  }
  return B200_OK;
}
static int pack_and_symbolic(const b200_problem_desc* d, Packed* pk) {
#define FAIL(code, msg) do { set_error(msg); return code; } while (0)
  if (!d || d->nvars < 0 || d->ngroups < 0) FAIL(B200_INVALID_ARGUMENT, "bad problem description");
  const int64_t n = d->nvars;
  pk->val_off.assign(n + 1, 0); pk->var_dof.assign(n + 1, 0); pk->var_dim.assign(n, 0);
  for (int64_t v = 0; v < n; v++) {
    const int t = d->var_type[v];
    if (t < 0 || t >= B200_NUM_VAR_TYPES) FAIL(B200_INVALID_ARGUMENT, "unknown variable type");
    pk->var_dim[v] = VAR_DIM[t];
    pk->val_off[v + 1] = pk->val_off[v] + VAR_STORAGE[t];
    pk->var_dof[v + 1] = pk->var_dof[v] + VAR_DIM[t];
  }
  int64_t total = 0, next = 0;
  for (int64_t g = 0; g < d->ngroups; g++) {
    if (d->groups[g].count < 0) FAIL(B200_INVALID_ARGUMENT, "negative factor count");
    total += d->groups[g].count;
  }
  pk->total = total;
  std::vector<char> used(total, 0);
  pk->groups.resize(d->ngroups);
  pk->fptr.assign(total + 1, 0);
  for (int64_t gi = 0; gi < d->ngroups; gi++) {   // pass 1: graph positions and arities -> CSR offsets
    const b200_factor_group& s = d->groups[gi];
    if (s.type < 0 || s.type >= B200_NUM_FACTOR_TYPES) FAIL(B200_UNSUPPORTED_FACTOR, "unsupported factor type");
    const int rc = resolve_positions(s.count, s.graph_index, s.graph_index0, total, &next, &used, &pk->groups[gi].pos);
    if (rc) return rc;
    for (int64_t i = 0; i < s.count; i++) pk->fptr[pk->groups[gi].pos[i] + 1] = F_ARITY[s.type];
  }
  for (int64_t i = 0; i < total; i++) pk->fptr[i + 1] += pk->fptr[i];
  pk->fkeys.assign(pk->fptr[total], -1);
  for (int64_t gi = 0; gi < d->ngroups; gi++) {
    const b200_factor_group& s = d->groups[gi];
    PackedGroup& g = pk->groups[gi];
    g.type = s.type; g.noise_kind = s.noise_kind; g.per_factor = s.noise_per_factor; g.count = s.count;
    g.d = F_DIM[s.type]; g.arity = F_ARITY[s.type]; g.meas = F_MEAS[s.type];
    g.ncols = VAR_DIM[F_VT[s.type][0]] + (g.arity == 2 ? VAR_DIM[F_VT[s.type][1]] : 0) + 1;
    g.noise_size = noise_payload(s.noise_kind, g.d);
    if (g.noise_size < 0) FAIL(B200_UNSUPPORTED_NOISE, "unsupported noise model (Constrained models need QR: out of scope)");
    g.robust_kind = s.robust_kind; g.robust_param = s.robust_param;
    if (s.robust_kind < 0 || s.robust_kind > B200_ROBUST_FAIR || (s.robust_kind && !(s.robust_param > 0)))
      FAIL(B200_UNSUPPORTED_NOISE, "unknown robust loss or non-positive parameter");
    if (s.robust_kind && s.type == B200_FACTOR_SFM_BUNDLER)
      FAIL(B200_UNSUPPORTED_NOISE, "GeneralSFMFactor::linearize whitens without reweighting: Robust models are not supported on it");
    for (int64_t i = 0; i < s.count; i++) {
      for (int a = 0; a < g.arity; a++) {
        const int64_t k = s.keys[i * g.arity + a];
        if (k < 0 || k >= n || d->var_type[k] != F_VT[s.type][a])
          FAIL(B200_INVALID_ARGUMENT, "factor key missing or of the wrong value type (ValuesKeyDoesNotExist / ValuesIncorrectType)");
        pk->fkeys[pk->fptr[g.pos[i]] + a] = k;
      }
    }
    if (s.type == B200_FACTOR_PROJECTION_CAL3S2) {
      if (d->ncal < 1) FAIL(B200_INVALID_ARGUMENT, "projection factors need a calibration");
      if (s.cal_index)
        for (int64_t i = 0; i < s.count; i++)
          if (s.cal_index[i] < 0 || s.cal_index[i] >= d->ncal) FAIL(B200_INVALID_ARGUMENT, "calibration index out of range");
    }
  }
  const char* serr = "";
  if (!build_symbolic(n, pk->var_dim.data(), d->ordering, total, pk->fptr.data(), pk->fkeys.data(), &pk->sym, &serr))
    FAIL(B200_INVALID_ARGUMENT, serr);
  return B200_OK;
}

// The same for a linear description (b200_linear_create): JacobianFactor groups of any arity.
static int pack_linear(const b200_linear_desc* d, Packed* pk) {
  if (!d || d->nvars < 0 || d->ngroups < 0 || d->nhgroups < 0) FAIL(B200_INVALID_ARGUMENT, "bad linear description");
  const int64_t n = d->nvars;
  pk->val_off.assign(n + 1, 0); pk->var_dof.assign(n + 1, 0); pk->var_dim.assign(n, 0);
  for (int64_t v = 0; v < n; v++) {
    if (d->var_dim[v] < 1) FAIL(B200_INVALID_ARGUMENT, "variable dimension < 1");
    pk->var_dim[v] = d->var_dim[v];
    if ((int64_t)pk->var_dof[v] + d->var_dim[v] > INT_MAX / 2) FAIL(B200_INVALID_ARGUMENT, "total dimension too large");
    pk->var_dof[v + 1] = pk->var_dof[v] + d->var_dim[v];
  }
  int64_t total = 0, next = 0;
  for (int64_t g = 0; g < d->ngroups; g++) {
    if (d->groups[g].count < 0) FAIL(B200_INVALID_ARGUMENT, "negative factor count");
    total += d->groups[g].count;
  }
  for (int64_t g = 0; g < d->nhgroups; g++) {
    if (d->hgroups[g].count < 0) FAIL(B200_INVALID_ARGUMENT, "negative factor count");
    total += d->hgroups[g].count;
  }
  pk->total = total;
  std::vector<char> used(total, 0);
  pk->groups.resize(d->ngroups + d->nhgroups);
  pk->fptr.assign(total + 1, 0);
  for (int64_t gi = 0; gi < d->ngroups; gi++) {
    const b200_jacobian_group& s = d->groups[gi];
    PackedGroup& g = pk->groups[gi];
    if (s.arity < 1 || s.arity > B200_JACOBIAN_MAX_ARITY) FAIL(B200_UNSUPPORTED_FACTOR, "JacobianFactor arity outside 1..B200_JACOBIAN_MAX_ARITY");
    if (s.rows < 0) FAIL(B200_INVALID_ARGUMENT, "negative row count");
    g.type = B200_FACTOR_JACOBIAN; g.d = s.rows; g.arity = s.arity; g.count = s.count;
    g.ncols = 1;
    for (int a = 0; a < s.arity; a++) {
      if (s.dims[a] < 1) FAIL(B200_INVALID_ARGUMENT, "block width < 1");
      g.dims[a] = s.dims[a];
      g.ncols += s.dims[a];
    }
    const int rc = resolve_positions(s.count, s.graph_index, s.graph_index0, total, &next, &used, &g.pos);
    if (rc) return rc;
    for (int64_t i = 0; i < s.count; i++) pk->fptr[g.pos[i] + 1] = s.arity;
    if (s.sigmas)
      for (int64_t i = 0; i < s.count * s.rows; i++)
        if (!(s.sigmas[i] > 0)) FAIL(B200_UNSUPPORTED_NOISE, "sigma <= 0: Constrained noise models need QR elimination (out of scope)");
  }
  for (int64_t hi = 0; hi < d->nhgroups; hi++) {   // HessianFactor groups follow the Jacobian groups
    const b200_hessian_group& s = d->hgroups[hi];
    PackedGroup& g = pk->groups[d->ngroups + hi];
    if (s.arity < 1 || s.arity > B200_JACOBIAN_MAX_ARITY) FAIL(B200_UNSUPPORTED_FACTOR, "HessianFactor arity outside 1..B200_JACOBIAN_MAX_ARITY");
    g.type = B200_FACTOR_HESSIAN; g.arity = s.arity; g.count = s.count;
    g.ncols = 1;
    for (int a = 0; a < s.arity; a++) {
      if (s.dims[a] < 1) FAIL(B200_INVALID_ARGUMENT, "block width < 1");
      g.dims[a] = s.dims[a];
      g.ncols += s.dims[a];
    }
    g.d = g.ncols;   // the augmented information matrix is (N+1) x (N+1)
    const int rc = resolve_positions(s.count, s.graph_index, s.graph_index0, total, &next, &used, &g.pos);
    if (rc) return rc;
    for (int64_t i = 0; i < s.count; i++) pk->fptr[g.pos[i] + 1] = s.arity;
  }
  for (int64_t i = 0; i < total; i++) pk->fptr[i + 1] += pk->fptr[i];
  pk->fkeys.assign(pk->fptr[total], -1);
  for (int64_t hi = 0; hi < d->nhgroups; hi++) {
    const b200_hessian_group& s = d->hgroups[hi];
    const PackedGroup& g = pk->groups[d->ngroups + hi];
    for (int64_t i = 0; i < s.count; i++)
      for (int a = 0; a < s.arity; a++) {
        const int64_t k = s.keys[i * s.arity + a];
        if (k < 0 || k >= n) FAIL(B200_INVALID_ARGUMENT, "HessianFactor key out of range");
        if (d->var_dim[k] != s.dims[a]) FAIL(B200_INVALID_ARGUMENT, "HessianFactor block width differs from the variable's dimension");
        pk->fkeys[pk->fptr[g.pos[i]] + a] = k;
      }
  }
  for (int64_t gi = 0; gi < d->ngroups; gi++) {
    const b200_jacobian_group& s = d->groups[gi];
    const PackedGroup& g = pk->groups[gi];
    for (int64_t i = 0; i < s.count; i++)
      for (int a = 0; a < s.arity; a++) {
        const int64_t k = s.keys[i * s.arity + a];
        if (k < 0 || k >= n) FAIL(B200_INVALID_ARGUMENT, "JacobianFactor key out of range");
        if (d->var_dim[k] != s.dims[a]) FAIL(B200_INVALID_ARGUMENT, "JacobianFactor block width differs from the variable's dimension");
        pk->fkeys[pk->fptr[g.pos[i]] + a] = k;
      }
  }
  const char* serr = "";
  if (!build_symbolic(n, pk->var_dim.data(), d->ordering, total, pk->fptr.data(), pk->fkeys.data(), &pk->sym, &serr))
    FAIL(B200_INVALID_ARGUMENT, serr);
#undef FAIL
  return B200_OK;
}

// ---- sharding plan (SURVEY §8e) ------------------------------------------------------
// Which leaf cliques take the fused path; which cliques form the replicated TOP of the junction
// tree; which rank owns every other clique.  The top T is ancestor-closed: starting from the
// roots, the heaviest subtree root is moved into T and replaced by its children until every
// remaining subtree is lighter than total/(4*world) (for BAL with Schur ordering T ends up being
// the camera cliques and the subtrees the points; for nested-dissection orderings T is the top
// separators and the subtrees the ND branches).  The remaining subtrees are assigned to ranks
// in clique order by prefix weight (keeps neighbouring leaves, and their shared separators,
// together).  Factors follow the clique that owns them; factors of top cliques belong to rank 0.
static void shard_plan(const Symbolic& S, int64_t ngroups, int64_t total, int world, std::vector<char>* fused,
                       std::vector<char>* is_top, std::vector<int>* clique_owner, std::vector<int>* factor_owner,
                       bool allow_leaf = true, std::vector<int>* top_owner = nullptr) {
  // the fused leaf kernels evaluate typed factor groups: never for the JacobianFactor groups of a linear problem
  const bool leaf_path = allow_leaf && ngroups <= kMaxGroups && !getenv("B200_NO_LEAF_FUSION");
  const int64_t nc = S.ncliques;
  fused->assign(nc, 0);
  for (int64_t c = 0; c < nc; c++) {
    const int64_t nn = S.nf[c] + S.ns[c] + 1;
    if (leaf_path && S.level[c] == 0 && S.nf[c] <= kLeafMaxF && (int64_t)S.nf[c] * nn <= kLeafMaxFN) (*fused)[c] = 1;
  }
  is_top->assign(nc, 0);
  clique_owner->assign(nc, 0);
  if (world > 1) {
    std::vector<int64_t> nfac(nc, 0);
    for (int64_t pos = 0; pos < total; pos++) nfac[S.fac_clique[pos]]++;
    std::vector<double> w(nc, 0.0);
    std::vector<int64_t> ch_ptr(nc + 1, 0);
    for (int64_t c = 0; c < nc; c++) if (S.parent[c] >= 0) ch_ptr[S.parent[c] + 1]++;
    for (int64_t c = 0; c < nc; c++) ch_ptr[c + 1] += ch_ptr[c];
    std::vector<int64_t> ch(ch_ptr[nc]), cur(ch_ptr.begin(), ch_ptr.end() - 1);
    for (int64_t c = 0; c < nc; c++) if (S.parent[c] >= 0) ch[cur[S.parent[c]]++] = c;
    double sum = 0;
    for (int64_t c = 0; c < nc; c++) {   // children have smaller ids than parents
      const double nn = S.nf[c] + S.ns[c] + 1;
      w[c] += nn * nn * (S.nf[c] + 1) + 200.0 * (double)nfac[c];
      if (S.parent[c] >= 0) w[S.parent[c]] += w[c]; else sum += w[c];
    }
    // Subtrees lighter than total / (top_factor * world).  A deeper top balances better; a shallower one has fewer levels —
    // each a communication stage of the distributed top — and less of the tree in the exchanged region.  So: the shallowest top whose
    // busiest rank stays within 20 % of the mean subtree load, deepening by 1.5x at a time (B200_TOP_FACTOR pins it).
    std::vector<int> assigned(nc, 0);
    const double pinned = getenv("B200_TOP_FACTOR") ? atof(getenv("B200_TOP_FACTOR")) : 0.0;
    for (double top_factor = pinned > 0 ? pinned : 1.0;; top_factor *= 1.5) {
    is_top->assign(nc, 0);
    std::fill(assigned.begin(), assigned.end(), 0);
    const double target = sum / (top_factor * world);
    std::vector<std::pair<double, int64_t>> heap;
    for (int64_t c = 0; c < nc; c++) if (S.parent[c] < 0) heap.push_back({w[c], c});
    std::make_heap(heap.begin(), heap.end());
    while (!heap.empty()) {
      const auto top = heap.front();
      const int64_t c = top.second;
      if (top.first <= target || ch_ptr[c + 1] == ch_ptr[c]) break;
      std::pop_heap(heap.begin(), heap.end());
      heap.pop_back();
      (*is_top)[c] = 1;
      for (int64_t q = ch_ptr[c]; q < ch_ptr[c + 1]; q++) {
        heap.push_back({w[ch[q]], ch[q]});
        std::push_heap(heap.begin(), heap.end());
      }
    }
    std::vector<int64_t> roots;
    double subsum = 0;
    for (auto& e : heap) { roots.push_back(e.second); subsum += e.first; }
    std::sort(roots.begin(), roots.end());
    double prefix = 0;
    std::vector<double> load(world, 0.0);
    for (int64_t r : roots) {
      assigned[r] = subsum > 0 ? (int)std::min<double>(world - 1, std::floor(prefix * world / subsum)) : 0;
      prefix += w[r];
      load[assigned[r]] += w[r];
    }
    // A few heavy subtrees (nested-dissection branches, camera chains) defeat the contiguous split: if
    // longest-processing-time-first packing lowers the heaviest rank by more than 10 %, take it instead.
    // (Many equal leaves - the BAL points of the default benchmark - stay contiguous: runs of points with
    // the same cameras remain on one rank.)
    {
      std::vector<int64_t> by_w(roots);
      std::sort(by_w.begin(), by_w.end(), [&](int64_t a, int64_t b) { return w[a] != w[b] ? w[a] > w[b] : a < b; });
      std::vector<double> lpt_load(world, 0.0);
      std::vector<int> lpt(nc, 0);
      for (int64_t r : by_w) {
        const int k = (int)(std::min_element(lpt_load.begin(), lpt_load.end()) - lpt_load.begin());
        lpt[r] = k;
        lpt_load[k] += w[r];
      }
      const double worst = *std::max_element(load.begin(), load.end());
      const double worst_lpt = *std::max_element(lpt_load.begin(), lpt_load.end());
      double final_worst = worst;
      if (worst_lpt < 0.9 * worst && !getenv("B200_NO_LPT")) {
        for (int64_t r : roots) assigned[r] = lpt[r];
        final_worst = worst_lpt;
      }
      if (pinned > 0 || top_factor >= 8.0 || final_worst <= 1.2 * subsum / world) break;
    }
    }
    for (int64_t c = nc - 1; c >= 0; c--) {
      if ((*is_top)[c]) (*clique_owner)[c] = -1;
      else if (S.parent[c] < 0 || (*is_top)[S.parent[c]]) (*clique_owner)[c] = assigned[c];
      else (*clique_owner)[c] = (*clique_owner)[S.parent[c]];
    }
  }
  // owners of the top fronts: level by level (a level's fronts are independent), heaviest first onto the rank with the
  // least work so far AT THAT LEVEL (what bounds a stage is its busiest owner), ties to the globally least loaded
  if (top_owner) {
    top_owner->assign(nc, -1);
    if (world > 1) {
      std::vector<double> total_load(world, 0.0);
      for (int64_t l = 0; l < S.nlevels; l++) {
        std::vector<int64_t> at;
        for (int64_t q = S.lvl_ptr[l]; q < S.lvl_ptr[l + 1]; q++) if ((*is_top)[S.lvl_cliques[q]]) at.push_back(S.lvl_cliques[q]);
        auto wt = [&](int64_t c) { const double nn = S.nf[c] + S.ns[c] + 1; return nn * nn * (S.nf[c] + 1); };
        std::sort(at.begin(), at.end(), [&](int64_t a, int64_t b) { return wt(a) != wt(b) ? wt(a) > wt(b) : a < b; });
        std::vector<double> load(world, 0.0);
        for (int64_t c : at) {
          int best = 0;
          for (int r = 1; r < world; r++)
            if (load[r] < load[best] || (load[r] == load[best] && total_load[r] < total_load[best])) best = r;
          (*top_owner)[c] = best;
          load[best] += wt(c); total_load[best] += wt(c);
        }
      }
    }
  }
  factor_owner->assign(total, 0);
  for (int64_t pos = 0; pos < total; pos++) {
    const int o = (*clique_owner)[S.fac_clique[pos]];
    (*factor_owner)[pos] = o < 0 ? 0 : o;
  }
}

// ---- NCCL, loaded lazily so the single-GPU path never needs it ------------------------
struct NcclApi {
  void* h = nullptr;
  int (*GetUniqueId)(void*) = nullptr;
  int (*CommInitRank)(void**, int, ncclUniqueIdBlob, int) = nullptr;
  int (*AllReduce)(const void*, void*, size_t, int, int, void*, cudaStream_t) = nullptr;
  int (*Reduce)(const void*, void*, size_t, int, int, int, void*, cudaStream_t) = nullptr;
  int (*GroupStart)() = nullptr;
  int (*GroupEnd)() = nullptr;
  int (*CommDestroy)(void*) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
};
static NcclApi g_nccl;
static int nccl_load() {
  if (g_nccl.h) return B200_OK;
  void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
  if (!h) { set_error(std::string("cannot load libnccl.so.2: ") + dlerror()); return B200_NCCL_ERROR; }
  g_nccl.GetUniqueId = (int (*)(void*))dlsym(h, "ncclGetUniqueId");
  g_nccl.CommInitRank = (int (*)(void**, int, ncclUniqueIdBlob, int))dlsym(h, "ncclCommInitRank");
  g_nccl.AllReduce = (int (*)(const void*, void*, size_t, int, int, void*, cudaStream_t))dlsym(h, "ncclAllReduce");
  g_nccl.Reduce = (int (*)(const void*, void*, size_t, int, int, int, void*, cudaStream_t))dlsym(h, "ncclReduce");
  g_nccl.GroupStart = (int (*)())dlsym(h, "ncclGroupStart");
  g_nccl.GroupEnd = (int (*)())dlsym(h, "ncclGroupEnd");
  g_nccl.CommDestroy = (int (*)(void*))dlsym(h, "ncclCommDestroy");
  g_nccl.GetErrorString = (const char* (*)(int))dlsym(h, "ncclGetErrorString");
  if (!g_nccl.GetUniqueId || !g_nccl.CommInitRank || !g_nccl.AllReduce) { set_error("libnccl.so.2 lacks required symbols"); return B200_NCCL_ERROR; }
  g_nccl.h = h;
  return B200_OK;
}
enum { kNcclInt32 = 2, kNcclFloat64 = 8, kNcclSum = 0, kNcclMax = 2, kNcclMin = 3 };  // ncclDataType_t / ncclRedOp_t (nccl.h)
#define B200_NCCL(call)                                                                              \
  do {                                                                                               \
    int r_ = (call);                                                                                 \
    if (r_ != 0) {                                                                                   \
      set_error(std::string(#call) + ": " + (g_nccl.GetErrorString ? g_nccl.GetErrorString(r_) : "nccl error")); \
      return B200_NCCL_ERROR;                                                                        \
    }                                                                                                \
  } while (0)
static int allreduce_sum(b200_problem* p, double* buf, size_t n) {
  if (p->ctx->world <= 1 || n == 0) return B200_OK;
  B200_NCCL(g_nccl.AllReduce(buf, buf, n, kNcclFloat64, kNcclSum, p->ctx->comm, p->ctx->stream));
  p->ctx->launches++;
  return B200_OK;
}
// one stage of the distributed top: the ranks' partial copies of every front of the level, summed onto the front's owner
// (ncclReduce in place; one group, so the fronts of the level travel concurrently over NVLink)
static int reduce_top_stage(b200_problem* p, size_t s) {
  static const bool use_reduce = getenv("B200_TOP_REDUCE") != nullptr;
  if (!use_reduce) {
    // the level's fronts are one contiguous range of the arena: ONE all-reduce (in-switch reduction where NVSwitch offers it),
    // instead of the grouped ncclReduce onto the owners, which moves every rank's full copy along a chain
    const auto& f0 = p->ts_fronts[p->ts_begin[s]];
    const auto& f1 = p->ts_fronts[p->ts_begin[s + 1] - 1];
    return allreduce_sum(p, p->d_arena + f0.off, (size_t)(f1.off + f1.count - f0.off));
  }
  if (!g_nccl.Reduce || !g_nccl.GroupStart || !g_nccl.GroupEnd) { set_error("libnccl.so.2 lacks ncclReduce / ncclGroupStart"); return B200_NCCL_ERROR; }
  B200_NCCL(g_nccl.GroupStart());
  for (int q = p->ts_begin[s]; q < p->ts_begin[s + 1]; q++) {
    const auto& tf = p->ts_fronts[q];
    B200_NCCL(g_nccl.Reduce(p->d_arena + tf.off, p->d_arena + tf.off, (size_t)tf.count, kNcclFloat64, kNcclSum, tf.owner, p->ctx->comm, p->ctx->stream));
  }
  B200_NCCL(g_nccl.GroupEnd());
  p->ctx->launches++;
  return B200_OK;
}
static int allreduce_max_int(b200_problem* p, int* buf, size_t n) {
  if (p->ctx->world <= 1) return B200_OK;
  B200_NCCL(g_nccl.AllReduce(buf, buf, n, kNcclInt32, kNcclMax, p->ctx->comm, p->ctx->stream));
  p->ctx->launches++;
  return B200_OK;
}

// One LM try = flags reset + damped solve + (speculative) retract + error.  The launch
// sequence does not depend on lambda (device resident), so it is captured once into a CUDA
// graph per problem and replayed: ~100-300 small kernels per try would otherwise be bound by
// the host's launch rate, not by the GPU.  Eager when profiling (phase timers), when sharded
// (NCCL on-stream) or when B200_NO_GRAPH is set.
static int enqueue_try(b200_problem* p, int diagonal, double min_diag, double max_diag) {
  int rc = reset_flags(p);
  if (rc) return rc;
  // sharded: the scalars LM branches on (two linear errors, the new error, the two failure codes) travel in ONE
  // all-reduce at the end of the try instead of three latency-bound ones (a SUM over [3 doubles | one slot per rank
  // for each code]; the maximum of the slots is taken on the device afterwards)
  const bool merged = p->ctx->world > 1 && p->ctx->world <= kMaxRanksMerged && !getenv("B200_NO_MERGED_SCALARS");
  p->defer_scalar_reduce = merged;
  rc = enqueue_solve(p, true, diagonal, min_diag, max_diag);
  if (!rc) rc = enqueue_try_step(p);
  p->defer_scalar_reduce = false;
  if (rc || !merged) return rc;
  if (!p->d_red) B200_CUDA(p->d_red.alloc(3 + 2 * kMaxRanksMerged));
  cudaStream_t st = p->ctx->stream;
  launch_k(scalars_pack_kernel, dim3(1), dim3(32), 0, st, p->d_scalars, p->d_red, p->ctx->rank, p->ctx->world, 0);
  rc = allreduce_sum(p, p->d_red, (size_t)(3 + 2 * p->ctx->world));
  if (rc) return rc;
  launch_k(scalars_pack_kernel, dim3(1), dim3(32), 0, st, p->d_scalars, p->d_red, p->ctx->rank, p->ctx->world, 1);
  p->ctx->launches += 2;
  return B200_OK;
}
static int launch_try(b200_problem* p, int diagonal, double min_diag, double max_diag) {
  static const bool no_graph = getenv("B200_NO_GRAPH") != nullptr;
  if (no_graph || p->profile || p->ctx->world > 1) return enqueue_try(p, diagonal, min_diag, max_diag);
  const int key = diagonal ? 1 : 0;
  if (p->try_graph[key] && (p->graph_min_diag[key] != min_diag || p->graph_max_diag[key] != max_diag)) {
    cudaGraphExecDestroy(p->try_graph[key]);
    p->try_graph[key] = nullptr;
  }
  if (!p->try_graph[key]) {
    cudaStream_t st = p->ctx->stream;
    const int64_t launches0 = p->ctx->launches;
    B200_CUDA(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
    const int rc = enqueue_try(p, diagonal, min_diag, max_diag);
    cudaGraph_t graph = nullptr;
    const cudaError_t ce = cudaStreamEndCapture(st, &graph);
    if (rc) { if (graph) cudaGraphDestroy(graph); return rc; }
    if (ce != cudaSuccess) { set_error(std::string("cudaStreamEndCapture: ") + cudaGetErrorString(ce)); return B200_CUDA_ERROR; }
    B200_CUDA(cudaGraphInstantiate(&p->try_graph[key], graph, 0));
    cudaGraphDestroy(graph);
    p->graph_min_diag[key] = min_diag; p->graph_max_diag[key] = max_diag;   // the clamps are baked into THIS key's graph
    p->try_launches = p->ctx->launches - launches0;   // kernels inside one replay
    p->ctx->launches = launches0;
  }
  B200_CUDA(cudaGraphLaunch(p->try_graph[key], p->ctx->stream));
  p->ctx->launches += p->try_launches;
  p->solved = p->factored = true;
  p->marg_ready = false;     // the LM try factors the damped system
  return B200_OK;
}
// the captured LM tries have the group views, buffers and kernel instantiations baked in
static void drop_try_graphs(b200_problem* p) {
  for (auto& g : p->try_graph)
    if (g) { cudaGraphExecDestroy(g); g = nullptr; }
}

}  // namespace b200

using namespace b200;

// ---------------------------------------------------------------------------
extern "C" {

int b200_var_storage(int32_t t) { return (t >= 0 && t < B200_NUM_VAR_TYPES) ? VAR_STORAGE[t] : -1; }
int b200_var_dim(int32_t t) { return (t >= 0 && t < B200_NUM_VAR_TYPES) ? VAR_DIM[t] : -1; }
int b200_factor_arity(int32_t t) { return (t >= 0 && t < B200_NUM_FACTOR_TYPES) ? F_ARITY[t] : -1; }
int b200_factor_meas_size(int32_t t) { return (t >= 0 && t < B200_NUM_FACTOR_TYPES) ? F_MEAS[t] : -1; }
int b200_factor_dim(int32_t t) { return (t >= 0 && t < B200_NUM_FACTOR_TYPES) ? F_DIM[t] : -1; }
const char* b200_last_error_string(void) { return g_err.c_str(); }

int b200_ctx_create(int device, b200_ctx** out) {
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    set_error("no CUDA device visible: gtsam_b200 has no CPU fallback");
    return B200_NO_DEVICE;
  }
  if (device < 0 || device >= ndev) { set_error("device index out of range"); return B200_INVALID_ARGUMENT; }
  B200_CUDA(cudaSetDevice(device));
  b200_ctx* c = new b200_ctx();
  c->device = device;
  // (every early return below releases the context and its stream)
  struct Guard { b200_ctx* c; ~Guard() { if (c) { if (c->stream) cudaStreamDestroy(c->stream); delete c; } } } guard{c};
  B200_CUDA(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
  cudaDeviceProp prop;
  B200_CUDA(cudaGetDeviceProperties(&prop, device));
  c->sm_count = prop.multiProcessorCount;
  {
    unsigned char pa[B200_NUM_FACTOR_TYPES][kMaxPairs] = {}, pb[B200_NUM_FACTOR_TYPES][kMaxPairs] = {};
    for (int ty = 0; ty < B200_NUM_FACTOR_TYPES; ty++) {
      const int nc = VAR_DIM[F_VT[ty][0]] + (F_ARITY[ty] == 2 ? VAR_DIM[F_VT[ty][1]] : 0) + 1;
      int q = 0;
      for (int a = 0; a < nc; a++) for (int b = a; b < nc; b++) { pa[ty][q] = (unsigned char)a; pb[ty][q] = (unsigned char)b; q++; }
    }
    B200_CUDA(cudaMemcpyToSymbol(kPairA, pa, sizeof pa));
    B200_CUDA(cudaMemcpyToSymbol(kPairB, pb, sizeof pb));
  }
#ifndef B200_EMULATE   // (no shared-memory limit to raise in the host emulation build)
  B200_CUDA(cudaFuncSetAttribute(leaf_fused_kernel<double>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)(kWarpsPerBlock * (kLeafMaxFN + kLeafAccMax) * sizeof(double))));
  B200_CUDA(cudaFuncSetAttribute(leaf_fused_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)(kWarpsPerBlock * (kLeafMaxFN + kLeafAccMax) * sizeof(double))));
  B200_CUDA(cudaFuncSetAttribute(elim_small_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)(kWarpsPerBlock * kSmallMaxN * kSmallMaxN * sizeof(double))));
  B200_CUDA(cudaFuncSetAttribute(front_df_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, kDfSmemBytes));
  B200_CUDA(cudaFuncSetAttribute(front_df_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, kDfSmemBytes));
  // the widest point-leaf instantiations stage more than the 48 KB a kernel gets by default
#define B200_SM_ATTR(DC_, T_)                                                                                                          \
  B200_CUDA(cudaFuncSetAttribute(leaf_point_fused_mma_kernel<DC_, T_, double>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024)); \
  B200_CUDA(cudaFuncSetAttribute(leaf_point_fused_mma_kernel<DC_, T_, float>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  B200_SM_ATTR(6, 4) B200_SM_ATTR(6, 5) B200_SM_ATTR(6, 7) B200_SM_ATTR(9, 4) B200_SM_ATTR(9, 5) B200_SM_ATTR(9, 7) B200_SM_ATTR(9, 10)
#undef B200_SM_ATTR
#endif
  guard.c = nullptr;
  *out = c;
  return B200_OK;
}
int b200_nccl_unique_id(void* out128) {
  const int rc = nccl_load();
  if (rc) return rc;
  B200_NCCL(g_nccl.GetUniqueId(out128));
  return B200_OK;
}
int b200_ctx_comm_init(b200_ctx* c, const void* id128, int rank, int world) {
  if (world < 1 || rank < 0 || rank >= world) { set_error("bad rank/world"); return B200_INVALID_ARGUMENT; }
  c->rank = rank; c->world = world;
  if (world == 1) return B200_OK;
  const int rc = nccl_load();
  if (rc) return rc;
  B200_CUDA(cudaSetDevice(c->device));
  ncclUniqueIdBlob id;
  memcpy(&id, id128, sizeof id);
  B200_NCCL(g_nccl.CommInitRank(&c->comm, world, id, rank));
  return B200_OK;
}
int b200_ctx_destroy(b200_ctx* c) {
  if (!c) return B200_OK;
  cudaSetDevice(c->device);
  if (c->comm && g_nccl.CommDestroy) g_nccl.CommDestroy(c->comm);
  cudaStreamDestroy(c->stream);
  delete c;
  return B200_OK;
}
int64_t b200_launch_count(const b200_ctx* c) { return c->launches; }
void* b200_ctx_stream(const b200_ctx* c) { return (void*)c->stream; }

int b200_problem_destroy(b200_problem* p) {
  if (!p) return B200_OK;
  cudaSetDevice(p->ctx->device);
  cudaStreamSynchronize(p->ctx->stream);
  drop_try_graphs(p);
  for (auto& e : p->ev_pool) { cudaEventDestroy(e.first); cudaEventDestroy(e.second); }
  delete p;   // the owners of the problem's buffers free them
  return B200_OK;
}
static int upload_jacobian_group(b200_problem* p, b200_problem::Group& g, const double* Ab, const double* sigmas);

// What the stages of create_problem hand on to each other.
struct ProblemPlan {
  const b200_problem_desc* d; const b200_linear_desc* ld;   // exactly one of them is non-null
  int64_t ngroups = 0;
  Packed pk;
  std::vector<char> fused, is_top;                          // per clique (shard_plan)
  std::vector<int> clique_owner, factor_owner, top_owner;
  std::vector<int> fused_list, run_ptr;                     // the fused leaf cliques THIS rank owns, in runs
  std::vector<int> leaf_kind;                               // per clique: 0 generic, 1 / 2: BAL point clique, 6- / 9-dof cameras
  std::vector<std::vector<int2>> hkeys; std::vector<std::vector<int4>> hscat;   // typed groups: keys, scatter records (device order)
};

static int setup_symbolic(b200_problem* p, ProblemPlan& P) {
  if (const int rc = P.d ? pack_and_symbolic(P.d, &P.pk) : pack_linear(P.ld, &P.pk)) return rc;
  const int64_t n = P.d ? P.d->nvars : P.ld->nvars;
  P.ngroups = P.d ? P.d->ngroups : P.ld->ngroups + P.ld->nhgroups;   // linear: Jacobian groups, then Hessian groups
  p->nvars = n; p->nval = P.pk.val_off[n]; p->ndelta = P.pk.var_dof[n]; p->nfactors = P.pk.total;
  if (P.d) p->var_type.assign(P.d->var_type, P.d->var_type + n);
  p->groups.resize(P.ngroups);
  for (int64_t gi = 0; gi < P.ngroups; gi++) {
    auto& g = p->groups[gi];
    const PackedGroup& q = P.pk.groups[gi];
    g.type = q.type; g.noise_kind = q.noise_kind; g.per_factor = q.per_factor; g.noise_size = q.noise_size;
    g.d = q.d; g.ncols = q.ncols; g.arity = q.arity; g.meas = q.meas; g.count = q.count; g.pos = q.pos;
    g.robust_kind = q.robust_kind; g.robust_param = q.robust_param;
    g.col0[0] = 0;
    for (int a = 0; a < B200_JACOBIAN_MAX_ARITY; a++) g.col0[a + 1] = g.col0[a] + (a < q.arity ? q.dims[a] : 0);
    g.col0[q.arity + 1] = g.col0[q.arity] + 1;   // the rhs column closes the list
  }
  p->sym = std::move(P.pk.sym);
  return B200_OK;
}
static int setup_values(b200_problem* p, ProblemPlan& P) {
  if (P.d) {
    B200_CUDA(upload(p->d_values, P.d->values, (size_t)p->nval, p->ctx->stream));
    B200_CUDA(p->d_new_values.alloc(p->nval));
    B200_CUDA(upload(p->d_val_off, P.pk.val_off, p->ctx->stream));
    B200_CUDA(upload(p->d_var_type, p->var_type, p->ctx->stream));
    B200_CUDA(upload(p->d_cal, P.d->cal, (size_t)P.d->ncal * 5, p->ctx->stream));
  }
  B200_CUDA(p->d_delta.alloc(p->ndelta));
  B200_CUDA(cudaMemsetAsync(p->d_delta, 0, std::max<int64_t>(1, p->ndelta) * sizeof(double), p->ctx->stream));
  B200_CUDA(p->d_hdiag.alloc(p->ndelta));
  B200_CUDA(upload(p->d_var_dof, P.pk.var_dof, p->ctx->stream));
  return B200_OK;
}
// Storage plan (fused leaf cliques keep only their f x n conditional; sharding), then the owned fused leaves grouped into
// runs that share (parent, separator variables): one warp / CTA reduces a run's Schur complements before the extend-add.
static int setup_leaf_runs(b200_problem* p, ProblemPlan& P) {
  const Symbolic& S = p->sym;
  const b200_ctx* ctx = p->ctx;
  shard_plan(S, P.ngroups, p->nfactors, ctx->world, &P.fused, &P.is_top, &P.clique_owner, &P.factor_owner, /*allow_leaf=*/P.d != nullptr, &P.top_owner);
  p->top_staged = ctx->world > 1 && getenv("B200_REPLICATED_TOP") == nullptr;
  std::vector<int>& fused_list = P.fused_list;
  for (int64_t c = 0; c < S.ncliques; c++)
    if (P.fused[c] && P.clique_owner[c] == p->ctx->rank) fused_list.push_back((int)c);
  auto sig_cmp = [&](int a, int b) {   // run signature: parent, then the separator variables
    if (S.parent[a] != S.parent[b]) return S.parent[a] < S.parent[b] ? -1 : 1;
    const int64_t la = S.sep_ptr[a + 1] - S.sep_ptr[a], lb = S.sep_ptr[b + 1] - S.sep_ptr[b];
    if (la != lb) return la < lb ? -1 : 1;
    for (int64_t q = 0; q < la; q++) {
      const int64_t va = S.sep_vars[S.sep_ptr[a] + q], vb = S.sep_vars[S.sep_ptr[b] + q];
      if (va != vb) return va < vb ? -1 : 1;
    }
    return 0;
  };
  // kind 1/2: BAL point cliques (one Point3 frontal, m <= kPtMaxObs binary projection factors on
  // distinct cameras) take the point-leaf kernels <6>/<9>; everything else the generic leaf kernel
  std::vector<int> cf_count(S.ncliques, 0), cf_mask(S.ncliques, 0);
  std::vector<int>& kind = P.leaf_kind;
  kind.assign(S.ncliques, 0);
  for (int64_t gi = 0; P.d && gi < P.d->ngroups; gi++)
    for (int64_t i = 0; i < P.d->groups[gi].count; i++) {
      const int c = S.fac_clique[p->groups[gi].pos[i]];
      if (P.fused[c]) { cf_count[c]++; cf_mask[c] |= 1 << P.d->groups[gi].type; }
    }
  const bool fast = !getenv("B200_NO_POINT_KERNEL");
  for (int c : fused_list) {
    const int64_t nsep = S.sep_ptr[c + 1] - S.sep_ptr[c];
    const bool point = S.front_ptr[c + 1] - S.front_ptr[c] == 1 && P.d->var_type[S.front_vars[S.front_ptr[c]]] == B200_VAR_POINT3;
    if (!fast || !point || cf_count[c] != nsep || cf_count[c] > kPtMaxObs || cf_count[c] < 1) continue;
    if (cf_mask[c] == (1 << B200_FACTOR_PROJECTION_CAL3S2)) kind[c] = 1;
    else if (cf_mask[c] == (1 << B200_FACTOR_SFM_BUNDLER)) kind[c] = 2;
  }
  std::sort(fused_list.begin(), fused_list.end(), [&](int a, int b) {
    if (kind[a] != kind[b]) return kind[a] < kind[b];
    const int s = sig_cmp(a, b);
    return s != 0 ? s < 0 : a < b;
  });
  const int nfl = (int)fused_list.size();
  // long enough to amortise the per-run extend-add, short enough for >= 8 CTAs per SM
  int run_max_pt = getenv("B200_NO_LEAF_RUNS") ? 1 : std::max(1, std::min(64, nfl / (ctx->sm_count * 8)));
  if (getenv("B200_LEAF_RUN_MAX")) run_max_pt = std::max(1, atoi(getenv("B200_LEAF_RUN_MAX")));
  std::vector<int>& run_ptr = P.run_ptr;
  run_ptr.push_back(0);
  for (int i = 1; i <= nfl; i++) {
    const int kprev = kind[fused_list[i - 1]];
    const int rmax = kprev == 0 ? 1 : run_max_pt;
    if (i == nfl || i - run_ptr.back() >= rmax || kind[fused_list[i]] != kprev || sig_cmp(fused_list[i - 1], fused_list[i]) != 0)
      run_ptr.push_back(i);
  }
  p->n_runs = (int)run_ptr.size() - 1;
  for (int kd = 0, r = 0; kd < 3; kd++) {
    p->leaf_run_begin[kd] = r;
    while (r < p->n_runs && kind[fused_list[run_ptr[r]]] == kd) r++;
    p->leaf_run_end[kd] = r;
    p->leaf_pos_begin[kd] = run_ptr[p->leaf_run_begin[kd]];
    p->leaf_pos_end[kd] = run_ptr[r];
  }
  // shared memory per warp of the generic leaf kernel: the widest [F S d] block
  for (int c : fused_list) {
    if (kind[c] == 0) p->leaf_lb_cap = std::max(p->leaf_lb_cap, S.nf[c] * (S.nf[c] + S.ns[c] + 1));
    p->leaf_max_w[kind[c]] = std::max(p->leaf_max_w[kind[c]], S.ns[c] + 1);
  }
  p->n_fused = nfl;
  p->schur_pb = (getenv("B200_SCHUR_PB") && atoi(getenv("B200_SCHUR_PB")) == 6) ? 6 : 4;
  p->schur_mma = !(getenv("B200_SCHUR_MMA") && atoi(getenv("B200_SCHUR_MMA")) == 0);
  if (getenv("B200_LIN_VARIANT")) p->lin_variant = atoi(getenv("B200_LIN_VARIANT"));
  return B200_OK;
}
static int setup_offsets(b200_problem* p, ProblemPlan& P) {
  const Symbolic& S = p->sym;
  p->h_off.assign(S.ncliques + 1, 0);
  p->h_ld.assign(S.ncliques, 0);
  int64_t o = 0;
  std::vector<int64_t> order(S.ncliques);     // top fronts level by level: a stage of the distributed top is one contiguous range
  for (int64_t c = 0; c < S.ncliques; c++) order[c] = c;
  std::stable_sort(order.begin(), order.end(), [&](int64_t a, int64_t b) { return (P.is_top[a] ? S.level[a] : -1) < (P.is_top[b] ? S.level[b] : -1); });
  for (int pass = 0; pass < 2; pass++) {   // replicated top first: it is the all-reduced region
    for (int64_t oc = 0; oc < S.ncliques; oc++) {
      const int64_t c = pass == 0 ? order[oc] : oc;
      if (!P.fused[c] && (P.is_top[c] != 0) == (pass == 0)) {
        const int64_t nn = S.nf[c] + S.ns[c] + 1; p->h_ld[c] = (int)nn;
        // the fronts of other ranks' subtrees take no storage here (nothing on this rank ever touches them)
        if (pass == 1 && P.clique_owner[c] != p->ctx->rank) { p->h_off[c] = 0; continue; }
        p->h_off[c] = o; o += nn * nn;
      }
    }
    if (pass == 0) p->top_doubles = o;
  }
  p->zero_doubles = o;   // everything below is accumulated into by atomics: zeroed per solve
  for (int64_t c = 0; c < S.ncliques; c++)
    if (P.fused[c]) {
      const int64_t nn = S.nf[c] + S.ns[c] + 1; p->h_ld[c] = S.nf[c];
      if (P.clique_owner[c] != p->ctx->rank) { p->h_off[c] = 0; continue; }
      p->h_off[c] = o; o += (int64_t)S.nf[c] * nn;
    }
  p->arena_doubles = o;
  p->h_off[S.ncliques] = o;
  return B200_OK;
}
// JacobianFactor / HessianFactor groups: keys, owning clique and front slot of every key, then the numbers
// (whitened [A|b], or the augmented information matrix) in the element-major SoA
static int setup_linear_groups(b200_problem* p, ProblemPlan& P) {
  if (!P.ld) return B200_OK;
  const Symbolic& S = p->sym;
  const b200_linear_desc* ld = P.ld;
  for (int64_t gi = 0; gi < P.ngroups; gi++) {
    auto& g = p->groups[gi];
    const bool hess = gi >= ld->ngroups;
    const int ar = g.arity;
    // keep only the factors this rank owns (all of them when world == 1): SURVEY 8(e), as for the typed groups
    g.full_count = g.count;
    for (int64_t i = 0; i < g.full_count; i++) if (P.factor_owner[g.pos[i]] == p->ctx->rank) g.local_index.push_back(i);
    const int64_t count = (int64_t)g.local_index.size();
    g.count = count;
    std::vector<int> jkeys((size_t)count * ar), jslots((size_t)count * ar), jclique((size_t)count);
    for (int64_t li = 0; li < count; li++) {
      const int64_t pos = g.pos[g.local_index[li]];
      jclique[li] = S.fac_clique[pos];
      for (int a = 0; a < ar; a++) {
        jkeys[(size_t)li * ar + a] = (int)P.pk.fkeys[P.pk.fptr[pos] + a];
        jslots[(size_t)li * ar + a] = S.fac_slots[P.pk.fptr[pos] + a];
      }
    }
    g.n_nonleaf = count;
    B200_CUDA(upload(g.d_jkeys, jkeys, p->ctx->stream));
    B200_CUDA(upload(g.d_jslots, jslots, p->ctx->stream));
    B200_CUDA(upload(g.d_jclique, jclique, p->ctx->stream));
    B200_CUDA(g.d_J.alloc((size_t)count * g.d * g.ncols));
    const int rc = hess ? upload_jacobian_group(p, g, ld->hgroups[gi - ld->ngroups].info, nullptr)   // (N+1)^2 entries, no whitening
                        : upload_jacobian_group(p, g, ld->groups[gi].Ab, ld->groups[gi].sigmas);
    if (rc) return rc;
  }
  return B200_OK;
}
static int setup_typed_groups(b200_problem* p, ProblemPlan& P) {
  if (!P.d) return B200_OK;
  const Symbolic& S = p->sym;
  const std::vector<int>& fused_list = P.fused_list;
  const bool reorder_leaf_factors = getenv("B200_NO_FACTOR_REORDER") == nullptr;
  std::vector<int> leaf_list_pos(S.ncliques, INT_MAX);      // position of a point leaf (kinds 1 / 2) in fused_list
  for (size_t i = 0; i < fused_list.size(); i++) if (P.leaf_kind[fused_list[i]] > 0) leaf_list_pos[fused_list[i]] = (int)i;
  P.hkeys.resize(P.ngroups);
  P.hscat.resize(P.ngroups);
  for (int64_t gi = 0; gi < P.ngroups; gi++) {
    const b200_factor_group& s = P.d->groups[gi];
    auto& g = p->groups[gi];
    // keep only the factors this rank owns (all of them when world == 1)
    std::vector<int64_t>& keep = g.local_index;
    for (int64_t i = 0; i < s.count; i++) if (P.factor_owner[g.pos[i]] == p->ctx->rank) keep.push_back(i);
    // Device order of a projection group = the order in which the leaf kernels visit its factors: by the position of the owning
    // point leaf in fused_list (points of one run next to each other), graph order inside a point; factors of other cliques
    // behind them.  Every row of the element-major SoA then holds a warp's 4 points x m factors contiguously.  In graph order
    // each point's 5 floats of a row sit alone in a 128-byte line, so the leaf kernels read several times the bytes of the
    // Jacobians they use.  It also puts factors that share cameras
    // (the points of a run) side by side for the gathers of linearize_kernel / error_kernel.  local_index maps back to the
    // caller's order wherever that is visible (b200_get_jacobians, b200_set_group_noise).
    if (reorder_leaf_factors && (s.type == B200_FACTOR_PROJECTION_CAL3S2 || s.type == B200_FACTOR_SFM_BUNDLER) && !fused_list.empty()) {
      // stable counting sort by list position (one bucket per leaf + one for "not a point leaf"): linear in the group
      const size_t nb = fused_list.size() + 1;
      std::vector<int64_t> start(nb + 1, 0);
      auto bucket = [&](int64_t i) { const int q = leaf_list_pos[S.fac_clique[g.pos[i]]]; return q == INT_MAX ? nb - 1 : (size_t)q; };
      for (int64_t i : keep) start[bucket(i) + 1]++;
      for (size_t b = 0; b < nb; b++) start[b + 1] += start[b];
      std::vector<int64_t> sorted(keep.size());
      for (int64_t i : keep) sorted[start[bucket(i)]++] = i;
      keep.swap(sorted);
    }
    const int64_t nl = (int64_t)keep.size();
    std::vector<int2>& hkeys = P.hkeys[gi];
    std::vector<int4>& hscat = P.hscat[gi];
    hkeys.resize(nl); hscat.resize(nl);
    std::vector<double> hmeas((size_t)nl * g.meas), hnoise;
    std::vector<int> hcal;
    if (s.noise_per_factor) hnoise.resize((size_t)nl * g.noise_size);
    const bool with_cal = s.type == B200_FACTOR_PROJECTION_CAL3S2 && s.cal_index;
    if (with_cal) hcal.resize((size_t)nl);
    int64_t nonleaf_part[16] = {0};
    parallel_chunks(nl, [&](int64_t l0, int64_t l1, int tid) {
      int64_t nonleaf = 0;
      for (int64_t li = l0; li < l1; li++) {
        const int64_t i = keep[li], pos = g.pos[i], k0 = P.pk.fptr[pos];
        hkeys[li] = make_int2((int)P.pk.fkeys[k0], g.arity == 2 ? (int)P.pk.fkeys[k0 + 1] : -1);
        const int isleaf = P.fused[S.fac_clique[pos]];
        hscat[li] = make_int4(S.fac_clique[pos], S.fac_slot0[pos], S.fac_slot1[pos], isleaf);
        if (!isleaf) nonleaf++;
        memcpy(hmeas.data() + (size_t)li * g.meas, s.meas + (size_t)i * g.meas, (size_t)g.meas * sizeof(double));
        if (s.noise_per_factor) memcpy(hnoise.data() + (size_t)li * g.noise_size, s.noise + (size_t)i * g.noise_size, (size_t)g.noise_size * sizeof(double));
        if (with_cal) hcal[(size_t)li] = s.cal_index[i];
      }
      nonleaf_part[tid] = nonleaf;
    });
    for (int t = 0; t < 16; t++) g.n_nonleaf += nonleaf_part[t];
    g.count = nl;
    B200_CUDA(upload(g.d_keys, hkeys, p->ctx->stream));
    B200_CUDA(upload(g.d_scat, hscat, p->ctx->stream));
    B200_CUDA(upload(g.d_meas, hmeas, p->ctx->stream));
    if (s.noise_per_factor) B200_CUDA(upload(g.d_noise, hnoise, p->ctx->stream));
    else B200_CUDA(upload(g.d_noise, s.noise, (size_t)g.noise_size, p->ctx->stream));
    if (!hcal.empty()) B200_CUDA(upload(g.d_cal, hcal, p->ctx->stream));
    if (s.type == B200_FACTOR_PROJECTION_CAL3S2 && s.body_P_sensor) B200_CUDA(upload(g.d_body, s.body_P_sensor, 12, p->ctx->stream));
    B200_CUDA(g.d_J.alloc((size_t)nl * g.d * g.ncols));
  }
  return B200_OK;
}
static int setup_tree_tables(b200_problem* p, ProblemPlan& P) {
  const Symbolic& S = p->sym;
  std::vector<int> parent32(S.ncliques);
  for (int64_t c = 0; c < S.ncliques; c++) parent32[c] = (int)S.parent[c];
  B200_CUDA(upload(p->d_off, p->h_off, p->ctx->stream));
  B200_CUDA(upload(p->d_ld, p->h_ld, p->ctx->stream));
  B200_CUDA(upload(p->d_nf, S.nf, p->ctx->stream));
  B200_CUDA(upload(p->d_ns, S.ns, p->ctx->stream));
  B200_CUDA(upload(p->d_parent, parent32, p->ctx->stream));
  B200_CUDA(upload(p->d_ea_ptr, S.ea_ptr, p->ctx->stream));
  B200_CUDA(upload(p->d_ea_map, S.ea_map, p->ctx->stream));
  B200_CUDA(upload(p->d_didx_ptr, S.didx_ptr, p->ctx->stream));
  B200_CUDA(upload(p->d_didx, S.didx, p->ctx->stream));
  std::vector<int64_t> diag_index(p->ndelta);
  for (int64_t v = 0; v < p->nvars; v++) {
    const int c = S.var_clique[v];
    const int64_t nn = S.nf[c] + S.ns[c] + 1;
    for (int k = 0; k < P.pk.var_dim[v]; k++)
      diag_index[P.pk.var_dof[v] + k] = (P.fused[c] || (P.is_top[c] ? p->ctx->rank != 0 : P.clique_owner[c] != p->ctx->rank))
                                            ? -1 : p->h_off[c] + (S.var_slot[v] + k) * (nn + 1);
  }
  B200_CUDA(upload(p->d_diag_index, diag_index, p->ctx->stream));
  return B200_OK;
}
// fused leaf cliques: CSR of their factors as (group, index), graph order; the BAL point table
static int setup_leaf_tables(b200_problem* p, ProblemPlan& P) {
  if (!p->n_fused) return B200_OK;
  const Symbolic& S = p->sym;
  const std::vector<int>& fused_list = P.fused_list;
  std::vector<int> lpos(S.ncliques, -1), fptr(p->n_fused + 1, 0);
  for (int i = 0; i < p->n_fused; i++) lpos[fused_list[i]] = i;
  for (int64_t pos = 0; pos < p->nfactors; pos++) if (lpos[S.fac_clique[pos]] >= 0) fptr[lpos[S.fac_clique[pos]] + 1]++;
  for (int i = 0; i < p->n_fused; i++) fptr[i + 1] += fptr[i];
  std::vector<int2> ffac(fptr[p->n_fused]);
  std::vector<int> cur(fptr.begin(), fptr.end() - 1);
  for (int64_t gi = 0; gi < P.ngroups; gi++)
    for (int64_t li = 0; li < p->groups[gi].count; li++) {
      const int64_t pos = p->groups[gi].pos[p->groups[gi].local_index[li]];
      if (lpos[S.fac_clique[pos]] >= 0) ffac[cur[lpos[S.fac_clique[pos]]]++] = make_int2((int)gi, (int)li);
    }
  // keep graph order inside each clique (groups may interleave in the graph; a clique whose factors come from one group
  // already has it)
  parallel_chunks(p->n_fused, [&](int64_t i0, int64_t i1, int) {
    auto gpos = [&](const int2& a) { return p->groups[a.x].pos[p->groups[a.x].local_index[a.y]]; };
    for (int64_t i = i0; i < i1; i++) {
      bool ordered = true;
      for (int q = fptr[i] + 1; q < fptr[i + 1] && ordered; q++) ordered = gpos(ffac[q - 1]) < gpos(ffac[q]);
      if (!ordered)
        std::sort(ffac.begin() + fptr[i], ffac.begin() + fptr[i + 1], [&](const int2& a, const int2& b) { return gpos(a) < gpos(b); });
    }
  });
  B200_CUDA(upload(p->d_fused_list, fused_list, p->ctx->stream));
  B200_CUDA(upload(p->d_fused_run_ptr, P.run_ptr, p->ctx->stream));
  B200_CUDA(upload(p->d_fused_fac_ptr, fptr, p->ctx->stream));
  B200_CUDA(upload(p->d_fused_fac, ffac, p->ctx->stream));
  // BAL point leaves: one flat record per (point position, factor slot 0..7) = (factor index in its group, group << 8 | camera
  // slot) and the offset of the point's conditional, so that the leaf kernels reach their operands through ONE level of index
  // loads (list -> fac_ptr -> fac -> scat was a chain of three dependent loads in front of every batch of points)
  if (p->leaf_pos_end[2] > p->leaf_pos_begin[1] || p->leaf_pos_end[1] > p->leaf_pos_begin[1]) {
    std::vector<int2> tab((size_t)p->n_fused * kPtMaxObs, make_int2(-1, 0));
    std::vector<int64_t> poff((size_t)p->n_fused, 0);
    parallel_chunks(p->n_fused, [&](int64_t i0, int64_t i1, int) {
      for (int64_t i = i0; i < i1; i++) {
        const int c = fused_list[i], kd = P.leaf_kind[c];
        poff[i] = p->h_off[c];
        if (kd == 0) continue;
        const int dc = kd == 1 ? 6 : 9;
        for (int q = fptr[i]; q < fptr[i + 1]; q++) {
          const int2 gf = ffac[q];
          tab[(size_t)i * kPtMaxObs + (q - fptr[i])] = make_int2(gf.y, (gf.x << 8) | ((P.hscat[gf.x][gf.y].y - 3) / dc));
        }
      }
    });
    B200_CUDA(upload(p->d_pt_tab, tab, p->ctx->stream));
    B200_CUDA(upload(p->d_pt_off, poff, p->ctx->stream));
  }
  return B200_OK;
}
// Tile grid of a dataflow front: K pivot column blocks of kDfB columns, NB column blocks in all.
static void df_shape(const Symbolic& S, int c, int& K, int& NB) {
  const int f = S.nf[c], nn = f + S.ns[c] + 1;
  K = (f + kDfB - 1) / kDfB; NB = K + (nn - f + kDfB - 1) / kDfB;
}
// The number of pivot steps tile (front, column block, row tile) has to see before it is done.
static int df_need(const Symbolic& S, const int4& t) {
  int K, NB; df_shape(S, t.x, K, NB);
  return std::min(K, std::min(std::min(kDfTR * t.z + kDfTR - 1, t.y), NB - 1) + 1);
}
// Every wait of front_df_kernel on the tiles T of one launch points to a smaller ticket of that launch (or to an earlier launch).
static bool df_order_is_safe(const Symbolic& S, const std::vector<int4>& T) {
  std::vector<int64_t> first(S.ncliques, -1), last(S.ncliques, -1), base(S.ncliques, -1);   // per front: smallest / largest ticket; offset into tk
  int64_t ntk = 0;
  for (size_t i = 0; i < T.size(); i++) {
    const int c = T[i].x;
    if (base[c] < 0) { int K, NB; df_shape(S, c, K, NB); base[c] = ntk; ntk += (int64_t)NB * ((NB + kDfTR - 1) / kDfTR); first[c] = (int64_t)i; }
    last[c] = (int64_t)i;
  }
  std::vector<int> tk((size_t)ntk, -1);             // ticket of tile (c, j, r)
  auto slot = [&](int c, int j, int r) { int K, NB; df_shape(S, c, K, NB); return base[c] + (int64_t)j * ((NB + kDfTR - 1) / kDfTR) + r; };
  for (size_t i = 0; i < T.size(); i++) tk[slot(T[i].x, T[i].y, T[i].z)] = (int)i;
  for (size_t i = 0; i < T.size(); i++) {
    const int c = T[i].x, j = T[i].y, r = T[i].z;
    int K, NB; df_shape(S, c, K, NB);
    const int last_rb = std::min(std::min(kDfTR * r + kDfTR - 1, j), NB - 1);
    auto before = [&](int jj, int rr) { const int d = tk[slot(c, jj, rr)]; return (jj == j && rr == r) || (d >= 0 && d < (int)i); };
    for (int k = 0; k < std::min(K, last_rb + 1); k++) {
      const int rk = k / kDfTR;
      if (k <= j && !before(k, rk)) return false;                      // R_kk from the diagonal tile of column k
      if (rk < r && !before(j, rk)) return false;                      // column piece (k, j)
      for (int ib = std::max(kDfTR * r, k + 1); ib <= last_rb; ib++)
        if (ib != j && !before(ib, rk)) return false;                  // row piece (k, ib)
    }
    const int par = S.parent[c];
    if (par >= 0 && first[par] >= 0 && first[par] < last[c]) return false;   // a parent's tiles wait for every tile of its children
  }
  return true;
}
// What the level planner hands on to the uploads.
struct LevelLists {
  std::vector<int> small, bsmall, blarge, bpoint;      // cliques of d_lvl_small / _bsmall / _blarge / _bpoint
  std::vector<int4> df_tasks[2];                       // per phase: dataflow tiles (front, column block, row tile), ticket order
  std::vector<int> df_flag_off, df_expect, df_tiles;   // per clique
  int64_t df_nflags = 0;
};

// Level plans: small (one warp per clique) / tile dataflow.  Phase 0: the subtrees this rank owns, leaves to subtree roots;
// phase 1: the replicated top.  p->levels = [phase-0 levels ..., phase-1 levels ...]; elimination walks it forwards (with the
// all-reduce of the top fronts between the phases), back-substitution walks it backwards.
static int plan_levels(b200_problem* p, const ProblemPlan& P, LevelLists& L) {
  const Symbolic& S = p->sym;
  p->levels.resize(2 * S.nlevels);
  p->n_sub_levels = (int)S.nlevels;
  p->max_small_n = 1;
  // tile dataflow (front_df.cuh): per phase, from the first level that holds a front wider than kSmallMaxN upwards,
  // every non-leaf front is a set of tiles of ONE launch; the levels below it (small fronts only) keep elim_small_kernel
  int df_first[2] = {INT_MAX, INT_MAX};
  L.df_flag_off.assign(S.ncliques, 0); L.df_expect.assign(S.ncliques, 0); L.df_tiles.assign(S.ncliques, 0);
  auto in_phase = [&](int phase, int c) {
    return phase == 0 ? (!P.is_top[c] && P.clique_owner[c] == p->ctx->rank) : (P.is_top[c] != 0 && (!p->top_staged || P.top_owner[c] == p->ctx->rank));
  };
  for (int phase = 0; phase < 2; phase++)
    for (int64_t c = 0; c < S.ncliques; c++)
      if (in_phase(phase, (int)c) && !P.fused[c] && S.nf[c] + S.ns[c] + 1 > kSmallMaxN) df_first[phase] = std::min(df_first[phase], S.level[c]);
  if (p->top_staged) df_first[1] = 0;     // every top front goes through its stage's reduce + dataflow launch
  for (int phase = 0; phase < 2; phase++)
  for (int64_t l = 0; l < S.nlevels; l++) {
    LevelPlan& lv = p->levels[phase * S.nlevels + l];
    lv = LevelPlan();
    lv.small_begin = (int)L.small.size();
    lv.bsmall_begin = (int)L.bsmall.size();
    lv.blarge_begin = (int)L.blarge.size();
    std::vector<int> pts[2];
    const size_t stage_task_begin = L.df_tasks[1].size();
    const size_t level_task_begin = L.df_tasks[phase].size();
    for (int64_t q = S.lvl_ptr[l]; q < S.lvl_ptr[l + 1]; q++) {
      const int c = S.lvl_cliques[q];
      const int nn = S.nf[c] + S.ns[c] + 1;
      if (!in_phase(phase, c)) continue;
      if (P.fused[c]) {
        // eliminated by the leaf kernels; back-substituted 8 lanes per point / one warp per clique
        if (P.leaf_kind[c] > 0 && !getenv("B200_NO_POINT_BACKSUB")) pts[P.leaf_kind[c] - 1].push_back(c);
        else L.bsmall.push_back(c);
      } else if (nn <= kSmallMaxN && l < df_first[phase]) {
        L.small.push_back(c);
        L.bsmall.push_back(c);
        p->max_small_n = std::max(p->max_small_n, nn);
      } else {
        if (l < df_first[phase]) { set_error("level plan: a front wider than kSmallMaxN below the first dataflow level (internal)"); return B200_INVALID_ARGUMENT; }
        // tiles (column block j, row tile r) of the upper trapezoid, ticket order: column-major (dependencies point backwards)
        int K, NB; df_shape(S, c, K, NB);
        if (p->df_level[phase] < 0) p->df_level[phase] = (int)(phase * S.nlevels + l);
        L.df_flag_off[c] = (int)L.df_nflags;
        L.df_nflags += (int64_t)K * NB;
        for (int j = 0; j < NB; j++)
          for (int r = 0; kDfTR * r <= j; r++) { L.df_tasks[phase].push_back(make_int4(c, j, r, 0)); L.df_tiles[c]++; }
        if (S.parent[c] >= 0) L.df_expect[S.parent[c]] += L.df_tiles[c];
        if (nn <= kSmallMaxN) { L.bsmall.push_back(c); continue; }
        // back-substitution cares about the pivots only: thin fronts (<= 8 pivots: one pass of the one-warp kernel
        // over the separator) skip the multi-CTA flag machinery (faster on the BAL trees, about even on sphere2500)
        if (S.nf[c] <= 8 && !getenv("B200_NO_THIN_BACKSUB")) L.bsmall.push_back(c);
        else { L.blarge.push_back(c); lv.blarge_max_nf = std::max(lv.blarge_max_nf, S.nf[c]); }
      }
    }
    lv.blarge_count = (int)L.blarge.size() - lv.blarge_begin;
    for (int kd = 0; kd < 2; kd++) {
      lv.bpoint_begin[kd] = (int)L.bpoint.size();
      lv.bpoint_count[kd] = (int)pts[kd].size();
      L.bpoint.insert(L.bpoint.end(), pts[kd].begin(), pts[kd].end());
    }
    lv.small_count = (int)L.small.size() - lv.small_begin;
    lv.bsmall_count = (int)L.bsmall.size() - lv.bsmall_begin;
    // ticket order inside a level: by column block first, across ALL the level's fronts (then front, row tile).  A tile of column
    // j has nothing to wait for once pivot step j is over, so the resident CTAs (2-3 per SM) are the columns next to every front's
    // pivot — the tiles with work — instead of all the columns of the first few fronts parked on their dependencies while the other
    // fronts of the level wait for a slot; columns further right start later and catch up at full rate (their pieces are all there).
    // Dependencies still point to smaller tickets (same front: smaller column, or same column and smaller row tile; children: lower level).
    if (!getenv("B200_DF_FRONT_ORDER")) {
      // ... refined: first by the number of pivot steps the tile has to see before it is done (its `need`): a tile that needs all K
      // steps of its front (every trailing tile of a front with few pivots and a wide separator) would otherwise sit on a slot
      // from the first step on, busy a small part of the time (one short update per pivot step, with every slot taken);
      // started late it finds its pieces ready and runs straight through.  A producer never
      // needs more steps than its consumers (smaller-or-equal row tile and column), so the order stays dependency-safe.
      const bool by_need = getenv("B200_DF_NO_NEED_ORDER") == nullptr;
      std::sort(L.df_tasks[phase].begin() + (int64_t)level_task_begin, L.df_tasks[phase].end(), [&](const int4& a, const int4& b) {
        if (by_need) { const int na = df_need(S, a), nb = df_need(S, b); if (na != nb) return na < nb; }
        return a.y != b.y ? a.y < b.y : (a.x != b.x ? a.x < b.x : a.z < b.z); });
    }
    if (phase == 1 && p->top_staged) {
      // the stage of this top level: ALL its fronts (whoever owns them: they are reduced onto their owners), this rank's tiles
      const int f0 = (int)p->ts_fronts.size();
      const int64_t x0 = p->topx_doubles;
      for (int64_t q = S.lvl_ptr[l]; q < S.lvl_ptr[l + 1]; q++) {
        const int c = S.lvl_cliques[q];
        if (!P.is_top[c]) continue;
        const int64_t nn = S.nf[c] + S.ns[c] + 1;
        p->ts_fronts.push_back({p->h_off[c], nn * nn, P.top_owner[c], c});
        p->topx_doubles += S.nf[c];
      }
      if ((int)p->ts_fronts.size() > f0) {
        p->ts_level.push_back((int)(S.nlevels + l));
        p->ts_begin.push_back(f0);
        p->ts_task_begin.push_back((int)stage_task_begin);
        p->ts_task_count.push_back((int)(L.df_tasks[1].size() - stage_task_begin));
        p->ts_x_begin.push_back((int)x0);
        p->ts_x_count.push_back((int)(p->topx_doubles - x0));
      }
    }
  }
  p->ts_begin.push_back((int)p->ts_fronts.size());
  return B200_OK;
}
// Ticket order across levels (B200_DF_ORDER=1, the default; 0 = level by level): by the ESTIMATED time a tile can finish, in pivot
// steps — its front's start (= the latest finish of a child front) + the pivot steps it has to see; trailing-column tiles
// optionally B200_DF_LAG steps later (they then find their pieces ready instead of idling on a slot).  A front whose
// children are done early no longer waits for the tickets of the rest of its level.  Dependency-safe: a producer's key
// is never larger than its consumer's (same front: fewer steps, pivot columns before trailing ones; children: finish
// <= the parent's start), ties broken as before — and df_order_is_safe() checks the result, whatever the order.
static void order_tickets(const b200_problem* p, LevelLists& L) {
  const Symbolic& S = p->sym;
  const int df_order = getenv("B200_DF_ORDER") ? atoi(getenv("B200_DF_ORDER")) : 1;
  const int df_lag = getenv("B200_DF_LAG") ? std::max(0, atoi(getenv("B200_DF_LAG"))) : 2;
  if (df_order < 1) return;
  std::vector<int64_t> est(S.ncliques, 0);
  for (int64_t c = 0; c < S.ncliques; c++) {      // children have smaller ids than parents
    if (!L.df_tiles[c] || S.parent[c] < 0) continue;
    int K, NB; df_shape(S, (int)c, K, NB);
    est[S.parent[c]] = std::max(est[S.parent[c]], est[c] + K + 1 + df_lag);
  }
  for (int phase = 0; phase < 2; phase++) {
    if (phase == 1 && p->top_staged) continue;     // the staged top is launched level by level
    auto key = [&](const int4& t) { int K, NB; df_shape(S, t.x, K, NB); return est[t.x] + df_need(S, t) + (t.y >= K ? df_lag : 0); };
    std::sort(L.df_tasks[phase].begin(), L.df_tasks[phase].end(), [&](const int4& a, const int4& b) {
      const int64_t ka = key(a), kb = key(b);
      if (ka != kb) return ka < kb;
      const int na = df_need(S, a), nb = df_need(S, b);
      if (na != nb) return na < nb;
      return a.y != b.y ? a.y < b.y : (a.x != b.x ? a.x < b.x : a.z < b.z); });
  }
}
static int setup_levels(b200_problem* p, ProblemPlan& P) {
  const Symbolic& S = p->sym;
  LevelLists L;
  if (const int rc = plan_levels(p, P, L)) return rc;
  order_tickets(p, L);
  for (int phase = 0; phase < 2; phase++)
    if (!df_order_is_safe(S, L.df_tasks[phase])) { set_error("front dataflow: ticket order is not dependency-safe (internal)"); return B200_INVALID_ARGUMENT; }
  if (p->top_staged && !p->ts_fronts.empty()) {
    std::vector<int> tc, tx, to;
    int64_t x = 0;
    for (auto& tf : p->ts_fronts) { tc.push_back(tf.clique); tx.push_back((int)x); to.push_back(tf.owner == p->ctx->rank ? 1 : 0); x += S.nf[tf.clique]; }
    B200_CUDA(upload(p->d_ts_cliques, tc, p->ctx->stream));
    B200_CUDA(upload(p->d_ts_xoff, tx, p->ctx->stream));
    B200_CUDA(upload(p->d_ts_owned, to, p->ctx->stream));
    B200_CUDA(p->d_topx.alloc(p->topx_doubles));
  }
  if (L.df_nflags + S.ncliques + 4 * (S.nlevels + 2) > (int64_t)INT_MAX) { set_error("front dataflow: flag table exceeds 2^31 entries"); return B200_INVALID_ARGUMENT; }
  for (int phase = 0; phase < 2; phase++) {
    p->df_ntasks[phase] = (int)L.df_tasks[phase].size();
    if (p->df_ntasks[phase]) B200_CUDA(upload(p->d_df_tasks[phase], L.df_tasks[phase], p->ctx->stream));
  }
  // backsub_large_kernel solves with the diagonal-block inverses W that front_df_kernel leaves behind
  for (int c : L.blarge)
    if (!L.df_tiles[c]) { set_error("level plan: a multi-CTA back-substitution front without diagonal-block inverses (internal)"); return B200_INVALID_ARGUMENT; }
  if (p->df_ntasks[0] + p->df_ntasks[1]) {
    std::vector<int64_t> woff(S.ncliques, -1);
    int64_t wtot = 0;
    for (int64_t c = 0; c < S.ncliques; c++)
      if (L.df_tiles[c]) { woff[c] = wtot; wtot += (int64_t)((S.nf[c] + kDfB - 1) / kDfB) * kDfB * kDfB; }
    B200_CUDA(upload(p->d_winv_off, woff, p->ctx->stream));
    B200_CUDA(p->d_winv.alloc(wtot));
    B200_CUDA(upload(p->d_df_flag_off, L.df_flag_off, p->ctx->stream));
    B200_CUDA(upload(p->d_df_expect, L.df_expect, p->ctx->stream));
    p->df_ctrl_ints = 2 * (2 + (int)S.nlevels);     // (ticket, abort) per launch: the two phases + one per stage of the top
    p->df_sync_ints = p->df_ctrl_ints + S.ncliques + L.df_nflags;
    // latency variant (2 CTAs per SM, 252 registers) unless the tree has more tiles than that keeps busy
    p->df_minb = (p->df_ntasks[0] + p->df_ntasks[1] > 6 * p->ctx->sm_count) ? 3 : 2;
    if (const char* e = getenv("B200_DF_MINB")) p->df_minb = atoi(e) == 3 ? 3 : 2;
    B200_CUDA(p->d_df_sync.alloc(p->df_sync_ints));
    if (getenv("B200_DF_TRACE") && p->df_ntasks[0]) {
      B200_CUDA(p->d_df_trace.alloc((size_t)p->df_ntasks[0] * 32));
      B200_CUDA(cudaMemsetAsync(p->d_df_trace, 0, (size_t)p->df_ntasks[0] * 32 * 8, p->ctx->stream));
    }
  }
  B200_CUDA(upload(p->d_lvl_small, L.small, p->ctx->stream));
  B200_CUDA(upload(p->d_lvl_bsmall, L.bsmall, p->ctx->stream));
  B200_CUDA(upload(p->d_lvl_blarge, L.blarge, p->ctx->stream));
  B200_CUDA(upload(p->d_lvl_bpoint, L.bpoint, p->ctx->stream));
  std::vector<int> fbase(L.blarge.size() + 1, 0);
  for (size_t i = 0; i < L.blarge.size(); i++) fbase[i + 1] = fbase[i] + (S.nf[L.blarge[i]] + kBsRows - 1) / kBsRows;
  B200_CUDA(upload(p->d_bs_flag_base, fbase, p->ctx->stream));
  p->n_bs_flags = fbase.back();
  B200_CUDA(p->d_bs_flags.alloc(fbase.back()));
  B200_CUDA(cudaMemsetAsync(p->d_bs_flags, 0, (size_t)std::max(1, fbase.back()) * sizeof(int), p->ctx->stream));
  return B200_OK;
}
// values views (sharded problems move only what a rank needs / owns between host and device)
static int setup_values_views(b200_problem* p, ProblemPlan& P) {
  if (!P.d) return B200_OK;
  const Symbolic& S = p->sym;
  const int64_t n = p->nvars;
  const int world = p->ctx->world;
  std::vector<char> need(n, world == 1), own(n, world == 1);
  if (world > 1) {
    for (int64_t c = 0; c < S.ncliques; c++) {
      if (!P.is_top[c] && P.clique_owner[c] != p->ctx->rank) continue;
      for (int64_t q = S.front_ptr[c]; q < S.front_ptr[c + 1]; q++) {
        need[S.front_vars[q]] = 1;
        if (!P.is_top[c] || p->ctx->rank == 0) own[S.front_vars[q]] = 1;     // the top's variables are reported by rank 0
      }
    }
    for (int64_t gi = 0; gi < P.ngroups; gi++)
      for (auto& k : P.hkeys[gi]) { need[k.x] = 1; if (k.y >= 0) need[k.y] = 1; }
  }
  for (int w = 0; w < 2; w++) {
    const std::vector<char>& m = w == 0 ? need : own;
    std::vector<int> idx;
    for (int64_t v = 0; v < n; v++)
      if (m[v]) { p->view_vars[w].push_back(v); for (int k = P.pk.val_off[v]; k < P.pk.val_off[v + 1]; k++) idx.push_back(k); }
    p->view_doubles[w] = (int64_t)idx.size();
    B200_CUDA(upload(p->d_view_idx[w], idx, p->ctx->stream));
  }
  B200_CUDA(p->d_view_buf.alloc(std::max(p->view_doubles[0], p->view_doubles[1])));
  return B200_OK;
}
static int setup_scratch(b200_problem* p, ProblemPlan& P) {
  B200_CUDA(p->d_arena.alloc(p->arena_doubles));
  p->partial_cap = 2 * p->ctx->sm_count * 8;
  B200_CUDA(p->d_partials.alloc(p->partial_cap));
  B200_CUDA(p->d_counters.alloc(4));
  B200_CUDA(cudaMemsetAsync(p->d_counters, 0, 4 * sizeof(unsigned), p->ctx->stream));
  B200_CUDA(p->d_scalars.alloc(1));
  B200_CUDA(cudaMemsetAsync(p->d_scalars, 0, sizeof(Scalars), p->ctx->stream));
  B200_CUDA(p->h_scalars.alloc(1));
  B200_CUDA(p->d_lambda.alloc(1));
  B200_CUDA(cudaMemsetAsync(p->d_lambda, 0, sizeof(double), p->ctx->stream));
  B200_CUDA(p->h_lambda.alloc(1));
  B200_CUDA(p->h_pinned.alloc(std::max<int64_t>(81, std::max(p->nval, p->ndelta))));   // >= 9 x 9: one marginal covariance
  return B200_OK;
}
// Problem creation, shared by the two descriptions: `d` (nonlinear graph + Values, b200_problem_create) or
// `ld` (JacobianFactors, b200_linear_create); exactly one of them is non-null.
static int create_problem(b200_ctx* ctx, const b200_problem_desc* d, const b200_linear_desc* ld, b200_problem** out) {
  if (!ctx || (!d && !ld) || !out) { set_error("null argument"); return B200_INVALID_ARGUMENT; }
  B200_CUDA(cudaSetDevice(ctx->device));
  std::unique_ptr<b200_problem, int (*)(b200_problem*)> p(new b200_problem(), b200_problem_destroy);   // freed on every early return
  p->ctx = ctx; p->linear = ld != nullptr;
  ProblemPlan P{d, ld};
  // B200_SETUP_TIMING=1: where the one-time setup goes (host wall clock per named stage, stderr)
  static const struct { int (*run)(b200_problem*, ProblemPlan&); const char* name; } stages[] = {
      {setup_symbolic, "validate + symbolic phase"}, {setup_values, "values + variable tables"}, {setup_leaf_runs, "shard plan + leaf runs"},
      {setup_offsets, "front offsets"}, {setup_linear_groups, nullptr}, {setup_typed_groups, "factor tables"}, {setup_tree_tables, "tree tables"},
      {setup_leaf_tables, "leaf factor lists + point table"}, {setup_levels, "level plans + dataflow tickets"},
      {setup_values_views, nullptr}, {setup_scratch, nullptr}};
  const bool setup_timing = getenv("B200_SETUP_TIMING") != nullptr;
  auto t_prev = std::chrono::steady_clock::now();
  for (const auto& s : stages) {
    if (const int rc = s.run(p.get(), P)) return rc;
    if (!setup_timing || !s.name) continue;
    const auto now = std::chrono::steady_clock::now();
    fprintf(stderr, "[b200 setup] %-28s %8.1f ms\n", s.name, std::chrono::duration<double, std::milli>(now - t_prev).count());
    t_prev = now;
  }
  B200_CUDA(cudaStreamSynchronize(ctx->stream));
  p->linearized = p->linear;   // a linear problem IS its linearization
  *out = p.release();
  return B200_OK;
}

// [A|b] blocks as the caller holds them (factor-major, column-major blocks) -> staging buffer -> whitened SoA
static int upload_jacobian_group(b200_problem* p, b200_problem::Group& g, const double* Ab, const double* sigmas) {
  p->hdiag_valid = false;
  cudaStream_t st = p->ctx->stream;
  const size_t per = (size_t)g.d * g.ncols, nel = per * (size_t)g.count;
  if (!nel) return B200_OK;
  if (!Ab) { set_error("JacobianFactor group without [A|b] data"); return B200_INVALID_ARGUMENT; }
  std::vector<double> own_Ab, own_sig;   // sharded: the caller passes the whole group, this rank stages its own factors
  if (g.count != g.full_count) {
    own_Ab.resize(nel);
    for (int64_t li = 0; li < g.count; li++) memcpy(own_Ab.data() + (size_t)li * per, Ab + (size_t)g.local_index[li] * per, per * sizeof(double));
    Ab = own_Ab.data();
    if (sigmas) {
      own_sig.resize((size_t)g.count * g.d);
      for (int64_t li = 0; li < g.count; li++) memcpy(own_sig.data() + (size_t)li * g.d, sigmas + (size_t)g.local_index[li] * g.d, (size_t)g.d * sizeof(double));
      sigmas = own_sig.data();
    }
  }
  DevPtr<double> d_stage, d_sig;
  B200_CUDA(upload(d_stage, Ab, nel, st));
  if (sigmas) B200_CUDA(upload(d_sig, sigmas, (size_t)g.count * g.d, st));
  const int nb = (int)std::min<int64_t>(((int64_t)nel + 255) / 256, (int64_t)p->ctx->sm_count * 16);
  launch_plain(jacobian_load_kernel, dim3(nb), dim3(256), 0, st, (const double*)d_stage, (const double*)d_sig, g.d, g.ncols, (int)g.count, g.d_J);
  p->ctx->launches++;
  B200_CUDA(cudaGetLastError());
  B200_CUDA(cudaStreamSynchronize(st));   // the caller's buffers and the staging copies die with this call
  return B200_OK;
}

int b200_problem_create(b200_ctx* ctx, const b200_problem_desc* d, b200_problem** out) {
  if (!d) { set_error("null argument"); return B200_INVALID_ARGUMENT; }
  return create_problem(ctx, d, nullptr, out);
}
int b200_linear_create(b200_ctx* ctx, const b200_linear_desc* d, b200_problem** out) {
  if (!d) { set_error("null argument"); return B200_INVALID_ARGUMENT; }
  return create_problem(ctx, nullptr, d, out);
}
int b200_linear_update_hessian(b200_problem* p, int64_t hi, const double* info) {
  if (!p || !p->linear) { set_error("b200_linear_update_hessian: not a linear problem"); return B200_INVALID_ARGUMENT; }
  int64_t gi = -1;
  for (int64_t q = 0, k = 0; q < (int64_t)p->groups.size(); q++)
    if (p->groups[q].type == B200_FACTOR_HESSIAN && k++ == hi) { gi = q; break; }
  if (hi < 0 || gi < 0) { set_error("HessianFactor group out of range"); return B200_INVALID_ARGUMENT; }
  B200_CUDA(cudaSetDevice(p->ctx->device));
  p->solved = p->factored = p->marg_ready = false;
  return upload_jacobian_group(p, p->groups[gi], info, nullptr);
}
int b200_linear_update(b200_problem* p, int64_t gi, const double* Ab, const double* sigmas) {
  if (!p || !p->linear) { set_error("b200_linear_update: not a linear problem"); return B200_INVALID_ARGUMENT; }
  if (gi < 0 || gi >= (int64_t)p->groups.size() || p->groups[gi].type != B200_FACTOR_JACOBIAN) { set_error("JacobianFactor group out of range"); return B200_INVALID_ARGUMENT; }
  auto& g = p->groups[gi];
  if (sigmas)
    for (int64_t i = 0; i < g.full_count * g.d; i++)
      if (!(sigmas[i] > 0)) { set_error("sigma <= 0: Constrained noise models need QR elimination (out of scope)"); return B200_UNSUPPORTED_NOISE; }
  B200_CUDA(cudaSetDevice(p->ctx->device));
  p->solved = p->factored = p->marg_ready = false;
  return upload_jacobian_group(p, g, Ab, sigmas);
}

int64_t b200_values_size(const b200_problem* p) { return p->nval; }
int64_t b200_delta_size(const b200_problem* p) { return p->ndelta; }

// Page-locked caller buffers (cudaHostAlloc / cudaHostRegister / torch pin_memory) are copied
// directly; pageable ones go through the problem's own pinned staging buffer.
static bool is_pinned_host(const void* ptr) {
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, ptr) != cudaSuccess) { cudaGetLastError(); return false; }
  return a.type == cudaMemoryTypeHost;
}

int b200_set_values(b200_problem* p, const double* v) {
  if (p->linear) { set_error("this call needs Values: not available on a linear problem (b200_linear_create)"); return B200_INVALID_ARGUMENT; }
  B200_CUDA(cudaSetDevice(p->ctx->device));
  const size_t bytes = (size_t)p->nval * sizeof(double);
  const void* src = v;
  if (!is_pinned_host(v)) { memcpy(p->h_pinned, v, bytes); src = p->h_pinned; }
  B200_CUDA(cudaMemcpyAsync(p->d_values, src, bytes, cudaMemcpyHostToDevice, p->ctx->stream));
  B200_CUDA(cudaStreamSynchronize(p->ctx->stream));   // the caller may reuse its buffer on return
  p->linearized = p->solved = p->marg_ready = false;
  return B200_OK;
}
/* New noise models on an existing group: GncOptimizer::makeWeightedGraph (gtsam/nonlinear/GncOptimizer.h:391-411)
 * between outer iterations, without the symbolic phase and the uploads of a new problem. */
int b200_set_group_noise(b200_problem* p, int64_t group, int32_t noise_kind, int32_t noise_per_factor, const double* noise) {
  if (!p) { set_error("null problem"); return B200_INVALID_ARGUMENT; }
  if (p->linear) { set_error("b200_set_group_noise: a linear problem carries its sigmas in b200_linear_update"); return B200_INVALID_ARGUMENT; }
  if (group < 0 || group >= (int64_t)p->groups.size()) { set_error("b200_set_group_noise: group index out of range"); return B200_INVALID_ARGUMENT; }
  auto& g = p->groups[group];
  const int payload = noise_payload(noise_kind, g.d);
  if (payload < 0) { set_error("unsupported noise model (Constrained models need QR: out of scope)"); return B200_UNSUPPORTED_NOISE; }
  if (payload > 0 && !noise) { set_error("b200_set_group_noise: null noise payload"); return B200_INVALID_ARGUMENT; }
  B200_CUDA(cudaSetDevice(p->ctx->device));
  B200_CUDA(cudaStreamSynchronize(p->ctx->stream));
  std::vector<double> h;
  if (noise_per_factor) {   // this rank's factors only (all of them when world == 1)
    h.resize((size_t)g.count * payload);
    for (int64_t li = 0; li < g.count; li++)
      memcpy(h.data() + (size_t)li * payload, noise + (size_t)g.local_index[li] * payload, (size_t)payload * sizeof(double));
  } else {
    h.assign(noise, noise + payload);
  }
  DevPtr<double> fresh;
  B200_CUDA(upload(fresh, h, p->ctx->stream));
  B200_CUDA(cudaStreamSynchronize(p->ctx->stream));   // h goes out of scope
  g.d_noise = std::move(fresh);
  g.noise_kind = noise_kind; g.per_factor = noise_per_factor ? 1 : 0; g.noise_size = payload;
  drop_try_graphs(p);
  p->linearized = p->solved = p->factored = p->marg_ready = false;
  return B200_OK;
}

/* Views of the packed Values of a (sharded) problem: which = 0 the variables this rank needs as INPUT (every variable one of
 * its factors touches + the frontal variables of its cliques and of the top), which = 1 the variables it OWNS (after a step
 * their new values are current here: its own subtrees; rank 0 reports the top).  Ascending variable ids; the packed view is
 * the storage of those variables, concatenated.  With one rank both views are all the variables. */
int b200_values_view(const b200_problem* p, int which, int64_t* nvars, int64_t* ndoubles, int64_t* var_ids) {
  if (!p || which < 0 || which > 1 || p->linear) { set_error("bad argument"); return B200_INVALID_ARGUMENT; }
  if (nvars) *nvars = (int64_t)p->view_vars[which].size();
  if (ndoubles) *ndoubles = p->view_doubles[which];
  if (var_ids && !p->view_vars[which].empty()) memcpy(var_ids, p->view_vars[which].data(), p->view_vars[which].size() * sizeof(int64_t));
  return B200_OK;
}
int b200_set_values_view(b200_problem* p, const double* packed) {
  if (!p || p->linear || !packed) { set_error("bad argument"); return B200_INVALID_ARGUMENT; }
  B200_CUDA(cudaSetDevice(p->ctx->device));
  const int64_t nd = p->view_doubles[0];
  const void* src = packed;
  if (!is_pinned_host(packed)) { memcpy(p->h_pinned, packed, (size_t)nd * sizeof(double)); src = p->h_pinned; }
  B200_CUDA(cudaMemcpyAsync(p->d_view_buf, src, (size_t)nd * sizeof(double), cudaMemcpyHostToDevice, p->ctx->stream));
  launch_plain(values_view_kernel, dim3((unsigned)((nd + 255) / 256)), dim3(256), 0, p->ctx->stream, p->d_values, p->d_view_buf, (const int*)p->d_view_idx[0], nd, 1);
  p->ctx->launches++;
  B200_CUDA(cudaStreamSynchronize(p->ctx->stream));
  p->linearized = p->solved = p->marg_ready = false;
  return B200_OK;
}
int b200_get_values_view(b200_problem* p, double* packed) {
  if (!p || p->linear || !packed) { set_error("bad argument"); return B200_INVALID_ARGUMENT; }
  B200_CUDA(cudaSetDevice(p->ctx->device));
  const int64_t nd = p->view_doubles[1];
  launch_plain(values_view_kernel, dim3((unsigned)((nd + 255) / 256)), dim3(256), 0, p->ctx->stream, p->d_values, p->d_view_buf, (const int*)p->d_view_idx[1], nd, 0);
  p->ctx->launches++;
  const bool direct = is_pinned_host(packed);
  B200_CUDA(cudaMemcpyAsync(direct ? (void*)packed : (void*)p->h_pinned, p->d_view_buf, (size_t)nd * sizeof(double), cudaMemcpyDeviceToHost, p->ctx->stream));
  B200_CUDA(cudaStreamSynchronize(p->ctx->stream));
  if (!direct) memcpy(packed, p->h_pinned, (size_t)nd * sizeof(double));
  return B200_OK;
}

/* The whole packed Values on EVERY rank of a sharded problem (each rank owns a part of the new estimate after a step):
 * the owned views are summed into a zeroed full-size buffer by one all-reduce.  One rank: the same as b200_get_values. */
int b200_get_values_all(b200_problem* p, double* v) {
  if (!p || !v || p->linear) { set_error("bad argument"); return B200_INVALID_ARGUMENT; }
  if (p->ctx->world <= 1) return b200_get_values(p, v);
  B200_CUDA(cudaSetDevice(p->ctx->device));
  cudaStream_t st = p->ctx->stream;
  if (!p->d_gather_buf) B200_CUDA(p->d_gather_buf.alloc(p->nval));
  B200_CUDA(cudaMemsetAsync(p->d_gather_buf, 0, (size_t)p->nval * sizeof(double), st));
  const int64_t nd = p->view_doubles[1];
  launch_plain(values_view_kernel, dim3((unsigned)((nd + 255) / 256)), dim3(256), 0, st, p->d_values, p->d_gather_buf, (const int*)p->d_view_idx[1], nd, 2);
  p->ctx->launches++;
  const int rc = allreduce_sum(p, p->d_gather_buf, (size_t)p->nval);
  if (rc) return rc;
  const bool direct = is_pinned_host(v);
  B200_CUDA(cudaMemcpyAsync(direct ? (void*)v : (void*)p->h_pinned, p->d_gather_buf, (size_t)p->nval * sizeof(double), cudaMemcpyDeviceToHost, st));
  B200_CUDA(cudaStreamSynchronize(st));
  if (!direct) memcpy(v, p->h_pinned, (size_t)p->nval * sizeof(double));
  return B200_OK;
}

int b200_get_values(b200_problem* p, double* v) {
  if (p->linear) { set_error("this call needs Values: not available on a linear problem (b200_linear_create)"); return B200_INVALID_ARGUMENT; }
  B200_CUDA(cudaSetDevice(p->ctx->device));
  const size_t bytes = (size_t)p->nval * sizeof(double);
  const bool direct = is_pinned_host(v);
  B200_CUDA(cudaMemcpyAsync(direct ? (void*)v : (void*)p->h_pinned, p->d_values, bytes, cudaMemcpyDeviceToHost, p->ctx->stream));
  B200_CUDA(cudaStreamSynchronize(p->ctx->stream));
  if (!direct) memcpy(v, p->h_pinned, bytes);
  return B200_OK;
}

int b200_error(b200_problem* p, double* err) {
  if (p->linear) { set_error("this call needs Values: not available on a linear problem (b200_linear_create)"); return B200_INVALID_ARGUMENT; }
  B200_CUDA(cudaSetDevice(p->ctx->device));
  int rc = enqueue_error(p, p->d_values, &p->d_scalars->error);
  if (rc) return rc;
  rc = fetch_scalars(p);
  if (rc) return rc;
  *err = p->h_scalars->error;
  return B200_OK;
}

int b200_linearize(b200_problem* p) {
  if (p->linear) { set_error("this call needs Values: not available on a linear problem (b200_linear_create)"); return B200_INVALID_ARGUMENT; }
  B200_CUDA(cudaSetDevice(p->ctx->device));
  return enqueue_linearize(p);
}

int b200_get_jacobians(b200_problem* p, int64_t gi, double* out) {
  if (gi < 0 || gi >= (int64_t)p->groups.size()) { set_error("group out of range"); return B200_INVALID_ARGUMENT; }
  if (!p->linearized) { set_error("b200_get_jacobians before b200_linearize"); return B200_INVALID_ARGUMENT; }
  B200_CUDA(cudaSetDevice(p->ctx->device));
  auto& g = p->groups[gi];
  const size_t per = (size_t)g.d * g.ncols;
  // the device order of a group is internal (create_problem): the caller's order when the whole group lives on this rank,
  // the rank's own factors in device order when sharded
  const bool whole = !p->linear && (int64_t)g.local_index.size() == g.count && g.count == (int64_t)g.pos.size();
  if (p->jac_f32) {   // stored as floats (b200_set_jacobian_precision): widened for the caller
    std::vector<float> soa(per * g.count);
    B200_CUDA(cudaMemcpyAsync(soa.data(), g.d_J, soa.size() * sizeof(float), cudaMemcpyDeviceToHost, p->ctx->stream));
    B200_CUDA(cudaStreamSynchronize(p->ctx->stream));
    for (int64_t f = 0; f < g.count; f++) {
      const int64_t o = whole ? g.local_index[f] : f;
      for (size_t e = 0; e < per; e++) out[o * per + e] = (double)soa[e * g.count + f];
    }
    return B200_OK;
  }
  std::vector<double> soa(per * g.count);
  B200_CUDA(cudaMemcpyAsync(soa.data(), g.d_J, soa.size() * sizeof(double), cudaMemcpyDeviceToHost, p->ctx->stream));
  B200_CUDA(cudaStreamSynchronize(p->ctx->stream));
  for (int64_t f = 0; f < g.count; f++) {
    const int64_t o = whole ? g.local_index[f] : f;
    for (size_t e = 0; e < per; e++) out[o * per + e] = soa[e * g.count + f];
  }
  return B200_OK;
}

/* "FP32 linearize + FP64 solve" (BASELINE configs[4]): store the whitened Jacobians as floats. */
int b200_set_jacobian_precision(b200_problem* p, int fp32) {
  if (!p) { set_error("null problem"); return B200_INVALID_ARGUMENT; }
  if (p->linear) { set_error("b200_set_jacobian_precision: a linear problem holds the caller's FP64 [A|b]"); return B200_INVALID_ARGUMENT; }
  const bool want = fp32 != 0;
  if (want == p->jac_f32) return B200_OK;
  B200_CUDA(cudaSetDevice(p->ctx->device));
  B200_CUDA(cudaStreamSynchronize(p->ctx->stream));
  // re-allocate at the new element size (the old contents are a stale linearization anyway); on failure nothing changes
  std::vector<DevPtr<double>> fresh(p->groups.size());
  for (size_t i = 0; i < fresh.size(); i++)
    B200_CUDA(fresh[i].alloc((size_t)p->groups[i].count * p->groups[i].d * p->groups[i].ncols, want ? sizeof(float) : sizeof(double)));
  for (size_t i = 0; i < fresh.size(); i++) p->groups[i].d_J = std::move(fresh[i]);
  drop_try_graphs(p);
  p->jac_f32 = want;
  p->linearized = p->solved = p->factored = p->marg_ready = false;
  return B200_OK;
}
int b200_get_jacobian_precision(const b200_problem* p) { return p && p->jac_f32 ? 1 : 0; }

/* Kernel-variant switches of one problem (A/B measurements, profiles/ab_r02.py; every variant computes the same thing). */
int b200_set_tuning(b200_problem* p, const char* key, int64_t value) {
  if (!p || !key) { set_error("null problem / key"); return B200_INVALID_ARGUMENT; }
  const std::string k(key);
  if (k == "schur_mma") p->schur_mma = value != 0;
  else if (k == "lin_variant") p->lin_variant = (int)value;
  else if (k == "factor_staged") {}   // accepted, no effect: the split path stores the point conditionals directly
  else if (k == "schur_pb") p->schur_pb = value == 6 ? 6 : 4;
  else if (k == "df_minb") p->df_minb = value == 3 ? 3 : 2;
  else { set_error("b200_set_tuning: unknown key " + k); return B200_INVALID_ARGUMENT; }
  B200_CUDA(cudaSetDevice(p->ctx->device));
  B200_CUDA(cudaStreamSynchronize(p->ctx->stream));
  drop_try_graphs(p);
  return B200_OK;
}

int b200_hessian_diagonal(b200_problem* p, double* out) {
  if (!p->linearized) { set_error("b200_hessian_diagonal before b200_linearize"); return B200_INVALID_ARGUMENT; }
  B200_CUDA(cudaSetDevice(p->ctx->device));
  int rc = enqueue_hdiag(p);
  if (rc) return rc;
  B200_CUDA(cudaMemcpyAsync(p->h_pinned, p->d_hdiag, (size_t)p->ndelta * sizeof(double), cudaMemcpyDeviceToHost, p->ctx->stream));
  B200_CUDA(cudaStreamSynchronize(p->ctx->stream));
  memcpy(out, p->h_pinned, (size_t)p->ndelta * sizeof(double));
  return B200_OK;
}

/* GaussianFactorGraph::gradientAtZero (gtsam/linear/GaussianFactorGraph.cpp:369-378): -A^T b of the current
 * linearization (typed problems) / of the graph (linear problems), summed over the factors. */
int b200_gradient_at_zero(b200_problem* p, double* out) {
  if (!p || !out) { set_error("null argument"); return B200_INVALID_ARGUMENT; }
  if (!p->linearized) { set_error("b200_gradient_at_zero before b200_linearize"); return B200_INVALID_ARGUMENT; }
  B200_CUDA(cudaSetDevice(p->ctx->device));
  cudaStream_t st = p->ctx->stream;
  if (!p->d_grad) B200_CUDA(p->d_grad.alloc(p->ndelta));
  double* grad = p->d_grad;
  B200_CUDA(cudaMemsetAsync(grad, 0, (size_t)p->ndelta * sizeof(double), st));
  for (auto& g : p->groups) {
    if (!g.count) continue;
    if (g.type == B200_FACTOR_JACOBIAN || g.type == B200_FACTOR_HESSIAN) {
      const int nb = (int)((g.count + 127) / 128);
      if (g.type == B200_FACTOR_JACOBIAN) launch_plain(gradient_jacobian_kernel, dim3(nb), dim3(128), 0, st, jview(g), (const int*)p->d_var_dof, grad);
      else launch_plain(gradient_hessian_kernel, dim3(nb), dim3(128), 0, st, jview(g), (const int*)p->d_var_dof, grad);
    } else {
      const int nb = reduce_blocks(g.count, 256, p->ctx->sm_count);
      DISPATCH_JT(p, DISPATCH_TYPE(g.type, (launch_plain(gradient_kernel<TY, JT>, dim3(nb), dim3(256), 0, st, view(g), (const int*)p->d_var_dof, grad))));
    }
    p->ctx->launches++;
  }
  B200_CUDA(cudaGetLastError());
  const int rc = allreduce_sum(p, grad, (size_t)p->ndelta);   // sharded: every rank summed its own factors
  if (rc) return rc;
  B200_CUDA(cudaMemcpyAsync(p->h_pinned, grad, (size_t)p->ndelta * sizeof(double), cudaMemcpyDeviceToHost, st));
  B200_CUDA(cudaStreamSynchronize(st));
  memcpy(out, p->h_pinned, (size_t)p->ndelta * sizeof(double));
  return B200_OK;
}

static int enqueue_linerr_of(b200_problem* p, const double* x, double bscale, double* out);
/* GaussianFactorGraph::error(x) (gtsam/linear/GaussianFactorGraph.cpp:71-78): sum of 0.5 |A x - b|^2 (JacobianFactor.cpp:479-491)
 * and 0.5 (f - 2 x'g + x'G x) (HessianFactor.cpp:331-346) at the caller's x. */
int b200_linear_graph_error(b200_problem* p, const double* x, double* err) {
  if (!p || !x || !err) { set_error("null argument"); return B200_INVALID_ARGUMENT; }
  if (!p->linearized) { set_error("b200_linear_graph_error before b200_linearize"); return B200_INVALID_ARGUMENT; }
  B200_CUDA(cudaSetDevice(p->ctx->device));
  cudaStream_t st = p->ctx->stream;
  if (!p->d_grad) B200_CUDA(p->d_grad.alloc(p->ndelta));
  memcpy(p->h_pinned, x, (size_t)p->ndelta * sizeof(double));
  B200_CUDA(cudaMemcpyAsync(p->d_grad, p->h_pinned, (size_t)p->ndelta * sizeof(double), cudaMemcpyHostToDevice, st));
  int rc = enqueue_linerr_of(p, p->d_grad, 1.0, &p->d_scalars->graph_err);
  if (rc) return rc;
  rc = allreduce_sum(p, &p->d_scalars->graph_err, 1);   // sharded: every rank summed its own factors
  if (rc) return rc;
  B200_CUDA(cudaMemcpyAsync(p->h_pinned, &p->d_scalars->graph_err, sizeof(double), cudaMemcpyDeviceToHost, st));
  B200_CUDA(cudaStreamSynchronize(st));
  *err = p->h_pinned[0];
  return B200_OK;
}

int b200_solve(b200_problem* p, double lambda, int diagonal, double min_diag, double max_diag, double* e0, double* e1,
               int64_t* fail_var) {
  if (!p->linearized) { set_error("b200_solve before b200_linearize"); return B200_INVALID_ARGUMENT; }
  B200_CUDA(cudaSetDevice(p->ctx->device));
  int rc = reset_flags(p);
  if (rc) return rc;
  rc = set_lambda(p, lambda);
  if (rc) return rc;
  rc = enqueue_solve(p, lambda > 0, diagonal, min_diag, max_diag);
  if (rc) return rc;
  rc = fetch_scalars(p);
  if (rc) return rc;
  if (p->d_df_trace) {   // B200_DF_TRACE=<file>: per-tile globaltimer stamps of the last solve (profiling aid, phase 0 only)
    std::vector<unsigned long long> tr((size_t)p->df_ntasks[0] * 32);
    std::vector<int4> tk((size_t)p->df_ntasks[0]);
    cudaMemcpy(tr.data(), p->d_df_trace, tr.size() * 8, cudaMemcpyDeviceToHost);
    cudaMemcpy(tk.data(), p->d_df_tasks[0], tk.size() * sizeof(int4), cudaMemcpyDeviceToHost);
    if (FILE* fh = fopen(getenv("B200_DF_TRACE"), "wb")) {
      const int64_t nt = p->df_ntasks[0];
      fwrite(&nt, 8, 1, fh); fwrite(tk.data(), sizeof(int4), tk.size(), fh); fwrite(tr.data(), 8, tr.size(), fh);
      fclose(fh);
    }
  }
  if (e0) *e0 = p->h_scalars->lin_err0;
  if (e1) *e1 = p->h_scalars->lin_err_delta;
  rc = solve_status(p, fail_var);
  if (rc) p->marg_ready = false;   // a failed factorisation is no basis for marginals
  return rc;
}

int b200_get_delta(b200_problem* p, double* out) {
  B200_CUDA(cudaSetDevice(p->ctx->device));
  B200_CUDA(cudaMemcpyAsync(p->h_pinned, p->d_delta, (size_t)p->ndelta * sizeof(double), cudaMemcpyDeviceToHost, p->ctx->stream));
  B200_CUDA(cudaStreamSynchronize(p->ctx->stream));
  memcpy(out, p->h_pinned, (size_t)p->ndelta * sizeof(double));
  return B200_OK;
}

int b200_try_step(b200_problem* p, double* new_error) {
  if (p->linear) { set_error("this call needs Values: not available on a linear problem (b200_linear_create)"); return B200_INVALID_ARGUMENT; }
  if (!p->solved) { set_error("b200_try_step before b200_solve"); return B200_INVALID_ARGUMENT; }
  B200_CUDA(cudaSetDevice(p->ctx->device));
  int rc = enqueue_try_step(p);
  if (rc) return rc;
  rc = fetch_scalars(p);
  if (rc) return rc;
  *new_error = p->h_scalars->new_error;
  return B200_OK;
}

int b200_accept_step(b200_problem* p) {
  if (p->linear) { set_error("this call needs Values: not available on a linear problem (b200_linear_create)"); return B200_INVALID_ARGUMENT; }
  B200_CUDA(cudaSetDevice(p->ctx->device));
  // copy, not pointer swap: the captured CUDA graph of the LM try has the buffer roles baked in
  B200_CUDA(cudaMemcpyAsync(p->d_values, p->d_new_values, (size_t)p->nval * sizeof(double), cudaMemcpyDeviceToDevice, p->ctx->stream));
  p->linearized = p->solved = p->marg_ready = false;
  return B200_OK;
}

/* device-side snapshot / restore of Values (benchmarks: reset without host traffic) */
int b200_save_values(b200_problem* p) {
  if (p->linear) { set_error("this call needs Values: not available on a linear problem (b200_linear_create)"); return B200_INVALID_ARGUMENT; }
  B200_CUDA(cudaSetDevice(p->ctx->device));
  if (!p->d_saved_values) B200_CUDA(p->d_saved_values.alloc(p->nval));
  B200_CUDA(cudaMemcpyAsync(p->d_saved_values, p->d_values, (size_t)p->nval * sizeof(double), cudaMemcpyDeviceToDevice, p->ctx->stream));
  return B200_OK;
}
int b200_restore_values(b200_problem* p) {
  if (p->linear) { set_error("this call needs Values: not available on a linear problem (b200_linear_create)"); return B200_INVALID_ARGUMENT; }
  if (!p->d_saved_values) { set_error("b200_restore_values before b200_save_values"); return B200_INVALID_ARGUMENT; }
  B200_CUDA(cudaSetDevice(p->ctx->device));
  B200_CUDA(cudaMemcpyAsync(p->d_values, p->d_saved_values, (size_t)p->nval * sizeof(double), cudaMemcpyDeviceToDevice, p->ctx->stream));
  p->linearized = p->solved = p->marg_ready = false;
  return B200_OK;
}
int b200_synchronize(b200_problem* p) {
  B200_CUDA(cudaSetDevice(p->ctx->device));
  B200_CUDA(cudaStreamSynchronize(p->ctx->stream));
  if (p->profile) resolve_profile(p);
  return B200_OK;
}
int b200_profile_enable(b200_problem* p, int on) {
  p->profile = on != 0;
  if (on == 1) {    // 1: start from zero; 2: resume (the accumulated times stay); 0: pause
    for (int i = 0; i < PH_COUNT; i++) { p->phase_ms[i] = 0; p->phase_calls[i] = 0; }
    p->ev_used = 0;
  }
  return B200_OK;
}
/* Measured FP64 peaks of this device (roofline denominators of the dense-front kernels): TFLOP/s of the tensor path at
 * its widest shape (m16n8k16.f64 on sm_90) and of the FMA pipe, registers only, every SM full; best of 3 launches. */
int b200_measure_fp64_peak(b200_ctx* ctx, double* dmma_tflops, double* dfma_tflops) {
  if (!ctx || !dmma_tflops || !dfma_tflops) { set_error("null argument"); return B200_INVALID_ARGUMENT; }
  B200_CUDA(cudaSetDevice(ctx->device));
  DevPtr<double> sink;
  B200_CUDA(sink.alloc(1));
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  const int iters = 4096, blocks = ctx->sm_count * 8;
  double best[3] = {0, 0, 0};   // indexed by fp64_peak_kernel's mode: FMA, m8n8k4, m16n8k16
  for (int mode = 0; mode < 3; mode++)
    for (int rep = 0; rep < 4; rep++) {
      cudaEventRecord(e0, ctx->stream);
      launch_plain(fp64_peak_kernel, dim3(blocks), dim3(256), 0, ctx->stream, iters, mode, sink);
      cudaEventRecord(e1, ctx->stream);
      B200_CUDA(cudaStreamSynchronize(ctx->stream));
      float ms = 0;
      cudaEventElapsedTime(&ms, e0, e1);
      // per warp and iteration: 32 FMA x 64 flop, 16 m8n8k4 x 512 flop, or 8 m16n8k16 x 4096 flop
      const double per_warp = mode == 0 ? 32.0 * 64.0 : (mode == 1 ? 16.0 * 512.0 : 8.0 * 4096.0);
      const double flop = (double)blocks * 8 * iters * per_warp;
      if (rep > 0 && ms > 0) best[mode] = std::max(best[mode], flop / (ms * 1e-3) / 1e12);
      ctx->launches++;
    }
  cudaEventDestroy(e0); cudaEventDestroy(e1);
  if (getenv("B200_PEAK_VERBOSE"))
    fprintf(stderr, "[b200 fp64 peak] m16n8k16 %.1f, m8n8k4 %.1f, FMA %.1f TFLOP/s\n", best[2], best[1], best[0]);
  *dmma_tflops = std::max(best[1], best[2]); *dfma_tflops = best[0];
  return B200_OK;
}
int b200_profile_phase_count(void) { return PH_COUNT; }
const char* b200_profile_phase_name(int i) {
  static const char* names[PH_COUNT] = {"linearize", "memset_fronts", "assemble", "damp", "eliminate_small",
                                        "eliminate_large", "back_substitute", "linear_error", "retract", "error",
                                        "leaf_fused", "allreduce_top", "linearize_small_groups", "leaf_schur", "backsub_exchange"};
  return (i >= 0 && i < PH_COUNT) ? names[i] : "";
}
int b200_profile_get(b200_problem* p, double* ms, int64_t* calls) {
  for (int i = 0; i < PH_COUNT; i++) { ms[i] = p->phase_ms[i]; calls[i] = p->phase_calls[i]; }
  return B200_OK;
}

// ---- symbolic introspection ------------------------------------------------------
static void fill_info(const Symbolic& S, int64_t ndelta, b200_symbolic_info* info) {
  // the junction tree as the reference builds it (what b200_get_cliques / b200_get_conditional report) ...
  const RefCliques& R = S.ref;
  info->ncliques = R.ncliques; info->nlevels = R.nlevels; info->total_dim = ndelta;
  info->max_frontal_dim = R.max_nf; info->max_separator_dim = R.max_ns;
  info->frontal_list_len = (int64_t)R.front_vars.size(); info->separator_list_len = (int64_t)R.sep_vars.size();
  info->factor_flops = R.flops; info->front_bytes = S.arena_doubles * 8;
  // ... and the supernodes the device eliminates (the same cliques after relaxed amalgamation, symbolic.h)
  info->supernodes = S.ncliques; info->supernode_levels = S.nlevels;
  info->supernode_max_frontal_dim = S.max_nf; info->supernode_max_separator_dim = S.max_ns;
  info->supernode_frontal_list_len = (int64_t)S.front_vars.size(); info->supernode_separator_list_len = (int64_t)S.sep_vars.size();
  info->supernode_flops = S.flops;
}
int b200_symbolic_info_get(const b200_problem* p, b200_symbolic_info* info) {
  fill_info(p->sym, p->ndelta, info);
  info->front_bytes = p->arena_doubles * 8;
  return B200_OK;
}
static void copy_i64(int64_t* dst, const std::vector<int64_t>& v) {   // an empty vector's data() may be null
  if (!v.empty()) memcpy(dst, v.data(), v.size() * sizeof(int64_t));
}
static void fill_cliques(const Symbolic& S, int64_t* fp, int64_t* fv, int64_t* sp, int64_t* sv, int64_t* parent) {
  const RefCliques& R = S.ref;
  copy_i64(fp, R.front_ptr); copy_i64(fv, R.front_vars); copy_i64(sp, R.sep_ptr); copy_i64(sv, R.sep_vars); copy_i64(parent, R.parent);
}
static void fill_supernodes(const Symbolic& S, int64_t* fp, int64_t* fv, int64_t* sp, int64_t* sv, int64_t* parent) {
  copy_i64(fp, S.front_ptr); copy_i64(fv, S.front_vars); copy_i64(sp, S.sep_ptr); copy_i64(sv, S.sep_vars); copy_i64(parent, S.parent);
}
int b200_get_cliques(const b200_problem* p, int64_t* fp, int64_t* fv, int64_t* sp, int64_t* sv, int64_t* parent) {
  fill_cliques(p->sym, fp, fv, sp, sv, parent);
  return B200_OK;
}
int b200_get_supernodes(const b200_problem* p, int64_t* fp, int64_t* fv, int64_t* sp, int64_t* sv, int64_t* parent) {
  fill_supernodes(p->sym, fp, fv, sp, sv, parent);
  return B200_OK;
}
/* conditional [R S d] of (reference) clique c after a solve: nf x (nf+ns+1) column-major.  The clique's rows live in
 * the supernode that absorbed it: its frontal rows, at the columns of its own frontals, its own separator variables
 * (frontals or separator of the supernode) and the rhs; every other column of those rows is structurally zero. */
int b200_get_conditional(b200_problem* p, int64_t c, double* out) {
  const Symbolic& S = p->sym;
  const RefCliques& R = S.ref;
  if (c < 0 || c >= R.ncliques || !p->factored) { set_error("bad clique or no solve yet"); return B200_INVALID_ARGUMENT; }
  B200_CUDA(cudaSetDevice(p->ctx->device));
  const int64_t C = R.super[c];
  const int64_t f = R.nf[c], nn = f + R.ns[c] + 1, ld = p->h_ld[C];
  const int64_t NN = S.nf[C] + S.ns[C] + 1;
  std::vector<double> M((size_t)(ld * NN));
  B200_CUDA(cudaMemcpyAsync(M.data(), p->d_arena + p->h_off[C], M.size() * sizeof(double), cudaMemcpyDeviceToHost, p->ctx->stream));
  B200_CUDA(cudaStreamSynchronize(p->ctx->stream));
  // scalar slot in the supernode of every row / column of the clique
  std::vector<int64_t> slot;
  slot.reserve((size_t)nn);
  auto push_var = [&](int64_t v) -> bool {
    int64_t s0 = -1;
    if (S.var_clique[v] == (int)C) s0 = S.var_slot[v];
    else {
      int64_t k = S.nf[C];
      for (int64_t q = S.sep_ptr[C]; q < S.sep_ptr[C + 1]; q++) {
        if (S.sep_vars[q] == v) { s0 = k; break; }
        k += S.var_dim[S.sep_vars[q]];
      }
    }
    if (s0 < 0) return false;
    for (int t = 0; t < S.var_dim[v]; t++) slot.push_back(s0 + t);
    return true;
  };
  for (int64_t q = R.front_ptr[c]; q < R.front_ptr[c + 1]; q++) if (!push_var(R.front_vars[q])) { set_error("internal: clique variable not in its supernode"); return B200_INVALID_ARGUMENT; }
  for (int64_t q = R.sep_ptr[c]; q < R.sep_ptr[c + 1]; q++) if (!push_var(R.sep_vars[q])) { set_error("internal: clique separator not in its supernode"); return B200_INVALID_ARGUMENT; }
  slot.push_back(NN - 1);
  for (int64_t j = 0; j < nn; j++)
    for (int64_t i = 0; i < f; i++) out[i + j * f] = (i <= j) ? M[(size_t)(slot[i] + slot[j] * ld)] : 0.0;
  return B200_OK;
}
struct b200_symbolic { Symbolic sym; int64_t ndelta; };
int b200_symbolic_create(const b200_problem_desc* d, b200_symbolic** out) {
  Packed pk;
  const int rc = pack_and_symbolic(d, &pk);
  if (rc) return rc;
  b200_symbolic* s = new b200_symbolic();
  s->ndelta = pk.var_dof[d->nvars];
  s->sym = std::move(pk.sym);
  *out = s;
  return B200_OK;
}
int b200_linear_symbolic_create(const b200_linear_desc* d, b200_symbolic** out) {
  Packed pk;
  const int rc = pack_linear(d, &pk);
  if (rc) return rc;
  b200_symbolic* s = new b200_symbolic();
  s->ndelta = pk.var_dof[d->nvars];
  s->sym = std::move(pk.sym);
  *out = s;
  return B200_OK;
}
int b200_symbolic_destroy(b200_symbolic* s) { delete s; return B200_OK; }
int b200_symbolic_get_info(const b200_symbolic* s, b200_symbolic_info* info) { fill_info(s->sym, s->ndelta, info); return B200_OK; }
int b200_symbolic_get_cliques(const b200_symbolic* s, int64_t* fp, int64_t* fv, int64_t* sp, int64_t* sv, int64_t* parent) {
  fill_cliques(s->sym, fp, fv, sp, sv, parent);
  return B200_OK;
}
int b200_symbolic_get_factor_slots(const b200_symbolic* s, int32_t* clique, int32_t* slots) {
  for (size_t i = 0; i < s->sym.fac_clique.size(); i++) clique[i] = s->sym.fac_clique[i];
  for (size_t i = 0; i < s->sym.fac_slots.size(); i++) slots[i] = s->sym.fac_slots[i];
  return B200_OK;
}
int b200_symbolic_get_supernodes(const b200_symbolic* s, int64_t* fp, int64_t* fv, int64_t* sp, int64_t* sv, int64_t* parent) {
  fill_supernodes(s->sym, fp, fv, sp, sv, parent);
  return B200_OK;
}
int b200_symbolic_get_levels(const b200_symbolic* s, int32_t* level) {
  for (int64_t c = 0; c < s->sym.ref.ncliques; c++) level[c] = s->sym.ref.level[c];
  return B200_OK;
}
int b200_symbolic_get_clique_supernode(const b200_symbolic* s, int32_t* super) {
  for (int64_t c = 0; c < s->sym.ref.ncliques; c++) super[c] = s->sym.ref.super[c];
  return B200_OK;
}

/* Host-only: the sharding plan problem creation uses at `world` ranks (SURVEY §8e).
 * clique_owner[c] = owning rank of a clique, -1 for the replicated top;
 * factor_owner[pos] = rank that linearizes the factor at graph position pos. */
int b200_shard_plan(const b200_problem_desc* d, int world, int32_t* clique_owner, int32_t* factor_owner) {
  if (world < 1) { set_error("world < 1"); return B200_INVALID_ARGUMENT; }
  Packed pk;
  const int rc = pack_and_symbolic(d, &pk);
  if (rc) return rc;
  std::vector<char> fused, is_top;
  std::vector<int> co, fo;
  shard_plan(pk.sym, d->ngroups, pk.total, world, &fused, &is_top, &co, &fo);
  for (int64_t c = 0; c < pk.sym.ref.ncliques; c++) clique_owner[c] = co[pk.sym.ref.super[c]];   // per reference clique
  for (size_t i = 0; i < fo.size(); i++) factor_owner[i] = fo[i];
  return B200_OK;
}

int b200_shared_front_buffer(b200_problem* p, void** ptr, int64_t* nd) {
  *ptr = p->d_arena; *nd = p->top_doubles;   // the replicated top fronts = the all-reduced region
  return B200_OK;
}

// ---- LM / GN host control (a17, a18) -----------------------------------------------
void b200_lm_params_legacy(b200_lm_params* P) {
  /* LevenbergMarquardtParams::SetLegacyDefaults, gtsam/nonlinear/LevenbergMarquardtParams.h:69-84 */
  P->max_iterations = 100; P->relative_error_tol = 1e-5; P->absolute_error_tol = 1e-5; P->error_tol = 0.0;
  P->lambda_initial = 1e-5; P->lambda_factor = 10.0; P->lambda_upper_bound = 1e5; P->lambda_lower_bound = 0.0;
  P->min_model_fidelity = 1e-3; P->diagonal_damping = 0; P->use_fixed_lambda_factor = 1;
  P->min_diagonal = 1e-6; P->max_diagonal = 1e32;
}
void b200_lm_params_ceres(b200_lm_params* P) {
  /* ::SetCeresDefaults, :87-99 */
  b200_lm_params_legacy(P);
  P->max_iterations = 50; P->absolute_error_tol = 0; P->relative_error_tol = 1e-6;
  P->lambda_upper_bound = 1e32; P->lambda_lower_bound = 1e-16; P->lambda_initial = 1e-4; P->lambda_factor = 2.0;
  P->min_model_fidelity = 1e-3; P->diagonal_damping = 1; P->use_fixed_lambda_factor = 0;
}

int b200_lm_reset(b200_lm* lm) {
  double e;
  int rc = b200_error(lm->prob, &e);
  if (rc) return rc;
  lm->state.error = e;
  lm->state.lambda = lm->params.lambda_initial;
  lm->state.current_factor = lm->params.lambda_factor;
  lm->state.iterations = 0;
  lm->state.total_inner_iterations = 0;
  return B200_OK;
}
int b200_lm_create(b200_problem* p, const b200_lm_params* params, b200_lm** out) {
  if (p->linear) { set_error("this call needs Values: not available on a linear problem (b200_linear_create)"); return B200_INVALID_ARGUMENT; }
  b200_lm* lm = new b200_lm();
  lm->prob = p;
  lm->params = *params;
  int rc = b200_lm_reset(lm);
  if (rc) { delete lm; return rc; }
  *out = lm;
  return B200_OK;
}
int b200_lm_destroy(b200_lm* lm) { delete lm; return B200_OK; }
int b200_lm_get_state(const b200_lm* lm, b200_lm_state* s) { *s = lm->state; return B200_OK; }

/* LevenbergMarquardtOptimizer::tryLambda (gtsam/nonlinear/LevenbergMarquardtOptimizer.cpp:121-270):
 * one damped solve + retract + error enqueued back to back, ONE host sync, then
 * the reference's accept/reject logic on four scalars.  *done = 1 when the
 * lambda search of this outer iteration is over. */
static int try_lambda(b200_lm* lm, int* done) {
  b200_problem* p = lm->prob;
  const b200_lm_params& P = lm->params;
  b200_lm_state& S = lm->state;
  int rc = set_lambda(p, S.lambda);
  if (rc) return rc;
  rc = launch_try(p, P.diagonal_damping, P.min_diagonal, P.max_diagonal);  // solve + retract + error
  if (rc) return rc;
  rc = fetch_scalars(p);
  if (rc) return rc;
  const bool solved = solve_status(p, nullptr) == B200_OK;
  double modelFidelity = 0.0, newError = INFINITY, costChange = 0.0;
  bool step_is_successful = false, stopSearchingLambda = false;
  if (solved) {
    const double oldLin = p->h_scalars->lin_err0, newLin = p->h_scalars->lin_err_delta;
    const double linearizedCostChange = oldLin - newLin;
    if (linearizedCostChange >= 0) {
      newError = p->h_scalars->new_error;
      costChange = S.error - newError;
      if (linearizedCostChange > std::numeric_limits<double>::epsilon() * oldLin) {
        modelFidelity = costChange / linearizedCostChange;
        step_is_successful = modelFidelity > P.min_model_fidelity;
      }
      const double minAbsoluteTolerance = P.relative_error_tol * S.error;
      if (std::abs(costChange) < minAbsoluteTolerance) stopSearchingLambda = true;
    }
  }
  if (step_is_successful) {
    /* decreaseLambda, internal/LevenbergMarquardtState.h:81-94 */
    double newLambda = S.lambda, newFactor = S.current_factor;
    if (P.use_fixed_lambda_factor) {
      newLambda /= S.current_factor;
    } else {
      newLambda *= std::max(1.0 / 3.0, 1.0 - std::pow(2.0 * modelFidelity - 1.0, 3));
      newFactor = 2.0 * S.current_factor;
    }
    newLambda = std::max(P.lambda_lower_bound, newLambda);
    b200_accept_step(p);
    S.error = newError; S.lambda = newLambda; S.current_factor = newFactor;
    S.iterations += 1; S.total_inner_iterations += 1;
    *done = 1;
  } else if (!stopSearchingLambda) {
    /* increaseLambda, :70-76 */
    S.lambda *= S.current_factor;
    S.total_inner_iterations += 1;
    if (!P.use_fixed_lambda_factor) S.current_factor *= 2.0;
    *done = S.lambda >= P.lambda_upper_bound ? 1 : 0;
  } else {
    *done = 1;
  }
  return B200_OK;
}

int b200_lm_iterate(b200_lm* lm) {
  B200_CUDA(cudaSetDevice(lm->prob->ctx->device));
  int rc = enqueue_linearize(lm->prob);
  if (rc) return rc;
  if (lm->params.diagonal_damping) {     // outside the captured try: one hessianDiagonal per linearization
    rc = enqueue_hdiag(lm->prob);
    if (rc) return rc;
    lm->prob->hdiag_valid = true;
  }
  int done = 0;
  while (!done) {
    rc = try_lambda(lm, &done);
    if (rc) return rc;
  }
  return B200_OK;
}

/* checkConvergence, gtsam/nonlinear/NonlinearOptimizer.cpp:182-231 */
static bool check_convergence(double rel, double absT, double errT, double cur, double nw) {
  if (nw <= errT) return true;
  const double absoluteDecrease = cur - nw;
  const double relativeDecrease = absoluteDecrease / cur;
  return (rel && (relativeDecrease <= rel)) || (absoluteDecrease <= absT);
}

/* NonlinearOptimizer::defaultOptimize, gtsam/nonlinear/NonlinearOptimizer.cpp:62-117 */
int b200_lm_optimize(b200_lm* lm) {
  const b200_lm_params& P = lm->params;
  double currentError = lm->state.error;
  if (currentError <= P.error_tol) return B200_OK;
  if (lm->state.iterations >= P.max_iterations) return B200_OK;
  double newError = currentError;
  do {
    currentError = newError;
    int rc = b200_lm_iterate(lm);
    if (rc) return rc;
    newError = lm->state.error;
  } while (lm->state.iterations < P.max_iterations &&
           !check_convergence(P.relative_error_tol, P.absolute_error_tol, P.error_tol, currentError, newError) &&
           std::isfinite(currentError));
  return B200_OK;
}

/* GaussNewtonOptimizer::iterate, gtsam/nonlinear/GaussNewtonOptimizer.cpp:44-67 */
int b200_gn_iterate(b200_problem* p, double* new_error) {
  if (p->linear) { set_error("this call needs Values: not available on a linear problem (b200_linear_create)"); return B200_INVALID_ARGUMENT; }
  B200_CUDA(cudaSetDevice(p->ctx->device));
  int rc = enqueue_linearize(p);
  if (rc) return rc;
  rc = reset_flags(p);
  if (rc) return rc;
  rc = set_lambda(p, 0.0);
  if (rc) return rc;
  rc = enqueue_solve(p, false, 0, 0, 0);
  if (rc) return rc;
  rc = enqueue_try_step(p);
  if (rc) return rc;
  rc = fetch_scalars(p);
  if (rc) return rc;
  int64_t fv;
  rc = solve_status(p, &fv);
  if (rc) { set_error("indeterminate linear system near variable " + std::to_string(fv)); return rc; }
  b200_accept_step(p);
  if (new_error) *new_error = p->h_scalars->new_error;
  return B200_OK;
}

// ---- Marginals ---------------------------------------------------------------------------
// the undamped factor of H at the current values, computed once and reused until the values change
static int prepare_marginals(b200_problem* p) {
  if (p->marg_ready) return B200_OK;
  int rc = enqueue_linearize(p);
  if (rc) return rc;
  rc = reset_flags(p);
  if (rc) return rc;
  rc = set_lambda(p, 0.0);
  if (rc) return rc;
  rc = enqueue_solve(p, false, 0, 0, 0);
  if (rc) return rc;
  rc = fetch_scalars(p);
  if (rc) return rc;
  int64_t fv;
  rc = solve_status(p, &fv);
  if (rc) { p->marg_ready = false; set_error("indeterminate linear system near variable " + std::to_string(fv)); return rc; }
  return B200_OK;
}

int b200_marginal_covariance(b200_problem* p, int64_t var, double* out) {
  b200_ctx* ctx = p->ctx;
  if (ctx->world > 1) { set_error("marginals are single-GPU: create the problem on a context without a communicator"); return B200_INVALID_ARGUMENT; }
  if (var < 0 || var >= p->nvars) { set_error("b200_marginal_covariance: variable id out of range"); return B200_INVALID_ARGUMENT; }
  B200_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  { const int rc = prepare_marginals(p); if (rc) return rc; }
  const Symbolic& S = p->sym;
  std::vector<int> path;
  for (int c = S.var_clique[var]; c >= 0; c = S.parent[c]) {
    if (S.nf[c] > kMargMaxF) { set_error("b200_marginal_covariance: a clique on the path has more than 4096 pivots"); return B200_INVALID_ARGUMENT; }
    path.push_back(c);
  }
  const int d = (int)(S.var_dof[var + 1] - S.var_dof[var]);
  if (d > 9) { set_error("b200_marginal_covariance: variable dimension > 9 (use b200_joint_marginal_covariance)"); return B200_INVALID_ARGUMENT; }
  if (!p->d_marg_work) B200_CUDA(p->d_marg_work.alloc((size_t)9 * std::max<int64_t>(1, p->ndelta)));
  if (!p->d_marg_path) B200_CUDA(p->d_marg_path.alloc(S.ncliques));
  if (!p->d_marg_out) B200_CUDA(p->d_marg_out.alloc(81));
  B200_CUDA(cudaMemcpyAsync(p->d_marg_path, path.data(), path.size() * sizeof(int), cudaMemcpyHostToDevice, st));
  B200_CUDA(cudaStreamSynchronize(st));   // `path` is pageable and dies with this call
  launch_plain(marginal_path_kernel, dim3(d), dim3(256), 0, st, tview(p), (const int*)p->d_marg_path, (int)path.size(), (int)S.var_dof[var], d,
               p->d_marg_work, p->ndelta, p->d_marg_out);
  ctx->launches++;
  B200_CUDA(cudaGetLastError());
  B200_CUDA(cudaMemcpyAsync(p->h_pinned, p->d_marg_out, (size_t)d * d * sizeof(double), cudaMemcpyDeviceToHost, st));
  B200_CUDA(cudaStreamSynchronize(st));
  memcpy(out, p->h_pinned, (size_t)d * d * sizeof(double));
  return B200_OK;
}

int b200_joint_marginal_covariance(b200_problem* p, const int64_t* vars, int64_t nv, double* out) {
  b200_ctx* ctx = p->ctx;
  if (ctx->world > 1) { set_error("marginals are single-GPU: create the problem on a context without a communicator"); return B200_INVALID_ARGUMENT; }
  if (nv <= 0) { set_error("b200_joint_marginal_covariance: no variables"); return B200_INVALID_ARGUMENT; }
  const Symbolic& S = p->sym;
  std::vector<int> dofs;
  for (int64_t a = 0; a < nv; a++) {
    if (vars[a] < 0 || vars[a] >= p->nvars || (a > 0 && vars[a] <= vars[a - 1])) {
      set_error("b200_joint_marginal_covariance: variable ids must be in range, distinct and ascending");
      return B200_INVALID_ARGUMENT;
    }
    for (int64_t q = S.var_dof[vars[a]]; q < S.var_dof[vars[a] + 1]; q++) dofs.push_back((int)q);
  }
  const int D = (int)dofs.size();
  if (D > 128) { set_error("b200_joint_marginal_covariance: more than 128 scalar dimensions requested"); return B200_INVALID_ARGUMENT; }
  B200_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  { const int rc = prepare_marginals(p); if (rc) return rc; }
  std::vector<char> on(S.ncliques, 0);
  for (int64_t a = 0; a < nv; a++)
    for (int c = S.var_clique[vars[a]]; c >= 0 && !on[c]; c = S.parent[c]) {
      if (S.nf[c] > kMargMaxF) { set_error("b200_joint_marginal_covariance: a clique on the path has more than 4096 pivots"); return B200_INVALID_ARGUMENT; }
      on[c] = 1;
    }
  std::vector<int> path;
  for (int c = 0; c < (int)S.ncliques; c++)
    if (on[c]) path.push_back(c);   // ascending clique id = elimination order
  DevPtr<double> d_work, d_out;
  DevPtr<int> d_path, d_dofs;
  B200_CUDA(d_work.alloc((size_t)D * std::max<int64_t>(1, p->ndelta)));
  B200_CUDA(d_out.alloc((size_t)D * D));
  B200_CUDA(upload(d_path, path, st));
  B200_CUDA(upload(d_dofs, dofs, st));
  B200_CUDA(cudaStreamSynchronize(st));
  launch_plain(marginal_joint_kernel, dim3(D), dim3(256), 0, st, tview(p), (const int*)d_path, (int)path.size(), (const int*)d_dofs, D, d_work,
               p->ndelta, d_out);
  ctx->launches++;
  B200_CUDA(cudaGetLastError());
  B200_CUDA(cudaMemcpyAsync(out, d_out, (size_t)D * D * sizeof(double), cudaMemcpyDeviceToHost, st));
  B200_CUDA(cudaStreamSynchronize(st));
  return B200_OK;
}

// ---- Dogleg ------------------------------------------------------------------------------
int b200_dl_create(b200_problem* p, double delta_initial, b200_dl** out) {
  // the sharded solve leaves each rank with its own slice of delta; Dogleg's global dot products
  // over dx_u / dx_n are not wired for that layout
  if (p->ctx->world > 1) { set_error("Dogleg is single-GPU: create the problem on a context without a communicator"); return B200_INVALID_ARGUMENT; }
  if (p->linear) { set_error("this call needs Values: not available on a linear problem (b200_linear_create)"); return B200_INVALID_ARGUMENT; }
  B200_CUDA(cudaSetDevice(p->ctx->device));
  std::unique_ptr<b200_dl> dl(new b200_dl);
  dl->prob = p;
  dl->delta = delta_initial;
  dl->iterations = 0;
  B200_CUDA(dl->d_grad.alloc(p->ndelta));
  B200_CUDA(dl->d_dxn.alloc(p->ndelta));
  const int rc = b200_error(p, &dl->error);
  if (rc) return rc;
  *out = dl.release();
  return B200_OK;
}
int b200_dl_destroy(b200_dl* dl) { delete dl; return B200_OK; }
int b200_dl_get_state(const b200_dl* dl, double* error, double* delta, int32_t* iterations) {
  if (error) *error = dl->error;
  if (delta) *delta = dl->delta;
  if (iterations) *iterations = dl->iterations;
  return B200_OK;
}

// 0.5*|A x - bscale*b|^2 into *out
static int enqueue_linerr_of(b200_problem* p, const double* x, double bscale, double* out) {
  b200_ctx* ctx = p->ctx;
  cudaStream_t st = ctx->stream;
  bool first = true;
  for (auto& g : p->groups) {
    if (!g.count) continue;
    const int nb = reduce_blocks(g.count, 256, ctx->sm_count);
    double* p0 = p->d_partials;
    double* p1 = p->d_partials + p->partial_cap / 2;
    if (g.type == B200_FACTOR_JACOBIAN)
      launch_k(linerr_jacobian_kernel, dim3(nb), dim3(256), 0, st, jview(g), x, (const int*)p->d_var_dof, p0, p1, p->d_counters + 1, &p->d_scalars->dl_scratch, out,
               first ? 0 : 1, bscale);
    else if (g.type == B200_FACTOR_HESSIAN)
      launch_k(linerr_hessian_kernel, dim3(nb), dim3(256), 0, st, jview(g), x, (const int*)p->d_var_dof, p0, p1, p->d_counters + 1, &p->d_scalars->dl_scratch, out,
               first ? 0 : 1, bscale);
    else
    DISPATCH_JT(p, DISPATCH_TYPE(g.type, (launch_k(linerr_kernel<TY, JT>, dim3(nb), dim3(256), 0, st, view(g), x, p->d_var_dof, p0, p1, p->d_counters + 1,
                                    &p->d_scalars->dl_scratch, out, first ? 0 : 1, bscale))));
    ctx->launches += 1;
    first = false;
  }
  if (first) B200_CUDA(cudaMemsetAsync(out, 0, sizeof(double), st));
  B200_CUDA(cudaGetLastError());
  return B200_OK;
}

int b200_dl_iterate(b200_dl* dl) {
  b200_problem* p = dl->prob;
  b200_ctx* ctx = p->ctx;
  cudaStream_t st = ctx->stream;
  B200_CUDA(cudaSetDevice(ctx->device));
  const int64_t n = p->ndelta;
  int rc = enqueue_linearize(p);
  if (rc) return rc;
  rc = reset_flags(p);
  if (rc) return rc;
  rc = set_lambda(p, 0.0);
  if (rc) return rc;
  rc = enqueue_solve(p, false, 0, 0, 0);     // d_delta = dx_n, lin_err0 = M(0)
  if (rc) return rc;
  B200_CUDA(cudaMemcpyAsync(dl->d_dxn, p->d_delta, (size_t)n * sizeof(double), cudaMemcpyDeviceToDevice, st));
  // gradientAtZero and |A g|^2
  B200_CUDA(cudaMemsetAsync(dl->d_grad, 0, (size_t)n * sizeof(double), st));
  for (auto& g : p->groups) {
    if (!g.count) continue;
    const int nb = reduce_blocks(g.count, 256, ctx->sm_count);
    DISPATCH_JT(p, DISPATCH_TYPE(g.type, (launch_plain(gradient_kernel<TY, JT>, dim3(nb), dim3(256), 0, st, view(g), (const int*)p->d_var_dof, dl->d_grad))));
    ctx->launches++;
  }
  B200_CUDA(cudaGetLastError());
  launch_plain(dot3_kernel, dim3(1), dim3(1024), 0, st, (const double*)dl->d_grad, (const double*)dl->d_dxn, n, p->d_scalars->dl_dots);
  ctx->launches++;
  rc = enqueue_linerr_of(p, dl->d_grad, 0.0, &p->d_scalars->dl_half_Ag2);
  if (rc) return rc;
  rc = fetch_scalars(p);
  if (rc) return rc;
  int64_t fv;
  rc = solve_status(p, &fv);
  if (rc) { set_error("indeterminate linear system near variable " + std::to_string(fv)); return rc; }
  const Scalars* s = p->h_scalars;
  const double gg = s->dl_dots[0], gn = s->dl_dots[1], nn = s->dl_dots[2];
  const double step = -gg / (2.0 * s->dl_half_Ag2);          // GaussianFactorGraph.cpp:397-403
  const double uu = step * step * gg, un = step * gn;
  const double f_error = dl->error, M_error = s->lin_err0;
  double delta = dl->delta, new_f = f_error;
  bool stay = true, zero_step = false;
  while (stay) {
    // ComputeDoglegPoint, DoglegOptimizerImpl.cpp:25-78
    double ca, cb;
    const double deltaSq = delta * delta;
    if (deltaSq < uu) { ca = std::sqrt(deltaSq / uu); cb = 0; }
    else if (deltaSq < nn) {
      const double a = uu - 2. * un + nn, b = 2. * (un - uu), c = uu - deltaSq;
      const double sq = std::sqrt(b * b - 4 * a * c);
      const double tau1 = (-b + sq) / (2. * a), tau2 = (-b - sq) / (2. * a);
      const double eps = std::numeric_limits<double>::epsilon();
      const double tau = (-eps <= tau1 && tau1 <= 1.0 + eps) ? tau1 : tau2;
      ca = 1. - tau; cb = tau;
    } else { ca = 0; cb = 1; }
    launch_plain(blend_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, st, (const double*)dl->d_grad, (const double*)dl->d_dxn, ca * step, cb, n, p->d_delta);
    ctx->launches++;
    B200_CUDA(cudaGetLastError());
    rc = enqueue_try_step(p);
    if (rc) return rc;
    rc = enqueue_linerr_of(p, p->d_delta, 1.0, &p->d_scalars->lin_err_delta);
    if (rc) return rc;
    rc = fetch_scalars(p);
    if (rc) return rc;
    new_f = s->new_error;
    const double new_M = s->lin_err_delta;
    const double rho = (std::fabs(f_error - new_f) < 1e-15 || std::fabs(M_error - new_M) < 1e-15)
                           ? 0.5 : (f_error - new_f) / (M_error - new_M);
    if (rho >= 0.75) {
      const double nd = std::sqrt(ca * ca * uu + 2. * ca * cb * un + cb * cb * nn);
      delta = std::max(delta, 3.0 * nd);
      stay = false;
    } else if (rho >= 0.25) {
      stay = false;
    } else if (rho >= 0.0) {
      if (delta > 1e-5) delta = 0.5 * delta;
      stay = false;
    } else {   // includes NaN
      if (delta > 1e-5) { delta *= 0.5; stay = true; }
      else { zero_step = true; new_f = f_error; stay = false; }
    }
  }
  if (!zero_step) b200_accept_step(p);
  else {
    B200_CUDA(cudaMemsetAsync(p->d_delta, 0, (size_t)n * sizeof(double), st));   // the reference leaves dx_d = 0 (DoglegOptimizerImpl.h:232-237)
    p->linearized = p->solved = p->marg_ready = false;
  }
  dl->error = new_f;
  dl->delta = delta;
  dl->iterations++;
  return B200_OK;
}

}  // extern "C"
