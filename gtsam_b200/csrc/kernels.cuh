// kernels.cuh — the sm_90a kernels of the hot path (FP64).  Reference rows of SURVEY.md §8(a):
//
//  linearize_kernel      a1-a7   residual + Jacobian + whitening (+ robust reweighting), one thread per
//                                factor, element-major SoA stores => every store instruction coalesced
//  error_kernel          a8      0.5*|R r|^2 or rho(|R r|); single launch, last-block reduction in index order
//  leaf_point_fused_mma_kernel<DC,..>  a10+a12+a13+a14  BAL point cliques, one CTA per run of points with the same
//                                cameras: per point assemble + damp + 3x3 Cholesky (8 lanes per point), the run's Schur
//                                complement as FP64 DMMA tiles, one extend-add per run
//  leaf_point_factor_kernel<DC>, leaf_point_schur_kernel<DC,..>  the same in two kernels (schur_mma = 0): per point,
//                                then the per-run SYRK in 3x3 register tiles
//  leaf_fused_kernel     a10+a12+a13+a14  any leaf clique with a small frontal block
//  assemble_kernel       a12     J^T J / J^T b / b^T b scatter-add into the owning non-leaf front
//  hdiag_kernel, damp_kernel  a10  hessianDiagonal; lambda*I or lambda*clip(diag H) on the diagonal
//  elim_small_kernel     a13/14  one warp per small non-leaf front in shared memory, fused extend-add
//  panel_kernel          a13     32x32 diagonal Cholesky (one warp, registers + shuffles) + TRSM of the row panel
//  update_kernel, update_dmma_kernel  a13  C -= S^T S on the upper trapezoid (FP64 FMA tiles / DMMA for big fronts)
//  extend_add_kernel     a12     child Schur complement into the parent front
//  backsub_point_kernel<DC>, backsub_small_kernel, backsub_large_kernel  a15  x_F = R^-1 (d - S x_S), level by level
//  linerr_kernel         a16     0.5*|A delta - b|^2 and 0.5*|b|^2 in one pass
//  retract_kernel        a9      x (+) delta per variable
//  assemble_hessian_kernel, hdiag_hessian_kernel, linerr_hessian_kernel   the same for HessianFactor groups
//  jacobian_load_kernel, assemble_jacobian_kernel, hdiag_jacobian_kernel, linerr_jacobian_kernel,
//  gradient_jacobian_kernel, gradient_hessian_kernel (GaussianFactorGraph::gradientAtZero)
//                                a12/a10/a16 for the JacobianFactor groups (any arity / block widths) of a linear problem
//                                (GaussianFactorGraph::optimize level, b200_linear_create)
//  gradient_kernel, dot3_kernel, blend_kernel        Dogleg (8f rank 3): gradientAtZero, dot products, dogleg point
//  marginal_path_kernel, marginal_joint_kernel        Marginals (8f rank 3): forward/back solves along clique paths
#pragma once
#include <climits>

#include "engine.cuh"
#ifdef B200_EMULATE
#include "cuda_emu_full.h"   // tests/emu: host model of the CUDA execution for the test-only emulation build (DESIGN.md 7i)
#define B200_DYN_SMEM(T, name) T* name = (T*)b200_emu::dyn_smem()
#else
#define B200_DYN_SMEM(T, name) extern __shared__ T name[]
#endif
#include "factors.cuh"

namespace b200 {

constexpr int kSmallMaxN = 48;   // fronts up to this size run one-warp-per-clique
constexpr int kWarpsPerBlock = 4;
constexpr int kNB = 32;          // panel width of the blocked large-front path
constexpr int kTile = 64;        // SYRK tile
constexpr int kLeafMaxF = 6;     // leaf cliques up to this frontal dim take the fused path
constexpr int kLeafMaxFN = 768;  // doubles of [F S d] staged per warp in shared memory
constexpr int kMaxGroups = 8;    // factor groups addressable by the fused leaf kernel

struct GroupTable { GroupView g[kMaxGroups]; };
__constant__ int kFD[B200_NUM_FACTOR_TYPES] = {6, 6, 3, 2, 2, 9, 3, 3};
__constant__ int kFN1[B200_NUM_FACTOR_TYPES] = {6, 6, 3, 6, 9, 9, 3, 3};
__constant__ int kFN2[B200_NUM_FACTOR_TYPES] = {6, 0, 0, 3, 3, 0, 3, 0};
// column pairs (ca <= cb) of a factor's [A1 A2 b] block, per factor type (filled at ctx creation)
constexpr int kMaxPairs = 96;   // 13*14/2 = 91
// (global memory, read through L1: the index differs per lane, which would serialise in the constant cache)
__device__ unsigned char kPairA[B200_NUM_FACTOR_TYPES][kMaxPairs];
__device__ unsigned char kPairB[B200_NUM_FACTOR_TYPES][kMaxPairs];

// ---------------------------------------------------------------------------
// Programmatic dependent launch: every kernel of the LM try is launched with
// cudaLaunchAttributeProgrammaticStreamSerialization, so its CTAs are scheduled while the
// previous kernel is still draining; it must therefore wait here before touching anything the
// previous kernel wrote, and it immediately lets the NEXT kernel start its own launch.  The
// try is a chain of ~50-300 small dependent kernels: the kernel-boundary latency, not the
// kernels, is what this hides.  No-ops when the kernel was launched without the attribute.
// ---------------------------------------------------------------------------
__device__ __forceinline__ void pdl_sync() {
#if defined(__CUDA_ARCH__) && __CUDA_ARCH__ >= 900
  cudaGridDependencySynchronize();
  cudaTriggerProgrammaticLaunchCompletion();
#endif
}

// ---------------------------------------------------------------------------
// block reduction helpers
// ---------------------------------------------------------------------------
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  return v;
}
template <int NT>
__device__ __forceinline__ double block_sum(double v, double* sh) {
  v = warp_sum(v);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (lane == 0) sh[w] = v;
  __syncthreads();
  double r = 0;
  if (w == 0) {
    r = lane < NT / 32 ? sh[lane] : 0.0;
    r = warp_sum(r);
  }
  __syncthreads();
  return r;  // valid in thread 0
}

// Deterministic single-launch reduction: every block writes its partial, the LAST block to
// finish (atomic ticket) adds them up in index order, so the result does not depend on the
// order in which blocks ran.  `counter` must be 0 on entry and is reset for the next use.
__device__ __forceinline__ void finish_sum(double block_value, double* partials, unsigned* counter, double* out,
                                           int accumulate, double* sh) {
  __shared__ bool last;
  __syncthreads();   // `last` may still be read by a previous call in the same kernel
  if (threadIdx.x == 0) {
    partials[blockIdx.x] = block_value;
    __threadfence();
    last = atomicInc(counter, gridDim.x - 1) == gridDim.x - 1;   // wraps back to 0
  }
  __syncthreads();
  if (!last) return;
  __threadfence();
  double s = 0;
  for (int i = threadIdx.x; i < (int)gridDim.x; i += blockDim.x) s += __ldcg(partials + i);
  s = block_sum<256>(s, sh);
  if (threadIdx.x == 0) *out = accumulate ? (*out + s) : s;
}

// ---------------------------------------------------------------------------
// linearize
// ---------------------------------------------------------------------------
// JT = storage type of the whitened Jacobians: double, or float for the "FP32 linearize + FP64 solve" mode of
// BASELINE configs[4] (b200_set_jacobian_precision): the math stays FP64 in registers, the element-major SoA holds
// floats (half the HBM traffic of the two bandwidth-bound phases); every consumer widens back to FP64 on load.
// MINB: resident CTAs per SM the kernel is compiled for.  The 2-row projection factors default to 8 (64 registers: ptxas
// spills 160 bytes of the 20-entry block) — variant 4 (128 registers, no spills) is switched in by b200_set_tuning("lin_variant").
template <int TYPE, typename JT = double, int MINB = (FactorTraits<TYPE>::D <= 3 ? 8 : 2)>
__global__ void __launch_bounds__(128, MINB) linearize_kernel(GroupView g, EvalCtx c) {
  pdl_sync();
  typedef FactorTraits<TYPE> FT;
  enum { D = FT::D, NC = FT::N1 + FT::N2 + 1 };
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= g.count) return;
  const int2 k = g.keys[f];
  double M[D * NC];
  Eval<TYPE, true>::run(c, k.x, k.y, g.meas + (size_t)f * FT::MEAS, g.cal_index ? g.cal_index[f] : 0, g.body, M);
  whiten<D, NC, 0>(M, g.noise_kind, g.noise + (g.per_factor ? (size_t)f * g.noise_size : 0));
  if (g.robust_kind) {   // Robust::WhitenSystem: scale A and b by sqrt(w(|b|)) (Block reweighting)
    double nrm = 0;
#pragma unroll
    for (int r = 0; r < D; r++) nrm += M[r * NC + NC - 1] * M[r * NC + NC - 1];
    const double w = sqrt(robust_weight(g.robust_kind, g.robust_param, sqrt(nrm)));
#pragma unroll
    for (int e = 0; e < D * NC; e++) M[e] *= w;
  }
  JT* J = reinterpret_cast<JT*>(g.J) + f;
#pragma unroll
  for (int cc = 0; cc < NC; cc++)
#pragma unroll
    for (int r = 0; r < D; r++) J[(size_t)(r + cc * D) * g.count] = (JT)M[r * NC + cc];
}

// ---------------------------------------------------------------------------
// nonlinear error: partial sums of 0.5*|whiten(r)|^2
// ---------------------------------------------------------------------------
template <int TYPE>
__global__ void __launch_bounds__(256) error_kernel(GroupView g, EvalCtx c, double* partials, unsigned* counter,
                                                    double* out, int accumulate) {
  pdl_sync();
  typedef FactorTraits<TYPE> FT;
  enum { D = FT::D, NC = FT::N1 + FT::N2 + 1 };
  __shared__ double sh[32];
  double acc = 0;
  for (int f = blockIdx.x * blockDim.x + threadIdx.x; f < g.count; f += gridDim.x * blockDim.x) {
    const int2 k = g.keys[f];
    double M[D * NC];
    Eval<TYPE, false>::run(c, k.x, k.y, g.meas + (size_t)f * FT::MEAS, g.cal_index ? g.cal_index[f] : 0, g.body, M);
    whiten<D, NC, NC - 1>(M, g.noise_kind, g.noise + (g.per_factor ? (size_t)f * g.noise_size : 0));
    double s = 0;
#pragma unroll
    for (int r = 0; r < D; r++) s += M[r * NC + NC - 1] * M[r * NC + NC - 1];
    acc += g.robust_kind ? robust_loss(g.robust_kind, g.robust_param, sqrt(s)) : 0.5 * s;
  }
  acc = block_sum<256>(acc, sh);
  finish_sum(acc, partials, counter, out, accumulate, sh);
}

// ---------------------------------------------------------------------------
// linear error on the undamped linearization
// ---------------------------------------------------------------------------
template <int TYPE, typename JT = double>
__global__ void __launch_bounds__(256) linerr_kernel(GroupView g, const double* __restrict__ delta,
                                                     const int* __restrict__ var_dof, double* p0, double* p1,
                                                     unsigned* counters, double* out0, double* out1, int accumulate,
                                                     double bscale) {
  // bscale = 1: 0.5*|A delta - b|^2; bscale = 0: 0.5*|A delta|^2 (Dogleg's |R g|^2)
  pdl_sync();
  typedef FactorTraits<TYPE> FT;
  enum { D = FT::D, N1 = FT::N1, N2 = FT::N2, NC = N1 + N2 + 1 };
  __shared__ double sh[32];
  double a0 = 0, a1 = 0;
  for (int f = blockIdx.x * blockDim.x + threadIdx.x; f < g.count; f += gridDim.x * blockDim.x) {
    const int2 k = g.keys[f];
    const JT* J = reinterpret_cast<const JT*>(g.J) + f;
    double e[D], b[D];
#pragma unroll
    for (int r = 0; r < D; r++) { b[r] = J[(size_t)(r + (NC - 1) * D) * g.count]; e[r] = -bscale * b[r]; }
    const double* d0 = delta + var_dof[k.x];
#pragma unroll
    for (int cc = 0; cc < N1; cc++) {
      const double x = d0[cc];
#pragma unroll
      for (int r = 0; r < D; r++) e[r] += J[(size_t)(r + cc * D) * g.count] * x;
    }
    if (N2 > 0) {
      const double* d1 = delta + var_dof[k.y];
#pragma unroll
      for (int cc = 0; cc < N2; cc++) {
        const double x = d1[cc];
#pragma unroll
        for (int r = 0; r < D; r++) e[r] += J[(size_t)(r + (N1 + cc) * D) * g.count] * x;
      }
    }
    double s0 = 0, s1 = 0;
#pragma unroll
    for (int r = 0; r < D; r++) { s0 += b[r] * b[r]; s1 += e[r] * e[r]; }
    a0 += 0.5 * s0;
    a1 += 0.5 * s1;
  }
  a0 = block_sum<256>(a0, sh);
  a1 = block_sum<256>(a1, sh);
  finish_sum(a0, p0, counters, out0, accumulate, sh);
  finish_sum(a1, p1, counters + 1, out1, accumulate, sh);
}

// ---------------------------------------------------------------------------
// Dogleg support (gtsam/linear/GaussianFactorGraph.cpp:381-407 optimizeGradientSearch,
// gtsam/nonlinear/DoglegOptimizerImpl.cpp:25-98): gradientAtZero = -A^T b per variable,
// the three dot products of the steepest-descent and Newton points, and the blend.
// ---------------------------------------------------------------------------
template <int TYPE, typename JT = double>
__global__ void __launch_bounds__(256) gradient_kernel(GroupView g, const int* __restrict__ var_dof, double* grad) {
  typedef FactorTraits<TYPE> FT;
  enum { D = FT::D, N1 = FT::N1, N2 = FT::N2, NC = N1 + N2 + 1 };
  for (int f = blockIdx.x * blockDim.x + threadIdx.x; f < g.count; f += gridDim.x * blockDim.x) {
    const int2 k = g.keys[f];
    const JT* J = reinterpret_cast<const JT*>(g.J) + f;
    double b[D];
#pragma unroll
    for (int r = 0; r < D; r++) b[r] = J[(size_t)(r + (NC - 1) * D) * g.count];
    double* g0 = grad + var_dof[k.x];
#pragma unroll
    for (int cc = 0; cc < N1; cc++) {
      double s = 0;
#pragma unroll
      for (int r = 0; r < D; r++) s += J[(size_t)(r + cc * D) * g.count] * b[r];
      atomicAdd(g0 + cc, -s);
    }
    if (N2 > 0) {
      double* g1 = grad + var_dof[k.y];
#pragma unroll
      for (int cc = 0; cc < N2; cc++) {
        double s = 0;
#pragma unroll
        for (int r = 0; r < D; r++) s += J[(size_t)(r + (N1 + cc) * D) * g.count] * b[r];
        atomicAdd(g1 + cc, -s);
      }
    }
  }
}

// out[0..2] = {u.u, u.n, n.n}; one block, fixed summation order
__global__ void __launch_bounds__(1024) dot3_kernel(const double* __restrict__ u, const double* __restrict__ n, int64_t count,
                                                    double* out) {
  __shared__ double sh[32];
  double a = 0, b = 0, c = 0;
  for (int64_t i = threadIdx.x; i < count; i += 1024) {
    const double x = u[i], y = n[i];
    a += x * x; b += x * y; c += y * y;
  }
  a = block_sum<1024>(a, sh);
  b = block_sum<1024>(b, sh);
  c = block_sum<1024>(c, sh);
  if (threadIdx.x == 0) { out[0] = a; out[1] = b; out[2] = c; }
}

// out = ca*u + cb*n (ComputeBlend); ca == 0 / cb == 0 select the pure points exactly
__global__ void blend_kernel(const double* __restrict__ u, const double* __restrict__ n, double ca, double cb, int64_t count,
                             double* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  out[i] = cb == 0.0 ? ca * u[i] : (ca == 0.0 ? cb * n[i] : ca * u[i] + cb * n[i]);
}

// ---------------------------------------------------------------------------
// Hessian assembly: updateHessian semantics (gtsam/linear/JacobianFactor.cpp:563-598,
// gtsam/linear/BinaryJacobianFactor.h:51-82) straight into the owning clique's
// front.  Upper triangle only; FP64 red.global.add.
// ---------------------------------------------------------------------------
template <int D, int NA, int NB_>
__device__ __forceinline__ void add_block(double* __restrict__ Mf, int ld, int sa, int sb, const double* A,
                                          const double* B, bool diag) {
  // entry (sa+ca, sb+cb) += A[:,ca] . B[:,cb]; stored in the upper triangle
#pragma unroll
  for (int ca = 0; ca < NA; ca++)
#pragma unroll
    for (int cb = 0; cb < NB_; cb++) {
      if (diag && ca > cb) continue;
      double s = 0;
#pragma unroll
      for (int r = 0; r < D; r++) s += A[ca * D + r] * B[cb * D + r];
      const int i = sa + ca, j = sb + cb;
      const int lo = i < j ? i : j, hi = i < j ? j : i;
      atomicAdd(Mf + lo + (size_t)hi * ld, s);
    }
}

template <int TYPE, typename JT = double>
__global__ void __launch_bounds__(128) assemble_kernel(GroupView g, TreeView t) {
  pdl_sync();
  typedef FactorTraits<TYPE> FT;
  enum { D = FT::D, N1 = FT::N1, N2 = FT::N2, NC = N1 + N2 + 1 };
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= g.count) return;
  const int4 sc = g.scat[f];
  if (sc.w) return;   // owned by a fused leaf clique: handled by leaf_fused_kernel
  double Jl[D * NC];  // column-major
  const JT* J = reinterpret_cast<const JT*>(g.J) + f;
#pragma unroll
  for (int e = 0; e < D * NC; e++) Jl[e] = J[(size_t)e * g.count];
  double* Mf = t.arena + t.off[sc.x];
  const int ld = t.nf[sc.x] + t.ns[sc.x] + 1;
  const int sb = ld - 1;
  const double* A1 = Jl;
  const double* bb = Jl + (N1 + N2) * D;
  add_block<D, N1, N1>(Mf, ld, sc.y, sc.y, A1, A1, true);
  add_block<D, N1, 1>(Mf, ld, sc.y, sb, A1, bb, false);
  if (N2 > 0) {
    const double* A2 = Jl + N1 * D;
    add_block<D, N1, (N2 > 0 ? N2 : 1)>(Mf, ld, sc.y, sc.z, A1, A2, false);
    add_block<D, (N2 > 0 ? N2 : 1), (N2 > 0 ? N2 : 1)>(Mf, ld, sc.z, sc.z, A2, A2, true);
    add_block<D, (N2 > 0 ? N2 : 1), 1>(Mf, ld, sc.z, sb, A2, bb, false);
  }
  add_block<D, 1, 1>(Mf, ld, sb, sb, bb, bb, true);
}

// hessianDiagonal: gtsam/linear/JacobianFactor.cpp:516-541
template <int TYPE, typename JT = double>
__global__ void __launch_bounds__(128) hdiag_kernel(GroupView g, const int* __restrict__ var_dof, double* hdiag) {
  pdl_sync();
  typedef FactorTraits<TYPE> FT;
  enum { D = FT::D, N1 = FT::N1, N2 = FT::N2 };
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= g.count) return;
  const int2 k = g.keys[f];
  const JT* J = reinterpret_cast<const JT*>(g.J) + f;
#pragma unroll
  for (int cc = 0; cc < N1 + N2; cc++) {
    double s = 0;
#pragma unroll
    for (int r = 0; r < D; r++) { const double a = J[(size_t)(r + cc * D) * g.count]; s += a * a; }
    const int idx = cc < N1 ? var_dof[k.x] + cc : var_dof[k.y] + (cc - N1);
    atomicAdd(hdiag + idx, s);
  }
}

// ---------------------------------------------------------------------------
// GaussianFactorGraph level (b200_linear_create): JacobianFactors of any arity and block widths
// (gtsam/linear/JacobianFactor.h:93-103).  Runtime shapes, one thread per factor, the same
// element-major SoA as the typed groups, so a warp's loads of one element are one segment.
// ---------------------------------------------------------------------------
// [A|b] blocks as the caller holds them (factor-major, column-major blocks = JacobianFactor::matrixObject())
// -> SoA, whitened by the Diagonal model's inverse sigmas (JacobianFactor::whiten, JacobianFactor.cpp:743-750;
// noiseModel::Diagonal::WhitenInPlace multiplies row r by invsigmas[r] = 1/sigmas[r])
__global__ void __launch_bounds__(256) jacobian_load_kernel(const double* __restrict__ Ab, const double* __restrict__ sigmas,
                                                            int rows, int ncols, int count, double* __restrict__ J) {
  const int64_t per = (int64_t)rows * ncols, total = per * count;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t e = i / count, f = i - e * count;   // consecutive threads -> consecutive factors: coalesced stores
    double x = Ab[f * per + e];
    if (sigmas) x *= 1.0 / sigmas[f * rows + e % rows];
    J[i] = x;
  }
}

// JacobianFactor::updateHessian (gtsam/linear/JacobianFactor.cpp:563-598): info(I,J) += A_i^T A_j over the
// blocks i <= j of [A1 .. Ak b], into the upper triangle of the owning clique's front
__global__ void __launch_bounds__(128) assemble_jacobian_kernel(JacobianView g, TreeView t) {
  pdl_sync();
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= g.count) return;
  const int c = g.clique[f];
  double* Mf = t.arena + t.off[c];
  const int ld = t.nf[c] + t.ns[c] + 1;
  const double* J = g.J + f;
  const int m = g.rows;
  const size_t cnt = (size_t)g.count;
  for (int a = 0; a <= g.arity; a++) {
    const int sa = a < g.arity ? g.slots[(size_t)f * g.arity + a] : ld - 1;   // block `arity` is the rhs column
    for (int ca = g.col0[a]; ca < g.col0[a + 1]; ca++) {
      const int i = sa + (ca - g.col0[a]);
      for (int b = a; b <= g.arity; b++) {
        const int sb = b < g.arity ? g.slots[(size_t)f * g.arity + b] : ld - 1;
        for (int cb = (b == a ? ca : g.col0[b]); cb < g.col0[b + 1]; cb++) {   // diagonal block: upper part only
          const int j = sb + (cb - g.col0[b]);
          double s = 0;
          for (int r = 0; r < m; r++) s += J[(size_t)(r + ca * m) * cnt] * J[(size_t)(r + cb * m) * cnt];
          const int lo = i < j ? i : j, hi = i < j ? j : i;
          atomicAdd(Mf + lo + (size_t)hi * ld, s);
        }
      }
    }
  }
}

// JacobianFactor::hessianDiagonalAdd, gtsam/linear/JacobianFactor.cpp:516-541
__global__ void __launch_bounds__(128) hdiag_jacobian_kernel(JacobianView g, const int* __restrict__ var_dof, double* hdiag) {
  pdl_sync();
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= g.count) return;
  const double* J = g.J + f;
  const int m = g.rows;
  const size_t cnt = (size_t)g.count;
  for (int a = 0; a < g.arity; a++) {
    const int base = var_dof[g.keys[(size_t)f * g.arity + a]];
    for (int cc = g.col0[a]; cc < g.col0[a + 1]; cc++) {
      double s = 0;
      for (int r = 0; r < m; r++) { const double x = J[(size_t)(r + cc * m) * cnt]; s += x * x; }
      atomicAdd(hdiag + base + (cc - g.col0[a]), s);
    }
  }
}

// JacobianFactor::gradientAtZero (gtsam/linear/JacobianFactor.cpp:690-699): -A^T b of the whitened factor, per key
__global__ void __launch_bounds__(128) gradient_jacobian_kernel(JacobianView g, const int* __restrict__ var_dof, double* grad) {
  pdl_sync();
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= g.count) return;
  const double* J = g.J + f;
  const int m = g.rows;
  const size_t cnt = (size_t)g.count;
  const double* b = J + (size_t)(g.ncols - 1) * m * cnt;
  for (int a = 0; a < g.arity; a++) {
    const int base = var_dof[g.keys[(size_t)f * g.arity + a]];
    for (int cc = g.col0[a]; cc < g.col0[a + 1]; cc++) {
      double s = 0;
      for (int r = 0; r < m; r++) s += J[(size_t)(r + cc * m) * cnt] * b[(size_t)r * cnt];
      atomicAdd(grad + base + (cc - g.col0[a]), -s);
    }
  }
}

// JacobianFactor::error (gtsam/linear/JacobianFactor.cpp:479-491): 0.5*|A x - bscale*b|^2 and 0.5*|b|^2
__global__ void __launch_bounds__(256) linerr_jacobian_kernel(JacobianView g, const double* __restrict__ delta,
                                                              const int* __restrict__ var_dof, double* p0, double* p1,
                                                              unsigned* counters, double* out0, double* out1, int accumulate,
                                                              double bscale) {
  pdl_sync();
  __shared__ double sh[32];
  double a0 = 0, a1 = 0;
  const int m = g.rows;
  const size_t cnt = (size_t)g.count;
  for (int f = blockIdx.x * blockDim.x + threadIdx.x; f < g.count; f += gridDim.x * blockDim.x) {
    const double* J = g.J + f;
    double s0 = 0, s1 = 0;
    for (int r = 0; r < m; r++) {
      const double b = J[(size_t)(r + g.col0[g.arity] * m) * cnt];
      double e = -bscale * b;
      for (int a = 0; a < g.arity; a++) {
        const double* d = delta + var_dof[g.keys[(size_t)f * g.arity + a]];
        for (int cc = g.col0[a]; cc < g.col0[a + 1]; cc++) e += J[(size_t)(r + cc * m) * cnt] * d[cc - g.col0[a]];
      }
      s0 += b * b;
      s1 += e * e;
    }
    a0 += 0.5 * s0;
    a1 += 0.5 * s1;
  }
  a0 = block_sum<256>(a0, sh);
  a1 = block_sum<256>(a1, sh);
  finish_sum(a0, p0, counters, out0, accumulate, sh);
  finish_sum(a1, p1, counters + 1, out1, accumulate, sh);
}

// HessianFactors of a linear problem (gtsam/linear/HessianFactor.h:99-110): the view's "rows" is N + 1 and J holds
// the augmented information matrix [G g; g' f] (element (r, c) at r + c*(N+1); upper triangle read).
// HessianFactor::updateHessian (gtsam/linear/HessianFactor.cpp:348-374): info(I,J) += this->info(i,j)
__global__ void __launch_bounds__(128) assemble_hessian_kernel(JacobianView g, TreeView t) {
  pdl_sync();
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= g.count) return;
  const int c = g.clique[f];
  double* Mf = t.arena + t.off[c];
  const int ld = t.nf[c] + t.ns[c] + 1;
  const double* H = g.J + f;
  const int n1 = g.rows;
  const size_t cnt = (size_t)g.count;
  for (int a = 0; a <= g.arity; a++) {
    const int sa = a < g.arity ? g.slots[(size_t)f * g.arity + a] : ld - 1;
    for (int ca = g.col0[a]; ca < g.col0[a + 1]; ca++) {
      const int i = sa + (ca - g.col0[a]);
      for (int b = a; b <= g.arity; b++) {
        const int sb = b < g.arity ? g.slots[(size_t)f * g.arity + b] : ld - 1;
        for (int cb = (b == a ? ca : g.col0[b]); cb < g.col0[b + 1]; cb++) {
          const int j = sb + (cb - g.col0[b]);
          const int lo = i < j ? i : j, hi = i < j ? j : i;
          atomicAdd(Mf + lo + (size_t)hi * ld, H[(size_t)(ca + cb * n1) * cnt]);   // ca <= cb: upper triangle of the factor
        }
      }
    }
  }
}

// HessianFactor::hessianDiagonalAdd (gtsam/linear/HessianFactor.cpp:292-304): the diagonal of G
__global__ void __launch_bounds__(128) hdiag_hessian_kernel(JacobianView g, const int* __restrict__ var_dof, double* hdiag) {
  pdl_sync();
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= g.count) return;
  const double* H = g.J + f;
  const int n1 = g.rows;
  const size_t cnt = (size_t)g.count;
  for (int a = 0; a < g.arity; a++) {
    const int base = var_dof[g.keys[(size_t)f * g.arity + a]];
    for (int cc = g.col0[a]; cc < g.col0[a + 1]; cc++) atomicAdd(hdiag + base + (cc - g.col0[a]), H[(size_t)(cc + cc * n1) * cnt]);
  }
}

// HessianFactor::gradientAtZero (gtsam/linear/HessianFactor.cpp:422-429): minus the linear term g of [G g; g' f]
__global__ void __launch_bounds__(128) gradient_hessian_kernel(JacobianView g, const int* __restrict__ var_dof, double* grad) {
  pdl_sync();
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= g.count) return;
  const double* H = g.J + f;
  const int n1 = g.rows;
  const size_t cnt = (size_t)g.count;
  for (int a = 0; a < g.arity; a++) {
    const int base = var_dof[g.keys[(size_t)f * g.arity + a]];
    for (int cc = g.col0[a]; cc < g.col0[a + 1]; cc++) atomicAdd(grad + base + (cc - g.col0[a]), -H[(size_t)(cc + (n1 - 1) * n1) * cnt]);
  }
}

// HessianFactor::error (gtsam/linear/HessianFactor.cpp:331-346): 0.5 (f - 2 x'g + x'G x); out0 gets the value at
// x = 0 (0.5 f), out1 the value at x = delta; bscale = 0 drops the f and g terms (0.5 x'G x)
__global__ void __launch_bounds__(256) linerr_hessian_kernel(JacobianView g, const double* __restrict__ delta,
                                                             const int* __restrict__ var_dof, double* p0, double* p1,
                                                             unsigned* counters, double* out0, double* out1, int accumulate,
                                                             double bscale) {
  pdl_sync();
  __shared__ double sh[32];
  double a0 = 0, a1 = 0;
  const int n1 = g.rows, N = n1 - 1;
  const size_t cnt = (size_t)g.count;
  for (int f = blockIdx.x * blockDim.x + threadIdx.x; f < g.count; f += gridDim.x * blockDim.x) {
    const double* H = g.J + f;
    double xGx = 0, xg = 0;
    for (int a = 0; a < g.arity; a++) {
      const double* da = delta + var_dof[g.keys[(size_t)f * g.arity + a]];
      for (int ca = g.col0[a]; ca < g.col0[a + 1]; ca++) {
        const double xa = da[ca - g.col0[a]];
        xg += xa * H[(size_t)(ca + N * n1) * cnt];
        xGx += xa * xa * H[(size_t)(ca + ca * n1) * cnt];
        for (int b = a; b < g.arity; b++) {   // strictly upper entries count twice
          const double* db = delta + var_dof[g.keys[(size_t)f * g.arity + b]];
          for (int cb = (b == a ? ca + 1 : g.col0[b]); cb < g.col0[b + 1]; cb++)
            xGx += 2.0 * xa * db[cb - g.col0[b]] * H[(size_t)(ca + cb * n1) * cnt];
        }
      }
    }
    const double ff = H[(size_t)(N + N * n1) * cnt];
    a0 += 0.5 * ff;
    a1 += 0.5 * (bscale * (ff - 2.0 * xg) + xGx);
  }
  a0 = block_sum<256>(a0, sh);
  a1 = block_sum<256>(a1, sh);
  finish_sum(a0, p0, counters, out0, accumulate, sh);
  finish_sum(a1, p1, counters + 1, out1, accumulate, sh);
}

// damping priors of buildDampedSystem (gtsam/nonlinear/internal/LevenbergMarquardtState.h:125-156)
__global__ void damp_kernel(double* arena, const int64_t* __restrict__ diag_index, int n,
                            const double* __restrict__ lambda_ptr, const double* __restrict__ hdiag, double min_diag,
                            double max_diag) {
  pdl_sync();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double lambda = *lambda_ptr;   // device resident: the launch sequence is lambda independent (CUDA graph)
  if (!(lambda > 0)) return;
  if (diag_index[i] < 0) return;  // variable of a fused leaf clique (damped inside leaf_fused_kernel)
  double a2 = 1.0;
  if (hdiag) {
    double h = fmin(fmax(hdiag[i], min_diag), max_diag);
    const double sq = sqrt(h);
    a2 = sq * sq;
  }
  const double sl = 1.0 / (1.0 / sqrt(lambda));
  arena[diag_index[i]] += (sl * sl) * a2;
}

// ---------------------------------------------------------------------------
// small fronts: one warp per clique, front staged in shared memory
//   choleskyPartial (gtsam/base/cholesky.cpp:107-158) + extend-add of the
//   Schur complement into the parent (gtsam/linear/HessianFactor.cpp:348-374)
// ---------------------------------------------------------------------------
__device__ __forceinline__ int dexp(double x) {
  int e;
  (void)frexp(x, &e);
  return e;
}

__global__ void __launch_bounds__(kWarpsPerBlock * 32)
elim_small_kernel(TreeView t, const int* __restrict__ list, int count, int smem_n, Scalars* sc) {
  pdl_sync();
  B200_DYN_SMEM(double, smem);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int idx = blockIdx.x * kWarpsPerBlock + warp;
  if (idx >= count) return;
  const int c = list[idx];
  const int f = t.nf[c], s = t.ns[c], n = f + s + 1;
  double* M = t.arena + t.off[c];
  double* A = smem + (size_t)warp * smem_n * smem_n;
  for (int e = lane; e < n * n; e += 32) A[e] = M[e];
  __syncwarp();
  bool ok = true;
  for (int k = 0; k < f; k++) {
    const double piv = A[k + k * n];
    if (!(piv > 0.0)) ok = false;  // Eigen LLT: fail when pivot <= 0
    const double r = sqrt(piv);
    __syncwarp();
    for (int j = k + lane; j < n; j += 32) A[k + j * n] = (j == k) ? r : A[k + j * n] / r;
    __syncwarp();
    const int w = n - k - 1;
    for (int e = lane; e < w * w; e += 32) {
      const int i = k + 1 + e % w, j = k + 1 + e / w;
      if (i <= j) A[i + j * n] -= A[k + i * n] * A[k + j * n];
    }
    __syncwarp();
  }
  if (f >= 2) {
    if (!(dexp(A[(f - 2) + (f - 2) * n]) - dexp(A[(f - 1) + (f - 1) * n]) < 12)) ok = false;
  } else if (f == 1) {
    if (!(dexp(A[0]) > -12)) ok = false;
  }
  if (!ok && lane == 0) atomicMax(&sc->fail_code, INT_MAX - c);
  // conditional [R S d] back to the front (rows 0..f-1)
  for (int e = lane; e < f * n; e += 32) {
    const int i = e % f, j = e / f;
    if (i <= j) M[i + (size_t)j * n] = A[i + j * n];
  }
  const int p = t.parent[c];
  if (p >= 0) {
    double* P = t.arena + t.off[p];
    const int pn = t.nf[p] + t.ns[p] + 1;
    const int* map = t.ea_map + t.ea_ptr[c];
    const int w = s + 1;
    for (int e = lane; e < w * w; e += 32) {
      const int i = e % w, j = e / w;
      if (i <= j) {
        const int pi = map[i], pj = map[j];
        const int lo = pi < pj ? pi : pj, hi = pi < pj ? pj : pi;
        atomicAdd(P + lo + (size_t)hi * pn, A[(f + i) + (f + j) * n]);
      }
    }
  }
}


// ---------------------------------------------------------------------------
// fused leaf path (the BAL "point" cliques, and any leaf clique with a small
// frontal block): ONE kernel does Hessian assembly of the clique's own factors
// (a12), the damping priors (a10), the partial Cholesky (a13/a14) and the
// extend-add of the Schur complement into the parent — without ever
// materialising the (f+s+1)^2 front in HBM.  One warp per clique; only the
// f x (f+s+1) block [F S d] lives in shared memory:
//   * factor contributions whose row is frontal accumulate into [F S d];
//   * contributions between separator variables (A_cam^T A_cam, A_cam^T b, b^T b)
//     do not take part in the elimination, so they go straight to the parent;
//   * after R = chol(F), S' = R^-T [S d], the update -S'^T S' goes to the parent.
// The conditional [R S' d'] is stored compactly (f x n, ld = f).
// ---------------------------------------------------------------------------
constexpr int kLeafAccMax = 1024;  // (s+1)(s+2)/2 accumulators per warp for grouped runs

// Triangular index e -> (i <= j) with e = j(j+1)/2 + i
__device__ __forceinline__ void tri_decode(int e, int& i, int& j) {
  j = (int)((sqrtf(8.0f * (float)e + 1.0f) - 1.0f) * 0.5f);
  while ((j + 1) * (j + 2) / 2 <= e) j++;
  while (j * (j + 1) / 2 > e) j--;
  i = e - j * (j + 1) / 2;
}

// One warp processes a RUN of leaf cliques that share parent and separator set (points seen by
// the same cameras).  Their contributions to the parent are first summed in shared memory
// (lane-private accumulators, no conflicts) and extend-added once per run, which divides the
// number of FP64 atomics into the top fronts by the run length.  A run of length 1 whose
// separator is too wide for the accumulators falls back to direct atomics.
template <typename JT = double>
__global__ void __launch_bounds__(kWarpsPerBlock * 32)
leaf_fused_kernel(TreeView t, GroupTable gt, const int* __restrict__ list, const int* __restrict__ run_ptr,
                  int nruns, const int* __restrict__ fac_ptr, const int2* __restrict__ fac,
                  const double* __restrict__ lambda_ptr, const double* __restrict__ hdiag, double min_diag,
                  double max_diag, Scalars* sc, int lb_cap, int acc_cap) {
  pdl_sync();
  B200_DYN_SMEM(double, leaf_sm);
  const double lambda = *lambda_ptr;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int run = blockIdx.x * kWarpsPerBlock + warp;
  if (run >= nruns) return;
  double* LB = leaf_sm + (size_t)warp * (lb_cap + acc_cap);  // row-major f x n
  double* acc = LB + lb_cap;
  const int r0 = run_ptr[run], r1 = run_ptr[run + 1];
  const int c0 = list[r0];
  const int s = t.ns[c0], w = s + 1, ntri = w * (w + 1) / 2;
  const int p = t.parent[c0];
  double* P = p >= 0 ? t.arena + t.off[p] : nullptr;
  const int pn = p >= 0 ? t.nf[p] + t.ns[p] + 1 : 0;
  const int* map = t.ea_map + t.ea_ptr[c0];
  const bool grouped = P && ntri <= acc_cap;
  if (grouped)
    for (int e = lane; e < ntri; e += 32) acc[e] = 0.0;
  for (int idx = r0; idx < r1; idx++) {
    const int c = list[idx];
    const int f = t.nf[c], n = f + s + 1;
    for (int e = lane; e < f * n; e += 32) LB[e] = 0.0;
    __syncwarp();
    for (int q = fac_ptr[idx]; q < fac_ptr[idx + 1]; q++) {
      const int2 gf = fac[q];
      const GroupView& g = gt.g[gf.x];
      const int D = kFD[g.type], N1 = kFN1[g.type], N2 = kFN2[g.type], NC = N1 + N2 + 1;
      const int4 scat = g.scat[gf.y];
      const JT* J = reinterpret_cast<const JT*>(g.J) + gf.y;
      const int NP = NC * (NC + 1) / 2;
      const size_t cnt = (size_t)g.count;
      for (int pi = lane; pi < NP; pi += 32) {
        const int ca = __ldg(&kPairA[g.type][pi]), cb = __ldg(&kPairB[g.type][pi]);
        const JT* Ja = J + (size_t)(ca * D) * cnt;
        const JT* Jb = J + (size_t)(cb * D) * cnt;
        double dot = 0;
        for (int r = 0; r < D; r++) dot += (double)Ja[r * cnt] * (double)Jb[r * cnt];
        int I = ca < N1 ? scat.y + ca : (ca < N1 + N2 ? scat.z + (ca - N1) : n - 1);
        int Jx = cb < N1 ? scat.y + cb : (cb < N1 + N2 ? scat.z + (cb - N1) : n - 1);
        if (I > Jx) { const int tmp = I; I = Jx; Jx = tmp; }
        if (I < f) {
          LB[I * n + Jx] += dot;  // distinct (ca,cb) -> distinct entries: no intra-warp conflict
        } else if (grouped) {
          const int i = I - f, j = Jx - f;
          acc[j * (j + 1) / 2 + i] += dot;   // separator-separator term: passes through to the parent
        } else if (P) {
          const int a = map[I - f], b = map[Jx - f];
          const int lo = a < b ? a : b, hi = a < b ? b : a;
          atomicAdd(P + lo + (size_t)hi * pn, dot);
        }
      }
      __syncwarp();
    }
    if (lambda > 0 && lane < f) {  // damping prior of each frontal scalar
      double a2 = 1.0;
      if (hdiag) {
        const double h = fmin(fmax(hdiag[t.didx[t.didx_ptr[c] + lane]], min_diag), max_diag);
        const double sq = sqrt(h);
        a2 = sq * sq;
      }
      const double sl = 1.0 / (1.0 / sqrt(lambda));
      LB[lane * n + lane] += (sl * sl) * a2;
    }
    __syncwarp();
    bool ok = true;
    for (int k = 0; k < f; k++) {
      const double piv = LB[k * n + k];
      if (!(piv > 0.0)) ok = false;
      const double r = sqrt(piv);
      __syncwarp();
      for (int j = k + lane; j < n; j += 32) LB[k * n + j] = (j == k) ? r : LB[k * n + j] / r;
      __syncwarp();
      for (int i = k + 1; i < f; i++) {
        const double rki = LB[k * n + i];
        for (int j = i + lane; j < n; j += 32) LB[i * n + j] -= rki * LB[k * n + j];
      }
      __syncwarp();
    }
    if (f >= 2) {
      if (!(dexp(LB[(f - 2) * n + f - 2]) - dexp(LB[(f - 1) * n + f - 1]) < 12)) ok = false;
    } else if (f == 1) {
      if (!(dexp(LB[0]) > -12)) ok = false;
    }
    if (!ok && lane == 0) atomicMax(&sc->fail_code, INT_MAX - c);
    double* M = t.arena + t.off[c];  // compact conditional, column-major f x n
    for (int j = lane; j < n; j += 32)
      for (int i = 0; i < f; i++) M[i + j * f] = (i <= j) ? LB[i * n + j] : 0.0;
    if (P) {
      int i, j;
      tri_decode(lane, i, j);
      for (int e = lane; e < ntri; e += 32) {
        if (e != lane) {   // advance (i,j) by 32 positions along the packed upper triangle
          i += 32;
          while (i > j) { i -= j + 1; j++; }
        }
        double v = 0;
        for (int k = 0; k < f; k++) v += LB[k * n + f + i] * LB[k * n + f + j];
        if (grouped) {
          acc[e] -= v;
        } else {
          const int a = map[i], b = map[j];
          const int lo = a < b ? a : b, hi = a < b ? b : a;
          atomicAdd(P + lo + (size_t)hi * pn, -v);
        }
      }
    }
    __syncwarp();
  }
  if (grouped) {
    int i, j;
    tri_decode(lane, i, j);
    for (int e = lane; e < ntri; e += 32) {
      if (e != lane) {
        i += 32;
        while (i > j) { i -= j + 1; j++; }
      }
      const int a = map[i], b = map[j];
      const int lo = a < b ? a : b, hi = a < b ? b : a;
      atomicAdd(P + lo + (size_t)hi * pn, acc[e]);
    }
  }
}

// ---------------------------------------------------------------------------
// BAL fast path of the fused leaf elimination: cliques whose single frontal variable is a Point3
// observed by m <= kPtMaxObs DISTINCT cameras through binary projection factors
// (GenericProjectionFactor: DC = 6, GeneralSFMFactor<Cal3Bundler>: DC = 9).  Same maths and same
// outputs as leaf_fused_kernel.  Per point, 8 lanes (one LANE per factor) assemble H_pp / g_p, damp, factor the 3x3
// block in registers and form S' = R^-T H_pc, d' = R^-T g_p: the compact conditional [R S' d'] (3 x n), PointFactor.
// Per RUN of points seen by the same cameras, the Schur complement  sum_p ( [A_c b]^T [A_c b] - [S' d']^T [S' d'] )  is a
// small SYRK (K = 3 per point, N = s + 1), added into the parent with ONE extend-add (FP64 atomics) per run.
//
//  leaf_point_fused_mma_kernel (default)  both, one CTA per run; the SYRK as 8x8 DMMA tiles (below).
//  leaf_point_factor_kernel + leaf_point_schur_kernel (schur_mma = 0)  a per-point kernel (50k points = 12.5k warps,
//      latency hidden by occupancy), then one CTA per run with 3x3 register tiles over the (s+1)^2 upper triangle and
//      the operands staged in shared memory 4 or 6 points at a time.
// ---------------------------------------------------------------------------
constexpr int kPtMaxObs = 8;

#ifdef B200_EMULATE   // host emulation build: the asynchronous copy is a plain copy
// (cp.async needs both addresses aligned to the copy size: checked here, the hardware would fault)
__device__ __forceinline__ void cp_async8(double* smem_dst, const double* gsrc) { if (((uintptr_t)smem_dst | (uintptr_t)gsrc) & 7) __builtin_trap(); *smem_dst = *gsrc; }
__device__ __forceinline__ void cp_async4(float* smem_dst, const float* gsrc) { if (((uintptr_t)smem_dst | (uintptr_t)gsrc) & 3) __builtin_trap(); *smem_dst = *gsrc; }
__device__ __forceinline__ void cp_async_commit() {}
#else
__device__ __forceinline__ void cp_async8(double* smem_dst, const double* gsrc) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;\n" ::"r"((unsigned)__cvta_generic_to_shared(smem_dst)), "l"(gsrc));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
__device__ __forceinline__ void cp_async4(float* smem_dst, const float* gsrc) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"((unsigned)__cvta_generic_to_shared(smem_dst)), "l"(gsrc));
}
#endif
__device__ __forceinline__ void cp_async_el(double* d, const double* s) { cp_async8(d, s); }
__device__ __forceinline__ void cp_async_el(float* d, const float* s) { cp_async4(d, s); }
#ifdef B200_EMULATE
template <int N>
__device__ __forceinline__ void cp_async_wait() {}
#else
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }
#endif

// The per-point arithmetic of the BAL point leaves.  leaf_point_factor_kernel and leaf_point_fused_mma_kernel both go
// through it, so the two store bitwise the same conditionals: every product and fused multiply-add is spelled out
// (fma / mul_rn), since where the compiler would contract a * b + c on its own depends on the surrounding kernel.
// 8 lanes per point, one factor per lane.
#ifdef B200_EMULATE
__device__ __forceinline__ double mul_rn(double a, double b) { return a * b; }
#else
__device__ __forceinline__ double mul_rn(double a, double b) { return __dmul_rn(a, b); }
#endif
struct PointFactor {
  double r00, r01, r02, r11, r12, r22, i00, i11, i22;   // R (upper) and the reciprocals of its diagonal
  double d0, d1, d2;                                    // d' = R^-T g_p
  bool ok;
  // this lane's factor's share of [H_pp g_p]: the upper triangle of A_p^T A_p (6) and A_p^T b (3)
  __device__ __forceinline__ static void lane_terms(const double Ap[2][3], const double b[2], double v[9]) {
    v[0] = fma(Ap[0][0], Ap[0][0], mul_rn(Ap[1][0], Ap[1][0]));
    v[1] = fma(Ap[0][0], Ap[0][1], mul_rn(Ap[1][0], Ap[1][1]));
    v[2] = fma(Ap[0][0], Ap[0][2], mul_rn(Ap[1][0], Ap[1][2]));
    v[3] = fma(Ap[0][1], Ap[0][1], mul_rn(Ap[1][1], Ap[1][1]));
    v[4] = fma(Ap[0][1], Ap[0][2], mul_rn(Ap[1][1], Ap[1][2]));
    v[5] = fma(Ap[0][2], Ap[0][2], mul_rn(Ap[1][2], Ap[1][2]));
    v[6] = fma(Ap[0][0], b[0], mul_rn(Ap[1][0], b[1]));
    v[7] = fma(Ap[0][1], b[0], mul_rn(Ap[1][1], b[1]));
    v[8] = fma(Ap[0][2], b[0], mul_rn(Ap[1][2], b[1]));
  }
  // v: the lane's terms; summed over the point's 8 lanes, damped (lambda, times the clipped diagonal of H at the point's
  // variables di when hd is given), then the 3x3 partial Cholesky in registers (every lane of the point, identical):
  // gtsam/base/cholesky.cpp:107-158 (rsqrt + multiplies instead of sqrt + divides: same result to ~1 ulp per operation,
  // a third of the latency)
  __device__ __forceinline__ void factor(double v[9], double lambda, const double* __restrict__ hd, const int* __restrict__ di,
                                         double min_diag, double max_diag) {
#pragma unroll
    for (int i = 0; i < 9; i++)
#pragma unroll
      for (int o = 4; o > 0; o >>= 1) v[i] += __shfl_xor_sync(0xffffffffu, v[i], o);
    if (lambda > 0) {
      const double sl = 1.0 / (1.0 / sqrt(lambda)), sl2 = mul_rn(sl, sl);
      double a2[3] = {1.0, 1.0, 1.0};
      if (hd) {
#pragma unroll
        for (int i = 0; i < 3; i++) { const double sq = sqrt(fmin(fmax(hd[di[i]], min_diag), max_diag)); a2[i] = mul_rn(sq, sq); }
      }
      v[0] = fma(sl2, a2[0], v[0]); v[3] = fma(sl2, a2[1], v[3]); v[5] = fma(sl2, a2[2], v[5]);
    }
    ok = v[0] > 0.0;
    i00 = rsqrt(v[0]);
    r00 = mul_rn(v[0], i00);
    r01 = mul_rn(v[1], i00); r02 = mul_rn(v[2], i00);
    const double p11 = fma(-r01, r01, v[3]);
    ok = ok && p11 > 0.0;
    i11 = rsqrt(p11);
    r11 = mul_rn(p11, i11);
    r12 = mul_rn(fma(-r01, r02, v[4]), i11);
    const double p22 = fma(-r12, r12, fma(-r02, r02, v[5]));
    ok = ok && p22 > 0.0;
    i22 = rsqrt(p22);
    r22 = mul_rn(p22, i22);
    if (!(dexp(r11) - dexp(r22) < 12)) ok = false;
    d0 = mul_rn(v[6], i00);
    d1 = mul_rn(fma(-r01, d0, v[7]), i11);
    d2 = mul_rn(fma(-r12, d1, fma(-r02, d0, v[8])), i22);
  }
  // one column of S' = R^-T A_p^T A_c, from the column (a0, a1) of this lane's A_c
  __device__ __forceinline__ void s_col(const double Ap[2][3], double a0, double a1, double& s0, double& s1, double& s2) const {
    const double w0 = fma(Ap[0][0], a0, mul_rn(Ap[1][0], a1));
    const double w1 = fma(Ap[0][1], a0, mul_rn(Ap[1][1], a1));
    const double w2 = fma(Ap[0][2], a0, mul_rn(Ap[1][2], a1));
    s0 = mul_rn(w0, i00);
    s1 = mul_rn(fma(-r01, s0, w1), i11);
    s2 = mul_rn(fma(-r12, s1, fma(-r02, s0, w2)), i22);
  }
};

// The split path (schur_mma = 0): every lane stores its camera's 3 x DC block of the conditional directly.
template <int DC, typename JT = double>
__global__ void __launch_bounds__(128)
leaf_point_factor_kernel(TreeView t, GroupTable gt, const int* __restrict__ list, int i_begin, int i_end,
                         const int* __restrict__ fac_ptr, const int2* __restrict__ fac, const double* __restrict__ lambda_ptr,
                         const double* __restrict__ hdiag, double min_diag, double max_diag, Scalars* sc,
                         const int2* __restrict__ pt_tab, const int64_t* __restrict__ pt_off) {
  pdl_sync();
  const double lambda = *lambda_ptr;
  const int sub = threadIdx.x & 7;
  const int idx = i_begin + (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 3);
  const bool live = idx < i_end;
  // one level of index loads: this lane's factor from the flat table, the conditional's offset, the clique id (failure
  // code / diagonal damping only)
  int c = 0;
  int2 rec = make_int2(-1, 0);
  int64_t moff = 0;
  if (live) { rec = pt_tab[(size_t)idx * kPtMaxObs + sub]; moff = pt_off[idx]; c = list[idx]; }
  int m = rec.x >= 0 ? 1 : 0;                                  // factors of this lane's point: summed over its 8 lanes
#pragma unroll
  for (int o = 4; o > 0; o >>= 1) m += __shfl_xor_sync(0xffffffffu, m, o);
  double Ac[2][DC], Ap[2][3], b[2];
  int tk = 0;
  double v[9];
#pragma unroll
  for (int i = 0; i < 9; i++) v[i] = 0.0;
  if (rec.x >= 0) {
    const GroupView& g = gt.g[rec.y >> 8];
    const size_t cnt = (size_t)g.count;
    const JT* J = reinterpret_cast<const JT*>(g.J) + rec.x;
    tk = DC * (rec.y & 0xff);
#pragma unroll
    for (int cc = 0; cc < DC; cc++) { Ac[0][cc] = J[(size_t)(2 * cc) * cnt]; Ac[1][cc] = J[(size_t)(2 * cc + 1) * cnt]; }
#pragma unroll
    for (int j = 0; j < 3; j++) { Ap[0][j] = J[(size_t)(2 * (DC + j)) * cnt]; Ap[1][j] = J[(size_t)(2 * (DC + j) + 1) * cnt]; }
    b[0] = J[(size_t)(2 * (DC + 3)) * cnt]; b[1] = J[(size_t)(2 * (DC + 3) + 1) * cnt];
    PointFactor::lane_terms(Ap, b, v);
  }
  const bool hd = hdiag && live;
  PointFactor f;
  f.factor(v, lambda, hd ? hdiag : nullptr, hd ? t.didx + t.didx_ptr[c] : nullptr, min_diag, max_diag);
  if (!live) return;
  if (!f.ok && sub == 0) atomicMax(&sc->fail_code, INT_MAX - c);
  const int n = 3 + DC * m + 1;     // (a point clique of these kinds: one factor per separator camera)
  double* M = t.arena + moff;       // compact conditional [R S' d'], column-major 3 x n
  if (sub == 0) {
    M[0] = f.r00; M[1] = 0.0; M[2] = 0.0;
    M[3] = f.r01; M[4] = f.r11; M[5] = 0.0;
    M[6] = f.r02; M[7] = f.r12; M[8] = f.r22;
    M[3 * (n - 1)] = f.d0; M[3 * (n - 1) + 1] = f.d1; M[3 * (n - 1) + 2] = f.d2;
  }
  if (rec.x >= 0) {
    double* Mc = M + 3 * (3 + tk);
#pragma unroll
    for (int cc = 0; cc < DC; cc++) {
      double s0, s1, s2;
      f.s_col(Ap, Ac[0][cc], Ac[1][cc], s0, s1, s2);
      Mc[3 * cc] = s0; Mc[3 * cc + 1] = s1; Mc[3 * cc + 2] = s2;
    }
  }
}

template <int DC, int TPT, int PB, typename JT = double>   // TPT: 3x3 tiles per thread = ceil(tiles of the widest separator / blockDim); PB: points per staged batch (<= 8)
__global__ void __launch_bounds__(128)
leaf_point_schur_kernel(TreeView t, GroupTable gt, const int* __restrict__ list, const int* __restrict__ run_ptr,
                        const int* __restrict__ fac_ptr, const int2* __restrict__ fac) {
  pdl_sync();
  constexpr int NTMAX = (kPtMaxObs * DC + 1 + 2) / 3; // 3-wide tiles along the widest separator (+ rhs column)
  constexpr int WP = NTMAX * 3;
  constexpr int AW = 2 * DC + 2;                      // per factor: A_c (2 x DC, column-major) and b (2)
  __shared__ double sS[2][PB][3 * WP];                // [S' d'] as stored: entry (r, col) at 3*col + r
  __shared__ JT sA[2][PB][kPtMaxObs][AW];            // staged in the Jacobians' storage type, widened on use
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int nthr = blockDim.x, nwarp = nthr >> 5;   // 96 or 128 threads: no idle warp on the common 6-camera point
  const int r0 = run_ptr[blockIdx.x], r1 = run_ptr[blockIdx.x + 1];
  const int c0 = list[r0];
  const int p = t.parent[c0];
  if (p < 0) return;
  const int s = t.ns[c0], w = s + 1;
  const int m = fac_ptr[r0 + 1] - fac_ptr[r0];
  const int nt = (w + 2) / 3, ts = s / 3;   // s = m*DC is a multiple of 3: the rhs column is entry 0 of tile ts
  int ti[TPT], tj[TPT];
  double acc[TPT][3][3];
#pragma unroll
  for (int u = 0; u < TPT; u++) {
    int e = tid + nthr * u, a = 0;
    while (a < nt && e >= nt - a) { e -= nt - a; a++; }
    ti[u] = a < nt ? a : -1;
    tj[u] = a + e;
#pragma unroll
    for (int x = 0; x < 3; x++)
#pragma unroll
      for (int y = 0; y < 3; y++) acc[u][x][y] = 0.0;
  }
  for (int e = tid; e < 2 * PB * (3 * WP - 3 * w); e += nthr) {   // zero padding behind the rhs column, written once
    const int pt = e / (3 * WP - 3 * w);
    (&sS[0][0][0])[(size_t)pt * 3 * WP + 3 * w + (e - pt * (3 * WP - 3 * w))] = 0.0;
  }
  // Software pipeline: the operands of batch b+1 stream into the other buffer (cp.async) while batch b
  // is multiplied, and the (dependent) index loads of batch b+2 are in flight behind them.
  const double* srcS[3];       // [S' d'] of the points this warp copies (points warp, warp + nwarp, ... of a batch)
  const JT* srcJ = nullptr;    // this thread's factor (point tid>>3, factor tid&7), staged by camera slot
  int cntJ = 0;
  int slotJ = -1;
  auto load_idx = [&](int b0) {
    const int nb = min(PB, r1 - b0);
#pragma unroll
    for (int q = 0; q < 3; q++) {
      const int pt = warp + nwarp * q;
      srcS[q] = pt < nb ? t.arena + t.off[list[b0 + pt]] + 9 : nullptr;
    }
    const int pt = tid >> 3, fi = tid & 7;
    slotJ = -1;
    if (pt < nb && fi < m) {
      const int2 gf = fac[fac_ptr[b0 + pt] + fi];
      const GroupView& g = gt.g[gf.x];
      cntJ = (size_t)g.count;
      srcJ = reinterpret_cast<const JT*>(g.J) + gf.y;
      slotJ = (g.scat[gf.y].y - 3) / DC;
    }
  };
  auto issue = [&](int buf) {
#pragma unroll
    for (int q = 0; q < 3; q++)
      if (srcS[q])
        for (int e = lane; e < 3 * w; e += 32) cp_async8(&sS[buf][warp + nwarp * q][e], srcS[q] + e);
    if (slotJ >= 0) {
      JT* dst = sA[buf][tid >> 3][slotJ];
#pragma unroll
      for (int el = 0; el < 2 * DC; el++) cp_async_el(dst + el, srcJ + (size_t)el * cntJ);
      cp_async_el(dst + 2 * DC, srcJ + (size_t)(2 * (DC + 3)) * cntJ);
      cp_async_el(dst + 2 * DC + 1, srcJ + (size_t)(2 * (DC + 3) + 1) * cntJ);
    }
    cp_async_commit();
  };
  load_idx(r0);
  issue(0);
  load_idx(r0 + PB);
  int buf = 0;
  for (int b0 = r0; b0 < r1; b0 += PB, buf ^= 1) {
    const int nbp = min(PB, r1 - b0);
    if (b0 + PB < r1) {
      issue(buf ^ 1);
      load_idx(b0 + 2 * PB);
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
#pragma unroll
    for (int u = 0; u < TPT; u++) {
      if (ti[u] < 0) continue;
      const int i0 = 3 * ti[u], j0 = 3 * tj[u];
      const int ci = i0 / DC, cj = j0 / DC;
      const int oi = i0 - ci * DC, oj = j0 - cj * DC;
      for (int pt = 0; pt < nbp; pt++) {
        const double* Si = sS[buf][pt] + 3 * i0;
        const double* Sj = sS[buf][pt] + 3 * j0;
#pragma unroll
        for (int r = 0; r < 3; r++) {
          double si[3], sj[3];
#pragma unroll
          for (int x = 0; x < 3; x++) { si[x] = Si[3 * x + r]; sj[x] = Sj[3 * x + r]; }
#pragma unroll
          for (int x = 0; x < 3; x++)
#pragma unroll
            for (int y = 0; y < 3; y++) acc[u][x][y] -= si[x] * sj[y];
        }
        if (tj[u] < ts) {
          if (ci == cj) {   // both inside one camera's block: A_c^T A_c
            const JT* A = sA[buf][pt][ci];
#pragma unroll
            for (int x = 0; x < 3; x++)
#pragma unroll
              for (int y = 0; y < 3; y++)
                acc[u][x][y] += (double)A[2 * (oi + x)] * (double)A[2 * (oj + y)] + (double)A[2 * (oi + x) + 1] * (double)A[2 * (oj + y) + 1];
          }
        } else if (ti[u] < ts) {   // rhs column: A_c^T b
          const JT* A = sA[buf][pt][ci];
#pragma unroll
          for (int x = 0; x < 3; x++) acc[u][x][0] += (double)A[2 * (oi + x)] * (double)A[2 * DC] + (double)A[2 * (oi + x) + 1] * (double)A[2 * DC + 1];
        } else {                   // constant term: b^T b
          for (int fi = 0; fi < m; fi++) {
            const JT* A = sA[buf][pt][fi];
            acc[u][0][0] += (double)A[2 * DC] * (double)A[2 * DC] + (double)A[2 * DC + 1] * (double)A[2 * DC + 1];
          }
        }
      }
    }
    __syncthreads();
  }
  // one extend-add per run (HessianFactor::updateHessian of the leaf's separator factor)
  double* P = t.arena + t.off[p];
  const int pn = t.nf[p] + t.ns[p] + 1;
  const int* map = t.ea_map + t.ea_ptr[c0];
#pragma unroll
  for (int u = 0; u < TPT; u++) {
    if (ti[u] < 0) continue;
#pragma unroll
    for (int x = 0; x < 3; x++)
#pragma unroll
      for (int y = 0; y < 3; y++) {
        const int i = 3 * ti[u] + x, j = 3 * tj[u] + y;
        if (i <= j && j < w) {
          const int a = map[i], bq = map[j];
          const int lo = a < bq ? a : bq, hi = a < bq ? bq : a;
          atomicAdd(P + lo + (size_t)hi * pn, acc[u][x][y]);
        }
      }
  }
}

// mma.sync.aligned.m8n8k4.row.col.f64 (SASS: DMMA); fragment layout (PTX ISA): A(row i = lane/4, col k = lane%4),
// B(row k = lane%4, col j = lane/4), C/D(row i = lane/4, cols 2*(lane%4) + {0,1}).
#ifdef B200_EMULATE   // host emulation build: the fragment layout above spelled out with warp exchanges
__device__ __forceinline__ void dmma_m8n8k4(double& d0, double& d1, double a, double b) {
  const int lane = threadIdx.x & 31, i = lane >> 2, j0 = 2 * (lane & 3);
  for (int k = 0; k < 4; k++) {
    const double ak = __shfl_sync(0xffffffffu, a, 4 * i + k);
    const double b0 = __shfl_sync(0xffffffffu, b, 4 * j0 + k), b1 = __shfl_sync(0xffffffffu, b, 4 * (j0 + 1) + k);
    d0 += ak * b0;
    d1 += ak * b1;
  }
}
#else
__device__ __forceinline__ void dmma_m8n8k4(double& d0, double& d1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
               : "+d"(d0), "+d"(d1)
               : "d"(a), "d"(b));
}
#endif

// ---------------------------------------------------------------------------
// Both halves of the BAL point leaves in one kernel, the Schur complement on the FP64 tensor path.  One CTA of 4 warps per
// RUN of points seen by the same cameras; the run's points are dealt to the warps in mini-batches of 4 (warp, warp + 4, ...)
// and every warp runs its own pipeline over them — no block barrier in the loop:
//   * it stages the next mini-batch's [A_c b] blocks ([camera][column][k = 2 pt + r]) and A_p ([element][lane]) with
//     cp.async, double-buffered;
//   * it factors the current mini-batch's points (PointFactor, lane = point lane>>3, factor lane&7, A_c read column by
//     column from shared memory) and writes [R S' d'] TRANSPOSED into shared memory ([column][k = 3 pt + r], 12 doubles per
//     column: conflict-free fragments, no padding); from there every point's conditional leaves as contiguous stores;
//   * per k-step of 4 rows it loads ONE fragment per 8-column strip and issues mma.sync.m8n8k4.f64 for every tile pair
//     of the upper triangle of -S'^T S' (the same fragment is the A operand, negated, and the B operand): 10 DMMAs = 2560
//     FMAs for 4 shared-memory loads at 32 columns; a camera's (DC+1)^2 block [A_c b]^T [A_c b] is one more tile (four at
//     9 dofs);
//   * the four warps' partial sums are added in shared memory in a FIXED order, then one extend-add per entry and run
//     (HessianFactor::updateHessian of the leaf's separator factor) — a run's contribution is bitwise reproducible.
// Every operand crosses HBM once: the split path (leaf_point_factor_kernel + leaf_point_schur_kernel) reads the [S' d'] the
// first kernel has just written and the [A_c b] it has just read a second time.
// ---------------------------------------------------------------------------
constexpr int kSmMP = 4;                 // points per warp mini-batch
constexpr int kSmKS = 3 * kSmMP;         // rows (and pitch) of a staged S'^T column: (q * 12 + g) mod 16 distinct over a half-warp
constexpr int kSmKA = 2 * kSmMP;         // rows of a staged [A_c b]^T column; pitch 12 (doubles and floats: conflict-free)
constexpr int kSmPA = 12;
constexpr int kSmPadA = 4;               // behind every camera's [A_c b]^T block: the 8 cameras of a factor-phase access hit
                                         // different banks (2 wavefronts per float access instead of 8)

// (min. 3 blocks = 168 registers at 6 dofs and up to 40 columns: at 4 blocks = 128 registers the factorisation spills)
template <int DC, int NTT, typename JT = double>   // NTT: 8-column strips of the widest separator (+ rhs column) of the kind
__global__ void __launch_bounds__(128, (NTT <= 5 && DC == 6) ? 3 : (NTT <= 7 ? 2 : 1))
leaf_point_fused_mma_kernel(TreeView t, GroupTable gt, const int* __restrict__ list, const int* __restrict__ run_ptr,
                            const double* __restrict__ lambda_ptr, const double* __restrict__ hdiag, double min_diag,
                            double max_diag, Scalars* sc, const int2* __restrict__ pt_tab, const int64_t* __restrict__ pt_off) {
  pdl_sync();
  constexpr int MP = kSmMP, KS = kSmKS, PA = kSmPA;
  constexpr int CP = DC < 8 ? 8 : 16, CT = CP / 8;           // [A_c b] has DC + 1 columns: one 8x8 tile, or 2 x 2 at 9 dofs
  constexpr int NAT = CT * (CT + 1) / 2;
  constexpr int SA = CP * PA + kSmPadA;                      // elements per camera of a staged [A_c b]^T
  constexpr int MC = (8 * NTT - 1) / DC < kPtMaxObs ? (8 * NTT - 1) / DC : kPtMaxObs;   // cameras of the widest separator
  B200_DYN_SMEM(double, sm_dyn);
  __shared__ int64_t sOff[4][2][MP];                         // per warp and buffer: the points' conditional offsets,
  __shared__ int sC[4][2][MP];                               // clique ids
  __shared__ int sSlot[4][2][32];                            // and every lane's camera slot (-1: no factor)
  const double lambda = *lambda_ptr;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, q = lane & 3;
  const int pl = lane >> 3, fl = lane & 7;                   // factorisation: point of the mini-batch, factor slot
  const int r0 = run_ptr[blockIdx.x], r1 = run_ptr[blockIdx.x + 1];
  const int c0 = list[r0];
  const int s = t.ns[c0], w = s + 1;
  const int m = s / DC;                                       // one factor per separator camera
  const int NT = (w + 7) >> 3, WP = 8 * NT;
  const int f_doubles = (3 + WP) * KS;                        // per warp: [R S' d']^T of the mini-batch (one buffer)
  const int a_elems = 2 * m * SA;                             // per warp: [A_c b]^T of m cameras, two buffers, in JT
  double* sF = sm_dyn + (size_t)warp * f_doubles;
  double* sS = sF + 3 * KS;                                   // the [S' d'] columns
  JT* sA = reinterpret_cast<JT*>(sm_dyn + (size_t)4 * f_doubles) + (size_t)warp * (a_elems + 2 * 6 * 32);
  JT* sP = sA + a_elems;                                      // per warp: A_p, [buffer][element 2 j + r][lane], in JT
  double acc[NTT][NTT][2];                                    // tile (ti <= tj) of -S'^T S'
  double accA[MC][NAT][2];                                    // per camera: tiles of [A_c b]^T [A_c b]
#pragma unroll
  for (int a = 0; a < NTT; a++)
#pragma unroll
    for (int b = 0; b < NTT; b++) acc[a][b][0] = acc[a][b][1] = 0.0;
#pragma unroll
  for (int ci = 0; ci < MC; ci++)
#pragma unroll
    for (int x = 0; x < NAT; x++) accA[ci][x][0] = accA[ci][x][1] = 0.0;
  // padding never written: columns behind the rhs column, columns behind b
  for (int e = lane; e < f_doubles; e += 32) if (e / KS >= 3 + w) sF[e] = 0.0;
  for (int e = lane; e < a_elems; e += 32) { const int r = e % SA; if (r / PA > DC || r % PA >= kSmKA) sA[e] = (JT)0; }
  const int npts = r1 - r0, nmb = (npts + MP - 1) / MP;       // mini-batches of the run; this warp takes warp, warp + 4, ...
  const JT* srcJ = nullptr;      // this lane's factor (point lane>>3 of the mini-batch, factor lane&7), staged by camera slot
  int cntJ = 0;
  int slotJ = -1, cJ = 0;
  int64_t offJ = 0;
  auto load_idx = [&](int mb) {
    const int b0 = r0 + MP * mb, nb = min(MP, r1 - b0);
    // one level of index loads (the flat table of the point leaves: engine.cu)
    slotJ = -1;
    if (pl < nb) {
      const int2 rec = pt_tab[(size_t)(b0 + pl) * kPtMaxObs + fl];
      offJ = pt_off[b0 + pl];
      cJ = list[b0 + pl];
      if (rec.x >= 0) {
        const GroupView& gv = gt.g[rec.y >> 8];
        cntJ = (int)gv.count;
        srcJ = reinterpret_cast<const JT*>(gv.J) + rec.x;
        slotJ = rec.y & 0xff;
      }
    }
  };
  auto issue = [&](int buf, int nb) {
    JT* A = sA + buf * m * SA;
    if (slotJ >= 0) {
      JT* dst = A + slotJ * SA + 2 * pl;
#pragma unroll
      for (int cc = 0; cc < DC; cc++) {
        cp_async_el(dst + cc * PA, srcJ + (size_t)(2 * cc) * cntJ);
        cp_async_el(dst + cc * PA + 1, srcJ + (size_t)(2 * cc + 1) * cntJ);
      }
      cp_async_el(dst + DC * PA, srcJ + (size_t)(2 * (DC + 3)) * cntJ);
      cp_async_el(dst + DC * PA + 1, srcJ + (size_t)(2 * (DC + 3) + 1) * cntJ);
      JT* P = sP + buf * 6 * 32 + lane;
#pragma unroll
      for (int el = 0; el < 6; el++) cp_async_el(P + 32 * el, srcJ + (size_t)(2 * DC + el) * cntJ);
    }
    cp_async_commit();
    sSlot[warp][buf][lane] = slotJ;
    if (fl == 0 && pl < nb) { sOff[warp][buf][pl] = offJ; sC[warp][buf][pl] = cJ; }
    if (nb < MP)       // a short last mini-batch: the rows of the missing points read as zero
      for (int e = lane; e < m * (DC + 1) * (kSmKA - 2 * nb); e += 32) {
        const int cc = e / (kSmKA - 2 * nb);
        A[cc / (DC + 1) * SA + cc % (DC + 1) * PA + 2 * nb + (e - cc * (kSmKA - 2 * nb))] = (JT)0;
      }
  };
  if (warp < nmb) {
    load_idx(warp);
    issue(0, min(MP, npts - MP * warp));
    if (warp + 4 < nmb) load_idx(warp + 4);
  }
  int buf = 0;
  for (int mb = warp; mb < nmb; mb += 4, buf ^= 1) {
    const int nb = min(MP, npts - MP * mb);
    if (mb + 4 < nmb) {
      issue(buf ^ 1, min(MP, npts - MP * (mb + 4)));
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncwarp();
    const JT* A = sA + buf * m * SA;
    {   // ---- the mini-batch's points: factor, [R S' d'] into sF; the rows of missing points are zero ----
      const int slot = sSlot[warp][buf][lane];
      const bool live = pl < nb;
      const JT* Al = A + slot * SA + 2 * pl;                  // this lane's [A_c b]^T (slot >= 0)
      double Ap[2][3], v[9];
#pragma unroll
      for (int i = 0; i < 9; i++) v[i] = 0.0;
      if (slot >= 0) {
        const JT* P = sP + buf * 6 * 32 + lane;
#pragma unroll
        for (int j = 0; j < 3; j++) { Ap[0][j] = (double)P[32 * (2 * j)]; Ap[1][j] = (double)P[32 * (2 * j + 1)]; }
        const double b[2] = {(double)Al[DC * PA], (double)Al[DC * PA + 1]};
        PointFactor::lane_terms(Ap, b, v);
      }
      const int c = live ? sC[warp][buf][pl] : 0;
      const bool hd = hdiag && live;
      PointFactor f;
      f.factor(v, lambda, hd ? hdiag : nullptr, hd ? t.didx + t.didx_ptr[c] : nullptr, min_diag, max_diag);
      if (live) {
        if (fl == 0) {
          if (!f.ok) atomicMax(&sc->fail_code, INT_MAX - c);
          double* F = sF + 3 * pl;
          F[0] = f.r00; F[1] = 0.0; F[2] = 0.0;
          F[KS] = f.r01; F[KS + 1] = f.r11; F[KS + 2] = 0.0;
          F[2 * KS] = f.r02; F[2 * KS + 1] = f.r12; F[2 * KS + 2] = f.r22;
          F[(3 + s) * KS] = f.d0; F[(3 + s) * KS + 1] = f.d1; F[(3 + s) * KS + 2] = f.d2;
        }
        if (slot >= 0) {
          double* F = sS + DC * slot * KS + 3 * pl;
#pragma unroll
          for (int cc = 0; cc < DC; cc++) {
            double s0, s1, s2;
            f.s_col(Ap, (double)Al[cc * PA], (double)Al[cc * PA + 1], s0, s1, s2);
            F[cc * KS] = s0; F[cc * KS + 1] = s1; F[cc * KS + 2] = s2;
          }
        }
      } else {
        for (int col = fl; col < w; col += 8) { double* F = sS + col * KS + 3 * pl; F[0] = F[1] = F[2] = 0.0; }
      }
    }
    __syncwarp();
    // ---- every point's conditional [R S' d'] (column-major 3 x (3 + w)) leaves as contiguous stores ----
#pragma unroll 1
    for (int z = 0; z < nb; z++) {
      double* dst = t.arena + sOff[warp][buf][z];
      const double* src = sF + 3 * z;
#pragma unroll 1
      for (int e = lane; e < 3 * (3 + w); e += 32) { const int col = e / 3; dst[e] = src[col * KS + (e - 3 * col)]; }
    }
    if (mb + 8 < nmb) load_idx(mb + 8);      // (here, not next to issue(): the factorisation's registers are free again)
    // ---- the mini-batch's share of the run's Schur complement ----
#pragma unroll
    for (int k4 = 0; k4 < KS / 4; k4++) {
      double fr[NTT];
#pragma unroll
      for (int a = 0; a < NTT; a++) fr[a] = a < NT ? sS[(8 * a + g) * KS + 4 * k4 + q] : 0.0;
#pragma unroll
      for (int a = 0; a < NTT; a++)
#pragma unroll
        for (int b = a; b < NTT; b++)
          if (b < NT) dmma_m8n8k4(acc[a][b][0], acc[a][b][1], -fr[a], fr[b]);     // (warp-uniform)
    }
#pragma unroll
    for (int ci = 0; ci < MC; ci++) {
      if (ci >= m) break;
#pragma unroll
      for (int k4 = 0; k4 < kSmKA / 4; k4++) {
        double fa[CT];
#pragma unroll
        for (int x = 0; x < CT; x++) fa[x] = (double)A[ci * SA + (8 * x + g) * PA + 4 * k4 + q];
#pragma unroll
        for (int x = 0; x < CT; x++)
#pragma unroll
          for (int y = x; y < CT; y++) dmma_m8n8k4(accA[ci][x * CT - x * (x - 1) / 2 + (y - x)][0], accA[ci][x * CT - x * (x - 1) / 2 + (y - x)][1], fa[x], fa[y]);
      }
    }
    __syncwarp();
  }
  const int p = t.parent[c0];
  if (p < 0) return;      // a root point clique: factored, nothing to extend-add into (block-uniform)
  // ---- the four warps' sums, added in a fixed order in shared memory (the staging buffers are free now) ----
  __syncthreads();
  double* R = sm_dyn;                                          // [WP][WP], upper triangle used (the launch sizes it)
  for (int round = 0; round < 4; round++) {
    if (warp == round) {
#pragma unroll
      for (int a = 0; a < NTT; a++)
#pragma unroll
        for (int b = a; b < NTT; b++)
          if (b < NT) {
#pragma unroll
            for (int h = 0; h < 2; h++) {
              double* dst = R + (8 * a + g) * WP + 8 * b + 2 * q + h;
              *dst = round == 0 ? acc[a][b][h] : *dst + acc[a][b][h];
            }
          }
      __syncwarp();
#pragma unroll
      for (int ci = 0; ci < MC; ci++) {
        if (ci >= m) break;
#pragma unroll
        for (int x = 0; x < CT; x++)
#pragma unroll
          for (int y = x; y < CT; y++)
#pragma unroll
            for (int h = 0; h < 2; h++) {
              const int lx = 8 * x + g, ly = 8 * y + 2 * q + h;          // entry of [A_c b]^T [A_c b]; column DC = b
              if (lx <= ly && ly <= DC) {
                const int i = lx < DC ? ci * DC + lx : s, j = ly < DC ? ci * DC + ly : s;
                R[i * WP + j] += accA[ci][x * CT - x * (x - 1) / 2 + (y - x)][h];
              }
            }
        __syncwarp();          // (the b^T b of every camera lands on the same entry)
      }
    }
    __syncthreads();
  }
  // one extend-add per run (HessianFactor::updateHessian of the leaf's separator factor)
  double* P = t.arena + t.off[p];
  const int pn = t.nf[p] + t.ns[p] + 1;
  const int* map = t.ea_map + t.ea_ptr[c0];
  for (int e = tid; e < w * w; e += 128) {
    const int i = e / w, j = e - i * w;
    if (i > j) continue;
    const int a = map[i], bq = map[j];
    const int lo = a < bq ? a : bq, hi = a < bq ? bq : a;
    atomicAdd(P + lo + (size_t)hi * pn, R[i * WP + j]);
  }
}

// ---------------------------------------------------------------------------
// large fronts: blocked right-looking partial Cholesky in global memory.
// Per panel [k0, k0+nb): (1) potrf of the nb x nb diagonal block + TRSM of the
// row panel (one CTA per clique), (2) SYRK update of the trailing upper
// triangle (grid of 64x64 tiles).
// ---------------------------------------------------------------------------
// (1) panel kernel: every CTA re-factors the kNB x kNB diagonal block in shared memory from
// the (fully updated, still unfactored) front, so no CTA waits for another and nobody reads a
// half-written block; CTA 0 publishes R_kk to a side buffer (rdiag) and does the pivot checks;
// then each CTA solves its kTrsmCols columns of the row panel (one thread per column).
// The following update kernel copies rdiag into the front.
constexpr int kTrsmCols = 128;

__global__ void __launch_bounds__(kTrsmCols)
panel_kernel(TreeView t, const int* __restrict__ list, int k0, Scalars* sc, double* __restrict__ rdiag) {
  pdl_sync();
  __shared__ double Dg[kNB][kNB + 1];
  __shared__ int bad;
  const int c = list[blockIdx.y];
  const int f = t.nf[c], n = f + t.ns[c] + 1;
  if (k0 >= f) return;
  const int nb = min(kNB, f - k0);
  const int j0 = k0 + nb + blockIdx.x * kTrsmCols;
  if (j0 >= n && blockIdx.x != 0) return;
  double* M = t.arena + t.off[c];
  const int tid = threadIdx.x;
  __shared__ double invd[kNB];
  if (tid == 0) bad = 0;
  // this thread's column of the row panel: issued now, consumed after the diagonal block is factored
  const int j = j0 + tid;
  double* col = M + k0 + (size_t)(j < n ? j : 0) * n;
  double x[kNB];
#pragma unroll
  for (int p = 0; p < kNB; p++) x[p] = (j < n && p < nb) ? col[p] : 0.0;
  __syncthreads();
  // Cholesky of the diagonal block by ONE warp, the matrix in registers: lane j owns column j.
  // Step k: r = sqrt(a_kk) (lane k), row k scaled, then lane j subtracts R(k,i) R(k,j) from its
  // a_ij with R(k,i) fetched from lane i by shuffle.  No block barrier inside the 32 steps.
  if (tid < 32) {
    const int lane = tid;
    double a[kNB];
#pragma unroll
    for (int i = 0; i < kNB; i++)
      a[i] = (lane < nb && i <= lane) ? M[(k0 + i) + (size_t)(k0 + lane) * n] : ((i == lane) ? 1.0 : 0.0);
    bool notpd = false;
#pragma unroll
    for (int k = 0; k < kNB; k++) {
      const double akk = __shfl_sync(0xffffffffu, a[k], k);
      if (k < nb && !(akk > 0.0)) notpd = true;
      // 600 sequential pivots are the critical path of the whole solve: one rsqrt (1 ulp) replaces
      // sqrt + divide (two long software sequences) per pivot; r = a*rsqrt(a), row scaled by rsqrt(a)
      const double rinv = rsqrt(akk);
      if (lane == k) a[k] = akk * rinv;
      else if (lane > k) a[k] = a[k] * rinv;
#pragma unroll
      for (int i = k + 1; i < kNB; i++) {
        const double rki = __shfl_sync(0xffffffffu, a[k], i);
        if (lane >= i) a[i] -= rki * a[k];
      }
    }
    if (notpd && lane == 0) bad = 1;
#pragma unroll
    for (int i = 0; i < kNB; i++) Dg[i][lane] = (i <= lane) ? a[i] : 0.0;
  }
  __syncthreads();
  if (tid < 32) invd[tid] = 1.0 / Dg[tid][tid];
  __syncthreads();
  if (blockIdx.x == 0) {
    if (tid == 0) {
      if (k0 + nb == f) {  // last panel: underconstrained check on the last two pivots
        if (f >= 2) {
          const double r2 = nb >= 2 ? Dg[nb - 2][nb - 2] : M[(f - 2) + (size_t)(f - 2) * n];
          if (!(dexp(r2) - dexp(Dg[nb - 1][nb - 1]) < 12)) bad = 1;
        } else if (!(dexp(Dg[0][0]) > -12)) bad = 1;
      }
      if (bad) atomicMax(&sc->fail_code, INT_MAX - c);
    }
    double* R = rdiag + (size_t)blockIdx.y * kNB * kNB;
    for (int e = tid; e < nb * nb; e += kTrsmCols) R[e] = Dg[e % nb][e / nb];
  }
  if (j < n) {  // x = R_kk^-T a, forward substitution
#pragma unroll
    for (int p = 0; p < kNB; p++) {
      if (p < nb) {
        double s = x[p];
#pragma unroll
        for (int q = 0; q < kNB; q++)
          if (q < p) s -= Dg[q][p] * x[q];
        x[p] = s * invd[p];
      }
    }
#pragma unroll
    for (int p = 0; p < kNB; p++)
      if (p < nb) col[p] = x[p];
  }
}

// (2) update kernel: C[i][j] -= sum_{p in [pa,pb)} M[p][i] M[p][j] for rows i in [ia,ib),
// columns j in [i, n), tiled TILE x TILE with RB x RB register blocking.  Modes:
//   0 SIMPLE  pa=k0      pb=k0+kNB  rows [pb, n)             (small fronts: full update per panel)
//   1 BAND    pa=k0      pb=k0+kNB  rows [pb, K0+kBig)       (rest of the current big panel only)
//   2 TRAIL   pa=K0      pb=K0+kBig rows [pb, n)             (one K=kBig update per big panel)
// The CTA with blockIdx.x == 0 also moves R_kk from rdiag into the front (modes 0 and 1).
constexpr int kBig = 128;

template <int TILE, int RB, int kKC>
__global__ void __launch_bounds__(256)
update_kernel(TreeView t, const int* __restrict__ list, int mode, int K0, int k0, const double* __restrict__ rdiag, int fuse_ea) {
  pdl_sync();
  __shared__ double Pi[kKC][TILE + 1];
  __shared__ double Pj[kKC][TILE + 1];
  const int c = list[blockIdx.y];
  const int f = t.nf[c], n = f + t.ns[c] + 1;
  double* M = t.arena + t.off[c];
  const int tid = threadIdx.x;
  if (mode != 2) {
    if (k0 >= f) return;
    if (blockIdx.x == 0) {
      const int nb = min(kNB, f - k0);
      const double* R = rdiag + (size_t)blockIdx.y * kNB * kNB;
      for (int e = tid; e < nb * nb; e += 256) {
        const int i = e % nb, j = e / nb;
        if (i <= j) M[(k0 + i) + (size_t)(k0 + j) * n] = R[e];
      }
    }
  } else if (K0 >= f) {
    return;
  }
  const int pa = mode == 2 ? K0 : k0;
  const int pb = mode == 2 ? min(K0 + kBig, f) : min(k0 + kNB, f);
  const int ia = pb;
  const int ib = mode == 1 ? min(K0 + kBig, f) : n;
  if (ia >= ib) return;
  const int TR = (ib - ia + TILE - 1) / TILE, TC = (n - ia + TILE - 1) / TILE;
  int rem = blockIdx.x, ti = 0;
  while (ti < TR && rem >= TC - ti) { rem -= TC - ti; ti++; }
  if (ti >= TR) return;
  const int tj = ti + rem;
  const int i0 = ia + ti * TILE, j0 = ia + tj * TILE;
  const int tx = tid & 15, ty = tid >> 4;
  double acc[RB][RB];
#pragma unroll
  for (int a = 0; a < RB; a++)
#pragma unroll
    for (int b = 0; b < RB; b++) acc[a][b] = 0.0;
  for (int kk = pa; kk < pb; kk += kKC) {
    for (int e = tid; e < kKC * TILE; e += 256) {
      const int p = e % kKC, cc = e / kKC;
      const int gi = i0 + cc, gj = j0 + cc;
      const bool pv = kk + p < pb;
      Pi[p][cc] = (pv && gi < ib) ? M[(kk + p) + (size_t)gi * n] : 0.0;
      Pj[p][cc] = (pv && gj < n) ? M[(kk + p) + (size_t)gj * n] : 0.0;
    }
    __syncthreads();
#pragma unroll 4
    for (int p = 0; p < kKC; p++) {
      double ai[RB], bj[RB];
#pragma unroll
      for (int a = 0; a < RB; a++) ai[a] = Pi[p][tx + 16 * a];
#pragma unroll
      for (int b = 0; b < RB; b++) bj[b] = Pj[p][ty + 16 * b];
#pragma unroll
      for (int a = 0; a < RB; a++)
#pragma unroll
        for (int b = 0; b < RB; b++) acc[a][b] += ai[a] * bj[b];
    }
    __syncthreads();
  }
  // The front's LAST update (its pivots end at pb) leaves the finished Schur complement: instead of
  // storing it and re-reading it in a separate extend-add launch, add it straight into the parent
  // (HessianFactor::updateHessian of the child factor, gtsam/linear/HessianFactor.cpp:348-374).
  const int par = t.parent[c];
  const bool to_parent = fuse_ea && mode != 1 && pb == f && par >= 0;
  if (to_parent) {
    double* P = t.arena + t.off[par];
    const int pn = t.nf[par] + t.ns[par] + 1;
    const int* map = t.ea_map + t.ea_ptr[c];
#pragma unroll
    for (int b = 0; b < RB; b++)
#pragma unroll
      for (int a = 0; a < RB; a++) {
        const int gi = i0 + tx + 16 * a, gj = j0 + ty + 16 * b;
        if (gi < ib && gj < n && gi <= gj) {
          const int pi = map[gi - f], pj = map[gj - f];
          const int lo = pi < pj ? pi : pj, hi = pi < pj ? pj : pi;
          atomicAdd(P + lo + (size_t)hi * pn, M[gi + (size_t)gj * n] - acc[a][b]);
        }
      }
    return;
  }
#pragma unroll
  for (int b = 0; b < RB; b++)
#pragma unroll
    for (int a = 0; a < RB; a++) {
      const int gi = i0 + tx + 16 * a, gj = j0 + ty + 16 * b;
      if (gi < ib && gj < n && gi <= gj) M[gi + (size_t)gj * n] -= acc[a][b];
    }
}

// (3) the same trailing update for genuinely dense big fronts on the FP64 tensor path:
// mma.sync.aligned.m8n8k4.row.col.f64 (SASS: DMMA).  128x128 tile per CTA, 8 warps as 2x4,
// each warp owns 64x32 = 8x4 MMA tiles (64 FP64 accumulators per thread).  Fragment layout
// (PTX ISA, m8n8k4 .f64): A(row i = lane/4, col k = lane%4), B(row k = lane%4, col j = lane/4),
// C/D(row i = lane/4, cols 2*(lane%4) + {0,1}).  With C -= P^T P: A[i][k] = P[k][i], B[k][j] = P[k][j],
// both straight out of the staged row panels.  Only mode 2 (TRAIL) of update_kernel.

__global__ void __launch_bounds__(256)
update_dmma_kernel(TreeView t, const int* __restrict__ list, int K0, int fuse_ea) {
  constexpr int TILE = 128, KC = 16;
  __shared__ double Pi[KC][TILE + 4];
  __shared__ double Pj[KC][TILE + 4];
  pdl_sync();
  const int c = list[blockIdx.y];
  const int f = t.nf[c], n = f + t.ns[c] + 1;
  if (K0 >= f) return;
  double* M = t.arena + t.off[c];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int pa = K0, pb = min(K0 + kBig, f), ia = pb;
  if (ia >= n) return;
  const int TC = (n - ia + TILE - 1) / TILE;
  int rem = blockIdx.x, ti = 0;
  while (ti < TC && rem >= TC - ti) { rem -= TC - ti; ti++; }
  if (ti >= TC) return;
  const int tj = ti + rem;
  const int i0 = ia + ti * TILE, j0 = ia + tj * TILE;
  const int wi = (warp >> 2) * 64, wj = (warp & 3) * 32;   // warp sub-tile origin inside the CTA tile
  const int g = lane >> 2, q = lane & 3;
  double acc[8][4][2];
#pragma unroll
  for (int a = 0; a < 8; a++)
#pragma unroll
    for (int b = 0; b < 4; b++) acc[a][b][0] = acc[a][b][1] = 0.0;
  for (int kk = pa; kk < pb; kk += KC) {
    for (int e = tid; e < KC * TILE; e += 256) {
      const int p = e % KC, cc = e / KC;
      const int gi = i0 + cc, gj = j0 + cc;
      const bool pv = kk + p < pb;
      Pi[p][cc] = (pv && gi < n) ? M[(kk + p) + (size_t)gi * n] : 0.0;
      Pj[p][cc] = (pv && gj < n) ? M[(kk + p) + (size_t)gj * n] : 0.0;
    }
    __syncthreads();
#pragma unroll
    for (int k4 = 0; k4 < KC; k4 += 4) {
      double af[8], bf[4];
#pragma unroll
      for (int a = 0; a < 8; a++) af[a] = Pi[k4 + q][wi + 8 * a + g];
#pragma unroll
      for (int b = 0; b < 4; b++) bf[b] = Pj[k4 + q][wj + 8 * b + g];
#pragma unroll
      for (int a = 0; a < 8; a++)
#pragma unroll
        for (int b = 0; b < 4; b++) dmma_m8n8k4(acc[a][b][0], acc[a][b][1], af[a], bf[b]);
    }
    __syncthreads();
  }
  const int par = t.parent[c];
  if (fuse_ea && pb == f && par >= 0) {   // last update of the front: extend-add into the parent (see update_kernel)
    double* P = t.arena + t.off[par];
    const int pn = t.nf[par] + t.ns[par] + 1;
    const int* map = t.ea_map + t.ea_ptr[c];
#pragma unroll
    for (int a = 0; a < 8; a++)
#pragma unroll
      for (int b = 0; b < 4; b++)
#pragma unroll
        for (int h = 0; h < 2; h++) {
          const int gi = i0 + wi + 8 * a + g, gj = j0 + wj + 8 * b + 2 * q + h;
          if (gi < n && gj < n && gi <= gj) {
            const int pi = map[gi - f], pj = map[gj - f];
            const int lo = pi < pj ? pi : pj, hi = pi < pj ? pj : pi;
            atomicAdd(P + lo + (size_t)hi * pn, M[gi + (size_t)gj * n] - acc[a][b][h]);
          }
        }
    return;
  }
#pragma unroll
  for (int a = 0; a < 8; a++)
#pragma unroll
    for (int b = 0; b < 4; b++)
#pragma unroll
      for (int h = 0; h < 2; h++) {
        const int gi = i0 + wi + 8 * a + g, gj = j0 + wj + 8 * b + 2 * q + h;
        if (gi < n && gj < n && gi <= gj) M[gi + (size_t)gj * n] -= acc[a][b][h];
      }
}

__global__ void __launch_bounds__(256) extend_add_kernel(TreeView t, const int* __restrict__ list) {
  pdl_sync();
  const int c = list[blockIdx.y];
  const int p = t.parent[c];
  if (p < 0) return;
  const int f = t.nf[c], s = t.ns[c], n = f + s + 1, w = s + 1;
  const int64_t total = (int64_t)w * w;
  const double* M = t.arena + t.off[c];
  double* P = t.arena + t.off[p];
  const int pn = t.nf[p] + t.ns[p] + 1;
  const int* map = t.ea_map + t.ea_ptr[c];
  for (int64_t e = (int64_t)blockIdx.x * 256 + threadIdx.x; e < total; e += (int64_t)gridDim.x * 256) {
    const int i = (int)(e % w), j = (int)(e / w);
    if (i <= j) {
      const int pi = map[i], pj = map[j];
      const int lo = pi < pj ? pi : pj, hi = pi < pj ? pj : pi;
      atomicAdd(P + lo + (size_t)hi * pn, M[(f + i) + (size_t)(f + j) * n]);
    }
  }
}

}  // namespace b200
#include "front_df.cuh"   // tile-dataflow partial Cholesky of all non-leaf fronts in one launch
namespace b200 {

// ---------------------------------------------------------------------------
// back-substitution (gtsam/linear/linearAlgorithms-inst.h:50-117)
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(kWarpsPerBlock * 32)
backsub_small_kernel(TreeView t, const int* __restrict__ list, int count, double* delta, Scalars* sc) {
  pdl_sync();
  __shared__ double xs[kWarpsPerBlock][kSmallMaxN];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int idx = blockIdx.x * kWarpsPerBlock + warp;
  if (idx >= count) return;
  const int c = list[idx];
  const int f = t.nf[c], s = t.ns[c], n = f + s + 1, ld = t.ld[c];
  const double* M = t.arena + t.off[c];
  const int* di = t.didx + t.didx_ptr[c];
  double* x = xs[warp];
  // small triangular block staged up front (f <= 8: every BAL point): the solve below then has no
  // dependent global load on its critical path
  __shared__ double Rst[kWarpsPerBlock][64];
  const bool staged = f <= 8;
  if (staged)
    for (int e = lane; e < f * f; e += 32) Rst[warp][e] = M[(e % f) + (size_t)(e / f) * ld];
  // rhs = d - S x_S with the lanes spread over the separator columns (coalesced: the f entries of a
  // column are contiguous and consecutive columns are adjacent), 8 rows at a time, warp-reduced
  for (int i0 = 0; i0 < f; i0 += 8) {
    double a[8];
#pragma unroll
    for (int k = 0; k < 8; k++) a[k] = 0.0;
    for (int cc = lane; cc < s; cc += 32) {
      const double xsv = delta[di[f + cc]];
      const double* col = M + (size_t)(f + cc) * ld + i0;
#pragma unroll
      for (int k = 0; k < 8; k++)
        if (i0 + k < f) a[k] += col[k] * xsv;
    }
#pragma unroll
    for (int k = 0; k < 8; k++) {
      const double sum = warp_sum(a[k]);
      if (lane == 0 && i0 + k < f) x[i0 + k] = M[(i0 + k) + (size_t)(n - 1) * ld] - sum;
    }
  }
  __syncwarp();
  for (int i = f - 1; i >= 0; i--) {
    if (lane == 0) x[i] = x[i] / (staged ? Rst[warp][i + i * f] : M[i + (size_t)i * ld]);
    __syncwarp();
    const double xi = x[i];
    for (int k = lane; k < i; k += 32) x[k] -= (staged ? Rst[warp][k + i * f] : M[k + (size_t)i * ld]) * xi;
    __syncwarp();
  }
  bool nan = false;
  for (int i = lane; i < f; i += 32) {
    delta[di[i]] = x[i];
    if (isnan(x[i])) nan = true;
  }
  if (nan) atomicMax(&sc->nan_code, INT_MAX - c);
}

// Large cliques: x_F = R^-1 (d - S x_S) with several CTAs per clique and no global barrier.
// CTA b owns a block of kBsRows rows of the clique (blockIdx.x = 0 is the BOTTOM block, which
// depends on nobody; a CTA only ever waits on CTAs with a smaller blockIdx.x, so the wait cannot
// deadlock).  Each CTA accumulates d - S x_S for its rows, then consumes the x blocks below it as
// they are published (flag = epoch of this solve, release/acquire through L2), solves its own
// 64x64 diagonal block as two 32x32 warp-shuffle solves, and publishes.  The critical path per
// block is one flag hop + one 64-column GEMV + the in-block solve; everything else overlaps.
constexpr int kBsRows = 64;

// BAL point leaves (compact conditional [R S' d'], 3 x n): 8 lanes per point, lane k multiplies
// camera k's 3 x DC block of S' with that camera's slice of delta, an 8-lane shuffle reduction
// gives d' - S' x_S, lane 0 solves the 3 x 3 triangle.  ~1/20 of the instructions of the generic
// one-warp-per-clique kernel on the same cliques.
template <int DC>
__global__ void __launch_bounds__(128)
backsub_point_kernel(TreeView t, const int* __restrict__ list, int count, double* delta, Scalars* sc) {
  pdl_sync();
  const int sub = threadIdx.x & 7;
  const int idx = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 3);
  const bool live = idx < count;
  const int c = live ? list[idx] : list[0];
  const int s = t.ns[c];
  const int m = live ? s / DC : 0;
  const double* M = t.arena + t.off[c];
  const int* di = t.didx + t.didx_ptr[c];
  double a0 = 0.0, a1 = 0.0, a2 = 0.0;
  if (sub < m) {
    const double* xs = delta + di[3 + DC * sub];   // a variable's dofs are contiguous in delta
    const double* S = M + 3 * (3 + DC * sub);
#pragma unroll
    for (int cc = 0; cc < DC; cc++) {
      const double x = xs[cc];
      a0 += S[3 * cc] * x; a1 += S[3 * cc + 1] * x; a2 += S[3 * cc + 2] * x;
    }
  }
#pragma unroll
  for (int o = 4; o > 0; o >>= 1) {
    a0 += __shfl_xor_sync(0xffffffffu, a0, o);
    a1 += __shfl_xor_sync(0xffffffffu, a1, o);
    a2 += __shfl_xor_sync(0xffffffffu, a2, o);
  }
  if (live && sub == 0) {
    const double* d = M + 3 * (3 + s);
    const double x2 = (d[2] - a2) / M[8];
    const double x1 = ((d[1] - a1) - M[7] * x2) / M[4];
    const double x0 = (((d[0] - a0) - M[6] * x2) - M[3] * x1) / M[0];
    double* xo = delta + di[0];
    xo[0] = x0; xo[1] = x1; xo[2] = x2;
    if (isnan(x0) || isnan(x1) || isnan(x2)) atomicMax(&sc->nan_code, INT_MAX - c);
  }
}

__global__ void __launch_bounds__(256)
backsub_large_kernel(TreeView t, const int* __restrict__ list, double* delta, Scalars* sc, int* flags,
                     const int* __restrict__ flag_base, int list_begin, int epoch,
                     const double* __restrict__ winv, const int64_t* __restrict__ winv_off) {
  pdl_sync();
  __shared__ double part[4][kBsRows];
  __shared__ double rhs[kBsRows];
  __shared__ double Dg[3][32][33];   // [0]: rows 0..31 diag, [1]: rows 32..63 diag, [2]: coupling rows 0..31 x cols 32..63
  __shared__ double invd[kBsRows];   // (with W: Dg[0] / Dg[1] hold W_lo / W_hi column-major, Dg[b][j][i] = W[i][j])
  const int c = list[blockIdx.y];
  const int f = t.nf[c], s = t.ns[c], n = f + s + 1;
  const int nblk = (f + kBsRows - 1) / kBsRows;
  if ((int)blockIdx.x >= nblk) return;
  const int rb = nblk - 1 - blockIdx.x;
  const int r0 = rb * kBsRows, r1 = min(f, r0 + kBsRows), nr = r1 - r0;
  const double* M = t.arena + t.off[c];
  const int* di = t.didx + t.didx_ptr[c];
  int* fl = flags + flag_base[list_begin + blockIdx.y];
  const int tid = threadIdx.x, row = tid & (kBsRows - 1), q = tid >> 6, lane = tid & 31, warp = tid >> 5;
  // front_df_kernel left W = R_kk^-1 of every 32 x 32 diagonal block: the two triangular solves become matrix-vector products
  const double* W = (winv && winv_off && winv_off[c] >= 0) ? winv + winv_off[c] + (size_t)(2 * rb) * 1024 : nullptr;
  // stage this block's diagonal data now: it overlaps with the waits below
  for (int e = tid; e < 3 * 1024; e += 256) {
    const int blk = e >> 10, i = e & 31, j = (e >> 5) & 31;
    double v = 0.0;
    if (W && blk < 2) {
      if (blk == 0 || nr > 32) v = W[(size_t)blk * 1024 + j * 32 + i];     // coalesced over i; Dg[blk][j][i] = W_blk[i][j]
      Dg[blk][j][i] = v;
    } else {
      const int gi = (blk == 1 ? 32 : 0) + i, gj = (blk == 0 ? 0 : 32) + j;
      if (gi < nr && gj < nr && gi <= gj) v = M[(r0 + gi) + (size_t)(r0 + gj) * n];
      Dg[blk][i][j] = v;
    }
  }
  double acc = 0.0;
  if (row < nr) {
    const double* Mr = M + r0 + row;
    for (int cc = q; cc < s; cc += 4) acc += Mr[(size_t)(f + cc) * n] * delta[di[f + cc]];
  }
  for (int jb = nblk - 1; jb > rb; jb--) {
    // the entries of R are there before the solution is: fetch them ahead of the wait (the last wait is the pivot chain)
    const int c0 = jb * kBsRows, c1 = min(f, c0 + kBsRows);
    double rv[kBsRows / 4];
#pragma unroll
    for (int u = 0; u < kBsRows / 4; u++) {
      const int j = c0 + q + 4 * u;
      rv[u] = (row < nr && j < c1) ? M[(r0 + row) + (size_t)j * n] : 0.0;
    }
    if (tid == 0) {
      int spins = 0;   // bounded: a scheduling surprise must never hang the GPU
#ifdef B200_EMULATE
      while (atomicAdd(fl + jb, 0) != epoch && ++spins < (1 << 22)) {}
#else
      while (df_ld_relaxed(fl + jb) != epoch && ++spins < (1 << 22)) {}
      df_fence_acquire();
#endif
      if (spins >= (1 << 22)) atomicMax(&sc->nan_code, INT_MAX - c);
    }
    __syncthreads();
#pragma unroll
    for (int u = 0; u < kBsRows / 4; u++) {
      const int j = c0 + q + 4 * u;
      if (j < c1) acc += rv[u] * __ldcg(delta + di[j]);
    }
  }
  part[q][row] = acc;
  __syncthreads();
  if (tid < kBsRows) {
    rhs[tid] = tid < nr ? M[r0 + tid + (size_t)(n - 1) * n] - (part[0][tid] + part[1][tid] + part[2][tid] + part[3][tid]) : 0.0;
    if (!W) invd[tid] = tid < nr ? 1.0 / Dg[tid >> 5][tid & 31][tid & 31] : 1.0;
  }
  __syncthreads();
  if (warp == 0) {   // one warp: solve rows 32..63, apply the coupling block, solve rows 0..31
    for (int sb = (nr > 32 ? 1 : 0); sb >= 0; sb--) {
      const int b0 = 32 * sb, nb = min(32, nr - b0);
      double xv;
      if (W) {
        xv = 0.0;
#pragma unroll 8
        for (int j = 0; j < 32; j++) xv += Dg[sb][j][lane] * rhs[b0 + j];   // x = W rhs (W upper: zero below the diagonal)
      } else {
        xv = lane < nb ? rhs[b0 + lane] : 0.0;
        for (int k = nb - 1; k >= 0; k--) {
          const double xk = __shfl_sync(0xffffffffu, xv, k) * invd[b0 + k];
          if (lane == k) xv = xk;
          else if (lane < k) xv -= Dg[sb][lane][k] * xk;
        }
      }
      __syncwarp();
      if (lane < nb) rhs[b0 + lane] = xv;
      __syncwarp();
      if (sb == 1) {
        double a = 0;
        for (int j = 0; j < nb; j++) a += Dg[2][lane][j] * rhs[32 + j];
        rhs[lane] -= a;
        __syncwarp();
      }
    }
  }
  __syncthreads();
  bool nan = false;
  if (tid < nr) {
    delta[di[r0 + tid]] = rhs[tid];
    nan = isnan(rhs[tid]);
  }
  if (nan) atomicMax(&sc->nan_code, INT_MAX - c);
  __syncthreads();
#ifdef B200_EMULATE
  __threadfence();
  if (tid == 0) atomicExch(fl + rb, epoch);
#else
  if (tid == 0) df_st_release(fl + rb, epoch);
#endif
}

// ---------------------------------------------------------------------------
// Marginals::marginalCovariance (gtsam/nonlinear/Marginals.cpp:118-154): the (j, j) block of H^-1 from the
// factor already on the device.  H = U^T U with the rows [R S] of U stored per clique, so column k of the
// block is x = U^-1 U^-T e_k restricted to variable j.  e_k lives in j's clique, the forward solve
// U^T y = e_k only touches the cliques on the path from there to the root, and x_j only depends on that
// same path: one CTA per column walks the path up (y_F = R^-T g_F, g_S -= S^T y_F) and down
// (x_F = R^-1 (y_F - S x_S)).  work: one scratch vector of ndelta doubles per column.
// ---------------------------------------------------------------------------
constexpr int kMargMaxF = 4096;   // pivots of one clique staged in shared memory

__global__ void __launch_bounds__(256)
marginal_path_kernel(TreeView t, const int* __restrict__ path, int npath, int dof0, int d, double* __restrict__ work,
                     int64_t ndelta, double* __restrict__ out) {
  __shared__ double yv[kMargMaxF];
  const int kcol = blockIdx.x, tid = threadIdx.x;
  double* w = work + (size_t)kcol * ndelta;
  // zero the entries this walk can touch (frontals of the path cliques cover their separators too), then e_k
  for (int q = 0; q < npath; q++) {
    const int c = path[q];
    const int* di = t.didx + t.didx_ptr[c];
    for (int i = tid; i < t.nf[c]; i += 256) w[di[i]] = 0.0;
  }
  __syncthreads();
  if (tid == 0) w[dof0 + kcol] = 1.0;
  __syncthreads();
  for (int q = 0; q < npath; q++) {   // U^T y = e_k, leaf-side clique first
    const int c = path[q];
    const int f = t.nf[c], s = t.ns[c], ld = t.ld[c];
    const double* M = t.arena + t.off[c];
    const int* di = t.didx + t.didx_ptr[c];
    for (int i = tid; i < f; i += 256) yv[i] = w[di[i]];
    __syncthreads();
    for (int i = 0; i < f; i++) {
      if (tid == 0) yv[i] = yv[i] / M[i + (size_t)i * ld];
      __syncthreads();
      const double yi = yv[i];
      for (int j = i + 1 + tid; j < f; j += 256) yv[j] -= M[i + (size_t)j * ld] * yi;
      __syncthreads();
    }
    for (int i = tid; i < f; i += 256) w[di[i]] = yv[i];
    for (int j = tid; j < s; j += 256) {
      const double* col = M + (size_t)(f + j) * ld;
      double acc = 0.0;
      for (int i = 0; i < f; i++) acc += col[i] * yv[i];
      w[di[f + j]] -= acc;
    }
    __syncthreads();
  }
  for (int q = npath - 1; q >= 0; q--) {   // U x = y, root first
    const int c = path[q];
    const int f = t.nf[c], s = t.ns[c], ld = t.ld[c];
    const double* M = t.arena + t.off[c];
    const int* di = t.didx + t.didx_ptr[c];
    for (int i = tid; i < f; i += 256) {
      double acc = w[di[i]];
      for (int j = 0; j < s; j++) acc -= M[i + (size_t)(f + j) * ld] * w[di[f + j]];
      yv[i] = acc;
    }
    __syncthreads();
    for (int i = f - 1; i >= 0; i--) {
      if (tid == 0) yv[i] = yv[i] / M[i + (size_t)i * ld];
      __syncthreads();
      const double xi = yv[i];
      for (int r = tid; r < i; r += 256) yv[r] -= M[r + (size_t)i * ld] * xi;
      __syncthreads();
    }
    for (int i = tid; i < f; i += 256) w[di[i]] = yv[i];
    __syncthreads();
  }
  for (int i = tid; i < d; i += 256) out[i + kcol * d] = w[dof0 + i];
}

// Marginals::jointMarginalCovariance: the same walk over the UNION of the variables' clique paths (ascending
// clique id = elimination order: parents have larger ids), one CTA per column of the D x D joint matrix;
// dofs[] lists the delta indices of the requested variables in sorted-variable order.
__global__ void __launch_bounds__(256)
marginal_joint_kernel(TreeView t, const int* __restrict__ path, int npath, const int* __restrict__ dofs, int D,
                      double* __restrict__ work, int64_t ndelta, double* __restrict__ out) {
  __shared__ double yv[kMargMaxF];
  const int kcol = blockIdx.x, tid = threadIdx.x;
  double* w = work + (size_t)kcol * ndelta;
  for (int q = 0; q < npath; q++) {
    const int c = path[q];
    const int* di = t.didx + t.didx_ptr[c];
    for (int i = tid; i < t.nf[c]; i += 256) w[di[i]] = 0.0;
  }
  __syncthreads();
  if (tid == 0) w[dofs[kcol]] = 1.0;
  __syncthreads();
  for (int q = 0; q < npath; q++) {   // U^T y = e_k in elimination order
    const int c = path[q];
    const int f = t.nf[c], s = t.ns[c], ld = t.ld[c];
    const double* M = t.arena + t.off[c];
    const int* di = t.didx + t.didx_ptr[c];
    for (int i = tid; i < f; i += 256) yv[i] = w[di[i]];
    __syncthreads();
    for (int i = 0; i < f; i++) {
      if (tid == 0) yv[i] = yv[i] / M[i + (size_t)i * ld];
      __syncthreads();
      const double yi = yv[i];
      for (int j = i + 1 + tid; j < f; j += 256) yv[j] -= M[i + (size_t)j * ld] * yi;
      __syncthreads();
    }
    for (int i = tid; i < f; i += 256) w[di[i]] = yv[i];
    for (int j = tid; j < s; j += 256) {
      const double* col = M + (size_t)(f + j) * ld;
      double acc = 0.0;
      for (int i = 0; i < f; i++) acc += col[i] * yv[i];
      w[di[f + j]] -= acc;
    }
    __syncthreads();
  }
  for (int q = npath - 1; q >= 0; q--) {   // U x = y, roots first
    const int c = path[q];
    const int f = t.nf[c], s = t.ns[c], ld = t.ld[c];
    const double* M = t.arena + t.off[c];
    const int* di = t.didx + t.didx_ptr[c];
    for (int i = tid; i < f; i += 256) {
      double acc = w[di[i]];
      for (int j = 0; j < s; j++) acc -= M[i + (size_t)(f + j) * ld] * w[di[f + j]];
      yv[i] = acc;
    }
    __syncthreads();
    for (int i = f - 1; i >= 0; i--) {
      if (tid == 0) yv[i] = yv[i] / M[i + (size_t)i * ld];
      __syncthreads();
      const double xi = yv[i];
      for (int r = tid; r < i; r += 256) yv[r] -= M[r + (size_t)i * ld] * xi;
      __syncthreads();
    }
    for (int i = tid; i < f; i += 256) w[di[i]] = yv[i];
    __syncthreads();
  }
  for (int i = tid; i < D; i += 256) out[i + (size_t)kcol * D] = w[dofs[i]];
}

// ---------------------------------------------------------------------------
// retract: Values::retract (gtsam/nonlinear/Values.cpp:52-63)
// ---------------------------------------------------------------------------
__global__ void retract_kernel(const double* __restrict__ values, const double* __restrict__ delta,
                               const int* __restrict__ val_off, const int* __restrict__ var_dof,
                               const int* __restrict__ var_type, int nvars, double* __restrict__ out) {
  pdl_sync();
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= nvars) return;
  const double* x = values + val_off[v];
  const double* d = delta + var_dof[v];
  double* y = out + val_off[v];
  const int ty = var_type[v];
  if (ty == B200_VAR_POINT3) {
    y[0] = x[0] + d[0]; y[1] = x[1] + d[1]; y[2] = x[2] + d[2];
  } else if (ty == B200_VAR_POSE2) {
    // x * ChartAtOrigin::Retract(d) = x * Pose2(d0, d1, d2) (gtsam/geometry/Pose2.cpp:99-109, Pose2.h:131-133)
    double s, c, sd, cd;
    sincos(x[2], &s, &c);
    sincos(d[2], &sd, &cd);
    double cn = c * cd - s * sd, sn = s * cd + c * sd;
    rot2_normalize(cn, sn);
    y[0] = x[0] + (c * d[0] - s * d[1]);
    y[1] = x[1] + (s * d[0] + c * d[1]);
    y[2] = atan2(sn, cn);
  } else {
    double xi[6];
#pragma unroll
    for (int i = 0; i < 6; i++) xi[i] = d[i];
    store_pose(pose_retract(load_pose(x), xi), y);
    if (ty == B200_VAR_CAM_BUNDLER) {
      // PinholeCamera::retract (gtsam/geometry/PinholeCamera.h:199-205), Cal3Bundler::retract
      y[12] = x[12] + d[6]; y[13] = x[13] + d[7]; y[14] = x[14] + d[8];
      y[15] = x[15]; y[16] = x[16];
    }
  }
}

}  // namespace b200
