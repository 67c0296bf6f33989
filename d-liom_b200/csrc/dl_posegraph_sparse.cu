// Block-sparse sparse pose adjustment: OptimizationProblem3D::Solve (optimization_problem_3d.cc:259-589) on whole trajectories,
// with frozen trajectories (:283-329).
//
// Structure: every residual of this fork is a SpaCostFunction3D between one submap and one node, so the normal equations are
//   [ blockdiag(H_ss)  H_sn            ]
//   [ H_ns             blockdiag(H_nn) ]
// Eliminating the node blocks (Schur complement) leaves a dense system over the submaps only, which one CTA factors with a
// Cholesky; the node steps follow by back-substitution. In exact arithmetic this is the LM step of the dense normal equations,
// as the oracle (oracle/orc_posegraph.h) takes it.
//
// Every pose owns a 6-slot block; its first dim(p) slots are live: 0 if frozen or if no constraint (on any rank) refers to it
// (Ceres's Program::RemoveFixedBlocks removes constant and unused blocks, so neither moves nor enters ||x||), 2 for the first
// submap (constant translation, ConstantYawQuaternionPlus), else 3 + tdof (fix_z: tdof = 2). Dead slots carry zeros in the
// Jacobian and an identity in the damped node blocks, so that they leave the live entries of every factor bit-unchanged.
//
// Per evaluation: one thread per constraint writes its residual and 6 x 12 local Jacobian; one thread per output scalar sums
// them into the pose blocks (H_pp, g_p) and pair blocks (H_sn) along fixed-order CSR lists (no floating-point atomics, so a
// solve is bit-reproducible on one GPU); with a communicator one ncclAllReduce(fp64) sums
//   2 + 42 (S + N) + 36 P doubles   (cost, fixed cost, g_p and H_pp per pose, H_sn per distinct (submap, node) pair)
// over the ranks. Every rank then does identical work, so the replicas cannot drift.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <map>
#include <utility>
#include <vector>

#include "dl_posegraph.cuh"

namespace dl {
namespace {
using namespace pg;

constexpr int kMaxReduced = 3072;  // the one-CTA factor's limit (DL_POSE_GRAPH_MAX_REDUCED)

struct SparseGraph {
  int S, N, tdof;
  const int* dim;   // [S + N] live local parameters per pose
  const int* roff;  // [S] offset of a submap's live parameters in the reduced system
  int n_red;
};

// One thread per constraint: residual, cost and the local Jacobian (6 x 12: submap slots 0..5, node slots 6..11).
__global__ void sp_evaluate_kernel(SparseGraph gr, const double* __restrict__ x, const dl_spa_constraint* __restrict__ constraints,
                                   int num_constraints, int with_jacobian, double* __restrict__ Jc, double* __restrict__ ec,
                                   double* __restrict__ c2) {
  const int ci = blockIdx.x * blockDim.x + threadIdx.x;
  if (ci >= num_constraints) return;
  const dl_spa_constraint c = constraints[ci];
  const int pi = c.submap, pj = gr.S + c.node;
  const double* xi = x + 7 * pi;
  const double* xj = x + 7 * pj;
  Dual e[6];
  spa_residual(c, xi + 3, xi, xj + 3, xj, e);
  double s = 0;
  for (int r = 0; r < 6; ++r) s += e[r].a * e[r].a;
  c2[ci] = s;
  if (!with_jacobian) return;
  const int di = gr.dim[pi], dj = gr.dim[pj];
  double* J = Jc + (size_t)ci * 72;
  for (int r = 0; r < 6; ++r) {
    double row[12];
    for (int k = 0; k < 12; ++k) row[k] = 0.;
    {
      const double w = xi[3], xx = xi[4], y = xi[5], zq = xi[6];
      const double* de = e[r].v;
      if (di == 2) {  // ConstantYawQuaternionPlus: d (q * (1, d0, d1, 0)) / d d0 = q * (0,1,0,0), / d d1 = q * (0,0,1,0)
        const double c0[4] = {-xx, w, zq, -y}, c1[4] = {-y, -zq, w, xx};
        for (int k = 0; k < 4; ++k) { row[0] += de[k] * c0[k]; row[1] += de[k] * c1[k]; }
      } else if (di > 0) {  // QuaternionParameterization::ComputeJacobian
        const double jj[4][3] = {{-xx, -y, -zq}, {w, zq, -y}, {-zq, w, xx}, {y, -xx, w}};
        for (int k = 0; k < 4; ++k)
          for (int a = 0; a < 3; ++a) row[a] += de[k] * jj[k][a];
        for (int k = 0; k < di - 3; ++k) row[3 + k] = de[4 + k];
      }
    }
    if (dj > 0) {
      const double w = xj[3], xx = xj[4], y = xj[5], zq = xj[6];
      const double* de = e[r].v + 7;
      const double jj[4][3] = {{-xx, -y, -zq}, {w, zq, -y}, {-zq, w, xx}, {y, -xx, w}};
      for (int k = 0; k < 4; ++k)
        for (int a = 0; a < 3; ++a) row[6 + a] += de[k] * jj[k][a];
      for (int k = 0; k < dj - 3; ++k) row[6 + 3 + k] = de[4 + k];
    }
    for (int k = 0; k < 12; ++k) J[r * 12 + k] = row[k];
    ec[(size_t)ci * 6 + r] = e[r].a;
  }
}

// Payload layout (one all-reduce): [0] sum of squared residuals, [1] the same over the constraints between frozen poses,
// then g (6 per pose), H_pp (36 per pose), H_sn (36 per pair, row = submap slot, column = node slot).
struct Payload {
  int P, K;
  __host__ __device__ size_t g(int p) const { return 2 + (size_t)6 * p; }
  __host__ __device__ size_t hp(int p) const { return 2 + (size_t)6 * P + (size_t)36 * p; }
  __host__ __device__ size_t hk(int k) const { return 2 + (size_t)42 * P + (size_t)36 * k; }
  __host__ __device__ size_t size() const { return 2 + (size_t)42 * P + (size_t)36 * K; }
};

// One thread per payload scalar (except the two costs): a sum over that pose's / pair's constraints in ascending order.
__global__ void sp_assemble_kernel(Payload pl, int S, const double* __restrict__ Jc, const double* __restrict__ ec,
                                   const int* __restrict__ pose_ptr, const int* __restrict__ pose_con,
                                   const int* __restrict__ pair_ptr, const int* __restrict__ pair_con, double* __restrict__ out) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t ng = (int64_t)6 * pl.P, nh = (int64_t)36 * pl.P, nk = (int64_t)36 * pl.K;
  if (t >= ng + nh + nk) return;
  double s = 0;
  if (t < ng) {                 // g_p[a] = sum_c sum_r J[r][a] e[r]
    const int p = (int)(t / 6), a = (int)(t % 6) + (p < S ? 0 : 6);
    for (int i = pose_ptr[p]; i < pose_ptr[p + 1]; ++i) {
      const int c = pose_con[i];
      const double* J = Jc + (size_t)c * 72;
      const double* e = ec + (size_t)c * 6;
      for (int r = 0; r < 6; ++r) s += J[r * 12 + a] * e[r];
    }
    out[2 + t] = s;
  } else if (t < ng + nh) {     // H_pp[a][b] = sum_c sum_r J[r][a] J[r][b]
    const int64_t u = t - ng;
    const int p = (int)(u / 36), off = p < S ? 0 : 6, a = (int)(u % 36) / 6 + off, b = (int)(u % 6) + off;
    for (int i = pose_ptr[p]; i < pose_ptr[p + 1]; ++i) {
      const double* J = Jc + (size_t)pose_con[i] * 72;
      for (int r = 0; r < 6; ++r) s += J[r * 12 + a] * J[r * 12 + b];
    }
    out[2 + t] = s;
  } else {                      // H_sn[a][b] = sum_c sum_r J[r][a] J[r][6 + b]
    const int64_t u = t - ng - nh;
    const int k = (int)(u / 36), a = (int)(u % 36) / 6, b = (int)(u % 6) + 6;
    for (int i = pair_ptr[k]; i < pair_ptr[k + 1]; ++i) {
      const double* J = Jc + (size_t)pair_con[i] * 72;
      for (int r = 0; r < 6; ++r) s += J[r * 12 + a] * J[r * 12 + b];
    }
    out[2 + t] = s;
  }
}

// One CTA, fixed shape: out = sum of v[0..n) (strided per thread, then a warp-shuffle tree, then the warps in order).
__device__ double cta_sum(const double* __restrict__ v, int n) {
  __shared__ double red[32];
  double part = 0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) part += v[i];
  for (int dd = 16; dd > 0; dd >>= 1) part += __shfl_xor_sync(0xffffffffu, part, dd);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = part;
  __syncthreads();
  double s = 0;
  if (threadIdx.x == 0)
    for (int w = 0; w < (int)(blockDim.x + 31) / 32; ++w) s += red[w];
  __syncthreads();
  return s;
}
__global__ void sp_cost_kernel(const double* __restrict__ c2, int n, const double* __restrict__ fixed2, double* out) {
  const double s = cta_sum(c2, n);
  if (threadIdx.x == 0) { out[0] = s; out[1] = fixed2 ? *fixed2 : 0.; }
}

// x (+) delta (6 slots per pose); one thread per pose. Frozen poses are copied.
__global__ void sp_plus_kernel(int P, const int* __restrict__ dim, const double* __restrict__ x, const double* __restrict__ delta,
                               size_t delta_stride_offset, double sign, double* __restrict__ out) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  const double* xp = x + 7 * p;
  const double* dl = delta + delta_stride_offset + 6 * p;
  double* o = out + 7 * p;
  const int d = dim[p];
  for (int k = 0; k < 7; ++k) o[k] = xp[k];
  if (d == 0) return;
  const Quatd q{xp[3], xp[4], xp[5], xp[6]};
  if (d == 2) {
    const double d0 = sign * dl[0], d1 = sign * dl[1];
    const double nn = sqrt(d0 * d0 + d1 * d1);
    const double s = nn < 1e-6 ? 1. : sin(nn) / nn;
    const Quatd r = qmul(q, Quatd{nn < 1e-6 ? 1. : cos(nn), s * d0, s * d1, 0.});
    o[3] = r.w; o[4] = r.x; o[5] = r.y; o[6] = r.z;
    return;
  }
  const double d0 = sign * dl[0], d1 = sign * dl[1], d2 = sign * dl[2];
  const double nn = sqrt(d0 * d0 + d1 * d1 + d2 * d2);
  if (nn > 0.) {
    const double s = sin(nn) / nn;
    const Quatd r = qmul(Quatd{cos(nn), s * d0, s * d1, s * d2}, q);
    o[3] = r.w; o[4] = r.x; o[5] = r.y; o[6] = r.z;
  }
  for (int k = 0; k < d - 3; ++k) o[k] = xp[k] + sign * dl[3 + k];
}

// Over the parameterised poses' ambient parameters (rotation of every live pose, translation of every live pose but the first
// submap): max |x - y|, ||x||, ||x - y||. One CTA, fixed shape.
__global__ void sp_norms_kernel(int P, const int* __restrict__ dim, const double* __restrict__ x, const double* __restrict__ y,
                                double* out3) {
  __shared__ double r0[32], r1[32], r2[32];
  double mx = 0, sx = 0, sd = 0;
  for (int i = threadIdx.x; i < 7 * P; i += blockDim.x) {
    const int p = i / 7, k = i % 7, d = dim[p];
    if (d == 0 || (d == 2 && k < 3)) continue;
    const double dxy = x[i] - y[i];
    mx = fmax(mx, fabs(dxy));
    sx += x[i] * x[i];
    sd += dxy * dxy;
  }
  for (int dd = 16; dd > 0; dd >>= 1) {
    mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, dd));
    sx += __shfl_xor_sync(0xffffffffu, sx, dd);
    sd += __shfl_xor_sync(0xffffffffu, sd, dd);
  }
  if ((threadIdx.x & 31) == 0) { r0[threadIdx.x >> 5] = mx; r1[threadIdx.x >> 5] = sx; r2[threadIdx.x >> 5] = sd; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double a = 0, b = 0, c = 0;
    for (int w = 0; w < (int)(blockDim.x + 31) / 32; ++w) { a = fmax(a, r0[w]); b += r1[w]; c += r2[w]; }
    out3[0] = a; out3[1] = sqrt(b); out3[2] = sqrt(c);
  }
}

// ---- the step. scalars: [0] radius, [1] reuse_diagonal, [2] compute_scale (in); [3] valid, [4] model_cost_change (out).
struct StepBufs {
  const double* sys;  // the payload at the current point
  double* scale;      // 6 per pose (Jacobi, from the first evaluation)
  double* diag;       // 6 per pose (LM diagonal of S H S, clamped)
  double* Lnode;      // 36 per pose (node Cholesky factor, lower, row-major)
  double* znode;      // 6 per pose: A_nn^-1 (S g)_n
  double* W;          // 36 per pair: S_s H_sn S_n
  double* Y;          // 36 per pair: A_nn^-1 W^T (row = node slot, column = submap slot)
  double* A;          // n_red x n_red reduced system, factored in place
  double* rhs;        // n_red: reduced right-hand side, then the submaps' y
  double* delta;      // 6 per pose: step * scale
  double* part;       // per pose: its share of the model cost change
  int* ok;            // 1 unless a factorisation failed or the step is not finite
  double* scalars;
};

// one thread per pose slot: Jacobi scale, LM diagonal
__global__ void sp_scale_kernel(Payload pl, const int* __restrict__ dim, StepBufs b) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t == 0) *b.ok = 1;
  if (t >= 6 * pl.P) return;
  const int p = t / 6, a = t % 6;
  const bool reuse = b.scalars[1] != 0., compute_scale = b.scalars[2] != 0.;
  if (a >= dim[p]) { b.scale[t] = 0.; b.diag[t] = 0.; return; }
  const double h = b.sys[pl.hp(p) + a * 6 + a];
  if (compute_scale) b.scale[t] = 1.0 / (1.0 + sqrt(h));
  const double hjj = b.scale[t] * h * b.scale[t];
  if (!reuse) b.diag[t] = fmin(fmax(hjj, lm_min_diag()), lm_max_diag());
}

// A = S H_pp S + D / radius over the live slots, identity over the dead ones
__device__ __forceinline__ void damped_block(const double* H, const double* sc, const double* dg, double radius, int d, double A[6][6]) {
#pragma unroll
  for (int a = 0; a < 6; ++a)
#pragma unroll
    for (int c = 0; c < 6; ++c) {
      double v = (a < d && c < d) ? sc[a] * H[a * 6 + c] * sc[c] : 0.;
      if (a == c) v = a < d ? v + dg[a] / radius : 1.;
      A[a][c] = v;
    }
}
__device__ __forceinline__ void chol_solve6(const double* L, double v[6]) {  // v <- (L L^T)^-1 v
#pragma unroll
  for (int i = 0; i < 6; ++i) {
    double s = v[i];
#pragma unroll
    for (int k = 0; k < i; ++k) s -= L[i * 6 + k] * v[k];
    v[i] = s / L[i * 6 + i];
  }
#pragma unroll
  for (int i = 5; i >= 0; --i) {
    double s = v[i];
#pragma unroll
    for (int k = i + 1; k < 6; ++k) s -= L[k * 6 + i] * v[k];
    v[i] = s / L[i * 6 + i];
  }
}

// one thread per node: factor the damped node block, z_n = A_nn^-1 (S g)_n
__global__ void sp_node_factor_kernel(Payload pl, int S, const int* __restrict__ dim, StepBufs b) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  const int p = S + n;
  if (p >= pl.P) return;
  const int d = dim[p];
  if (d == 0) {  // frozen: no parameters; z = 0 keeps its pairs out of the reduced right-hand side
    for (int a = 0; a < 6; ++a) b.znode[6 * p + a] = 0.;
    return;
  }
  const double radius = b.scalars[0];
  double A[6][6];
  damped_block(b.sys + pl.hp(p), b.scale + 6 * p, b.diag + 6 * p, radius, d, A);
  bool ok = true;
#pragma unroll
  for (int j = 0; j < 6; ++j) {
    double s = A[j][j];
#pragma unroll
    for (int k = 0; k < j; ++k) s -= A[j][k] * A[j][k];
    if (!(s > 0.)) ok = false;
    const double djj = sqrt(s);
    A[j][j] = djj;
#pragma unroll
    for (int i = j + 1; i < 6; ++i) {
      double t = A[i][j];
#pragma unroll
      for (int k = 0; k < j; ++k) t -= A[i][k] * A[j][k];
      A[i][j] = t / djj;
    }
  }
  if (!ok) *b.ok = 0;
  double* L = b.Lnode + (size_t)36 * p;
#pragma unroll
  for (int i = 0; i < 6; ++i)
#pragma unroll
    for (int k = 0; k < 6; ++k) L[i * 6 + k] = k <= i ? A[i][k] : 0.;
  double z[6];
#pragma unroll
  for (int a = 0; a < 6; ++a) z[a] = a < d ? b.scale[6 * p + a] * b.sys[pl.g(p) + a] : 0.;
  chol_solve6(L, z);
#pragma unroll
  for (int a = 0; a < 6; ++a) b.znode[6 * p + a] = z[a];
}

// one thread per pair: W = S_s H_sn S_n, Y = A_nn^-1 W^T
__global__ void sp_pair_kernel(Payload pl, int S, const int* __restrict__ dim, const int2* __restrict__ pairs, StepBufs b) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= pl.K) return;
  const int s = pairs[k].x, pn = S + pairs[k].y, ds = dim[s], dn = dim[pn];
  const double* H = b.sys + pl.hk(k);
  const double* L = b.Lnode + (size_t)36 * pn;
  double* W = b.W + (size_t)36 * k;
  double* Y = b.Y + (size_t)36 * k;
  for (int a = 0; a < 6; ++a) {
    double w[6];
#pragma unroll
    for (int c = 0; c < 6; ++c) {
      w[c] = (a < ds && c < dn) ? b.scale[6 * s + a] * H[a * 6 + c] * b.scale[6 * pn + c] : 0.;
      W[a * 6 + c] = w[c];
    }
    if (dn > 0) chol_solve6(L, w);
#pragma unroll
    for (int c = 0; c < 6; ++c) Y[c * 6 + a] = dn > 0 ? w[c] : 0.;
  }
}

// One CTA per reduced block (s1 <= s2): threads 0..35 the upper-triangle entries A_red[s1][s2] = [s1 == s2] (S H_ss S + D / radius)
//   - sum_n W_(s1,n) Y_(s2,n) over the block's node list (ascending node); on diagonal blocks threads 36..41 the right-hand side
//   (S g)_s - sum_n W_(s,n) z_n over the submap's pairs (ascending node).
__global__ void sp_reduce_kernel(Payload pl, int S, const int* __restrict__ dim, const int* __restrict__ roff, int n_red,
                                 const int2* __restrict__ blocks, const int* __restrict__ blk_ptr, const int2* __restrict__ blk_terms,
                                 const int2* __restrict__ pairs, const int* __restrict__ sub_ptr, StepBufs b) {
  const int r = blockIdx.x, t = threadIdx.x;
  const int s1 = blocks[r].x, s2 = blocks[r].y, d1 = dim[s1], d2 = dim[s2];
  if (t < 36) {
    const int a = t / 6, c = t % 6;
    // only the upper triangle is written (and read by the factor and the solves): on a diagonal block the entries (a, c) and
    // (c, a) round differently, and one writer per address keeps the solve bit-reproducible
    if (a >= d1 || c >= d2 || (s1 == s2 && c < a)) return;
    double v = 0;
    if (s1 == s2) {
      v = b.scale[6 * s1 + a] * b.sys[pl.hp(s1) + a * 6 + c] * b.scale[6 * s1 + c];
      if (a == c) v += b.diag[6 * s1 + a] / b.scalars[0];
    }
    for (int i = blk_ptr[r]; i < blk_ptr[r + 1]; ++i) {
      const double* W = b.W + (size_t)36 * blk_terms[i].x;
      const double* Y = b.Y + (size_t)36 * blk_terms[i].y;
      double s = 0;
#pragma unroll
      for (int k = 0; k < 6; ++k) s += W[a * 6 + k] * Y[k * 6 + c];
      v -= s;
    }
    b.A[(size_t)(roff[s1] + a) * n_red + roff[s2] + c] = v;
  } else if (t < 42 && s1 == s2) {
    const int a = t - 36;
    if (a >= d1) return;
    double v = b.scale[6 * s1 + a] * b.sys[pl.g(s1) + a];
    for (int k = sub_ptr[s1]; k < sub_ptr[s1 + 1]; ++k) {
      const double* W = b.W + (size_t)36 * k;
      const double* z = b.znode + 6 * (S + pairs[k].y);
      double s = 0;
#pragma unroll
      for (int c = 0; c < 6; ++c) s += W[a * 6 + c] * z[c];
      v -= s;
    }
    b.rhs[roff[s1] + a] = v;
  }
}

// One CTA: the reduced system's dense Cholesky and solves (cta_cholesky_*, dl_posegraph.cuh).
__global__ void __launch_bounds__(1024) sp_reduced_solve_kernel(int n_red, StepBufs b) {
  __shared__ int ok_s;
  cta_cholesky_factor(b.A, n_red, &ok_s);
  if (!ok_s) {
    if (threadIdx.x == 0) *b.ok = 0;
    return;
  }
  cta_cholesky_solve(b.A, n_red, b.rhs);
}

// One thread per pose: y (submaps from the reduced solve, nodes by back-substitution y_n = z_n - sum Y_(s,n) y_s), step = -y,
// delta = step * scale, and the pose's share of step . gs + 1/2 step^T (S H S) step (a node carries its pairs' cross terms).
__global__ void sp_backsub_kernel(Payload pl, int S, const int* __restrict__ dim, const int* __restrict__ roff,
                                  const int2* __restrict__ pairs, const int* __restrict__ node_ptr, const int* __restrict__ node_pairs,
                                  StepBufs b) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= pl.P) return;
  const int d = dim[p];
  const double* sc = b.scale + 6 * p;
  double st[6];
  bool finite = true;
#pragma unroll
  for (int a = 0; a < 6; ++a) st[a] = 0.;
  if (p < S) {
    for (int a = 0; a < d; ++a) st[a] = -b.rhs[roff[p] + a];
  } else if (d > 0) {
    const int n = p - S;
    double y[6];
#pragma unroll
    for (int a = 0; a < 6; ++a) y[a] = b.znode[6 * p + a];
    for (int i = node_ptr[n]; i < node_ptr[n + 1]; ++i) {
      const int k = node_pairs[i], s = pairs[k].x;
      const double* Y = b.Y + (size_t)36 * k;
      for (int c = 0; c < dim[s]; ++c) {
        const double ys = b.rhs[roff[s] + c];
#pragma unroll
        for (int a = 0; a < 6; ++a) y[a] -= Y[a * 6 + c] * ys;
      }
    }
#pragma unroll
    for (int a = 0; a < 6; ++a) st[a] = a < d ? -y[a] : 0.;
  }
  double part = 0;
  const double* H = b.sys + pl.hp(p);
  for (int a = 0; a < d; ++a) {
    if (!isfinite(st[a])) finite = false;
    double row = 0;
    for (int c = 0; c < d; ++c) row += (sc[a] * H[a * 6 + c] * sc[c]) * st[c];
    part += st[a] * (sc[a] * b.sys[pl.g(p) + a]) + 0.5 * st[a] * row;
    b.delta[6 * p + a] = st[a] * sc[a];
  }
  if (p >= S && d > 0) {  // cross terms step_s^T W step_n, counted once for both halves of the symmetric product
    const int n = p - S;
    for (int i = node_ptr[n]; i < node_ptr[n + 1]; ++i) {
      const int k = node_pairs[i], s = pairs[k].x;
      const double* W = b.W + (size_t)36 * k;
      for (int a = 0; a < dim[s]; ++a) {
        double row = 0;
        for (int c = 0; c < d; ++c) row += W[a * 6 + c] * st[c];
        part += -b.rhs[roff[s] + a] * row;
      }
    }
  }
  if (!finite) *b.ok = 0;
  b.part[p] = part;
}

__global__ void sp_finish_kernel(int P, StepBufs b) {
  const double s = cta_sum(b.part, P);
  if (threadIdx.x == 0) {
    const double mcc = -s;
    const bool valid = *b.ok != 0;
    b.scalars[3] = valid && mcc > 0. ? 1. : 0.;
    b.scalars[4] = valid ? mcc : 0.;
  }
}

// host-side CSR over a list of (key, value) appended in the order the values must be walked
struct Csr {
  std::vector<int> ptr, idx;
};
template <typename F>
Csr make_csr(int keys, int count, F key_of) {
  Csr c;
  c.ptr.assign(keys + 1, 0);
  for (int i = 0; i < count; ++i) c.ptr[key_of(i) + 1]++;
  for (int k = 0; k < keys; ++k) c.ptr[k + 1] += c.ptr[k];
  c.idx.resize(count);
  std::vector<int> fill(c.ptr.begin(), c.ptr.end() - 1);
  for (int i = 0; i < count; ++i) c.idx[fill[key_of(i)]++] = i;
  return c;
}

}  // namespace
}  // namespace dl

using namespace dl;

extern "C" int dl_pose_graph_solve_sparse(dl_context* ctx, dl_comm* comm, const dl_pose_graph_options* options, int32_t num_submaps,
                                          int32_t num_nodes, double* poses, const uint8_t* frozen,
                                          const dl_spa_constraint* constraints, int32_t num_constraints, dl_solve_summary* summary,
                                          dl_pose_graph_sparse_info* info) {
  // ---- everything the call can reject, before the first collective
  if (!ctx || !options || num_submaps < 1 || num_nodes < 0 || !poses || num_constraints < 0 || (num_constraints > 0 && !constraints))
    return DL_ERR_ARG;
  const int S = num_submaps, N = num_nodes, P = S + N, tdof = options->fix_z ? 2 : 3;
  for (int k = 0; k < num_constraints; ++k)
    if (constraints[k].submap < 0 || constraints[k].submap >= S || constraints[k].node < 0 || constraints[k].node >= N)
      return ctx->fail(DL_ERR_ARG, "constraint refers to a submap / node outside the graph");
  auto is_frozen = [&](int p) { return frozen && frozen[p]; };
  // The reduced system's limit holds for every submap that is not frozen, referenced or not, so that every rank can check it
  // before the first collective (which submaps the constraints refer to is only known after the exchange).
  int submap_capacity = 0;
  for (int s = 0; s < S; ++s) submap_capacity += is_frozen(s) ? 0 : s == 0 ? 2 : 3 + tdof;
  if (submap_capacity > kMaxReduced)
    return ctx->fail(DL_ERR_ARG, "pose graph has more submap parameters than the reduced system's one-CTA factor holds (> 3072)");
  cudaError_t e0 = cudaSetDevice(ctx->device);
  if (e0 != cudaSuccess) return ctx->cuda_fail(e0, "cudaSetDevice");
  // ---- setup: live constraints (not between two frozen poses) first, then those between two frozen poses (fixed cost only)
  std::vector<dl_spa_constraint> cons;
  cons.reserve(num_constraints);
  for (int pass = 0; pass < 2; ++pass)
    for (int k = 0; k < num_constraints; ++k) {
      const bool live = !(is_frozen(constraints[k].submap) && is_frozen(S + constraints[k].node));
      if (live == (pass == 0)) cons.push_back(constraints[k]);
    }
  int M = 0;
  while (M < (int)cons.size() && !(is_frozen(cons[M].submap) && is_frozen(S + cons[M].node))) ++M;
  const int F = (int)cons.size() - M;
  std::vector<std::pair<int, int>> local_pairs(M);
  for (int i = 0; i < M; ++i) local_pairs[i] = {cons[i].submap, cons[i].node};
  std::sort(local_pairs.begin(), local_pairs.end());
  local_pairs.erase(std::unique(local_pairs.begin(), local_pairs.end()), local_pairs.end());
  std::vector<std::pair<int, int>> pairs = local_pairs;
  int64_t setup_bytes = 0;
  // With a communicator every rank must take the same path through the collectives below. The set-up exchange: (pair count,
  // non-frozen submap parameters, S, N, hash of the frozen flags, fix_z, max_num_iterations) from every rank, checked on every rank
  // alike; then the pair lists padded to the largest count. Every scratch reservation made after the first collective is agreed on
  // by a one-int all-gather of its status, so that a rank that cannot reserve does not leave its peers waiting in the next
  // collective.
  const int world = comm ? dl_comm_world_size(comm) : 1;
  DeviceBuffer<int32_t> control;
  constexpr int kMeta = 8;
  if (comm) DL_TRY(alloc(ctx, control, (size_t)(kMeta + 1) * (world + 1)));
  int32_t* d_meta = control.get();
  int32_t* d_meta_all = d_meta ? d_meta + kMeta : nullptr;
  int32_t* d_st = d_meta ? d_meta + kMeta * (world + 1) : nullptr;
  int32_t* d_st_all = d_st ? d_st + 1 : nullptr;
  auto agree = [&](int st) -> int {  // the first failing rank's status on every rank
    if (!comm) return st;
    const int32_t mine = st;
    DL_CUDA(ctx, cudaMemcpyAsync(d_st, &mine, 4, cudaMemcpyHostToDevice, ctx->stream));
    DL_TRY(dl_comm_all_gather_dev(comm, d_st, d_st_all, 4));
    std::vector<int32_t> all(world);
    DL_CUDA(ctx, cudaMemcpyAsync(all.data(), d_st_all, 4 * (size_t)world, cudaMemcpyDeviceToHost, ctx->stream));
    DL_CUDA(ctx, ctx->wait_stream());
    setup_bytes += 4 * (int64_t)world;
    if (st != DL_OK) return st;
    for (int r = 0; r < world; ++r)
      if (all[r] != DL_OK) return ctx->fail(all[r], "another rank could not reserve the pose graph's device memory");
    return DL_OK;
  };
  if (comm) {
    uint32_t hash = 2166136261u;  // FNV-1a over the frozen flags
    for (int p = 0; p < P; ++p) hash = (hash ^ (uint32_t)(is_frozen(p) ? 1 : 0)) * 16777619u;
    const int32_t meta[kMeta] = {(int32_t)local_pairs.size(), submap_capacity, S, N, (int32_t)hash, options->fix_z ? 1 : 0,
                                 options->max_num_iterations, 0};
    DL_CUDA(ctx, cudaMemcpyAsync(d_meta, meta, sizeof(meta), cudaMemcpyHostToDevice, ctx->stream));
    DL_TRY(dl_comm_all_gather_dev(comm, d_meta, d_meta_all, (int64_t)sizeof(meta)));
    std::vector<int32_t> all(kMeta * world);
    DL_CUDA(ctx, cudaMemcpyAsync(all.data(), d_meta_all, sizeof(meta) * world, cudaMemcpyDeviceToHost, ctx->stream));
    DL_CUDA(ctx, ctx->wait_stream());
    setup_bytes += (int64_t)sizeof(meta) * world;
    int most = 0;
    for (int r = 0; r < world; ++r) {
      for (int k = 1; k < kMeta; ++k)
        if (all[kMeta * r + k] != meta[k])
          return ctx->fail(DL_ERR_ARG, "pose graph differs between the ranks (submaps, nodes, frozen poses, reduced size or options)");
      most = std::max(most, (int)all[kMeta * r]);
    }
    if (most > 0) {
      const size_t per = (size_t)most * sizeof(int2);
      int2 *d_send, *d_recv;
      DL_TRY(agree(carve_scratch(ctx, [&](Arena& a) {
        d_send = a.take<int2>(most);
        d_recv = a.take<int2>((size_t)most * world);
      })));
      std::vector<int2> send(most, make_int2(-1, -1));
      for (size_t i = 0; i < local_pairs.size(); ++i) send[i] = make_int2(local_pairs[i].first, local_pairs[i].second);
      DL_CUDA(ctx, cudaMemcpyAsync(d_send, send.data(), per, cudaMemcpyHostToDevice, ctx->stream));
      DL_TRY(dl_comm_all_gather_dev(comm, d_send, d_recv, (int64_t)per));
      std::vector<int2> recv((size_t)most * world);
      DL_CUDA(ctx, cudaMemcpyAsync(recv.data(), d_recv, per * world, cudaMemcpyDeviceToHost, ctx->stream));
      DL_CUDA(ctx, ctx->wait_stream());
      setup_bytes += (int64_t)per * world;
      pairs.clear();
      for (const int2& v : recv)
        if (v.x >= 0) pairs.push_back({v.x, v.y});
      std::sort(pairs.begin(), pairs.end());
      pairs.erase(std::unique(pairs.begin(), pairs.end()), pairs.end());
    }
  }
  // A pose that no constraint refers to is not in Ceres's minimised program (Program::RemoveFixedBlocks drops unused parameter
  // blocks as well as constant ones): like a frozen pose it gets no parameters, so it neither moves nor enters ||x||. A pose that
  // is not frozen and is referenced on some rank sits in a live constraint there, so it is in the pair list every rank now holds:
  // the pairs decide, and every rank forms the same dims without another exchange.
  std::vector<uint8_t> used(P, 0);
  for (const auto& pr : pairs) used[pr.first] = used[S + pr.second] = 1;
  std::vector<int> dim(P), roff(S);
  int n_red = 0, n_local = 0;
  for (int p = 0; p < P; ++p) {
    dim[p] = (is_frozen(p) || !used[p]) ? 0 : p == 0 ? 2 : 3 + tdof;
    if (p < S) { roff[p] = n_red; n_red += dim[p]; }
    n_local += dim[p];
  }
  const int K = (int)pairs.size();
  std::vector<int> con_pair(M);
  for (int i = 0; i < M; ++i)
    con_pair[i] = (int)(std::lower_bound(pairs.begin(), pairs.end(), std::make_pair(cons[i].submap, cons[i].node)) - pairs.begin());
  // pose -> live constraints (a constraint sits in its submap's and its node's list, ascending index)
  Csr pose_con;
  {
    std::vector<int> key(2 * M);
    for (int i = 0; i < M; ++i) { key[2 * i] = cons[i].submap; key[2 * i + 1] = S + cons[i].node; }
    Csr c = make_csr(P, 2 * M, [&](int i) { return key[i]; });
    for (int& v : c.idx) v /= 2;
    pose_con = c;
  }
  Csr pair_con = make_csr(K, M, [&](int i) { return con_pair[i]; });
  Csr sub_pairs = make_csr(S, K, [&](int k) { return pairs[k].first; });   // ascending node within a submap
  Csr node_pairs = make_csr(N, K, [&](int k) { return pairs[k].second; }); // ascending submap within a node
  // reduced blocks (s1 <= s2, both live) and, per block, the (pair s1, pair s2) terms of the nodes that see both, ascending node
  std::map<std::pair<int, int>, int> block_of;
  for (int s = 0; s < S; ++s)
    if (dim[s] > 0) block_of.emplace(std::make_pair(s, s), 0);
  for (int n = 0; n < N; ++n) {
    if (dim[S + n] == 0) continue;
    for (int i = node_pairs.ptr[n]; i < node_pairs.ptr[n + 1]; ++i)
      for (int j = i; j < node_pairs.ptr[n + 1]; ++j) {
        const int s1 = pairs[node_pairs.idx[i]].first, s2 = pairs[node_pairs.idx[j]].first;
        if (dim[s1] > 0 && dim[s2] > 0) block_of.emplace(std::make_pair(s1, s2), 0);
      }
  }
  std::vector<int2> blocks;
  for (auto& kv : block_of) { kv.second = (int)blocks.size(); blocks.push_back(make_int2(kv.first.first, kv.first.second)); }
  const int R = (int)blocks.size();
  std::vector<int> term_block;
  std::vector<int2> terms_raw;
  for (int n = 0; n < N; ++n) {
    if (dim[S + n] == 0) continue;
    for (int i = node_pairs.ptr[n]; i < node_pairs.ptr[n + 1]; ++i)
      for (int j = i; j < node_pairs.ptr[n + 1]; ++j) {
        const int k1 = node_pairs.idx[i], k2 = node_pairs.idx[j], s1 = pairs[k1].first, s2 = pairs[k2].first;
        if (dim[s1] == 0 || dim[s2] == 0) continue;
        term_block.push_back(block_of[{s1, s2}]);
        terms_raw.push_back(make_int2(k1, k2));
      }
  }
  Csr blk = make_csr(R, (int)terms_raw.size(), [&](int i) { return term_block[i]; });
  std::vector<int2> terms(terms_raw.size());
  for (size_t i = 0; i < terms.size(); ++i) terms[i] = terms_raw[blk.idx[i]];
  std::vector<int2> pairs2(K);
  for (int k = 0; k < K; ++k) pairs2[k] = make_int2(pairs[k].first, pairs[k].second);

  // ---- device memory
  const Payload pl{P, K};
  const size_t sys = pl.size(), nr = (size_t)std::max(n_red, 1);
  auto I = [](size_t v) { return std::max<size_t>(v, 1); };
  double *d_sys[2], *d_x, *d_cand, *d_tmp, *d_best, *d_J, *d_e, *d_c2, *d_misc;
  StepBufs sb;
  sb.sys = nullptr;
  dl_spa_constraint* d_c;
  int *d_dim, *d_roff, *d_pose_ptr, *d_pose_con, *d_pair_ptr, *d_pair_con, *d_sub_ptr, *d_node_ptr, *d_node_pairs, *d_blk_ptr;
  int2 *d_pairs, *d_blocks, *d_terms;
  DL_TRY(agree(carve_scratch(ctx, [&](Arena& a) {
    d_sys[0] = a.take<double>(sys);
    d_sys[1] = a.take<double>(sys);
    d_x = a.take<double>((size_t)7 * P);
    d_cand = a.take<double>((size_t)7 * P);
    d_tmp = a.take<double>((size_t)7 * P);
    d_best = a.take<double>((size_t)7 * P);
    d_J = a.take<double>(I((size_t)M * 72));
    d_e = a.take<double>(I((size_t)M * 6));
    d_c2 = a.take<double>(I(cons.size()));
    d_misc = a.take<double>(8);  // [0] fixed cost2, [1..3] norms, [4..7] step scalars out
    sb.scale = a.take<double>((size_t)6 * P);
    sb.diag = a.take<double>((size_t)6 * P);
    sb.znode = a.take<double>((size_t)6 * P);
    sb.delta = a.take<double>((size_t)6 * P);
    sb.Lnode = a.take<double>((size_t)36 * P);
    sb.part = a.take<double>((size_t)P);
    sb.W = a.take<double>(I(K) * 36);
    sb.Y = a.take<double>(I(K) * 36);
    sb.A = a.take<double>(nr * nr);
    sb.rhs = a.take<double>(nr);
    sb.scalars = a.take<double>(8);
    sb.ok = a.take<int>(4);
    d_c = a.take<dl_spa_constraint>(I(cons.size()));
    d_dim = a.take<int>(P);
    d_roff = a.take<int>(S);
    d_pose_ptr = a.take<int>(I(pose_con.ptr.size()));
    d_pose_con = a.take<int>(I(pose_con.idx.size()));
    d_pair_ptr = a.take<int>(I(pair_con.ptr.size()));
    d_pair_con = a.take<int>(I(pair_con.idx.size()));
    d_pairs = a.take<int2>(I(pairs2.size()));
    d_sub_ptr = a.take<int>(I(sub_pairs.ptr.size()));
    d_node_ptr = a.take<int>(I(node_pairs.ptr.size()));
    d_node_pairs = a.take<int>(I(node_pairs.idx.size()));
    d_blocks = a.take<int2>(I(blocks.size()));
    d_blk_ptr = a.take<int>(I(blk.ptr.size()));
    d_terms = a.take<int2>(I(terms.size()));
  })));
  auto up = [&](auto* d, const auto& v) { return h2d(ctx, d, v.data(), v.size()); };
  DL_TRY(up(d_pose_ptr, pose_con.ptr));
  DL_TRY(up(d_pose_con, pose_con.idx));
  DL_TRY(up(d_pair_ptr, pair_con.ptr));
  DL_TRY(up(d_pair_con, pair_con.idx));
  DL_TRY(up(d_pairs, pairs2));
  DL_TRY(up(d_sub_ptr, sub_pairs.ptr));
  DL_TRY(up(d_node_ptr, node_pairs.ptr));
  DL_TRY(up(d_node_pairs, node_pairs.idx));
  DL_TRY(up(d_blocks, blocks));
  DL_TRY(up(d_blk_ptr, blk.ptr));
  DL_TRY(up(d_terms, terms));
  DL_CUDA(ctx, cudaMemcpyAsync(d_dim, dim.data(), (size_t)P * 4, cudaMemcpyHostToDevice, ctx->stream));
  DL_CUDA(ctx, cudaMemcpyAsync(d_roff, roff.data(), (size_t)S * 4, cudaMemcpyHostToDevice, ctx->stream));
  DL_CUDA(ctx, cudaMemcpyAsync(d_x, poses, (size_t)P * 56, cudaMemcpyHostToDevice, ctx->stream));
  DL_CUDA(ctx, cudaMemcpyAsync(d_best, poses, (size_t)P * 56, cudaMemcpyHostToDevice, ctx->stream));
  if (!cons.empty())
    DL_CUDA(ctx, cudaMemcpyAsync(d_c, cons.data(), cons.size() * sizeof(dl_spa_constraint), cudaMemcpyHostToDevice, ctx->stream));
  DL_CUDA(ctx, cudaGetLastError());
  const SparseGraph gr{S, N, tdof, d_dim, d_roff, n_red};
  // the constraints between frozen poses: their cost once
  if (F > 0) {
    sp_evaluate_kernel<<<(F + 127) / 128, 128, 0, ctx->stream>>>(gr, d_x, d_c + M, F, 0, nullptr, nullptr, d_c2 + M);
    DL_LAUNCH_CHECK(ctx, "sp_evaluate_kernel");
  }
  sp_cost_kernel<<<1, 256, 0, ctx->stream>>>(d_c2 + M, F, nullptr, d_misc);  // d_misc[0] = fixed cost2
  DL_LAUNCH_CHECK(ctx, "sp_cost_kernel");

  cudaEvent_t ev0, ev1;
  cudaEventCreate(&ev0);
  cudaEventCreate(&ev1);
  float reduce_ms = 0.f, reduce_min_ms = 1e30f;
  int reductions = 0;
  const int64_t scalars_total = (int64_t)6 * P + (int64_t)36 * P + (int64_t)36 * K;
  auto evaluate = [&](const double* at, int buf) -> int {
    if (M > 0) {
      sp_evaluate_kernel<<<(M + 63) / 64, 64, 0, ctx->stream>>>(gr, at, d_c, M, 1, d_J, d_e, d_c2);
      DL_LAUNCH_CHECK(ctx, "sp_evaluate_kernel");
    }
    sp_assemble_kernel<<<(unsigned)((scalars_total + 127) / 128), 128, 0, ctx->stream>>>(pl, S, d_J, d_e, d_pose_ptr, d_pose_con,
                                                                                       d_pair_ptr, d_pair_con, d_sys[buf]);
    DL_LAUNCH_CHECK(ctx, "sp_assemble_kernel");
    sp_cost_kernel<<<1, 256, 0, ctx->stream>>>(d_c2, M, d_misc, d_sys[buf]);
    DL_LAUNCH_CHECK(ctx, "sp_cost_kernel");
    if (comm) {
      DL_CUDA(ctx, cudaEventRecord(ev0, ctx->stream));
      DL_TRY(dl_comm_all_reduce_f64_dev(comm, d_sys[buf], (int64_t)sys));
      DL_CUDA(ctx, cudaEventRecord(ev1, ctx->stream));
      DL_CUDA(ctx, cudaEventSynchronize(ev1));
      float ms = 0.f;
      cudaEventElapsedTime(&ms, ev0, ev1);
      reduce_ms += ms;
      reduce_min_ms = std::fmin(reduce_min_ms, ms);
      ++reductions;
    }
    return DL_OK;
  };
  double fixed_cost = 0;
  auto cost_of = [&](int buf, double* c) -> int {
    double c2[2];
    DL_CUDA(ctx, cudaMemcpyAsync(c2, d_sys[buf], 16, cudaMemcpyDeviceToHost, ctx->stream));
    DL_CUDA(ctx, ctx->wait_stream());
    *c = 0.5 * c2[0];
    fixed_cost = 0.5 * c2[1];
    return DL_OK;
  };
  auto norms = [&](const double* x, const double* y, double* o) -> int {
    sp_norms_kernel<<<1, 256, 0, ctx->stream>>>(P, d_dim, x, y, d_misc + 1);
    DL_LAUNCH_CHECK(ctx, "sp_norms_kernel");
    DL_CUDA(ctx, cudaMemcpyAsync(o, d_misc + 1, 24, cudaMemcpyDeviceToHost, ctx->stream));
    DL_CUDA(ctx, ctx->wait_stream());
    return DL_OK;
  };
  // projected gradient max norm at (at, system buf): || at - Plus(at, -g) ||_max, and ||at||
  auto gradient_norms = [&](const double* at, int buf, double* gmax, double* xnorm) -> int {
    sp_plus_kernel<<<(P + 127) / 128, 128, 0, ctx->stream>>>(P, d_dim, at, d_sys[buf], 2, -1.0, d_tmp);
    DL_LAUNCH_CHECK(ctx, "sp_plus_kernel");
    double o[3];
    DL_TRY(norms(at, d_tmp, o));
    *gmax = o[0];
    *xnorm = o[1];
    return DL_OK;
  };
  int cur = 0;
  dl_solve_summary sum{};
  if (n_local == 0) {  // nothing to optimise: Ceres reports the fixed cost and converges without iterating
    DL_TRY(evaluate(d_x, cur));
    double c = 0;
    DL_TRY(cost_of(cur, &c));
    sum.initial_cost = sum.final_cost = c + fixed_cost;
    sum.termination = 0;
    sum.num_evaluations = 1;
  } else {
    LmCallbacks cb;
    cb.initial = [&](double* cost, double* gmax, double* x_norm) -> int {
      DL_TRY(evaluate(d_x, cur));
      DL_TRY(cost_of(cur, cost));
      return gradient_norms(d_x, cur, gmax, x_norm);
    };
    cb.save_best = [&]() -> int {
      DL_CUDA(ctx, cudaMemcpyAsync(d_best, d_x, (size_t)P * 56, cudaMemcpyDeviceToDevice, ctx->stream));
      return DL_OK;
    };
    cb.step = [&](double radius, bool reuse_diagonal, bool first_step, bool* valid, double* model_cost_change) -> int {
      const double sc[3] = {radius, reuse_diagonal ? 1. : 0., first_step ? 1. : 0.};
      DL_CUDA(ctx, cudaMemcpyAsync(sb.scalars, sc, 24, cudaMemcpyHostToDevice, ctx->stream));
      sb.sys = d_sys[cur];
      sp_scale_kernel<<<(6 * P + 127) / 128, 128, 0, ctx->stream>>>(pl, d_dim, sb);
      DL_LAUNCH_CHECK(ctx, "sp_scale_kernel");
      if (N > 0) {
        sp_node_factor_kernel<<<(N + 63) / 64, 64, 0, ctx->stream>>>(pl, S, d_dim, sb);
        DL_LAUNCH_CHECK(ctx, "sp_node_factor_kernel");
      }
      if (K > 0) {
        sp_pair_kernel<<<(K + 63) / 64, 64, 0, ctx->stream>>>(pl, S, d_dim, d_pairs, sb);
        DL_LAUNCH_CHECK(ctx, "sp_pair_kernel");
      }
      if (R > 0) {
        DL_CUDA(ctx, cudaMemsetAsync(sb.A, 0, (size_t)n_red * n_red * 8, ctx->stream));
        sp_reduce_kernel<<<R, 64, 0, ctx->stream>>>(pl, S, d_dim, d_roff, n_red, d_blocks, d_blk_ptr, d_terms, d_pairs, d_sub_ptr, sb);
        DL_LAUNCH_CHECK(ctx, "sp_reduce_kernel");
        sp_reduced_solve_kernel<<<1, 1024, 0, ctx->stream>>>(n_red, sb);
        DL_LAUNCH_CHECK(ctx, "sp_reduced_solve_kernel");
      }
      sp_backsub_kernel<<<(P + 127) / 128, 128, 0, ctx->stream>>>(pl, S, d_dim, d_roff, d_pairs, d_node_ptr, d_node_pairs, sb);
      DL_LAUNCH_CHECK(ctx, "sp_backsub_kernel");
      sp_finish_kernel<<<1, 256, 0, ctx->stream>>>(P, sb);
      DL_LAUNCH_CHECK(ctx, "sp_finish_kernel");
      double outv[2];
      DL_CUDA(ctx, cudaMemcpyAsync(outv, sb.scalars + 3, 16, cudaMemcpyDeviceToHost, ctx->stream));
      DL_CUDA(ctx, ctx->wait_stream());
      *valid = outv[0] != 0.;
      *model_cost_change = outv[1];
      return DL_OK;
    };
    cb.candidate = [&](double* cand_cost, double* step_norm) -> int {
      sp_plus_kernel<<<(P + 127) / 128, 128, 0, ctx->stream>>>(P, d_dim, d_x, sb.delta, 0, 1.0, d_cand);
      DL_LAUNCH_CHECK(ctx, "sp_plus_kernel");
      DL_TRY(evaluate(d_cand, cur ^ 1));
      DL_TRY(cost_of(cur ^ 1, cand_cost));
      double o[3];
      DL_TRY(norms(d_x, d_cand, o));
      *step_norm = o[2];
      return DL_OK;
    };
    cb.accept = [&](double* gmax, double* x_norm) -> int {
      std::swap(d_x, d_cand);
      cur ^= 1;
      return gradient_norms(d_x, cur, gmax, x_norm);
    };
    DL_TRY(run_trust_region(cb, options->max_num_iterations, &sum));
    // Ceres 1.13 reports x_cost + fixed_cost; its tolerances above saw x_cost only
    sum.initial_cost += fixed_cost;
    sum.final_cost += fixed_cost;
  }
  cudaEventDestroy(ev0);
  cudaEventDestroy(ev1);
  DL_CUDA(ctx, cudaMemcpyAsync(poses, d_best, (size_t)P * 56, cudaMemcpyDeviceToHost, ctx->stream));
  DL_CUDA(ctx, ctx->wait_stream());
  if (summary) *summary = sum;
  if (info) {
    info->num_local_parameters = n_local;
    info->all_reduce_count = reductions;
    info->all_reduce_bytes = (int64_t)sys * 8;
    info->all_reduce_ms = reduce_ms;
    info->all_reduce_min_ms = reductions ? reduce_min_ms : 0.f;
    info->num_reduced_parameters = n_red;
    info->num_pairs = K;
    info->setup_exchange_bytes = setup_bytes;
  }
  return DL_OK;
}

// The factors alone: each constraint's residual and local Jacobian at the given poses, from sp_evaluate_kernel as the solve
// launches it. Every pose of a constraint is referenced, so its dim is 0 if frozen, 2 for the first submap, else 3 + tdof.
extern "C" int dl_pose_graph_evaluate(dl_context* ctx, const dl_pose_graph_options* options, int32_t num_submaps, int32_t num_nodes,
                                      const double* poses, const uint8_t* frozen, const dl_spa_constraint* constraints,
                                      int32_t num_constraints, double* residuals, double* jacobians) {
  if (!ctx || !options || num_submaps < 1 || num_nodes < 0 || !poses || num_constraints < 0 ||
      (num_constraints > 0 && (!constraints || !residuals || !jacobians)))
    return DL_ERR_ARG;
  const int S = num_submaps, N = num_nodes, P = S + N, M = num_constraints, tdof = options->fix_z ? 2 : 3;
  for (int k = 0; k < M; ++k)
    if (constraints[k].submap < 0 || constraints[k].submap >= S || constraints[k].node < 0 || constraints[k].node >= N)
      return ctx->fail(DL_ERR_ARG, "constraint refers to a submap / node outside the graph");
  if (M == 0) return DL_OK;
  std::vector<int> dim(P);
  for (int p = 0; p < P; ++p) dim[p] = (frozen && frozen[p]) ? 0 : p == 0 ? 2 : 3 + tdof;
  cudaError_t e0 = cudaSetDevice(ctx->device);
  if (e0 != cudaSuccess) return ctx->cuda_fail(e0, "cudaSetDevice");
  double *d_x, *d_J, *d_e, *d_c2;
  dl_spa_constraint* d_c;
  int* d_dim;
  DL_TRY(carve_scratch(ctx, [&](Arena& a) {
    d_x = a.take<double>((size_t)7 * P);
    d_J = a.take<double>((size_t)M * 72);
    d_e = a.take<double>((size_t)M * 6);
    d_c2 = a.take<double>((size_t)M);
    d_c = a.take<dl_spa_constraint>((size_t)M);
    d_dim = a.take<int>((size_t)P);
  }));
  DL_TRY(h2d(ctx, d_x, poses, (size_t)7 * P));
  DL_TRY(h2d(ctx, d_c, constraints, (size_t)M));
  DL_TRY(h2d(ctx, d_dim, dim.data(), (size_t)P));
  const SparseGraph gr{S, N, tdof, d_dim, nullptr, 0};
  sp_evaluate_kernel<<<(M + 63) / 64, 64, 0, ctx->stream>>>(gr, d_x, d_c, M, 1, d_J, d_e, d_c2);
  DL_LAUNCH_CHECK(ctx, "sp_evaluate_kernel");
  DL_TRY(d2h(ctx, residuals, d_e, (size_t)M * 6));
  DL_TRY(d2h(ctx, jacobians, d_J, (size_t)M * 72));
  return sync(ctx);
}
