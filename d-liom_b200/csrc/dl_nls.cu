// Point-to-probability-grid nonlinear least squares with the whole Levenberg-Marquardt loop on the device.
//
// Replaces CeresScanMatcher3D::Match -> ceres::Solve (SM/ceres_scan_matcher_3d.cc:71-123) for the problem the
// reference assembles: one OccupiedSpaceCostFunction3D block per (cloud, grid) pair
// (SM/occupied_space_cost_function_3d.h:46-80, interpolation SM/interpolated_grid.h:50-146), a
// TranslationDeltaCostFunctor3D and a RotationDeltaCostFunctor3D (SM/*_delta_cost_functor_3d.h), pose parameter
// blocks t[3], q[4] with ceres::QuaternionParameterization or YawOnlyQuaternionPlus
// (C/mapping/internal/3d/rotation_parameterization.h:27-39), LM trust region + DENSE_QR, Ceres 1.13 defaults.
//
// Design: ONE CTA per registration problem, many problems per launch (the reference solves them one at a time on
// one thread, or 8 at a time in the loop-closure thread pool). Each evaluation is a single fused pass
//   transform (fp64) -> float cell selection -> 8 voxel reads -> smoothstep interpolation -> analytic gradient ->
//   chain rule to the 6 local parameters -> J^T J (21) / J^T r (6) / cost (1) accumulation
// reduced with a butterfly reduce-scatter over the warp (31 shuffles for all 28 quantities) and then over the warps in
// index order (fixed order: bit-reproducible run to run). The N x 6 Jacobian the reference
// materialises (N x 7 doubles, then QR) never exists: the normal equations carry everything the LM loop needs —
// Jacobi scaling, the LM diagonal, the step (6x6 Cholesky of S J^T J S + D^2, algebraically the stacked QR
// solution), the model cost change and the projected gradient. Candidate points are evaluated speculatively
// WITH their normal equations, so an accepted step costs one pass instead of Ceres's two (cost-only, then
// re-evaluation with Jacobians). All accumulation is fp64; cell selection mirrors the reference's float/double
// mix exactly, so the piecewise-polynomial pieces are the same ones the CPU path picks.
//
// Algorithmic bytes: 12 B point + 8 corners * 2 B = 28 B per point per evaluation (SURVEY 8d).
#include <cstring>
#include <type_traits>
#include <vector>

#include <cooperative_groups.h>

#include "dl_internal.cuh"

namespace dl {
namespace {

// Threads per problem. The kernels are written for any multiple of 32 up to kBlock: the evaluation pass strides by the
// number of point threads, WARP 0 drives the LM state machine between passes (lane i owns row i of the 6x6 / 15x15 systems,
// all matrices in shared memory — round 1 ran it on thread 0 with the matrices in local memory: 7.5 KB of stack for the
// fused kernel, ~2/3 of the solve's time), and with the IMU term the last warp evaluates that term while the others
// walk the points. A scan-matching problem has only a few hundred points after the adaptive filters.
constexpr int kBlock = 256;
constexpr int kWarps = kBlock / 32;
constexpr int kRed = 28;  // cost, g[6], H upper triangle [21]

struct Lm {  // Ceres 1.13 Solver::Options defaults (trust_region_minimizer.cc, levenberg_marquardt_strategy.cc)
  static constexpr double initial_radius = 1e4, max_radius = 1e16, min_radius = 1e-32;
  static constexpr double min_relative_decrease = 1e-3, min_lm_diagonal = 1e-6, max_lm_diagonal = 1e32;
  static constexpr double function_tolerance = 1e-6, gradient_tolerance = 1e-10, parameter_tolerance = 1e-8;
  static constexpr int max_consecutive_invalid = 5, max_consecutive_nonmonotonic = 5;
};

__device__ __forceinline__ int tri(int a, int b) {  // a <= b, row-major upper triangle of 6x6
  return a * 6 - a * (a - 1) / 2 + (b - a);
}

// brick index of the brick containing the (shifted, in-bounds) cell, or -1
__device__ __forceinline__ int find_brick(const GridView& g, unsigned sx, unsigned sy, unsigned sz) {
  const int node = __ldg(g.top + ((((sz >> 6) << g.bits) + (sy >> 6)) << g.bits) + (sx >> 6));
  if (node < 0) return -1;
  return __ldg(g.nodes + (size_t)node * 512 + ((((sz >> 3) & 7) << 6) | (((sy >> 3) & 7) << 3) | ((sx >> 3) & 7)));
}

// InterpolatedGrid::GetProbability at (x, y, z) plus its spatial gradient.
__device__ __forceinline__ void interpolate(const GridView& g, double x, double y, double z, double* value,
                                            double* gx, double* gy, double* gz) {
  const float res = g.resolution;
  // CenterOfLowerVoxel (interpolated_grid.h:120-139): float cell of the narrowed point, float centre compared
  // with the double coordinate.
  const Int3 ci = cell_index(Vec3f{(float)x, (float)y, (float)z}, res);
  float cx = (float)ci.x * res, cy = (float)ci.y * res, cz = (float)ci.z * res;
  if ((double)cx > x) cx -= res;
  if ((double)cy > y) cy -= res;
  if ((double)cz > z) cz -= res;
  const double x1 = cx, y1 = cy, z1 = cz;
  const double x2 = (double)(cx + res), y2 = (double)(cy + res), z2 = (double)(cz + res);
  const Int3 i1 = cell_index(Vec3f{cx, cy, cz}, res);

  // 8 corners: one tree walk when the 2x2x2 block sits inside one brick (probability (7/8)^3), else 8 walks.
  float q[8];  // index = dx*4 + dy*2 + dz
  const int gs = 64 << g.bits, half = gs >> 1;
  const unsigned sx = (unsigned)(i1.x + half), sy = (unsigned)(i1.y + half), sz = (unsigned)(i1.z + half);
  if (sx < (unsigned)gs - 1 && sy < (unsigned)gs - 1 && sz < (unsigned)gs - 1 && (sx & 7) != 7 && (sy & 7) != 7 &&
      (sz & 7) != 7) {
    const int brick = find_brick(g, sx, sy, sz);
    if (brick < 0) {
#pragma unroll
      for (int k = 0; k < 8; ++k) q[k] = 0.1f;
    } else {
      const uint16_t* b = g.bricks + (size_t)brick * 512 + (((sz & 7) << 6) | ((sy & 7) << 3) | (sx & 7));
#pragma unroll
      for (int k = 0; k < 8; ++k) q[k] = value_to_probability(__ldg(b + ((k & 1) << 6) + (((k >> 1) & 1) << 3) + (k >> 2)));
    }
  } else {
#pragma unroll
    for (int k = 0; k < 8; ++k) q[k] = value_to_probability(grid_value(g, i1.x + (k >> 2), i1.y + ((k >> 1) & 1), i1.z + (k & 1)));
  }
  const double q111 = q[0], q112 = q[1], q121 = q[2], q122 = q[3], q211 = q[4], q212 = q[5], q221 = q[6], q222 = q[7];

  const double ix = 1.0 / (x2 - x1), iy = 1.0 / (y2 - y1), iz = 1.0 / (z2 - z1);
  const double nx = (x - x1) / (x2 - x1), ny = (y - y1) / (y2 - y1), nz = (z - z1) / (z2 - z1);
  const double nxx = nx * nx, nxxx = nx * nxx, nyy = ny * ny, nyyy = ny * nyy, nzz = nz * nz, nzzz = nz * nzz;
  // value: the reference's expression order (interpolated_grid.h:84-102)
  const double q11 = (q111 - q112) * nzzz * 2. + (q112 - q111) * nzz * 3. + q111;
  const double q12 = (q121 - q122) * nzzz * 2. + (q122 - q121) * nzz * 3. + q121;
  const double q21 = (q211 - q212) * nzzz * 2. + (q212 - q211) * nzz * 3. + q211;
  const double q22 = (q221 - q222) * nzzz * 2. + (q222 - q221) * nzz * 3. + q221;
  const double q1 = (q11 - q12) * nyyy * 2. + (q12 - q11) * nyy * 3. + q11;
  const double q2 = (q21 - q22) * nyyy * 2. + (q22 - q21) * nyy * 3. + q21;
  *value = (q1 - q2) * nxxx * 2. + (q2 - q1) * nxx * 3. + q1;
  // gradient of the same polynomial: S(t) = 3t^2 - 2t^3, S'(t) = 6t(1 - t)
  const double sx_ = 3. * nxx - 2. * nxxx, sy_ = 3. * nyy - 2. * nyyy;
  const double dsx = 6. * nx * (1. - nx), dsy = 6. * ny * (1. - ny), dsz = 6. * nz * (1. - nz);
  *gx = (q2 - q1) * dsx * ix;
  *gy = ((q12 - q11) * (1. - sx_) + (q22 - q21) * sx_) * dsy * iy;
  const double dz1 = (q112 - q111) * (1. - sy_) + (q122 - q121) * sy_;
  const double dz2 = (q212 - q211) * (1. - sy_) + (q222 - q221) * sy_;
  *gz = (dz1 * (1. - sx_) + dz2 * sx_) * dsz * iz;
}

// d(q_delta (x) x)/d(delta) at delta = 0: 4 x 3 for ceres::QuaternionParameterization, 4 x 1 for yaw-only.
__device__ __forceinline__ void plus_jacobian(const double* x, bool only_yaw, double P[4][3]) {
  const double q0 = x[3], q1 = x[4], q2 = x[5], q3 = x[6];
  if (!only_yaw) {
    P[0][0] = -q1; P[0][1] = -q2; P[0][2] = -q3;
    P[1][0] = q0;  P[1][1] = q3;  P[1][2] = -q2;
    P[2][0] = -q3; P[2][1] = q0;  P[2][2] = q1;
    P[3][0] = q2;  P[3][1] = -q1; P[3][2] = q0;
  } else {
    P[0][0] = -q3; P[1][0] = -q2; P[2][0] = q1; P[3][0] = q0;
    for (int i = 0; i < 4; ++i) P[i][1] = P[i][2] = 0.0;
  }
}

__device__ __forceinline__ void plus(const double* x, const double* delta, bool only_yaw, double* out) {
  out[0] = x[0] + delta[0]; out[1] = x[1] + delta[1]; out[2] = x[2] + delta[2];
  const Quatd q{x[3], x[4], x[5], x[6]};
  Quatd r = q;
  if (!only_yaw) {
    const double n = sqrt(delta[3] * delta[3] + delta[4] * delta[4] + delta[5] * delta[5]);
    if (n > 0.0) {
      const double sbd = sin(n) / n;
      r = qmul(Quatd{cos(n), sbd * delta[3], sbd * delta[4], sbd * delta[5]}, q);
    }
  } else {
    double d = delta[3];
    d = d > 0.5 ? 0.5 : (d < -0.5 ? -0.5 : d);
    r = qmul(Quatd{sqrt(1. - d * d), 0., 0., d}, q);
  }
  out[3] = r.w; out[4] = r.x; out[5] = r.y; out[6] = r.z;
}

struct Shared {
  double red[kWarps][32];  // per-warp partial sums of the 28 reduced quantities (lane l holds quantity l)
  double acc[32];          // block total of the last evaluation: cost*2, J^T r (6), J^T J upper triangle (21)
  double x[7];             // evaluation point broadcast
  int n[DL_MAX_PAIRS];
  double scaling[DL_MAX_PAIRS];
  int stop;
};

// Butterfly reduce-scatter of 32 per-lane values over the warp: 31 double shuffles instead of the 5 x 28 of a plain
// xor tree per quantity. On return lane l holds the warp total of v[l] in v[0]. Fixed order -> run-to-run reproducible.
__device__ __forceinline__ double warp_reduce_scatter32(double (&v)[32], int lane) {
#pragma unroll
  for (int h = 16; h >= 1; h >>= 1) {
    const bool up = (lane & h) != 0;
#pragma unroll
    for (int i = 0; i < h; ++i) {
      const double send = up ? v[i] : v[i + h];
      const double keep = up ? v[i + h] : v[i];
      v[i] = keep + __shfl_xor_sync(0xffffffffu, send, h);
    }
  }
  return v[0];
}

// Point pass of one evaluation at sh.x: every participating thread accumulates cost*2, J^T r and J^T J (local
// parameterisation) over its points; each warp leaves its partial sums in sh.red[warp][0..27].
// Threads [0, point_threads) take part (whole warps); the caller synchronises the block afterwards.
// A problem may be spread over the CTAs of a thread-block cluster (full-cloud solves): CTA `rank` of `ranks` takes points
// rank * point_threads + threadIdx.x, + ranks * point_threads, ... and leaves its partial sums in ITS sh.red.
__device__ __forceinline__ void evaluate_points(const NlsOptions& opt, const NlsProblem& prob, Shared& sh, int point_threads,
                                                int rank = 0, int ranks = 1) {
  if ((int)threadIdx.x >= point_threads) return;
  double x[7];
#pragma unroll
  for (int i = 0; i < 7; ++i) x[i] = sh.x[i];
  double P[4][3];
  plus_jacobian(x, opt.only_yaw != 0, P);
  const Quatd q{x[3], x[4], x[5], x[6]};
  const Vec3d a{x[4], x[5], x[6]};
  double acc[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) acc[i] = 0.0;

  for (int k = 0; k < opt.num_pairs; ++k) {
    const int n = sh.n[k];
    const double s = sh.scaling[k];
    const float* __restrict__ cloud = prob.cloud[k];
    const GridView g = prob.grid[k];
    for (int i = rank * point_threads + threadIdx.x; i < n; i += ranks * point_threads) {
      const Vec3d v{(double)cloud[3 * i], (double)cloud[3 * i + 1], (double)cloud[3 * i + 2]};
      const Vec3d w = add(rotate(q, v), Vec3d{x[0], x[1], x[2]});
      double m, gx, gy, gz;
      interpolate(g, w.x, w.y, w.z, &m, &gx, &gy, &gz);
      const double r = s * (1. - m);
      // ambient Jacobian row: -s * grad(M) . [ I | d world / d(qw, qx, qy, qz) ]
      const double jx = -s * gx, jy = -s * gy, jz = -s * gz;
      const Vec3d dw = mul(2.0, cross3(a, v));                       // d/d qw
      const double av = dot3(a, v);
      // d/d a_j = 2 qw (e_j x v) + 2 (e_j (a.v) + a v_j - 2 v a_j), e_x x v = (0, -v_z, v_y) etc.
      const Vec3d dxv{2. * (av + a.x * v.x - 2. * v.x * a.x), 2. * (-q.w * v.z + a.y * v.x - 2. * v.y * a.x),
                      2. * (q.w * v.y + a.z * v.x - 2. * v.z * a.x)};
      const Vec3d dyv{2. * (q.w * v.z + a.x * v.y - 2. * v.x * a.y), 2. * (av + a.y * v.y - 2. * v.y * a.y),
                      2. * (-q.w * v.x + a.z * v.y - 2. * v.z * a.y)};
      const Vec3d dzv{2. * (-q.w * v.y + a.x * v.z - 2. * v.x * a.z), 2. * (q.w * v.x + a.y * v.z - 2. * v.y * a.z),
                      2. * (av + a.z * v.z - 2. * v.z * a.z)};
      const double gq0 = jx * dw.x + jy * dw.y + jz * dw.z;
      const double gq1 = jx * dxv.x + jy * dxv.y + jz * dxv.z;
      const double gq2 = jx * dyv.x + jy * dyv.y + jz * dyv.z;
      const double gq3 = jx * dzv.x + jy * dzv.y + jz * dzv.z;
      double J[6];
      J[0] = jx; J[1] = jy; J[2] = jz;
#pragma unroll
      for (int j = 0; j < 3; ++j) J[3 + j] = gq0 * P[0][j] + gq1 * P[1][j] + gq2 * P[2][j] + gq3 * P[3][j];
      acc[0] += r * r;
#pragma unroll
      for (int c = 0; c < 6; ++c) acc[1 + c] += J[c] * r;
      int t = 7;
#pragma unroll
      for (int c = 0; c < 6; ++c)
#pragma unroll
        for (int d = c; d < 6; ++d) acc[t++] += J[c] * J[d];
    }
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  sh.red[warp][lane] = warp_reduce_scatter32(acc, lane);
}

// Warp 0, after the block barrier that follows evaluate_points: warps are summed in index order, then the two
// 3-residual blocks (translation_delta_cost_functor_3d.h:38-44, rotation_delta_cost_functor_3d.h:42-53) are added.
// Leaves the totals in sh.acc (visible to warp 0 after the trailing __syncwarp).
// With a cluster, CTA 0 reads the other CTAs' partial sums through distributed shared memory, CTAs in rank order.
__device__ __forceinline__ void finish_points(const NlsOptions& opt, Shared& sh, int point_warps, const double* target_q_inv,
                                              const double* target_t, int lane, int ranks = 1) {
  double v = 0.0;
  for (int w = 0; w < point_warps; ++w) v += sh.red[w][lane];
  if (ranks > 1) {
    cooperative_groups::cluster_group cluster = cooperative_groups::this_cluster();
    for (int r = 1; r < ranks; ++r) {
      const double* remote = cluster.map_shared_rank(&sh.red[0][0], r);
      for (int w = 0; w < point_warps; ++w) v += remote[w * 32 + lane];
    }
  }
  const double* x = sh.x;
  if (opt.trans_weight > 0.) {
    const double s = opt.trans_weight;
    if (lane == 0) {
      double c2 = 0;
      for (int c = 0; c < 3; ++c) {
        const double r = s * (x[c] - target_t[c]);
        c2 += r * r;
      }
      v += c2;
    } else if (lane >= 1 && lane <= 3) {
      v += s * (s * (x[lane - 1] - target_t[lane - 1]));
    } else if (lane == 7 + tri(0, 0) || lane == 7 + tri(1, 1) || lane == 7 + tri(2, 2)) {
      v += s * s;
    }
  }
  if (opt.rot_weight > 0.) {
    const double s = opt.rot_weight;
    double P[4][3];
    plus_jacobian(x, opt.only_yaw != 0, P);
    const double zw = target_q_inv[0], zx = target_q_inv[1], zy = target_q_inv[2], zz = target_q_inv[3];
    const double* w = x + 3;
    const double d[3] = {zw * w[1] + zx * w[0] + zy * w[3] - zz * w[2], zw * w[2] - zx * w[3] + zy * w[0] + zz * w[1],
                         zw * w[3] + zx * w[2] - zy * w[1] + zz * w[0]};
    const double dd[3][4] = {{zx, zw, -zz, zy}, {zy, zz, zw, -zx}, {zz, -zy, zx, zw}};
    double Jr[3][3];  // residual c, rotation parameter j
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
      for (int j = 0; j < 3; ++j)
        Jr[c][j] = s * (dd[c][0] * P[0][j] + dd[c][1] * P[1][j] + dd[c][2] * P[2][j] + dd[c][3] * P[3][j]);
    if (lane == 0) {
      for (int c = 0; c < 3; ++c) v += (s * d[c]) * (s * d[c]);
    } else if (lane >= 4 && lane <= 6) {
      const int e = lane - 4;
      for (int c = 0; c < 3; ++c) v += Jr[c][e] * (s * d[c]);
    } else {
#pragma unroll
      for (int e = 0; e < 3; ++e)
#pragma unroll
        for (int f = e; f < 3; ++f)
          if (lane == 7 + tri(3 + e, 3 + f))
            for (int c = 0; c < 3; ++c) v += Jr[c][e] * Jr[c][f];
    }
  }
  sh.acc[lane] = v;
  __syncwarp();
}

// ---------------------------------------------------------------------------------------------------------------
// Everything below is templated on N, the size of the local parameter vector held by the LM state:
//   N = 6   the reference's scan matcher (pose only; 4 of the 6 used with only_optimize_yaw), ambient size 7
//   N = 15  the fused solve: pose + velocity + accelerometer / gyroscope biases of state j (ambient size 16), with
//           the IMU pre-integration residual of integration_base.h:267-301 added to the normal equations.
template <int N>
struct Dims {
  static constexpr int ambient = N == 15 ? 16 : 7;
};

// The Jacobian of the residual w.r.t. the local parameters of state j is block diagonal: R_i^T for p and v, a 3x3
// block that depends on q_j for theta, identity for the biases. Only the three 3x3 blocks are stored.
struct ImuShared {
  double W[225];
  double r[15], Wr[15];
  double B[3][3][3];  // B[blk][row][col]: J[3 blk + row][3 blk + col], blk = 0 (p), 1 (theta), 2 (v)
  double WJ[15][15];
  double H[15][15], g[15], cost2;
};

// One warp: residual, block Jacobian, then H = J^T W J, g = J^T W r, cost2 = r^T W r. The sums skip the structural
// zeros of J, everything else is the dense formula.
__device__ void imu_normal_equations(const ImuTerm& m, const double* x /*16*/, ImuShared& is, int lane) {
  if (lane == 0) {
    const double T = m.sum_dt;
    const Quatd qi_inv{m.qi[0], -m.qi[1], -m.qi[2], -m.qi[3]};
    const Vec3d G{m.G[0], m.G[1], m.G[2]};
    const Vec3d pj{x[0], x[1], x[2]}, vj{x[7], x[8], x[9]};
    const Vec3d pi{m.pi[0], m.pi[1], m.pi[2]}, vi{m.vi[0], m.vi[1], m.vi[2]};
    const Vec3d rp = sub(rotate(qi_inv, sub(sub(add(mul(0.5 * T * T, G), pj), pi), mul(T, vi))), Vec3d{m.dp[0], m.dp[1], m.dp[2]});
    const Vec3d rv = sub(rotate(qi_inv, sub(add(mul(T, G), vj), vi)), Vec3d{m.dv[0], m.dv[1], m.dv[2]});
    is.r[0] = rp.x; is.r[1] = rp.y; is.r[2] = rp.z;
    is.r[6] = rv.x; is.r[7] = rv.y; is.r[8] = rv.z;
  } else if (lane == 1) {
    const Quatd qi_inv{m.qi[0], -m.qi[1], -m.qi[2], -m.qi[3]};
    const Quatd qj{x[3], x[4], x[5], x[6]};
    const Quatd A = qmul(Quatd{m.dq[0], -m.dq[1], -m.dq[2], -m.dq[3]}, qi_inv);
    const Quatd e = qmul(A, qj);
    is.r[3] = 2 * e.x; is.r[4] = 2 * e.y; is.r[5] = 2 * e.z;
  } else if (lane >= 2 && lane < 5) {
    const int b = lane - 2;  // column b of R_i^T (blocks 0 and 2) and of the theta block
    const Quatd qi_inv{m.qi[0], -m.qi[1], -m.qi[2], -m.qi[3]};
    const Quatd qj{x[3], x[4], x[5], x[6]};
    const Vec3d col = rotate(qi_inv, Vec3d{b == 0 ? 1.0 : 0.0, b == 1 ? 1.0 : 0.0, b == 2 ? 1.0 : 0.0});
    is.B[0][0][b] = col.x; is.B[0][1][b] = col.y; is.B[0][2][b] = col.z;
    is.B[2][0][b] = col.x; is.B[2][1][b] = col.y; is.B[2][2][b] = col.z;
    const Quatd A = qmul(Quatd{m.dq[0], -m.dq[1], -m.dq[2], -m.dq[3]}, qi_inv);
    const Quatd c = qmul(qmul(A, Quatd{0.0, b == 0 ? 1.0 : 0.0, b == 1 ? 1.0 : 0.0, b == 2 ? 1.0 : 0.0}), qj);
    is.B[1][0][b] = 2 * c.x; is.B[1][1][b] = 2 * c.y; is.B[1][2][b] = 2 * c.z;
  } else if (lane >= 5 && lane < 11) {
    const int a = lane - 5;
    is.r[9 + a] = x[10 + a] - (a < 3 ? m.bai[a] : m.bgi[a - 3]);
  }
  __syncwarp();
  // WJ[c][b] = sum_d W[c][d] J[d][b]
  for (int e = lane; e < 225; e += 32) {
    const int c = e / 15, b = e % 15;
    double s;
    if (b < 9) {
      const int blk = b / 3, col = b % 3;
      s = 0;
#pragma unroll
      for (int d = 0; d < 3; ++d) s += is.W[c * 15 + 3 * blk + d] * is.B[blk][d][col];
    } else {
      s = is.W[c * 15 + b];
    }
    is.WJ[c][b] = s;
  }
  if (lane < 15) {
    double s = 0;
    for (int d = 0; d < 15; ++d) s += is.W[lane * 15 + d] * is.r[d];
    is.Wr[lane] = s;
  }
  __syncwarp();
  // H[a][b] = sum_c J[c][a] WJ[c][b]
  for (int e = lane; e < 225; e += 32) {
    const int a = e / 15, b = e % 15;
    double s;
    if (a < 9) {
      const int blk = a / 3, col = a % 3;
      s = 0;
#pragma unroll
      for (int c = 0; c < 3; ++c) s += is.B[blk][c][col] * is.WJ[3 * blk + c][b];
    } else {
      s = is.WJ[a][b];
    }
    is.H[a][b] = s;
  }
  if (lane < 15) {
    const int a = lane;
    double s;
    if (a < 9) {
      const int blk = a / 3, col = a % 3;
      s = 0;
#pragma unroll
      for (int c = 0; c < 3; ++c) s += is.B[blk][c][col] * is.Wr[3 * blk + c];
    } else {
      s = is.Wr[a];
    }
    is.g[a] = s;
  }
  if (lane == 31) {
    double s = 0;
    for (int c = 0; c < 15; ++c) s += is.r[c] * is.Wr[c];
    is.cost2 = s;
  }
  __syncwarp();
}

__device__ __forceinline__ void setup_problem(const NlsOptions& opt, const NlsProblem& prob, Shared& sh, double* x0,
                                              double* target_t, double* target_q_inv) {
  if (threadIdx.x == 0) {
    for (int k = 0; k < opt.num_pairs; ++k) {
      const int n = prob.count_dev[k] ? *prob.count_dev[k] : prob.count[k];
      sh.n[k] = n;
      sh.scaling[k] = opt.occ_weight[k] / sqrt((double)n);  // ceres_scan_matcher_3d.cc:98-99
    }
    const double* init = prob.initial_dev ? prob.initial_dev : prob.initial;
    for (int i = 0; i < 7; ++i) sh.x[i] = init[i];
  }
  __syncthreads();
  for (int i = 0; i < 7; ++i) x0[i] = sh.x[i];
  if (prob.target_dev) {
    for (int i = 0; i < 3; ++i) target_t[i] = prob.target_dev[i];
  } else if (prob.initial_dev) {
    for (int i = 0; i < 3; ++i) target_t[i] = x0[i];
  } else {
    for (int i = 0; i < 3; ++i) target_t[i] = prob.target_t[i];
  }
  target_q_inv[0] = x0[3]; target_q_inv[1] = -x0[4]; target_q_inv[2] = -x0[5]; target_q_inv[3] = -x0[6];
}

// Trust-region state of one problem (names follow Ceres 1.13 TrustRegionMinimizer / LevenbergMarquardtStrategy /
// TrustRegionStepEvaluator members). Lives in shared memory and is driven by WARP 0: lane i owns row i of every
// N x N matrix (Jacobi scaling, LM diagonal, Cholesky, triangular solves, model cost), lane 0 the scalar bookkeeping.
// The accepted point's and the candidate's normal equations sit in two buffers that swap on a successful step.
template <int N>
struct LmStateT {
  static constexpr int NA = Dims<N>::ambient;
  double H[2][N][N], g[2][N], cost[2];
  double A[N][N];  // scaled + damped system, overwritten by its Cholesky factor (lower triangle; diagonal = 1 / L[j][j])
  double gs[N], step[N], scale[N], diag[N];
  double x[NA], cand[NA], best_x[NA], target_t[3], target_q_inv[4];
  double x_norm, minimum_cost, radius, decrease_factor, gradient_max_norm, initial_cost, final_cost, last_cost;
  double model_cost_change;
  double ev_minimum, ev_current, ev_reference, ev_candidate, ev_acc_ref, ev_acc_cand;
  int ev_num_nonmono, max_nonmono;
  int cur;  // which buffer holds the accepted point
  int reuse_diagonal, last_successful, num_invalid, iteration, recorded, successful, unsuccessful, termination, evals;
  int nl, only_yaw, max_iter;
  int flag;  // lane 0 -> warp broadcast of the state machine's decisions
};

template <int NA>
__device__ __forceinline__ double norm_ambient(const double* v) {
  double s = 0;
  for (int i = 0; i < NA; ++i) s += v[i] * v[i];
  return sqrt(s);
}
// x (+) delta for the N-dim local vector: pose like the scan matcher, the remaining 9 parameters additively.
template <int N>
__device__ __forceinline__ void plus_n(const double* x, const double* delta, bool only_yaw, double* out) {
  plus(x, delta, only_yaw, out);
  if (N == 15)
    for (int i = 0; i < 9; ++i) out[7 + i] = x[7 + i] + delta[6 + i];
}
// max-norm of x - Plus(x, -g): the projected gradient Ceres tests against gradient_tolerance
template <int N>
__device__ double projected_gradient_max_norm(const double* at, const double* g, bool only_yaw) {
  constexpr int NA = Dims<N>::ambient;
  double ng[N], px[NA];
  for (int j = 0; j < N; ++j) ng[j] = -g[j];
  plus_n<N>(at, ng, only_yaw, px);
  double mx = 0;
  for (int i = 0; i < NA; ++i) mx = fmax(mx, fabs(at[i] - px[i]));
  return mx;
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
  return v;
}

// Assembles the normal equations of the last evaluation (sh.acc [+ the IMU term]) into buffer `buf`. Warp 0.
template <int N>
__device__ __forceinline__ void load_eval(LmStateT<N>& st, const Shared& sh, const ImuShared* is, int buf, int lane) {
  if (lane < N) {
    const int c = lane;
    double gv = c < 6 ? sh.acc[1 + c] : 0.0;
    if (N == 15 && is) gv += is->g[c];
    st.g[buf][c] = gv;
    for (int d = 0; d < N; ++d) {
      double h = (c < 6 && d < 6) ? sh.acc[7 + (c <= d ? tri(c, d) : tri(d, c))] : 0.0;
      if (N == 15 && is) h += is->H[c][d];
      st.H[buf][c][d] = h;
    }
  }
  if (lane == 0) {
    double c2 = sh.acc[0];
    if (N == 15 && is) c2 += is->cost2;
    st.cost[buf] = 0.5 * c2;
  }
  __syncwarp();
}

template <int N>
__device__ void lm_iteration_zero(LmStateT<N>& st, const Shared& sh, const ImuShared* is, int lane) {
  load_eval<N>(st, sh, is, 0, lane);
  if (lane < N) st.scale[lane] = lane < st.nl ? 1.0 / (1.0 + sqrt(st.H[0][lane][lane])) : 0.0;
  if (lane == 0) {
    st.cur = 0;
    st.evals = 1;
    const double c = st.cost[0];
    st.x_norm = norm_ambient<Dims<N>::ambient>(st.x);
    st.gradient_max_norm = projected_gradient_max_norm<N>(st.x, st.g[0], st.only_yaw);
    st.initial_cost = st.final_cost = st.last_cost = c;
    st.ev_minimum = st.ev_current = st.ev_reference = st.ev_candidate = c;
    st.ev_acc_ref = st.ev_acc_cand = 0;
    st.ev_num_nonmono = 0;
    st.minimum_cost = 1.7976931348623157e308;
    st.radius = Lm::initial_radius;
    st.decrease_factor = 2.0;
    st.reuse_diagonal = 0;
    st.last_successful = 1;
    st.num_invalid = st.iteration = st.recorded = st.successful = st.unsuccessful = 0;
    st.termination = 1;
  }
  __syncwarp();
}

// LevenbergMarquardtStrategy::ComputeStep on the Jacobi-scaled system, warp-cooperative. Returns (warp-uniform) whether the
// step is valid; on success st.step holds the scaled step and st.model_cost_change the predicted decrease.
template <int N>
__device__ __forceinline__ bool lm_compute_step(LmStateT<N>& st, int lane) {
  const int nl = st.nl, cur = st.cur;
  const bool row = lane < nl;
  const double radius = st.radius;
  if (row) {
    const double sc = st.scale[lane];
    st.gs[lane] = sc * st.g[cur][lane];
    for (int d = 0; d < nl; ++d) st.A[lane][d] = sc * st.H[cur][lane][d] * st.scale[d];
    if (!st.reuse_diagonal) st.diag[lane] = fmin(fmax(st.A[lane][lane], Lm::min_lm_diagonal), Lm::max_lm_diagonal);
    st.A[lane][lane] += st.diag[lane] / radius;
  }
  __syncwarp();
  // Cholesky, left-looking by columns; lane i owns row i. The factor overwrites the lower triangle of A.
  bool valid = true;
  for (int j = 0; j < nl; ++j) {
    double s = 0.0;
    if (row && lane >= j) {
      s = st.A[lane][j];
      for (int k = 0; k < j; ++k) s -= st.A[lane][k] * st.A[j][k];
    }
    const double pivot = __shfl_sync(0xffffffffu, s, j);
    if (!(pivot > 0.0)) { valid = false; break; }
    // one reciprocal square root per column instead of a square root and a division on the critical path
    // (fp64 rsqrt: 1 ulp); the diagonal slot keeps 1 / L[j][j], which is what the triangular solves need
    const double rinv = rsqrt(pivot);
    if (row && lane >= j) st.A[lane][j] = lane == j ? rinv : s * rinv;
    __syncwarp();
  }
  if (valid) {
    // L z = gs (forward), L^T y = z (backward); lane i carries the running right-hand side of row i
    const double inv_diag = row ? st.A[lane][lane] : 0.0;
    double rhs = row ? st.gs[lane] : 0.0;
    for (int k = 0; k < nl; ++k) {
      const double zk = __shfl_sync(0xffffffffu, rhs * inv_diag, k);
      if (lane == k) rhs = zk;
      else if (row && lane > k) rhs -= st.A[lane][k] * zk;
    }
    for (int k = nl - 1; k >= 0; --k) {
      const double yk = __shfl_sync(0xffffffffu, rhs * inv_diag, k);
      if (lane == k) rhs = yk;
      else if (row && lane < k) rhs -= st.A[k][lane] * yk;
    }
    const double y = rhs;
    valid = __all_sync(0xffffffffu, !row || isfinite(y));
    if (valid) {
      const double stp = row ? -y : 0.0;
      if (row) st.step[lane] = stp;
      __syncwarp();
      double lin = 0.0, quad = 0.0;
      if (row) {
        lin = stp * st.gs[lane];
        const double sc = st.scale[lane];
        double r = 0;
        for (int d = 0; d < nl; ++d) r += (sc * st.H[cur][lane][d] * st.scale[d]) * st.step[d];
        quad = stp * r;
      }
      lin = warp_sum(lin);
      quad = warp_sum(quad);
      const double mcc = -(lin + 0.5 * quad);
      if (lane == 0) st.model_cost_change = mcc;
      valid = mcc > 0.0;
    }
  }
  if (lane == 0) st.reuse_diagonal = 1;
  __syncwarp();
  return valid;
}

// FinalizeIterationAndCheckIfMinimizerCanContinue + ComputeTrustRegionStep (+ HandleInvalidStep retries).
// Returns 1 to stop; otherwise st.cand holds the candidate point. Warp 0, warp-uniform result.
template <int N>
__device__ int lm_prepare_step(LmStateT<N>& st, int lane) {
  constexpr int NA = Dims<N>::ambient;
  if (lane == 0) {
    int stop = 0;
    if (st.last_successful) {
      ++st.successful;
      if (st.cost[st.cur] < st.minimum_cost) {
        st.minimum_cost = st.cost[st.cur];
        for (int i = 0; i < NA; ++i) st.best_x[i] = st.x[i];
      }
    } else {
      ++st.unsuccessful;
    }
    ++st.recorded;
    st.final_cost = fmin(st.final_cost, st.last_cost);
    if (st.iteration >= st.max_iter) { st.termination = 1; stop = 1; }
    else if (st.last_successful && st.gradient_max_norm <= Lm::gradient_tolerance) { st.termination = 0; stop = 1; }
    else if (st.radius <= Lm::min_radius) { st.termination = 0; stop = 1; }
    st.flag = stop;
  }
  __syncwarp();
  if (st.flag) return 1;
  for (;;) {
    if (lane == 0) ++st.iteration;
    __syncwarp();
    if (lm_compute_step<N>(st, lane)) {
      if (lane == 0) {
        st.num_invalid = 0;
        double delta[N];
        for (int c = 0; c < N; ++c) delta[c] = c < st.nl ? st.step[c] * st.scale[c] : 0.0;
        plus_n<N>(st.x, delta, st.only_yaw, st.cand);
      }
      __syncwarp();
      return 0;
    }
    // HandleInvalidStep, then finalize that iteration and retry with the smaller radius
    if (lane == 0) {
      int stop = 0;
      if (++st.num_invalid >= Lm::max_consecutive_invalid) { st.termination = 2; stop = 1; }
      else {
        st.radius *= 0.5;
        st.last_successful = 0;
        st.last_cost = st.cost[st.cur];
        ++st.unsuccessful;
        ++st.recorded;
        if (st.iteration >= st.max_iter) { st.termination = 1; stop = 1; }
        else if (st.radius <= Lm::min_radius) { st.termination = 0; stop = 1; }
      }
      st.flag = stop;
    }
    __syncwarp();
    if (st.flag) return 1;
  }
}

// Tolerance tests, step acceptance and trust-region update for the evaluated candidate. Returns 1 to stop. Warp 0.
template <int N>
__device__ int lm_process_candidate(LmStateT<N>& st, const Shared& sh, const ImuShared* is, int lane) {
  constexpr int NA = Dims<N>::ambient;
  const int nb = st.cur ^ 1;
  load_eval<N>(st, sh, is, nb, lane);  // the candidate's normal equations were computed speculatively in the same pass
  if (lane == 0) {
    int stop = 0;
    ++st.evals;
    double candidate_cost = st.cost[nb];
    if (!isfinite(candidate_cost)) candidate_cost = 1.7976931348623157e308;
    const double cur_cost = st.cost[st.cur];
    // ParameterToleranceReached
    double sn = 0;
    for (int i = 0; i < NA; ++i) sn += (st.x[i] - st.cand[i]) * (st.x[i] - st.cand[i]);
    if (sqrt(sn) <= Lm::parameter_tolerance * (st.x_norm + Lm::parameter_tolerance)) { st.termination = 0; stop = 1; }
    // FunctionToleranceReached
    else if (fabs(cur_cost - candidate_cost) <= Lm::function_tolerance * cur_cost) { st.termination = 0; stop = 1; }
    else {
      const double relative = (st.ev_current - candidate_cost) / st.model_cost_change;
      const double historical = (st.ev_reference - candidate_cost) / (st.ev_acc_ref + st.model_cost_change);
      const double relative_decrease = fmax(relative, historical);
      if (relative_decrease > Lm::min_relative_decrease) {
        // HandleSuccessfulStep
        for (int i = 0; i < NA; ++i) st.x[i] = st.cand[i];
        st.x_norm = norm_ambient<NA>(st.x);
        st.cur = nb;
        st.cost[nb] = candidate_cost;
        st.gradient_max_norm = projected_gradient_max_norm<N>(st.x, st.g[nb], st.only_yaw);
        st.last_successful = 1;
        st.last_cost = candidate_cost;
        const double t = 2.0 * relative_decrease - 1.0;
        st.radius = st.radius / fmax(1.0 / 3.0, 1.0 - t * t * t);
        st.radius = fmin(Lm::max_radius, st.radius);
        st.decrease_factor = 2.0;
        st.reuse_diagonal = 0;
        st.ev_current = candidate_cost;
        st.ev_acc_cand += st.model_cost_change;
        st.ev_acc_ref += st.model_cost_change;
        if (st.ev_current < st.ev_minimum) {
          st.ev_minimum = st.ev_current;
          st.ev_num_nonmono = 0;
          st.ev_candidate = st.ev_current;
          st.ev_acc_cand = 0;
        } else {
          ++st.ev_num_nonmono;
          if (st.ev_current > st.ev_candidate) {
            st.ev_candidate = st.ev_current;
            st.ev_acc_cand = 0;
          }
        }
        if (st.ev_num_nonmono == st.max_nonmono) {
          st.ev_reference = st.ev_candidate;
          st.ev_acc_ref = st.ev_acc_cand;
        }
      } else {
        // HandleUnsuccessfulStep
        st.last_successful = 0;
        st.last_cost = candidate_cost;
        st.radius = st.radius / st.decrease_factor;
        st.decrease_factor *= 2.0;
        st.reuse_diagonal = 1;
      }
    }
    st.flag = stop;
  }
  __syncwarp();
  return st.flag;
}

// The trust-region loop of Ceres 1.13 (TrustRegionMinimizer::Minimize). Per round: one evaluation pass by every warp
// (with FUSED the last warp computes the IMU term instead of points, concurrently), one block barrier, then warp 0 alone
// finishes the reduction and runs the state machine up to the next candidate, one block barrier. FUSED adds the IMU
// term (15 local parameters).
template <bool FUSED>
__device__ __forceinline__ void solve_body(const NlsOptions& opt, const NlsProblem& prob, const ImuTerm* imu,
                                           const double* initial16, double* pose_out /*7 or 16*/,
                                           dl_solve_summary* summary) {
  constexpr int N = FUSED ? 15 : 6;
  constexpr int NA = Dims<N>::ambient;
  __shared__ Shared sh;
  __shared__ LmStateT<N> st;
  __shared__ typename std::conditional<FUSED, ImuShared, int>::type is_storage;
  __shared__ double xfull[16];
  ImuShared* is = FUSED ? reinterpret_cast<ImuShared*>(&is_storage) : nullptr;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, warps = blockDim.x >> 5;
  // Thread-block cluster (opt.cluster CTAs per problem, launched with cudaLaunchAttributeClusterDimension): every CTA evaluates
  // its share of the points, CTA 0 gathers the partial normal equations through distributed shared memory, runs the trust-region
  // step and pushes the next evaluation point (or the stop flag) into every CTA's shared memory. cluster.sync() replaces the
  // block barriers. One CTA per problem (ranks == 1) is the path of the ~400-point pipeline solves: unchanged arithmetic.
  cooperative_groups::cluster_group cluster = cooperative_groups::this_cluster();
  const int ranks = opt.cluster > 1 ? (int)cluster.num_blocks() : 1;
  const int rank = ranks > 1 ? (int)cluster.block_rank() : 0;
  auto barrier = [&]() {
    if (ranks > 1) cluster.sync(); else __syncthreads();
  };
  // with the IMU term and more than one warp, the last warp is the IMU warp (in CTA 0) and the others take the points
  const int imu_warp = FUSED ? warps - 1 : -1;
  const int point_warps = (FUSED && warps > 1) ? warps - 1 : warps;
  {
    double x[7], target_t[3], target_q_inv[4];
    setup_problem(opt, prob, sh, x, target_t, target_q_inv);
    if (threadIdx.x == 0) {
      for (int i = 0; i < 7; ++i) st.x[i] = x[i];
      if (FUSED)
        for (int i = 7; i < 16; ++i) st.x[i] = initial16[i];
      for (int i = 0; i < NA; ++i) xfull[i] = st.x[i];
      for (int i = 0; i < 3; ++i) st.target_t[i] = target_t[i];
      for (int i = 0; i < 4; ++i) st.target_q_inv[i] = target_q_inv[i];
      st.only_yaw = FUSED ? 0 : (opt.only_yaw != 0);
      st.nl = FUSED ? 15 : (st.only_yaw ? 4 : 6);
      st.max_iter = opt.max_iter;
      st.max_nonmono = opt.nonmono ? Lm::max_consecutive_nonmonotonic : 0;
      sh.stop = 0;
    }
    if (FUSED)
      for (int e = threadIdx.x; e < 225; e += blockDim.x) is->W[e] = imu->W[e];
  }
  barrier();
  bool first = true;
  for (;;) {
    evaluate_points(opt, prob, sh, point_warps * 32, rank, ranks);
    if (FUSED && rank == 0 && warp == imu_warp) imu_normal_equations(*imu, xfull, *is, lane);
    barrier();  // partial sums (and the IMU term) are in (distributed) shared memory
    if (rank == 0 && warp == 0) {
      finish_points(opt, sh, point_warps, st.target_q_inv, st.target_t, lane, ranks);
      int stop = 0;
      if (first) lm_iteration_zero<N>(st, sh, is, lane);
      else stop = lm_process_candidate<N>(st, sh, is, lane);
      if (!stop) stop = lm_prepare_step<N>(st, lane);
      if (lane == 0) {
        for (int r = 0; r < ranks; ++r) {  // r = 0 is this CTA itself
          Shared* dst = ranks > 1 ? cluster.map_shared_rank(&sh, r) : &sh;
          dst->stop = stop;
          if (!stop)
            for (int i = 0; i < 7; ++i) dst->x[i] = st.cand[i];
        }
        if (!stop)
          for (int i = 0; i < NA; ++i) xfull[i] = st.cand[i];
      }
    }
    first = false;
    barrier();  // the next evaluation point (or the stop flag) is visible to every CTA of the problem
    if (sh.stop) break;
  }
  if (rank != 0) return;
  if (threadIdx.x == 0) {
    for (int i = 0; i < NA; ++i) pose_out[i] = st.best_x[i];
    summary->initial_cost = st.initial_cost;
    summary->final_cost = st.final_cost;
    summary->num_iterations = st.recorded;
    summary->num_successful_steps = st.successful;
    summary->num_unsuccessful_steps = st.unsuccessful;
    summary->termination = st.termination;
    summary->num_evaluations = st.evals;
    summary->reserved = 0;
  }
}

__global__ void __launch_bounds__(kBlock, 2) nls_solve_kernel(NlsOptions opt, const NlsProblem* __restrict__ problems,
                                                           NlsOutput* __restrict__ outputs) {
  const int p = blockIdx.x / (opt.cluster > 1 ? opt.cluster : 1);
  NlsOutput& o = outputs[p];
  if (problems[p].enabled_dev && *problems[p].enabled_dev == 0) return;  // uniform over the problem's CTA(s)
  solve_body<false>(opt, problems[p], nullptr, nullptr, o.pose, &o.summary);
}

__global__ void __launch_bounds__(kBlock, 2) nls_fused_kernel(NlsOptions opt, const NlsProblem* __restrict__ problems,
                                                           const ImuTerm* __restrict__ imu,
                                                           const double* __restrict__ initial16,
                                                           FusedOutput* __restrict__ outputs) {
  const int p = blockIdx.x / (opt.cluster > 1 ? opt.cluster : 1);
  FusedOutput& o = outputs[p];
  if (problems[p].enabled_dev && *problems[p].enabled_dev == 0) return;  // uniform over the problem's CTA(s)
  solve_body<true>(opt, problems[p], imu + p, initial16 + 16 * p, o.state, &o.summary);
}

// One evaluation pass at a given pose; writes the 28 reduced doubles (cost, g, H upper triangle).
__global__ void __launch_bounds__(kBlock) nls_normal_equations_kernel(NlsOptions opt, const NlsProblem* problems,
                                                                      const double* at_pose, double* out28) {
  __shared__ Shared sh;
  const NlsProblem& prob = problems[blockIdx.x];
  __shared__ double target_t[3], target_q_inv[4];
  {
    double x[7], tt[3], tq[4];
    setup_problem(opt, prob, sh, x, tt, tq);
    if (threadIdx.x == 0) {
      for (int i = 0; i < 3; ++i) target_t[i] = tt[i];
      for (int i = 0; i < 4; ++i) target_q_inv[i] = tq[i];
    }
  }
  __syncthreads();
  if (threadIdx.x == 0)
    for (int i = 0; i < 7; ++i) sh.x[i] = at_pose[i];
  __syncthreads();
  evaluate_points(opt, prob, sh, blockDim.x);
  __syncthreads();
  if (threadIdx.x < 32) {
    finish_points(opt, sh, blockDim.x >> 5, target_q_inv, target_t, threadIdx.x);
    if (threadIdx.x < kRed) out28[blockIdx.x * kRed + threadIdx.x] = threadIdx.x == 0 ? 0.5 * sh.acc[0] : sh.acc[threadIdx.x];
  }
}

// The IMU term of the fused solve alone, one warp per prepared factor: residual, H = J^T W J, g = J^T W r and r^T W r at x16
// (submap frame). Factors whose covariance was not positive definite (ok == 0) are skipped.
__global__ void __launch_bounds__(32) imu_factor_evaluate_kernel(const ImuTerm* __restrict__ terms, const int32_t* __restrict__ ok,
                                                                 const double* __restrict__ x16, double* __restrict__ out) {
  __shared__ ImuShared is;
  __shared__ double x[16];
  const int b = blockIdx.x, lane = threadIdx.x;
  if (!ok[b]) return;
  for (int e = lane; e < 225; e += 32) is.W[e] = terms[b].W[e];
  if (lane < 16) x[lane] = x16[16 * (size_t)b + lane];
  __syncwarp();
  imu_normal_equations(terms[b], x, is, lane);
  double* o = out + (size_t)b * kImuFactorOutDoubles;  // r(15) H(225) g(15) cost2
  if (lane < 15) {
    o[lane] = is.r[lane];
    o[240 + lane] = is.g[lane];
  }
  for (int e = lane; e < 225; e += 32) o[15 + e] = is.H[e / 15][e % 15];
  if (lane == 0) o[255] = is.cost2;
}

__global__ void interpolate_kernel(GridView g, int64_t n, const double* __restrict__ xyz, double* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double v, gx, gy, gz;
  interpolate(g, xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], &v, &gx, &gy, &gz);
  out[4 * i] = v; out[4 * i + 1] = gx; out[4 * i + 2] = gy; out[4 * i + 3] = gz;
}

__global__ void grid_lookup_kernel(GridView g, int64_t n, const int32_t* __restrict__ xyz, uint16_t* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  out[i] = grid_value(g, xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]);
}

}  // namespace

// One CTA of kBlock threads per problem, or opt.cluster CTAs (a thread-block cluster) per problem. The kernels find their
// problem as blockIdx.x / cluster size. (Fewer threads per ~400-point problem measured slower: the evaluation pass serialises
// inside a thread.)
template <typename Kernel, typename... Args>
static cudaError_t launch_solve(Kernel kernel, const NlsOptions& opt, int count, cudaStream_t stream, Args... args) {
  const int cs = opt.cluster > 1 ? opt.cluster : 1;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3((unsigned)(count * cs));
  cfg.blockDim = dim3((unsigned)kBlock);
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = (unsigned)cs;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = cs > 1 ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, args...);
}

int launch_nls(dl_context* ctx, const NlsOptions& opt, const NlsProblem* problems_dev, int count, NlsOutput* out_dev) {
  if (count <= 0) return DL_OK;
  DL_CUDA(ctx, launch_solve(nls_solve_kernel, opt, count, ctx->stream, opt, problems_dev, out_dev));
  DL_LAUNCH_CHECK(ctx, "nls_solve_kernel");
  return DL_OK;
}

int launch_nls_fused(dl_context* ctx, const NlsOptions& opt, const NlsProblem* problems_dev, const ImuTerm* imu_terms_dev,
                     const double* initial16_dev, int count, FusedOutput* out_dev) {
  if (count <= 0) return DL_OK;
  DL_CUDA(ctx, launch_solve(nls_fused_kernel, opt, count, ctx->stream, opt, problems_dev, imu_terms_dev, initial16_dev, out_dev));
  DL_LAUNCH_CHECK(ctx, "nls_fused_kernel");
  return DL_OK;
}

int launch_nls_normal_equations(dl_context* ctx, const NlsOptions& opt, const NlsProblem* problems_dev,
                                const double* at_pose_dev, double* out28_dev) {
  nls_normal_equations_kernel<<<1, kBlock, 0, ctx->stream>>>(opt, problems_dev, at_pose_dev, out28_dev);
  DL_LAUNCH_CHECK(ctx, "nls_normal_equations_kernel");
  return DL_OK;
}

int launch_imu_factor_evaluate(dl_context* ctx, int count, const ImuTerm* terms_dev, const int32_t* ok_dev, const double* x16_dev,
                               double* out_dev) {
  if (count <= 0) return DL_OK;
  imu_factor_evaluate_kernel<<<count, 32, 0, ctx->stream>>>(terms_dev, ok_dev, x16_dev, out_dev);
  DL_LAUNCH_CHECK(ctx, "imu_factor_evaluate_kernel");
  return DL_OK;
}

int launch_interpolate(dl_context* ctx, const GridView& grid, int64_t n, const double* xyz, double* out) {
  if (n <= 0) return DL_OK;
  interpolate_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(grid, n, xyz, out);
  DL_LAUNCH_CHECK(ctx, "interpolate_kernel");
  return DL_OK;
}

int launch_grid_lookup(dl_context* ctx, const GridView& grid, int64_t n, const int32_t* xyz, uint16_t* out) {
  if (n <= 0) return DL_OK;
  grid_lookup_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(grid, n, xyz, out);
  DL_LAUNCH_CHECK(ctx, "grid_lookup_kernel");
  return DL_OK;
}

}  // namespace dl

// ------------------------------------------------------------------------------------------------ Ceres-equivalent matcher
namespace dl {
int check_ceres_options(dl_context* ctx, const dl_ceres_options* o, int num_pairs) {
  if (!o) return DL_ERR_ARG;
  if (num_pairs < 1 || num_pairs > DL_MAX_PAIRS) return ctx->fail(DL_ERR_ARG, "num_pairs out of range");
  if (o->num_occupied_space_weights != num_pairs)
    return ctx->fail(DL_ERR_ARG, "occupied_space_weight count != number of (cloud, grid) pairs (CHECK_EQ)");
  for (int i = 0; i < num_pairs; ++i)
    if (!(o->occupied_space_weight[i] > 0.)) return ctx->fail(DL_ERR_ARG, "occupied_space_weight must be > 0 (CHECK_GT)");
  if (o->max_num_iterations <= 0) return ctx->fail(DL_ERR_ARG, "max_num_iterations must be > 0 (CHECK_GT)");
  return DL_OK;
}
NlsOptions to_nls_options(const dl_ceres_options& o, int num_pairs) {
  NlsOptions n{};
  n.num_pairs = num_pairs;
  for (int i = 0; i < num_pairs; ++i) n.occ_weight[i] = o.occupied_space_weight[i];
  n.trans_weight = o.translation_weight;
  n.rot_weight = o.rotation_weight;
  n.only_yaw = o.only_optimize_yaw;
  n.nonmono = o.use_nonmonotonic_steps;
  n.max_iter = o.max_num_iterations;
  return n;
}
}  // namespace dl

using namespace dl;

extern "C" {

int dl_ceres_match_batch(dl_context* ctx, const dl_ceres_options* options, int32_t count, int32_t num_pairs,
                         const double* target_translations, const double* initial_poses, const float* const* clouds,
                         const int64_t* sizes, const dl_grid* const* grids, double* poses_out,
                         dl_solve_summary* summaries) {
  if (!ctx) return DL_ERR_ARG;
  DL_TRY(check_ceres_options(ctx, options, num_pairs));
  if (count < 0 || (count > 0 && (!target_translations || !initial_poses || !clouds || !sizes || !grids || !poses_out)))
    return DL_ERR_ARG;
  if (count == 0) return DL_OK;
  DL_CUDA(ctx, cudaSetDevice(ctx->device));
  for (int i = 0; i < count * num_pairs; ++i) {
    if (sizes[i] < 0 || !grids[i] || (sizes[i] > 0 && !clouds[i])) return DL_ERR_ARG;
    if (sizes[i] == 0) return ctx->fail(DL_ERR_EMPTY, "empty point cloud");
    if (grids[i]->structure_dirty) return ctx->fail(DL_ERR_ARG, "dl_grid_sync not called after dl_grid_set_cells");
  }
  std::vector<float*> d_clouds(count * num_pairs);
  NlsProblem* d_problems;
  NlsOutput* d_out;
  DL_TRY(carve_scratch(ctx, [&](Arena& a) {
    for (int i = 0; i < count * num_pairs; ++i) d_clouds[i] = a.take<float>(3 * sizes[i]);
    d_problems = a.take<NlsProblem>(count);
    d_out = a.take<NlsOutput>(count);
  }));
  std::vector<NlsProblem> problems(count);
  for (int c = 0; c < count; ++c) {
    NlsProblem& p = problems[c];
    std::memset(&p, 0, sizeof(p));
    for (int k = 0; k < num_pairs; ++k) {
      const int i = c * num_pairs + k;
      DL_TRY(h2d(ctx, d_clouds[i], clouds[i], 3 * sizes[i]));
      p.cloud[k] = d_clouds[i];
      p.count[k] = (int32_t)sizes[i];
      p.grid[k] = grids[i]->view();
    }
    for (int j = 0; j < 3; ++j) p.target_t[j] = target_translations[3 * c + j];
    for (int j = 0; j < 7; ++j) p.initial[j] = initial_poses[7 * c + j];
  }
  DL_TRY(h2d(ctx, d_problems, problems.data(), count));
  DL_TRY(launch_nls(ctx, to_nls_options(*options, num_pairs), d_problems, count, d_out));
  std::vector<NlsOutput> out(count);
  DL_TRY(d2h(ctx, out.data(), d_out, count));
  DL_TRY(sync(ctx));
  for (int c = 0; c < count; ++c) {
    std::memcpy(poses_out + 7 * c, out[c].pose, 7 * sizeof(double));
    if (summaries) summaries[c] = out[c].summary;
  }
  return DL_OK;
}

int dl_ceres_match(dl_context* ctx, const dl_ceres_options* options, const double* target_translation,
                   const double* initial_pose, int32_t num_pairs, const float* const* clouds, const int64_t* sizes,
                   const dl_grid* const* grids, double* pose_out, dl_solve_summary* summary) {
  return dl_ceres_match_batch(ctx, options, 1, num_pairs, target_translation, initial_pose, clouds, sizes, grids,
                              pose_out, summary);
}

int dl_ceres_normal_equations(dl_context* ctx, const dl_ceres_options* options, const double* target_translation,
                              const double* reference_pose, const double* at_pose, int32_t num_pairs,
                              const float* const* clouds, const int64_t* sizes, const dl_grid* const* grids,
                              double* cost, double* gradient6, double* hessian36) {
  if (!ctx) return DL_ERR_ARG;
  DL_TRY(check_ceres_options(ctx, options, num_pairs));
  if (!target_translation || !reference_pose || !at_pose || !clouds || !sizes || !grids || !cost || !gradient6 || !hessian36)
    return DL_ERR_ARG;
  DL_CUDA(ctx, cudaSetDevice(ctx->device));
  float* d_clouds[DL_MAX_PAIRS];
  NlsProblem* d_p;
  double *d_at, *d_out;
  DL_TRY(carve_scratch(ctx, [&](Arena& a) {
    for (int k = 0; k < num_pairs; ++k) d_clouds[k] = a.take<float>(3 * sizes[k]);
    d_p = a.take<NlsProblem>(1);
    d_at = a.take<double>(7);
    d_out = a.take<double>(28);
  }));
  NlsProblem p;
  std::memset(&p, 0, sizeof(p));
  for (int k = 0; k < num_pairs; ++k) {
    DL_TRY(h2d(ctx, d_clouds[k], clouds[k], 3 * sizes[k]));
    p.cloud[k] = d_clouds[k];
    p.count[k] = (int32_t)sizes[k];
    p.grid[k] = grids[k]->view();
  }
  for (int j = 0; j < 3; ++j) p.target_t[j] = target_translation[j];
  for (int j = 0; j < 7; ++j) p.initial[j] = reference_pose[j];
  DL_TRY(h2d(ctx, d_p, &p, 1));
  DL_TRY(h2d(ctx, d_at, at_pose, 7));
  DL_TRY(launch_nls_normal_equations(ctx, to_nls_options(*options, num_pairs), d_p, d_at, d_out));
  double out[28];
  DL_TRY(d2h(ctx, out, d_out, 28));
  DL_TRY(sync(ctx));
  *cost = out[0];
  for (int i = 0; i < 6; ++i) gradient6[i] = out[1 + i];
  int t = 7;
  for (int r = 0; r < 6; ++r)
    for (int c = r; c < 6; ++c) hessian36[r * 6 + c] = hessian36[c * 6 + r] = out[t++];
  return DL_OK;
}

}  // extern "C"
