// The reference's two-stage front end, second stage: LocalTrajectoryBuilder3D::WindowOptimize (LTB:693-863) without GTSAM.
//
// The reference feeds the scan matcher's pose as a PriorFactor<Pose3> (sigmas ceres_pose_noise_{t,r}, LTB:94-101, :815-818) into
// an iSAM2 smoother next to the IMU factor and the bias random walk between the previous key and the new one (:801-812), and
// re-seeds the graph every num_range_data keys from the marginal covariances of the last key (:750-797). iSAM2 never drops a
// key inside one segment, but the NEWEST key — the only estimate the front end reads (:846-852) — depends on the older ones only
// through the marginal of the previous key, which is exactly what a fixed-lag smoother with lag one carries. That is what is
// built here (SURVEY 8f-3):
//   variables  x_i (previous key), x_j (new key): 15 local parameters each, order p, theta, v, b_a, b_g
//   factors    prior on x_i     : mean = the previous estimate, information = the marginal carried from the previous step
//              IMU factor       : the in-repo pre-integration residual with the first-order bias correction
//                                 (integration_base.h:267-301) weighted by the propagated covariance^-1 (:156-236); its last six
//                                 rows are the bias random walk between the two keys
//              pose prior on x_j: the matched pose, diagonal sigmas (translation, rotation)
//              optional gravity prior on x_j's roll / pitch (gravity_factor.cc:10-31): the body-frame reference direction must
//                                 map to the estimated gravity direction. Both are directions: the host refuses a zero or
//                                 non-finite one and normalises both (Unit3 does the same), so their lengths do not enter
//   solve     Gauss-Newton on the 30 x 30 normal equations (Jacobians by forward-mode duals: one code path for every factor),
//              then the Schur complement on x_i gives the information of x_j = the prior of the next step
//   difference from GTSAM, stated: GTSAM's PreintegratedImuMeasurements / ImuFactor integrate on the manifold with a 9-dim
//              residual and a separate bias BetweenFactor; the integrator here is the reference's own IntegrationBase. Neither
//              library is in this image, so the row's parity is pinned oracle <-> device only (DESIGN.md).
//   difference from gravity_factor.cc, stated: the reference rotates b_ref by x_j's roll and pitch only (Rot3::RzRyRx(r.x, r.y, 0),
//              :20, :25) and adds k_cost_value = 1e-5 to both error components (:12, :27-28); here b_ref is rotated by the whole
//              R_j and the residual has no offset.
// dl_window_evaluate runs window_weights and window_residuals alone at given (x_i, x_j), so the factors can be checked on their own.
// One warp per trajectory: lane 0 forms the residuals and their duals, the 32 lanes share the 30 x 30 linear algebra.
#include <cmath>
#include <cstring>
#include <vector>

#include "dl_internal.cuh"

namespace dl {
namespace {

constexpr int kVars = 30;
constexpr int kRes = 38;  // 15 prior + 15 imu + 6 pose + 2 gravity

struct D30 {  // dual number over the 30 local parameters
  double a;
  double v[kVars];
};
__device__ __forceinline__ D30 dc(double s) { D30 d; d.a = s; for (int i = 0; i < kVars; ++i) d.v[i] = 0.; return d; }
__device__ __forceinline__ D30 operator+(const D30& f, const D30& g) { D30 h; h.a = f.a + g.a; for (int i = 0; i < kVars; ++i) h.v[i] = f.v[i] + g.v[i]; return h; }
__device__ __forceinline__ D30 operator-(const D30& f, const D30& g) { D30 h; h.a = f.a - g.a; for (int i = 0; i < kVars; ++i) h.v[i] = f.v[i] - g.v[i]; return h; }
__device__ __forceinline__ D30 operator*(const D30& f, const D30& g) { D30 h; h.a = f.a * g.a; for (int i = 0; i < kVars; ++i) h.v[i] = f.a * g.v[i] + f.v[i] * g.a; return h; }
__device__ __forceinline__ D30 operator*(double s, const D30& f) { D30 h; h.a = s * f.a; for (int i = 0; i < kVars; ++i) h.v[i] = s * f.v[i]; return h; }
__device__ __forceinline__ D30 operator/(const D30& f, const D30& g) {
  const double gi = 1.0 / g.a, fg = f.a * gi;
  D30 h; h.a = fg; for (int i = 0; i < kVars; ++i) h.v[i] = (f.v[i] - fg * g.v[i]) * gi; return h;
}
__device__ __forceinline__ D30 dsqrt(const D30& f) { const double r = sqrt(f.a), d = 0.5 / r; D30 h; h.a = r; for (int i = 0; i < kVars; ++i) h.v[i] = f.v[i] * d; return h; }
struct DQ { D30 w, x, y, z; };
struct DV { D30 x, y, z; };
__device__ DQ dqmul(const DQ& a, const DQ& b) {
  return {a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z, a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y,
          a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z, a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x};
}
__device__ DQ dqconj(const DQ& q) { return {q.w, -1.0 * q.x, -1.0 * q.y, -1.0 * q.z}; }
__device__ DQ dqinverse(const DQ& q) {  // Eigen inverse(): conjugate / squared norm
  const D30 n2 = q.w * q.w + q.x * q.x + q.y * q.y + q.z * q.z;
  const DQ c = dqconj(q);
  return {c.w / n2, c.x / n2, c.y / n2, c.z / n2};
}
__device__ DV dqrotate(const DQ& q, const DV& v) {  // v + w uv + q x uv, uv = 2 q x v
  DV uv{q.y * v.z - q.z * v.y, q.z * v.x - q.x * v.z, q.x * v.y - q.y * v.x};
  uv = {uv.x + uv.x, uv.y + uv.y, uv.z + uv.z};
  return {v.x + q.w * uv.x + (q.y * uv.z - q.z * uv.y), v.y + q.w * uv.y + (q.z * uv.x - q.x * uv.z),
          v.z + q.w * uv.z + (q.x * uv.y - q.y * uv.x)};
}
// x (+) delta of the fused solve (dl_nls.cu plus()): q <- (cos|d|, sin|d|/|d| d) (x) q, everything else additive. As duals with the
// perturbation variables [base, base + 15) active at delta = 0: d(sin|d|/|d| d)/dd = I, d cos|d| / dd = 0 there.
struct DState { DV p; DQ q; DV v, ba, bg; };
__device__ DState lift(const double* x16, int base) {
  DState s;
  auto var = [&](double val, int k) { D30 d = dc(val); d.v[base + k] = 1.; return d; };
  s.p = {var(x16[0], 0), var(x16[1], 1), var(x16[2], 2)};
  const Quatd q{x16[3], x16[4], x16[5], x16[6]};
  // (1, d) (x) q: w' = w - d.qv, v' = w d + qv x ... ; partial w.r.t. d_k at 0 = e_k (x) q
  D30 qw = dc(q.w), qx = dc(q.x), qy = dc(q.y), qz = dc(q.z);
  for (int k = 0; k < 3; ++k) {
    const Quatd e{0., k == 0 ? 1. : 0., k == 1 ? 1. : 0., k == 2 ? 1. : 0.};
    const Quatd d = qmul(e, q);
    qw.v[base + 3 + k] = d.w; qx.v[base + 3 + k] = d.x; qy.v[base + 3 + k] = d.y; qz.v[base + 3 + k] = d.z;
  }
  s.q = {qw, qx, qy, qz};
  s.v = {var(x16[7], 6), var(x16[8], 7), var(x16[9], 8)};
  s.ba = {var(x16[10], 9), var(x16[11], 10), var(x16[12], 11)};
  s.bg = {var(x16[13], 12), var(x16[14], 13), var(x16[15], 14)};
  return s;
}
__device__ void state_plus(const double* x, const double* delta, double* out) {
  for (int k = 0; k < 3; ++k) out[k] = x[k] + delta[k];
  const double n = sqrt(delta[3] * delta[3] + delta[4] * delta[4] + delta[5] * delta[5]);
  Quatd r{x[3], x[4], x[5], x[6]};
  if (n > 0.) {
    const double s = sin(n) / n;
    r = qmul(Quatd{cos(n), s * delta[3], s * delta[4], s * delta[5]}, r);
  }
  out[3] = r.w; out[4] = r.x; out[5] = r.y; out[6] = r.z;
  for (int k = 0; k < 9; ++k) out[7 + k] = x[7 + k] + delta[6 + k];
}
// x (-) mean in the same chart: rotation part = the vector d with (cos|d|, sin|d|/|d| d) = q (x) mean^-1, as duals
__device__ void state_minus(const DState& s, const double* mean16, D30 out[15]) {
  out[0] = s.p.x - dc(mean16[0]); out[1] = s.p.y - dc(mean16[1]); out[2] = s.p.z - dc(mean16[2]);
  const DQ mi{dc(mean16[3]), dc(-mean16[4]), dc(-mean16[5]), dc(-mean16[6])};
  DQ e = dqmul(s.q, mi);
  if (e.w.a < 0.) e = {-1.0 * e.w, -1.0 * e.x, -1.0 * e.y, -1.0 * e.z};
  const D30 vn2 = e.x * e.x + e.y * e.y + e.z * e.z;
  // d = atan2(|v|, w) / |v| * v; near zero the factor is 1 / w (series), which keeps the duals finite at v = 0
  if (vn2.a < 1e-16) {
    const D30 f = dc(1.) / e.w;
    out[3] = f * e.x; out[4] = f * e.y; out[5] = f * e.z;
  } else {
    const D30 vn = dsqrt(vn2);
    D30 ang; ang.a = atan2(vn.a, e.w.a);
    const double dd = 1.0 / (e.w.a * e.w.a + vn.a * vn.a);
    for (int i = 0; i < kVars; ++i) ang.v[i] = dd * (e.w.a * vn.v[i] - vn.a * e.w.v[i]);
    const D30 f = ang / vn;
    out[3] = f * e.x; out[4] = f * e.y; out[5] = f * e.z;
  }
  out[6] = s.v.x - dc(mean16[7]); out[7] = s.v.y - dc(mean16[8]); out[8] = s.v.z - dc(mean16[9]);
  out[9] = s.ba.x - dc(mean16[10]); out[10] = s.ba.y - dc(mean16[11]); out[11] = s.ba.z - dc(mean16[12]);
  out[12] = s.bg.x - dc(mean16[13]); out[13] = s.bg.y - dc(mean16[14]); out[14] = s.bg.z - dc(mean16[15]);
}

struct WindowShared {
  double r[kRes];
  double J[kRes][kVars];
  double W[kRes][kRes];   // block-diagonal weight: prior information, IMU information, pose and gravity 1/sigma^2
  double WJ[kRes][kVars];
  double H[kVars][kVars], g[kVars], L[kVars][kVars], delta[kVars];
  double xi[16], xj[16];
  double cost;
  int ok;
};

__device__ void store(const D30& d, WindowShared& sh, int row) {
  sh.r[row] = d.a;
  for (int k = 0; k < kVars; ++k) sh.J[row][k] = d.v[k];
}

struct WindowArgs {
  int count;
  const dl_nav_state* states_i;      // prior mean (the previous estimate), local frame
  const double* prior_information;   // 225 per problem
  const dl_preintegration* preint;
  const double* matched_pose;        // 7 per problem
  const dl_nav_state* initial_j;     // optional start for x_j (default: the IMU prediction)
  dl_window_options opt;
  dl_nav_state* states_i_out;        // smoothed previous state (optional)
  dl_nav_state* states_j_out;
  double* information_out;           // 225 per problem
  dl_solve_summary* summaries;
};

__device__ void nav_to16(const dl_nav_state& s, double* x) {
  for (int k = 0; k < 3; ++k) { x[k] = s.p[k]; x[7 + k] = s.v[k]; x[10 + k] = s.ba[k]; x[13 + k] = s.bg[k]; }
  for (int k = 0; k < 4; ++k) x[3 + k] = s.q[k];
}
__device__ void nav_from16(const double* x, dl_nav_state* s) {
  for (int k = 0; k < 3; ++k) { s->p[k] = x[k]; s->v[k] = x[7 + k]; s->ba[k] = x[10 + k]; s->bg[k] = x[13 + k]; }
  for (int k = 0; k < 4; ++k) s->q[k] = x[3 + k];
}

// lane 0: residuals and duals of all factors at (xi, xj)
__device__ void window_residuals(const WindowArgs& a, int b, WindowShared& sh) {
  const dl_preintegration& m = a.preint[b];
  const DState si = lift(sh.xi, 0), sj = lift(sh.xj, 15);
  double mean[16];
  nav_to16(a.states_i[b], mean);
  // ---- prior on x_i
  {
    D30 d[15];
    state_minus(si, mean, d);
    for (int k = 0; k < 15; ++k) store(d[k], sh, k);
  }
  // ---- IMU factor (integration_base.h:267-301)
  {
    const double T = m.sum_dt;
    const double* Jm = m.jacobian;
    auto blk = [&](int r0, int c0, const DV& v) {  // 3x3 block of the bias Jacobian times a dual vector
      DV o;
      o.x = Jm[(r0 + 0) * 15 + c0] * v.x + Jm[(r0 + 0) * 15 + c0 + 1] * v.y + Jm[(r0 + 0) * 15 + c0 + 2] * v.z;
      o.y = Jm[(r0 + 1) * 15 + c0] * v.x + Jm[(r0 + 1) * 15 + c0 + 1] * v.y + Jm[(r0 + 1) * 15 + c0 + 2] * v.z;
      o.z = Jm[(r0 + 2) * 15 + c0] * v.x + Jm[(r0 + 2) * 15 + c0 + 1] * v.y + Jm[(r0 + 2) * 15 + c0 + 2] * v.z;
      return o;
    };
    const DV dba{si.ba.x - dc(m.linearized_ba[0]), si.ba.y - dc(m.linearized_ba[1]), si.ba.z - dc(m.linearized_ba[2])};
    const DV dbg{si.bg.x - dc(m.linearized_bg[0]), si.bg.y - dc(m.linearized_bg[1]), si.bg.z - dc(m.linearized_bg[2])};
    const DV th = blk(3, 12, dbg);  // dq_dbg * dbg
    const DQ dq{dc(m.delta_q[0]), dc(m.delta_q[1]), dc(m.delta_q[2]), dc(m.delta_q[3])};
    const DQ corrected_q = dqmul(dq, DQ{dc(1.), 0.5 * th.x, 0.5 * th.y, 0.5 * th.z});  // delta_q * deltaQ(.)
    const DV pa = blk(0, 9, dba), pg = blk(0, 12, dbg), va = blk(6, 9, dba), vg = blk(6, 12, dbg);
    const DV corrected_p{dc(m.delta_p[0]) + pa.x + pg.x, dc(m.delta_p[1]) + pa.y + pg.y, dc(m.delta_p[2]) + pa.z + pg.z};
    const DV corrected_v{dc(m.delta_v[0]) + va.x + vg.x, dc(m.delta_v[1]) + va.y + vg.y, dc(m.delta_v[2]) + va.z + vg.z};
    const double G[3] = {a.opt.gravity[0], a.opt.gravity[1], a.opt.gravity[2]};
    const DQ qi_inv = dqconj(si.q);  // unit quaternion
    const DV tp{dc(0.5 * G[0] * T * T) + sj.p.x - si.p.x - T * si.v.x, dc(0.5 * G[1] * T * T) + sj.p.y - si.p.y - T * si.v.y,
                dc(0.5 * G[2] * T * T) + sj.p.z - si.p.z - T * si.v.z};
    const DV rp = dqrotate(qi_inv, tp);
    const DV tv{dc(G[0] * T) + sj.v.x - si.v.x, dc(G[1] * T) + sj.v.y - si.v.y, dc(G[2] * T) + sj.v.z - si.v.z};
    const DV rv = dqrotate(qi_inv, tv);
    const DQ e = dqmul(dqinverse(corrected_q), dqmul(qi_inv, sj.q));
    store(rp.x - corrected_p.x, sh, 15); store(rp.y - corrected_p.y, sh, 16); store(rp.z - corrected_p.z, sh, 17);
    store(2.0 * e.x, sh, 18); store(2.0 * e.y, sh, 19); store(2.0 * e.z, sh, 20);
    store(rv.x - corrected_v.x, sh, 21); store(rv.y - corrected_v.y, sh, 22); store(rv.z - corrected_v.z, sh, 23);
    store(sj.ba.x - si.ba.x, sh, 24); store(sj.ba.y - si.ba.y, sh, 25); store(sj.ba.z - si.ba.z, sh, 26);
    store(sj.bg.x - si.bg.x, sh, 27); store(sj.bg.y - si.bg.y, sh, 28); store(sj.bg.z - si.bg.z, sh, 29);
  }
  // ---- pose prior on x_j: translation difference, 2 vec(q_m^-1 q_j)
  {
    const double* z = a.matched_pose + 7 * (size_t)b;
    store(sj.p.x - dc(z[0]), sh, 30); store(sj.p.y - dc(z[1]), sh, 31); store(sj.p.z - dc(z[2]), sh, 32);
    const DQ zi{dc(z[3]), dc(-z[4]), dc(-z[5]), dc(-z[6])};
    DQ e = dqmul(zi, sj.q);
    if (e.w.a < 0.) e = {-1.0 * e.w, -1.0 * e.x, -1.0 * e.y, -1.0 * e.z};
    store(2.0 * e.x, sh, 33); store(2.0 * e.y, sh, 34); store(2.0 * e.z, sh, 35);
  }
  // ---- gravity direction on x_j: R_j * b_ref should point along g_dir (both unit: the host normalised them, as Unit3 does);
  //      residual = the two components of R_j b_ref orthogonal to g_dir in a fixed basis of its tangent plane (the role of
  //      Unit3::error in gravity_factor.cc:10-31)
  if (a.opt.use_gravity_factor) {
    const double* gd = a.opt.gravity_direction;
    const double* br = a.opt.body_reference_direction;
    const DV n = dqrotate(sj.q, DV{dc(br[0]), dc(br[1]), dc(br[2])});
    // basis of the plane orthogonal to gd
    const Vec3d g{gd[0], gd[1], gd[2]};
    const Vec3d helper = fabs(g.x) < 0.9 ? Vec3d{1, 0, 0} : Vec3d{0, 1, 0};
    Vec3d b1 = cross3(g, helper);
    b1 = mul(1.0 / norm3(b1), b1);
    const Vec3d b2 = cross3(g, b1);
    store(b1.x * n.x + b1.y * n.y + b1.z * n.z, sh, 36);
    store(b2.x * n.x + b2.y * n.y + b2.z * n.z, sh, 37);
  } else {
    store(dc(0.), sh, 36);
    store(dc(0.), sh, 37);
  }
}

// Cholesky solve of the n x n SPD system in sh.L (copied from M) for `rhs` (in place); lanes = rows. Returns (uniform) success.
__device__ bool warp_cholesky(double (*L)[kVars], int n, int lane) {
  for (int j = 0; j < n; ++j) {
    double s = 0.;
    if (lane >= j && lane < n) {
      s = L[lane][j];
      for (int k = 0; k < j; ++k) s -= L[lane][k] * L[j][k];
    }
    const double pivot = __shfl_sync(0xffffffffu, s, j);
    if (!(pivot > 0.)) return false;
    const double d = sqrt(pivot);
    if (lane >= j && lane < n) L[lane][j] = lane == j ? d : s / d;
    __syncwarp();
  }
  return true;
}
__device__ void warp_solve(double (*L)[kVars], int n, double* x /* rhs in, solution out */, int lane) {
  double rhs = lane < n ? x[lane] : 0.;
  for (int k = 0; k < n; ++k) {
    const double zk = __shfl_sync(0xffffffffu, lane < n ? rhs / L[lane][lane] : 0., k);
    if (lane == k) rhs = zk; else if (lane > k && lane < n) rhs -= L[lane][k] * zk;
  }
  for (int k = n - 1; k >= 0; --k) {
    const double yk = __shfl_sync(0xffffffffu, lane < n ? rhs / L[lane][lane] : 0., k);
    if (lane == k) rhs = yk; else if (lane < k) rhs -= L[k][lane] * yk;
  }
  if (lane < n) x[lane] = rhs;
  __syncwarp();
}

constexpr int kWarpsPerBlock = 2;

// The block-diagonal weight of problem b into sh.W (whole warp): prior information, imu_weight^2 covariance^-1, the pose prior's and
// the gravity factor's 1 / sigma^2. Returns (uniform) false when the covariance is not positive definite; the IMU block is then 0.
__device__ bool window_weights(const WindowArgs& a, int b, WindowShared& sh, int lane) {
  const dl_preintegration& m = a.preint[b];
  for (int e = lane; e < kRes * kRes; e += 32) sh.W[e / kRes][e % kRes] = 0.;
  __syncwarp();
  for (int e = lane; e < 225; e += 32) sh.W[e / 15][e % 15] = a.prior_information[(size_t)b * 225 + e];
  // IMU information = covariance^-1 by Cholesky (lanes = rows), scratch in sh.L / sh.H
  for (int e = lane; e < 225; e += 32) sh.L[e / 15][e % 15] = m.covariance[e];
  __syncwarp();
  bool ok = warp_cholesky(sh.L, 15, lane);
  if (ok) {
    // columns of the inverse: solve L L^T x = e_c
    for (int c = 0; c < 15; ++c) {
      if (lane < 15) sh.delta[lane] = lane == c ? 1. : 0.;
      __syncwarp();
      warp_solve(sh.L, 15, sh.delta, lane);
      if (lane < 15) sh.W[15 + lane][15 + c] = a.opt.imu_weight * a.opt.imu_weight * sh.delta[lane];
      __syncwarp();
    }
  }
  if (lane == 0) {
    const double wt = 1.0 / (a.opt.pose_sigma_translation * a.opt.pose_sigma_translation);
    const double wr = 1.0 / (a.opt.pose_sigma_rotation * a.opt.pose_sigma_rotation);
    for (int k = 0; k < 3; ++k) { sh.W[30 + k][30 + k] = wt; sh.W[33 + k][33 + k] = wr; }
    const double wg = a.opt.use_gravity_factor ? 1.0 / (a.opt.gravity_sigma * a.opt.gravity_sigma) : 0.;
    sh.W[36][36] = sh.W[37][37] = wg;
  }
  return ok;
}

__global__ void __launch_bounds__(kWarpsPerBlock * 32) window_optimize_kernel(WindowArgs a) {
  extern __shared__ __align__(16) unsigned char smem[];
  WindowShared* all = reinterpret_cast<WindowShared*>(smem);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int b = blockIdx.x * kWarpsPerBlock + warp;
  if (b >= a.count) return;
  WindowShared& sh = all[warp];
  const dl_preintegration& m = a.preint[b];
  bool ok = window_weights(a, b, sh, lane);
  if (lane == 0) {
    nav_to16(a.states_i[b], sh.xi);
    if (a.initial_j) {
      nav_to16(a.initial_j[b], sh.xj);
    } else {  // IMU prediction (dl_imu_predict's arithmetic)
      const dl_nav_state& si = a.states_i[b];
      const double T = m.sum_dt;
      const Quatd qi{si.q[0], si.q[1], si.q[2], si.q[3]};
      const Vec3d G{a.opt.gravity[0], a.opt.gravity[1], a.opt.gravity[2]};
      const Vec3d pi{si.p[0], si.p[1], si.p[2]}, vi{si.v[0], si.v[1], si.v[2]};
      const Vec3d pj = add(sub(add(pi, mul(T, vi)), mul(0.5 * T * T, G)), rotate(qi, Vec3d{m.delta_p[0], m.delta_p[1], m.delta_p[2]}));
      const Vec3d vj = add(sub(vi, mul(T, G)), rotate(qi, Vec3d{m.delta_v[0], m.delta_v[1], m.delta_v[2]}));
      const Quatd qj = qnormalized(qmul(qi, Quatd{m.delta_q[0], m.delta_q[1], m.delta_q[2], m.delta_q[3]}));
      dl_nav_state sj = si;
      for (int k = 0; k < 3; ++k) sj.p[k] = (&pj.x)[k], sj.v[k] = (&vj.x)[k];
      sj.q[0] = qj.w; sj.q[1] = qj.x; sj.q[2] = qj.y; sj.q[3] = qj.z;
      nav_to16(sj, sh.xj);
    }
    sh.ok = ok ? 1 : 0;
  }
  __syncwarp();
  int iterations = 0;
  double initial_cost = 0., cost = 0.;
  const int max_iter = a.opt.max_num_iterations > 0 ? a.opt.max_num_iterations : 10;
  bool converged = false;
  while (ok) {
    if (lane == 0) window_residuals(a, b, sh);
    __syncwarp();
    // WJ = W J, H = J^T W J, g = J^T W r, cost = 1/2 r^T W r
    for (int e = lane; e < kRes * kVars; e += 32) {
      const int r = e / kVars, c = e % kVars;
      double s = 0.;
      const int r0 = r < 15 ? 0 : (r < 30 ? 15 : r), r1 = r < 15 ? 15 : (r < 30 ? 30 : r + 1);  // block-diagonal W
      for (int k = r0; k < r1; ++k) s += sh.W[r][k] * sh.J[k][c];
      sh.WJ[r][c] = s;
    }
    __syncwarp();
    if (lane < kVars) {
      for (int c = 0; c < kVars; ++c) {
        double s = 0.;
        for (int r = 0; r < kRes; ++r) s += sh.J[r][lane] * sh.WJ[r][c];
        sh.H[lane][c] = s;
      }
      double gs = 0.;
      for (int r = 0; r < kRes; ++r) gs += sh.WJ[r][lane] * sh.r[r];
      sh.g[lane] = gs;
    }
    if (lane == 31) {
      double c2 = 0.;
      for (int r = 0; r < kRes; ++r) {
        const int r0 = r < 15 ? 0 : (r < 30 ? 15 : r), r1 = r < 15 ? 15 : (r < 30 ? 30 : r + 1);
        double s = 0.;
        for (int k = r0; k < r1; ++k) s += sh.W[r][k] * sh.r[k];
        c2 += sh.r[r] * s;
      }
      sh.cost = 0.5 * c2;
    }
    __syncwarp();
    cost = sh.cost;
    if (iterations == 0) initial_cost = cost;
    if (converged || iterations >= max_iter) break;
    // Gauss-Newton step: H delta = -g
    for (int e = lane; e < kVars * kVars; e += 32) sh.L[e / kVars][e % kVars] = sh.H[e / kVars][e % kVars];
    if (lane < kVars) sh.delta[lane] = -sh.g[lane];
    __syncwarp();
    if (!warp_cholesky(sh.L, kVars, lane)) { ok = false; break; }
    warp_solve(sh.L, kVars, sh.delta, lane);
    double n2 = lane < kVars ? sh.delta[lane] * sh.delta[lane] : 0.;
    for (int d = 16; d > 0; d >>= 1) n2 += __shfl_xor_sync(0xffffffffu, n2, d);
    if (lane == 0) {
      double t[16];
      state_plus(sh.xi, sh.delta, t);
      for (int k = 0; k < 16; ++k) sh.xi[k] = t[k];
      state_plus(sh.xj, sh.delta + 15, t);
      for (int k = 0; k < 16; ++k) sh.xj[k] = t[k];
    }
    __syncwarp();
    ++iterations;
    converged = sqrt(n2) < 1e-10;  // one more evaluation at the converged point gives the final cost and linearisation
  }
  // marginal information of x_j: H_jj - H_ji H_ii^-1 H_ij at the final linearisation
  if (ok) {
    for (int e = lane; e < 225; e += 32) sh.L[e / 15][e % 15] = sh.H[e / 15][e % 15];
    __syncwarp();
    ok = warp_cholesky(sh.L, 15, lane);
    if (ok) {
      for (int c = 0; c < 15; ++c) {  // column c of H_ii^-1 H_ij, then the Schur complement's column c
        if (lane < 15) sh.delta[lane] = sh.H[lane][15 + c];
        __syncwarp();
        warp_solve(sh.L, 15, sh.delta, lane);
        if (lane < 15) {
          double s = sh.H[15 + lane][15 + c];
          for (int k = 0; k < 15; ++k) s -= sh.H[15 + lane][k] * sh.delta[k];
          a.information_out[(size_t)b * 225 + lane * 15 + c] = s;
        }
        __syncwarp();
      }
    }
  }
  if (lane == 0) {
    if (ok) {
      nav_from16(sh.xj, &a.states_j_out[b]);
      if (a.states_i_out) nav_from16(sh.xi, &a.states_i_out[b]);
    }
    if (a.summaries) {
      dl_solve_summary s{};
      s.initial_cost = initial_cost;
      s.final_cost = cost;
      s.num_iterations = iterations;
      s.num_successful_steps = iterations;
      s.termination = !ok ? 2 : (converged ? 0 : 1);
      s.num_evaluations = iterations + 1;
      a.summaries[b] = s;
    }
  }
}

// The factors alone at given (x_i, x_j) (dl_window_evaluate): the weight and residual code of window_optimize_kernel, written out.
// x: 32 doubles per problem (x_i then x_j, p q v ba bg each); out: kWindowEvalDoubles per problem, r (38), J (38 x 30), W (38 x 38).
__global__ void __launch_bounds__(kWarpsPerBlock * 32) window_evaluate_kernel(WindowArgs a, const double* __restrict__ x,
                                                                              int32_t* __restrict__ ok_out, double* __restrict__ out) {
  extern __shared__ __align__(16) unsigned char smem[];
  WindowShared* all = reinterpret_cast<WindowShared*>(smem);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int b = blockIdx.x * kWarpsPerBlock + warp;
  if (b >= a.count) return;
  WindowShared& sh = all[warp];
  const bool ok = window_weights(a, b, sh, lane);
  if (lane < 16) { sh.xi[lane] = x[(size_t)b * 32 + lane]; sh.xj[lane] = x[(size_t)b * 32 + 16 + lane]; }
  __syncwarp();
  if (ok && lane == 0) window_residuals(a, b, sh);
  __syncwarp();
  double* o = out + (size_t)b * kWindowEvalDoubles;
  for (int e = lane; e < kRes; e += 32) o[e] = ok ? sh.r[e] : 0.;
  for (int e = lane; e < kRes * kVars; e += 32) o[kRes + e] = ok ? sh.J[e / kVars][e % kVars] : 0.;
  for (int e = lane; e < kRes * kRes; e += 32) o[kRes + kRes * kVars + e] = ok ? sh.W[e / kRes][e % kRes] : 0.;
  if (lane == 0) ok_out[b] = ok ? 1 : 0;
}

}  // namespace

int launch_window_evaluate(dl_context* ctx, int count, const dl_nav_state* states_i, const double* prior_information,
                           const dl_preintegration* preint, const double* matched_pose, const dl_window_options& opt, const double* x,
                           int32_t* ok, double* out) {
  if (count <= 0) return DL_OK;
  WindowArgs a{count, states_i, prior_information, preint, matched_pose, nullptr, opt, nullptr, nullptr, nullptr, nullptr};
  const size_t smem = sizeof(WindowShared) * kWarpsPerBlock;
  DL_CUDA(ctx, cudaFuncSetAttribute(window_evaluate_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  window_evaluate_kernel<<<(count + kWarpsPerBlock - 1) / kWarpsPerBlock, kWarpsPerBlock * 32, smem, ctx->stream>>>(a, x, ok, out);
  DL_LAUNCH_CHECK(ctx, "window_evaluate_kernel");
  return DL_OK;
}

int launch_window_optimize(dl_context* ctx, int count, const dl_nav_state* states_i, const double* prior_information,
                           const dl_preintegration* preint, const double* matched_pose, const dl_nav_state* initial_j,
                           const dl_window_options& opt, dl_nav_state* states_i_out, dl_nav_state* states_j_out,
                           double* information_out, dl_solve_summary* summaries) {
  if (count <= 0) return DL_OK;
  WindowArgs a{count, states_i, prior_information, preint, matched_pose, initial_j, opt, states_i_out, states_j_out, information_out, summaries};
  const size_t smem = sizeof(WindowShared) * kWarpsPerBlock;
  DL_CUDA(ctx, cudaFuncSetAttribute(window_optimize_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  window_optimize_kernel<<<(count + kWarpsPerBlock - 1) / kWarpsPerBlock, kWarpsPerBlock * 32, smem, ctx->stream>>>(a);
  DL_LAUNCH_CHECK(ctx, "window_optimize_kernel");
  return DL_OK;
}

}  // namespace dl

// ------------------------------------------------------------------------------------------------ two-stage window
using namespace dl;

namespace {
// The options of dl_window_optimize_batch and dl_window_evaluate as the kernels take them: sigmas and the IMU weight positive and,
// with the gravity factor on, both directions finite and non-zero. Only their orientation enters the factor (Unit3 normalises
// too), so both are normalised here, the one place that does it.
int window_options_checked(dl_context* ctx, const dl_window_options& in, dl_window_options* out) {
  if (!(in.pose_sigma_translation > 0.) || !(in.pose_sigma_rotation > 0.) || !(in.imu_weight > 0.) ||
      (in.use_gravity_factor && !(in.gravity_sigma > 0.)))
    return ctx->fail(DL_ERR_ARG, "dl_window_options: sigmas and the IMU weight must be positive");
  *out = in;
  if (!in.use_gravity_factor) return DL_OK;
  for (double* d : {out->gravity_direction, out->body_reference_direction}) {
    const double n = std::sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
    if (!std::isfinite(n) || !(n > 0.))
      return ctx->fail(DL_ERR_ARG, "dl_window_options: the gravity and body reference directions must be finite and non-zero");
    for (int k = 0; k < 3; ++k) d[k] /= n;
  }
  return DL_OK;
}
}  // namespace

namespace dl {
void carve_window(Arena& a, int count, WindowBuffers* w) {
  const size_t n = (size_t)count;
  w->si = a.take<dl_nav_state>(n);
  w->prior = a.take<double>(n * 225);
  w->pre = a.take<dl_preintegration>(n);
  w->z = a.take<double>(n * 7);
  w->init = a.take<dl_nav_state>(n);
  w->si_out = a.take<dl_nav_state>(n);
  w->sj_out = a.take<dl_nav_state>(n);
  w->info = a.take<double>(n * 225);
  w->sum = a.take<dl_solve_summary>(n);
}
int window_optimize(dl_context* ctx, const dl_window_options& options, int count, const WindowBuffers& w, const dl_nav_state* states_i,
                    const double* prior_information, const dl_preintegration* preintegrations, const double* matched_poses,
                    const dl_nav_state* initial_states_j, dl_nav_state* states_i_out, dl_nav_state* states_j_out,
                    double* information_out, dl_solve_summary* summaries) {
  const size_t n = (size_t)count;
  DL_TRY(h2d(ctx, w.si, states_i, n));
  DL_TRY(h2d(ctx, w.prior, prior_information, n * 225));
  DL_TRY(h2d(ctx, w.pre, preintegrations, n));
  DL_TRY(h2d(ctx, w.z, matched_poses, n * 7));
  if (initial_states_j) DL_TRY(h2d(ctx, w.init, initial_states_j, n));
  DL_CUDA(ctx, cudaMemsetAsync(w.sj_out, 0, n * sizeof(dl_nav_state), ctx->stream));
  DL_CUDA(ctx, cudaMemsetAsync(w.info, 0, n * 225 * 8, ctx->stream));
  DL_TRY(launch_window_optimize(ctx, count, w.si, w.prior, w.pre, w.z, initial_states_j ? w.init : nullptr, options, w.si_out, w.sj_out,
                                w.info, w.sum));
  DL_TRY(d2h(ctx, states_j_out, w.sj_out, n));
  if (states_i_out) DL_TRY(d2h(ctx, states_i_out, w.si_out, n));
  DL_TRY(d2h(ctx, information_out, w.info, n * 225));
  std::vector<dl_solve_summary> sums(n);
  DL_TRY(d2h(ctx, sums.data(), w.sum, n));
  DL_TRY(sync(ctx));
  if (summaries) std::memcpy(summaries, sums.data(), n * sizeof(dl_solve_summary));
  return DL_OK;
}
}  // namespace dl

extern "C" int dl_window_optimize_batch(dl_context* ctx, const dl_window_options* options, int32_t count, const dl_nav_state* states_i,
                                        const double* prior_information, const dl_preintegration* preintegrations,
                                        const double* matched_poses, const dl_nav_state* initial_states_j, dl_nav_state* states_i_out,
                                        dl_nav_state* states_j_out, double* information_out, dl_solve_summary* summaries) {
  if (!ctx || !options || count < 0) return DL_ERR_ARG;
  if (count == 0) return DL_OK;
  if (!states_i || !prior_information || !preintegrations || !matched_poses || !states_j_out || !information_out) return DL_ERR_ARG;
  dl_window_options o;
  DL_TRY(window_options_checked(ctx, *options, &o));
  DL_CUDA(ctx, cudaSetDevice(ctx->device));
  WindowBuffers w;
  DL_TRY(carve_scratch(ctx, [&](Arena& a) { carve_window(a, count, &w); }));
  return window_optimize(ctx, o, count, w, states_i, prior_information, preintegrations, matched_poses, initial_states_j,
                         states_i_out, states_j_out, information_out, summaries);
}

extern "C" int dl_window_evaluate(dl_context* ctx, const dl_window_options* options, int32_t count, const dl_nav_state* states_i,
                                  const double* prior_information, const dl_preintegration* preintegrations, const double* matched_poses,
                                  const dl_nav_state* x_i, const dl_nav_state* x_j, int32_t* ok, double* residuals, double* jacobians,
                                  double* weights) {
  if (!ctx || !options || count < 0) return DL_ERR_ARG;
  if (count == 0) return DL_OK;
  if (!states_i || !prior_information || !preintegrations || !matched_poses || !x_i || !x_j || !ok || !residuals || !jacobians ||
      !weights)
    return DL_ERR_ARG;
  dl_window_options o;
  DL_TRY(window_options_checked(ctx, *options, &o));
  DL_CUDA(ctx, cudaSetDevice(ctx->device));
  const size_t n = (size_t)count;
  dl_nav_state* d_si;
  dl_preintegration* d_pre;
  double *d_prior, *d_z, *d_x, *d_out;
  int32_t* d_ok;
  DL_TRY(carve_scratch(ctx, [&](Arena& a) {
    d_si = a.take<dl_nav_state>(n);
    d_prior = a.take<double>(n * 225);
    d_pre = a.take<dl_preintegration>(n);
    d_z = a.take<double>(n * 7);
    d_x = a.take<double>(n * 32);
    d_out = a.take<double>(n * kWindowEvalDoubles);
    d_ok = a.take<int32_t>(n);
  }));
  std::vector<double> x(n * 32);
  for (size_t k = 0; k < n; ++k)
    for (int s = 0; s < 2; ++s) {
      const dl_nav_state& v = (s == 0 ? x_i : x_j)[k];
      double* d = x.data() + 32 * k + 16 * s;
      for (int c = 0; c < 3; ++c) { d[c] = v.p[c]; d[7 + c] = v.v[c]; d[10 + c] = v.ba[c]; d[13 + c] = v.bg[c]; }
      for (int c = 0; c < 4; ++c) d[3 + c] = v.q[c];
    }
  DL_TRY(h2d(ctx, d_si, states_i, n));
  DL_TRY(h2d(ctx, d_prior, prior_information, n * 225));
  DL_TRY(h2d(ctx, d_pre, preintegrations, n));
  DL_TRY(h2d(ctx, d_z, matched_poses, n * 7));
  DL_TRY(h2d(ctx, d_x, x.data(), n * 32));
  DL_TRY(launch_window_evaluate(ctx, count, d_si, d_prior, d_pre, d_z, o, d_x, d_ok, d_out));
  std::vector<double> out(n * kWindowEvalDoubles);
  DL_TRY(d2h(ctx, ok, d_ok, n));
  DL_TRY(d2h(ctx, out.data(), d_out, out.size()));
  DL_TRY(sync(ctx));
  for (size_t k = 0; k < n; ++k) {
    const double* s = out.data() + k * kWindowEvalDoubles;
    std::memcpy(residuals + 38 * k, s, 38 * sizeof(double));
    std::memcpy(jacobians + 38 * 30 * k, s + 38, 38 * 30 * sizeof(double));
    std::memcpy(weights + 38 * 38 * k, s + 38 + 38 * 30, 38 * 38 * sizeof(double));
  }
  return DL_OK;
}
