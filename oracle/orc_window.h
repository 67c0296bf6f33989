// TEST INFRASTRUCTURE — CPU oracle (see orc_math.h header).
//
// The two-stage front end's second stage, restated for the checks of csrc/dl_window.cu: the fixed-lag (lag one) smoother that
// stands in for LocalTrajectoryBuilder3D::WindowOptimize (LTB:693-863): prior on the previous key, the in-repo pre-integration
// residual with first-order bias correction (integration_base.h:267-301) weighted by its propagated covariance, the matched
// pose as a diagonal prior on the new key (LTB:94-101, :815-818), optional gravity-direction prior (gravity_factor.cc:10-31).
// Written independently of the device code on purpose: residuals in plain doubles, Jacobians by CENTRAL DIFFERENCES in the
// tangent space (the device uses forward-mode duals), dense Cholesky from orc_nls.h.
// parity unpinned against GTSAM (absent from this image and from /root/reference): see DESIGN.md.
#pragma once
#include <cmath>
#include <vector>

#include "orc_imu.h"
#include "orc_math.h"
#include "orc_nls.h"

namespace orc {

struct WindowOptions {
  double pose_sigma_t = 0.05, pose_sigma_r = 0.01, imu_weight = 1.0;
  V3d gravity{0, 0, 9.8};
  int max_num_iterations = 10;
  bool use_gravity_factor = false;
  double gravity_sigma = 0.05;
  V3d gravity_direction{0, 0, 1}, body_reference_direction{0, 0, 1};
};

inline void window_plus(const double* x, const double* d, double* out) {  // chart of the fused solve: q <- exp(d) q, |d| = half angle
  for (int k = 0; k < 3; ++k) out[k] = x[k] + d[k];
  const double n = std::sqrt(d[3] * d[3] + d[4] * d[4] + d[5] * d[5]);
  Quatd r{x[3], x[4], x[5], x[6]};
  if (n > 0.) {
    const double s = std::sin(n) / n;
    r = qmul(Quatd{std::cos(n), s * d[3], s * d[4], s * d[5]}, r);
  }
  out[3] = r.w; out[4] = r.x; out[5] = r.y; out[6] = r.z;
  for (int k = 0; k < 9; ++k) out[7 + k] = x[7 + k] + d[6 + k];
}

// the 38 residuals at (xi, xj): 15 prior, 15 imu, 6 pose, 2 gravity
inline void window_residuals(const WindowOptions& o, const double* mean_i, const Preintegration& m, const Rigid3d& matched,
                             const double* xi, const double* xj, double* r) {
  // prior: xi (-) mean
  for (int k = 0; k < 3; ++k) r[k] = xi[k] - mean_i[k];
  {
    Quatd e = qmul(Quatd{xi[3], xi[4], xi[5], xi[6]}, Quatd{mean_i[3], -mean_i[4], -mean_i[5], -mean_i[6]});
    if (e.w < 0) e = {-e.w, -e.x, -e.y, -e.z};
    const double vn = std::sqrt(e.x * e.x + e.y * e.y + e.z * e.z);
    const double f = vn < 1e-8 ? 1.0 / e.w : std::atan2(vn, e.w) / vn;
    r[3] = f * e.x; r[4] = f * e.y; r[5] = f * e.z;
  }
  for (int k = 0; k < 9; ++k) r[6 + k] = xi[7 + k] - mean_i[7 + k];
  // IMU
  const V3d pi{xi[0], xi[1], xi[2]}, vi{xi[7], xi[8], xi[9]}, bai{xi[10], xi[11], xi[12]}, bgi{xi[13], xi[14], xi[15]};
  const V3d pj{xj[0], xj[1], xj[2]}, vj{xj[7], xj[8], xj[9]}, baj{xj[10], xj[11], xj[12]}, bgj{xj[13], xj[14], xj[15]};
  const Quatd qi{xi[3], xi[4], xi[5], xi[6]}, qj{xj[3], xj[4], xj[5], xj[6]};
  auto blk = [&](int r0, int c0, const V3d& v) {
    return V3d{m.jacobian[r0][c0] * v.x + m.jacobian[r0][c0 + 1] * v.y + m.jacobian[r0][c0 + 2] * v.z,
               m.jacobian[r0 + 1][c0] * v.x + m.jacobian[r0 + 1][c0 + 1] * v.y + m.jacobian[r0 + 1][c0 + 2] * v.z,
               m.jacobian[r0 + 2][c0] * v.x + m.jacobian[r0 + 2][c0 + 1] * v.y + m.jacobian[r0 + 2][c0 + 2] * v.z};
  };
  const V3d dba = bai - m.ba, dbg = bgi - m.bg;
  const V3d th = blk(3, 12, dbg);
  const Quatd cq = qmul(m.delta_q, Quatd{1.0, 0.5 * th.x, 0.5 * th.y, 0.5 * th.z});
  const V3d cp = m.delta_p + blk(0, 9, dba) + blk(0, 12, dbg);
  const V3d cv = m.delta_v + blk(6, 9, dba) + blk(6, 12, dbg);
  const double T = m.sum_dt;
  const Quatd qi_inv = conj(qi);
  const V3d rp = rotate(qi_inv, scale(0.5 * T * T, o.gravity) + pj - pi - scale(T, vi)) - cp;
  const V3d rv = rotate(qi_inv, scale(T, o.gravity) + vj - vi) - cv;
  const double n2 = cq.w * cq.w + cq.x * cq.x + cq.y * cq.y + cq.z * cq.z;
  const Quatd cq_inv{cq.w / n2, -cq.x / n2, -cq.y / n2, -cq.z / n2};
  const Quatd e = qmul(cq_inv, qmul(qi_inv, qj));
  r[15] = rp.x; r[16] = rp.y; r[17] = rp.z;
  r[18] = 2 * e.x; r[19] = 2 * e.y; r[20] = 2 * e.z;
  r[21] = rv.x; r[22] = rv.y; r[23] = rv.z;
  r[24] = baj.x - bai.x; r[25] = baj.y - bai.y; r[26] = baj.z - bai.z;
  r[27] = bgj.x - bgi.x; r[28] = bgj.y - bgi.y; r[29] = bgj.z - bgi.z;
  // pose prior
  r[30] = pj.x - matched.t.x; r[31] = pj.y - matched.t.y; r[32] = pj.z - matched.t.z;
  Quatd ez = qmul(conj(matched.q), qj);
  if (ez.w < 0) ez = {-ez.w, -ez.x, -ez.y, -ez.z};
  r[33] = 2 * ez.x; r[34] = 2 * ez.y; r[35] = 2 * ez.z;
  // gravity direction
  r[36] = r[37] = 0;
  if (o.use_gravity_factor) {
    const V3d n = rotate(qj, o.body_reference_direction);   // both directions unit (window_optimize normalised them)
    const V3d& g = o.gravity_direction;
    const V3d helper = std::fabs(g.x) < 0.9 ? V3d{1, 0, 0} : V3d{0, 1, 0};
    auto cross = [](const V3d& a, const V3d& b) { return V3d{a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; };
    V3d b1 = cross(g, helper);
    b1 = scale(1.0 / std::sqrt(b1.x * b1.x + b1.y * b1.y + b1.z * b1.z), b1);
    const V3d b2 = cross(g, b1);
    r[36] = b1.x * n.x + b1.y * n.y + b1.z * n.z;
    r[37] = b2.x * n.x + b2.y * n.y + b2.z * n.z;
  }
}

// Returns false if a matrix is not positive definite or, with the gravity factor on, a direction is zero or not finite.
// xi_out / xj_out: 16 doubles; info_out: 225.
inline bool window_optimize(const WindowOptions& o_in, const double* mean_i, const double* prior_info, const Preintegration& m,
                            const Rigid3d& matched, const double* initial_j, double* xi_out, double* xj_out, double* info_out,
                            int* iterations_out, double* initial_cost_out, double* final_cost_out, int* termination_out) {
  WindowOptions o = o_in;
  constexpr int R = 38, N = 30;
  if (o_in.use_gravity_factor) {  // both are directions (Unit3): only their orientation enters the factor
    for (V3d* d : {&o.gravity_direction, &o.body_reference_direction}) {
      const double n = std::sqrt(d->x * d->x + d->y * d->y + d->z * d->z);
      if (!std::isfinite(n) || !(n > 0.)) return false;
      *d = scale(1.0 / n, *d);
    }
  }
  std::vector<double> W((size_t)R * R, 0.0);
  for (int a = 0; a < 15; ++a)
    for (int b = 0; b < 15; ++b) W[(size_t)a * R + b] = prior_info[a * 15 + b];
  {  // IMU information = covariance^-1
    for (int c = 0; c < 15; ++c) {
      std::vector<double> A(225), e(15, 0.0), x(15);
      for (int a = 0; a < 15; ++a)
        for (int b = 0; b < 15; ++b) A[a * 15 + b] = m.covariance[a][b];
      e[c] = 1.0;
      if (!cholesky_solve_dense(A.data(), e.data(), 15, x.data())) return false;
      for (int a = 0; a < 15; ++a) W[(size_t)(15 + a) * R + 15 + c] = o.imu_weight * o.imu_weight * x[a];
    }
  }
  for (int k = 0; k < 3; ++k) {
    W[(size_t)(30 + k) * R + 30 + k] = 1.0 / (o.pose_sigma_t * o.pose_sigma_t);
    W[(size_t)(33 + k) * R + 33 + k] = 1.0 / (o.pose_sigma_r * o.pose_sigma_r);
  }
  if (o.use_gravity_factor) W[(size_t)36 * R + 36] = W[(size_t)37 * R + 37] = 1.0 / (o.gravity_sigma * o.gravity_sigma);
  double xi[16], xj[16];
  for (int k = 0; k < 16; ++k) xi[k] = mean_i[k];
  if (initial_j) {
    for (int k = 0; k < 16; ++k) xj[k] = initial_j[k];
  } else {
    const NavState p = imu_predict(FusedProblem::unpack(mean_i), m, o.gravity);
    FusedProblem::pack(p, xj);
  }
  std::vector<double> r(R), J((size_t)R * N), H((size_t)N * N), g(N);
  int iterations = 0;
  bool converged = false;
  double cost = 0, initial_cost = 0;
  const int max_iter = o.max_num_iterations > 0 ? o.max_num_iterations : 10;
  for (;;) {
    window_residuals(o, mean_i, m, matched, xi, xj, r.data());
    const double h = 1e-6;
    for (int k = 0; k < N; ++k) {  // central differences in the tangent space
      double d[15] = {0}, a[16], b[16], rp[R], rm[R];
      d[k % 15] = h;
      if (k < 15) { window_plus(xi, d, a); window_residuals(o, mean_i, m, matched, a, xj, rp); }
      else { window_plus(xj, d, a); window_residuals(o, mean_i, m, matched, xi, a, rp); }
      d[k % 15] = -h;
      if (k < 15) { window_plus(xi, d, b); window_residuals(o, mean_i, m, matched, b, xj, rm); }
      else { window_plus(xj, d, b); window_residuals(o, mean_i, m, matched, xi, b, rm); }
      for (int q = 0; q < R; ++q) J[(size_t)q * N + k] = (rp[q] - rm[q]) / (2 * h);
    }
    std::vector<double> WJ((size_t)R * N, 0.0), Wr(R, 0.0);
    for (int a = 0; a < R; ++a)
      for (int b = 0; b < R; ++b) {
        const double w = W[(size_t)a * R + b];
        if (w == 0.0) continue;
        Wr[a] += w * r[b];
        for (int k = 0; k < N; ++k) WJ[(size_t)a * N + k] += w * J[(size_t)b * N + k];
      }
    cost = 0;
    for (int a = 0; a < R; ++a) cost += 0.5 * r[a] * Wr[a];
    for (int a = 0; a < N; ++a) {
      g[a] = 0;
      for (int q = 0; q < R; ++q) g[a] += J[(size_t)q * N + a] * Wr[q];
      for (int b = 0; b < N; ++b) {
        double s = 0;
        for (int q = 0; q < R; ++q) s += J[(size_t)q * N + a] * WJ[(size_t)q * N + b];
        H[(size_t)a * N + b] = s;
      }
    }
    if (iterations == 0) initial_cost = cost;
    if (converged || iterations >= max_iter) break;
    std::vector<double> A(H), rhs(N), delta(N);
    for (int a = 0; a < N; ++a) rhs[a] = -g[a];
    if (!cholesky_solve_dense(A.data(), rhs.data(), N, delta.data())) return false;
    double t[16], n2 = 0;
    window_plus(xi, delta.data(), t);
    for (int k = 0; k < 16; ++k) xi[k] = t[k];
    window_plus(xj, delta.data() + 15, t);
    for (int k = 0; k < 16; ++k) xj[k] = t[k];
    for (int a = 0; a < N; ++a) n2 += delta[a] * delta[a];
    ++iterations;
    converged = std::sqrt(n2) < 1e-10;
  }
  // Schur complement on x_i
  for (int c = 0; c < 15; ++c) {
    std::vector<double> A(225), b(15), x(15);
    for (int a = 0; a < 15; ++a) {
      b[a] = H[(size_t)a * N + 15 + c];
      for (int k = 0; k < 15; ++k) A[a * 15 + k] = H[(size_t)a * N + k];
    }
    if (!cholesky_solve_dense(A.data(), b.data(), 15, x.data())) return false;
    for (int a = 0; a < 15; ++a) {
      double s = H[(size_t)(15 + a) * N + 15 + c];
      for (int k = 0; k < 15; ++k) s -= H[(size_t)(15 + a) * N + k] * x[k];
      info_out[a * 15 + c] = s;
    }
  }
  for (int k = 0; k < 16; ++k) { xi_out[k] = xi[k]; xj_out[k] = xj[k]; }
  *iterations_out = iterations;
  *initial_cost_out = initial_cost;
  *final_cost_out = cost;
  *termination_out = converged ? 0 : 1;
  return true;
}

}  // namespace orc
