// TEST INFRASTRUCTURE — CPU oracle (see orc_math.h header).
//
// IMU pre-integration and the scan-match solve with the pre-integration residual FUSED in (SURVEY 8a row a12).
//
// (1) Pre-integration: restated from the reference's in-repo integrator
//       C/mapping/internal/3d/initialization/integration_base.h:109-123 (push_back: the first sample only latches
//       acc_0 / gyr_0), :156-236 (midPointIntegration: state, 15x15 Jacobian F and noise map V), :238-265 (propagate,
//       delta_q re-normalised after every step), noise layout :36-51.
//     Row/column order of `jacobian` / `covariance` follows the F matrix code: [0:3] delta_p, [3:6] delta_theta,
//     [6:9] delta_v, [9:12] b_a, [12:15] b_g. (The file's StateOrder enum swaps O_P / O_R, but nothing live reads it.)
// (2) Residual: the 15-dim residual the same file documents (commented `evaluate`, :267-301):
//       r_p = R_i^T (1/2 G T^2 + p_j - p_i - v_i T) - dp,  r_th = 2 vec(dq^-1 (x) q_i^-1 (x) q_j),
//       r_v = R_i^T (G T + v_j - v_i) - dv,  r_ba = ba_j - ba_i,  r_bg = bg_j - bg_i,   G = +9.8 z by default.
// (3) Fused solve — an EXTENSION, not reference behaviour: the reference runs CeresScanMatcher3D::Match and then
//     hands the pose to GTSAM iSAM2 as a prior next to a gtsam::ImuFactor (LTB:535-555, :693-863; SURVEY F1).
//     BASELINE.json's north star asks for one solve: here the previous state i is held fixed and the 15 local
//     parameters of state j (dp, dtheta [left-multiplied like ceres::QuaternionParameterization], dv, dba, dbg) are
//     estimated from the occupied-space residuals + the (optional) translation / rotation priors + the IMU residual
//     whitened by the pre-integration covariance, with the same Levenberg-Marquardt loop as the scan matcher.
//     GTSAM 4.0.2 is not available here: parity for this row is oracle <-> GPU only ("parity unpinned" against the
//     reference).
#pragma once
#include <cmath>
#include <vector>

#include "orc_math.h"
#include "orc_nls.h"

namespace orc {

struct ImuNoise {
  double acc_n, gyr_n, acc_w, gyr_w;
};

struct Preintegration {
  double sum_dt = 0;
  V3d delta_p{0, 0, 0}, delta_v{0, 0, 0};
  Quatd delta_q{1, 0, 0, 0};
  V3d ba{0, 0, 0}, bg{0, 0, 0};
  double jacobian[15][15];
  double covariance[15][15];
  bool started = false;
  V3d acc_0{0, 0, 0}, gyr_0{0, 0, 0};
};

inline void preint_reset(Preintegration* p, const V3d& ba, const V3d& bg) {
  *p = Preintegration();
  p->ba = ba;
  p->bg = bg;
  for (int i = 0; i < 15; ++i)
    for (int j = 0; j < 15; ++j) {
      p->jacobian[i][j] = i == j ? 1.0 : 0.0;
      p->covariance[i][j] = 0.0;
    }
}

// Eigen Quaternion::toRotationMatrix (no normalisation)
inline void to_rotation_matrix(const Quatd& q, double R[3][3]) {
  const double tx = 2 * q.x, ty = 2 * q.y, tz = 2 * q.z;
  const double twx = tx * q.w, twy = ty * q.w, twz = tz * q.w;
  const double txx = tx * q.x, txy = ty * q.x, txz = tz * q.x, tyy = ty * q.y, tyz = tz * q.y, tzz = tz * q.z;
  R[0][0] = 1 - (tyy + tzz); R[0][1] = txy - twz; R[0][2] = txz + twy;
  R[1][0] = txy + twz; R[1][1] = 1 - (txx + tzz); R[1][2] = tyz - twx;
  R[2][0] = txz - twy; R[2][1] = tyz + twx; R[2][2] = 1 - (txx + tyy);
}
inline void skew(const V3d& v, double S[3][3]) {
  S[0][0] = 0; S[0][1] = -v.z; S[0][2] = v.y;
  S[1][0] = v.z; S[1][1] = 0; S[1][2] = -v.x;
  S[2][0] = -v.y; S[2][1] = v.x; S[2][2] = 0;
}
inline void mat3_mul(const double A[3][3], const double B[3][3], double C[3][3]) {
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) C[i][j] = A[i][0] * B[0][j] + A[i][1] * B[1][j] + A[i][2] * B[2][j];
}

// IntegrationBase::push_back + propagate + midPointIntegration
inline void preint_push(Preintegration* p, double dt, const V3d& acc_1, const V3d& gyr_1, const ImuNoise& n) {
  if (!p->started) {  // integration_base.h:111-118
    p->started = true;
    p->acc_0 = acc_1;
    p->gyr_0 = gyr_1;
    return;
  }
  const V3d un_acc_0 = rotate(p->delta_q, p->acc_0 - p->ba);
  const V3d un_gyr = scale(0.5, p->gyr_0 + gyr_1) - p->bg;
  const Quatd result_q = qmul(p->delta_q, Quatd{1, un_gyr.x * dt / 2, un_gyr.y * dt / 2, un_gyr.z * dt / 2});
  const V3d un_acc_1 = rotate(result_q, acc_1 - p->ba);
  const V3d un_acc = scale(0.5, un_acc_0 + un_acc_1);
  const V3d result_p = p->delta_p + scale(dt, p->delta_v) + scale(0.5 * dt * dt, un_acc);
  const V3d result_v = p->delta_v + scale(dt, un_acc);

  // F (15x15) and V (15x18), integration_base.h:176-232
  const V3d w_x = un_gyr, a_0_x = p->acc_0 - p->ba, a_1_x = acc_1 - p->ba;
  double Rw[3][3], Ra0[3][3], Ra1[3][3], R0[3][3], R1[3][3], I_Rw[3][3];
  skew(w_x, Rw); skew(a_0_x, Ra0); skew(a_1_x, Ra1);
  to_rotation_matrix(p->delta_q, R0);
  to_rotation_matrix(result_q, R1);
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) I_Rw[i][j] = (i == j ? 1.0 : 0.0) - Rw[i][j] * dt;
  double R0a0[3][3], R1a1[3][3], R1a1I[3][3];
  mat3_mul(R0, Ra0, R0a0);
  mat3_mul(R1, Ra1, R1a1);
  mat3_mul(R1a1, I_Rw, R1a1I);
  static thread_local std::vector<double> Fm(225), Vm(270);
  auto F = [&](int r, int c) -> double& { return Fm[r * 15 + c]; };
  auto V = [&](int r, int c) -> double& { return Vm[r * 18 + c]; };
  std::fill(Fm.begin(), Fm.end(), 0.0);
  std::fill(Vm.begin(), Vm.end(), 0.0);
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) {
      const double id = i == j ? 1.0 : 0.0;
      F(i, j) = id;
      F(i, 3 + j) = -0.25 * R0a0[i][j] * dt * dt + -0.25 * R1a1I[i][j] * dt * dt;
      F(i, 6 + j) = id * dt;
      F(i, 9 + j) = -0.25 * (R0[i][j] + R1[i][j]) * dt * dt;
      F(i, 12 + j) = -0.25 * R1a1[i][j] * dt * dt * -dt;
      F(3 + i, 3 + j) = I_Rw[i][j];
      F(3 + i, 12 + j) = -1.0 * id * dt;
      F(6 + i, 3 + j) = -0.5 * R0a0[i][j] * dt - 0.5 * R1a1I[i][j] * dt;
      F(6 + i, 6 + j) = id;
      F(6 + i, 9 + j) = -0.5 * (R0[i][j] + R1[i][j]) * dt;
      F(6 + i, 12 + j) = -0.5 * R1a1[i][j] * dt * -dt;
      F(9 + i, 9 + j) = id;
      F(12 + i, 12 + j) = id;
      V(i, j) = 0.25 * R0[i][j] * dt * dt;
      V(i, 3 + j) = 0.25 * -R1a1[i][j] * dt * dt * 0.5 * dt;
      V(i, 6 + j) = 0.25 * R1[i][j] * dt * dt;
      V(i, 9 + j) = V(i, 3 + j);
      V(3 + i, 3 + j) = 0.5 * id * dt;
      V(3 + i, 9 + j) = 0.5 * id * dt;
      V(6 + i, j) = 0.5 * R0[i][j] * dt;
      V(6 + i, 3 + j) = 0.5 * -R1a1[i][j] * dt * 0.5 * dt;
      V(6 + i, 6 + j) = 0.5 * R1[i][j] * dt;
      V(6 + i, 9 + j) = V(6 + i, 3 + j);
      V(9 + i, 12 + j) = id * dt;
      V(12 + i, 15 + j) = id * dt;
    }
  }
  const double nd[18] = {n.acc_n * n.acc_n, n.acc_n * n.acc_n, n.acc_n * n.acc_n, n.gyr_n * n.gyr_n, n.gyr_n * n.gyr_n,
                         n.gyr_n * n.gyr_n, n.acc_n * n.acc_n, n.acc_n * n.acc_n, n.acc_n * n.acc_n, n.gyr_n * n.gyr_n,
                         n.gyr_n * n.gyr_n, n.gyr_n * n.gyr_n, n.acc_w * n.acc_w, n.acc_w * n.acc_w, n.acc_w * n.acc_w,
                         n.gyr_w * n.gyr_w, n.gyr_w * n.gyr_w, n.gyr_w * n.gyr_w};
  double FJ[15][15], FP[15][15], NP[15][15];
  for (int i = 0; i < 15; ++i)
    for (int j = 0; j < 15; ++j) {
      double a = 0, b = 0;
      for (int k = 0; k < 15; ++k) {
        a += F(i, k) * p->jacobian[k][j];
        b += F(i, k) * p->covariance[k][j];
      }
      FJ[i][j] = a;
      FP[i][j] = b;
    }
  for (int i = 0; i < 15; ++i)
    for (int j = 0; j < 15; ++j) {
      double a = 0, b = 0;
      for (int k = 0; k < 15; ++k) a += FP[i][k] * F(j, k);
      for (int k = 0; k < 18; ++k) b += V(i, k) * nd[k] * V(j, k);
      NP[i][j] = a + b;
    }
  for (int i = 0; i < 15; ++i)
    for (int j = 0; j < 15; ++j) {
      p->jacobian[i][j] = FJ[i][j];
      p->covariance[i][j] = NP[i][j];
    }
  p->delta_p = result_p;
  p->delta_v = result_v;
  p->delta_q = qnormalized(result_q);
  p->sum_dt += dt;
  p->acc_0 = acc_1;
  p->gyr_0 = gyr_1;
}

struct NavState {  // pose, velocity, biases of one key (the reference's X(k), V(k), B(k))
  V3d p{0, 0, 0};
  Quatd q{1, 0, 0, 0};
  V3d v{0, 0, 0};
  V3d ba{0, 0, 0}, bg{0, 0, 0};
};

// State at the end of the pre-integrated interval (what the front end uses as pose prediction, LTB:188-199).
inline NavState imu_predict(const NavState& i, const Preintegration& m, const V3d& G) {
  NavState j = i;
  const double T = m.sum_dt;
  j.p = i.p + scale(T, i.v) - scale(0.5 * T * T, G) + rotate(i.q, m.delta_p);
  j.v = i.v - scale(T, G) + rotate(i.q, m.delta_v);
  j.q = qnormalized(qmul(i.q, m.delta_q));
  return j;
}

// The 15 residuals (order p, theta, v, ba, bg) of integration_base.h:267-301, and their Jacobian (15 x 15) w.r.t. the
// local parameters of state j. State i's biases may differ from the linearisation biases m.ba / m.bg: the deltas then take
// the first-order correction of :283-290 (corrected_delta_p / _v, corrected_delta_q = delta_q * deltaQ(J_q,bg dbg), whose
// Eigen inverse() divides the conjugate by the squared norm). Sums run left to right. At the linearisation biases the raw
// deltas are used as they are.
inline void imu_residual(const NavState& si, const NavState& sj, const Preintegration& m, const V3d& G, double* r,
                         double (*J)[15]) {
  const double T = m.sum_dt;
  const V3d dba = si.ba - m.ba, dbg = si.bg - m.bg;
  V3d dp = m.delta_p, dv = m.delta_v;
  Quatd dq_inv = conj(m.delta_q);
  if (!(dba.x == 0 && dba.y == 0 && dba.z == 0 && dbg.x == 0 && dbg.y == 0 && dbg.z == 0)) {
    auto blk = [&](int r0, int c0, const V3d& d) {
      const double(*Jm)[15] = m.jacobian;
      return V3d{Jm[r0][c0] * d.x + Jm[r0][c0 + 1] * d.y + Jm[r0][c0 + 2] * d.z,
                 Jm[r0 + 1][c0] * d.x + Jm[r0 + 1][c0 + 1] * d.y + Jm[r0 + 1][c0 + 2] * d.z,
                 Jm[r0 + 2][c0] * d.x + Jm[r0 + 2][c0 + 1] * d.y + Jm[r0 + 2][c0 + 2] * d.z};
    };
    dp = m.delta_p + blk(0, 9, dba) + blk(0, 12, dbg);
    dv = m.delta_v + blk(6, 9, dba) + blk(6, 12, dbg);
    const V3d th = blk(3, 12, dbg);
    const Quatd c = qmul(m.delta_q, Quatd{1.0, 0.5 * th.x, 0.5 * th.y, 0.5 * th.z});
    const double n2 = (c.x * c.x + c.y * c.y) + (c.z * c.z + c.w * c.w);
    dq_inv = {c.w / n2, -c.x / n2, -c.y / n2, -c.z / n2};
  }
  const Quatd qi_inv = conj(si.q);
  const V3d rp = rotate(qi_inv, scale(0.5 * T * T, G) + sj.p - si.p - scale(T, si.v)) - dp;
  const Quatd A = qmul(dq_inv, qi_inv);
  const Quatd e = qmul(A, sj.q);
  const V3d rv = rotate(qi_inv, scale(T, G) + sj.v - si.v) - dv;
  r[0] = rp.x; r[1] = rp.y; r[2] = rp.z;
  r[3] = 2 * e.x; r[4] = 2 * e.y; r[5] = 2 * e.z;
  r[6] = rv.x; r[7] = rv.y; r[8] = rv.z;
  r[9] = sj.ba.x - si.ba.x; r[10] = sj.ba.y - si.ba.y; r[11] = sj.ba.z - si.ba.z;
  r[12] = sj.bg.x - si.bg.x; r[13] = sj.bg.y - si.bg.y; r[14] = sj.bg.z - si.bg.z;
  if (!J) return;
  for (int a = 0; a < 15; ++a)
    for (int b = 0; b < 15; ++b) J[a][b] = 0;
  double Rit[3][3];
  to_rotation_matrix(qi_inv, Rit);
  for (int a = 0; a < 3; ++a)
    for (int b = 0; b < 3; ++b) {
      J[a][b] = Rit[a][b];          // d r_p / d dp
      J[6 + a][6 + b] = Rit[a][b];  // d r_v / d dv
    }
  // d r_theta / d dtheta: q_j <- (1, d) (x) q_j  =>  2 vec(A (x) (0, d) (x) q_j), column by column
  for (int b = 0; b < 3; ++b) {
    Quatd d{0, b == 0 ? 1.0 : 0.0, b == 1 ? 1.0 : 0.0, b == 2 ? 1.0 : 0.0};
    const Quatd c = qmul(qmul(A, d), sj.q);
    J[3][3 + b] = 2 * c.x; J[4][3 + b] = 2 * c.y; J[5][3 + b] = 2 * c.z;
  }
  for (int a = 0; a < 6; ++a) J[9 + a][9 + a] = 1.0;
}

// L with Sigma = L L^T (lower). Returns false if Sigma is not positive definite.
inline bool cholesky15(const double S[15][15], double L[15][15]) {
  for (int i = 0; i < 15; ++i)
    for (int j = 0; j < 15; ++j) L[i][j] = 0;
  for (int i = 0; i < 15; ++i)
    for (int j = 0; j <= i; ++j) {
      double s = S[i][j];
      for (int k = 0; k < j; ++k) s -= L[i][k] * L[j][k];
      if (i == j) {
        if (!(s > 0)) return false;
        L[i][i] = std::sqrt(s);
      } else {
        L[i][j] = s / L[j][j];
      }
    }
  return true;
}

// Scan-match problem over the 15 local parameters of state j with state i fixed (see the header, (3)).
// Ambient vector: p(3) q(4) v(3) ba(3) bg(3) = 16.
class FusedProblem {
 public:
  FusedProblem(const CeresMatcherOptions& opt, const V3d& target_translation, const NavState& state_i,
               const NavState& initial_j, const Preintegration& m, const V3d& G, double imu_weight,
               const std::vector<CloudAndGrid>& pairs)
      : scan_(opt, target_translation, Rigid3d{initial_j.p, initial_j.q}, pairs), si_(state_i), m_(m), G_(G),
        imu_weight_(imu_weight) {
    ok_ = cholesky15(m.covariance, L_);
  }
  bool ok() const { return ok_; }
  int num_residuals() const { return scan_.num_residuals() + 15; }
  int num_local() const { return 15; }
  int num_ambient() const { return 16; }

  static NavState unpack(const double* x) {
    NavState s;
    s.p = {x[0], x[1], x[2]}; s.q = {x[3], x[4], x[5], x[6]}; s.v = {x[7], x[8], x[9]};
    s.ba = {x[10], x[11], x[12]}; s.bg = {x[13], x[14], x[15]};
    return s;
  }
  static void pack(const NavState& s, double* x) {
    x[0] = s.p.x; x[1] = s.p.y; x[2] = s.p.z; x[3] = s.q.w; x[4] = s.q.x; x[5] = s.q.y; x[6] = s.q.z;
    x[7] = s.v.x; x[8] = s.v.y; x[9] = s.v.z; x[10] = s.ba.x; x[11] = s.ba.y; x[12] = s.ba.z;
    x[13] = s.bg.x; x[14] = s.bg.y; x[15] = s.bg.z;
  }

  void Evaluate(const double* x, double* residuals, double* J) const {
    const int ms = scan_.num_residuals();
    std::vector<double> J6;
    if (J) J6.resize((size_t)ms * 6);
    scan_.Evaluate(x, residuals, J ? J6.data() : nullptr);
    if (J) {
      for (int i = 0; i < ms; ++i) {
        double* row = J + (size_t)i * 15;
        for (int c = 0; c < 15; ++c) row[c] = c < 6 ? J6[(size_t)i * 6 + c] : 0.0;
      }
    }
    double r[15], Ji[15][15];
    imu_residual(si_, unpack(x), m_, G_, r, J ? Ji : nullptr);
    // whiten with L^-1 (forward substitution): ||L^-1 r||^2 = r^T Sigma^-1 r
    auto solve_lower = [&](double* v) {
      for (int i = 0; i < 15; ++i) {
        double s = v[i];
        for (int k = 0; k < i; ++k) s -= L_[i][k] * v[k];
        v[i] = s / L_[i][i];
      }
    };
    solve_lower(r);
    for (int a = 0; a < 15; ++a) residuals[ms + a] = imu_weight_ * r[a];
    if (J) {
      for (int c = 0; c < 15; ++c) {
        double col[15];
        for (int a = 0; a < 15; ++a) col[a] = Ji[a][c];
        solve_lower(col);
        for (int a = 0; a < 15; ++a) J[(size_t)(ms + a) * 15 + c] = imu_weight_ * col[a];
      }
    }
  }

  void Plus(const double* x, const double* delta, double* out) const {
    scan_.Plus(x, delta, out);  // p += d[0:3]; q <- dq(d[3:6]) (x) q
    for (int i = 0; i < 9; ++i) out[7 + i] = x[7 + i] + delta[6 + i];
  }

 private:
  ScanMatchProblem scan_;
  NavState si_;
  Preintegration m_;
  V3d G_;
  double imu_weight_;
  double L_[15][15];
  bool ok_ = false;
};

inline bool fused_scan_match(const CeresMatcherOptions& opt, const V3d& target_translation, const NavState& state_i,
                             const NavState& initial_j, const Preintegration& m, const V3d& G, double imu_weight,
                             const std::vector<CloudAndGrid>& pairs, NavState* state_j, SolveSummary* summary) {
  FusedProblem problem(opt, target_translation, state_i, initial_j, m, G, imu_weight, pairs);
  if (!problem.ok()) return false;
  double x[16];
  FusedProblem::pack(initial_j, x);
  solve_trust_region(problem, opt.use_nonmonotonic_steps, opt.max_num_iterations, x, summary);
  *state_j = FusedProblem::unpack(x);
  return true;
}

}  // namespace orc
