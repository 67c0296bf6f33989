// TEST INFRASTRUCTURE — CPU oracle (see orc_math.h header).
//
// The sparse pose adjustment the fork's OptimizationProblem3D::Solve reduces to (SURVEY 8f-4): in this tree the IMU
// acceleration / rotation terms and the consecutive-node terms are commented out (optimization_problem_3d.cc:350-489) and loop
// closures get a TrivialLoss (:336-338), so with no landmarks and no fixed-frame data the problem is
//   parameters  one CeresPose (rotation block 4, translation block 3) per submap and per node (:283-329);
//               first submap: translation constant, rotation with ConstantYawQuaternionPlus (4 -> 2,
//               mapping/internal/3d/rotation_parameterization.h:43-64); every other rotation QuaternionParameterization
//               (4 -> 3); translations free (fix_z: SubsetParameterization of index 2)
//   residuals   SpaCostFunction3D per constraint (cost_functions/spa_cost_function_3d.h:35-58): ScaleError(
//               ComputeUnscaledError(zbar_ij, c_i, c_j)) (cost_helpers_impl.h:58-100) with
//               RotationQuaternionToAngleAxisVector (transform/transform.h:59-83), 6 per constraint, autodiff Jacobians
//   solver      ceres::Solve with pose_graph.lua's options (LM, 50 iterations, no non-monotonic steps); the linear solver
//               there is SPARSE_NORMAL_CHOLESKY: here the normal equations are formed and factored densely (default), or the
//               dense QR of the scan matcher's loop is used as a cross-check: the same LM step in exact arithmetic.
// Jets use one summation order for norms (x^2 + y^2 + z^2 + w^2 left to right) in both the double and the Jet instantiation;
// Eigen would pair the doubles differently (1 ulp). Pinned to the reference's own test of this function
// (optimization_problem_3d_test.cc:106-196, a statistical property) in tests/test_posegraph_oracle.py.
#pragma once
#include <cmath>
#include <vector>

#include "orc_math.h"
#include "orc_nls.h"

namespace orc {

template <int N>
struct JetN {
  double a = 0.;
  double v[N];
  JetN() { for (int i = 0; i < N; ++i) v[i] = 0.; }
  JetN(double s) : a(s) { for (int i = 0; i < N; ++i) v[i] = 0.; }  // NOLINT: implicit like ceres::Jet
  static JetN variable(double s, int k) { JetN j(s); j.v[k] = 1.; return j; }
};
#define ORC_JET_BIN(op, expr_a, expr_v)                                                         \
  template <int N> inline JetN<N> operator op(const JetN<N>& f, const JetN<N>& g) {              \
    JetN<N> h; h.a = expr_a; for (int i = 0; i < N; ++i) h.v[i] = expr_v; return h; }
ORC_JET_BIN(+, f.a + g.a, f.v[i] + g.v[i])
ORC_JET_BIN(-, f.a - g.a, f.v[i] - g.v[i])
ORC_JET_BIN(*, f.a * g.a, f.a * g.v[i] + f.v[i] * g.a)
#undef ORC_JET_BIN
template <int N> inline JetN<N> operator/(const JetN<N>& f, const JetN<N>& g) {
  const double gi = 1.0 / g.a, fg = f.a * gi;  // ceres/jet.h: h = f/g, dh = (df - h dg) / g
  JetN<N> h; h.a = fg; for (int i = 0; i < N; ++i) h.v[i] = (f.v[i] - fg * g.v[i]) * gi; return h;
}
template <int N> inline JetN<N> operator-(const JetN<N>& f) { JetN<N> h; h.a = -f.a; for (int i = 0; i < N; ++i) h.v[i] = -f.v[i]; return h; }
template <int N> inline JetN<N> operator*(double s, const JetN<N>& f) { return JetN<N>(s) * f; }
template <int N> inline JetN<N> operator*(const JetN<N>& f, double s) { return f * JetN<N>(s); }
template <int N> inline JetN<N> operator-(double s, const JetN<N>& f) { return JetN<N>(s) - f; }
template <int N> inline JetN<N> operator/(const JetN<N>& f, double s) { return f / JetN<N>(s); }
template <int N> inline bool operator<(const JetN<N>& f, double s) { return f.a < s; }
template <int N> inline JetN<N> jsqrt(const JetN<N>& f) { const double r = std::sqrt(f.a), d = 1.0 / (2.0 * r); JetN<N> h; h.a = r; for (int i = 0; i < N; ++i) h.v[i] = f.v[i] * d; return h; }
template <int N> inline JetN<N> jsin(const JetN<N>& f) { const double c = std::cos(f.a); JetN<N> h; h.a = std::sin(f.a); for (int i = 0; i < N; ++i) h.v[i] = c * f.v[i]; return h; }
template <int N> inline JetN<N> jatan2(const JetN<N>& g, const JetN<N>& f) {  // atan2(g, f): d = (f dg - g df) / (f^2 + g^2)
  const double d = 1.0 / (f.a * f.a + g.a * g.a);
  JetN<N> h; h.a = std::atan2(g.a, f.a); for (int i = 0; i < N; ++i) h.v[i] = d * (f.a * g.v[i] - g.a * f.v[i]); return h;
}
inline double jsqrt(double x) { return std::sqrt(x); }
inline double jsin(double x) { return std::sin(x); }
inline double jatan2(double y, double x) { return std::atan2(y, x); }
inline double jet_value(double x) { return x; }
template <int N> inline double jet_value(const JetN<N>& x) { return x.a; }

// transform::RotationQuaternionToAngleAxisVector (transform.h:59-83), q = (w, x, y, z)
template <typename T>
inline void quaternion_to_angle_axis(const T q[4], T out[3]) {
  const T n = jsqrt(q[1] * q[1] + q[2] * q[2] + q[3] * q[3] + q[0] * q[0]);
  T w = q[0] / n, x = q[1] / n, y = q[2] / n, z = q[3] / n;
  if (w < 0.) { w = -1. * w; x = -1. * x; y = -1. * y; z = -1. * z; }
  const T vec_norm = jsqrt(x * x + y * y + z * z);
  const T angle = 2. * jatan2(vec_norm, w);
  const T scale = angle < 1e-7 ? T(2.) : angle / jsin(angle / 2.);
  out[0] = scale * x; out[1] = scale * y; out[2] = scale * z;
}
template <typename T>
inline void quaternion_product(const T a[4], const T b[4], T out[4]) {  // Eigen's generic product, (w, x, y, z)
  out[0] = a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3];
  out[1] = a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2];
  out[2] = a[0] * b[2] + a[2] * b[0] + a[3] * b[1] - a[1] * b[3];
  out[3] = a[0] * b[3] + a[3] * b[0] + a[1] * b[2] - a[2] * b[1];
}
template <typename T>
inline void quaternion_rotate(const T q[4], const T v[3], T out[3]) {  // Eigen: v + w uv + q x uv, uv = 2 q x v
  T uv[3] = {q[2] * v[2] - q[3] * v[1], q[3] * v[0] - q[1] * v[2], q[1] * v[1] - q[2] * v[0]};
  for (int i = 0; i < 3; ++i) uv[i] = uv[i] + uv[i];
  out[0] = v[0] + q[0] * uv[0] + (q[2] * uv[2] - q[3] * uv[1]);
  out[1] = v[1] + q[0] * uv[1] + (q[3] * uv[0] - q[1] * uv[2]);
  out[2] = v[2] + q[0] * uv[2] + (q[1] * uv[1] - q[2] * uv[0]);
}

struct SpaConstraint {
  int submap, node;
  Rigid3d zbar_ij;
  double translation_weight, rotation_weight;
};

// SpaCostFunction3D::operator() : c_i = submap, c_j = node
template <typename T>
inline void spa_residual(const SpaConstraint& c, const T* qi, const T* ti, const T* qj, const T* tj, T* e) {
  const T r_i_inverse[4] = {qi[0], -qi[1], -qi[2], -qi[3]};
  const T delta[3] = {tj[0] - ti[0], tj[1] - ti[1], tj[2] - ti[2]};
  T h_translation[3];
  quaternion_rotate(r_i_inverse, delta, h_translation);
  const T qj_conj[4] = {qj[0], -qj[1], -qj[2], -qj[3]};
  T h_rotation_inverse[4], prod[4], aa[3];
  quaternion_product(qj_conj, qi, h_rotation_inverse);
  const T z[4] = {T(c.zbar_ij.q.w), T(c.zbar_ij.q.x), T(c.zbar_ij.q.y), T(c.zbar_ij.q.z)};
  quaternion_product(h_rotation_inverse, z, prod);
  quaternion_to_angle_axis(prod, aa);
  e[0] = (T(c.zbar_ij.t.x) - h_translation[0]) * c.translation_weight;
  e[1] = (T(c.zbar_ij.t.y) - h_translation[1]) * c.translation_weight;
  e[2] = (T(c.zbar_ij.t.z) - h_translation[2]) * c.translation_weight;
  for (int k = 0; k < 3; ++k) e[3 + k] = aa[k] * c.rotation_weight;
}

// The problem orc_nls.h's solve_trust_region drives. Only the poses some constraint refers to are in it: Ceres 1.13's
// Program::RemoveFixedBlocks drops parameter blocks no residual uses, so an unreferenced pose has no parameters, keeps its start
// value and does not enter ||x||. Ambient layout over the referenced poses in order: submap 0 rotation (4) [its translation is
// constant and lives outside], every other pose rotation (4), translation (3).
class PoseGraphProblem {
 public:
  PoseGraphProblem(int num_submaps, int num_nodes, const V3d& first_submap_translation, std::vector<SpaConstraint> constraints,
                   bool fix_z)
      : S_(num_submaps), N_(num_nodes), t0_(first_submap_translation), constraints_(std::move(constraints)), fix_z_(fix_z) {
    used_.assign(S_ + N_, false);
    for (const SpaConstraint& c : constraints_) used_[c.submap] = used_[pose_of_node(c.node)] = true;
    amb_.assign(S_ + N_ + 1, 0);
    loc_.assign(S_ + N_ + 1, 0);
    for (int p = 0; p < S_ + N_; ++p) {
      amb_[p + 1] = amb_[p] + (!used_[p] ? 0 : p == 0 ? 4 : 7);
      loc_[p + 1] = loc_[p] + (!used_[p] ? 0 : p == 0 ? 2 : 3 + translation_dof());
    }
  }

  int num_residuals() const { return 6 * (int)constraints_.size(); }
  int num_ambient() const { return amb_[S_ + N_]; }
  int translation_dof() const { return fix_z_ ? 2 : 3; }
  int num_local() const { return loc_[S_ + N_]; }
  bool used(int pose) const { return used_[pose]; }
  int rotation_offset(int pose) const { return amb_[pose]; }                                      // ambient
  int translation_offset(int pose) const { return amb_[pose] + 4; }                               // ambient, pose > 0
  int local_offset(int pose) const { return loc_[pose]; }
  int pose_of_node(int node) const { return S_ + node; }

  void Plus(const double* x, const double* delta, double* out) const {
    for (int p = 0; p < S_ + N_; ++p) {
      if (!used_[p]) continue;
      const double* q = x + rotation_offset(p);
      const double* d = delta + local_offset(p);
      double* o = out + rotation_offset(p);
      if (p == 0) {  // ConstantYawQuaternionPlus: x * (cos|d|, sin|d|/|d| d0, sin|d|/|d| d1, 0)
        const double n = std::sqrt(d[0] * d[0] + d[1] * d[1]);
        const double s = n < 1e-6 ? 1. : std::sin(n) / n;
        const double qd[4] = {n < 1e-6 ? 1. : std::cos(n), s * d[0], s * d[1], 0.};
        quaternion_product(q, qd, o);
      } else {  // ceres::QuaternionParameterization: (cos|d|, sin|d|/|d| d) * x, identity for d = 0
        const double n = std::sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
        if (n > 0.) {
          const double s = std::sin(n) / n;
          const double qd[4] = {std::cos(n), s * d[0], s * d[1], s * d[2]};
          quaternion_product(qd, q, o);
        } else {
          for (int k = 0; k < 4; ++k) o[k] = q[k];
        }
        const double* t = x + translation_offset(p);
        double* ot = out + translation_offset(p);
        for (int k = 0; k < 3; ++k) ot[k] = t[k] + (k < translation_dof() ? d[3 + k] : 0.);
      }
    }
  }

  // residuals (6 per constraint) and the local Jacobian (row-major, num_residuals x num_local)
  void Evaluate(const double* x, double* residuals, double* jacobian) const {
    using J = JetN<14>;
    const int n = num_local();
    if (jacobian) std::fill(jacobian, jacobian + (size_t)num_residuals() * n, 0.);
    for (size_t ci = 0; ci < constraints_.size(); ++ci) {
      const SpaConstraint& c = constraints_[ci];
      const int pi = c.submap, pj = pose_of_node(c.node);
      const double* qi = x + rotation_offset(pi);
      const double ti_const[3] = {t0_.x, t0_.y, t0_.z};
      const double* ti = pi == 0 ? ti_const : x + translation_offset(pi);
      const double* qj = x + rotation_offset(pj);
      const double* tj = x + translation_offset(pj);
      J jqi[4], jti[3], jqj[4], jtj[3], e[6];
      for (int k = 0; k < 4; ++k) { jqi[k] = J::variable(qi[k], k); jqj[k] = J::variable(qj[k], 7 + k); }
      for (int k = 0; k < 3; ++k) { jti[k] = J::variable(ti[k], 4 + k); jtj[k] = J::variable(tj[k], 11 + k); }
      spa_residual(c, jqi, jti, jqj, jtj, e);
      for (int r = 0; r < 6; ++r) residuals[6 * ci + r] = e[r].a;
      if (!jacobian) continue;
      for (int r = 0; r < 6; ++r) {
        double* row = jacobian + (6 * ci + r) * (size_t)n;
        accumulate_rotation(row, pi, qi, e[r].v + 0);
        if (pi != 0) accumulate_translation(row, pi, e[r].v + 4);
        accumulate_rotation(row, pj, qj, e[r].v + 7);
        accumulate_translation(row, pj, e[r].v + 11);
      }
    }
  }

 private:
  // row[local] += d e / d q (1 x 4) * plus-Jacobian (4 x 2 or 4 x 3) at delta = 0
  void accumulate_rotation(double* row, int pose, const double* q, const double* de_dq) const {
    double* out = row + local_offset(pose);
    const double w = q[0], x = q[1], y = q[2], z = q[3];
    if (pose == 0) {  // d (q * (1, d0, d1, 0)) / d d0 = q * (0, 1, 0, 0), / d d1 = q * (0, 0, 1, 0)
      const double c0[4] = {-x, w, z, -y}, c1[4] = {-y, -z, w, x};
      for (int k = 0; k < 4; ++k) { out[0] += de_dq[k] * c0[k]; out[1] += de_dq[k] * c1[k]; }
    } else {  // QuaternionParameterization::ComputeJacobian
      const double j[4][3] = {{-x, -y, -z}, {w, z, -y}, {-z, w, x}, {y, -x, w}};
      for (int k = 0; k < 4; ++k)
        for (int a = 0; a < 3; ++a) out[a] += de_dq[k] * j[k][a];
    }
  }
  void accumulate_translation(double* row, int pose, const double* de_dt) const {
    double* out = row + local_offset(pose) + 3;
    for (int k = 0; k < translation_dof(); ++k) out[k] += de_dt[k];
  }

  int S_, N_;
  V3d t0_;
  std::vector<SpaConstraint> constraints_;
  bool fix_z_;
  std::vector<bool> used_;
  std::vector<int> amb_, loc_;  // per pose: ambient / local offsets (prefix sums over the referenced poses)
};

// OptimizationProblem3D::Solve for the SPA-only problem. poses: S submaps then N nodes, 7 doubles each (t xyz, q wxyz), in-out.
inline void solve_pose_graph(int num_submaps, int num_nodes, double* poses7, const std::vector<SpaConstraint>& constraints,
                             bool fix_z, int max_num_iterations, SolveSummary* summary,
                             LinearSolver linear_solver = kNormalCholesky) {
  PoseGraphProblem problem(num_submaps, num_nodes, V3d{poses7[0], poses7[1], poses7[2]}, constraints, fix_z);
  std::vector<double> x(problem.num_ambient());
  for (int p = 0; p < num_submaps + num_nodes; ++p) {
    if (!problem.used(p)) continue;
    const double* s = poses7 + 7 * p;
    double* q = x.data() + problem.rotation_offset(p);
    q[0] = s[3]; q[1] = s[4]; q[2] = s[5]; q[3] = s[6];
    if (p > 0) {
      double* t = x.data() + problem.translation_offset(p);
      t[0] = s[0]; t[1] = s[1]; t[2] = s[2];
    }
  }
  solve_trust_region(problem, /*use_nonmonotonic_steps=*/false, max_num_iterations, x.data(), summary, linear_solver);
  for (int p = 0; p < num_submaps + num_nodes; ++p) {
    if (!problem.used(p)) continue;  // not in the program: unchanged
    double* s = poses7 + 7 * p;
    const double* q = x.data() + problem.rotation_offset(p);
    s[3] = q[0]; s[4] = q[1]; s[5] = q[2]; s[6] = q[3];
    if (p > 0) {
      const double* t = x.data() + problem.translation_offset(p);
      s[0] = t[0]; s[1] = t[1]; s[2] = t[2];
    }
  }
}

}  // namespace orc
