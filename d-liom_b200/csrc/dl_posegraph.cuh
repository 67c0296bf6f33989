// Building blocks of the block-sparse pose-graph solve (dl_posegraph_sparse.cu):
//   - forward-mode duals over the 14 ambient parameters of one SpaCostFunction3D and the residual itself,
//   - the one-CTA dense Cholesky factor and triangular solves,
//   - the Ceres 1.13 TrustRegionMinimizer state machine (LM, monotonic steps, pose_graph.lua's options) run on the host, with
//     the device evaluation and step behind callbacks (tests/schur_oracle.py mirrors the same state machine on the CPU).
#pragma once
#include <cmath>
#include <functional>

#include "dl_internal.cuh"

namespace dl {
namespace pg {

__host__ __device__ inline double lm_min_diag() { return 1e-6; }   // Ceres min / max_lm_diagonal
__host__ __device__ inline double lm_max_diag() { return 1e32; }

// forward-mode dual number over the 14 ambient parameters of a constraint: q_i (4), t_i (3), q_j (4), t_j (3)
struct Dual {
  double a;
  double v[14];
};
__device__ __forceinline__ Dual dconst(double s) { Dual d; d.a = s; for (int i = 0; i < 14; ++i) d.v[i] = 0.; return d; }
__device__ __forceinline__ Dual dvar(double s, int k) { Dual d = dconst(s); d.v[k] = 1.; return d; }
__device__ __forceinline__ Dual operator+(const Dual& f, const Dual& g) { Dual h; h.a = f.a + g.a; for (int i = 0; i < 14; ++i) h.v[i] = f.v[i] + g.v[i]; return h; }
__device__ __forceinline__ Dual operator-(const Dual& f, const Dual& g) { Dual h; h.a = f.a - g.a; for (int i = 0; i < 14; ++i) h.v[i] = f.v[i] - g.v[i]; return h; }
__device__ __forceinline__ Dual operator*(const Dual& f, const Dual& g) { Dual h; h.a = f.a * g.a; for (int i = 0; i < 14; ++i) h.v[i] = f.a * g.v[i] + f.v[i] * g.a; return h; }
__device__ __forceinline__ Dual operator/(const Dual& f, const Dual& g) {
  const double gi = 1.0 / g.a, fg = f.a * gi;
  Dual h; h.a = fg; for (int i = 0; i < 14; ++i) h.v[i] = (f.v[i] - fg * g.v[i]) * gi; return h;
}
__device__ __forceinline__ Dual operator*(double s, const Dual& f) { Dual h; h.a = s * f.a; for (int i = 0; i < 14; ++i) h.v[i] = s * f.v[i]; return h; }
__device__ __forceinline__ Dual dneg(const Dual& f) { return -1.0 * f; }
__device__ __forceinline__ Dual dsqrt(const Dual& f) { const double r = sqrt(f.a), d = 1.0 / (2.0 * r); Dual h; h.a = r; for (int i = 0; i < 14; ++i) h.v[i] = f.v[i] * d; return h; }
__device__ __forceinline__ Dual dsin(const Dual& f) { const double c = cos(f.a); Dual h; h.a = sin(f.a); for (int i = 0; i < 14; ++i) h.v[i] = c * f.v[i]; return h; }
__device__ __forceinline__ Dual datan2(const Dual& g, const Dual& f) {
  const double d = 1.0 / (f.a * f.a + g.a * g.a);
  Dual h; h.a = atan2(g.a, f.a); for (int i = 0; i < 14; ++i) h.v[i] = d * (f.a * g.v[i] - g.a * f.v[i]); return h;
}
__device__ inline void dq_mul(const Dual a[4], const Dual b[4], Dual out[4]) {
  out[0] = a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3];
  out[1] = a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2];
  out[2] = a[0] * b[2] + a[2] * b[0] + a[3] * b[1] - a[1] * b[3];
  out[3] = a[0] * b[3] + a[3] * b[0] + a[1] * b[2] - a[2] * b[1];
}
__device__ inline void dq_rotate(const Dual q[4], const Dual v[3], Dual out[3]) {  // v + w uv + q x uv, uv = 2 q x v
  Dual uv[3] = {q[2] * v[2] - q[3] * v[1], q[3] * v[0] - q[1] * v[2], q[1] * v[1] - q[2] * v[0]};
  for (int i = 0; i < 3; ++i) uv[i] = uv[i] + uv[i];
  out[0] = v[0] + q[0] * uv[0] + (q[2] * uv[2] - q[3] * uv[1]);
  out[1] = v[1] + q[0] * uv[1] + (q[3] * uv[0] - q[1] * uv[2]);
  out[2] = v[2] + q[0] * uv[2] + (q[1] * uv[1] - q[2] * uv[0]);
}
__device__ inline void dq_to_angle_axis(const Dual q[4], Dual out[3]) {  // transform.h:59-83
  const Dual n = dsqrt(q[1] * q[1] + q[2] * q[2] + q[3] * q[3] + q[0] * q[0]);
  Dual w = q[0] / n, x = q[1] / n, y = q[2] / n, z = q[3] / n;
  if (w.a < 0.) { w = dneg(w); x = dneg(x); y = dneg(y); z = dneg(z); }
  const Dual vec_norm = dsqrt(x * x + y * y + z * z);
  const Dual angle = 2.0 * datan2(vec_norm, w);
  const Dual scale = angle.a < 1e-7 ? dconst(2.) : angle / dsin(0.5 * angle);
  out[0] = scale * x; out[1] = scale * y; out[2] = scale * z;
}

// SpaCostFunction3D (c_i = submap, c_j = node): h = c_i^-1 c_j; e = scale(zbar - h). Derivatives with respect to
// (q_i, t_i, q_j, t_j) in the duals' 14 slots.
__device__ inline void spa_residual(const dl_spa_constraint& c, const double* qi, const double* ti, const double* qj,
                                    const double* tj, Dual e[6]) {
  Dual jqi[4], jti[3], jqj[4], jtj[3];
  for (int k = 0; k < 4; ++k) { jqi[k] = dvar(qi[k], k); jqj[k] = dvar(qj[k], 7 + k); }
  for (int k = 0; k < 3; ++k) { jti[k] = dvar(ti[k], 4 + k); jtj[k] = dvar(tj[k], 11 + k); }
  const Dual ri_inv[4] = {jqi[0], dneg(jqi[1]), dneg(jqi[2]), dneg(jqi[3])};
  const Dual delta[3] = {jtj[0] - jti[0], jtj[1] - jti[1], jtj[2] - jti[2]};
  Dual h_t[3];
  dq_rotate(ri_inv, delta, h_t);
  const Dual qj_conj[4] = {jqj[0], dneg(jqj[1]), dneg(jqj[2]), dneg(jqj[3])};
  Dual h_r_inv[4], prod[4], aa[3];
  dq_mul(qj_conj, jqi, h_r_inv);
  const Dual z[4] = {dconst(c.zbar[3]), dconst(c.zbar[4]), dconst(c.zbar[5]), dconst(c.zbar[6])};
  dq_mul(h_r_inv, z, prod);
  dq_to_angle_axis(prod, aa);
  for (int k = 0; k < 3; ++k) {
    e[k] = c.translation_weight * (dconst(c.zbar[k]) - h_t[k]);
    e[3 + k] = c.rotation_weight * aa[k];
  }
}

// One CTA: Cholesky A = U^T U of the row-major n x n matrix A, left-looking by columns of U; U overwrites the UPPER triangle, so
// that for a fixed k the threads (one per column i) read consecutive addresses U[k][i] and U[k][j] is a broadcast: coalesced,
// unlike rows of L. Only the upper triangle of A is read. ok_s: a __shared__ flag, 0 on return if a pivot was not positive.
__device__ inline void cta_cholesky_factor(double* A, int n, int* ok_s) {
  const int tid = threadIdx.x, nt = blockDim.x;
  if (tid == 0) *ok_s = 1;
  __syncthreads();
  for (int j = 0; j < n; ++j) {
    for (int i = j + tid; i < n; i += nt) {  // s_i = A[j][i] - sum_k U[k][i] U[k][j], the diagonal (i == j) included
      double s = A[(size_t)j * n + i];
      for (int k = 0; k < j; ++k) s -= A[(size_t)k * n + i] * A[(size_t)k * n + j];
      A[(size_t)j * n + i] = s;
    }
    __syncthreads();
    if (tid == 0) {
      const double s = A[(size_t)j * n + j];
      if (!(s > 0.)) *ok_s = 0; else A[(size_t)j * n + j] = sqrt(s);
    }
    __syncthreads();
    if (!*ok_s) break;
    const double djj = A[(size_t)j * n + j];
    for (int i = j + 1 + tid; i < n; i += nt) A[(size_t)j * n + i] /= djj;
    __syncthreads();
  }
}
// One CTA: y <- (U^T U)^-1 y with U from cta_cholesky_factor; the triangular solves as parallel axpys: U^T z = y (row i of U is
// contiguous), then U y = z.
__device__ inline void cta_cholesky_solve(const double* U, int n, double* y) {
  const int tid = threadIdx.x, nt = blockDim.x;
  for (int i = 0; i < n; ++i) {
    if (tid == 0) y[i] /= U[(size_t)i * n + i];
    __syncthreads();
    const double zi = y[i];
    const double* row = U + (size_t)i * n;
    for (int j = i + 1 + tid; j < n; j += nt) y[j] -= row[j] * zi;
    __syncthreads();
  }
  for (int i = n - 1; i >= 0; --i) {
    if (tid == 0) y[i] /= U[(size_t)i * n + i];
    __syncthreads();
    const double yi = y[i];
    for (int j = tid; j < i; j += nt) y[j] -= U[(size_t)j * n + i] * yi;
    __syncthreads();
  }
}

// ---- Ceres 1.13 TrustRegionMinimizer as pose_graph.lua runs it (LM, monotonic steps), scalars on the host. The solver keeps the
// current point, the candidate and the best point; the driver only sees costs, norms and the step's validity. The minimised
// program holds the parameters of the poses that are neither frozen nor unreferenced (no constraint refers to them), so x, ||x||
// and the parameter tolerance built from it cover those poses only.
struct LmCallbacks {
  // evaluate at the starting point: cost (the minimised program's: fixed cost excluded), projected-gradient max norm, ||x||
  std::function<int(double* cost, double* gradient_max_norm, double* x_norm)> initial;
  std::function<int()> save_best;  // the current point is the best so far
  // solve for the step at the current point: (S H S + D / radius) y = S g, D refreshed unless reuse_diagonal, the Jacobi scale S
  // computed when compute_scale (first step only). valid: factorisations succeeded, the step is finite and the model decreases.
  std::function<int(double radius, bool reuse_diagonal, bool compute_scale, bool* valid, double* model_cost_change)> step;
  // candidate = Plus(x, step): its cost (with the normal equations there, for when it is accepted) and ||x - candidate||
  std::function<int(double* cost, double* step_norm)> candidate;
  // make the candidate the current point: projected-gradient max norm and ||x|| there
  std::function<int(double* gradient_max_norm, double* x_norm)> accept;
};

inline int run_trust_region(const LmCallbacks& cb, int max_iter, dl_solve_summary* out) {
  const double kMinRelDecrease = 1e-3, kFunctionTol = 1e-6, kGradientTol = 1e-10, kParameterTol = 1e-8, kMinRadius = 1e-32, kMaxRadius = 1e16;
  double cur_cost = 0, gmax = 0, x_norm = 0;
  DL_TRY(cb.initial(&cur_cost, &gmax, &x_norm));
  dl_solve_summary sum{};
  sum.initial_cost = sum.final_cost = cur_cost;
  sum.termination = 1;
  sum.num_evaluations = 1;
  double radius = 1e4, decrease_factor = 2.0, minimum_cost = 1.7976931348623157e308, last_cost = cur_cost;
  bool reuse_diagonal = false, last_successful = true, first_step = true;
  int iteration = 0, num_invalid = 0;
  bool stop = false;
  while (!stop) {
    if (last_successful) {
      ++sum.num_successful_steps;
      if (cur_cost < minimum_cost) {
        minimum_cost = cur_cost;
        DL_TRY(cb.save_best());
      }
    } else {
      ++sum.num_unsuccessful_steps;
    }
    ++sum.num_iterations;
    sum.final_cost = std::fmin(sum.final_cost, last_cost);
    if (iteration >= max_iter) { sum.termination = 1; break; }
    if (last_successful && gmax <= kGradientTol) { sum.termination = 0; break; }
    if (radius <= kMinRadius) { sum.termination = 0; break; }
    bool have_step = false;
    double model_cost_change = 0;
    while (!have_step) {
      ++iteration;
      bool valid = false;
      double mcc = 0;
      DL_TRY(cb.step(radius, reuse_diagonal, first_step, &valid, &mcc));
      first_step = false;
      reuse_diagonal = true;
      if (valid) {
        model_cost_change = mcc;
        have_step = true;
        num_invalid = 0;
        break;
      }
      if (++num_invalid >= 5) { sum.termination = 2; stop = true; break; }
      radius *= 0.5;
      last_successful = false;
      last_cost = cur_cost;
      ++sum.num_unsuccessful_steps;
      ++sum.num_iterations;
      if (iteration >= max_iter) { sum.termination = 1; stop = true; break; }
      if (radius <= kMinRadius) { sum.termination = 0; stop = true; break; }
    }
    if (stop) break;
    double cand_cost = 0, step_norm = 0;
    DL_TRY(cb.candidate(&cand_cost, &step_norm));  // candidate cost + speculative normal equations in one pass
    ++sum.num_evaluations;
    if (!std::isfinite(cand_cost)) cand_cost = 1.7976931348623157e308;
    if (step_norm <= kParameterTol * (x_norm + kParameterTol)) { sum.termination = 0; break; }
    if (std::fabs(cur_cost - cand_cost) <= kFunctionTol * cur_cost) { sum.termination = 0; break; }
    const double relative_decrease = (cur_cost - cand_cost) / model_cost_change;  // monotonic steps only (pose_graph.lua)
    if (relative_decrease > kMinRelDecrease) {
      cur_cost = cand_cost;
      DL_TRY(cb.accept(&gmax, &x_norm));
      last_successful = true;
      last_cost = cand_cost;
      const double t = 2.0 * relative_decrease - 1.0;
      radius = std::fmin(kMaxRadius, radius / std::fmax(1.0 / 3.0, 1.0 - t * t * t));
      decrease_factor = 2.0;
      reuse_diagonal = false;
    } else {
      last_successful = false;
      last_cost = cand_cost;
      radius /= decrease_factor;
      decrease_factor *= 2.0;
      reuse_diagonal = true;
    }
  }
  *out = sum;
  return DL_OK;
}

}  // namespace pg
}  // namespace dl
