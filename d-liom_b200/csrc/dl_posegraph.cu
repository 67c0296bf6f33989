// Sparse pose adjustment on the device, with the normal equations reduced over NCCL (SURVEY 8f-4, VERDICT "missing" 2).
//
// Replaces OptimizationProblem3D::Solve as this fork runs it (C/mapping/internal/optimization/optimization_problem_3d.cc:259-589):
// the IMU / consecutive-node terms are commented out there (:350-489) and loop closures get a TrivialLoss (:336-338), so the
// problem is pure SPA — one CeresPose per submap and node (:283-329; first submap: constant translation + ConstantYawQuaternionPlus,
// C/mapping/internal/3d/rotation_parameterization.h:43-64; all others QuaternionParameterization; fix_z = SubsetParameterization),
// one SpaCostFunction3D per constraint (cost_functions/spa_cost_function_3d.h:35-58, cost_helpers_impl.h:58-100,
// RotationQuaternionToAngleAxisVector transform.h:59-83), ceres LM with pose_graph.lua's options.
//
// Multi-GPU shape (BASELINE configs[4], "loop-closure/global constraint reduction over NCCL"): the CONSTRAINTS are sharded —
// every rank holds the constraints it found (dl_constraint_search_exchange's shard) — and the pose variables are replicated.
// Per LM evaluation each rank forms J^T J / J^T r / cost of ITS constraints on its device (one thread per constraint, forward-mode
// duals for the 6 x 14 ambient Jacobian, projected through the parameterisations, scattered with fp64 atomics), then ONE
// ncclAllReduce(sum, fp64) of the (n^2 + n + 1)-double block gives every rank the same global normal equations, and every rank
// takes the same trust-region step (dense Cholesky of S H S + D / r by one CTA). NCCL returns bit-identical sums on all ranks, so
// the replicas cannot drift apart.
// Size: dense n x n normal equations, n = 2 + (3 + tdof)(poses - 1) <= kMaxLocal; whole trajectories: dl_posegraph_sparse.cu.
#include <cmath>
#include <cstring>
#include <vector>

#include "dl_posegraph.cuh"

namespace dl {
namespace {
using namespace pg;

constexpr int kMaxLocal = 3072;

struct GraphDims {
  int S, N, tdof;
  __host__ __device__ int poses() const { return S + N; }
  __host__ __device__ int num_local() const { return 2 + (3 + tdof) * (S + N - 1); }
  __host__ __device__ int num_ambient() const { return 4 + 7 * (S + N - 1); }
  __host__ __device__ int rot(int p) const { return p == 0 ? 0 : 4 + 7 * (p - 1); }
  __host__ __device__ int trans(int p) const { return 4 + 7 * (p - 1) + 4; }
  __host__ __device__ int loc(int p) const { return p == 0 ? 0 : 2 + (3 + tdof) * (p - 1); }
};

// One thread per constraint: residuals (6), ambient Jacobian (6 x 14) by duals, projection to the local parameters, and the
// scatter of J^T J, J^T r, r^T r into the dense system.
__global__ void spa_evaluate_kernel(GraphDims d, const double* __restrict__ x, const double* __restrict__ t0,
                                    const dl_spa_constraint* __restrict__ constraints, int num_constraints, double* H, double* g,
                                    double* cost2, int with_jacobian) {
  const int ci = blockIdx.x * blockDim.x + threadIdx.x;
  if (ci >= num_constraints) return;
  const dl_spa_constraint c = constraints[ci];
  const int pi = c.submap, pj = d.S + c.node;
  const double* qi = x + d.rot(pi);
  const double* ti = pi == 0 ? t0 : x + d.trans(pi);
  const double* qj = x + d.rot(pj);
  const double* tj = x + d.trans(pj);
  Dual e[6];
  spa_residual(c, qi, ti, qj, tj, e);
  double c2 = 0;
  for (int r = 0; r < 6; ++r) c2 += e[r].a * e[r].a;
  atomicAdd(cost2, c2);
  if (!with_jacobian) return;
  // local Jacobian: columns [loc(pi), ...) and [loc(pj), ...)
  const int ni = pi == 0 ? 2 : 3 + d.tdof, nj = 3 + d.tdof;
  double J[6][12];
  for (int r = 0; r < 6; ++r) {
    double* row = J[r];
    for (int k = 0; k < 12; ++k) row[k] = 0.;
    {
      const double w = qi[0], xx = qi[1], y = qi[2], zq = qi[3];
      const double* de = e[r].v;
      if (pi == 0) {  // ConstantYawQuaternionPlus: d (q * (1, d0, d1, 0)) / d d0 = q * (0,1,0,0), / d d1 = q * (0,0,1,0)
        const double c0[4] = {-xx, w, zq, -y}, c1[4] = {-y, -zq, w, xx};
        for (int k = 0; k < 4; ++k) { row[0] += de[k] * c0[k]; row[1] += de[k] * c1[k]; }
      } else {        // QuaternionParameterization::ComputeJacobian
        const double jj[4][3] = {{-xx, -y, -zq}, {w, zq, -y}, {-zq, w, xx}, {y, -xx, w}};
        for (int k = 0; k < 4; ++k)
          for (int a = 0; a < 3; ++a) row[a] += de[k] * jj[k][a];
        for (int k = 0; k < d.tdof; ++k) row[3 + k] = de[4 + k];
      }
    }
    {
      const double w = qj[0], xx = qj[1], y = qj[2], zq = qj[3];
      const double* de = e[r].v + 7;
      const double jj[4][3] = {{-xx, -y, -zq}, {w, zq, -y}, {-zq, w, xx}, {y, -xx, w}};
      for (int k = 0; k < 4; ++k)
        for (int a = 0; a < 3; ++a) row[6 + a] += de[k] * jj[k][a];
      for (int k = 0; k < d.tdof; ++k) row[6 + 3 + k] = de[4 + k];
    }
  }
  const int n = d.num_local();
  const int li = d.loc(pi), lj = d.loc(pj);
  auto col = [&](int k) { return k < 6 ? li + k : lj + (k - 6); };
  auto live = [&](int k) { return k < 6 ? k < ni : (k - 6) < nj; };
  for (int a = 0; a < 12; ++a) {
    if (!live(a)) continue;
    double ga = 0;
    for (int r = 0; r < 6; ++r) ga += J[r][a] * e[r].a;
    atomicAdd(g + col(a), ga);
    for (int b = 0; b < 12; ++b) {
      if (!live(b)) continue;
      double hab = 0;
      for (int r = 0; r < 6; ++r) hab += J[r][a] * J[r][b];
      atomicAdd(H + (size_t)col(a) * n + col(b), hab);
    }
  }
}

// x (+) delta for all poses (PoseGraphProblem::Plus semantics); one thread per pose.
__global__ void spa_plus_kernel(GraphDims d, const double* __restrict__ x, const double* __restrict__ delta, double sign, double* out) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= d.poses()) return;
  const double* q = x + d.rot(p);
  const double* dl = delta + d.loc(p);
  double* o = out + d.rot(p);
  if (p == 0) {
    const double d0 = sign * dl[0], d1 = sign * dl[1];
    const double nn = sqrt(d0 * d0 + d1 * d1);
    const double s = nn < 1e-6 ? 1. : sin(nn) / nn;
    const Quatd qd{nn < 1e-6 ? 1. : cos(nn), s * d0, s * d1, 0.};
    const Quatd r = qmul(Quatd{q[0], q[1], q[2], q[3]}, qd);
    o[0] = r.w; o[1] = r.x; o[2] = r.y; o[3] = r.z;
    return;
  }
  const double d0 = sign * dl[0], d1 = sign * dl[1], d2 = sign * dl[2];
  const double nn = sqrt(d0 * d0 + d1 * d1 + d2 * d2);
  if (nn > 0.) {
    const double s = sin(nn) / nn;
    const Quatd r = qmul(Quatd{cos(nn), s * d0, s * d1, s * d2}, Quatd{q[0], q[1], q[2], q[3]});
    o[0] = r.w; o[1] = r.x; o[2] = r.y; o[3] = r.z;
  } else {
    for (int k = 0; k < 4; ++k) o[k] = q[k];
  }
  const double* t = x + d.trans(p);
  double* ot = out + d.trans(p);
  for (int k = 0; k < 3; ++k) ot[k] = t[k] + (k < d.tdof ? sign * dl[3 + k] : 0.);
}

// One CTA: Jacobi scaling (first call), LM diagonal, A = S H S + D / radius, dense Cholesky, the step and the model cost change.
// scalars: [0] radius (in), [1] reuse_diagonal (in), [2] compute_scale (in) -> out: [3] valid, [4] model_cost_change
struct StepArgs {
  int n;
  const double* H;
  const double* g;
  double* scale;
  double* diag;
  double* A;      // n x n scratch
  double* gs;     // n
  double* step;   // n: scaled step (y * -1)
  double* delta;  // n: step * scale
  double* scalars;
};
__global__ void __launch_bounds__(1024) spa_step_kernel(StepArgs a) {
  __shared__ double red[32];
  __shared__ int ok_s;
  const int n = a.n, tid = threadIdx.x, nt = blockDim.x;
  const double radius = a.scalars[0];
  const bool reuse = a.scalars[1] != 0., compute_scale = a.scalars[2] != 0.;
  if (compute_scale)
    for (int j = tid; j < n; j += nt) a.scale[j] = 1.0 / (1.0 + sqrt(a.H[(size_t)j * n + j]));
  __syncthreads();
  for (int j = tid; j < n; j += nt) {
    a.gs[j] = a.scale[j] * a.g[j];
    const double hjj = a.scale[j] * a.H[(size_t)j * n + j] * a.scale[j];
    if (!reuse) a.diag[j] = fmin(fmax(hjj, lm_min_diag()), lm_max_diag());
  }
  __syncthreads();
  for (size_t e = tid; e < (size_t)n * n; e += nt) {
    const int r = (int)(e / n), c = (int)(e % n);
    double v = a.scale[r] * a.H[e] * a.scale[c];
    if (r == c) v += a.diag[r] / radius;
    a.A[e] = v;
  }
  cta_cholesky_factor(a.A, n, &ok_s);
  int valid = ok_s;
  if (valid) {
    for (int j = tid; j < n; j += nt) a.step[j] = a.gs[j];
    __syncthreads();
    cta_cholesky_solve(a.A, n, a.step);
    if (tid == 0) ok_s = 1;
    __syncthreads();
    for (int j = tid; j < n; j += nt) {
      if (!isfinite(a.step[j])) ok_s = 0;
      a.step[j] = -a.step[j];
    }
    __syncthreads();
    valid = ok_s;
  }
  double mcc = 0.;
  if (valid) {
    // model_cost_change = -(step . gs + 1/2 step^T (S H S) step)
    double part = 0.;
    for (int r = tid; r < n; r += nt) {
      double row = 0.;
      for (int c = 0; c < n; ++c) row += (a.scale[r] * a.H[(size_t)r * n + c] * a.scale[c]) * a.step[c];
      part += a.step[r] * a.gs[r] + 0.5 * a.step[r] * row;
    }
    for (int dd = 16; dd > 0; dd >>= 1) part += __shfl_xor_sync(0xffffffffu, part, dd);
    if ((tid & 31) == 0) red[tid >> 5] = part;
    __syncthreads();
    if (tid == 0) {
      double s = 0;
      for (int w = 0; w < (nt + 31) / 32; ++w) s += red[w];
      mcc = -s;
      a.scalars[4] = mcc;
      a.scalars[3] = mcc > 0. ? 1. : 0.;
    }
    for (int j = tid; j < n; j += nt) a.delta[j] = a.step[j] * a.scale[j];
  } else if (tid == 0) {
    a.scalars[3] = 0.;
    a.scalars[4] = 0.;
  }
}

// max_i |x_i - y_i| and ||x||, ||x - y|| (ambient): one CTA
__global__ void spa_norms_kernel(int na, const double* __restrict__ x, const double* __restrict__ y, double* out3) {
  __shared__ double r0[32], r1[32], r2[32];
  double mx = 0, sx = 0, sd = 0;
  for (int i = threadIdx.x; i < na; i += blockDim.x) {
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

}  // namespace
}  // namespace dl

using namespace dl;

extern "C" int dl_pose_graph_solve(dl_context* ctx, dl_comm* comm, const dl_pose_graph_options* options, int32_t num_submaps,
                                   int32_t num_nodes, double* poses, const dl_spa_constraint* constraints, int32_t num_constraints,
                                   dl_solve_summary* summary, dl_pose_graph_info* info) {
  if (!ctx || !options || num_submaps < 1 || num_nodes < 0 || !poses || num_constraints < 0 || (num_constraints > 0 && !constraints))
    return DL_ERR_ARG;
  GraphDims d{num_submaps, num_nodes, options->fix_z ? 2 : 3};
  const int n = d.num_local(), na = d.num_ambient(), P = d.poses();
  if (n > kMaxLocal) return ctx->fail(DL_ERR_ARG, "pose graph too large for the dense solver (local size > 3072)");
  for (int k = 0; k < num_constraints; ++k)
    if (constraints[k].submap < 0 || constraints[k].submap >= num_submaps || constraints[k].node < 0 || constraints[k].node >= num_nodes)
      return ctx->fail(DL_ERR_ARG, "constraint refers to a submap / node outside the graph");
  cudaError_t e0 = cudaSetDevice(ctx->device);
  if (e0 != cudaSuccess) return ctx->cuda_fail(e0, "cudaSetDevice");
  const size_t nn = (size_t)n * n;
  const size_t sys = nn + n + 1;  // H, g, cost2: one all-reduce block
  auto A8 = [](size_t v) { return (v + 31) & ~size_t(31); };
  const size_t doubles = A8(sys) * 2 + A8(nn) + A8(na) * 3 + A8(n) * 6 + 64 + 8;
  const int st0 = ctx->reserve_device(doubles * 8 + (size_t)std::max(num_constraints, 1) * sizeof(dl_spa_constraint) + 4096);
  if (st0 != DL_OK) return st0;
  Arena a(ctx->d_scratch);
  double* d_sys[2] = {a.take<double>(A8(sys)), a.take<double>(A8(sys))};  // accepted point / candidate
  double* d_A = a.take<double>(A8(nn));
  double* d_x = a.take<double>(A8(na));
  double* d_cand = a.take<double>(A8(na));
  double* d_tmp = a.take<double>(A8(na));
  double* d_scale = a.take<double>(A8(n));
  double* d_diag = a.take<double>(A8(n));
  double* d_gs = a.take<double>(A8(n));
  double* d_step = a.take<double>(A8(n));
  double* d_delta = a.take<double>(A8(n));
  double* d_negg = a.take<double>(A8(n));
  double* d_scalars = a.take<double>(16);
  double* d_norms = a.take<double>(8);
  double* d_t0 = a.take<double>(4);
  dl_spa_constraint* d_c = a.take<dl_spa_constraint>(std::max(num_constraints, 1));
#define PG_CUDA(call)                                              \
  do {                                                             \
    cudaError_t e__ = (call);                                      \
    if (e__ != cudaSuccess) return ctx->cuda_fail(e__, #call);     \
  } while (0)
  std::vector<double> x(na), best(na);
  for (int p = 0; p < P; ++p) {
    const double* s = poses + 7 * p;
    double* q = x.data() + d.rot(p);
    q[0] = s[3]; q[1] = s[4]; q[2] = s[5]; q[3] = s[6];
    if (p > 0) { double* t = x.data() + d.trans(p); t[0] = s[0]; t[1] = s[1]; t[2] = s[2]; }
  }
  best = x;
  PG_CUDA(cudaMemcpyAsync(d_x, x.data(), na * 8, cudaMemcpyHostToDevice, ctx->stream));
  PG_CUDA(cudaMemcpyAsync(d_t0, poses, 3 * 8, cudaMemcpyHostToDevice, ctx->stream));
  if (num_constraints) PG_CUDA(cudaMemcpyAsync(d_c, constraints, (size_t)num_constraints * sizeof(dl_spa_constraint), cudaMemcpyHostToDevice, ctx->stream));
  cudaEvent_t ev0, ev1;
  cudaEventCreate(&ev0);
  cudaEventCreate(&ev1);
  float reduce_ms = 0.f, reduce_min_ms = 1e30f;
  int reductions = 0;
  // evaluation at `at` into system `buf`: local constraints, then the all-reduce over the ranks
  auto evaluate = [&](const double* at, int buf) -> int {
    PG_CUDA(cudaMemsetAsync(d_sys[buf], 0, sys * 8, ctx->stream));
    if (num_constraints) {
      spa_evaluate_kernel<<<(num_constraints + 63) / 64, 64, 0, ctx->stream>>>(d, at, d_t0, d_c, num_constraints, d_sys[buf], d_sys[buf] + nn,
                                                                               d_sys[buf] + nn + n, 1);
      ctx->launches++;
      PG_CUDA(cudaGetLastError());
    }
    if (comm) {
      PG_CUDA(cudaEventRecord(ev0, ctx->stream));
      const int st = dl_comm_all_reduce_f64_dev(comm, d_sys[buf], (int64_t)sys);
      if (st != DL_OK) return st;
      PG_CUDA(cudaEventRecord(ev1, ctx->stream));
      PG_CUDA(cudaEventSynchronize(ev1));
      float ms = 0.f;
      cudaEventElapsedTime(&ms, ev0, ev1);
      reduce_ms += ms;
      reduce_min_ms = std::fmin(reduce_min_ms, ms);
      ++reductions;
    }
    return DL_OK;
  };
  auto cost_of = [&](int buf, double* c) -> int {
    double c2 = 0;
    PG_CUDA(cudaMemcpyAsync(&c2, d_sys[buf] + nn + n, 8, cudaMemcpyDeviceToHost, ctx->stream));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    *c = 0.5 * c2;
    return DL_OK;
  };
  // projected gradient max norm at (at, system buf): || at - Plus(at, -g) ||_max, and ||at||
  auto gradient_norms = [&](const double* at, int buf, double* gmax, double* xnorm) -> int {
    spa_plus_kernel<<<(P + 127) / 128, 128, 0, ctx->stream>>>(d, at, d_sys[buf] + nn, -1.0, d_tmp);
    spa_norms_kernel<<<1, 256, 0, ctx->stream>>>(na, at, d_tmp, d_norms);
    ctx->launches += 2;
    double o[3];
    PG_CUDA(cudaMemcpyAsync(o, d_norms, 24, cudaMemcpyDeviceToHost, ctx->stream));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    *gmax = o[0];
    *xnorm = o[1];
    return DL_OK;
  };
  (void)d_negg;
  // ---- Ceres 1.13 TrustRegionMinimizer (dl_posegraph.cuh), scalars on the host
  int cur = 0;
  LmCallbacks cb;
  cb.initial = [&](double* cost, double* gmax, double* x_norm) -> int {
    DL_TRY_STATUS(evaluate(d_x, cur));
    DL_TRY_STATUS(cost_of(cur, cost));
    return gradient_norms(d_x, cur, gmax, x_norm);
  };
  cb.save_best = [&]() -> int {
    PG_CUDA(cudaMemcpyAsync(best.data(), d_x, na * 8, cudaMemcpyDeviceToHost, ctx->stream));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    return DL_OK;
  };
  cb.step = [&](double radius, bool reuse_diagonal, bool first_step, bool* valid, double* model_cost_change) -> int {
    const double sc[3] = {radius, reuse_diagonal ? 1. : 0., first_step ? 1. : 0.};
    PG_CUDA(cudaMemcpyAsync(d_scalars, sc, 24, cudaMemcpyHostToDevice, ctx->stream));
    StepArgs sa{n, d_sys[cur], d_sys[cur] + nn, d_scale, d_diag, d_A, d_gs, d_step, d_delta, d_scalars};
    spa_step_kernel<<<1, 1024, 0, ctx->stream>>>(sa);
    ctx->launches++;
    double outv[2];
    PG_CUDA(cudaMemcpyAsync(outv, d_scalars + 3, 16, cudaMemcpyDeviceToHost, ctx->stream));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    *valid = outv[0] != 0.;
    *model_cost_change = outv[1];
    return DL_OK;
  };
  cb.candidate = [&](double* cand_cost, double* step_norm) -> int {
    spa_plus_kernel<<<(P + 127) / 128, 128, 0, ctx->stream>>>(d, d_x, d_delta, 1.0, d_cand);
    ctx->launches++;
    DL_TRY_STATUS(evaluate(d_cand, cur ^ 1));
    DL_TRY_STATUS(cost_of(cur ^ 1, cand_cost));
    spa_norms_kernel<<<1, 256, 0, ctx->stream>>>(na, d_x, d_cand, d_norms);
    ctx->launches++;
    double o[3];
    PG_CUDA(cudaMemcpyAsync(o, d_norms, 24, cudaMemcpyDeviceToHost, ctx->stream));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    *step_norm = o[2];
    return DL_OK;
  };
  cb.accept = [&](double* gmax, double* x_norm) -> int {
    std::swap(d_x, d_cand);
    cur ^= 1;
    return gradient_norms(d_x, cur, gmax, x_norm);
  };
  dl_solve_summary sum{};
  DL_TRY_STATUS(run_trust_region(cb, options->max_num_iterations, &sum));
  cudaEventDestroy(ev0);
  cudaEventDestroy(ev1);
  for (int p = 0; p < P; ++p) {
    double* s = poses + 7 * p;
    const double* q = best.data() + d.rot(p);
    s[3] = q[0]; s[4] = q[1]; s[5] = q[2]; s[6] = q[3];
    if (p > 0) { const double* t = best.data() + d.trans(p); s[0] = t[0]; s[1] = t[1]; s[2] = t[2]; }
  }
  if (summary) *summary = sum;
  if (info) {
    info->num_local_parameters = n;
    info->all_reduce_count = reductions;
    info->all_reduce_bytes = (int64_t)sys * 8;
    info->all_reduce_ms = reduce_ms;
    info->all_reduce_min_ms = reductions ? reduce_min_ms : 0.f;
  }
#undef PG_CUDA
  return DL_OK;
}
