// IMU pre-integration on the device: one warp per scan interval.
//
// Replaces the per-sample work of LocalTrajectoryBuilder3D::AddImuData (LTB:164-201) for the in-repo mid-point
// integrator (C/mapping/internal/3d/initialization/integration_base.h:109-123 push_back, :156-236
// midPointIntegration incl. the 15x15 Jacobian F and the 15x18 noise map V, :238-265 propagate). The samples of
// one interval are inherently sequential (~20 at 200 Hz), so the parallelism is (a) across scans: one warp each, and
// (b) inside a step: the three 15x15 products F*J, F*P*F^T, V*N*V^T are spread over the 32 lanes. The state lives in
// shared memory (4 warps per CTA, 9.6 KB each). Row/column order: delta_p, delta_theta, delta_v, b_a, b_g.
#include "dl_internal.cuh"
#include "dl_pipeline.cuh"

namespace dl {
namespace {

constexpr int kWarpsPerBlock = 4;

struct WarpState {
  double J[225], P[225], F[225], T[225], V[270];
  double R0[3][3], R1[3][3], IRw[3][3], R0a0[3][3], R1a1[3][3], R1a1I[3][3];  // 3x3 building blocks of F and V
};

__device__ __forceinline__ void rotation_matrix(const Quatd& q, double R[3][3]) {  // Eigen toRotationMatrix
  const double tx = 2 * q.x, ty = 2 * q.y, tz = 2 * q.z;
  const double twx = tx * q.w, twy = ty * q.w, twz = tz * q.w;
  const double txx = tx * q.x, txy = ty * q.x, txz = tz * q.x, tyy = ty * q.y, tyz = tz * q.y, tzz = tz * q.z;
  R[0][0] = 1 - (tyy + tzz); R[0][1] = txy - twz; R[0][2] = txz + twy;
  R[1][0] = txy + twz; R[1][1] = 1 - (txx + tzz); R[1][2] = tyz - twx;
  R[2][0] = txz - twy; R[2][1] = tyz + twx; R[2][2] = 1 - (txx + tyy);
}
__device__ __forceinline__ void skew(const Vec3d& v, double S[3][3]) {
  S[0][0] = 0; S[0][1] = -v.z; S[0][2] = v.y;
  S[1][0] = v.z; S[1][1] = 0; S[1][2] = -v.x;
  S[2][0] = -v.y; S[2][1] = v.x; S[2][2] = 0;
}
__device__ __forceinline__ void mul33(const double A[3][3], const double B[3][3], double C[3][3]) {
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) C[i][j] = A[i][0] * B[0][j] + A[i][1] * B[1][j] + A[i][2] * B[2][j];
}

__global__ void __launch_bounds__(kWarpsPerBlock * 32) imu_preintegrate_kernel(
    int count, const int32_t* __restrict__ offsets /* count + 1 */, const double* __restrict__ dts,
    const double* __restrict__ accs, const double* __restrict__ gyrs,
    const double* __restrict__ biases /* ba, bg of scan k at biases + k * bias_stride */, int bias_stride, double acc_n, double gyr_n, double acc_w, double gyr_w, dl_preintegration* __restrict__ out) {
  __shared__ WarpState states[kWarpsPerBlock];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int scan = blockIdx.x * kWarpsPerBlock + warp;
  if (scan >= count) return;
  WarpState& st = states[warp];
  for (int e = lane; e < 225; e += 32) {
    st.J[e] = (e / 15 == e % 15) ? 1.0 : 0.0;
    st.P[e] = 0.0;
  }
  const double* bias = biases + (size_t)bias_stride * scan;
  const Vec3d ba{bias[0], bias[1], bias[2]};
  const Vec3d bg{bias[3], bias[4], bias[5]};
  Vec3d dp{0, 0, 0}, dv{0, 0, 0};
  Quatd dq{1, 0, 0, 0};
  double sum_dt = 0;
  const int first = offsets[scan], last = offsets[scan + 1];
  Vec3d acc_0{0, 0, 0}, gyr_0{0, 0, 0};
  if (last > first) {  // the first sample only latches acc_0 / gyr_0 (integration_base.h:111-118)
    acc_0 = {accs[3 * first], accs[3 * first + 1], accs[3 * first + 2]};
    gyr_0 = {gyrs[3 * first], gyrs[3 * first + 1], gyrs[3 * first + 2]};
  }
  const double nd[18] = {acc_n * acc_n, acc_n * acc_n, acc_n * acc_n, gyr_n * gyr_n, gyr_n * gyr_n, gyr_n * gyr_n,
                         acc_n * acc_n, acc_n * acc_n, acc_n * acc_n, gyr_n * gyr_n, gyr_n * gyr_n, gyr_n * gyr_n,
                         acc_w * acc_w, acc_w * acc_w, acc_w * acc_w, gyr_w * gyr_w, gyr_w * gyr_w, gyr_w * gyr_w};
  __syncwarp();
  for (int k = first + 1; k < last; ++k) {
    const double dt = dts[k];
    const Vec3d acc_1{accs[3 * k], accs[3 * k + 1], accs[3 * k + 2]};
    const Vec3d gyr_1{gyrs[3 * k], gyrs[3 * k + 1], gyrs[3 * k + 2]};
    // state update (every lane computes it redundantly: ~100 flops, keeps the state in registers)
    const Vec3d un_acc_0 = rotate(dq, sub(acc_0, ba));
    const Vec3d un_gyr = sub(mul(0.5, add(gyr_0, gyr_1)), bg);
    const Quatd rq = qmul(dq, Quatd{1, un_gyr.x * dt / 2, un_gyr.y * dt / 2, un_gyr.z * dt / 2});
    const Vec3d un_acc_1 = rotate(rq, sub(acc_1, ba));
    const Vec3d un_acc = mul(0.5, add(un_acc_0, un_acc_1));
    const Vec3d rp = add(add(dp, mul(dt, dv)), mul(0.5 * dt * dt, un_acc));
    const Vec3d rv = add(dv, mul(dt, un_acc));
    // F and V of this step (integration_base.h:176-232): lane 0 forms the 3x3 building blocks, every lane clears its share
    // of the two matrices, then lanes 0..8 each write the entries of one (i, j) position of the blocks.
    if (lane == 0) {
      double Rw[3][3], Ra0[3][3], Ra1[3][3];
      skew(un_gyr, Rw); skew(sub(acc_0, ba), Ra0); skew(sub(acc_1, ba), Ra1);
      rotation_matrix(dq, st.R0);
      rotation_matrix(rq, st.R1);
      for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) st.IRw[i][j] = (i == j ? 1.0 : 0.0) - Rw[i][j] * dt;
      mul33(st.R0, Ra0, st.R0a0);
      mul33(st.R1, Ra1, st.R1a1);
      mul33(st.R1a1, st.IRw, st.R1a1I);
    }
    for (int e = lane; e < 225; e += 32) st.F[e] = 0.0;
    for (int e = lane; e < 270; e += 32) st.V[e] = 0.0;
    __syncwarp();
    if (lane < 9) {
      const int i = lane / 3, j = lane % 3;
      const double id = i == j ? 1.0 : 0.0;
      const double R0 = st.R0[i][j], R1 = st.R1[i][j], R0a0 = st.R0a0[i][j], R1a1 = st.R1a1[i][j], R1a1I = st.R1a1I[i][j];
      st.F[i * 15 + j] = id;
      st.F[i * 15 + 3 + j] = -0.25 * R0a0 * dt * dt + -0.25 * R1a1I * dt * dt;
      st.F[i * 15 + 6 + j] = id * dt;
      st.F[i * 15 + 9 + j] = -0.25 * (R0 + R1) * dt * dt;
      st.F[i * 15 + 12 + j] = -0.25 * R1a1 * dt * dt * -dt;
      st.F[(3 + i) * 15 + 3 + j] = st.IRw[i][j];
      st.F[(3 + i) * 15 + 12 + j] = -1.0 * id * dt;
      st.F[(6 + i) * 15 + 3 + j] = -0.5 * R0a0 * dt - 0.5 * R1a1I * dt;
      st.F[(6 + i) * 15 + 6 + j] = id;
      st.F[(6 + i) * 15 + 9 + j] = -0.5 * (R0 + R1) * dt;
      st.F[(6 + i) * 15 + 12 + j] = -0.5 * R1a1 * dt * -dt;
      st.F[(9 + i) * 15 + 9 + j] = id;
      st.F[(12 + i) * 15 + 12 + j] = id;
      const double v03 = 0.25 * -R1a1 * dt * dt * 0.5 * dt, v63 = 0.5 * -R1a1 * dt * 0.5 * dt;
      st.V[i * 18 + j] = 0.25 * R0 * dt * dt;
      st.V[i * 18 + 3 + j] = v03;
      st.V[i * 18 + 6 + j] = 0.25 * R1 * dt * dt;
      st.V[i * 18 + 9 + j] = v03;
      st.V[(3 + i) * 18 + 3 + j] = 0.5 * id * dt;
      st.V[(3 + i) * 18 + 9 + j] = 0.5 * id * dt;
      st.V[(6 + i) * 18 + j] = 0.5 * R0 * dt;
      st.V[(6 + i) * 18 + 3 + j] = v63;
      st.V[(6 + i) * 18 + 6 + j] = 0.5 * R1 * dt;
      st.V[(6 + i) * 18 + 9 + j] = v63;
      st.V[(9 + i) * 18 + 12 + j] = id * dt;
      st.V[(12 + i) * 18 + 15 + j] = id * dt;
    }
    __syncwarp();
    // T = F * J ; then J = T
    for (int e = lane; e < 225; e += 32) {
      const int i = e / 15, j = e % 15;
      double s = 0;
      for (int c = 0; c < 15; ++c) s += st.F[i * 15 + c] * st.J[c * 15 + j];
      st.T[e] = s;
    }
    __syncwarp();
    for (int e = lane; e < 225; e += 32) st.J[e] = st.T[e];
    __syncwarp();
    // T = F * P ; P = T * F^T + V N V^T
    for (int e = lane; e < 225; e += 32) {
      const int i = e / 15, j = e % 15;
      double s = 0;
      for (int c = 0; c < 15; ++c) s += st.F[i * 15 + c] * st.P[c * 15 + j];
      st.T[e] = s;
    }
    __syncwarp();
    for (int e = lane; e < 225; e += 32) {
      const int i = e / 15, j = e % 15;
      double a = 0, b = 0;
      for (int c = 0; c < 15; ++c) a += st.T[i * 15 + c] * st.F[j * 15 + c];
      for (int c = 0; c < 18; ++c) b += st.V[i * 18 + c] * nd[c] * st.V[j * 18 + c];
      st.P[e] = a + b;
    }
    __syncwarp();
    dp = rp;
    dv = rv;
    dq = qnormalized(rq);
    sum_dt += dt;
    acc_0 = acc_1;
    gyr_0 = gyr_1;
  }
  dl_preintegration& o = out[scan];
  for (int e = lane; e < 225; e += 32) {
    o.jacobian[e] = st.J[e];
    o.covariance[e] = st.P[e];
  }
  if (lane == 0) {
    o.sum_dt = sum_dt;
    o.delta_p[0] = dp.x; o.delta_p[1] = dp.y; o.delta_p[2] = dp.z;
    o.delta_q[0] = dq.w; o.delta_q[1] = dq.x; o.delta_q[2] = dq.y; o.delta_q[3] = dq.z;
    o.delta_v[0] = dv.x; o.delta_v[1] = dv.y; o.delta_v[2] = dv.z;
    o.linearized_ba[0] = ba.x; o.linearized_ba[1] = ba.y; o.linearized_ba[2] = ba.z;
    o.linearized_bg[0] = bg.x; o.linearized_bg[1] = bg.y; o.linearized_bg[2] = bg.z;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Everything between the pre-integration and the fused solve, on the device, so that a batch of scans with their raw
// IMU samples needs no host round trip: state prediction (dl_imu_predict's arithmetic = the front end's
// pose prediction, LTB:188-199), the deskew constants of LTB:426-428, the pre-integration factor moved into the submap
// frame, and its information matrix W = weight^2 * Sigma^-1 (Sigma = L L^T, W = L^-T L^-1; the same operation order as the
// host path in dl_api.cu, so both produce the same bits). One warp per scan; lane i owns row / column i of the 15x15 work.
struct PrepareShared {
  double L[15][15], Li[15][15];
};

__global__ void __launch_bounds__(kWarpsPerBlock * 32) imu_prepare_kernel(ImuPrepareArgs a) {
  __shared__ PrepareShared shared[kWarpsPerBlock];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int b = blockIdx.x * kWarpsPerBlock + warp;
  if (b >= a.count) return;
  PrepareShared& sh = shared[warp];
  const dl_preintegration& m = a.preint[b];
  const dl_nav_state& si = a.states_i[b];
  ImuTerm& t = a.terms[b];
  if (lane == 0) {
    // prediction at the end of the interval
    const double T = m.sum_dt;
    const Quatd qi{si.q[0], si.q[1], si.q[2], si.q[3]};
    const Vec3d G{a.gravity[0], a.gravity[1], a.gravity[2]};
    const Vec3d pi{si.p[0], si.p[1], si.p[2]}, vi{si.v[0], si.v[1], si.v[2]};
    const Vec3d pj = add(sub(add(pi, mul(T, vi)), mul(0.5 * T * T, G)), rotate(qi, Vec3d{m.delta_p[0], m.delta_p[1], m.delta_p[2]}));
    const Vec3d vj = add(sub(vi, mul(T, G)), rotate(qi, Vec3d{m.delta_v[0], m.delta_v[1], m.delta_v[2]}));
    const Quatd qj = qnormalized(qmul(qi, Quatd{m.delta_q[0], m.delta_q[1], m.delta_q[2], m.delta_q[3]}));
    if (a.predicted) {
      dl_nav_state& o = a.predicted[b];
      o = si;
      o.p[0] = pj.x; o.p[1] = pj.y; o.p[2] = pj.z;
      o.v[0] = vj.x; o.v[1] = vj.y; o.v[2] = vj.z;
      o.q[0] = qj.w; o.q[1] = qj.x; o.q[2] = qj.y; o.q[3] = qj.z;
    }
    const Rigidd prev{pi, qi}, cur{pj, qj};
    a.scans[b] = make_scan_constants(prev, cur);
    // the factor in the submap frame (the grids live there and the solve is frame-invariant)
    const Rigidd to_submap = a.to_submap[b];
    const Rigidd pose_i = compose(to_submap, prev), pose_j = compose(to_submap, cur);
    const Vec3d wi = rotate(to_submap.q, vi), wj = rotate(to_submap.q, vj), Gs = rotate(to_submap.q, G);
    t.pi[0] = pose_i.t.x; t.pi[1] = pose_i.t.y; t.pi[2] = pose_i.t.z;
    t.qi[0] = pose_i.q.w; t.qi[1] = pose_i.q.x; t.qi[2] = pose_i.q.y; t.qi[3] = pose_i.q.z;
    t.vi[0] = wi.x; t.vi[1] = wi.y; t.vi[2] = wi.z;
    imu_term_deltas(m, si.ba, si.bg, &t);
    t.G[0] = Gs.x; t.G[1] = Gs.y; t.G[2] = Gs.z;
    t.sum_dt = m.sum_dt;
    double* x = a.init16 + 16 * (size_t)b;
    pose_to7(pose_j, x);
    x[7] = wj.x; x[8] = wj.y; x[9] = wj.z;
    for (int k = 0; k < 3; ++k) { x[10 + k] = si.ba[k]; x[13 + k] = si.bg[k]; }
  }
  // Cholesky of the covariance, column by column (lane = row)
  const bool row = lane < 15;
  bool pd = true;
  for (int j = 0; j < 15; ++j) {
    double s = 0.0;
    if (row && lane >= j) {
      s = m.covariance[lane * 15 + j];
      for (int k = 0; k < j; ++k) s -= sh.L[lane][k] * sh.L[j][k];
    }
    const double pivot = __shfl_sync(0xffffffffu, s, j);
    if (!(pivot > 0)) { pd = false; break; }
    const double d = sqrt(pivot);
    if (row && lane >= j) sh.L[lane][j] = lane == j ? d : s / d;
    __syncwarp();
  }
  if (lane == 0) a.ok[b] = pd ? 1 : 0;
  if (!pd) return;
  // L^-1 (lower): lane c solves column c
  if (row) {
    const int c = lane;
    for (int i = 0; i < c; ++i) sh.Li[i][c] = 0.0;
    for (int i = c; i < 15; ++i) {
      double s = i == c ? 1.0 : 0.0;
      for (int k = c; k < i; ++k) s -= sh.L[i][k] * sh.Li[k][c];
      sh.Li[i][c] = s / sh.L[i][i];
    }
  }
  __syncwarp();
  for (int e = lane; e < 225; e += 32) {
    const int r = e / 15, c = e % 15;
    double s = 0;
    for (int k = (r > c ? r : c); k < 15; ++k) s += sh.Li[k][r] * sh.Li[k][c];
    t.W[e] = a.imu_weight * a.imu_weight * s;
  }
}

}  // namespace

int launch_imu_prepare(dl_context* ctx, const ImuPrepareArgs& a) {
  if (a.count <= 0) return DL_OK;
  imu_prepare_kernel<<<(a.count + kWarpsPerBlock - 1) / kWarpsPerBlock, kWarpsPerBlock * 32, 0, ctx->stream>>>(a);
  DL_LAUNCH_CHECK(ctx, "imu_prepare_kernel");
  return DL_OK;
}

int launch_imu_preintegrate(dl_context* ctx, int count, const int32_t* offsets, const double* dts, const double* accs,
                            const double* gyrs, const double* biases, int bias_stride, const dl_imu_noise& noise,
                            dl_preintegration* out) {
  if (count <= 0) return DL_OK;
  imu_preintegrate_kernel<<<(count + kWarpsPerBlock - 1) / kWarpsPerBlock, kWarpsPerBlock * 32, 0, ctx->stream>>>(
      count, offsets, dts, accs, gyrs, biases, bias_stride, noise.acc_n, noise.gyr_n, noise.acc_w, noise.gyr_w, out);
  DL_LAUNCH_CHECK(ctx, "imu_preintegrate_kernel");
  return DL_OK;
}

}  // namespace dl
