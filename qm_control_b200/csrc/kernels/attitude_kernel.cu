// Attitude filter between the IMU reading and the base state estimator (DESIGN.md §4.6).
//
// attitude_step_kernel, one thread per robot: a multiplicative (error-state) Kalman filter on SO(3) with gyro-bias states.  Nominal state q_hat
// (world <- body, xyzw) and b_hat, error x = [dtheta, db] with the right (body-frame) perturbation R = R_hat Exp(dtheta), P 6x6 packed.  Per call:
//   predict   w = gyro - b_hat (the reading that ends the step), q_hat <- q_hat (x) Exp(w dt),
//             P <- F P F^T + dt diag(process_attitude 1_3, process_gyro_bias 1_3),  F = [[Exp(w dt)^T, -dt 1], [0, 1]]
//   update    dq = q_hat^-1 (x) q_m with w >= 0, r = Log(dq); H = [1 0], S = P_tt + meas_orientation 1 (3x3), K = P H^T S^-1, dx = K r,
//             q_hat <- q_hat (x) Exp(dtheta) renormalised, b_hat += db, P <- P - K H P symmetrised (no reset Jacobian: first order)
//   output    sensors[SEN_QUAT..+4) = q_hat with w >= 0, sensors[SEN_GYRO..+3) = gyro - b_hat; the other columns are untouched
// Exp(v) = [v sin(|v|/2) / |v|, cos(|v|/2)] and Log(q) = v 2 atan2(|v|, w) / |v|: no (1 - cos) / theta^2 form, whose cancellation at the per-step angles
// (1e-3 rad) and corrections (1e-5 rad) loses digits.  The first call after a reset only takes the normalised reading.
// status: QMB200_ST_NAN for a non-finite quaternion or gyro input (neither the row nor the state is touched) or update (the state is kept and the row
// written from it).  meas_orientation > 0 (validated by the API) keeps S positive definite.
#include "attitude_api.cuh"
#include "wlinalg.cuh"

namespace qmb {

namespace {
constexpr int AT_THREADS = 128;

__device__ __forceinline__ double pk6(const double* P, int i, int j) { return i >= j ? P[tri(i) + j] : P[tri(j) + i]; }
// o = a (x) b, xyzw
__device__ __forceinline__ void qmul(const double* a, const double* b, double* o) {
  o[0] = a[3] * b[0] + b[3] * a[0] + (a[1] * b[2] - a[2] * b[1]);
  o[1] = a[3] * b[1] + b[3] * a[1] + (a[2] * b[0] - a[0] * b[2]);
  o[2] = a[3] * b[2] + b[3] * a[2] + (a[0] * b[1] - a[1] * b[0]);
  o[3] = a[3] * b[3] - (a[0] * b[0] + a[1] * b[1] + a[2] * b[2]);
}
__device__ __forceinline__ void qexp(const double* v, double* o) {
  const double th = sqrt(dot3(v, v));
  if (th == 0.0) { o[0] = 0.0; o[1] = 0.0; o[2] = 0.0; o[3] = 1.0; return; }
  double s, c; sincos(0.5 * th, &s, &c); const double f = s / th;
  o[0] = v[0] * f; o[1] = v[1] * f; o[2] = v[2] * f; o[3] = c;
}
// the rotation vector of q (w >= 0); 2 atan2(|v|, w) does not need |q| = 1
__device__ __forceinline__ void qlog(const double* q, double* o) {
  const double n = sqrt(dot3(q, q)), f = n > 0.0 ? 2.0 * atan2(n, q[3]) / n : 0.0;
  o[0] = q[0] * f; o[1] = q[1] * f; o[2] = q[2] * f;
}
// R of a unit quaternion, row-major
__device__ __forceinline__ void quat_rot(const double* q, double* R) {
  const double x = q[0], y = q[1], z = q[2], w = q[3];
  R[0] = 1.0 - 2.0 * (y * y + z * z); R[1] = 2.0 * (x * y - z * w); R[2] = 2.0 * (x * z + y * w);
  R[3] = 2.0 * (x * y + z * w); R[4] = 1.0 - 2.0 * (x * x + z * z); R[5] = 2.0 * (y * z - x * w);
  R[6] = 2.0 * (x * z - y * w); R[7] = 2.0 * (y * z + x * w); R[8] = 1.0 - 2.0 * (x * x + y * y);
}
}  // namespace

__global__ void __launch_bounds__(AT_THREADS) attitude_step_kernel(qmb200_attitude_params prm, int B, double dt, double* __restrict__ sensors,
                                                                   double* __restrict__ state, int32_t* __restrict__ status) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  double* sn = sensors + (size_t)b * QMB200_SENSORS; double* st = state + (size_t)b * AT_DBL;
  double qm[4], gy[3]; bool finite = true;
#pragma unroll
  for (int i = 0; i < 4; ++i) { qm[i] = sn[SEN_QUAT + i]; finite = finite && isfinite(qm[i]); }
#pragma unroll
  for (int i = 0; i < 3; ++i) { gy[i] = sn[SEN_GYRO + i]; finite = finite && isfinite(gy[i]); }
  if (!finite) { status[b] = QMB200_ST_NAN; return; }   // dt: checked by the API
  double qh[4], bh[3];
#pragma unroll
  for (int i = 0; i < 4; ++i) qh[i] = st[AT_Q + i];
#pragma unroll
  for (int i = 0; i < 3; ++i) bh[i] = st[AT_B + i];
  const double n_prev = st[AT_N];

  int code = 0;
  if (n_prev == 0.0) {   // first call after a reset: the reading; b_hat = 0 and P = diag(p0) come from the reset
    const double nn = 1.0 / sqrt(qm[0] * qm[0] + qm[1] * qm[1] + qm[2] * qm[2] + qm[3] * qm[3]);
#pragma unroll
    for (int i = 0; i < 4; ++i) { qh[i] = qm[i] * nn; st[AT_Q + i] = qh[i]; }
  } else {
    double P[AT_TRI];
#pragma unroll
    for (int t = 0; t < AT_TRI; ++t) P[t] = st[AT_P + t];
    // ---- predict ----
    const double om[3] = {(gy[0] - bh[0]) * dt, (gy[1] - bh[1]) * dt, (gy[2] - bh[2]) * dt};
    double dq[4], qp[4], E[9]; qexp(om, dq); qmul(qh, dq, qp); quat_rot(dq, E);   // F's top-left block is E^T
    double FP[AT_NX][AT_NX];   // F P: rows 0..2 = E^T P[0:3, :] - dt P[3:6, :], rows 3..5 = P[3:6, :]
#pragma unroll
    for (int j = 0; j < AT_NX; ++j) {
#pragma unroll
      for (int i = 0; i < 3; ++i) FP[i][j] = E[i] * pk6(P, 0, j) + E[3 + i] * pk6(P, 1, j) + E[6 + i] * pk6(P, 2, j) - dt * pk6(P, 3 + i, j);
#pragma unroll
      for (int i = 3; i < AT_NX; ++i) FP[i][j] = pk6(P, i, j);
    }
    double Pp[AT_TRI];   // F P F^T + dt diag(q), lower triangle
#pragma unroll
    for (int i = 0; i < AT_NX; ++i) {
#pragma unroll
      for (int j = 0; j <= i; ++j) {
        double v = j < 3 ? FP[i][0] * E[j] + FP[i][1] * E[3 + j] + FP[i][2] * E[6 + j] - dt * FP[i][3 + j] : FP[i][j];
        if (i == j) v += dt * (i < 3 ? prm.process_attitude : prm.process_gyro_bias);
        Pp[tri(i) + j] = v;
      }
    }
    // ---- update with the orientation reading ----
    const double qc[4] = {-qp[0], -qp[1], -qp[2], qp[3]};
    double dm[4], r[3]; qmul(qc, qm, dm);
    if (dm[3] < 0.0) { dm[0] = -dm[0]; dm[1] = -dm[1]; dm[2] = -dm[2]; dm[3] = -dm[3]; }   // q_m and -q_m give one residual
    qlog(dm, r);
    double S[9], Si[9];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int j = 0; j < 3; ++j) S[3 * i + j] = pk6(Pp, i, j) + (i == j ? prm.meas_orientation : 0.0);
    inv3(S, Si);
    double K[AT_NX][3], dx[AT_NX];
#pragma unroll
    for (int i = 0; i < AT_NX; ++i) {
#pragma unroll
      for (int j = 0; j < 3; ++j) K[i][j] = pk6(Pp, i, 0) * Si[j] + pk6(Pp, i, 1) * Si[3 + j] + pk6(Pp, i, 2) * Si[6 + j];
      dx[i] = K[i][0] * r[0] + K[i][1] * r[1] + K[i][2] * r[2];
    }
    double ex[4], qn[4]; qexp(dx, ex); qmul(qp, ex, qn);
    const double nn = 1.0 / sqrt(qn[0] * qn[0] + qn[1] * qn[1] + qn[2] * qn[2] + qn[3] * qn[3]);
    bool bad = false;
#pragma unroll
    for (int i = 0; i < 4; ++i) { qn[i] *= nn; bad = bad || !isfinite(qn[i]); }
    double bn[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) { bn[i] = bh[i] + dx[3 + i]; bad = bad || !isfinite(bn[i]); }
#pragma unroll
    for (int i = 0; i < AT_NX; ++i) {
#pragma unroll
      for (int j = 0; j <= i; ++j) {   // (K H P)_ij = K_i . P[0:3, j]
        const double kp = K[i][0] * pk6(Pp, 0, j) + K[i][1] * pk6(Pp, 1, j) + K[i][2] * pk6(Pp, 2, j) +
                          (K[j][0] * pk6(Pp, 0, i) + K[j][1] * pk6(Pp, 1, i) + K[j][2] * pk6(Pp, 2, i));
        P[tri(i) + j] = Pp[tri(i) + j] - 0.5 * kp; bad = bad || !isfinite(P[tri(i) + j]);
      }
    }
    if (bad) code = QMB200_ST_NAN;   // the state before this call is kept
    else {
#pragma unroll
      for (int i = 0; i < 4; ++i) { qh[i] = qn[i]; st[AT_Q + i] = qn[i]; }
#pragma unroll
      for (int i = 0; i < 3; ++i) { bh[i] = bn[i]; st[AT_B + i] = bn[i]; }
#pragma unroll
      for (int t = 0; t < AT_TRI; ++t) st[AT_P + t] = P[t];
    }
  }
  // ---- the row the state estimator reads, from the stored state ----
  const double sg = qh[3] < 0.0 ? -1.0 : 1.0;
#pragma unroll
  for (int i = 0; i < 4; ++i) sn[SEN_QUAT + i] = sg * qh[i];
#pragma unroll
  for (int i = 0; i < 3; ++i) sn[SEN_GYRO + i] = gy[i] - bh[i];
  st[AT_N] = n_prev + 1.0; status[b] = code;
}

int launch_attitude_step(const qmb200_attitude_params& prm, int B, double dt, double* sensors, double* state, int32_t* status, cudaStream_t s) {
  attitude_step_kernel<<<(B + AT_THREADS - 1) / AT_THREADS, AT_THREADS, 0, s>>>(prm, B, dt, sensors, state, status);
  return 1;
}

}  // namespace qmb
