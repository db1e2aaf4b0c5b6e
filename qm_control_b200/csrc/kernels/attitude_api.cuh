// Host-visible interface of the attitude filter (attitude_kernel.cu): a batched multiplicative Kalman filter on SO(3) with gyro-bias states that
// replaces the orientation and gyro columns of a sensor row (state_est_api.cuh: SEN_*) with the filtered orientation and the bias-corrected rate
// (include/qmb200.h: qmb200_attitude_*; DESIGN.md §4.6).
#pragma once
#include <cuda_runtime.h>

#include "state_est_api.cuh"

namespace qmb {

// Filter state of one robot, AT_DBL doubles in one device block [B][AT_DBL]:
//   [0, 4)     q_hat, world <- body, xyzw (not re-signed: it stays continuous from call to call)
//   [4, 7)     gyro bias b_hat (rad/s, body axes)
//   [7, 28)    P on the error [dtheta (body, right perturbation R = R_hat Exp(dtheta)), db], packed lower triangle (entry (i, j <= i) at i(i+1)/2 + j)
//   [28]       calls since the reset (0: the next call only takes its reading)
constexpr int AT_NX = 6, AT_TRI = AT_NX * (AT_NX + 1) / 2;
constexpr int AT_Q = 0, AT_B = AT_Q + 4, AT_P = AT_B + 3, AT_N = AT_P + AT_TRI, AT_DBL = AT_N + 1;
// The reset row st [AT_DBL] of one robot: the identity (replaced by the first call's reading), zero bias, P diagonal with p's p0 variances, no call yet.
// qmb200_attitude_reset and the spawn sampler both write it.
QMB_HD void attitude_reset_row(const qmb200_attitude_params& p, double* st) {
  for (int i = 0; i < AT_DBL; ++i) st[i] = 0.0;
  st[AT_Q + 3] = 1.0;
  for (int i = 0; i < AT_NX; ++i) st[AT_P + i * (i + 1) / 2 + i] = i < 3 ? p.p0_attitude : p.p0_gyro_bias;
}

// one filter call per robot on sensors [B][46] (in-out: quaternion and gyro columns replaced); writes status [B]
int launch_attitude_step(const qmb200_attitude_params& prm, int B, double dt, double* sensors, double* state, int32_t* status, cudaStream_t s);

}  // namespace qmb
