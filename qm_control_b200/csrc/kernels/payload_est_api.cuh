// Host-visible interface of the online payload estimator (payload_est_kernel.cu): per-robot recursive least squares on the arm rows of the nominal
// model, committed to the controller's model payload on the device (include/qmb200.h: qmb200_payload_est_*; DESIGN.md §4.6).
#pragma once
#include <cuda_runtime.h>

#include "dev_common.cuh"
#include "../../../include/qmb200.h"

namespace qmb {

// Estimator state of one robot, EST_DBL doubles in one device block [B][EST_DBL]:
//   [0, 10)    theta = [m, m c(3), I(6)]: the load's inertial parameters in the end-effector frame about its origin, I = (xx, xy, xz, yy, yz, zz)
//   [10, 65)   P, packed lower triangle (entry (i, j <= i) at i(i+1)/2 + j)
//   [65, 89)   q of the previous sample, [89, 113) its v (euler rates)
//   [113]      samples stored since the reset (0: the next call only stores its sample)
constexpr int EST_NP = 10, EST_TRI = EST_NP * (EST_NP + 1) / 2;
constexpr int EST_THETA = 0, EST_P = EST_THETA + EST_NP, EST_Q = EST_P + EST_TRI, EST_V = EST_Q + NQ, EST_N = EST_V + NQ, EST_DBL = EST_N + 1;

// One RLS update per robot from the measurement rbd [B][55] and the effort [B][18] held over the dt seconds that ended at it; status [B] is written.
int launch_payload_est_step(const DevModel* mdl, const qmb200_payload_est_params& prm, int B, double dt, const double* effort, const double* rbd, double* state,
                            int32_t* status, cudaStream_t s);
// theta → the end-effector half of each robot's model payload row mpayload [B][8] and its SRBD constants srbd [B][SRBD_DBL]
int launch_payload_est_commit(const DevModel* mdl, const qmb200_payload_est_params& prm, int B, const double* state, double* mpayload, double* srbd, cudaStream_t s);

}  // namespace qmb
