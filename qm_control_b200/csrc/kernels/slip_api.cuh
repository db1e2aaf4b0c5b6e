// Host-visible interface of the slip detector (slip_step_kernel in state_est_kernel.cu): per robot, a test of each stance foot's velocity against the
// base state estimator's prior that turns the plant's contact mask into the mask of the stance feet the estimator may trust (include/qmb200.h:
// qmb200_slip_*; DESIGN.md §4.6).
#pragma once
#include <cuda_runtime.h>

#include "state_est_api.cuh"

namespace qmb {

// Detector state of one robot, SL_DBL doubles in one device block [B][SL_DBL]:
//   [0]        slip mask (contact bit order: foot f at bit 3 - f)
//   [1, 5)     per foot: consecutive calls with d^2 < release while slipping
//   [5, 9)     per foot: onsets since the reset (calls on which the foot became slipping)
constexpr int SL_MASK = 0, SL_HOLD = 1, SL_ONSET = SL_HOLD + 4, SL_DBL = SL_ONSET + 4;

// one detector call per robot from sensors [B][46], the contact mask [B] and the estimator's state se [B][SE_DBL] (read only);
// writes stance [B], slip [B] and status [B]
int launch_slip_step(const DevModel* mdl, const qmb200_slip_params& prm, const qmb200_state_est_params& se_prm, int B, double dt, const double* sensors,
                     const int32_t* contact, const double* se, double* state, int32_t* stance, int32_t* slip, int32_t* status, cudaStream_t s);

}  // namespace qmb
