// Host-visible interface of the sensor model and the base state estimator (state_est_kernel.cu): the IMU and joint-encoder readings of the plant state
// (include/qmb200.h: qmb200_sim_read_sensors) and a batched linear Kalman filter that turns them, with the plant's contact flags, into the measurement
// rbd[55] the controller consumes (qmb200_state_est_*; DESIGN.md §4.6).
#pragma once
#include <cuda_runtime.h>

#include "dev_common.cuh"
#include "sim_api.cuh"
#include "../../../include/qmb200.h"

namespace qmb {

// sensors[B][QMB200_SENSORS] = [quat xyzw(4), gyro(3), accel(3), joint pos(18), joint vel(18)]
constexpr int SEN_QUAT = 0, SEN_GYRO = 4, SEN_ACCEL = 7, SEN_JPOS = 10, SEN_JVEL = 28;
static_assert(SEN_JVEL + NJ == QMB200_SENSORS, "sensor layout of include/qmb200.h");
// noise channels of one reading: orientation (3), gyro (3), accel (3), joint pos (18), joint vel (18)
constexpr int CH_ORI = 0, CH_GYRO = 3, CH_ACCEL = 6, CH_JPOS = 9, CH_JVEL = 27;

// One standard normal draw, a pure function of (seed, robot, sample, channel): the four words are hashed in turn, two 53-bit uniforms in (0, 1) are cut
// from two more hashes, and Box-Muller's cosine branch turns them into N(0, 1).  No generator state, so a draw does not depend on the batch or the launch.
QMB_HD double sensor_normal(uint64_t seed, uint64_t robot, uint64_t sample, int channel) {
  const uint64_t h = mix64(mix64(mix64(mix64(seed ^ 0x9e3779b97f4a7c15ull) ^ robot) ^ sample) ^ (uint64_t)channel);
  const double u1 = ((double)(mix64(h) >> 11) + 0.5) * 1.1102230246251565e-16, u2 = ((double)(mix64(h ^ 0xd1b54a32d192ed03ull) >> 11) + 0.5) * 1.1102230246251565e-16;
  return sqrt(-2.0 * log(u1)) * cos(6.283185307179586 * u2);
}

// Filter state of one robot, SE_DBL doubles in one device block [B][SE_DBL]:
//   [0, 18)     x = [p_base(3), v_base(3), p_foot(4 x 3, contact order LF, RF, LH, RH)], world frame
//   [18, 189)   P, packed lower triangle (entry (i, j <= i) at i(i+1)/2 + j)
//   [189]       calls since the reset (0: the next call only places the feet)
constexpr int SE_NX = 18, SE_TRI = SE_NX * (SE_NX + 1) / 2, SE_NY = 28;
constexpr int SE_X = 0, SE_P = SE_X + SE_NX, SE_N = SE_P + SE_TRI, SE_DBL = SE_N + 1;

// sensors of robots [0, B) at the plant state (q, v) after a step of dt seconds that started at velocity v_prev; robot b draws its noise as robot robot0 + b
int launch_read_sensors(const qmb200_sensor_params& prm, int B, int64_t robot0, double dt, int64_t sample, const double* q, const double* v, const double* v_prev,
                        double* sensors, cudaStream_t s);
// one filter call per robot from sensors [B][46] and the contact mask [B]; writes rbd_est [B][55] and status [B].  map: the estimator's ground map on
// the plant's tile library (map.robot [B][3] = [tile, origin_x, origin_y]; NULL: every foot-height row on the plane), ground_height: the plant's plane
int launch_state_est_step(const DevModel* mdl, const qmb200_state_est_params& prm, int B, double dt, const double* sensors, const int32_t* contact, double* state,
                          double* rbd_est, int32_t* status, const SimTerrain& map, double ground_height, cudaStream_t s);

}  // namespace qmb
