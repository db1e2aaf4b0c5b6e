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

// One standard normal draw, a pure function of (seed, robot, sample, channel): two 53-bit uniforms in (0, 1) are cut from the key (keyed_hash with the
// sensor domain) and from the key xor-ed with a second constant, and Box-Muller's cosine branch turns them into N(0, 1).
QMB_HD double sensor_normal(uint64_t seed, uint64_t robot, uint64_t sample, int channel) {
  const uint64_t h = keyed_hash(seed, 0x9e3779b97f4a7c15ull, robot, sample, channel);
  const double u1 = hash_uniform(h), u2 = hash_uniform(h ^ 0xd1b54a32d192ed03ull);
  return sqrt(-2.0 * log(u1)) * cos(6.283185307179586 * u2);
}

// Filter state of one robot, SE_DBL doubles in one device block [B][SE_DBL]:
//   [0, 18)     x = [p_base(3), v_base(3), p_foot(4 x 3, contact order LF, RF, LH, RH)], world frame
//   [18, 189)   P, packed lower triangle (entry (i, j <= i) at i(i+1)/2 + j)
//   [189]       calls since the reset (0: the next call only places the feet)
constexpr int SE_NX = 18, SE_TRI = SE_NX * (SE_NX + 1) / 2, SE_NY = 28;
constexpr int SE_X = 0, SE_P = SE_X + SE_NX, SE_N = SE_P + SE_TRI, SE_DBL = SE_N + 1;
// The reset row st [SE_DBL] of one robot at base position base_pos [3]: zero velocity and feet, P diagonal with p's p0 variances, no call yet (the next
// call places the feet).  qmb200_state_est_reset and the spawn sampler both write it.
QMB_HD void state_est_reset_row(const qmb200_state_est_params& p, const double* base_pos, double* st) {
  for (int i = 0; i < SE_DBL; ++i) st[i] = 0.0;
  for (int i = 0; i < 3; ++i) st[SE_X + i] = base_pos[i];
  for (int i = 0; i < SE_NX; ++i) st[SE_P + i * (i + 1) / 2 + i] = i < 3 ? p.p0_base_pos : (i < 6 ? p.p0_base_vel : p.p0_foot);
}

// sensors of robots [0, B) at the plant state (q, v) after a step of dt seconds that started at velocity v_prev; robot b draws its noise as robot robot0 + b
int launch_read_sensors(const qmb200_sensor_params& prm, int B, int64_t robot0, double dt, int64_t sample, const double* q, const double* v, const double* v_prev,
                        double* sensors, cudaStream_t s);
// one filter call per robot from sensors [B][46] and the contact mask [B]; writes rbd_est [B][55] and status [B].  map: the estimator's ground map on
// the plant's tile library (map.robot [B][3] = [tile, origin_x, origin_y]; NULL: every foot-height row on the plane), ground_height: the plant's plane
int launch_state_est_step(const DevModel* mdl, const qmb200_state_est_params& prm, int B, double dt, const double* sensors, const int32_t* contact, double* state,
                          double* rbd_est, int32_t* status, const SimTerrain& map, double ground_height, cudaStream_t s);

}  // namespace qmb
