// Per-episode plant draws (episode_kernel.cu; include/qmb200.h: qmb200_episode_*; DESIGN.md §4.11): the row of one episode of one robot, a pure function
// of (seed, global robot, episode, channel) and the robot's ranges.  Host + device: the sampler kernel, qmb200_episode_draw and tests/episode_host.cpp
// compile the same core, so host and device agree bit for bit.
#pragma once
#include <math.h>
#include <stdint.h>

#include <cmath>
#include <string>

#include "dev_common.cuh"

namespace qmb {

// an episode row [EP_DBL] (_lib.EPISODE_LAYOUT): friction_mu, the payload row [8], push t_on and duration (s from the episode's start), the push wrench
// [12] (qmb200_sim_step_ext's layout), cmd_vel (vx, vy, vz, yaw rate; base frame)
constexpr int EP_MU = 0, EP_PAYLOAD = 1, EP_PUSH_T_ON = 9, EP_PUSH_DURATION = 10, EP_WRENCH = 11, EP_CMD_VEL = 23, EP_DBL = 27;
// xor-ed into the seed so that a plant draw and a sensor-noise draw of the same words are unrelated
constexpr uint64_t EPISODE_DOMAIN = 0x6a09e667f3bcc909ull;

// u in (0, 1) of (seed, robot, episode, channel): the keyed uniform (dev_common.cuh) on the plant draws' domain
QMB_HD double episode_uniform(uint64_t seed, uint64_t robot, uint64_t episode, int channel) { return keyed_uniform(seed, EPISODE_DOMAIN, robot, episode, channel); }
// row[c] = fma(u_c, hi[c] - lo[c], lo[c]): one rounding whatever the compiler contracts.  A fixed column (lo[c] == hi[c]) is lo[c] itself, byte for
// byte: the fma would turn lo = hi = -0.0 into +0.0
QMB_HD void episode_row(const double* lo, const double* hi, uint64_t seed, uint64_t robot, uint64_t episode, double* row) {
  for (int c = 0; c < EP_DBL; ++c) row[c] = hi[c] == lo[c] ? lo[c] : fma(episode_uniform(seed, robot, episode, c), hi[c] - lo[c], lo[c]);
}

// The check of qmb200_episode_set_ranges on ranges lo, hi [B][EP_DBL] (ranges_error): friction_mu's lo must be > 0, the masses' and the push times' >= 0
inline std::string episode_ranges_error(const double* lo, const double* hi, size_t B) {
  static const char* const names[EP_DBL] = {"friction_mu", "m_ee", "o_ee_x", "o_ee_y", "o_ee_z", "m_base", "o_base_x", "o_base_y", "o_base_z", "push_t_on",
                                            "push_duration", "f_base_x", "f_base_y", "f_base_z", "n_base_x", "n_base_y", "n_base_z", "f_ee_x", "f_ee_y", "f_ee_z",
                                            "n_ee_x", "n_ee_y", "n_ee_z", "cmd_vel_x", "cmd_vel_y", "cmd_vel_z", "cmd_yaw_rate"};
  return ranges_error("qmb200_episode_set_ranges", names, EP_DBL, lo, hi, B, [](int c, double l, double) -> std::string {
    const bool at_least_zero = c == EP_PAYLOAD || c == EP_PAYLOAD + 4 || c == EP_PUSH_T_ON || c == EP_PUSH_DURATION;
    return (c == EP_MU && !(l > 0.0)) ? "lo must be > 0" : (at_least_zero && l < 0.0) ? "lo must be >= 0" : "";
  });
}

#ifdef __CUDACC__
// Where a sampled row goes besides rows[B][EP_DBL]: the plant's robot params (always), and as linked the model payload with its SRBD rows and the
// tuning rows' friction coefficients.  NULL: not written.
struct EpisodeTargets {
  double *mu, *payload;          // [B], [B][8]
  double *mpayload, *srbd;       // [B][8], [B][SRBD_DBL]
  double* tuning; int mpc_mu, wbc_mu;   // [B][TUNING_DBL]; write friction_mu into the row's MPC / WBC friction coefficient
};
// one thread per robot: robots with mask[b] != 0 draw episode[b] as global robot robot0 + b
int launch_episode_sample(const DevModel* mdl, int B, int64_t robot0, const double* lo, const double* hi, uint64_t seed, const int32_t* mask, const int32_t* episode,
                          double* rows, const EpisodeTargets& t, cudaStream_t s);
#endif

}  // namespace qmb
