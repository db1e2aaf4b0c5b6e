// Per-episode command timelines (timeline_kernel.cu; include/qmb200.h: qmb200_timeline_*; DESIGN.md §4.14): the n_cmd command slots of one episode of
// one robot, a pure function of (seed, global robot, episode, slot, channel) and the robot's ranges.  A drawn slot is one command of the device gait
// schedule's timeline (gait_api.cuh: GsCommands), which gs_step consumes unchanged.  Host + device: the sampler kernel, qmb200_timeline_draw and
// tests/timeline_host.cpp compile the same core, so host and device agree bit for bit.
#pragma once
#include <math.h>
#include <stdint.h>

#include <cmath>
#include <cstring>
#include <string>

#include "dev_common.cuh"
#include "../../../include/qmb200.h"

namespace qmb {

// a ranges row [TL_DBL] (_lib.TIMELINE_LAYOUT): slot 0's time on the robot's observation clock, the time between consecutive slots, the probability that a
// slot inserts a gait and the bitmask of the templates it picks among, the weights of the slot's target command (none, cmd_vel, ee_cmd_vel, ee goal), the
// cmd_vel row (base frame), the end-effector velocity and goal position (world frame), the goal quaternion xyzw
constexpr int TL_T_FIRST = 0, TL_GAP = 1, TL_P_GAIT = 2, TL_GAIT_SET = 3, TL_W = 4, TL_CMD_VEL = 8, TL_EE_VEL = 12, TL_EE_POS = 15, TL_EE_QUAT = 18, TL_DBL = 22;
// a drawn slot [TLC_DBL] (_lib.TIMELINE_CMD_LAYOUT): one command of qmb200_gait_dev_set_commands_ee
constexpr int TLC_T = 0, TLC_TMPL = 1, TLC_CMD_VEL = 2, TLC_EE_KIND = 6, TLC_EE = 7, TLC_DBL = 14;
// the slot's target kinds, in the order of their weights
constexpr int TL_KIND_NONE = 0, TL_KIND_CMD_VEL = 1, TL_KIND_EE_CMD_VEL = 2, TL_KIND_EE_GOAL = 3;
// channels per slot: slot j reads channels TL_CHANNELS j + c
constexpr int TL_CHANNELS = 16, TLC_GAIT = 1, TLC_TEMPLATE = 2, TLC_KIND = 3, TLC_VEL = 4, TLC_EEV = 8, TLC_EEP = 11;
// xor-ed into the seed so that a timeline draw and a plant, spawn or sensor-noise draw of the same words are unrelated
constexpr uint64_t TIMELINE_DOMAIN = 0x3c6ef372fe94f82bull;

// the "none" of a cmd_vel row: the quiet NaN 0x7FF8000000000000, the same bits on host, device and numpy
QMB_HD double timeline_nan() {
#ifdef __CUDA_ARCH__
  return __longlong_as_double(0x7FF8000000000000ll);
#else
  const uint64_t bits = 0x7FF8000000000000ull; double d; std::memcpy(&d, &bits, 8); return d;
#endif
}
// u in (0, 1) of (seed, robot, episode, channel): the keyed uniform (dev_common.cuh) on the timeline draws' domain
QMB_HD double timeline_uniform(uint64_t seed, uint64_t robot, uint64_t episode, int channel) { return keyed_uniform(seed, TIMELINE_DOMAIN, robot, episode, channel); }
// column c drawn on channel ch: a fixed column (lo == hi) is lo itself, byte for byte; a box column fma(u, hi - lo, lo), one rounding
QMB_HD double timeline_box(const double* lo, const double* hi, int c, uint64_t seed, uint64_t robot, uint64_t episode, int ch) {
  return hi[c] == lo[c] ? lo[c] : fma(timeline_uniform(seed, robot, episode, ch), hi[c] - lo[c], lo[c]);
}
// the number of set bits of m, and the bit index of its k-th set bit in increasing order (k < the count)
QMB_HD int timeline_popcount(uint32_t m) {
  m = m - ((m >> 1) & 0x55555555u); m = (m & 0x33333333u) + ((m >> 2) & 0x33333333u); return (int)((((m + (m >> 4)) & 0x0F0F0F0Fu) * 0x01010101u) >> 24);
}
QMB_HD int timeline_kth_bit(uint32_t m, int k) {
  for (int i = 0; i < 32; ++i)
    if ((m >> i) & 1u) { if (k == 0) return i; --k; }
  return -1;
}

// Slot j of one robot (its ranges lo, hi [TL_DBL]) after slot j - 1's time t_prev (ignored for j = 0) → out[TLC_DBL].  Time: draw(t_first) on
// channel 0, else t_prev + draw(gap) on channel 16 j, so the times are sorted.  Gait: inserted when u < p_gait (channel 16 j + 1); the template is the
// k-th set bit of gait_set with k = min(floor(u popcount), popcount - 1) (channel + 2).  Kind: the first whose running sum of the weights exceeds u W,
// W their sum in order (channel + 3), else the last with a positive weight.  cmd_vel on channels + 4..7, the end-effector velocity on + 8..10, the goal
// position on + 11..13.  Every choice reads its own channel, so changing one weight shifts no other column's draw.
QMB_HD void timeline_slot(const double* lo, const double* hi, uint64_t seed, uint64_t robot, uint64_t episode, int j, double t_prev, double* out) {
  const int ch = TL_CHANNELS * j;
  out[TLC_T] = j == 0 ? timeline_box(lo, hi, TL_T_FIRST, seed, robot, episode, 0) : t_prev + timeline_box(lo, hi, TL_GAP, seed, robot, episode, ch);
  int tmpl = -1;
  if (timeline_uniform(seed, robot, episode, ch + TLC_GAIT) < lo[TL_P_GAIT]) {
    const uint32_t m = (uint32_t)(uint64_t)lo[TL_GAIT_SET]; const int pc = timeline_popcount(m);
    const double k = fmin(floor(timeline_uniform(seed, robot, episode, ch + TLC_TEMPLATE) * (double)pc), (double)(pc - 1));
    tmpl = timeline_kth_bit(m, (int)k);
  }
  out[TLC_TMPL] = (double)tmpl;
  const double w0 = lo[TL_W], w1 = lo[TL_W + 1], w2 = lo[TL_W + 2], w3 = lo[TL_W + 3];
  const double s1 = w0 + w1, s2 = s1 + w2, s3 = s2 + w3, x = timeline_uniform(seed, robot, episode, ch + TLC_KIND) * s3;
  const int last = w3 > 0.0 ? TL_KIND_EE_GOAL : w2 > 0.0 ? TL_KIND_EE_CMD_VEL : w1 > 0.0 ? TL_KIND_CMD_VEL : TL_KIND_NONE;
  const int kind = w0 > x ? TL_KIND_NONE : s1 > x ? TL_KIND_CMD_VEL : s2 > x ? TL_KIND_EE_CMD_VEL : s3 > x ? TL_KIND_EE_GOAL : last;
  const double nan = timeline_nan();
#pragma unroll
  for (int i = 0; i < 4; ++i) out[TLC_CMD_VEL + i] = kind == TL_KIND_CMD_VEL ? timeline_box(lo, hi, TL_CMD_VEL + i, seed, robot, episode, ch + TLC_VEL + i) : nan;
  out[TLC_EE_KIND] = kind == TL_KIND_EE_CMD_VEL ? (double)QMB200_TARGET_EE_CMD_VEL : kind == TL_KIND_EE_GOAL ? (double)QMB200_TARGET_EE_GOAL : -1.0;
#pragma unroll
  for (int i = 0; i < 3; ++i)
    out[TLC_EE + i] = kind == TL_KIND_EE_CMD_VEL ? timeline_box(lo, hi, TL_EE_VEL + i, seed, robot, episode, ch + TLC_EEV + i)
                    : kind == TL_KIND_EE_GOAL ? timeline_box(lo, hi, TL_EE_POS + i, seed, robot, episode, ch + TLC_EEP + i) : 0.0;
#pragma unroll
  for (int i = 0; i < 4; ++i) out[TLC_EE + 3 + i] = kind == TL_KIND_EE_GOAL ? lo[TL_EE_QUAT + i] : 0.0;
}
// the n_cmd slots [n_cmd][TLC_DBL] of one episode of one robot
QMB_HD void timeline_rows(const double* lo, const double* hi, uint64_t seed, uint64_t robot, uint64_t episode, int n_cmd, double* rows) {
  double t = 0.0;
  for (int j = 0; j < n_cmd; ++j) { timeline_slot(lo, hi, seed, robot, episode, j, t, rows + (size_t)j * TLC_DBL); t = rows[(size_t)j * TLC_DBL + TLC_T]; }
}

// The check of qmb200_timeline_set_ranges on ranges lo, hi [B][TL_DBL] (ranges_error): p_gait, gait_set, the weights and the quaternion are fixed columns
// (lo == hi); p_gait lies in [0, 1]; gait_set is an integer in [0, 2^32), non-zero when p_gait > 0; the weights are >= 0 with a positive sum; the
// quaternion has unit norm within 1e-9; gap's lo is >= 0
inline std::string timeline_ranges_error(const double* lo, const double* hi, size_t B) {
  static const char* const names[TL_DBL] = {"t_first", "gap", "p_gait", "gait_set", "w_none", "w_cmd_vel", "w_ee_cmd_vel", "w_ee_goal", "cmd_vel_x", "cmd_vel_y",
                                            "cmd_vel_z", "cmd_yaw_rate", "ee_vx", "ee_vy", "ee_vz", "ee_x", "ee_y", "ee_z", "ee_qx", "ee_qy", "ee_qz", "ee_qw"};
  const char* who = "qmb200_timeline_set_ranges";
  const std::string e = ranges_error(who, names, TL_DBL, lo, hi, B, [](int c, double l, double u) -> std::string {
    const bool fixed = (c >= TL_P_GAIT && c < TL_CMD_VEL) || c >= TL_EE_QUAT;
    if (fixed && l != u) return "must be fixed (lo == hi)";
    if (c == TL_GAP && l < 0.0) return "lo must be >= 0";
    if (c == TL_P_GAIT && !(l >= 0.0 && l <= 1.0)) return "must lie in [0, 1]";
    if (c == TL_GAIT_SET && !(std::floor(l) == l && l >= 0.0 && l < 4294967296.0)) return "must be an integer in [0, 2^32)";
    if (c >= TL_W && c < TL_CMD_VEL && l < 0.0) return "must be >= 0";
    return "";
  });
  if (!e.empty()) return e;
  for (size_t b = 0; b < B; ++b) {
    const double* r = lo + b * TL_DBL; const std::string of = " of robot " + std::to_string(b) + ": ";
    if (r[TL_P_GAIT] > 0.0 && r[TL_GAIT_SET] == 0.0) return std::string(who) + ": gait_set" + of + "must be non-zero when p_gait > 0";
    if (!(r[TL_W] + r[TL_W + 1] + r[TL_W + 2] + r[TL_W + 3] > 0.0)) return std::string(who) + ": weights" + of + "must have a positive sum";
    const double* q = r + TL_EE_QUAT;
    if (!(std::fabs(std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]) - 1.0) <= 1e-9))
      return std::string(who) + ": ee_quat" + of + "must have unit norm (within 1e-9)";
  }
  return "";
}

#ifdef __CUDACC__
// The device gait schedule's timeline rows the sampler writes ([B][n_cmd], gait_api.cuh's GsCommands layout; ee_kind / ee NULL: the timeline has no
// end-effector rows) and the robots' cursors [B]
struct TimelineTargets { double* t; int32_t* tmpl; double* vel; int32_t* ee_kind; double* ee; int32_t* cursor; };
// one thread per robot: robots with mask[b] != 0 draw episode[b]'s n_cmd slots as global robot robot0 + b
int launch_timeline_sample(int B, int n_cmd, int64_t robot0, const double* lo, const double* hi, uint64_t seed, const int32_t* mask, const int32_t* episode, double* rows,
                           const TimelineTargets& t, cudaStream_t s);
#endif

}  // namespace qmb
