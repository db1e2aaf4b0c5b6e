// Per-episode end-effector paths (ee_path_draw_kernel.cu; include/qmb200.h: qmb200_ee_path_*; DESIGN.md §4.21): the waypoints of one episode's path of
// one robot, a pure function of (seed, global robot, episode, waypoint, channel) and the robot's ranges.  A drawn path is one row of the end-effector
// path table (ctrl_api.cuh: EE_PATH_MAX waypoints of EE_PATH_WAY doubles), which target_path follows unchanged.  Host + device: the sampler kernel,
// qmb200_ee_path_draw and tests/ee_path_draw_host.cpp compile the same core, so host and device agree bit for bit.
#pragma once
#include <math.h>
#include <stdint.h>

#include <cmath>
#include <string>

#include "ctrl_api.cuh"
#include "gait_api.cuh"
#include "timeline_api.cuh"

namespace qmb {

// a ranges row [EPR_DBL] (_lib.EE_PATH_RANGES_LAYOUT): the waypoint count, the first waypoint's time after the path's start, the time between
// consecutive waypoints, the waypoint position in the path's frame, the yaw that turns the hand about that frame's z axis, the quaternion xyzw it turns
constexpr int EPR_N_WAY = 0, EPR_TAU_FIRST = 1, EPR_GAP = 2, EPR_POS = 3, EPR_YAW = 6, EPR_QUAT = 7, EPR_DBL = 11;
// channels of waypoint i: 8 i + c, c one of these (time: tau_first for waypoint 0, gap after it)
constexpr int EPC_TIME = 0, EPC_POS = 1, EPC_YAW = 4, EPC_CHANNELS = 8;
// xor-ed into the seed so that a path draw and a plant, spawn, timeline or sensor-noise draw of the same words are unrelated
constexpr uint64_t EE_PATH_DOMAIN = 0xa54ff53a5f1d36f1ull;
// the largest last waypoint time the ranges may allow (s), so that every drawn time is finite
constexpr double EE_PATH_TAU_MAX = 1e300;

// a * b and a + b each rounded once: the device compiler would otherwise contract a product and a sum into an fma, which the host does not
QMB_HD double epd_mul(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}
QMB_HD double epd_add(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}
// sine and cosine of h in [-pi/2, pi/2] (half a yaw in [-pi, pi]): Taylor polynomials to h^21 / h^22 (truncation below 2e-17) in Horner form on
// epd_mul / epd_add, so that host and device give the same bits.  The library sines (spawn_sincos: sincospi on the device, std::sin on the host) differ
// by an ulp between the two.  No argument reduction, no table, no stack.
QMB_HD void epd_sincos(double h, double& s, double& c) {
  const double z = epd_mul(h, h);
  // sin h = h + h z P(z), cos h = 1 + z Q(z): the coefficients (-1)^k / (2k + 1)! and (-1)^k / (2k)!, highest first (tests/test_ee_path_draw_cpu.py: SIN, COS)
  double p = 1.9572941063391263e-20;
  p = epd_add(epd_mul(p, z), -8.22063524662433e-18); p = epd_add(epd_mul(p, z), 2.8114572543455206e-15);
  p = epd_add(epd_mul(p, z), -7.647163731819816e-13); p = epd_add(epd_mul(p, z), 1.6059043836821613e-10);
  p = epd_add(epd_mul(p, z), -2.505210838544172e-08); p = epd_add(epd_mul(p, z), 2.7557319223985893e-06);
  p = epd_add(epd_mul(p, z), -0.0001984126984126984); p = epd_add(epd_mul(p, z), 0.008333333333333333);
  p = epd_add(epd_mul(p, z), -0.16666666666666666);
  s = epd_add(h, epd_mul(epd_mul(h, z), p));
  double q = -8.896791392450574e-22;
  q = epd_add(epd_mul(q, z), 4.110317623312165e-19); q = epd_add(epd_mul(q, z), -1.5619206968586225e-16);
  q = epd_add(epd_mul(q, z), 4.779477332387385e-14); q = epd_add(epd_mul(q, z), -1.1470745597729725e-11);
  q = epd_add(epd_mul(q, z), 2.08767569878681e-09); q = epd_add(epd_mul(q, z), -2.755731922398589e-07);
  q = epd_add(epd_mul(q, z), 2.48015873015873e-05); q = epd_add(epd_mul(q, z), -0.001388888888888889);
  q = epd_add(epd_mul(q, z), 0.041666666666666664); q = epd_add(epd_mul(q, z), -0.5);
  c = epd_add(1.0, epd_mul(z, q));
}

// u in (0, 1) of (seed, robot, episode, channel): the keyed uniform (dev_common.cuh) on the path draws' domain
QMB_HD double ee_path_uniform(uint64_t seed, uint64_t robot, uint64_t episode, int channel) { return keyed_uniform(seed, EE_PATH_DOMAIN, robot, episode, channel); }
// column c drawn on channel ch: a fixed column (lo == hi) is lo itself, byte for byte; a box column fma(u, hi - lo, lo), one rounding
QMB_HD double ee_path_box(const double* lo, const double* hi, int c, uint64_t seed, uint64_t robot, uint64_t episode, int ch) {
  return hi[c] == lo[c] ? lo[c] : fma(ee_path_uniform(seed, robot, episode, ch), hi[c] - lo[c], lo[c]);
}
// t + g with g >= 0, rounded up where the nearest rounding falls short of the exact sum (its error by TwoSum), so that (t + g) - t >= g: the drawn
// waypoints then keep the table's gap rule at every gap the ranges allow
QMB_HD double ee_path_after(double t, double g) {
  const double s = epd_add(t, g), v = epd_add(s, -t), e = epd_add(epd_add(t, -epd_add(s, -v)), epd_add(g, -v));
  return e > 0.0 ? nextafter(s, HUGE_VAL) : s;
}
// the robot's waypoint count: its fixed n_way column
QMB_HD int ee_path_n_way(const double* lo) { return (int)lo[EPR_N_WAY]; }

// Waypoint i of one robot (its ranges lo, hi [EPR_DBL]) after waypoint i - 1's time t_prev (ignored for i = 0) → w[EE_PATH_WAY] (tau, position 3,
// quaternion xyzw 4).  tau: draw(tau_first) on channel 0, else ee_path_after(t_prev, draw(gap)) on channel 8 i; the position on channels 8 i + 1..3; the quaternion
// Rz(draw(yaw)) (x) quat (channel 8 i + 4), the product heading_to_world applies.  Every column reads its own channel, so changing one box moves no other.
QMB_HD void ee_path_waypoint(const double* lo, const double* hi, uint64_t seed, uint64_t robot, uint64_t episode, int i, double t_prev, double* w) {
  const int ch = EPC_CHANNELS * i;
  w[0] = i == 0 ? ee_path_box(lo, hi, EPR_TAU_FIRST, seed, robot, episode, ch + EPC_TIME) : ee_path_after(t_prev, ee_path_box(lo, hi, EPR_GAP, seed, robot, episode, ch + EPC_TIME));
#pragma unroll
  for (int k = 0; k < 3; ++k) w[1 + k] = ee_path_box(lo, hi, EPR_POS + k, seed, robot, episode, ch + EPC_POS + k);
  double sh, chh; epd_sincos(epd_mul(0.5, ee_path_box(lo, hi, EPR_YAW, seed, robot, episode, ch + EPC_YAW)), sh, chh);
  const double qx = lo[EPR_QUAT], qy = lo[EPR_QUAT + 1], qz = lo[EPR_QUAT + 2], qw = lo[EPR_QUAT + 3];
  w[4] = epd_add(epd_mul(chh, qx), -epd_mul(sh, qy)); w[5] = epd_add(epd_mul(chh, qy), epd_mul(sh, qx));
  w[6] = epd_add(epd_mul(chh, qz), epd_mul(sh, qw)); w[7] = epd_add(epd_mul(chh, qw), -epd_mul(sh, qz));
}
// one episode's path of one robot as a row of the path table: way [EE_PATH_MAX][EE_PATH_WAY], zeros past its n_way waypoints; returns n_way
QMB_HD int ee_path_rows(const double* lo, const double* hi, uint64_t seed, uint64_t robot, uint64_t episode, double* way) {
  const int n = ee_path_n_way(lo); double t = 0.0;
  for (int i = 0; i < EE_PATH_MAX; ++i) {
    double* w = way + (size_t)i * EE_PATH_WAY;
    if (i < n) { ee_path_waypoint(lo, hi, seed, robot, episode, i, t, w); t = w[0]; }
    else for (int k = 0; k < EE_PATH_WAY; ++k) w[k] = 0.0;
  }
  return n;
}

// The check of qmb200_ee_path_set_ranges on ranges lo, hi [B][EPR_DBL] for a handle of time horizon T (ranges_error): n_way and the quaternion are fixed
// columns (lo == hi); n_way is an integer in [1, QMB200_EE_PATH_MAX]; tau_first's lo is > 0; gap's lo is >= T/2; the yaw bounds lie in [-pi, pi]; the
// quaternion has unit norm within 1e-9; tau_first hi + (n_way - 1) gap hi is at most EE_PATH_TAU_MAX.  Every row these ranges draw then passes
// ee_paths_error at T.
inline std::string ee_path_ranges_error(const double* lo, const double* hi, size_t B, double T) {
  static const char* const names[EPR_DBL] = {"n_way", "tau_first", "gap", "x", "y", "z", "yaw", "qx", "qy", "qz", "qw"};
  const char* who = "qmb200_ee_path_set_ranges";
  const std::string e = ranges_error(who, names, EPR_DBL, lo, hi, B, [T](int c, double l, double u) -> std::string {
    if ((c == EPR_N_WAY || c >= EPR_QUAT) && l != u) return "must be fixed (lo == hi)";
    if (c == EPR_N_WAY && !(std::floor(l) == l && l >= 1.0 && l <= (double)EE_PATH_MAX)) return "must be an integer in [1, QMB200_EE_PATH_MAX (32)]";
    if (c == EPR_TAU_FIRST && !(l > 0.0)) return "lo must be > 0 (seconds after the path starts)";
    if (c == EPR_GAP && !(l >= 0.5 * T)) return "lo must be >= T/2 = " + std::to_string(0.5 * T) + " s";
    if (c == EPR_YAW && !(l >= -M_PI && u <= M_PI)) return "bounds must lie in [-pi, pi]";
    return "";
  });
  if (!e.empty()) return e;
  for (size_t b = 0; b < B; ++b) {
    const double* q = lo + b * EPR_DBL + EPR_QUAT; const double* u = hi + b * EPR_DBL;
    if (!(std::fabs(std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]) - 1.0) <= 1e-9))
      return std::string(who) + ": quat of robot " + std::to_string(b) + ": must have unit norm (within 1e-9)";
    // the last waypoint's time is at most this bound plus an ulp per waypoint: far below it every drawn time stays finite
    if (!(u[EPR_TAU_FIRST] + (lo[b * EPR_DBL + EPR_N_WAY] - 1.0) * u[EPR_GAP] <= EE_PATH_TAU_MAX))
      return std::string(who) + ": gap of robot " + std::to_string(b) + ": tau_first hi + (n_way - 1) gap hi must be <= 1e300 s";
  }
  return "";
}

#ifdef __CUDACC__
// What the sampler writes besides the caller's record rows: the path table's drawn rows (row p0 + b of n_way [p0 + B] and way [p0 + B][EE_PATH_MAX][8])
// and the device gait schedule's pending slots [B]
struct EePathTargets { int32_t* n_way; double* way; int p0; GsPending* pending; };
// one thread per robot: robots with mask[b] != 0 draw episode[b]'s path as global robot robot0 + b into rows[b][0:n_way] ([B][EE_PATH_MAX][8]) and
// table row p0 + b, and set their pending slot to a start of that row
int launch_ee_path_sample(int B, int64_t robot0, const double* lo, const double* hi, uint64_t seed, const int32_t* mask, const int32_t* episode, double* rows,
                          const EePathTargets& t, cudaStream_t s);
#endif

}  // namespace qmb
