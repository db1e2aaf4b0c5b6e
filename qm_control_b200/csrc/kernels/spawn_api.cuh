// Per-episode spawns (spawn_kernel.cu; include/qmb200.h: qmb200_spawn_*; DESIGN.md §4.12): the spawn row of one episode of one robot (its tile, its
// offset along the tile and its yaw), a pure function of (seed, global robot, episode, column) and the robot's ranges.  Host + device: the sampler
// kernel, qmb200_spawn_draw and tests/spawn_host.cpp compile the same core, so host and device agree bit for bit.  The robot stands on the drawn ground
// with standing_on_tile (sim_api.cuh), the pose qmb200_sim_standing_state gives.  A restart "here" (DESIGN.md §4.18) writes its row with spawn_here_row
// and places it after the device check spawn_place_ok; both are host + device too (tests/spawn_place_host.cpp).
#pragma once
#include <math.h>
#include <stdint.h>

#include <cmath>
#include <string>

#include "dev_common.cuh"
#include "sim_api.cuh"
#include "../../../include/qmb200.h"

namespace qmb {

// a spawn row [SP_DBL] (_lib.SPAWN_LAYOUT): the plant's tile (-1: the plane), the offset (dx, dy) the robot stands further along its tile (world axes:
// the tile's origin moves by -(dx, dy)), the base yaw
constexpr int SP_TILE = 0, SP_DX = 1, SP_DY = 2, SP_YAW = 3, SP_DBL = 4;
// xor-ed into the seed so that a spawn draw, a plant draw and a sensor-noise draw of the same words are unrelated
constexpr uint64_t SPAWN_DOMAIN = 0xbb67ae8584caa73bull;

// u in (0, 1) of (seed, robot, episode, column): the keyed uniform (dev_common.cuh) on the spawn draws' domain
QMB_HD double spawn_uniform(uint64_t seed, uint64_t robot, uint64_t episode, int column) { return keyed_uniform(seed, SPAWN_DOMAIN, robot, episode, column); }
// row[c]: a fixed column (lo[c] == hi[c]) is lo[c] itself, byte for byte; the tile is the integer lo + min(floor(u (hi - lo + 1)), hi - lo), each of
// the hi - lo + 1 tiles with probability 1 / (hi - lo + 1); dx, dy and yaw are fma(u, hi - lo, lo), one rounding whatever the compiler contracts
QMB_HD void spawn_row(const double* lo, const double* hi, uint64_t seed, uint64_t robot, uint64_t episode, double* row) {
#pragma unroll
  for (int c = 0; c < SP_DBL; ++c) {
    const double u = spawn_uniform(seed, robot, episode, c), d = hi[c] - lo[c];
    row[c] = hi[c] == lo[c] ? lo[c] : c == SP_TILE ? lo[c] + fmin(floor(u * (d + 1.0)), d) : fma(u, d, lo[c]);
  }
}

// The check of qmb200_spawn_set_ranges on ranges lo, hi [B][SP_DBL] on a tile library of n_tiles tiles (ranges_error): the tile's bounds must be
// integers in [-1, n_tiles), the yaw's lie in [-pi, pi]
inline std::string spawn_ranges_error(const double* lo, const double* hi, size_t B, int n_tiles) {
  static const char* const names[SP_DBL] = {"tile", "dx", "dy", "yaw"};
  return ranges_error("qmb200_spawn_set_ranges", names, SP_DBL, lo, hi, B, [n_tiles](int c, double l, double u) -> std::string {
    const double pi = 3.141592653589793;
    if (c == SP_TILE && !(std::floor(l) == l && std::floor(u) == u)) return "bounds must be integers";
    if (c == SP_TILE && !(l >= -1.0 && u < n_tiles)) return "bounds must lie in [-1, " + std::to_string(n_tiles) + "), the tiles of the library in force";
    if (c == SP_YAW && !(l >= -pi && u <= pi)) return "bounds must lie in [-pi, pi]";
    return "";
  });
}

// A yaw in [-pi, pi] with the same heading: y itself there; else y - 2 pi floor((y + pi) / (2 pi)), held inside [-pi, pi] against the rounding.  The
// product is rounded on its own (no fma contraction), so that the kernel and a host build agree bit for bit.  A non-finite y is returned as it is.
QMB_HD double spawn_wrap_yaw(double y) {
  const double pi = 3.141592653589793, two_pi = 6.283185307179586;
  if (fabs(y) <= pi || !isfinite(y)) return y;
  const double k = floor((y + pi) / two_pi);
#ifdef __CUDA_ARCH__
  const double m = __dmul_rn(two_pi, k);
#else
  const double m = two_pi * k;
#endif
  return fmin(fmax(y - m, -pi), pi);
}

// The "here" row (qmb200_spawn_here): the spawn row that, once the robot is back at its start pose q_start [NQ], stands it on the ground point under its
// base now (rbd [QMB200_RBD]) with its heading now.  ter: the plant's robot terrain row now [tile, origin] (NULL: none, the plane); origin [2]: the
// origin the row's offsets count from (the run's).  The tile stays; the ground moves by the base's travel plus the origin's shift, so the base's
// point in tile coordinates, x - ter origin, is the same after the place; the yaw is the base's, wrapped.  Without terrain rows only the heading
// matters to the place; dx, dy then hold the base's travel from its start.
QMB_HD void spawn_here_row(const double* rbd, const double* q_start, const double* origin, const double* ter, double* row) {
  const double ox = ter ? ter[1] : origin[0], oy = ter ? ter[2] : origin[1];
  row[SP_TILE] = ter ? ter[0] : -1.0;
  row[SP_DX] = (rbd[RBD_POS] - q_start[0]) + (origin[0] - ox);
  row[SP_DY] = (rbd[RBD_POS + 1] - q_start[1]) + (origin[1] - oy);
  row[SP_YAW] = spawn_wrap_yaw(rbd[RBD_ZYX]);
}

// The device check of a row given to qmb200_spawn_place on a library of n_tiles tiles: the tile an integer in [-1, n_tiles), a tile >= 0 only where the
// plant has robot terrain rows (rows: whether it has), finite dx and dy, the yaw in [-pi, pi].  NaN fails every comparison.
QMB_HD bool spawn_place_ok(const double* row, int n_tiles, bool rows) {
  const double pi = 3.141592653589793, t = row[SP_TILE];
  return floor(t) == t && t >= -1.0 && t < (double)n_tiles && (t < 0.0 || rows) && isfinite(row[SP_DX]) && isfinite(row[SP_DY]) && row[SP_YAW] >= -pi &&
         row[SP_YAW] <= pi;
}

// The held end-effector target e [7] of a robot the spawn turns from yaw0 to yaw about the vertical through its base (x, y): a world-frame hold turns
// with the base; a heading-frame hold (heading: qmb200_set_ee_frame, DESIGN.md §4.19) is stated in the base's frame already and stays as it is.
QMB_HD void spawn_turn_hold(double* e, double x, double y, double yaw0, double yaw, bool heading) {
  if (yaw == yaw0 || heading) return;
  const double dyaw = yaw - yaw0; double sn, c, sh, ch; spawn_sincos(dyaw, sn, c); spawn_sincos(0.5 * dyaw, sh, ch);
  const double ex = e[0] - x, ey = e[1] - y, qx = e[3], qy = e[4], qz = e[5], qw = e[6];
  e[0] = x + (c * ex - sn * ey); e[1] = y + (sn * ex + c * ey);
  e[3] = ch * qx - sh * qy; e[4] = ch * qy + sh * qx; e[5] = ch * qz + sh * qw; e[6] = ch * qw - sh * qz;   // Rz(dyaw) quaternion times e's
}

#ifdef __CUDACC__
// What qmb200_spawn_sample_dev and qmb200_spawn_place_dev read and write besides their per-call buffers.  NULL pointers: not written.
struct SpawnArgs {
  const double *lo, *hi; uint64_t seed; int64_t robot0;   // the sampler's ranges [B][SP_DBL], seed, global rank of robot 0
  const double* origin;     // [B][2] the robots' tile origins at the set (the run's), from which the drawn or given offsets count
  const double* qj;         // [NJ] the standing pose's joints (defaultJointState)
  double z_plane, radius, delta0, ground_height;   // the plane pose's base height and delta0 (plane_pose), the contact law's r, the plane
  SimTerrain ter;           // the tile library; ter.robot: the plant's robot terrain rows [B][3] the sampler writes (NULL: none, every robot on the plane)
  double* ground;           // [B][3] the estimator's ground map (the ground-map link), else NULL
  double* se; qmb200_state_est_params se_prm;   // state estimator [B][SE_DBL] and the parameters of its reset row
  double* at; qmb200_attitude_params at_prm;    // attitude filter [B][AT_DBL] and the parameters of its reset row
  double* sl;                    // slip detector [B][SL_DBL]
  const int32_t* frame;          // [B] the robots' end-effector frames (qmb200_set_ee_frame), NULL: every robot in the world frame
};
// one thread per robot: robots with mask[b] != 0 draw episode[b] as global robot robot0 + b and stand there
int launch_spawn_sample(const DevModel* mdl, int B, const SpawnArgs& a, const int32_t* mask, const int32_t* episode, double* rows, double* q, double* v, double* rbd,
                        int32_t* contact, double* x_obs, double* last_ee, double* rbd_est, cudaStream_t s);
// one thread per robot: robots with mask[b] != 0 whose row rows[b] passes spawn_place_ok stand there; status[b] (written) QMB200_ST_SPAWN for a
// rejected row, else 0
int launch_spawn_place(const DevModel* mdl, int B, int n_tiles, const SpawnArgs& a, const int32_t* mask, const double* rows, double* q, double* v, double* rbd,
                       int32_t* contact, double* x_obs, double* last_ee, double* rbd_est, int32_t* status, cudaStream_t s);
// one thread per robot: robots with mask[b] != 0 write spawn_here_row into rows[b]; ter: the plant's robot terrain rows [B][3] or NULL
int launch_spawn_here(int B, const int32_t* mask, const double* rbd, const double* q_start, const double* origin, const double* ter, double* rows, cudaStream_t s);
#endif

}  // namespace qmb
