// Per-episode spawns (spawn_kernel.cu; include/qmb200.h: qmb200_spawn_*; DESIGN.md §4.12): the spawn row of one episode of one robot (its tile, its
// offset along the tile and its yaw), a pure function of (seed, global robot, episode, column) and the robot's ranges.  Host + device: the sampler
// kernel, qmb200_spawn_draw and tests/spawn_host.cpp compile the same core, so host and device agree bit for bit.  The robot stands on the drawn ground
// with standing_on_tile (sim_api.cuh), the pose qmb200_sim_standing_state gives.
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

#ifdef __CUDACC__
// What qmb200_spawn_sample_dev reads and writes besides its per-call buffers.  NULL pointers: not written.
struct SpawnArgs {
  const double *lo, *hi; uint64_t seed; int64_t robot0;   // ranges [B][SP_DBL], seed, global rank of robot 0
  const double* origin;     // [B][2] the robots' tile origins at the set (the run's), from which the drawn offsets count
  const double* qj;         // [NJ] the standing pose's joints (defaultJointState)
  double z_plane, radius, delta0, ground_height;   // the plane pose's base height and delta0 (plane_pose), the contact law's r, the plane
  SimTerrain ter;           // the tile library; ter.robot: the plant's robot terrain rows [B][3] the sampler writes (NULL: none, every robot on the plane)
  double* ground;           // [B][3] the estimator's ground map (the ground-map link), else NULL
  double* se; qmb200_state_est_params se_prm;   // state estimator [B][SE_DBL] and the parameters of its reset row
  double* at; qmb200_attitude_params at_prm;    // attitude filter [B][AT_DBL] and the parameters of its reset row
  double* sl;                    // slip detector [B][SL_DBL]
};
// one thread per robot: robots with mask[b] != 0 draw episode[b] as global robot robot0 + b and stand there
int launch_spawn_sample(const DevModel* mdl, int B, const SpawnArgs& a, const int32_t* mask, const int32_t* episode, double* rows, double* q, double* v, double* rbd,
                        int32_t* contact, double* x_obs, double* last_ee, double* rbd_est, cudaStream_t s);
#endif

}  // namespace qmb
