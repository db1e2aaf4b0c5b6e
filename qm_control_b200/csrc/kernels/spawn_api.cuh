// Per-episode spawns (spawn_kernel.cu; include/qmb200.h: qmb200_spawn_*; DESIGN.md §4.12): the spawn row of one episode of one robot (its tile, its
// offset along the tile and its yaw), a pure function of (seed, global robot, episode, column) and the robot's ranges, and the standing pose on that
// ground.  Host + device: the sampler kernel, qmb200_spawn_draw and tests/spawn_host.cpp compile the same core, so host and device agree bit for bit.
#pragma once
#include <math.h>
#include <stdint.h>

#include <cmath>
#include <string>

#include "dev_common.cuh"
#include "sim_api.cuh"

namespace qmb {

// a spawn row [SP_DBL] (_lib.SPAWN_LAYOUT): the plant's tile (-1: the plane), the offset (dx, dy) the robot stands further along its tile (world axes:
// the tile's origin moves by -(dx, dy)), the base yaw
constexpr int SP_TILE = 0, SP_DX = 1, SP_DY = 2, SP_YAW = 3, SP_DBL = 4;
// xor-ed into the seed so that a spawn draw, a plant draw and a sensor-noise draw of the same words are unrelated
constexpr uint64_t SPAWN_DOMAIN = 0xbb67ae8584caa73bull;

// u in (0, 1): (seed ^ SPAWN_DOMAIN, robot, episode, column) hashed in turn as episode_uniform hashes its words, then a 53-bit uniform of one more hash
QMB_HD double spawn_uniform(uint64_t seed, uint64_t robot, uint64_t episode, int column) {
  const uint64_t h = mix64(mix64(mix64(mix64(seed ^ SPAWN_DOMAIN) ^ robot) ^ episode) ^ (uint64_t)column);
  return ((double)(mix64(h) >> 11) + 0.5) * 1.1102230246251565e-16;
}
// row[c]: a fixed column (lo[c] == hi[c]) is lo[c] itself, byte for byte; the tile is the integer lo + min(floor(u (hi - lo + 1)), hi - lo), each of
// the hi - lo + 1 tiles with probability 1 / (hi - lo + 1); dx, dy and yaw are fma(u, hi - lo, lo), one rounding whatever the compiler contracts
QMB_HD void spawn_row(const double* lo, const double* hi, uint64_t seed, uint64_t robot, uint64_t episode, double* row) {
#pragma unroll
  for (int c = 0; c < SP_DBL; ++c) {
    const double u = spawn_uniform(seed, robot, episode, c), d = hi[c] - lo[c];
    row[c] = hi[c] == lo[c] ? lo[c] : c == SP_TILE ? lo[c] + fmin(floor(u * (d + 1.0)), d) : fma(u, d, lo[c]);
  }
}

// The check of qmb200_spawn_set_ranges on ranges lo, hi [B][SP_DBL] on a tile library of n_tiles tiles: "" when valid, else the first offence naming
// the field and the robot
inline std::string spawn_ranges_error(const double* lo, const double* hi, size_t B, int n_tiles) {
  static const char* const names[SP_DBL] = {"tile", "dx", "dy", "yaw"};
  const double pi = 3.141592653589793;
  for (size_t b = 0; b < B; ++b) for (int c = 0; c < SP_DBL; ++c) {
    const double l = lo[b * SP_DBL + c], u = hi[b * SP_DBL + c];
    std::string why;
    if (!(std::isfinite(l) && std::isfinite(u))) why = "bounds must be finite";
    else if (!(l <= u)) why = "lo must be <= hi";
    else if (!std::isfinite(u - l)) why = "hi - lo must be finite";
    else if (c == SP_TILE && !(std::floor(l) == l && std::floor(u) == u)) why = "bounds must be integers";
    else if (c == SP_TILE && !(l >= -1.0 && u < n_tiles)) why = "bounds must lie in [-1, " + std::to_string(n_tiles) + "), the tiles of the library in force";
    else if (c == SP_YAW && !(l >= -pi && u <= pi)) why = "bounds must lie in [-pi, pi]";
    if (!why.empty()) return std::string("qmb200_spawn_set_ranges: ") + names[c] + " of robot " + std::to_string(b) + ": " + why;
  }
  return "";
}

// ---- the standing pose, one thread per robot: every chain walked from the base with a running (R, p), so no per-body arrays are held ----
// Sine and cosine of an angle of a few radians.  The device takes sincospi, whose argument reduction is exact and needs no stack: sin / cos carry a
// Payne-Hanek slow path for huge arguments whose 40-byte frame would put the kernel in local memory.  The two differ by about an ulp.
QMB_HD void spawn_sincos(double x, double& s, double& c) {
#ifdef __CUDA_ARCH__
  sincospi(x * 0.31830988618379067, &s, &c);
#else
  s = std::sin(x); c = std::cos(x);
#endif
}
// R = Rz(z) Ry(y) Rx(x), rot_zyx's formula on spawn_sincos
QMB_HD void spawn_rot_zyx(double z, double y, double x, double* R) {
  double sz, cz, sy, cy, sx, cx; spawn_sincos(z, sz, cz); spawn_sincos(y, sy, cy); spawn_sincos(x, sx, cx);
  R[0] = cz * cy; R[1] = cz * sy * sx - sz * cx; R[2] = cz * sy * cx + sz * sx;
  R[3] = sz * cy; R[4] = sz * sy * sx + cz * cx; R[5] = sz * sy * cx - cz * sx;
  R[6] = -sy;     R[7] = cy * sx;                R[8] = cy * cx;
}
// M := M A with A the rotation about axis (I, K)'s normal by an angle of sine s and cosine c: columns I and K turn, the third stays
template <int I, int K> QMB_HD void turn_columns(double* M, double s, double c) {
#pragma unroll
  for (int r = 0; r < 3; ++r) { const double a = M[3 * r + I], b = M[3 * r + K]; M[3 * r + I] = c * a + s * b; M[3 * r + K] = c * b - s * a; }
}
// (R, p): the base pose on entry, body `body`'s pose on exit, with the joints at qj [NJ].  body's chain is the serial chain of joints chain_start..body-1
// hanging off the base (a leg, the arm), each step as host_fk takes it: p += R pj, R := R Rj Rot(axis, q).
QMB_HD void chain_pose(const DevModel& d, const double* qj, int body, double* R, double* p) {
  const int last = body - 1;
  for (int j = d.chain_start[last]; j <= last; ++j) {
    double t[3]; matvec3(R, d.pj[j], t); p[0] += t[0]; p[1] += t[1]; p[2] += t[2];
    double RR[9]; matmul3(R, d.Rj[j], RR);
    double s, c; spawn_sincos(qj[j], s, c);
    if (d.axis[j] == 0) turn_columns<1, 2>(RR, s, c); else if (d.axis[j] == 1) turn_columns<2, 0>(RR, s, c); else turn_columns<0, 1>(RR, s, c);
#pragma unroll
    for (int i = 0; i < 9; ++i) R[i] = RR[i];
  }
}
// world origin of foot frame f of the base at (pb, Rb)
QMB_HD void spawn_foot(const DevModel& d, const double* qj, const double* Rb, const double* pb, int f, double* pf) {
  double R[9], p[3] = {pb[0], pb[1], pb[2]};
#pragma unroll
  for (int i = 0; i < 9; ++i) R[i] = Rb[i];
  chain_pose(d, qj, d.foot_body[f], R, p);
  matvec3(R, d.foot_p[f], pf); pf[0] += p[0]; pf[1] += p[1]; pf[2] += p[2];
}
// the end-effector frame of the base at (pb, Rb): origin pe and rotation Re (world)
QMB_HD void spawn_ee(const DevModel& d, const double* qj, const double* Rb, const double* pb, double* pe, double* Re) {
  double R[9], p[3] = {pb[0], pb[1], pb[2]};
#pragma unroll
  for (int i = 0; i < 9; ++i) R[i] = Rb[i];
  chain_pose(d, qj, d.ee_body, R, p);
  matvec3(R, d.ee_p, pe); pe[0] += p[0]; pe[1] += p[1]; pe[2] += p[2];
  matmul3(R, d.ee_R, Re);
}

// The standing pose of a robot at world (x, y) with yaw and joints qj on the ground of terrain row `row` ([tile >= 0, origin_x, origin_y]): the port of
// the host's standing_on_terrain (capi_sim.inc).  Roll and pitch tilt the base's z axis onto the normal of the least-squares plane through the ground
// heights under the four feet, iterated eight times because the feet's xy move with the tilt; then the base height at which the deepest foot has the
// static penetration delta0 of the contact law, max_f (H_f - p_fz + (r - delta0) s_f) with the feet computed at base height 0.  → z, pitch, roll.
QMB_HD void standing_on_tile(const DevModel& d, const SimTerrain& t, const double* row, double radius, double delta0, const double* qj, double x, double y,
                             double yaw, double& z, double& pitch, double& roll) {
  double sy, cy; spawn_sincos(yaw, sy, cy); const double pb[3] = {x, y, 0.0};
  pitch = 0.0; roll = 0.0;
  for (int it = 0; it < 8; ++it) {
    double Rb[9]; spawn_rot_zyx(yaw, pitch, roll, Rb);
    double px[4], py[4], H[4], mx = 0.0, my = 0.0, mh = 0.0;
#pragma unroll
    for (int f = 0; f < 4; ++f) {
      double pf[3], gx, gy; spawn_foot(d, qj, Rb, pb, f, pf); ground_at(t, row, 0.0, pf[0], pf[1], H[f], gx, gy);
      px[f] = pf[0]; py[f] = pf[1]; mx += 0.25 * pf[0]; my += 0.25 * pf[1]; mh += 0.25 * H[f];
    }
    double sxx = 0.0, sxy = 0.0, syy = 0.0, sxh = 0.0, syh = 0.0;
#pragma unroll
    for (int f = 0; f < 4; ++f) {
      const double a = px[f] - mx, b = py[f] - my, h = H[f] - mh;
      sxx += a * a; sxy += a * b; syy += b * b; sxh += a * h; syh += b * h;
    }
    const double det = sxx * syy - sxy * sxy, bx = (syy * sxh - sxy * syh) / det, by = (sxx * syh - sxy * sxh) / det;
    const double nn = sqrt(1.0 + bx * bx + by * by), n0 = -bx / nn, n1 = -by / nn, n2 = 1.0 / nn;
    const double nxp = cy * n0 + sy * n1, nyp = -sy * n0 + cy * n1;   // the normal in the yawed frame
    pitch = atan2(nxp, n2); roll = asin(-nyp);
  }
  double Rb[9]; spawn_rot_zyx(yaw, pitch, roll, Rb);
  z = -INFINITY;
#pragma unroll
  for (int f = 0; f < 4; ++f) {
    double pf[3], H, gx, gy; spawn_foot(d, qj, Rb, pb, f, pf); ground_at(t, row, 0.0, pf[0], pf[1], H, gx, gy);
    z = fmax(z, H - pf[2] + (radius - delta0) * sqrt(1.0 + gx * gx + gy * gy));
  }
}

#ifdef __CUDACC__
// What qmb200_spawn_sample_dev reads and writes besides its per-call buffers.  NULL pointers: not written.
struct SpawnArgs {
  const double *lo, *hi; uint64_t seed; int64_t robot0;   // ranges [B][SP_DBL], seed, global rank of robot 0
  const double* origin;     // [B][2] the robots' tile origins at the set (the run's), from which the drawn offsets count
  const double* qj;         // [NJ] the standing pose's joints (defaultJointState)
  double z_plane, radius, delta0, ground_height;   // the plane pose's base height (as qmb200_sim_standing_state), the contact law's r, delta0, plane
  SimTerrain ter;           // the tile library; ter.robot: the plant's robot terrain rows [B][3] the sampler writes (NULL: none, every robot on the plane)
  double* ground;           // [B][3] the estimator's ground map (the ground-map link), else NULL
  double* se; double se_p0[3];   // state estimator [B][SE_DBL] and its reset's P diagonal (base position, base velocity, foot)
  double* at; double at_p0[2];   // attitude filter [B][AT_DBL] and its reset's P diagonal (attitude, gyro bias)
  double* sl;                    // slip detector [B][SL_DBL]
};
// one thread per robot: robots with mask[b] != 0 draw episode[b] as global robot robot0 + b and stand there
int launch_spawn_sample(const DevModel* mdl, int B, const SpawnArgs& a, const int32_t* mask, const int32_t* episode, double* rows, double* q, double* v, double* rbd,
                        int32_t* contact, double* x_obs, double* last_ee, double* rbd_est, cudaStream_t s);
#endif

}  // namespace qmb
