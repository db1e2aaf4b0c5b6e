// Host-visible interface of the batched plant step (sim_kernel.cu): rigid-body forward dynamics of the 24-DoF tree with compliant
// foot-ground contact, the stand-in for Gazebo's physics step behind QMHWSim (qm_gazebo/src/QMHWSim.cpp).
#pragma once
#include <cuda_runtime.h>

#include "dev_common.cuh"

namespace qmb {

// Contact and joint constants of the plant (include/qmb200.h: qmb200_sim_params; DESIGN.md §4.6 explains the defaults).
struct SimParams {
  double ground_height;        // height of the flat ground plane (m)
  double foot_radius;          // collision sphere of the *_FOOT links, centred on the foot frame (m)
  double stiffness;            // normal penalty spring k (N/m)
  double damping;              // normal damper d (N s/m)
  double tangential_damping;   // regularised Coulomb friction: viscous slope gamma below the friction cone (N s/m)
  double friction_mu;          // Coulomb coefficient mu
  double joint_damping[NJ];    // viscous joint damping (N m s/rad)
  int substeps_per_ms;         // semi-implicit Euler steps per millisecond of simulated time
};

// Heightfield terrain under the feet (include/qmb200.h: qmb200_sim_set_terrain, qmb200_sim_set_robot_terrain; DESIGN.md §4.6).
struct SimTerrain {
  const double* heights;   // tile library [n_tiles][ny][nx], absolute world z (m); NULL when none is set
  const double* robot;     // [B][3] = [tile, origin_x, origin_y] per robot (tile -1: the plane z = ground_height); NULL: every robot on the plane
  int nx, ny;              // nodes per tile in x and y (>= 2); node (i, j) of robot b's tile lies at origin + (i cell, j cell)
  double cell;             // node spacing (m)
};

// Height H and gradient (gx, gy) at world (x, y) of one tile whose node (0, 0) lies at (ox, oy): bilinear inside the tile, the border value outside it
// with a zero gradient across the clamped axis.  The clamp uses fmin / fmax, which return the non-NaN operand, so a non-finite (x, y) still reads
// inside the tile.  For a constant tile H is exactly the tile's value and the gradient exactly zero.
QMB_HD void terrain_height(const double* tile, int nx, int ny, double cell, double ox, double oy, double x, double y, double& H, double& gx, double& gy) {
  const double ur = (x - ox) / cell, vr = (y - oy) / cell;
  const double u = fmin(fmax(ur, 0.0), (double)(nx - 1)), v = fmin(fmax(vr, 0.0), (double)(ny - 1));
  int i = (int)floor(u), j = (int)floor(v);
  if (i > nx - 2) i = nx - 2;
  if (j > ny - 2) j = ny - 2;
  const double fx = u - i, fy = v - j;
  const double* r0 = tile + (size_t)j * nx + i; const double* r1 = r0 + nx;
  const double h00 = r0[0], h10 = r0[1], h01 = r1[0], h11 = r1[1], hxy = h11 - h10 - h01 + h00;
  H = h00 + fx * (h10 - h00) + fy * (h01 - h00) + fx * fy * hxy;
  gx = ur == u ? ((h10 - h00) + fy * hxy) / cell : 0.0;   // ur != u: clamped, or NaN
  gy = vr == v ? ((h01 - h00) + fx * hxy) / cell : 0.0;
}

// Ground under robot b's foot at world (x, y): the plane when no terrain is set or the robot's tile is -1, else its tile
QMB_HD void ground_at(const SimTerrain& t, const double* row, double ground_height, double x, double y, double& H, double& gx, double& gy) {
  H = ground_height; gx = 0.0; gy = 0.0;
  const int tile = row ? (int)row[0] : -1;
  if (tile >= 0) terrain_height(t.heights + (size_t)tile * t.nx * t.ny, t.nx, t.ny, t.cell, row[1], row[2], x, y, H, gx, gy);
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

// The standing pose of a robot at world (x, y) with yaw and joints qj on the ground of terrain row `row` ([tile >= 0, origin_x, origin_y]), for
// qmb200_sim_standing_state and the spawn sampler.  Roll and pitch tilt the base's z axis onto the normal of the least-squares plane through the ground
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
    pitch = atan2(nxp, n2); roll = asin(-nyp);                        // base z = Rz(yaw) Ry(pitch) Rx(roll) e_z = (s_p c_r, -s_r, c_p c_r) in that frame
  }
  double Rb[9]; spawn_rot_zyx(yaw, pitch, roll, Rb);
  z = -INFINITY;
#pragma unroll
  for (int f = 0; f < 4; ++f) {
    double pf[3], H, gx, gy; spawn_foot(d, qj, Rb, pb, f, pf); ground_at(t, row, 0.0, pf[0], pf[1], H, gx, gy);
    z = fmax(z, H - pf[2] + (radius - delta0) * sqrt(1.0 + gx * gx + gy * gy));
  }
}

// mu [B], payload [B][8], wrench [B][12]: optional per-robot plant variation (NULL = not used; sim_kernel.cu has the layouts); terrain: see SimTerrain
int launch_sim_step(const DevModel* mdl, const SimParams& prm, int B, int substeps, double h, const double* effort, double* q, double* v, double* rbd, int32_t* contact,
                    int32_t* status, const double* mu, const double* payload, const double* wrench, const SimTerrain& terrain, cudaStream_t s);

}  // namespace qmb
