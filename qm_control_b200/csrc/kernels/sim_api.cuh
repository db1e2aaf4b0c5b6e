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

// mu [B], payload [B][8], wrench [B][12]: optional per-robot plant variation (NULL = not used; sim_kernel.cu has the layouts); terrain: see SimTerrain
int launch_sim_step(const DevModel* mdl, const SimParams& prm, int B, int substeps, double h, const double* effort, double* q, double* v, double* rbd, int32_t* contact,
                    int32_t* status, const double* mu, const double* payload, const double* wrench, const SimTerrain& terrain, cudaStream_t s);

}  // namespace qmb
