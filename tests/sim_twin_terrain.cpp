// TEST INFRASTRUCTURE ONLY: the CPU twin of the plant step on heightfield terrain (qm_control_b200/csrc/kernels/sim_kernel.cu with a tile library,
// include/qmb200.h: qmb200_sim_set_terrain).  It builds on the twin with per-robot variation (tests/sim_twin_ext.cpp, included as source, so payload,
// wrench and friction reach the robot exactly as there) and adds, on its own code:
//   lookup    the tile's height by interpolation along x on the cell's two rows, then along y; the border height outside the tile with a zero gradient
//             across the clamped axis (a NaN coordinate counts as clamped to node 0)
//   contact   the tangent-plane law of include/qmb200.h at the foot positions and velocities of orc::compute_rbd
// twin_step_ext of tests/sim_twin_ext.cpp stays the plane law the terrain law must reproduce bit for bit at zero gradient.
// Compiled by tests/_sim_twin_terrain.py together with oracle/src/model.cpp; the product never loads it.
#include "sim_twin_ext.cpp"

namespace {
// one robot's tile [ny][nx], nodes `cell` apart, node (0, 0) at (ox, oy)
struct Tile { const double* h; int nx, ny; double cell, ox, oy; };

// node index and fraction along one axis; inside = false when the coordinate was clamped to the border (or is NaN)
void cell_of(double w, double o, double cell, int n, int& i, double& f, bool& inside) {
  const double u = (w - o) / cell; inside = u >= 0.0 && u <= n - 1.0;
  const double c = inside ? u : (u > n - 1.0 ? n - 1.0 : 0.0);
  i = std::min((int)std::floor(c), n - 2); f = c - i;
}

void tile_height(const Tile& g, double x, double y, double& H, double& gx, double& gy) {
  int i, j; double fx, fy; bool inx, iny; cell_of(x, g.ox, g.cell, g.nx, i, fx, inx); cell_of(y, g.oy, g.cell, g.ny, j, fy, iny);
  auto h = [&](int a, int b) { return g.h[(size_t)(j + b) * g.nx + (i + a)]; };
  const double a0 = h(0, 0) + fx * (h(1, 0) - h(0, 0)), a1 = h(0, 1) + fx * (h(1, 1) - h(0, 1));
  H = a0 + fy * (a1 - a0);
  gx = inx ? ((1.0 - fy) * (h(1, 0) - h(0, 0)) + fy * (h(1, 1) - h(0, 1))) / g.cell : 0.0;
  gy = iny ? (a1 - a0) / g.cell : 0.0;
}

// contact force (world) on a foot at pos moving with vel against the tile's local tangent plane; returns F_n
double contact_on_tile(const Prm& p, const Tile& g, const V3<double>& pos, const V3<double>& vel, double* F) {
  double H, gx, gy; tile_height(g, pos[0], pos[1], H, gx, gy);
  const double s = std::sqrt(1.0 + gx * gx + gy * gy), n[3] = {-gx / s, -gy / s, 1.0 / s};
  const double pen = (H - (pos[2] - p.radius * s)) / s, vn = vel[0] * n[0] + vel[1] * n[1] + vel[2] * n[2];
  double fn = 0.0; if (pen > 0.0) fn = std::max(0.0, p.k * pen - p.d * vn);
  const double t[3] = {vel[0] - vn * n[0], vel[1] - vn * n[1], vel[2] - vn * n[2]}, vt = std::sqrt(t[0] * t[0] + t[1] * t[1] + t[2] * t[2]);
  const double c = fn > 0.0 && vt > 0.0 ? std::min(p.gamma, p.mu * fn / vt) : 0.0;
  for (int i = 0; i < 3; ++i) F[i] = fn > 0.0 ? fn * n[i] - c * t[i] : 0.0;
  return fn;
}

// accel of tests/sim_twin_ext.cpp with the feet on the tile
bool accel_on_tile(const Model& mdl, const Prm& p, const Tile& g, const double* tau_sat, const double* wrench, const double* q, const double* v, double* qdd, double* F12,
                   int* mask) {
  RbdData d; compute_rbd(mdl, q, v, d, 1);
  Vec Q(NQ, 0.0); *mask = 0;
  for (int f = 0; f < 4; ++f) {
    double* F = F12 + 3 * f;
    if (contact_on_tile(p, g, d.foot_pos[f], d.foot_vel[f], F) > 0.0) *mask |= 8 >> f;
    for (int c = 0; c < NQ; ++c) for (int i = 0; i < 3; ++i) Q[c] += d.Jfoot(3 * f + i, c) * F[i];
  }
  for (int c = 0; c < NQ; ++c) Q[c] -= d.nle[c];
  for (int j = 0; j < NJ; ++j) Q[6 + j] += tau_sat[j] - p.jd[j] * v[6 + j];
  if (wrench)
    for (int c = 0; c < NQ; ++c) for (int i = 0; i < 6; ++i) Q[c] += d.Jbase(i, c) * wrench[i] + d.Jee(i, c) * wrench[6 + i];
  Mat L; if (!cholesky(d.M, L)) return false;
  Mat x = chol_solve(L, col(Q)); for (int c = 0; c < NQ; ++c) qdd[c] = x(c, 0);
  return true;
}
}  // namespace

extern "C" {

// twin_accel_ext on the tile [ny][nx] (nodes `cell` apart, node (0, 0) at (ox, oy))
int twin_accel_terrain(void* tp, const double* params, const double* payload, const double* wrench, const double* tile, int nx, int ny, double cell, double ox, double oy,
                       const double* effort, const double* q, const double* v, double* qdd, double* F12, int* mask) {
  const Model m = with_payload(static_cast<Twin*>(tp)->m, payload); double tau[NJ]; saturate(m, effort, tau);
  return accel_on_tile(m, unpack(params), Tile{tile, nx, ny, cell, ox, oy}, tau, wrench, q, v, qdd, F12, mask) ? 0 : -1;
}

// twin_step_ext on the tile
void twin_step_terrain(void* tp, const double* params, const double* payload, const double* wrench, const double* tile, int nx, int ny, double cell, double ox, double oy,
                       int substeps, double h, const double* effort, double* q, double* v, double* rbd, int* contact, int* status) {
  const Model m = with_payload(static_cast<Twin*>(tp)->m, payload); const Prm p = unpack(params); const Tile g{tile, nx, ny, cell, ox, oy};
  double tau[NJ]; saturate(m, effort, tau);
  int st = 0, mask = 0; double qdd[NQ], F[12];
  for (int k = 0; k < substeps; ++k) {
    if (!accel_on_tile(m, p, g, tau, wrench, q, v, qdd, F, &mask)) { st |= 8; break; }
    for (int c = 0; c < NQ; ++c) { v[c] += h * qdd[c]; q[c] += h * v[c]; }
  }
  for (int c = 0; c < NQ; ++c) if (!std::isfinite(q[c]) || !std::isfinite(v[c])) st |= 4;
  RbdData d; compute_rbd(m, q, v, d, 0);
  rbd[0] = q[3]; rbd[1] = q[4]; rbd[2] = q[5]; rbd[3] = q[0]; rbd[4] = q[1]; rbd[5] = q[2];
  for (int j = 0; j < NJ; ++j) { rbd[6 + j] = q[6 + j]; rbd[30 + j] = v[6 + j]; }
  const M3<double> T = euler_rate_map<double>(q[3], q[4]); const V3<double> w = T * V3<double>(v[3], v[4], v[5]);
  for (int i = 0; i < 3; ++i) { rbd[24 + i] = w[i]; rbd[27 + i] = v[i]; rbd[48 + i] = d.ee_pos[i]; }
  quat_xyzw(d.ee_rot, rbd + 51);
  *contact = mask; *status = st;
}

// height H and gradient (gx, gy) of the tile at (x, y)
void twin_ground(const double* tile, int nx, int ny, double cell, double ox, double oy, double x, double y, double* H, double* gx, double* gy) {
  tile_height(Tile{tile, nx, ny, cell, ox, oy}, x, y, *H, *gx, *gy);
}

}  // extern "C"
