// TEST INFRASTRUCTURE: host build (g++) of the per-episode spawn core (qm_control_b200/csrc/kernels/spawn_api.cuh), the same functions the sampler
// kernel and qmb200_spawn_draw compile, so that the CPU suite can check the draw against a numpy statement and the ported standing pose against the
// host's standing_on_terrain (tests/test_spawn_cpu.py).  The suite compiles this file with -DHOST_STANDING naming a file that holds the host function's
// text as capi_sim.inc has it, and links host/qm_config.cpp for the model and the host kinematics.
#include <algorithm>
#include <cstring>

#include "host/qm_config.h"
#include "kernels/spawn_api.cuh"

namespace qmb {
namespace host_twin {
#include HOST_STANDING
}  // namespace host_twin
}  // namespace qmb

using namespace qmb;

extern "C" {

void sp_uniform(int n, const uint64_t* seed, const uint64_t* robot, const uint64_t* episode, const int32_t* column, double* u) {
  for (int i = 0; i < n; ++i) u[i] = spawn_uniform(seed[i], robot[i], episode[i], column[i]);
}
void sp_rows(int n, const uint64_t* seed, const uint64_t* robot, const uint64_t* episode, const double* lo, const double* hi, double* rows) {
  for (int i = 0; i < n; ++i) spawn_row(lo + (size_t)i * SP_DBL, hi + (size_t)i * SP_DBL, seed[i], robot[i], episode[i], rows + (size_t)i * SP_DBL);
}
int sp_ranges_error(int B, const double* lo, const double* hi, int n_tiles, char* msg, int cap) {
  const std::string e = spawn_ranges_error(lo, hi, (size_t)B, n_tiles);
  std::strncpy(msg, e.c_str(), cap - 1); msg[cap - 1] = 0;
  return e.empty() ? 0 : 1;
}

void* sp_create(const char* task, const char* urdf, const char* reference, const char* gains) {
  try { return new HostModel(build_host_model(task, urdf, reference, gains)); } catch (const std::exception&) { return nullptr; }
}
void sp_destroy(void* h) { delete static_cast<HostModel*>(h); }
// whether every foot's and the end effector's chain is the serial chain chain_start..body-1 hanging off the base, as chain_pose walks it
int sp_chains_serial(void* h) {
  const DevModel& d = static_cast<HostModel*>(h)->dev;
  int bodies[5] = {d.foot_body[0], d.foot_body[1], d.foot_body[2], d.foot_body[3], d.ee_body};
  for (int body : bodies) {
    const int last = body - 1, first = d.chain_start[last];
    if (d.parent[first] != 0) return 0;
    for (int j = first + 1; j <= last; ++j) if (d.parent[j] != j) return 0;
  }
  return 1;
}
// n robots at xy_yaw [n][3] on terrain rows [n][3] of the library tiles [n_tiles][ny][nx]: the port (standing_on_tile) into port [n][3] = (z, pitch,
// roll) and the host's standing_on_terrain into host [n][3]; both at defaultJointState
void sp_standing(void* hp, const double* tiles, int nx, int ny, double cell, int n, const double* rows, const double* xy_yaw, double radius, double delta0, double* port,
                 double* host) {
  const HostModel& hm = *static_cast<HostModel*>(hp); const SimTerrain t{tiles, nullptr, nx, ny, cell};
  for (int i = 0; i < n; ++i) {
    const double* r = rows + 3 * i; const double* p = xy_yaw + 3 * i;
    double z, pitch, roll; standing_on_tile(hm.dev, t, r, radius, delta0, hm.default_joint_state, p[0], p[1], p[2], z, pitch, roll);
    port[3 * i] = z; port[3 * i + 1] = pitch; port[3 * i + 2] = roll;
    double q[NQ] = {0}; q[0] = p[0]; q[1] = p[1]; q[3] = p[2]; for (int j = 0; j < NJ; ++j) q[6 + j] = hm.default_joint_state[j];
    host_twin::standing_on_terrain(hm.dev, t, r, radius, delta0, q);
    host[3 * i] = q[2]; host[3 * i + 1] = q[4]; host[3 * i + 2] = q[5];
  }
}
// the end-effector pose and the four feet of the port's forward kinematics at the standing configuration (x, y, z, yaw, pitch, roll): ee [7] (position,
// quaternion xyzw), feet [4][3]; and the host kinematics' (host_fk) into ee_host, feet_host
void sp_kinematics(void* hp, const double* base, double* ee, double* feet, double* ee_host, double* feet_host) {
  const HostModel& hm = *static_cast<HostModel*>(hp); const DevModel& d = hm.dev; const double* qj = hm.default_joint_state;
  double Rb[9]; spawn_rot_zyx(base[3], base[4], base[5], Rb);
  double Re[9]; spawn_ee(d, qj, Rb, base, ee, Re); rot_to_quat_xyzw(Re, ee + 3);
  for (int f = 0; f < 4; ++f) spawn_foot(d, qj, Rb, base, f, feet + 3 * f);
  double q[NQ] = {0}; for (int i = 0; i < 6; ++i) q[i] = base[i]; for (int j = 0; j < NJ; ++j) q[6 + j] = qj[j];
  double Rw[NB][9], pw[NB][3], pf[4][3]; host_fk(d, q, Rw, pw); host_feet(d, Rw, pw, pf);
  double R[9]; matmul3(Rw[d.ee_body], d.ee_R, R); matvec3(Rw[d.ee_body], d.ee_p, ee_host); for (int i = 0; i < 3; ++i) ee_host[i] += pw[d.ee_body][i];
  rot_to_quat_xyzw(R, ee_host + 3);
  for (int f = 0; f < 4; ++f) for (int i = 0; i < 3; ++i) feet_host[3 * f + i] = pf[f][i];
}

}  // extern "C"
