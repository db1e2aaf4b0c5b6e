// TEST INFRASTRUCTURE: host build (g++) of the per-episode metrics core (qm_control_b200/csrc/kernels/metrics_api.cuh), the same per-robot functions
// metrics_step_kernel and metrics_close_kernel compile, so that the CPU suite can check them against a numpy statement of the column table
// (tests/test_metrics_cpu.py).  Links host/qm_config.cpp for the model.
#include "host/qm_config.h"
#include "kernels/metrics_api.cuh"

using namespace qmb;

extern "C" {

void* mt_create(const char* task, const char* urdf, const char* reference, const char* gains) {
  try { return new HostModel(build_host_model(task, urdf, reference, gains)); } catch (const std::exception&) { return nullptr; }
}
void mt_destroy(void* h) { delete static_cast<HostModel*>(h); }

// one metrics_step launch of B robots, as qmb200_metrics_step_dev passes it: the library tiles [n_tiles][ny][nx] (NULL: none), the robots' terrain rows
// [B][3] (NULL: none); kind and rbd_est may be NULL
void mt_step(void* hp, const double* tiles, int nx, int ny, double cell, const double* terrain_rows, double ground_height, int B, double dt, const double* rbd,
             const int32_t* contact, const double* effort, const double* cmd, const int32_t* kind, const int32_t* n_target, const double* target_times,
             const double* target_states, const double* time, const int32_t* status, const double* rbd_est, double* acc) {
  const DevModel& d = static_cast<HostModel*>(hp)->dev; const SimTerrain t{tiles, terrain_rows, nx, ny, cell};
  const MetricsStep p{dt, rbd, effort, cmd, target_times, target_states, time, rbd_est, contact, kind, n_target, status, acc};
  for (int b = 0; b < B; ++b) metrics_step_robot(d, t, ground_height, p, b);
}

// one metrics_close launch of B robots on out [B][n_episodes][QMB200_METRICS]
void mt_close(int B, const int32_t* mask, const int32_t* end, const int32_t* episode, int n_episodes, double* acc, double* out, int32_t* status) {
  for (int b = 0; b < B; ++b)
    if (mask[b]) metrics_close_robot(acc + (size_t)b * MA_DBL, end[b], episode[b], n_episodes, out + (size_t)b * n_episodes * MT_DBL, status[b]);
}

}  // extern "C"
