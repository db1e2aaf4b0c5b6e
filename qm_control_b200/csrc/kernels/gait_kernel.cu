// Device gait schedule: one thread per robot rolls the robot's GaitSchedule once per MPC tick (gait_api.cuh: gs_step).  The work is a few dozen
// doubles per robot every 10 ms, so the state stays in global memory and each step works on a copy that is written back only on success.
// gait_command_kernel: one thread per robot checks a masked robot's command row (gs_command_check) and writes it to the robot's pending slot.
#include "gait_api.cuh"

namespace qmb {
namespace {

constexpr int GS_THREADS = 128;

__global__ void __launch_bounds__(GS_THREADS) gait_step_kernel(int B, const GsTemplate* __restrict__ table, GsRobot* __restrict__ robots,
                                                                int32_t* __restrict__ cursor, GsCommands c, double horizon, double stance_time,
                                                                const double* __restrict__ t_obs, int32_t* __restrict__ n_events, double* __restrict__ event_times,
                                                                int32_t* __restrict__ modes, double* __restrict__ cmd, int32_t* __restrict__ tmpl,
                                                                int32_t* __restrict__ mode, int32_t* __restrict__ status, int32_t* __restrict__ target_kind,
                                                                GsPending* __restrict__ pending) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const double t = t_obs[b];
  status[b] = gs_step(robots[b], cursor + b, table, c, b, t, horizon, stance_time, n_events + b, event_times + (size_t)b * QMB200_EMAX,
                      modes + (size_t)b * (QMB200_EMAX + 1), cmd + (size_t)b * 7, target_kind ? target_kind + b : nullptr, pending + b);
  if (tmpl) tmpl[b] = robots[b].tmpl;
  if (mode) mode[b] = gs_mode_at(robots[b].s, t);
}

__global__ void __launch_bounds__(GS_THREADS) gait_command_kernel(int B, int n_templates, int n_paths, GsPending* __restrict__ pending, const int32_t* __restrict__ mask,
                                                                   const int32_t* __restrict__ tmpl, const double* __restrict__ vel,
                                                                   const int32_t* __restrict__ ee_kind, const double* __restrict__ ee, int32_t* __restrict__ status) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  if (!mask[b]) { status[b] = 0; return; }
  double v[4], e[7];
#pragma unroll
  for (int i = 0; i < 4; ++i) v[i] = vel[(size_t)b * 4 + i];
#pragma unroll
  for (int i = 0; i < 7; ++i) e[i] = ee[(size_t)b * 7 + i];
  const int tm = tmpl[b], kind = ee_kind[b];
  const int st = gs_command_check(tm, v, kind, e, n_templates, n_paths);
  status[b] = st;
  if (st) return;
  GsPending& p = pending[b];
  p.set = 1; p.tmpl = tm; p.ee_kind = kind; p.pad = 0;
#pragma unroll
  for (int i = 0; i < 4; ++i) p.vel[i] = v[i];
#pragma unroll
  for (int i = 0; i < 7; ++i) p.ee[i] = e[i];
}

}  // namespace

int launch_gait_step(int B, const GsTemplate* table, GsRobot* robots, int32_t* cursor, GsCommands c, double horizon, double stance_time, const double* t_obs,
                     int32_t* n_events, double* event_times, int32_t* modes, double* cmd, int32_t* tmpl, int32_t* mode, int32_t* status, int32_t* target_kind,
                     GsPending* pending, cudaStream_t s) {
  gait_step_kernel<<<(B + GS_THREADS - 1) / GS_THREADS, GS_THREADS, 0, s>>>(B, table, robots, cursor, c, horizon, stance_time, t_obs, n_events, event_times,
                                                                           modes, cmd, tmpl, mode, status, target_kind, pending);
  return 1;
}

int launch_gait_command(int B, int n_templates, int n_paths, GsPending* pending, const int32_t* mask, const int32_t* tmpl, const double* vel, const int32_t* ee_kind,
                        const double* ee, int32_t* status, cudaStream_t s) {
  gait_command_kernel<<<(B + GS_THREADS - 1) / GS_THREADS, GS_THREADS, 0, s>>>(B, n_templates, n_paths, pending, mask, tmpl, vel, ee_kind, ee, status);
  return 1;
}

}  // namespace qmb
