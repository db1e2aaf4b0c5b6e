// TEST INFRASTRUCTURE: host build (g++) of the device gait schedule's core (qm_control_b200/csrc/kernels/gait_api.cuh) with each robot's pending
// command slot, so that the CPU suite can check the command channel of qmb200_gait_dev_command without a GPU (tests/test_session_cpu.py).  Every robot
// step is gs_step with the pending slot, the function gait_step_kernel runs; gsh_command is gait_command_kernel's body.
#include <cstring>
#include <vector>

#include "host/qm_config.h"
#include "kernels/gait_api.cuh"

using namespace qmb;

namespace {
struct SessionHost {
  std::vector<GsTemplate> table; GsSchedule init; std::vector<GsRobot> robots; std::vector<int32_t> cursor; std::vector<GsPending> pending;
  std::vector<double> t, vel, ee; std::vector<int32_t> tmpl, ee_kind; int n_cmd = 0; double horizon = 0.0, stance = 0.0;
};
}  // namespace

extern "C" {

// templates names[0..n) of gait_file; B robots; the initial schedule of reference (initialModeSchedule), the stance time of task
void* gsh_create(const char* task, const char* reference, const char* gait_file, const char* const* names, int n, int B, double horizon) {
  try {
    SessionHost* g = new SessionHost(); InfoFile f(gait_file), tk(task), ref(reference);
    g->horizon = horizon; g->stance = tk.number("model_settings.phaseTransitionStanceTime", 0.4);
    g->table.resize(n);
    for (int i = 0; i < n; ++i) {
      const ModeTemplate t = read_mode_template(f, names[i]); GsTemplate& x = g->table[i]; std::memset(&x, 0, sizeof(x));
      x.n = (int32_t)t.modes.size(); for (int k = 0; k < x.n; ++k) x.md[k] = t.modes[k]; for (int k = 0; k <= x.n; ++k) x.sw[k] = t.switching_times[k];
    }
    std::memset(&g->init, 0, sizeof(g->init));
    const std::vector<std::string> md = ref.list("initialModeSchedule.modeSequence"), ev = ref.list("initialModeSchedule.eventTimes");
    g->init.n = (int32_t)ev.size();
    for (size_t i = 0; i < md.size(); ++i) g->init.md[i] = mode_from_name(md[i]);
    for (size_t i = 0; i < ev.size(); ++i) g->init.ev[i] = std::stod(ev[i]);
    g->robots.resize(B); g->cursor.assign(B, 0); g->pending.assign(B, GsPending{});
    return g;
  } catch (const std::exception&) { return nullptr; }
}
void gsh_destroy(void* h) { delete static_cast<SessionHost*>(h); }

// robot b as qmb200_gait_dev_reset leaves it: the initial schedule, then template tmpl inserted at t_start; cursor 0, no pending command
int gsh_reset(void* h, int b, int tmpl, double t_start) {
  SessionHost* g = static_cast<SessionHost*>(h); GsRobot& r = g->robots[b];
  std::memset(&r, 0, sizeof(r)); r.s = g->init; r.tmpl = tmpl; g->cursor[b] = 0; std::memset(&g->pending[b], 0, sizeof(GsPending));
  return gs_insert(r.s, g->table[tmpl], t_start, g->horizon, g->stance);
}
// the timeline with end-effector rows [B][n_cmd]; every cursor back to 0
void gsh_set_commands(void* h, int n_cmd, const double* t, const int32_t* tmpl, const double* vel, const int32_t* ee_kind, const double* ee) {
  SessionHost* g = static_cast<SessionHost*>(h); const size_t n = g->robots.size() * n_cmd;
  g->n_cmd = n_cmd; g->t.assign(t, t + n); g->tmpl.assign(tmpl, tmpl + n); g->vel.assign(vel, vel + 4 * n);
  g->ee_kind.assign(ee_kind, ee_kind + n); g->ee.assign(ee, ee + 7 * n);
  for (int32_t& c : g->cursor) c = 0;
}
// gait_command_kernel's body for every robot
void gsh_command(void* h, const int32_t* mask, const int32_t* tmpl, const double* vel, const int32_t* ee_kind, const double* ee, int32_t* status) {
  SessionHost* g = static_cast<SessionHost*>(h);
  for (size_t b = 0; b < g->robots.size(); ++b) {
    if (!mask[b]) { status[b] = 0; continue; }
    status[b] = gs_command_check(tmpl[b], vel + 4 * b, ee_kind[b], ee + 7 * b, (int)g->table.size());
    if (status[b]) continue;
    GsPending& p = g->pending[b];
    p.set = 1; p.tmpl = tmpl[b]; p.ee_kind = ee_kind[b]; p.pad = 0;
    for (int i = 0; i < 4; ++i) p.vel[i] = vel[4 * b + i];
    for (int i = 0; i < 7; ++i) p.ee[i] = ee[7 * b + i];
  }
}
// the step kernel's body for every robot; with_pending 0: gs_step without a pending slot (the step before this feature)
void gsh_step(void* h, const double* t_obs, int32_t* n_events, double* event_times, int32_t* modes, double* cmd, int32_t* target_kind, int32_t* status, int with_pending) {
  SessionHost* g = static_cast<SessionHost*>(h);
  const GsCommands c{g->n_cmd, g->t.data(), g->tmpl.data(), g->vel.data(), g->ee_kind.data(), g->ee.data()};
  for (size_t b = 0; b < g->robots.size(); ++b)
    status[b] = with_pending ? gs_step(g->robots[b], &g->cursor[b], g->table.data(), c, (int)b, t_obs[b], g->horizon, g->stance, n_events + b, event_times + b * QMB200_EMAX,
                                       modes + b * (QMB200_EMAX + 1), cmd + b * 7, target_kind + b, &g->pending[b])
                             : gs_step(g->robots[b], &g->cursor[b], g->table.data(), c, (int)b, t_obs[b], g->horizon, g->stance, n_events + b, event_times + b * QMB200_EMAX,
                                       modes + b * (QMB200_EMAX + 1), cmd + b * 7, target_kind + b);
}
// the bytes of each robot's GsRobot [B][robot_bytes], its cursor and its pending slot's set flag
int gsh_robot_bytes() { return (int)sizeof(GsRobot); }
void gsh_get(void* h, unsigned char* robots, int32_t* cursor, int32_t* set) {
  SessionHost* g = static_cast<SessionHost*>(h);
  std::memcpy(robots, g->robots.data(), g->robots.size() * sizeof(GsRobot));
  for (size_t b = 0; b < g->robots.size(); ++b) { cursor[b] = g->cursor[b]; set[b] = g->pending[b].set; }
}
// gs_command_check of m rows against a table of n_templates templates
void gsh_check(int m, const int32_t* tmpl, const double* vel, const int32_t* ee_kind, const double* ee, int n_templates, int32_t* out) {
  for (int i = 0; i < m; ++i) out[i] = gs_command_check(tmpl[i], vel + 4 * i, ee_kind[i], ee + 7 * i, n_templates);
}

}  // extern "C"
