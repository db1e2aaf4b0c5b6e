// TEST INFRASTRUCTURE: host build (g++) of the device gait schedule's core (qm_control_b200/csrc/kernels/gait_api.cuh) with end-effector commands on
// the timeline, so that the CPU suite can check the target-source protocol without a GPU (tests/test_ee_commands_cpu.py).  Every robot step is gs_step
// with the end-effector rows and the target_kind output, the function gait_step_kernel runs.
#include <cstring>
#include <vector>

#include "host/qm_config.h"
#include "kernels/gait_api.cuh"

using namespace qmb;

namespace {
struct EeHost {
  std::vector<GsTemplate> table; GsSchedule init; std::vector<GsRobot> robots; std::vector<int32_t> cursor;
  std::vector<double> t, vel, ee; std::vector<int32_t> tmpl, ee_kind; bool with_ee = false; int n_cmd = 0; double horizon = 0.0, stance = 0.0;
};
}  // namespace

extern "C" {

// templates names[0..n) of gait_file; B robots; the initial schedule of reference (initialModeSchedule), the stance time of task
void* geh_create(const char* task, const char* reference, const char* gait_file, const char* const* names, int n, int B, double horizon) {
  try {
    EeHost* g = new EeHost(); InfoFile f(gait_file), tk(task), ref(reference);
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
    g->robots.resize(B); g->cursor.assign(B, 0);
    return g;
  } catch (const std::exception&) { return nullptr; }
}
void geh_destroy(void* h) { delete static_cast<EeHost*>(h); }

// robot b: zeroed (cmd_vel source), the initial schedule, then template tmpl inserted at t_start with final horizon; its cursor back to 0
int geh_reset(void* h, int b, int tmpl, double t_start) {
  EeHost* g = static_cast<EeHost*>(h); GsRobot& r = g->robots[b];
  std::memset(&r, 0, sizeof(r)); r.s = g->init; r.tmpl = tmpl; g->cursor[b] = 0;
  return gs_insert(r.s, g->table[tmpl], t_start, g->horizon, g->stance);
}
// the timeline; ee_kind / ee NULL: none of its rows is an end-effector command (the GsCommands of qmb200_gait_dev_set_commands)
void geh_set_commands(void* h, int n_cmd, const double* t, const int32_t* tmpl, const double* vel, const int32_t* ee_kind, const double* ee) {
  EeHost* g = static_cast<EeHost*>(h); const size_t n = g->robots.size() * n_cmd;
  g->n_cmd = n_cmd; g->t.assign(t, t + n); g->tmpl.assign(tmpl, tmpl + n); g->vel.assign(vel, vel + 4 * n);
  g->with_ee = ee_kind != nullptr;
  if (g->with_ee) { g->ee_kind.assign(ee_kind, ee_kind + n); g->ee.assign(ee, ee + 7 * n); } else { g->ee_kind.clear(); g->ee.clear(); }
  for (int32_t& c : g->cursor) c = 0;
}
// the kernel's body for every robot
void geh_step(void* h, const double* t_obs, int32_t* n_events, double* event_times, int32_t* modes, double* cmd, int32_t* tmpl, int32_t* mode, int32_t* status,
              int32_t* target_kind) {
  EeHost* g = static_cast<EeHost*>(h);
  const GsCommands c{g->n_cmd, g->t.data(), g->tmpl.data(), g->vel.data(), g->with_ee ? g->ee_kind.data() : nullptr, g->with_ee ? g->ee.data() : nullptr};
  for (size_t b = 0; b < g->robots.size(); ++b) {
    status[b] = gs_step(g->robots[b], &g->cursor[b], g->table.data(), c, (int)b, t_obs[b], g->horizon, g->stance, n_events + b, event_times + b * QMB200_EMAX,
                        modes + b * (QMB200_EMAX + 1), cmd + b * 7, target_kind + b);
    tmpl[b] = g->robots[b].tmpl; mode[b] = gs_mode_at(g->robots[b].s, t_obs[b]);
  }
}
// each robot's target source and cursor
void geh_get(void* h, int32_t* src, int32_t* cursor) {
  EeHost* g = static_cast<EeHost*>(h);
  for (size_t b = 0; b < g->robots.size(); ++b) { src[b] = g->robots[b].src; cursor[b] = g->cursor[b]; }
}

}  // extern "C"
