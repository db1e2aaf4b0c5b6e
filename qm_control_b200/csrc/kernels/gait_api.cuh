// Device gait schedule (gait_kernel.cu): per robot, ocs2::legged_robot::GaitSchedule as the host object qmb200_gait keeps it (capi_mpc.inc), on
// fixed-capacity arrays, with a timeline of gait, cmd_vel and end-effector commands, rolled once per MPC tick (include/qmb200.h: qmb200_gait_dev_*;
// DESIGN.md §4.7, §4.8).
// The core (gs_*) is host + device: tests/gait_host.cpp compiles it with g++ and checks it against the host objects on the CPU.  Its arithmetic is
// that of qmb200_gait_insert_template / qmb200_gait_get_mode_schedule: the event times come out bit for bit equal.
#pragma once
#include "dev_common.cuh"
#include "../../../include/qmb200.h"

namespace qmb {

constexpr int GS_MAXM = QMB200_GAIT_MAXM;   // modes of one template
constexpr int GS_CAP = QMB200_GAIT_CAP;     // events of one robot's schedule while a step works on it (a window holds at most QMB200_EMAX)
constexpr int GS_STANCE = 15;

// one ModeSequenceTemplate: modes md[n], switching times sw[n + 1] (strictly increasing)
struct GsTemplate { int32_t n; int32_t md[GS_MAXM]; double sw[GS_MAXM + 1]; };
// one robot's schedule: event times ev[n] (strictly increasing) and the n + 1 modes md[0..n] before, between and after them
struct GsSchedule { int32_t n; int32_t md[GS_CAP + 1]; double ev[GS_CAP]; };
// the target source of a robot's publisher (DESIGN.md §4.8): the cmd_vel stream (0, a zeroed robot's), the ee_cmd_vel stream, a published goal
// that is held, or an end-effector path that is followed (DESIGN.md §4.20)
constexpr int GS_SRC_CMD_VEL = QMB200_TARGET_CMD_VEL, GS_SRC_EE_CMD_VEL = QMB200_TARGET_EE_CMD_VEL, GS_SRC_EE_GOAL = QMB200_TARGET_EE_GOAL;
constexpr int GS_SRC_EE_PATH = QMB200_TARGET_EE_PATH;
constexpr int GS_KIND_HELD = -1;   // target kind of a robot whose goal is held: its target call writes nothing
constexpr int GS_KIND_FOLLOW = QMB200_TARGET_EE_PATH_FOLLOW;   // target kind of a robot that follows its path
// one robot's device state: the stored schedule, the active template (its index in the handle's table) and the target source
struct GsRobot { GsSchedule s; int32_t tmpl; int32_t src; };
// one robot's commands (robot-major arrays [B][n_cmd]): time t (sorted per robot), template (-1: none), cmd_vel row [4] (NaN: none), and optionally
// an end-effector command: kind (-1: none, QMB200_TARGET_EE_CMD_VEL, QMB200_TARGET_EE_GOAL, QMB200_TARGET_EE_PATH) with its row [7] (ee_cmd_vel:
// vx, vy, vz; goal: pos, quat xyzw; path: the path index).  NULL ee_kind: no end-effector rows.  A row carries at most one of cmd_vel and an end-effector command.
struct GsCommands { int n; const double* t; const int32_t* tmpl; const double* vel; const int32_t* ee_kind = nullptr; const double* ee = nullptr; };
// one robot's pending command (qmb200_gait_dev_command): one row of GsCommands without its time, applied by the robot's next step.  set 0: none.
// Zeroed words are an empty slot, so the restore clears it with one zero segment.
struct GsPending { int32_t set; int32_t tmpl; double vel[4]; int32_t ee_kind; int32_t pad; double ee[7]; };

QMB_HD int gs_lower_bound(const double* a, int n, double t) { int lo = 0, hi = n; while (lo < hi) { const int mid = (lo + hi) >> 1; if (a[mid] < t) lo = mid + 1; else hi = mid; } return lo; }

// GaitSchedule::tileModeSequenceTemplate(startTime, finalTime): [.. last mode] start [template repeated until the last event >= final] STANCE.
// -2 when start is not after the last event (as the host) or the events would exceed GS_CAP; s is then partly written.
QMB_HD int gs_tile(GsSchedule& s, const GsTemplate& t, double start, double final_time) {
  if (s.n > 0 && start <= s.ev[s.n - 1]) return -2;
  if (s.n >= GS_CAP) return -2;
  s.ev[s.n++] = start;
  while (s.ev[s.n - 1] < final_time)
    for (int i = 0; i < t.n; ++i) {
      if (s.n >= GS_CAP) return -2;
      s.md[s.n] = t.md[i]; s.ev[s.n] = s.ev[s.n - 1] + (t.sw[i + 1] - t.sw[i]); ++s.n;
    }
  s.md[s.n] = GS_STANCE; return 0;
}

// GaitSchedule::insertModeSequenceTemplate(template, startTime, finalTime): drop the events from start on, stance_time of stance unless the
// schedule already ends standing, then the template.  0 or -2 (s partly written).
QMB_HD int gs_insert(GsSchedule& s, const GsTemplate& t, double start, double final_time, double stance_time) {
  const int idx = gs_lower_bound(s.ev, s.n, start);
  if (idx < s.n) s.n = idx;
  const double stance = s.md[s.n] == GS_STANCE ? 0.0 : stance_time;
  if (stance > 0.0) { if (s.n >= GS_CAP) return -2; s.ev[s.n++] = start; s.md[s.n] = GS_STANCE; }
  return gs_tile(s, t, start + stance, final_time);
}

// GaitSchedule::getModeSchedule(lower, upper): keep one event before lower (its mode forced to stance), drop the final stance phase, re-tile from
// the last event to upper.  The schedule then is the window: returns its event count (<= QMB200_EMAX) or -2 (s partly written).
// A schedule is never empty here: every tile leaves at least its start event.
QMB_HD int gs_get(GsSchedule& s, const GsTemplate& t, double lower, double upper) {
  const int idx = gs_lower_bound(s.ev, s.n, lower);
  if (idx > 0) {
    const int d = idx - 1; s.n -= d;
    for (int i = 0; i < s.n; ++i) { s.ev[i] = s.ev[i + d]; s.md[i] = s.md[i + d]; }
    s.md[s.n] = s.md[s.n + d]; s.md[0] = GS_STANCE;
  }
  const double tiling_start = s.ev[s.n - 1];
  --s.n;
  if (int rc = gs_tile(s, t, tiling_start, upper)) return rc;
  return s.n > QMB200_EMAX ? -2 : s.n;
}

// the target kind of a robot's target call on a tick: a goal or path started by this tick's step (applied = QMB200_TARGET_EE_GOAL or _EE_PATH), else
// the source's stream, GS_KIND_HELD for a held goal, GS_KIND_FOLLOW for a path
QMB_HD int gs_target_kind(int src, int applied) {
  return applied == GS_SRC_EE_GOAL || applied == GS_SRC_EE_PATH ? applied : src == GS_SRC_EE_GOAL ? GS_KIND_HELD : src == GS_SRC_EE_PATH ? GS_KIND_FOLLOW : src;
}

// the rules qmb200_gait_dev_set_commands_ee checks on the host, for one command row: QMB200_ST_COMMAND when the template lies outside [-1, n_templates),
// the cmd_vel row is neither all finite nor all NaN, the kind is not -1, QMB200_TARGET_EE_CMD_VEL, QMB200_TARGET_EE_GOAL or QMB200_TARGET_EE_PATH, an
// end-effector value (ee[0:3] of ee_cmd_vel, ee[0:7] of a goal) is not finite, a goal quaternion's norm differs from 1 by more than 1e-9, a path index
// ee[0] is not an integer in [0, n_paths), or the row carries both a cmd_vel and an end-effector command; else 0
QMB_HD int gs_command_check(int tmpl, const double* vel, int ee_kind, const double* ee, int n_templates, int n_paths = 0) {
  if (tmpl < -1 || tmpl >= n_templates) return QMB200_ST_COMMAND;
  const bool none = isnan(vel[0]);
  for (int i = 0; i < 4; ++i) if (none ? !isnan(vel[i]) : !isfinite(vel[i])) return QMB200_ST_COMMAND;
  if (ee_kind == -1) return 0;
  if (ee_kind != GS_SRC_EE_CMD_VEL && ee_kind != GS_SRC_EE_GOAL && ee_kind != GS_SRC_EE_PATH) return QMB200_ST_COMMAND;
  if (!none) return QMB200_ST_COMMAND;
  if (ee_kind == GS_SRC_EE_PATH) return ee[0] >= 0.0 && ee[0] < (double)n_paths && floor(ee[0]) == ee[0] ? 0 : QMB200_ST_COMMAND;
  const bool goal = ee_kind == GS_SRC_EE_GOAL;
  for (int i = 0; i < (goal ? 7 : 3); ++i) if (!isfinite(ee[i])) return QMB200_ST_COMMAND;
  const double qn = sqrt(ee[3] * ee[3] + ee[4] * ee[4] + ee[5] * ee[5] + ee[6] * ee[6]);
  return goal && !(fabs(qn - 1.0) <= 1e-9) ? QMB200_ST_COMMAND : 0;
}

// one command row due at t applied to w: a template is inserted at t + horizon with final horizon, a cmd_vel row fills row[0:4], an ee_cmd_vel row
// row[0:3], a goal row row[0:7], a path row row[0:1]; wrote grows to the longest prefix written, applied becomes the row's target command.  QMB200_ST_OVERFLOW (w partly
// written) or 0.
QMB_HD int gs_apply(GsRobot& w, const GsTemplate* table, int tmpl, const double* vel, int ee_kind, const double* ee, double t, double horizon, double stance_time,
                    double* row, int& wrote, int& applied) {
  if (tmpl >= 0) {
    if (gs_insert(w.s, table[tmpl], t + horizon, horizon, stance_time)) return QMB200_ST_OVERFLOW;
    w.tmpl = tmpl;
  }
  if (!isnan(vel[0])) { for (int i = 0; i < 4; ++i) row[i] = vel[i]; wrote = wrote > 4 ? wrote : 4; applied = GS_SRC_CMD_VEL; }
  if (ee_kind >= 0) {
    const int m = ee_kind == GS_SRC_EE_GOAL ? 7 : ee_kind == GS_SRC_EE_PATH ? 1 : 3;
    for (int i = 0; i < m; ++i) row[i] = ee[i];
    wrote = wrote > m ? wrote : m; applied = ee_kind;
  }
  return 0;
}

// One step of robot b at time t: the robot's commands due at t (time <= t, from *cursor on) in order: a template is inserted at t + horizon with
// final horizon (GaitReceiver::preSolverRun), a cmd_vel row goes to cmd[0:4], an ee_cmd_vel row to cmd[0:3], a goal row to cmd[0:7]; the last of
// these target commands sets the robot's source.  A set pending command (non-NULL pending) is applied after them as one more row due at t, and its
// slot is cleared (set = 0) when the step succeeds.  Then the window [t - horizon, t + 2 horizon] is taken.  All or nothing: status QMB200_ST_NAN
// (non-finite t) or QMB200_ST_OVERFLOW (a window above QMB200_EMAX events, or GS_CAP exceeded) leaves r (its source included), *cursor, the pending
// slot, the MPC rows and cmd untouched.  Otherwise writes n_events, event_times[EMAX] (0 past the count), modes[EMAX + 1] (stance past the count) and cmd.
// target_kind (when non-NULL) is written on every path: gs_target_kind of the source after the step and the last target command it applied.
// Returns the status.
QMB_HD int gs_step(GsRobot& r, int32_t* cursor, const GsTemplate* table, const GsCommands& c, int b, double t, double horizon, double stance_time,
                   int32_t* n_events, double* event_times, int32_t* modes, double* cmd, int32_t* target_kind = nullptr, GsPending* pending = nullptr) {
  if (target_kind) *target_kind = gs_target_kind(r.src, -1);   // a failed step leaves the source as it was
  if (!isfinite(t)) return QMB200_ST_NAN;
  GsRobot w = r; int cur = *cursor; double row[7]; int wrote = 0, applied = -1;   // row[0:wrote]: the cmd slots written (every command writes a prefix)
  for (; cur < c.n && c.t[(size_t)b * c.n + cur] <= t; ++cur) {
    const size_t k = (size_t)b * c.n + cur;
    if (gs_apply(w, table, c.tmpl[k], c.vel + 4 * k, c.ee_kind ? c.ee_kind[k] : -1, c.ee ? c.ee + 7 * k : nullptr, t, horizon, stance_time, row, wrote, applied))
      return QMB200_ST_OVERFLOW;
  }
  const bool pend = pending && pending->set;   // the pending command: one more row due at t, after the timeline's
  if (pend && gs_apply(w, table, pending->tmpl, pending->vel, pending->ee_kind, pending->ee, t, horizon, stance_time, row, wrote, applied))
    return QMB200_ST_OVERFLOW;
  const int n = gs_get(w.s, table[w.tmpl], t - horizon, t + 2.0 * horizon);
  if (n < 0) return QMB200_ST_OVERFLOW;
  *n_events = n;
  for (int i = 0; i < QMB200_EMAX; ++i) event_times[i] = i < n ? w.s.ev[i] : 0.0;
  for (int i = 0; i <= QMB200_EMAX; ++i) modes[i] = i <= n ? w.s.md[i] : GS_STANCE;
  for (int i = 0; i < wrote; ++i) cmd[i] = row[i];
  if (applied >= 0) w.src = applied;
  if (target_kind) *target_kind = gs_target_kind(w.src, applied);
  r = w; *cursor = cur;
  if (pend) pending->set = 0;
  return 0;
}

// the mode of schedule s at t, as the MPC reads it (mode_at_time: the mode after the last event before t)
QMB_HD int gs_mode_at(const GsSchedule& s, double t) { return s.md[gs_lower_bound(s.ev, s.n, t)]; }

// one step per robot (gs_step) at t_obs [B] on the MPC problem rows n_events [B], event_times [B][EMAX], modes [B][EMAX + 1] and cmd [B][7];
// writes status [B], and tmpl [B] (active template), mode [B] (gs_mode_at t_obs of the stored schedule) and target_kind [B] when non-NULL; consumes the
// pending slots [B]
int launch_gait_step(int B, const GsTemplate* table, GsRobot* robots, int32_t* cursor, GsCommands c, double horizon, double stance_time, const double* t_obs,
                     int32_t* n_events, double* event_times, int32_t* modes, double* cmd, int32_t* tmpl, int32_t* mode, int32_t* status, int32_t* target_kind,
                     GsPending* pending, cudaStream_t s);

// one thread per robot: a masked robot's row (tmpl [B], vel [B][4], ee_kind [B], ee [B][7]) that passes gs_command_check (on n_templates templates
// and n_paths end-effector paths) overwrites its pending slot; status [B] = that check's word for masked robots, 0 for the others, whose slots are not
// written
int launch_gait_command(int B, int n_templates, int n_paths, GsPending* pending, const int32_t* mask, const int32_t* tmpl, const double* vel, const int32_t* ee_kind,
                        const double* ee, int32_t* status, cudaStream_t s);

}  // namespace qmb
