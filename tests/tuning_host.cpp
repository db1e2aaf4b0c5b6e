// TEST INFRASTRUCTURE: host build (g++) of the node evaluator's cost value (qm_control_b200/csrc/kernels/node_eval.cuh) with a per-robot tuning row, so that
// the CPU suite can check a row against the oracle built from a task.info edited to that row (tests/test_robot_tuning_cpu.py).
#include <string>

#include "host/qm_config.h"
#include "kernels/node_eval.cuh"

using namespace qmb;

extern "C" {

void* tun_create(const char* task, const char* urdf, const char* reference, const char* gains) {
  try { return new HostModel(build_host_model(task, urdf, reference, gains)); } catch (const std::exception&) { return nullptr; }
}
void tun_destroy(void* h) { delete static_cast<HostModel*>(h); }

// the cost value at one node; row: a tuning row [TUNING_DBL] read through tuning_of as the kernels read it, or NULL for the model's own values
double tun_cost(void* h, const double* row, int ne_, const double* ev, const int* modes, int nk, const double* tt, const double* ts, double t, const double* x, const double* u, int terminal) {
  const DevModel* mdl = &static_cast<HostModel*>(h)->dev; ne::BaseKin bk;
  ne::base_eval<false>(mdl, x, bk);
  const int mode = mode_at_time(ev, modes, ne_, t); int fm = 0; for (int i = 0; i < 4; ++i) if (contact_flag(mode, i)) fm |= 1 << i; if (terminal) fm = 0;
  const ne::TargetSeg sg = ne::target_segment(tt, ts, nk, t); double pref[3], qref[4], ee[6]; ne::target_pose(sg, nk, pref, qref);
  ne::ee_eval<false>(mdl, x, bk, pref, qref, ee, nullptr);
  return ne::cost_value(mdl, x, u, sg, ee, fm, terminal != 0, nullptr, row ? tuning_of(mdl, row, 0) : nullptr);
}

}  // extern "C"
