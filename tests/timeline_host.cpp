// TEST INFRASTRUCTURE: host build (g++) of the per-episode timeline draw core (qm_control_b200/csrc/kernels/timeline_api.cuh), the same functions the
// sampler kernel and qmb200_timeline_draw compile, so that the CPU suite can check it against a numpy statement (tests/test_timeline_cpu.py).
#include <cstring>

#include "kernels/timeline_api.cuh"

using namespace qmb;

extern "C" {

// the slots [m][n_cmd][TLC_DBL] of m (seed, robot, episode) triples on ranges lo, hi [m][TL_DBL]
void tl_rows(int m, int n_cmd, const uint64_t* seed, const uint64_t* robot, const uint64_t* episode, const double* lo, const double* hi, double* rows) {
  for (int i = 0; i < m; ++i)
    timeline_rows(lo + (size_t)i * TL_DBL, hi + (size_t)i * TL_DBL, seed[i], robot[i], episode[i], n_cmd, rows + (size_t)i * n_cmd * TLC_DBL);
}
// qmb200_timeline_set_ranges' check on B robots' ranges: 0 when valid, else 1 with the message in msg
int tl_ranges_error(int B, const double* lo, const double* hi, char* msg, int cap) {
  const std::string e = timeline_ranges_error(lo, hi, (size_t)B);
  std::strncpy(msg, e.c_str(), cap - 1); msg[cap - 1] = 0;
  return e.empty() ? 0 : 1;
}

}  // extern "C"
