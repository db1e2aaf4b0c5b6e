// TEST INFRASTRUCTURE: host build (g++) of the per-episode draw core (qm_control_b200/csrc/kernels/episode_api.cuh), the same functions the sampler kernel
// and qmb200_episode_draw compile, so that the CPU suite can check it against a numpy statement of the hash, the uniform and the fma
// (tests/test_episode_cpu.py).
#include <cstring>

#include "kernels/episode_api.cuh"

using namespace qmb;

extern "C" {

// u of n (seed, robot, episode, channel) tuples
void ep_uniform(int n, const uint64_t* seed, const uint64_t* robot, const uint64_t* episode, const int32_t* channel, double* u) {
  for (int i = 0; i < n; ++i) u[i] = episode_uniform(seed[i], robot[i], episode[i], channel[i]);
}
// the rows [n][EP_DBL] of n (seed, robot, episode) triples on ranges lo, hi [n][EP_DBL]
void ep_rows(int n, const uint64_t* seed, const uint64_t* robot, const uint64_t* episode, const double* lo, const double* hi, double* rows) {
  for (int i = 0; i < n; ++i) episode_row(lo + (size_t)i * EP_DBL, hi + (size_t)i * EP_DBL, seed[i], robot[i], episode[i], rows + (size_t)i * EP_DBL);
}
// qmb200_episode_set_ranges' check on B robots' ranges: 0 when valid, else 1 with the message in msg
int ep_ranges_error(int B, const double* lo, const double* hi, char* msg, int cap) {
  const std::string e = episode_ranges_error(lo, hi, (size_t)B);
  std::strncpy(msg, e.c_str(), cap - 1); msg[cap - 1] = 0;
  return e.empty() ? 0 : 1;
}

}  // extern "C"
