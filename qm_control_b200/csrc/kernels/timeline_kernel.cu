// Per-episode command timelines (include/qmb200.h: qmb200_timeline_sample_dev; DESIGN.md §4.14).
//   timeline_sample_kernel   one thread per robot: a masked robot draws its episode's n_cmd slots from its ranges (timeline_slot, the host's core) and
//                            writes them to the row buffer and to the device gait schedule's timeline rows, and sets its cursor to 0.  Unmasked robots
//                            are not written.
#include "timeline_api.cuh"

namespace qmb {

namespace {
constexpr int TL_THREADS = 128;

__global__ void __launch_bounds__(TL_THREADS) timeline_sample_kernel(int B, int n_cmd, int64_t robot0, const double* __restrict__ lo, const double* __restrict__ hi,
                                                                     uint64_t seed, const int32_t* __restrict__ mask, const int32_t* __restrict__ episode,
                                                                     double* __restrict__ rows, const TimelineTargets t) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B || !mask[b]) return;
  const double* l = lo + (size_t)b * TL_DBL; const double* h = hi + (size_t)b * TL_DBL;
  const uint64_t robot = (uint64_t)(robot0 + b), ep = (uint64_t)(int64_t)episode[b];
  double tp = 0.0;
  for (int j = 0; j < n_cmd; ++j) {
    double r[TLC_DBL];
    timeline_slot(l, h, seed, robot, ep, j, tp, r);
    tp = r[TLC_T];
    const size_t k = (size_t)b * n_cmd + j;
#pragma unroll
    for (int c = 0; c < TLC_DBL; ++c) rows[k * TLC_DBL + c] = r[c];
    t.t[k] = r[TLC_T]; t.tmpl[k] = (int32_t)r[TLC_TMPL];
#pragma unroll
    for (int i = 0; i < 4; ++i) t.vel[4 * k + i] = r[TLC_CMD_VEL + i];
    if (t.ee_kind) {
      t.ee_kind[k] = (int32_t)r[TLC_EE_KIND];
#pragma unroll
      for (int i = 0; i < 7; ++i) t.ee[7 * k + i] = r[TLC_EE + i];
    }
  }
  t.cursor[b] = 0;
}
}  // namespace

int launch_timeline_sample(int B, int n_cmd, int64_t robot0, const double* lo, const double* hi, uint64_t seed, const int32_t* mask, const int32_t* episode, double* rows,
                           const TimelineTargets& t, cudaStream_t s) {
  timeline_sample_kernel<<<(B + TL_THREADS - 1) / TL_THREADS, TL_THREADS, 0, s>>>(B, n_cmd, robot0, lo, hi, seed, mask, episode, rows, t);
  return 1;
}

}  // namespace qmb
