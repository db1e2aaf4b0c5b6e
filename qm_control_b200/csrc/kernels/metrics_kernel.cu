// Per-episode metrics (include/qmb200.h: qmb200_metrics_*; DESIGN.md §4.13).
//   metrics_step_kernel    one thread per robot: one sample of the plant's state after a step into the robot's accumulator row (metrics_step_robot).
//   metrics_close_kernel   one thread per robot: the masked robots' rows out of their accumulators, then the accumulators zeroed (metrics_close_robot).
#include <cstdint>

#include "metrics_api.cuh"

namespace qmb {

namespace {
constexpr int METRICS_THREADS = 128;

__global__ void __launch_bounds__(METRICS_THREADS) metrics_step_kernel(const DevModel* __restrict__ mdl, const SimTerrain terrain, double ground_height, int B,
                                                                       const MetricsStep p) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  metrics_step_robot(*mdl, terrain, ground_height, p, b);
}

__global__ void __launch_bounds__(METRICS_THREADS) metrics_close_kernel(int B, const int32_t* __restrict__ mask, const int32_t* __restrict__ end,
                                                                        const int32_t* __restrict__ episode, int n_episodes, double* __restrict__ acc,
                                                                        double* __restrict__ out, int32_t* __restrict__ status) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B || !mask[b]) return;
  metrics_close_robot(acc + (size_t)b * MA_DBL, end[b], episode[b], n_episodes, out + (size_t)b * n_episodes * MT_DBL, status[b]);
}
}  // namespace

int launch_metrics_step(const DevModel* mdl, const SimTerrain& terrain, double ground_height, int B, const MetricsStep& p, cudaStream_t s) {
  metrics_step_kernel<<<(B + METRICS_THREADS - 1) / METRICS_THREADS, METRICS_THREADS, 0, s>>>(mdl, terrain, ground_height, B, p);
  return 1;
}

int launch_metrics_close(int B, const int32_t* mask, const int32_t* end, const int32_t* episode, int n_episodes, double* acc, double* out, int32_t* status,
                         cudaStream_t s) {
  metrics_close_kernel<<<(B + METRICS_THREADS - 1) / METRICS_THREADS, METRICS_THREADS, 0, s>>>(B, mask, end, episode, n_episodes, acc, out, status);
  return 1;
}

}  // namespace qmb
