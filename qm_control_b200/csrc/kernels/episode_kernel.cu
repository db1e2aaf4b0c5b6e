// Per-episode plant draws (include/qmb200.h: qmb200_episode_sample_dev; DESIGN.md §4.11).
//   episode_sample_kernel   one thread per robot: a masked robot draws its episode's row from its ranges (episode_row, the host's core) and writes it to
//                           the row buffer, the plant's robot params and, as linked, the controller's model payload (SRBD rows through srbd_payload_fold,
//                           as the payload estimator's commit) and the tuning rows' friction coefficients.  Unmasked robots are not written.
#include "episode_api.cuh"

namespace qmb {

namespace {
constexpr int EP_THREADS = 128;

__global__ void __launch_bounds__(EP_THREADS) episode_sample_kernel(const DevModel* __restrict__ mdl, int B, int64_t robot0, const double* __restrict__ lo,
                                                                    const double* __restrict__ hi, uint64_t seed, const int32_t* __restrict__ mask,
                                                                    const int32_t* __restrict__ episode, double* __restrict__ rows, const EpisodeTargets t) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B || !mask[b]) return;
  double r[EP_DBL];
  episode_row(lo + (size_t)b * EP_DBL, hi + (size_t)b * EP_DBL, seed, (uint64_t)(robot0 + b), (uint64_t)(int64_t)episode[b], r);
#pragma unroll
  for (int c = 0; c < EP_DBL; ++c) rows[(size_t)b * EP_DBL + c] = r[c];
  t.mu[b] = r[EP_MU];
#pragma unroll
  for (int i = 0; i < 8; ++i) t.payload[(size_t)b * 8 + i] = r[EP_PAYLOAD + i];
  if (t.mpayload) {
#pragma unroll
    for (int i = 0; i < 8; ++i) t.mpayload[(size_t)b * 8 + i] = r[EP_PAYLOAD + i];
    srbd_payload_fold(*mdl, r + EP_PAYLOAD, t.srbd + (size_t)b * SRBD_DBL);
  }
  if (t.tuning) {
    double* tn = t.tuning + (size_t)b * TUNING_DBL;
    if (t.mpc_mu) tn[offsetof(Tuning, friction_mu) / 8] = r[EP_MU];
    if (t.wbc_mu) tn[offsetof(Tuning, wbc_friction) / 8] = r[EP_MU];
  }
}
}  // namespace

int launch_episode_sample(const DevModel* mdl, int B, int64_t robot0, const double* lo, const double* hi, uint64_t seed, const int32_t* mask, const int32_t* episode,
                          double* rows, const EpisodeTargets& t, cudaStream_t s) {
  episode_sample_kernel<<<(B + EP_THREADS - 1) / EP_THREADS, EP_THREADS, 0, s>>>(mdl, B, robot0, lo, hi, seed, mask, episode, rows, t);
  return 1;
}

}  // namespace qmb
