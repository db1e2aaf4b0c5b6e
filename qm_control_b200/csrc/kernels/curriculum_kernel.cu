// Per-robot curricula (include/qmb200.h: qmb200_curriculum_update_dev; DESIGN.md §4.15).
//   curriculum_update_kernel   one thread per robot: a masked robot whose episode closed with end 1 or 2 updates its state from the end code and, when
//                              the rule has conditions, the episode's metrics row (curriculum_outcome, curriculum_step, the host's core), writes its level
//                              and writes the box at that level into the ranges of every attached kind.  Unmasked robots are not written.
#include "curriculum_api.cuh"

namespace qmb {

namespace {
constexpr int CU_THREADS = 128;

// robot b's box of one kind of width W (round_col: the integer column, -1 none) at `level` into the kind's ranges
template <int W, int ROUND_COL>
__device__ __forceinline__ void write_box(const CurriculumKind k, size_t b, int level, int n_levels) {
  const size_t o = b * W;
#pragma unroll
  for (int c = 0; c < W; ++c) {
    k.lo[o + c] = curriculum_value(k.base_lo[o + c], k.top_lo[o + c], level, n_levels, c == ROUND_COL);
    k.hi[o + c] = curriculum_value(k.base_hi[o + c], k.top_hi[o + c], level, n_levels, c == ROUND_COL);
  }
}

__global__ void __launch_bounds__(CU_THREADS) curriculum_update_kernel(int B, const CurriculumArgs a, const int32_t* __restrict__ mask, const int32_t* __restrict__ end,
                                                                       const int32_t* __restrict__ episode, const double* __restrict__ metrics, int n_episodes,
                                                                       int32_t* __restrict__ level, int32_t* __restrict__ status) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B || !mask[b]) return;
  const int e = end[b];
  if (e != 1 && e != 2) return;
  const double* m = nullptr;
  if (a.rule.n_cond > 0) {
    const int ep = episode[b];
    if (ep < 0 || ep >= n_episodes) { status[b] |= QMB200_ST_OVERFLOW; return; }
    m = metrics + ((size_t)b * n_episodes + ep) * QMB200_METRICS;
  }
  const double* row = a.rows + (size_t)b * CU_DBL;
  int32_t s[CUS_INT];
#pragma unroll
  for (int i = 0; i < CUS_INT; ++i) s[i] = a.state[(size_t)b * CUS_INT + i];
  curriculum_step(a.rule.n_levels, row, curriculum_outcome(a.rule, row, e, m), s);
#pragma unroll
  for (int i = 0; i < CUS_INT; ++i) a.state[(size_t)b * CUS_INT + i] = s[i];
  level[b] = s[CUS_LEVEL];
  if (a.kind[QMB200_CURRICULUM_EPISODE].lo) write_box<EP_DBL, -1>(a.kind[QMB200_CURRICULUM_EPISODE], b, s[CUS_LEVEL], a.rule.n_levels);
  if (a.kind[QMB200_CURRICULUM_SPAWN].lo) write_box<SP_DBL, SP_TILE>(a.kind[QMB200_CURRICULUM_SPAWN], b, s[CUS_LEVEL], a.rule.n_levels);
  if (a.kind[QMB200_CURRICULUM_TIMELINE].lo) write_box<TL_DBL, -1>(a.kind[QMB200_CURRICULUM_TIMELINE], b, s[CUS_LEVEL], a.rule.n_levels);
  if (a.kind[QMB200_CURRICULUM_EE_PATH].lo) write_box<EPR_DBL, -1>(a.kind[QMB200_CURRICULUM_EE_PATH], b, s[CUS_LEVEL], a.rule.n_levels);
}
}  // namespace

int launch_curriculum_update(int B, const CurriculumArgs& a, const int32_t* mask, const int32_t* end, const int32_t* episode, const double* metrics, int n_episodes,
                             int32_t* level, int32_t* status, cudaStream_t s) {
  curriculum_update_kernel<<<(B + CU_THREADS - 1) / CU_THREADS, CU_THREADS, 0, s>>>(B, a, mask, end, episode, metrics, n_episodes, level, status);
  return 1;
}

}  // namespace qmb
