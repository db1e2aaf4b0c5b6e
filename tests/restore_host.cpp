// TEST INFRASTRUCTURE: host build (g++) of the masked row gather of image_restore_kernel (qm_control_b200/csrc/kernels/respawn_api.cuh), so that the CPU
// suite can check the rule behind the start image's restore and the robot-state snapshots without a GPU (tests/test_robot_state_cpu.py).  rh_gather
// walks every word of every segment in the kernel's order and applies the very functions the kernel runs.
#include <cstdint>

#include "kernels/respawn_api.cuh"

using namespace qmb;

extern "C" {

// n segments: dst[i] [B][words[i]] (in-out), src[i] [B][words[i]] or NULL (zeros); mask [B] or NULL (every robot), row [B] or NULL (b); status [B] or NULL
int rh_gather(int n, uint32_t* const* dst, const uint32_t* const* src, const int32_t* words, int B, const int32_t* mask, const int32_t* row, int32_t* status) {
  if (n > RESTORE_MAX_SEGS) return -1;
  RestoreTable t{};
  for (int i = 0; i < n; ++i) t.seg[t.n++] = RestoreSeg{dst[i], src[i], words[i]};
  for (int s = 0; s < t.n; ++s) {
    const RestoreSeg g = t.seg[s];
    for (int64_t i = 0; i < (int64_t)B * g.words; ++i) {
      const int b = (int)(i / g.words); int r;
      if (restore_source(B, mask, row, b, r)) g.dst[i] = restore_word(g, r, i - (int64_t)b * g.words);
    }
  }
  if (status)
    for (int b = 0; b < B; ++b) status[b] = restore_status(B, mask, row, b);
  return 0;
}

int rh_max_segs() { return RESTORE_MAX_SEGS; }

}  // extern "C"
