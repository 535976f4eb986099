// Host-side view of the four-step row pass's work split (reevr_b200/csrc/kernels_fourstep.cuh item_range), for
// tests/test_fourstep_range.py: the same inline function the kernel uses, compiled by g++ (no GPU needed).
#include "../../reevr_b200/csrc/kernels_fourstep.cuh"

extern "C" {
int fsr_rows() { return pc::fs::kRows; }
// the ranges of all ctas CTAs over items items
void fsr_ranges(unsigned items, unsigned ctas, unsigned* begin, unsigned* end) {
  for (unsigned b = 0; b < ctas; ++b) {
    const pc::fs::ItemRange r = pc::fs::item_range(items, ctas, b);
    begin[b] = r.begin;
    end[b] = r.end;
  }
}
}
