// Host-side view of the FP16 tensor-core sweep's geometry, layout and scale functions (reevr_b200/csrc/kernels_tc.cuh),
// for tests/test_tc_f16_layout.py: the same inline functions the kernels use, compiled by g++ (no GPU needed).
#include "../../reevr_b200/csrc/kernels_tc.cuh"

extern "C" {
void tc16_geom(int P, int nb, int* out) {
  const pc::tc::Geom g = pc::tc::make_geom(P, nb);
  out[0] = g.Q; out[1] = pc::tc::nchunk_f16(g.Q); out[2] = g.nseg; out[3] = g.ntile; out[4] = g.rows;
}
int tc16_geom_ok(int P, int nb, int B) { return pc::tc::geom_ok(pc::tc::make_geom(P, nb), B) ? 1 : 0; }
unsigned tc16_sw128_h(unsigned r, unsigned e) { return pc::tc::sw128_h(r, e); }
unsigned long long tc16_xf_index(long long line, int comp, long long tau, int rows) { return pc::tc::xf_index(line, comp, tau, rows); }
unsigned long long tc16_a_image_bytes(unsigned long long lines, int nchunk) { return pc::tc::a_image_bytes(lines, nchunk); }
int tc16_scale_exp(unsigned m) { return pc::tc::scale_exp(m); }
void tc16_consts(int* out) {
  out[0] = pc::tc::kR; out[1] = pc::tc::kN; out[2] = pc::tc::kStripRows; out[3] = pc::tc::kStripBytes; out[4] = pc::tc::kATileBytes;
  out[5] = pc::tc::kChunkK; out[6] = pc::tc::kMaxChunksF16; out[7] = pc::tc::kStageBytes; out[8] = pc::tc::kSmemBytesF16;
  out[9] = pc::tc::kFlushF16; out[10] = pc::tc::kAStages; out[11] = pc::tc::kStripThreads;
}
}
