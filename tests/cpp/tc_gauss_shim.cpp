// Host-side view of the three-product tensor-core sweep's geometry and layout (reevr_b200/csrc/kernels_tc.cuh), for
// tests/test_tc_gauss.py: the same inline functions the kernels use, compiled by g++ (no GPU needed).
#include "../../reevr_b200/csrc/kernels_tc.cuh"

extern "C" {
void tcg_consts(int* out) {
  out[0] = pc::tc::kGRows; out[1] = pc::tc::kGSliceBytes; out[2] = pc::tc::kGImageBytes; out[3] = pc::tc::kGStages;
  out[4] = pc::tc::kGStripBytes; out[5] = pc::tc::kSmemBytesGauss; out[6] = pc::tc::kStripBytes; out[7] = pc::tc::kGProducts;
  out[8] = pc::tc::kFlushF16; out[9] = pc::tc::kStripRows;
}
void tcg_geom(int P, int nb, int* out) {
  const pc::tc::Geom g = pc::tc::make_geom(P, nb);
  out[0] = g.Q; out[1] = pc::tc::nchunk_f16(g.Q); out[2] = g.ntile; out[3] = g.rows; out[4] = pc::tc::npair(g);
}
int tcg_pair_rows(int ntile, int m) { return pc::tc::pair_rows(ntile, m); }
unsigned long long tcg_a_image_bytes(unsigned long long lines, int nchunk) { return pc::tc::a_image_bytes_gauss(lines, nchunk); }
unsigned tcg_sw128_h(unsigned r, unsigned e) { return pc::tc::sw128_h(r, e); }
unsigned long long tcg_xf_index(long long line, int comp, long long tau, int rows) { return pc::tc::xf_index(line, comp, tau, rows); }
int tcg_scale_exp(unsigned m) { return pc::tc::scale_exp(m); }
}
