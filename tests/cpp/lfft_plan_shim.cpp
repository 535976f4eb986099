// Host-side view of the line-FFT sweep's segment plan (reevr_b200/csrc/kernels_lfft.cuh), for
// tests/test_lfft_sweep.py: the same inline functions the kernels use, compiled by g++ (no GPU needed).
#include "../../reevr_b200/csrc/kernels_lfft.cuh"

extern "C" {
int lfp_n() { return pc::lfft::kN; }
void lfp_plan(int P, int nb, long long* out) {
  const pc::lfft::Plan p = pc::lfft::make_plan(P, nb);
  out[0] = p.P; out[1] = p.Q; out[2] = p.L; out[3] = p.nseg; out[4] = p.Lt; out[5] = p.Lty;
}
long long lfp_window_start(int P, int nb, int q) { return pc::lfft::window_start(pc::lfft::make_plan(P, nb), q); }
long long lfp_output_of(int P, int nb, int q, int m) { return pc::lfft::output_of(pc::lfft::make_plan(P, nb), q, m); }
unsigned long long lfp_spectra_bytes(unsigned long long lines, int C) { return pc::lfft::spectra_bytes(lines, C); }
}
