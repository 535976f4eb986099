// Host-side view of the four-step sweep's segment plan (reevr_b200/csrc/kernels_fourstep.cuh), for
// tests/test_fourstep_model.py: the same inline functions the kernels use, compiled by g++ (no GPU needed).
#include "../../reevr_b200/csrc/kernels_fourstep.cuh"

extern "C" {
long long fsp_m() { return pc::fs::kM; }
int fsp_n1() { return pc::fs::kN1; }
int fsp_n2() { return pc::fs::kN2; }
int fsp_rows() { return pc::fs::kRows; }
int fsp_plan_ok(int P) { return pc::fs::plan_ok(P) ? 1 : 0; }
void fsp_plan(int P, long long n, long long* out) {
  const pc::fs::Plan p = pc::fs::make_plan(P, n);
  out[0] = p.P; out[1] = p.nseg; out[2] = p.Lh; out[3] = p.L; out[4] = p.n;
}
long long fsp_window_start(int P, long long n, int q) { return pc::fs::window_start(pc::fs::make_plan(P, n), q); }
long long fsp_output_of(int P, long long n, int q, long long m) { return pc::fs::output_of(pc::fs::make_plan(P, n), q, m); }
unsigned long long fsp_work_bytes(int P, long long n, int C) { return pc::fs::work_bytes(pc::fs::make_plan(P, n), C); }
unsigned long long fsp_spectrum_bytes(int C) { return pc::fs::spectrum_bytes(C); }
unsigned long long fsp_hist_bytes(int P, int C) { return pc::fs::hist_bytes(P, C); }
}
