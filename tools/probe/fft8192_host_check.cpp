// Host emulation of csrc/fft8192.cuh: the 512 threads of the CTA are looped over sequentially between the
// points where the kernel has a barrier.  Checks both transform
// directions against a double-precision O(N^2)-free reference (recursive radix-2) and prints the max error.
//   g++ -O2 -std=c++17 -I dasp_pytorch_b200/csrc tools/probe/fft8192_host_check.cpp -o /tmp/fft8192_host_check
#include <cmath>
#include <complex>
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "fft8192.cuh"

using namespace dasp::fft8k;
using cd = std::complex<double>;

static void ref_fft(std::vector<cd>& a, int sign) {
  const size_t n = a.size();
  if (n == 1) return;
  std::vector<cd> e(n / 2), o(n / 2);
  for (size_t i = 0; i < n / 2; ++i) { e[i] = a[2 * i]; o[i] = a[2 * i + 1]; }
  ref_fft(e, sign); ref_fft(o, sign);
  for (size_t k = 0; k < n / 2; ++k) {
    const cd w = std::polar(1.0, sign * 2.0 * M_PI * (double)k / (double)n) * o[k];
    a[k] = e[k] + w; a[k + n / 2] = e[k] - w;
  }
}

template <bool INV>
static double run(unsigned seed) {
  std::vector<float> tab(kTabFloats), gr(kPlaneG), gi(kPlaneG), yr(kPlaneY, 1e30f), yi(kPlaneY, 1e30f);
  for (int e = 0; e < kTabEntries; ++e) {
    int co, so, dup; double turns;
    table_entry(e, co, so, dup, turns);
    const float c = (float)std::cos(2.0 * M_PI * turns), s = (float)std::sin(2.0 * M_PI * turns);
    tab[co] = c; tab[so] = s;
    if (dup) { tab[co + 1] = c; tab[so + 1] = s; }
  }
  const Tables tb = carve_tables(tab.data());
  srand(seed);
  std::vector<cd> ref(kN);
  for (int n = 0; n < kN; ++n) {
    gr[n] = (float)rand() / RAND_MAX - 0.5f; gi[n] = (float)rand() / RAND_MAX - 0.5f;
    ref[n] = cd(gr[n], gi[n]);
  }
  ref_fft(ref, INV ? +1 : -1);
  for (int t = 0; t < kThreads; ++t) p1<INV>(gr.data(), gi.data(), tb, t);
  for (int t = 0; t < kThreads; ++t) p2<INV>(gr.data(), gi.data(), yr.data(), yi.data(), tb, t);
  std::vector<P3Regs> regs(kThreads);
  for (int t = 0; t < kThreads; ++t) p3_load<INV>(yr.data(), yi.data(), t, regs[t]);
  for (int t = 0; t < kThreads; ++t) p3_store<INV>(yr.data(), yi.data(), tb, t, regs[t]);
  double err = 0.0, mag = 0.0;
  for (int t = 0; t < kThreads; ++t) {
    float xr[16], xi[16];
    p4<INV>(yr.data(), yi.data(), t, xr, xi);
    for (int k4 = 0; k4 < 16; ++k4) {
      const cd d = cd(xr[k4], xi[k4]) - ref[t + 512 * k4];
      err = std::fmax(err, std::abs(d));
      mag = std::fmax(mag, std::abs(ref[t + 512 * k4]));
    }
  }
  return err / mag;
}

int main() {
  const double ei = run<true>(1), ef = run<false>(2);
  printf("inverse_rel_err %.3e\nforward_rel_err %.3e\n", ei, ef);
  return (ei < 2e-6 && ef < 2e-6) ? 0 : 1;
}
