// noise_shaped_reverberation forward + backward (reference: dasp_pytorch/functional.py:406-577,
// filter bank dasp_pytorch/signal.py:42-92).
//
// The reference builds, per item and channel, an impulse response as the mean of 12 band-filtered
// white-noise signals (1023-tap FIRs, time-domain conv1d, functional.py:551-556), each shaped by an
// exponential envelope and a gain (:561-567), then convolves the audio with it by a second
// time-domain conv1d with an L-tap kernel (:570-572).  >99.9 % of its time is those two direct
// convolutions.  Here both are FFT convolutions (SURVEY.md Appendix A.5) built from ONE transform shape,
// the 8192-point batched C2C that cuFFT runs as a single shared-memory kernel (long transforms take several
// passes over HBM), with everything between the transforms fused:
//
//   * Only the first Leff = min(L, N) taps of the impulse response can reach the N output samples
//     (y[n] = sum_{t<=n} IR[t] x[n-t], n < N), so only those are synthesised -- an exact saving.
//   * The LEFT and RIGHT channel of a band / of the audio are packed as real/imag of one complex sequence.
//   * IR synthesis, device noise (default): spectral_gen_kernel draws the FILTERED noise spectrum directly
//     (Philox4x32-10 + Box-Muller; see the comment at the kernel); ifft_shape_kernel = own in-shared-memory inverse
//     FFT (fft8192.cuh) fused with envelope * gain * band mean -> IR written straight into the partition layout of
//     the convolution.  For R <= 6 both run as one warp-specialised cluster kernel (ir_synth_cluster_kernel), so the
//     spectrum never goes to HBM.  (Test-hook variants: batched cuFFT + shape_ir_pp_kernel, and the two kernels.)
//   * IR synthesis, parity mode (caller's noise tensor): overlap-save blocks -> C2C -> cmul_filter_pairs ->
//     inverse C2C -> shape_ir_pairs_kernel.
//   * Audio convolution: uniformly partitioned overlap-save in the frequency domain: x_fft_kernel (window gather +
//     FFT, and the FFT of the IR partitions), partition_mac_kernel, ifft_mix_kernel (inverse FFT + crop + wet/dry mix),
//     all on the own FFT; rows that are not 16-byte aligned use x_blocks_kernel, cuFFT C2C, mix_blocks_kernel.
//   * Items are processed in chunks (chosen by the caller; the Python host uses one item per SM) to bound the workspace.
//
// Backward (A.5): g_fft_kernel, two correlation passes of partition_mac_kernel against the saved block spectra (dL/dx
// windows, dL/dIR partitions), ifft_dx_kernel (+ dL/dmix partials), ifft_irgrad_kernel (dL/dIR * env * f reductions for
// the 24 band parameters; deterministic two-stage sums); the cuFFT variants are g_blocks_kernel, C2C,
// finish_dx_blocks_kernel, inverse C2C, ir_grad_*_kernel.
//
// convolution_reverberation is the audio convolution with the caller's IR (ir_pack_kernel fills the partitions).  The
// convolution is written once on the host: conv_fwd_chunk / conv_bwd_chunk run a chunk for both ops, on one ConvGeom,
// one plan set (conv_setup) and one workspace layout per direction; each op adds only its IR fill, its mix stride and
// its dL/dIR consumer.  One IR for the whole batch (dasp_conv_shared_*) is the item stride 0 of the IR spectra: they
// are transformed once, and irgrad_sum_kernel sums the items' dL/dIR spectra in fp64 before one inverse transform.  A
// true-stereo IR (ir_chs 4) is two partition sets per IR (ConvGeom::sets), multiplied by the TS variants of the MAC
// kernels.
//
// Steps that several kernels share are written once: FftSmem (the shared-memory layout of the FFT kernels and their
// double-buffered bulk-copy input), fft8192_in_smem (the four passes), shape_band / store_ir_taps (the epilogue of both
// own-FFT IR syntheses, which therefore give the same bits), band_gain / band_rate (the parameter layout), ir_slot (the
// partition layout of the IR taps) and block_band_sums (the reduction of the 24 band-parameter partials).
#include <cufft.h>
#include <curand_kernel.h>
#include <math.h>

#include <map>
#include <mutex>
#include <tuple>
#include <vector>

#include "common.cuh"
#include "fft8192.cuh"

namespace dasp {
namespace {

constexpr int kBands = 12;
constexpr int kB = 4096;          // partition / hop of the audio convolution
constexpr int kNbA = 2 * kB;      // its FFT length (single-kernel cuFFT C2C size)
constexpr double kPi = 3.14159265358979323846;

#define DASP_CUFFT_OK(expr)                                                        \
  do {                                                                             \
    cufftResult r__ = (expr);                                                      \
    if (r__ != CUFFT_SUCCESS) {                                                    \
      ::dasp::set_error("%s failed: cufft error %d (%s:%d)", #expr, (int)r__, __FILE__, __LINE__); \
      return DASP_ERR_CUFFT;                                                       \
    }                                                                              \
  } while (0)

// ------------------------------------------------------------------ filter bank (host, fp64)
// scipy.signal.firwin(numtaps, cutoff, window="hamming", pass_zero, scale=True, fs) restated.
// band = [lo, hi] in Hz; lo == 0 -> low-pass, hi == nyquist -> high-pass.
void firwin_hamming(int numtaps, double lo_hz, double hi_hz, double fs, double* h) {
  const double nyq = 0.5 * fs;
  const double left = lo_hz / nyq, right = hi_hz / nyq;
  const double alpha = 0.5 * (numtaps - 1);
  auto sinc = [](double x) { return x == 0.0 ? 1.0 : sin(kPi * x) / (kPi * x); };
  for (int i = 0; i < numtaps; ++i) {
    const double m = i - alpha;
    double v = right * sinc(right * m) - left * sinc(left * m);
    const double w = (numtaps == 1) ? 1.0 : 0.54 - 0.46 * cos(2.0 * kPi * i / (numtaps - 1));
    h[i] = v * w;
  }
  double scale_frequency;
  if (left == 0.0) scale_frequency = 0.0;
  else if (right == 1.0) scale_frequency = 1.0;
  else scale_frequency = 0.5 * (left + right);
  double s = 0.0;
  for (int i = 0; i < numtaps; ++i) s += h[i] * cos(kPi * (i - alpha) * scale_frequency);
  for (int i = 0; i < numtaps; ++i) h[i] /= s;
}

// the 12 filters of signal.octave_band_filterbank (signal.py:42-92), cast to fp32 like the reference
void octave_filterbank(int taps, double sr, std::vector<float>& out) {
  static const double centres[10] = {31.5, 63, 125, 250, 500, 1000, 2000, 4000, 8000, 16000};
  out.assign((size_t)kBands * taps, 0.f);
  std::vector<double> h(taps);
  auto put = [&](int k) { for (int i = 0; i < taps; ++i) out[(size_t)k * taps + i] = (float)h[i]; };
  firwin_hamming(taps, 0.0, 12.0, sr, h.data());                       // low-pass 12 Hz (signal.py:60-64)
  put(0);
  for (int b = 0; b < 10; ++b) {                                       // octave band-passes (:69-78)
    const double lo = centres[b] / sqrt(2.0);
    double hi = centres[b] * sqrt(2.0);
    const double cap = 0.999 * sr / 2.0;
    if (hi > cap) hi = cap;
    firwin_hamming(taps, lo, hi, sr, h.data());
    put(1 + b);
  }
  firwin_hamming(taps, 18000.0, sr / 2.0, sr, h.data());               // high-pass 18 kHz (:84)
  put(11);
}

// ------------------------------------------------------------------ geometry
// the partitioned audio convolution, shared by the reverb and convolution_reverberation
struct ConvGeom {
  int64_t bs, n, L;
  int64_t leff;                 // min(L, n): the only IR taps that can reach the output
  int64_t ib, jb;               // output/input blocks of kB samples, IR partitions of kB taps
  int64_t chunk;
  bool shared = false;          // one impulse response for the whole batch (convolution_reverberation only)
  int sets = 1;                 // partition sets per IR: 2 for a true-stereo IR (convolution_reverberation only)
};

int make_conv_geom(int64_t bs, int64_t n, int64_t L, int64_t chunk, ConvGeom& g) {
  DASP_REQUIRE(bs >= 0 && n >= 1 && L >= 1, "conv: bad shape bs=%lld n=%lld ir_len=%lld", (long long)bs, (long long)n,
               (long long)L);
  g.bs = bs; g.n = n; g.L = L;
  g.leff = L < n ? L : n;
  g.ib = (n + kB - 1) / kB;
  g.jb = (g.leff + kB - 1) / kB;
  if (chunk <= 0) chunk = 4;
  g.chunk = chunk < bs ? chunk : (bs > 0 ? bs : 1);
  return DASP_OK;
}

// the reverb adds the IR synthesis: band filters of taps = P + 1, overlap-save blocks of nb with hop, or polyphase
struct Geom : ConvGeom {
  int64_t taps, P;
  int64_t nb, hop, nbk;
  int64_t rpp;                  // polyphase factor of the spectral synthesis: n1 = rpp*nb >= leff + P
  int64_t n1() const { return rpp * nb; }
  int64_t n1c() const { return n1() / 2 + 1; }
  int64_t nparts_pp() const { return (nb + 255) / 256; }
  // complex samples per (item, band) pair in either filtered-noise layout (overlap-save / polyphase)
  int64_t pair_c64() const { return (nbk > rpp ? nbk : rpp) * nb; }
};

int make_geom(int64_t bs, int64_t n, int64_t L, int64_t taps, int64_t chunk, Geom& g) {
  DASP_REQUIRE(bs >= 0 && n >= 1 && L >= 2, "reverb: bad shape bs=%lld n=%lld num_samples=%lld", (long long)bs,
               (long long)n, (long long)L);
  DASP_REQUIRE(taps >= 1 && (taps % 2) == 1, "num_bandpass_taps must be odd");
  int rc = make_conv_geom(bs, n, L, chunk, g);
  if (rc != DASP_OK) return rc;
  g.taps = taps; g.P = taps - 1;
  const int64_t discard = ((g.P + 3) / 4) * 4;            // >= P, keeps every block 16-byte aligned
  int64_t nb = 8192;
  while (nb < 4 * (discard + 1)) nb *= 2;
  g.nb = nb;
  g.hop = nb - discard;
  g.nbk = (g.leff + g.hop - 1) / g.hop;
  g.rpp = (g.leff + g.P + nb - 1) / nb;
  return DASP_OK;
}

// ------------------------------------------------------------------ plan / filter cache
struct PlanKey {
  int dev; int type; int64_t n, batch, idist, odist;
  bool operator<(const PlanKey& o) const {
    return std::tie(dev, type, n, batch, idist, odist) < std::tie(o.dev, o.type, o.n, o.batch, o.idist, o.odist);
  }
};
struct PlanVal { cufftHandle h; size_t work; };
struct FbKey {
  int dev; int64_t taps, nb; double sr;      // nb < 0: half spectrum at n1 = -nb points (spectral synthesis)
  bool operator<(const FbKey& o) const { return std::tie(dev, taps, nb, sr) < std::tie(o.dev, o.taps, o.nb, o.sr); }
};

std::mutex g_mu;
std::map<PlanKey, PlanVal> g_plans;
std::map<FbKey, cufftComplex*> g_fb;

int get_plan(int type /*0 = R2C, 1 = C2R, 2 = C2C*/, int64_t n, int64_t batch, int64_t idist, int64_t odist, PlanVal& out) {
  int dev = 0;
  DASP_CUDA_OK(cudaGetDevice(&dev));
  PlanKey key{dev, type, n, batch, idist, odist};
  auto it = g_plans.find(key);
  if (it != g_plans.end()) { out = it->second; return DASP_OK; }
  PlanVal pv{};
  DASP_CUFFT_OK(cufftCreate(&pv.h));
  DASP_CUFFT_OK(cufftSetAutoAllocation(pv.h, 0));
  long long nn[1] = {(long long)n};
  long long inembed[1] = {(long long)(type == 1 ? n / 2 + 1 : n)};
  long long onembed[1] = {(long long)(type == 0 ? n / 2 + 1 : n)};
  const cufftType ct = type == 0 ? CUFFT_R2C : (type == 1 ? CUFFT_C2R : CUFFT_C2C);
  DASP_CUFFT_OK(cufftMakePlanMany64(pv.h, 1, nn, inembed, 1, (long long)idist, onembed, 1, (long long)odist, ct,
                                    (long long)batch, &pv.work));
  g_plans[key] = pv;
  out = pv;
  return DASP_OK;
}

// in-place C2C of a plan on stream st with the work area `work`
int exec_c2c(const PlanVal& plan, void* work, void* data, int direction, cudaStream_t st) {
  DASP_CUFFT_OK(cufftSetStream(plan.h, st));
  DASP_CUFFT_OK(cufftSetWorkArea(plan.h, work));
  DASP_CUFFT_OK(cufftExecC2C(plan.h, (cufftComplex*)data, (cufftComplex*)data, direction));
  return DASP_OK;
}

// ------------------------------------------------------------------ kernels
// Overlap-save block layout shared by the kernels below.  For item i (chunk-local), band k, block b,
// sample m < nb the complex element  C[((i*12 + k)*nbk + b)*nb + m]  holds (left, right) of the band
// signal at absolute noise position b*hop + m; after the two FFTs it holds the filtered noise f at time
// t = b*hop + m - P (valid for P <= m < P + hop).

// parity mode: gather the user noise (bs*2 rows x 12 bands x (L+P) samples) into the block layout
__global__ void noise_pairs_layout_kernel(const float* __restrict__ noise, float2* __restrict__ C, int64_t item0,
                                          int nbk, int nb, int hop, int64_t lp) {
  // grid = (nbk, 12, items); threads stride over m
  const int b = blockIdx.x, k = blockIdx.y;
  const int64_t il = blockIdx.z;
  const float* nl = noise + (((item0 + il) * 2 + 0) * kBands + k) * lp;
  const float* nr = noise + (((item0 + il) * 2 + 1) * kBands + k) * lp;
  float2* out = C + ((il * kBands + k) * nbk + b) * (int64_t)nb;
  for (int m = threadIdx.x; m < nb; m += blockDim.x) {
    const int64_t pos = (int64_t)b * hop + m;
    float2 v = make_float2(0.f, 0.f);
    if (pos < lp) v = make_float2(nl[pos], nr[pos]);
    out[m] = v;
  }
}

// performance mode: N(0,1) from Philox4x32-10 (cuRAND device API).  The stream of a band signal is
// addressed by its absolute sample position, so the overlapping part of consecutive blocks is simply
// generated twice and nothing depends on the chunking.
__global__ void noise_pairs_philox_kernel(float2* __restrict__ C, int64_t item0, int nbk, int nb, int hop,
                                          const unsigned long long* seed) {
  const int b = blockIdx.x, k = blockIdx.y;
  const int64_t il = blockIdx.z;
  const unsigned long long sig_l = (unsigned long long)(((item0 + il) * 2 + 0) * kBands + k);
  const unsigned long long sig_r = (unsigned long long)(((item0 + il) * 2 + 1) * kBands + k);
  float4* out = reinterpret_cast<float4*>(C + ((il * kBands + k) * nbk + b) * (int64_t)nb);
  for (int q4 = threadIdx.x; q4 < nb / 4; q4 += blockDim.x) {
    const unsigned long long quad = (unsigned long long)(((int64_t)b * hop) / 4 + q4);   // hop % 4 == 0
    curandStatePhilox4_32_10_t sl, sr;
    curand_init(__ldg(seed), (sig_l << 24) + quad, 0ull, &sl);
    curand_init(__ldg(seed), (sig_r << 24) + quad, 0ull, &sr);
    const float4 l = curand_normal4(&sl), r = curand_normal4(&sr);
    out[q4 * 2 + 0] = make_float4(l.x, r.x, l.y, r.y);
    out[q4 * 2 + 1] = make_float4(l.z, r.z, l.w, r.w);
  }
}

// block spectra *= H_band (full nb-point spectrum of the real filter, 1/nb of the inverse FFT folded in)
__global__ void cmul_filter_pairs_kernel(float2* __restrict__ C, const float2* __restrict__ H, int nbk, int nb) {
  const int b = blockIdx.x, k = blockIdx.y;
  const int64_t il = blockIdx.z;
  float2* c = C + ((il * kBands + k) * nbk + b) * (int64_t)nb;
  const float2* h = H + (int64_t)k * nb;
  for (int f = threadIdx.x; f < nb; f += blockDim.x) {
    const float2 a = c[f], w = h[f];
    c[f] = make_float2(a.x * w.x - a.y * w.y, a.x * w.y + a.y * w.x);
  }
}

// lane-pair helpers of the generator's R-point DFT
__device__ __forceinline__ float2 gen_ffma2(float2 a, float2 b, float2 c) { return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }
__device__ __forceinline__ float2 gen_fmul2(float2 a, float2 b) { return make_float2(a.x * b.x, a.y * b.y); }

// ---- spectral synthesis (device-noise mode) ------------------------------------------------------
// The band-filtered noise only has to be a stationary Gaussian process with the FIR's autocovariance on
// the window [0, leff).  A length-n1 PERIODIC white sequence filtered circularly has exactly that
// covariance for every lag inside the window once n1 >= leff + P, and its spectrum has independent bins:
//   G[j] = H_k[j] Z[j],  Z[j] ~ CN(0, n1)  (real N(0, n1) at j = 0 and n1/2),  G[n1-j] = conj(G[j]).
// So the spectrum is drawn directly (no forward FFT, no separate filter pass) and only ONE inverse
// transform remains.  n1 = R*nb is split Cooley-Tukey style so that the inverse is the fast single-kernel
// nb-point batched C2C:   f[R a + b] = sum_{j1<nb} Q_b[j1] e^{2 pi i j1 a / nb},
//   Q_b[j1] = e^{2 pi i j1 b / n1} * sum_{j2<R} G[j1 + nb j2] e^{2 pi i j2 b / R}
// Polyphase layout: C[((item*12 + k)*R + b)*nb + a] = (f_left, f_right)[R a + b].
// Left/right are packed as G_left + i G_right; one Philox call per canonical bin yields both channels.
// Philox4x32-10 (Salmon et al., SC'11), counter = (c0, c1, c2, c3), key = (k0, k1); written out instead of the
// cuRAND state machinery because this kernel needs exactly one block of 4 words per call site
struct PhiloxKeys { uint2 k[10]; };           // the ten round keys (key + r * Weyl constants): one schedule per thread
__device__ __forceinline__ PhiloxKeys philox_keys(unsigned long long sd) {
  PhiloxKeys ks;
  uint2 k = make_uint2((unsigned)sd, (unsigned)(sd >> 32));
#pragma unroll
  for (int r = 0; r < 10; ++r) { ks.k[r] = k; k.x += 0x9E3779B9u; k.y += 0xBB67AE85u; }
  return ks;
}
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, const PhiloxKeys& ks) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const unsigned long long p0 = (unsigned long long)0xD2511F53u * c.x;
    const unsigned long long p1 = (unsigned long long)0xCD9E8D57u * c.z;
    c = make_uint4((unsigned)(p1 >> 32) ^ c.y ^ ks.k[r].x, (unsigned)p1, (unsigned)(p0 >> 32) ^ c.w ^ ks.k[r].y, (unsigned)p0);
  }
  return c;
}
// two independent N(0,1) from two 32-bit words (Box-Muller; u1 in (0,1], angle in turns)
// MUFU-only transcendental path (lg2, rsq, sin, cos: |abs err| ~ 1e-6, irrelevant for a noise source) -- the
// generator kernel is instruction-issue bound and the accurate logf/sqrtf/sincospif were ~55 % of it
__device__ __forceinline__ float2 box_muller(unsigned a, unsigned b) {
  // uniforms from the top 23 bits placed in the mantissa of [1, 2): no I2F (the conversions share the XU pipe with the
  // four MUFU calls below).  u1 = 2 - [1,2) lies in (0, 1]; the angle (v - 1.5) * 2 pi in [-pi, pi)
  const float u1 = 2.0f - __uint_as_float(0x3f800000u | (a >> 9));
  const float ang = fmaf(__uint_as_float(0x3f800000u | (b >> 9)), 6.283185307179586f, -9.42477796076938f);
  const float m = -2.0f * __logf(u1);                                  // >= 0
  const float r = m * rsqrtf(fmaxf(m, 1e-30f));                        // sqrt(m)
  return make_float2(r * __cosf(ang), r * __sinf(ang));
}

// e^{2 pi i m / R} for every polyphase factor R <= 16 (filled once per device on the host side)
__constant__ float2 c_root[17][16];

// One residue class pair (j1, nb - j1) of one band signal: draws the R bins of each class, runs the R-point
// DFT + twiddle ladder and hands  Q_b[j1], Q_b[nb - j1]  (b = 0 .. R-1) to `emit(b, q_j1, q_mirror)`.
// Shared by the stand-alone generator kernel and the fused synthesis kernel, so both produce the same stream.
template <int R, class Emit>
__device__ __forceinline__ void spectral_unit(int j1, int nb, const float2* __restrict__ h, unsigned long long pair,
                                              const PhiloxKeys& keys, Emit&& emit) {
  const int n1 = R * nb, n1h = n1 / 2;
  // the real-valued bins 0 and n1/2 (variance n1 on the real axis instead of n1/2 per component) only occur in the two
  // self-mirrored classes j1 = 0 and j1 = nb/2: everything else takes the branch-free path
  const bool special_unit = (j1 == 0) || (2 * j1 == nb);
  // value of the packed spectrum G_left + i G_right at bin j (0 <= j < n1) and at its mirror n1 - j
  // `canonical` (j <= n1/2) is a compile-time fact of the unrolled call site: for j1 in [0, nb/2] the bin
  // j1 + nb j2 lies in the lower half exactly when 2 j2 < R (the only tie, j = n1/2, is its own mirror)
  auto draw = [&](int j, bool canonical, float2& at_j, float2& at_mirror) {
    const int jc = canonical ? j : n1 - j;
    // counter = (canonical bin, band pair), key = seed: one Philox block -> both channels' complex Gaussian
    const uint4 rnd = philox4x32_10(make_uint4((unsigned)jc, (unsigned)pair, (unsigned)(pair >> 32), 0x5eedu), keys);
    float2 zl = box_muller(rnd.x, rnd.y), zr = box_muller(rnd.z, rnd.w);
    if (special_unit && (jc == 0 || jc == n1h)) {
      zl = make_float2(zl.x * 1.4142135623730951f, 0.f);
      zr = make_float2(zr.x * 1.4142135623730951f, 0.f);
    }
    const float2 w = h[jc];                                          // H_k / n1 * sqrt(n1 / 2), folded on the host
    const float2 sl = make_float2(w.x * zl.x - w.y * zl.y, w.x * zl.y + w.y * zl.x);   // H Z_left
    const float2 sr = make_float2(w.x * zr.x - w.y * zr.y, w.x * zr.y + w.y * zr.x);   // H Z_right
    const float2 canon = make_float2(sl.x - sr.y, sl.y + sr.x);      // S_l + i S_r           (bin jc)
    const float2 mirr = make_float2(sl.x + sr.y, sr.x - sl.y);       // conj(S_l) + i conj(S_r) (bin n1 - jc)
    if (canonical) { at_j = canon; at_mirror = mirr; } else { at_j = mirr; at_mirror = canon; }
  };

  float2 ga[R], gb[R];
#pragma unroll
  for (int j2 = 0; j2 < R; ++j2) {
    float2 a, m;
    draw(j1 + nb * j2, 2 * j2 < R, a, m);
    ga[j2] = a;
    gb[R - 1 - j2] = m;          // mirror of bin j1 + nb j2 is bin (nb - j1) + nb (R-1-j2)
  }
  // The two residue classes (j1 and nb - j1) go through the SAME R-point DFT and twiddle ladder, so they are
  // carried as the two lanes of float2 values.
  float2 gx[R], gy[R];                       // (class A, class B) real parts / imaginary parts
#pragma unroll
  for (int j2 = 0; j2 < R; ++j2) { gx[j2] = make_float2(ga[j2].x, gb[j2].x); gy[j2] = make_float2(ga[j2].y, gb[j2].y); }
  float2 rx[R], ry[R], nry[R];               // roots of unity broadcast to both lanes
#pragma unroll
  for (int m = 0; m < R; ++m) {
    const float2 r = c_root[R][m];
    rx[m] = make_float2(r.x, r.x); ry[m] = make_float2(r.y, r.y); nry[m] = make_float2(-r.y, -r.y);
  }
  // per-class twiddle steps e^{2 pi i j1 / n1} and e^{2 pi i (nb - j1) / n1} = e^{2 pi i / R} conj(the former)
  float2 w1a, w1b;
  __sincosf(6.283185307179586f * (float)j1 / (float)n1, &w1a.y, &w1a.x);      // argument <= pi / R
  {
    const float2 r1 = (R == 1) ? make_float2(1.f, 0.f) : c_root[R][1 % R];
    w1b = make_float2(fmaf(r1.x, w1a.x, r1.y * w1a.y), fmaf(r1.y, w1a.x, -r1.x * w1a.y));
  }
  const float2 wx = make_float2(w1a.x, w1b.x), wy = make_float2(w1a.y, w1b.y), nwy = make_float2(-w1a.y, -w1b.y);
  float2 tx = make_float2(1.f, 1.f), ty = make_float2(0.f, 0.f);      // twiddle e^{2 pi i j b / n1}, both classes
  // S[b] = sum_{j2} g[j2] e^{+2 pi i j2 b / R}: generic O(R^2) form, or for R = 6 (IR 96000 on 48000 samples, the
  // BASELINE geometry) radix 2 x 3 with literal constants -- 48 pair operations instead of 144
  float2 Sre[R], Sim[R];
  if constexpr (R == 6) {
    const float2 hlf = make_float2(0.5f, 0.5f), nhlf = make_float2(-0.5f, -0.5f);
    const float2 c3 = make_float2(0.8660254037844386f, 0.8660254037844386f), nc3 = make_float2(-0.8660254037844386f, -0.8660254037844386f);
    const float2 one = make_float2(1.f, 1.f), mone = make_float2(-1.f, -1.f);
    auto add = [&](float2 a, float2 b) { return gen_ffma2(b, one, a); };
    auto sub = [&](float2 a, float2 b) { return gen_ffma2(b, mone, a); };
    // 3-point DFT (positive exponent) of (a0, a1, a2): Y0 = a0 + t, Y1/2 = (a0 - t/2) +- i (sqrt3/2) d
    auto dft3 = [&](float2 a0r, float2 a0i, float2 a1r, float2 a1i, float2 a2r, float2 a2i, float2 (&yr)[3], float2 (&yi)[3]) {
      const float2 tr = add(a1r, a2r), ti = add(a1i, a2i), dr = sub(a1r, a2r), di = sub(a1i, a2i);
      yr[0] = add(a0r, tr); yi[0] = add(a0i, ti);
      const float2 mr = gen_ffma2(tr, nhlf, a0r), mi = gen_ffma2(ti, nhlf, a0i);
      yr[1] = gen_ffma2(di, nc3, mr); yi[1] = gen_ffma2(dr, c3, mi);       // + i c d = (-c d_i, c d_r)
      yr[2] = gen_ffma2(di, c3, mr);  yi[2] = gen_ffma2(dr, nc3, mi);
    };
    float2 er[3], ei[3], orr[3], oi[3];
    dft3(gx[0], gy[0], gx[2], gy[2], gx[4], gy[4], er, ei);
    dft3(gx[1], gy[1], gx[3], gy[3], gx[5], gy[5], orr, oi);
    // X[k] = E[k] + W6^k O[k], X[k+3] = E[k] - W6^k O[k];  W6 = (1/2, sqrt3/2), W6^2 = (-1/2, sqrt3/2)
    float2 pr[3], pi[3];
    pr[0] = orr[0]; pi[0] = oi[0];
    pr[1] = gen_ffma2(orr[1], hlf, gen_fmul2(oi[1], nc3));  pi[1] = gen_ffma2(orr[1], c3, gen_fmul2(oi[1], hlf));
    pr[2] = gen_ffma2(orr[2], nhlf, gen_fmul2(oi[2], nc3)); pi[2] = gen_ffma2(orr[2], c3, gen_fmul2(oi[2], nhlf));
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      Sre[k] = add(er[k], pr[k]); Sim[k] = add(ei[k], pi[k]);
      Sre[k + 3] = sub(er[k], pr[k]); Sim[k + 3] = sub(ei[k], pi[k]);
    }
  } else {
#pragma unroll
    for (int b = 0; b < R; ++b) {
      float2 sre = make_float2(0.f, 0.f), sim = make_float2(0.f, 0.f);
#pragma unroll
      for (int j2 = 0; j2 < R; ++j2) {
        const int m = (j2 * b) % R;
        sre = gen_ffma2(gx[j2], rx[m], gen_ffma2(gy[j2], nry[m], sre));
        sim = gen_ffma2(gx[j2], ry[m], gen_ffma2(gy[j2], rx[m], sim));
      }
      Sre[b] = sre; Sim[b] = sim;
    }
  }
#pragma unroll
  for (int b = 0; b < R; ++b) {
    const float2 sre = Sre[b], sim = Sim[b];
    const float2 ore = gen_ffma2(sre, tx, gen_fmul2(sim, make_float2(-ty.x, -ty.y)));
    const float2 oim = gen_ffma2(sre, ty, gen_fmul2(sim, tx));
    emit(b, make_float2(ore.x, oim.x), make_float2(ore.y, oim.y));
    const float2 ntx = gen_ffma2(tx, wx, gen_fmul2(ty, nwy));
    ty = gen_ffma2(tx, wy, gen_fmul2(ty, wx));
    tx = ntx;
  }
}

// PLANAR == false: C[((item*12 + k)*R + b)*nb + j] = (re, im) pairs, the input layout of the batched cuFFT C2C.
// PLANAR == true : the same 64 KB block per (item, band, class) holds [re plane nb][im plane nb] -- the shared-memory
//                  layout of fft8192.cuh, so ifft_shape_kernel can fetch a class with plain bulk copies.
template <int R, bool PLANAR>
__global__ void spectral_gen_kernel(float2* __restrict__ C, const float2* __restrict__ H1, int64_t item0, int nb,
                                    const unsigned long long* seed) {
  const int j1 = blockIdx.x * blockDim.x + threadIdx.x;       // residue class 0 .. nb/2
  if (j1 > nb / 2) return;
  const int k = blockIdx.y;
  const int64_t il = blockIdx.z;
  const unsigned long long pair = (unsigned long long)((item0 + il) * kBands + k);
  const PhiloxKeys keys = philox_keys(__ldg(seed));
  const bool self_mirror = (j1 == 0) || (2 * j1 == nb);     // class nb - j1 is class j1 itself
  float2* outp = C + ((il * kBands + k) * R) * (int64_t)nb;
  spectral_unit<R>(j1, nb, H1 + (int64_t)k * (R * nb / 2 + 1), pair, keys, [&](int b, float2 q, float2 qm) {
    if (PLANAR) {
      float* pl = reinterpret_cast<float*>(outp + (int64_t)b * nb);
      pl[j1] = q.x; pl[nb + j1] = q.y;
      if (!self_mirror) { pl[nb - j1] = qm.x; pl[2 * nb - j1] = qm.y; }
    } else {
      outp[(int64_t)b * nb + j1] = q;
      if (!self_mirror) outp[(int64_t)b * nb + (nb - j1)] = qm;
    }
  });
}

// torch.linspace(0, 1, L) in fp32 (functional.py:561): symmetric fill around the midpoint
__device__ __forceinline__ float time_axis(int64_t t, int64_t L, float step) {
  return (t < L / 2) ? step * (float)t : 1.0f - step * (float)(L - 1 - t);
}

// same values for L < 2^31 without 64-bit integer conversions
__device__ __forceinline__ float time_axis32(int t, int L, float step) {
  return (t < L / 2) ? step * (float)t : 1.0f - step * (float)(L - 1 - t);
}

// the 25 parameters of item il: band gains (0..11), band decays (12..23), mix (24).  Band k contributes
// band_gain exp(band_rate tt) f_k to the IR (the 1/12 of the band mean folded into the gain).
__device__ __forceinline__ float band_gain(const float* params, int64_t il, int k) {
  return params[il * 25 + k] * (1.0f / kBands);
}
__device__ __forceinline__ float band_rate(const float* params, int64_t il, int k) {
  return -(params[il * 25 + kBands + k] * 10.0f + 1.0f);
}

// The partition layout of the audio convolution: IR tap t < leff of item il (and, in the backward, dL/dIR tap t) is the
// (left, right) pair at element ir_slot(il, J, t), the first half of partition slot t / kB.  The offset inside the
// item is computed in the tap's own type (int or int64_t), which keeps 32-bit index arithmetic in the FFT kernels.
template <class Tap>
__device__ __forceinline__ int64_t ir_slot(int64_t il, int J, Tap t) {
  return il * J * (int64_t)kNbA + ((t / kB) * kNbA + t % kB);
}

// IR[c][t] = (1/12) sum_k gain_k exp(-(10 decay_k + 1) tt(t)) f_c[k][t]  for t < leff, written as (left, right)
// complex pairs into the partition layout of the audio convolution (first half of partition t / kB; every synthesis
// variant writes these taps and nothing else).
// grid = (nbk, items): CTA (b, item) produces samples [b*hop, (b+1)*hop).
__global__ void shape_ir_pairs_kernel(const float2* __restrict__ C, const float* __restrict__ params /* chunk x 25 */,
                                      float2* __restrict__ Hb, int64_t L, int64_t leff, int jb, int nbk, int nb,
                                      int hop, int P) {
  const int b = blockIdx.x;
  const int64_t il = blockIdx.y;
  __shared__ float gk[kBands], rk[kBands];
  if (threadIdx.x < kBands) {
    gk[threadIdx.x] = band_gain(params, il, threadIdx.x);
    rk[threadIdx.x] = band_rate(params, il, threadIdx.x);
  }
  __syncthreads();
  const float step = 1.0f / (float)(L - 1);
  for (int m = threadIdx.x; m < hop; m += blockDim.x) {
    const int64_t t = (int64_t)b * hop + m;
    if (t >= leff) break;
    const float tt = time_axis(t, L, step);
    const float2* c = C + ((il * kBands) * nbk + b) * (int64_t)nb + m + P;
    float al = 0.f, ar = 0.f;
#pragma unroll
    for (int k = 0; k < kBands; ++k) {
      const float2 v = c[(int64_t)k * nbk * nb];
      const float e = gk[k] * expf(rk[k] * tt);
      al = fmaf(e, v.x, al);
      ar = fmaf(e, v.y, ar);
    }
    Hb[ir_slot(il, jb, t)] = make_float2(al, ar);
  }
}

// polyphase layout variant, threads in TIME order (coalesced IR stores; the 12 band loads of a thread are
// issued together).  grid = (ceil(leff / 256), items)
__global__ void shape_ir_pp_kernel(const float2* __restrict__ C, const float* __restrict__ params, float2* __restrict__ Hb,
                                   int64_t L, int64_t leff, int jb, int R, int nb) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t il = blockIdx.y;
  __shared__ float gk[kBands], rk[kBands];
  if (threadIdx.x < kBands) {
    gk[threadIdx.x] = band_gain(params, il, threadIdx.x);
    rk[threadIdx.x] = band_rate(params, il, threadIdx.x);
  }
  __syncthreads();
  if (t >= leff) return;
  const int a = t / R, ph = t - a * R;
  const float tt = time_axis(t, L, 1.0f / (float)(L - 1));
  const float2* c0 = C + ((il * kBands) * (int64_t)R + ph) * nb + a;
  float2 v[kBands];
#pragma unroll
  for (int k = 0; k < kBands; ++k) v[k] = c0[(int64_t)k * R * nb];
  float al = 0.f, ar = 0.f;
#pragma unroll
  for (int k = 0; k < kBands; ++k) {
    const float e = gk[k] * __expf(rk[k] * tt);
    al = fmaf(e, v[k].x, al);
    ar = fmaf(e, v[k].y, ar);
  }
  Hb[ir_slot(il, jb, t)] = make_float2(al, ar);
}

// ---- the in-shared-memory FFT of fft8192.cuh as the kernels below use it ---------------------------------------
// One 512-thread CTA per SM; its input is bulk-copied into the planar double buffer G while the other half is transformed.
constexpr int kFusedThreads = fft8k::kThreads;
// G [buffer][re, im][8192], Y (re, im planes of the padded layouts), the twiddle tables, and 32 floats of per-kernel
// scratch (the pad; ifft_shape_kernel keeps the item's band gains and rates there)
constexpr int kFusedSmemFloats = 2 * 2 * fft8k::kPlaneG + 2 * fft8k::kPlaneY + fft8k::kTabFloats + 32;
constexpr size_t kFftSmemBytes = sizeof(float) * kFusedSmemFloats + 2 * sizeof(uint64_t);   // + the two mbarriers
struct FftSmem {
  float* G; float* Yr; float* Yi; float* tabf; float* pad; uint64_t* full;
  __device__ __forceinline__ explicit FftSmem(float* sm) {
    G = sm;
    Yr = sm + 4 * fft8k::kPlaneG;
    Yi = Yr + fft8k::kPlaneY;
    tabf = Yi + fft8k::kPlaneY;
    pad = tabf + fft8k::kTabFloats;
    full = reinterpret_cast<uint64_t*>(pad + 32);
  }
  __device__ __forceinline__ void init(const float* twiddles, int t) {
    if (t == 0) {
      mbar_init(&full[0], 1);
      mbar_init(&full[1], 1);
      fence_barrier_init();
    }
    for (int e = t; e < fft8k::kTabFloats; e += kFusedThreads) tabf[e] = twiddles[e];
    __syncthreads();
  }
  // the planar buffer of unit `it` of a CTA's work list (units alternate between the two halves)
  __device__ __forceinline__ float* buf(int it) const { return G + (it & 1) * 2 * fft8k::kPlaneG; }
  // until the input of unit `it` has landed in buf(it)
  __device__ __forceinline__ void wait(int it) const { mbar_wait(&full[it & 1], (uint32_t)((it >> 1) & 1)); }
  // thread 0 only: bulk-copy the 64 KB planar block src (re plane, im plane) into buf(it)
  __device__ __forceinline__ void load_planar(int it, const float* src) const {
    uint64_t* bar = &full[it & 1];
    float* dst = buf(it);
    mbar_arrive_expect_tx(bar, 2u * kNbA * 4u);
#pragma unroll
    for (int q = 0; q < 4; ++q) tma_load_1d(dst + q * 4096, src + q * 4096, 16384u, bar);
  }
};
// the 512 FFT threads only (named barrier 1; barrier 0 is __syncthreads): the FFT warps of ir_synth_cluster_kernel
__device__ __forceinline__ void fft_sync() { asm volatile("bar.sync 1, %0;" ::"n"(kFusedThreads) : "memory"); }
// the four passes on buffer (gr, gi); `refill()` runs as soon as nobody reads the buffer any more, `early()` two
// passes before the results exist (the place to issue global loads the epilogue needs, so that their latency is
// covered by passes 3 and 4 -- with one lock-stepped CTA per SM nothing else would hide it).  FFT_WARPS: the barriers
// are fft_sync() instead of __syncthreads().
template <bool INV, bool FFT_WARPS = false, class Refill, class Early>
__device__ __forceinline__ void fft8192_in_smem(float* gr, float* gi, const FftSmem& s, const fft8k::Tables& tb, int t,
                                                Refill&& refill, Early&& early, float (&xr)[16], float (&xi)[16]) {
  auto sync = [] { if constexpr (FFT_WARPS) fft_sync(); else __syncthreads(); };
  fft8k::p1<INV>(gr, gi, tb, t);
  sync();
  fft8k::p2<INV>(gr, gi, s.Yr, s.Yi, tb, t);
  fence_proxy_async_smem();                        // pass-1 stores to G (generic proxy) before the refill's async writes
  sync();
  refill();
  fft8k::P3Regs q3;
  fft8k::p3_load<INV>(s.Yr, s.Yi, t, q3);
  sync();
  early();
  fft8k::p3_store<INV>(s.Yr, s.Yi, tb, t, q3);
  sync();
  fft8k::p4<INV>(s.Yr, s.Yi, t, xr, xi);
}

// ---- inverse FFT + envelope / gain / band mean (device-noise mode, nb == 8192) ----------------------------------
// One band of the IR synthesis after its inverse transform (x = the pass-4 outputs of FFT thread t, i.e. the filtered
// noise f of band k at the taps tau_q = R (t + 512 q) + c of polyphase class c): acc += gain_k env_k(tau) f(tau), and f
// is stored as (left, right) pairs at fout[t + 512 q] unless fout is null.  The envelope g_k exp(rr tt(tau)) is
// evaluated at every 4th tap; the three taps in between follow by the constant ratio exp(rr step 512 R) (tt is linear in
// tau up to fp32 rounding of the linspace, so this stays within ~1e-6 of the per-tap evaluation).
__device__ __forceinline__ void shape_band(const float (&xr)[16], const float (&xi)[16], float g_k, float rr, int R, int c,
                                           int L, float step, int t, float2* fout, float (&accr)[16], float (&acci)[16]) {
  float e_prev = 0.f;
  const float rho = __expf(rr * step * (float)(512 * R));
#pragma unroll
  for (int q = 0; q < 16; ++q) {
    const int a = t + 512 * q;
    float e;
    if ((q & 3) == 0) e = g_k * __expf(rr * time_axis32(R * a + c, L, step));
    else e = e_prev * rho;
    e_prev = e;
    accr[q] = fmaf(e, xr[q], accr[q]);
    acci[q] = fmaf(e, xi[q], acci[q]);
    if (fout) fout[a] = make_float2(xr[q], xi[q]);
  }
}
// the accumulated IR taps tau_q = R (t + 512 q) + c below leff of item il into the partition layout
__device__ __forceinline__ void store_ir_taps(float2* Hb, int64_t il, int jb, int R, int c, int leff, int t,
                                              const float (&accr)[16], const float (&acci)[16]) {
#pragma unroll
  for (int q = 0; q < 16; ++q) {
    const int tau = R * (t + 512 * q) + c;
    if (tau < leff) Hb[ir_slot(il, jb, tau)] = make_float2(accr[q], acci[q]);
  }
}

// Replaces the batched cuFFT C2C + shape_ir_pp_kernel pair: the generator's spectrum is read ONCE (bulk copies
// straight into the planar shared-memory layout of fft8192.cuh, double buffered across the 12 bands), transformed
// in shared memory, and each thread accumulates  gain_k env_k(t) f_k(t) / 12  for its 16 taps in registers.  The
// filtered noise f is written back (over the consumed spectrum block, as (left, right) pairs) only when the
// backward needs it.  grid = (R, items): CTA (c, item) owns polyphase class c, i.e. the IR taps R a + c.
__global__ void __launch_bounds__(kFusedThreads, 1)
ifft_shape_kernel(float* __restrict__ Cpl, const float* __restrict__ twiddles, const float* __restrict__ params,
                  float2* __restrict__ Hb, int save_f, int L, int leff, int jb, int R) {
  constexpr int nb = fft8k::kN;
  extern __shared__ __align__(128) float sm[];
  FftSmem s(sm);
  float* gk = s.pad;
  float* rk = s.pad + 16;
  const int t = threadIdx.x, c = blockIdx.x;
  const int64_t il = blockIdx.y;
  float* blk = Cpl + ((il * kBands) * R + c) * (int64_t)(2 * nb);      // band k at blk + k * R * 2 nb
  const int64_t band_stride = (int64_t)R * 2 * nb;

  if (t < kBands) {
    gk[t] = band_gain(params, il, t);
    rk[t] = band_rate(params, il, t);
  }
  s.init(twiddles, t);
  if (t == 0) { s.load_planar(0, blk); s.load_planar(1, blk + band_stride); }
  const fft8k::Tables tb = fft8k::carve_tables(s.tabf);
  const float step = 1.0f / (float)(L - 1);
  float accr[16], acci[16];
#pragma unroll
  for (int q = 0; q < 16; ++q) { accr[q] = 0.f; acci[q] = 0.f; }

  for (int k = 0; k < kBands; ++k) {
    s.wait(k);
    float* gr = s.buf(k);
    float xr[16], xi[16];
    fft8192_in_smem<true>(gr, gr + fft8k::kPlaneG, s, tb, t,
                          [&] { if (t == 0 && k + 2 < kBands) s.load_planar(k + 2, blk + (k + 2) * band_stride); },
                          [] {}, xr, xi);
    shape_band(xr, xi, gk[k], rk[k], R, c, L, step, t,
               save_f ? reinterpret_cast<float2*>(blk + k * band_stride) : nullptr, accr, acci);
    // (Y is next written by pass 2 of the following band, behind the barrier after its pass 1)
  }
  store_ir_taps(Hb, il, jb, R, c, leff, t, accr, acci);
}

// ---- block transforms of the audio convolution on the same in-shared-memory FFT ---------------------------
// One CTA per SM at a time; the input of block m + 2 is bulk-copied into the free half of the double buffer while block
// m is transformed, so the copy engine, the FFT and the epilogue stores overlap.  The forward's two kernels (x_fft_kernel,
// ifft_mix_kernel) give each CTA a bounded run of kConvRun consecutive units (grid = ceil(units / kConvRun)) rather than
// a persistent share: while the next chunk's IR synthesis holds most SMs, a CTA that lands on a freed SM gives it back
// after about 40 us, so the synthesis clusters find whole GPCs again, and the hardware scheduler balances the tail.
#ifndef DASP_CONV_RUN
#define DASP_CONV_RUN 8
#endif
constexpr int kConvRun = DASP_CONV_RUN;

// Both forward block transforms of the audio convolution, one work list of nwin + items*J units (runs of kConvRun):
//   unit m < nwin = items*I:  Xb[(il*I + i)*kNbA + f] = FFT of the window (x_left + i x_right)[(i-1) kB + m], m < kNbA
//                             (zero outside [0, n)): x_blocks_kernel + forward C2C in one kernel.
//   unit nwin + il*J + j:     IR partition j of item il, in place in Hb: only the first kB (left, right) pairs of the slot
//                             are read (the synthesis writes nothing else), taps >= leff and the second half are zeroed in
//                             shared memory, so Hb needs no zero-fill and nobody reads the rest of the slot.
// Requires n % 4 == 0 and 16-byte aligned rows (bulk copies).
__global__ void __launch_bounds__(kFusedThreads, 1)
x_fft_kernel(const float* __restrict__ x, float2* __restrict__ Xb, float2* __restrict__ Hb,
             const float* __restrict__ twiddles, int64_t item0, int I, int J, int64_t n, int64_t leff, int in_chs,
             int nwin, int nunits) {
  extern __shared__ __align__(128) float sm[];
  FftSmem s(sm);
  const int t = threadIdx.x;
  s.init(twiddles, t);
  const fft8k::Tables tb = fft8k::carve_tables(s.tabf);
  const int m0 = blockIdx.x * kConvRun;            // this CTA's units [m0, m1)
  const int m1 = nunits - m0 < kConvRun ? nunits : m0 + kConvRun;
  // all threads: zero padding; thread 0: the bulk copies.  The buffer is addressed as below rather than by s.buf(it):
  // with s.buf(it), nvcc 12.9 schedules the whole kernel differently (same arithmetic); this form keeps the code the
  // timings in DESIGN.md were taken with.
  auto fetch = [&](int it, int m) {
    if (m >= m1) return;
    if (m >= nwin) {                               // partition: its 32 KB of taps land in the im plane, see below
      if (t == 0) {
        float* im = s.G + (it & 1) * 2 * fft8k::kPlaneG + fft8k::kPlaneG;
        const float* src = reinterpret_cast<const float*>(Hb + (int64_t)(m - nwin) * kNbA);
        uint64_t* bar = &s.full[it & 1];
        mbar_arrive_expect_tx(bar, 2u * kB * 4u);
        tma_load_1d(im, src, 16384u, bar);
        tma_load_1d(im + 4096, src + 4096, 16384u, bar);
      }
      return;
    }
    const int64_t il = m / I;
    const int i = m - (int)il * I;
    float* re = s.G + (it & 1) * 2 * fft8k::kPlaneG;
    float* im = re + fft8k::kPlaneG;
    const int64_t s0 = (int64_t)(i - 1) * kB;      // first sample of the window
    const int lo = (i == 0) ? kB : 0;
    const int64_t rem = n - s0;
    const int hi = rem < kNbA ? (int)rem : kNbA;   // valid window samples are [lo, hi)
    for (int e = t; e < lo; e += kFusedThreads) { re[e] = 0.f; im[e] = 0.f; }
    for (int e = hi + t; e < kNbA; e += kFusedThreads) { re[e] = 0.f; im[e] = 0.f; }
    if (t == 0) {
      const float* xl = x + ((item0 + il) * in_chs) * n + s0;
      const float* xr = in_chs == 1 ? xl : xl + n;
      uint64_t* bar = &s.full[it & 1];
      mbar_arrive_expect_tx(bar, 2u * (uint32_t)(hi - lo) * 4u);
      for (int o = lo; o < hi; o += 4096) {
        const uint32_t bytes = (uint32_t)((hi - o < 4096 ? hi - o : 4096) * 4);
        tma_load_1d(re + o, xl + o, bytes, bar);
        tma_load_1d(im + o, xr + o, bytes, bar);
      }
    }
  };
  fetch(0, m0);
  fetch(1, m0 + 1);
  __syncthreads();                                 // the zero padding of the first two buffers is in place
  int it = 0;
  for (int m = m0; m < m1; ++m, ++it) {
    s.wait(it);
    float* gr = s.buf(it);
    float* gi = gr + fft8k::kPlaneG;
    if (m >= nwin) {                               // deinterleave the partition's (left, right) pairs into the planes
      const int64_t lim = leff - (int64_t)((m - nwin) % J) * kB;      // taps e < lim exist (lim > 0)
      float2 v[8];
#pragma unroll
      for (int q = 0; q < 8; ++q) v[q] = reinterpret_cast<const float2*>(gi)[t + 512 * q];
      __syncthreads();
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const int e = t + 512 * q;
        const bool tap = e < lim;                  // a select, not a product: the bytes past leff are never written
        gr[e] = tap ? v[q].x : 0.f;
        gi[e] = tap ? v[q].y : 0.f;
        gr[kB + e] = 0.f;
        gi[kB + e] = 0.f;
      }
      __syncthreads();
    }
    float xr[16], xi[16];
    fft8192_in_smem<false>(gr, gi, s, tb, t, [&] { fetch(it + 2, m + 2); }, [] {}, xr, xi);
    float2* out = m < nwin ? Xb + (int64_t)m * kNbA : Hb + (int64_t)(m - nwin) * kNbA;
#pragma unroll
    for (int q = 0; q < 16; ++q) out[t + 512 * q] = make_float2(xr[q], xi[q]);
  }
}

// inverse C2C of the (planar) product spectra + mix_blocks_kernel in one kernel: block i of item il yields the wet
// samples [i kB, (i+1) kB) as the second half of the transform; y = x + mix (wet - x).
__global__ void __launch_bounds__(kFusedThreads, 1)
ifft_mix_kernel(const float* __restrict__ Ypl, const float* __restrict__ twiddles, const float* __restrict__ x,
                const float* __restrict__ mix_p, int mix_stride, float* __restrict__ y, int64_t item0, int I, int64_t n,
                int in_chs, int nblocks) {
  extern __shared__ __align__(128) float sm[];
  FftSmem s(sm);
  const int t = threadIdx.x;
  s.init(twiddles, t);
  const fft8k::Tables tb = fft8k::carve_tables(s.tabf);
  const int m0 = blockIdx.x * kConvRun;            // this CTA's blocks [m0, m1)
  const int m1 = nblocks - m0 < kConvRun ? nblocks : m0 + kConvRun;
  auto fetch = [&](int it, int m) {
    if (t == 0 && m < m1) s.load_planar(it, Ypl + (int64_t)m * 2 * kNbA);
  };
  fetch(0, m0);
  fetch(1, m0 + 1);
  int it = 0;
  for (int m = m0; m < m1; ++m, ++it) {
    s.wait(it);
    float* gr = s.buf(it);
    float xr[16], xi[16];
    const int64_t il = m / I, b = item0 + il;
    const int i = m - (int)il * I;
    const float mix = mix_p[b * mix_stride];
    const float* xl = x + (b * in_chs) * n;
    const float* xrr = in_chs == 1 ? xl : xl + n;
    float a0[8], a1[8];                            // the dry samples of this thread's 8 outputs
    fft8192_in_smem<true>(gr, gr + fft8k::kPlaneG, s, tb, t, [&] { fetch(it + 2, m + 2); },
                          [&] {
#pragma unroll
                            for (int q = 0; q < 8; ++q) {
                              const int64_t tg = (int64_t)i * kB + (t + 512 * q);
                              a0[q] = tg < n ? xl[tg] : 0.f;
                              a1[q] = tg < n ? xrr[tg] : 0.f;
                            }
                          },
                          xr, xi);
#pragma unroll
    for (int q = 8; q < 16; ++q) {                 // outputs kB .. 2 kB - 1 of the transform
      const int64_t tg = (int64_t)i * kB + (t + 512 * q - kB);
      if (tg < n) {
        y[(b * 2 + 0) * n + tg] = fmaf(mix, xr[q] - a0[q - 8], a0[q - 8]);
        y[(b * 2 + 1) * n + tg] = fmaf(mix, xi[q] - a1[q - 8], a1[q - 8]);
      }
    }
  }
}

// ---- the backward's block transforms on the same in-shared-memory FFT --------------------------------------
// g_fft_kernel     = g_blocks_kernel + forward C2C:  Gs[i] = FFT([0 .. 0 | g block i])  (not scaled by mix)
// ifft_dx_kernel   = inverse C2C + finish_dx_blocks_kernel: one CTA walks the windows of an item in order and keeps
//                    the second half of window i in registers until the first half of window i + 1 arrives, so the
//                    overlap-add of the two windows that cover a sample needs no second pass and no atomics; it also
//                    forms the dL/dmix partials (see there)
// ifft_irgrad_kernel = inverse C2C of the dL/dIR partitions + ir_grad_pp_kernel: the 4096 taps of a partition go to
//                    shared memory and are correlated with the filtered noise f read class by class (coalesced)
//
// Why G is not scaled: the inverse transforms of the dx windows then yield c(s) = sum_tau IR(tau) g(s + tau), the
// gradient of the wet signal with respect to x, and since sum_t g(t) wet(t) = sum_s x(s) c(s),
//   dL/dmix = sum over both channels of g (wet - x) = sum_s x (c - g)
// needs x but not the wet signal, so the forward does not save it.  mix is applied to c in ifft_dx_kernel and to the
// dL/dIR band sums in reverb_param_grad_kernel.

// Gb[(il*I + i)*kNbA + f] = FFT of [zeros(kB) | (g_left + i g_right)[i kB + m], m < kB]
__global__ void __launch_bounds__(kFusedThreads, 1)
g_fft_kernel(const float* __restrict__ gy, float2* __restrict__ Gb, const float* __restrict__ twiddles, int64_t item0,
             int I, int64_t n, int nblocks) {
  extern __shared__ __align__(128) float sm[];
  FftSmem s(sm);
  const int t = threadIdx.x;
  s.init(twiddles, t);
  const fft8k::Tables tb = fft8k::carve_tables(s.tabf);
  auto fetch = [&](int it, int m) {                // all threads: zero padding; thread 0: the bulk copies
    if (m >= nblocks) return;
    const int64_t il = m / I;
    const int i = m - (int)il * I;
    float* re = s.buf(it);
    float* im = re + fft8k::kPlaneG;
    const int64_t s0 = (int64_t)i * kB;            // first sample of the block (lands at offset kB of the window)
    const int64_t rem = n - s0;
    const int len = rem < kB ? (int)rem : kB;
    for (int e = t; e < kB; e += kFusedThreads) { re[e] = 0.f; im[e] = 0.f; }
    for (int e = kB + len + t; e < kNbA; e += kFusedThreads) { re[e] = 0.f; im[e] = 0.f; }
    if (t == 0) {
      const float* gl = gy + ((item0 + il) * 2) * n + s0;
      uint64_t* bar = &s.full[it & 1];
      mbar_arrive_expect_tx(bar, 2u * (uint32_t)len * 4u);
      tma_load_1d(re + kB, gl, (uint32_t)len * 4u, bar);
      tma_load_1d(im + kB, gl + n, (uint32_t)len * 4u, bar);
    }
  };
  fetch(0, blockIdx.x);
  fetch(1, blockIdx.x + gridDim.x);
  __syncthreads();
  int it = 0;
  for (int m = blockIdx.x; m < nblocks; m += gridDim.x, ++it) {
    s.wait(it);
    float* gr = s.buf(it);
    float xr_[16], xi_[16];
    fft8192_in_smem<false>(gr, gr + fft8k::kPlaneG, s, tb, t, [&] { fetch(it + 2, m + 2 * gridDim.x); }, [] {}, xr_, xi_);
    float2* out = Gb + (int64_t)m * kNbA;
#pragma unroll
    for (int q = 0; q < 16; ++q) out[t + 512 * q] = make_float2(xr_[q], xi_[q]);
  }
}

// gx[t] = (1-mix) g[t] + mix c[t],  c[t] = D[q][kB + t - q kB] + D[q+1][t - q kB], q = t / kB, from the planar product
// spectra Dpl (one CTA per item at a time; mono input receives the sum of both channel gradients);
// mix_part[il*I + q] = sum over block q and both channels of x (c - g)  (mono: x counted once per channel)
__global__ void __launch_bounds__(kFusedThreads, 1)
ifft_dx_kernel(const float* __restrict__ Dpl, const float* __restrict__ twiddles, const float* __restrict__ gy,
               const float* __restrict__ x, const float* __restrict__ mix_p, int mix_stride, float* __restrict__ gx,
               float* __restrict__ mix_part, int64_t item0, int items, int I, int64_t n, int in_chs) {
  extern __shared__ __align__(128) float sm[];
  FftSmem s(sm);
  __shared__ float wp[2][kFusedThreads / 32];
  const int t = threadIdx.x;
  s.init(twiddles, t);
  const fft8k::Tables tb = fft8k::carve_tables(s.tabf);
  // work list of this CTA: windows (il, i), il = blockIdx.x, blockIdx.x + gridDim.x, ..., i = 0 .. I-1
  const int my_items = (items - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
  const int total = my_items * I;
  auto fetch = [&](int it) {
    if (t != 0 || it >= total) return;
    const int64_t il = blockIdx.x + (int64_t)(it / I) * gridDim.x;
    const int i = it % I;
    s.load_planar(it, Dpl + (il * I + i) * (int64_t)(2 * kNbA));
  };
  fetch(0);
  fetch(1);
  float pr[8], pi[8];                                // second half of the previous window of this item
  for (int it = 0; it < total; ++it) {
    s.wait(it);
    float* gr = s.buf(it);
    const int64_t il = blockIdx.x + (int64_t)(it / I) * gridDim.x, b = item0 + il;
    const int i = it % I;
    const float mix = mix_p[b * mix_stride];
    const float* g0p = gy + (b * 2) * n;
    const float* xl = x + (b * in_chs) * n;
    const float* xrr = in_chs == 1 ? xl : xl + n;
    // the block finished by this window is i - 1 (its first half); after the last window also block I - 1
    float ga[8], gb[8], xa[8], xb[8];
    float xr[16], xi[16];
    fft8192_in_smem<true>(gr, gr + fft8k::kPlaneG, s, tb, t, [&] { fetch(it + 2); },
                          [&] {
#pragma unroll
                            for (int q = 0; q < 8; ++q) {
                              const int64_t t0 = (int64_t)(i - 1) * kB + (t + 512 * q);
                              const bool in = i > 0 && t0 < n;
                              ga[q] = in ? g0p[t0] : 0.f;
                              gb[q] = in ? g0p[n + t0] : 0.f;
                              xa[q] = in ? xl[t0] : 0.f;
                              xb[q] = in ? xrr[t0] : 0.f;
                            }
                          },
                          xr, xi);
    const float om = 1.0f - mix;
    float acc0 = 0.f, acc1 = 0.f;                    // dL/dmix partials of blocks i - 1 and (last window) I - 1
    if (i > 0) {
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const int64_t tg = (int64_t)(i - 1) * kB + (t + 512 * q);
        if (tg < n) {
          const float c0 = pr[q] + xr[q], c1 = pi[q] + xi[q];
          const float o0 = fmaf(om, ga[q], mix * c0), o1 = fmaf(om, gb[q], mix * c1);
          acc0 = fmaf(xa[q], c0 - ga[q], fmaf(xb[q], c1 - gb[q], acc0));
          if (in_chs == 1) gx[b * n + tg] = o0 + o1;
          else { gx[(b * 2) * n + tg] = o0; gx[(b * 2 + 1) * n + tg] = o1; }
        }
      }
    }
#pragma unroll
    for (int q = 0; q < 8; ++q) { pr[q] = xr[q + 8]; pi[q] = xi[q + 8]; }
    if (i == I - 1) {
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const int64_t tg = (int64_t)i * kB + (t + 512 * q);
        if (tg < n) {
          const float g0 = g0p[tg], g1 = g0p[n + tg];
          const float o0 = fmaf(om, g0, mix * pr[q]), o1 = fmaf(om, g1, mix * pi[q]);
          acc1 = fmaf(xl[tg], pr[q] - g0, fmaf(xrr[tg], pi[q] - g1, acc1));
          if (in_chs == 1) gx[b * n + tg] = o0 + o1;
          else { gx[(b * 2) * n + tg] = o0; gx[(b * 2 + 1) * n + tg] = o1; }
        }
      }
    }
    if (i > 0 || i == I - 1) {                       // uniform over the CTA
      acc0 = warp_sum(acc0);
      acc1 = warp_sum(acc1);
      if ((t & 31) == 0) { wp[0][t >> 5] = acc0; wp[1][t >> 5] = acc1; }
      __syncthreads();
      if (t == 0) {
        float s0 = 0.f, s1 = 0.f;
#pragma unroll
        for (int w = 0; w < kFusedThreads / 32; ++w) { s0 += wp[0][w]; s1 += wp[1][w]; }
        if (i > 0) mix_part[il * I + i - 1] = s0;
        if (i == I - 1) mix_part[il * I + i] = s1;
      }
      // (wp is next written after the barriers inside the following transform)
    }
  }
}

// The partials of the 24 band-parameter gradients of a block: part[2k] = the sum of s0[k] and part[2k + 1] = the sum of
// s1[k] over the block's threads (t = threadIdx.x), warp by warp and then over the nwarps warps in order from warp 0
// (the order fixes the bits of the parameter gradients).  red: [nwarps][24] floats of shared memory, which the caller
// rewrites only behind a later barrier.
__device__ __forceinline__ void block_band_sums(const float (&s0)[kBands], const float (&s1)[kBands],
                                                float (*red)[2 * kBands], int nwarps, int t, float* part) {
  const int lane = t & 31, warp = t >> 5;
#pragma unroll
  for (int k = 0; k < kBands; ++k) {
    const float x0 = warp_sum(s0[k]), x1 = warp_sum(s1[k]);
    if (lane == 0) { red[warp][2 * k] = x0; red[warp][2 * k + 1] = x1; }
  }
  __syncthreads();
  if (t < 2 * kBands) {
    float acc = 0.f;
    for (int w = 0; w < nwarps; ++w) acc += red[w][t];
    part[t] = acc;
  }
}

// unit (il, j): dIR taps [j kB, (j+1) kB) = first half of IFFT(Epl[il][j]) (left, right);
// part[((il*J + j)*12 + k)*2 + {0,1}] = sum_t (dIR_l f_l + dIR_r f_r) env_k(t) {1, tt(t)}  over the partition's taps,
// f in the polyphase layout C[((il*12 + k)*R + c)*nb + a] = f[R a + c].
__global__ void __launch_bounds__(kFusedThreads, 1)
ifft_irgrad_kernel(const float* __restrict__ Epl, const float* __restrict__ twiddles, const float2* __restrict__ C,
                   const float* __restrict__ params /* chunk x 25 */, float* __restrict__ part, int L, int leff, int J,
                   int R, int nunits) {
  constexpr int nb = fft8k::kN;
  extern __shared__ __align__(128) float sm[];
  FftSmem s(sm);
  __shared__ float red[kFusedThreads / 32][2 * kBands];
  __shared__ float rk[kBands];
  __shared__ int cls_lo[17], cls_off[17];            // per class: first a of the partition, prefix count of taps
  const int t = threadIdx.x;
  s.init(twiddles, t);
  const fft8k::Tables tb = fft8k::carve_tables(s.tabf);
  auto fetch = [&](int it, int m) {
    if (t == 0 && m < nunits) s.load_planar(it, Epl + (int64_t)m * 2 * kNbA);
  };
  fetch(0, blockIdx.x);
  fetch(1, blockIdx.x + gridDim.x);
  const float step = 1.0f / (float)(L - 1);
  float2* D = reinterpret_cast<float2*>(s.Yr);        // the partition's taps, after pass 4 has consumed Y
  int it = 0;
  for (int m = blockIdx.x; m < nunits; m += gridDim.x, ++it) {
    s.wait(it);
    float* gr = s.buf(it);
    const int64_t il = m / J;
    const int j = m - (int)il * J;
    const int lo = j * kB, hi = (lo + kB < leff) ? lo + kB : leff;      // taps [lo, hi)
    float xr[16], xi[16];
    fft8192_in_smem<true>(gr, gr + fft8k::kPlaneG, s, tb, t, [&] { fetch(it + 2, m + 2 * gridDim.x); }, [] {}, xr, xi);
    __syncthreads();                                  // every thread is done reading Y (pass 4) and the previous unit's D
    if (t < kBands) rk[t] = band_rate(params, il, t);
    if (t == 0) {
      int off = 0;
      for (int c = 0; c < R; ++c) {
        const int a_lo = (lo - c + R - 1) / R, a_hi = (hi - c + R - 1) / R;      // taps R a + c in [lo, hi)
        cls_lo[c] = a_lo;
        cls_off[c] = off;
        off += (a_hi > a_lo) ? a_hi - a_lo : 0;
      }
      cls_off[R] = off;
    }
#pragma unroll
    for (int q = 0; q < 8; ++q) D[t + 512 * q] = make_float2(xr[q], xi[q]);
    __syncthreads();
    float s0[kBands], s1[kBands];
#pragma unroll
    for (int k = 0; k < kBands; ++k) { s0[k] = 0.f; s1[k] = 0.f; }
    const float2* cb = C + (il * kBands) * (int64_t)R * nb;
    const int ntaps = cls_off[R];
    for (int idx = t; idx < ntaps; idx += kFusedThreads) {
      int c = 0;
      while (c + 1 < R && idx >= cls_off[c + 1]) ++c;
      const int a = cls_lo[c] + (idx - cls_off[c]);
      const int tau = R * a + c;
      const float2 gd = D[tau - lo];
      const float tt = time_axis32(tau, L, step);
      const float2* c0 = cb + (int64_t)c * nb + a;
      float2 v[kBands];
#pragma unroll
      for (int k = 0; k < kBands; ++k) v[k] = c0[(int64_t)k * R * nb];
#pragma unroll
      for (int k = 0; k < kBands; ++k) {
        const float w = fmaf(gd.x, v[k].x, gd.y * v[k].y) * __expf(rk[k] * tt);
        s0[k] += w;
        s1[k] = fmaf(w, tt, s1[k]);
      }
    }
    block_band_sums(s0, s1, red, kFusedThreads / 32, t, part + ((int64_t)m * kBands) * 2);
    // red / rk / cls_* / D are rewritten only after the __syncthreads that follows the next transform
  }
}

// ---- warp-specialised cluster IR synthesis (device-noise mode, nb == 8192, R <= 6; the default) --------------
// spectral_gen_kernel + ifft_shape_kernel as ONE kernel: the 4.7 MB-per-item noise spectrum never leaves the SMs, only
// the IR taps (and f, when a backward follows) are written.
//
// One thread-block CLUSTER of R CTAs per item; CTA c owns polyphase class c, i.e. the IR taps R a + c.  The clusters are
// persistent (as many as the device co-schedules) and walk the chunk's items.  Every CTA has two roles:
//   * warps 0-15 (4 warpgroups): the band loop of ifft_shape_kernel on the same device functions (fft8192_in_smem on
//     the class spectrum of each band, shape_band, store_ir_taps; f into the polyphase f_save layout), so the two give
//     the same bits;
//   * warps 16-27 (3 warpgroups): spectral_unit<R> for the bands ahead of the one being transformed.  The 12 (nb/2 + 1)
//     class pairs of an item are dealt round-robin over the R * 384 generator threads of the cluster; a unit's R
//     results go to the R CTAs as st.async stores into the planar buffer G[band & 1] of that CTA, which complete bytes
//     on its mbarrier full[band & 1] (armed with expect_tx of 64 KB per band by the FFT side).
// After FFT pass 2 the FFT side no longer reads G[band & 1]: one thread arrives (remotely) on empty[band & 1] of every
// CTA of the cluster (arrival count R), and the generators wait on their local empty before writing band + 2 there.
// No cluster-wide barrier is left in the band loop.  setmaxnreg moves the registers to the FFT warps.
// Generation is the slower role (H100: 1.6x faster with 256 than with 128 generator threads, 1.15x more with 384), so
// the generators get every register the FFT side can spare: 512 * 80 + 384 * 56 <= 896 * 72, the pool at launch.  At
// R = 7, 8 (64 registers per generator) only 128 generators would fit, which is slower than the two-kernel synthesis.
constexpr int kMaxClusterR = 6;
constexpr int kSynthGen = 384, kSynthThreads = kFusedThreads + kSynthGen;
constexpr int kSynthFftRegs = 80, kSynthGenRegs = 56;
// dasp_debug_reverb_path(2) selects the two-kernel synthesis for R <= 8 (the test matrix pins it there)
constexpr int kMaxHookR = 8;
constexpr size_t kSynthSmemBytes =
    sizeof(float) * (2 * 2 * fft8k::kPlaneG + 2 * fft8k::kPlaneY + fft8k::kTabFloats) + 4 * sizeof(uint64_t);

__device__ __forceinline__ void cluster_arrive() { asm volatile("barrier.cluster.arrive.release;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.acquire;" ::: "memory"); }
__device__ __forceinline__ unsigned cluster_ctarank() {
  unsigned r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
// shared::cluster address of the same shared-memory location in CTA `rank` (32-bit arithmetic only: see st_async)
__device__ __forceinline__ uint32_t mapa_u32(uint32_t smem_addr, uint32_t rank) {
  uint32_t r;
  asm("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(smem_addr), "r"(rank));
  return r;
}
// 4-byte store into (possibly remote) shared memory that completes 4 bytes of the transaction count of `bar` (same CTA
// as the destination); the completion has release semantics at cluster scope
__device__ __forceinline__ void st_async(uint32_t addr, float v, uint32_t bar) {
  asm volatile("st.async.shared::cluster.mbarrier::complete_tx::bytes.b32 [%0], %1, [%2];" ::"r"(addr),
               "r"(__float_as_uint(v)), "r"(bar)
               : "memory");
}
// relaxed arrive on an mbarrier of any CTA of the cluster; the caller orders its earlier accesses with fence_cluster()
// (one fence for the R arrives of a band instead of one release each)
__device__ __forceinline__ void mbar_arrive_remote(uint32_t cluster_bar) {
  asm volatile("mbarrier.arrive.relaxed.cluster.shared::cluster.b64 _, [%0];" ::"r"(cluster_bar) : "memory");
}
__device__ __forceinline__ void fence_cluster() { asm volatile("fence.acq_rel.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_wait_cluster(uint64_t* bar, uint32_t parity) {
  uint32_t done;
  do {
    asm volatile(
        "{\n.reg .pred p;\n"
        "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n}\n"
        : "=r"(done)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
  } while (!done);
}
template <int R>
__global__ void __launch_bounds__(kSynthThreads, 1)
ir_synth_cluster_kernel(const float2* __restrict__ H1, const float* __restrict__ twiddles, const float* __restrict__ params,
                        float2* __restrict__ Hb, float2* __restrict__ Csave, int64_t item0, int items, int L, int leff,
                        int jb, const unsigned long long* seed) {
  constexpr int nb = fft8k::kN, U = nb / 2 + 1, NG = kSynthGen, NT = kSynthThreads;
  constexpr int CT = R * NG, total = kBands * U;
  constexpr uint32_t kBandBytes = 2u * nb * 4u;    // one class spectrum, planar re / im
  extern __shared__ __align__(128) float sm[];
  const FftSmem s(sm);                             // G, Y and the tables; s.full is not used:
  // full[2] and empty[2] follow the tables directly (no pad, kSynthSmemBytes)
  uint64_t* full = reinterpret_cast<uint64_t*>(s.tabf + fft8k::kTabFloats);
  uint64_t* empty = full + 2;
  const int t = threadIdx.x;
  const unsigned c = cluster_ctarank();
  const int my_items = items > (int)blockIdx.y ? (items - 1 - (int)blockIdx.y) / (int)gridDim.y + 1 : 0;
  const int nbands = my_items * kBands;            // bands this cluster walks: g = item iteration * 12 + band

  for (int e = t; e < fft8k::kTabFloats; e += NT) s.tabf[e] = twiddles[e];
  if (t == 0) {
    mbar_init(&full[0], 1);
    mbar_init(&full[1], 1);
    mbar_init(&empty[0], R);
    mbar_init(&empty[1], R);
    fence_barrier_init();
    if (nbands > 0) mbar_arrive_expect_tx(&full[0], kBandBytes);
    if (nbands > 1) mbar_arrive_expect_tx(&full[1], kBandBytes);
  }
  __syncthreads();
  // every CTA of the cluster must be resident with its barriers initialised before the first remote store
  cluster_arrive();
  cluster_wait();

  if (t >= kFusedThreads) {
    // ---------------- generators
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kSynthGenRegs));
    const int gt = t - kFusedThreads;
    const PhiloxKeys keys = philox_keys(__ldg(seed));
    const uint32_t g_local = smem_u32(s.G), full_local = smem_u32(full);
    int waited = 1;                                // bands < 2 need no free buffer
    for (int i = 0; i < my_items; ++i) {
      const int64_t il = blockIdx.y + (int64_t)i * gridDim.y;
      for (int u = (int)c * NG + gt; u < total; u += CT) {
        const int k = u / U, j1 = u - k * U;
        const int g = i * kBands + k;
        if (g > waited) {                          // G[k & 1] of this CTA is free once every CTA finished band g - 2
          mbar_wait_cluster(&empty[k & 1], (uint32_t)(((g - 2) >> 1) & 1));
          waited = g;
        }
        const unsigned long long pair = (unsigned long long)((item0 + il) * kBands + k);
        const bool self_mirror = (j1 == 0) || (2 * j1 == nb);
        const uint32_t off = (uint32_t)(k & 1) * kBandBytes;
        spectral_unit<R>(j1, nb, H1 + (int64_t)k * (R * nb / 2 + 1), pair, keys, [&](int b, float2 q, float2 qm) {
          const uint32_t base = mapa_u32(g_local + off, (uint32_t)b);
          const uint32_t bar = mapa_u32(full_local + 8u * (uint32_t)(k & 1), (uint32_t)b);
          st_async(base + 4u * j1, q.x, bar);
          st_async(base + 4u * (fft8k::kPlaneG + j1), q.y, bar);
          if (!self_mirror) {
            st_async(base + 4u * (nb - j1), qm.x, bar);
            st_async(base + 4u * (fft8k::kPlaneG + nb - j1), qm.y, bar);
          }
        });
      }
    }
  } else {
    // ---------------- inverse FFT + shaping (the band loop of ifft_shape_kernel)
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kSynthFftRegs));
    const fft8k::Tables tb = fft8k::carve_tables(s.tabf);
    const float step = 1.0f / (float)(L - 1);
    for (int i = 0; i < my_items; ++i) {
      const int64_t il = blockIdx.y + (int64_t)i * gridDim.y;
      float accr[16], acci[16];
#pragma unroll
      for (int q = 0; q < 16; ++q) { accr[q] = 0.f; acci[q] = 0.f; }
      for (int k = 0; k < kBands; ++k) {
        const int g = i * kBands + k;
        // one warp polls the barrier, the others sleep in bar.sync instead of taking issue slots from the generators
        if (t < 32) mbar_wait_cluster(&full[k & 1], (uint32_t)((g >> 1) & 1));
        fft_sync();
        float* gr = s.buf(k);
        float xr[16], xi[16];
        fft8192_in_smem<true, true>(gr, gr + fft8k::kPlaneG, s, tb, t,
                                    [&] {
                                      if (t == 0 && g + 2 < nbands) {      // hand G[k & 1] back for band g + 2
                                        mbar_arrive_expect_tx(&full[k & 1], kBandBytes);
                                        fence_cluster();
#pragma unroll
                                        for (int b = 0; b < R; ++b) {
                                          mbar_arrive_remote(mapa_u32(smem_u32(&empty[k & 1]), (uint32_t)b));
                                        }
                                      }
                                    },
                                    [] {}, xr, xi);
        shape_band(xr, xi, band_gain(params, il, k), band_rate(params, il, k), R, (int)c, L, step, t,
                   Csave ? Csave + ((il * kBands + k) * R + c) * (int64_t)nb : nullptr, accr, acci);
        // (Y is next written by pass 2 of the following band, behind the barrier after its pass 1)
      }
      store_ir_taps(Hb, il, jb, R, (int)c, leff, t, accr, acci);
    }
  }
  // no CTA may leave while a remote store or arrive could still target it
  cluster_arrive();
  cluster_wait();
}

// part[((item*nparts + blockIdx.x)*12 + k)*2 + {0,1}], nparts = gridDim.x; threads stride over time
__global__ void ir_grad_pp_kernel(const float2* __restrict__ Et, const float2* __restrict__ C,
                                  const float* __restrict__ params, float* __restrict__ part, int64_t L, int64_t leff,
                                  int jb, int R, int nb) {
  const int64_t il = blockIdx.y;
  __shared__ float rk[kBands];
  __shared__ float red[8][2 * kBands];
  if (threadIdx.x < kBands) rk[threadIdx.x] = band_rate(params, il, threadIdx.x);
  __syncthreads();
  const float step = 1.0f / (float)(L - 1);
  const float2* cb = C + (il * kBands) * (int64_t)R * nb;
  float s0[kBands], s1[kBands];
#pragma unroll
  for (int k = 0; k < kBands; ++k) { s0[k] = 0.f; s1[k] = 0.f; }
  // two time points per iteration: 24 independent 8-byte loads in flight per thread
  const int stride = gridDim.x * blockDim.x;
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < leff; t += 2 * stride) {
    const int t2 = t + stride;
    const bool has2 = t2 < leff;
    const int a = t / R, ph = t - a * R;
    const int a2 = has2 ? t2 / R : a, ph2 = has2 ? t2 - a2 * R : ph;
    const float2 gd = Et[ir_slot(il, jb, t)];
    const float2 gd2 = has2 ? Et[ir_slot(il, jb, t2)] : make_float2(0.f, 0.f);
    const float2* c0 = cb + (int64_t)ph * nb + a;
    const float2* c1 = cb + (int64_t)ph2 * nb + a2;
    float2 v[kBands], v2[kBands];
#pragma unroll
    for (int k = 0; k < kBands; ++k) { v[k] = c0[(int64_t)k * R * nb]; v2[k] = c1[(int64_t)k * R * nb]; }
    const float tt = time_axis(t, L, step), tt2 = time_axis(has2 ? t2 : t, L, step);
#pragma unroll
    for (int k = 0; k < kBands; ++k) {
      const float w = fmaf(gd.x, v[k].x, gd.y * v[k].y) * __expf(rk[k] * tt);
      const float w2 = fmaf(gd2.x, v2[k].x, gd2.y * v2[k].y) * __expf(rk[k] * tt2);
      s0[k] += w + w2;
      s1[k] = fmaf(w, tt, fmaf(w2, tt2, s1[k]));
    }
  }
  block_band_sums(s0, s1, red, (int)(blockDim.x >> 5), threadIdx.x,
                  part + ((il * gridDim.x + blockIdx.x) * kBands) * 2);
}

// ---- audio convolution: uniformly partitioned overlap-save in the frequency domain -----------------
// y[n] = sum_{t<=n} IR[t] x[n-t] (n < N) with the IR split into J partitions of kB taps and the audio into
// I blocks of kB samples; every transform is the fast single-kernel kNbA-point batched C2C, with the LEFT
// and RIGHT channel packed as real/imag (the channels have different IRs, so the multiply kernels untangle
// the packed spectra through their Hermitian symmetry and re-pack the products).
//   Xs[i] = FFT(x window [(i-1) kB, (i+1) kB)),  Hs[j] = FFT(IR[j kB, (j+1) kB) zero padded)
//   y block i = last kB samples of IFFT(sum_{j<=i} Xs[i-j] Hs[j]) / kNbA
// Backward: Gs[i] = FFT(mix g block i, in the second half), dx windows = IFFT(sum_j conj(Hs[j]) Gs[q+j]),
//   dIR partition j = first kB samples of IFFT(sum_i conj(Xs[i-j]) Gs[i]).

// Xb[(il*I + i)*kNbA + m] = (x_left, x_right)[(i-1) kB + m]
__global__ void x_blocks_kernel(const float* __restrict__ x, float2* __restrict__ Xb, int64_t item0, int I, int64_t n,
                                int in_chs) {
  const int i = blockIdx.x;
  const int64_t il = blockIdx.y;
  const float* xl = x + ((item0 + il) * in_chs) * n;
  const float* xr = in_chs == 1 ? xl : xl + n;
  float2* out = Xb + (il * I + i) * (int64_t)kNbA;
  for (int m = threadIdx.x; m < kNbA; m += blockDim.x) {
    const int64_t idx = (int64_t)(i - 1) * kB + m;
    float2 v = make_float2(0.f, 0.f);
    if (idx >= 0 && idx < n) v = make_float2(xl[idx], xr[idx]);
    out[m] = v;
  }
}

// packed spectrum of (a + i b), a and b real: A[f] = (Z[f] + conj(Z[-f]))/2, B[f] = (Z[f] - conj(Z[-f]))/(2i)
__device__ __forceinline__ void untangle(float2 z, float2 zm, float2& a, float2& b) {
  a = make_float2(0.5f * (z.x + zm.x), 0.5f * (z.y - zm.y));
  b = make_float2(0.5f * (z.y + zm.y), -0.5f * (z.x - zm.x));
}
__device__ __forceinline__ void cfma(float2& acc, float2 p, float2 q) {          // acc += p q
  acc.x = fmaf(p.x, q.x, fmaf(-p.y, q.y, acc.x));
  acc.y = fmaf(p.x, q.y, fmaf(p.y, q.x, acc.y));
}
__device__ __forceinline__ void cfma_conj(float2& acc, float2 p, float2 q) {     // acc += p conj(q)
  acc.x = fmaf(p.x, q.x, fmaf(p.y, q.y, acc.x));
  acc.y = fmaf(p.y, q.x, fmaf(-p.x, q.y, acc.y));
}

// CORR == false: out[o] = sum_{j<nbm, j<=o} A[o-j] B[j]           (o < nout)      forward
// CORR == true : out[o] = sum_{j<nbm, o+j<na} A[o+j] conj(B[j])   (o < nout)      both backward products
// A: [items][na][kNbA], Bm: [items][nbm][kNbA] (bstep 1) or [nbm][kNbA] read by every item (bstep 0: the spectra of an
// IR shared by the batch), Out: [items][nout][kNbA]; per channel, packed spectra.
// grid = (ceil((kNbA/2+1)/128), items); thread = frequency pair (f, kNbA - f).  MAXB > 0: operands cached
// in registers (na, nbm <= MAXB); MAXB == 0: generic loop straight from L2.
// PLANAR: every output block is stored as [re plane kNbA][im plane kNbA] (what ifft_mix_kernel bulk-copies into the
// shared-memory layout of fft8192.cuh) instead of (re, im) pairs (what cuFFT reads).
// TS: a true-stereo IR, stored as two partition sets per IR, set A = h_LL + i h_LR then set B = h_RL + i h_RR:
//   TS == 1, forward: out[o] = sum_j XL[o-j] SA[j] + XR[o-j] SB[j], A untangled into (XL, XR), the sets SA = Bm[j] and
//            SB = Bm[nbm + j] used as stored (A = H_LL + i H_LR, so this is the packed wet spectrum WL + i WR)
//   TS == 1, CORR: DL[o] = sum_j GL[o+j] conj(H_LL[j]) + GR[o+j] conj(H_LR[j]), DR[o] likewise with H_RL, H_RR (both
//            operands untangled), stored packed as DL + i DR: the dL/dx windows
//   TS == 2, CORR: out[o] = sum_j A[o+j] conj(BL[j]), out[nout + o] = sum_j A[o+j] conj(BR[j]), A used as stored, B
//            untangled: the dL/dIR partitions of set A (from XL) and set B (from XR)
// Bm (TS == 1) and Out (TS == 2) then hold 2 nbm / 2 nout blocks per item.
template <int MAXB, bool CORR, bool PLANAR = false, int TS = 0>
__global__ void __launch_bounds__(128) partition_mac_kernel(const float2* __restrict__ A, const float2* __restrict__ Bm,
                                                            float2* __restrict__ Out, int na, int nbm, int nout,
                                                            float scale, int bstep) {
  static_assert(TS == 0 || TS == 1 || (TS == 2 && CORR), "TS == 2 is the dL/dIR correlation");
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f > kNbA / 2) return;
  const int fm = (kNbA - f) & (kNbA - 1);
  const int64_t il = blockIdx.y;
  const float2* a = A + il * (int64_t)na * kNbA;
  const float2* bq = Bm + (il * bstep) * (int64_t)(TS == 1 ? 2 : 1) * nbm * kNbA;
  float2* out = Out + il * (int64_t)(TS == 2 ? 2 : 1) * nout * kNbA;
  auto emit = [&](int o, float2 sl, float2 sr) {
    sl.x *= scale; sl.y *= scale; sr.x *= scale; sr.y *= scale;
    if (PLANAR) {
      float* pl = reinterpret_cast<float*>(out + (int64_t)o * kNbA);
      pl[f] = sl.x - sr.y; pl[kNbA + f] = sl.y + sr.x;
      if (fm != f) { pl[fm] = sl.x + sr.y; pl[kNbA + fm] = sr.x - sl.y; }
    } else {
      out[(int64_t)o * kNbA + f] = make_float2(sl.x - sr.y, sl.y + sr.x);                 // L + i R
      if (fm != f) out[(int64_t)o * kNbA + fm] = make_float2(sl.x + sr.y, sr.x - sl.y);   // conj(L) + i conj(R)
    }
  };
  if constexpr (TS != 0) {
    // a0, a1: block i of A (untangled, or for TS == 2 as stored at f and fm); b0..b3: partition j of Bm (TS == 1
    // forward: set A at f, fm, set B at f, fm; TS == 1 CORR: H_LL, H_LR, H_RL, H_RR; TS == 2: BL, BR)
    auto load_a = [&](int i, float2& a0, float2& a1) {
      if (TS == 1) untangle(a[(int64_t)i * kNbA + f], a[(int64_t)i * kNbA + fm], a0, a1);
      else { a0 = a[(int64_t)i * kNbA + f]; a1 = a[(int64_t)i * kNbA + fm]; }
    };
    auto load_b = [&](int j, float2& b0, float2& b1, float2& b2, float2& b3) {
      const float2* sa = bq + (int64_t)j * kNbA;
      const float2* sb = sa + (int64_t)nbm * kNbA;
      if (TS == 2) { untangle(sa[f], sa[fm], b0, b1); b2 = b3 = make_float2(0.f, 0.f); }
      else if (CORR) { untangle(sa[f], sa[fm], b0, b1); untangle(sb[f], sb[fm], b2, b3); }
      else { b0 = sa[f]; b1 = sa[fm]; b2 = sb[f]; b3 = sb[fm]; }
    };
    // one product term: block ia of A with partition j of Bm into the accumulators (p, q) of output pair (f, fm) or
    // (TS == 1 CORR) (DL, DR), and for TS == 2 (r, s) of set B's output
    auto term = [&](float2 a0, float2 a1, float2 b0, float2 b1, float2 b2, float2 b3, float2& p, float2& q, float2& r,
                    float2& s) {
      if (TS == 2) { cfma_conj(p, a0, b0); cfma(q, a1, b0); cfma_conj(r, a0, b1); cfma(s, a1, b1); }
      else if (CORR) { cfma_conj(p, a0, b0); cfma_conj(p, a1, b1); cfma_conj(q, a0, b2); cfma_conj(q, a1, b3); }
      else { cfma(p, a0, b0); cfma(p, a1, b2); cfma_conj(q, b1, a0); cfma_conj(q, b3, a1); }   // conj(XL(f)) = XL(fm)
    };
    auto store = [&](int o, float2 p, float2 q) {
      p.x *= scale; p.y *= scale; q.x *= scale; q.y *= scale;
      if (PLANAR) {
        float* pl = reinterpret_cast<float*>(out + (int64_t)o * kNbA);
        pl[f] = p.x; pl[kNbA + f] = p.y;
        if (fm != f) { pl[fm] = q.x; pl[kNbA + fm] = q.y; }
      } else {
        out[(int64_t)o * kNbA + f] = p;
        if (fm != f) out[(int64_t)o * kNbA + fm] = q;
      }
    };
    auto finish = [&](int o, float2 p, float2 q, float2 r, float2 s) {
      if (TS == 2) { store(o, p, q); store(nout + o, r, s); }
      else if (CORR) emit(o, p, q);
      else store(o, p, q);
    };
    if constexpr (MAXB > 0) {
      float2 a0[MAXB], a1[MAXB], b0[MAXB], b1[MAXB], b2[MAXB], b3[MAXB];
#pragma unroll
      for (int i = 0; i < MAXB; ++i) {
        a0[i] = a1[i] = b0[i] = b1[i] = b2[i] = b3[i] = make_float2(0.f, 0.f);   // operands beyond na / nbm are zero
        if (i < na) load_a(i, a0[i], a1[i]);
        if (i < nbm) load_b(i, b0[i], b1[i], b2[i], b3[i]);
      }
#pragma unroll
      for (int o = 0; o < MAXB; ++o) {
        if (o < nout) {
          float2 p = make_float2(0.f, 0.f), q = p, r = p, s = p;
#pragma unroll
          for (int j = 0; j < MAXB; ++j) {
            const int ia = CORR ? o + j : o - j;                     // compile-time after unrolling
            if (ia >= 0 && ia < MAXB) term(a0[ia], a1[ia], b0[j], b1[j], b2[j], b3[j], p, q, r, s);
          }
          finish(o, p, q, r, s);
        }
      }
    } else {
      for (int o = 0; o < nout; ++o) {
        float2 p = make_float2(0.f, 0.f), q = p, r = p, s = p;
        for (int j = 0; j < nbm; ++j) {
          const int ia = CORR ? o + j : o - j;
          if (ia < 0 || ia >= na) continue;
          float2 a0, a1, b0, b1, b2, b3;
          load_a(ia, a0, a1);
          load_b(j, b0, b1, b2, b3);
          term(a0, a1, b0, b1, b2, b3, p, q, r, s);
        }
        finish(o, p, q, r, s);
      }
    }
  } else if constexpr (MAXB > 0) {
    float2 al[MAXB], ar[MAXB], bl[MAXB], br[MAXB];
#pragma unroll
    for (int i = 0; i < MAXB; ++i) {
      al[i] = ar[i] = bl[i] = br[i] = make_float2(0.f, 0.f);      // operands beyond na / nbm are zero
      if (i < na) untangle(a[(int64_t)i * kNbA + f], a[(int64_t)i * kNbA + fm], al[i], ar[i]);
      if (i < nbm) untangle(bq[(int64_t)i * kNbA + f], bq[(int64_t)i * kNbA + fm], bl[i], br[i]);
    }
#pragma unroll
    for (int o = 0; o < MAXB; ++o) {
      if (o < nout) {
        float2 sl = make_float2(0.f, 0.f), sr = make_float2(0.f, 0.f);
#pragma unroll
        for (int j = 0; j < MAXB; ++j) {
          const int ia = CORR ? o + j : o - j;                       // compile-time after unrolling
          if (ia >= 0 && ia < MAXB) {
            if (CORR) { cfma_conj(sl, al[ia], bl[j]); cfma_conj(sr, ar[ia], br[j]); }
            else      { cfma(sl, al[ia], bl[j]); cfma(sr, ar[ia], br[j]); }
          }
        }
        emit(o, sl, sr);
      }
    }
  } else {
    for (int o = 0; o < nout; ++o) {
      float2 sl = make_float2(0.f, 0.f), sr = make_float2(0.f, 0.f);
      for (int j = 0; j < nbm; ++j) {
        const int ia = CORR ? o + j : o - j;
        if (ia < 0 || ia >= na) continue;
        float2 pl, pr, ql, qr;
        untangle(a[(int64_t)ia * kNbA + f], a[(int64_t)ia * kNbA + fm], pl, pr);
        untangle(bq[(int64_t)j * kNbA + f], bq[(int64_t)j * kNbA + fm], ql, qr);
        if (CORR) { cfma_conj(sl, pl, ql); cfma_conj(sr, pr, qr); }
        else      { cfma(sl, pl, ql); cfma(sr, pr, qr); }
      }
      emit(o, sl, sr);
    }
  }
}

// Both correlation products of the backward in ONE pass over the gradient spectra (each was HBM bound on its own):
//   D[q] = sum_{j<J, q+j<I} G[q+j] conj(H[j])  (q < I)   dL/dx windows
//   E[j] = sum_{p<I, j+p<I} G[j+p] conj(X[p])  (j < J)   dL/dIR partitions
// G is read and untangled once; H and X take turns in the same registers.  Planar outputs (own inverse FFT kernels).
// H's item stride is hstride (J kNbA, or 0 for IR spectra shared by the batch).
// TS: a true-stereo IR (two partition sets, see partition_mac_kernel; hstride 2 J kNbA or 0): the products of
// partition_mac_kernel<TS 1, CORR> into D and of <TS 2> into the 2 J partitions per item of E, the latter from G
// repacked out of its untangled halves.
template <int MAXB, bool TS = false>
__global__ void __launch_bounds__(128) partition_mac_bwd_kernel(const float2* __restrict__ G, const float2* __restrict__ H,
                                                                int64_t hstride, const float2* __restrict__ X,
                                                                float2* __restrict__ D, float2* __restrict__ E, int I,
                                                                int J, float scale) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f > kNbA / 2) return;
  const int fm = (kNbA - f) & (kNbA - 1);
  const int64_t il = blockIdx.y;
  const float2* g = G + il * (int64_t)I * kNbA;
  float2 al[MAXB], ar[MAXB], bl[MAXB], br[MAXB];
#pragma unroll
  for (int i = 0; i < MAXB; ++i) {
    al[i] = ar[i] = make_float2(0.f, 0.f);
    if (i < I) untangle(g[(int64_t)i * kNbA + f], g[(int64_t)i * kNbA + fm], al[i], ar[i]);
  }
  if constexpr (TS) {
    auto store = [&](float2* blk, float2 p, float2 q) {
      float* pl = reinterpret_cast<float*>(blk);
      pl[f] = p.x * scale; pl[kNbA + f] = p.y * scale;
      if (fm != f) { pl[fm] = q.x * scale; pl[kNbA + fm] = q.y * scale; }
    };
    float2 cl[MAXB], cr[MAXB];                     // bl, br, cl, cr: H_LL, H_LR, H_RL, H_RR, then XL, XR
    const float2* h = H + il * hstride;
#pragma unroll
    for (int j = 0; j < MAXB; ++j) {
      bl[j] = br[j] = cl[j] = cr[j] = make_float2(0.f, 0.f);
      if (j < J) {
        untangle(h[(int64_t)j * kNbA + f], h[(int64_t)j * kNbA + fm], bl[j], br[j]);
        untangle(h[(int64_t)(J + j) * kNbA + f], h[(int64_t)(J + j) * kNbA + fm], cl[j], cr[j]);
      }
    }
#pragma unroll
    for (int o = 0; o < MAXB; ++o) {
      if (o < I) {
        float2 dl = make_float2(0.f, 0.f), dr = dl;
#pragma unroll
        for (int j = 0; j < MAXB; ++j) {
          if (o + j < MAXB) {
            cfma_conj(dl, al[o + j], bl[j]); cfma_conj(dl, ar[o + j], br[j]);
            cfma_conj(dr, al[o + j], cl[j]); cfma_conj(dr, ar[o + j], cr[j]);
          }
        }
        store(D + (il * I + o) * (int64_t)kNbA, make_float2(dl.x - dr.y, dl.y + dr.x), make_float2(dl.x + dr.y, dr.x - dl.y));
      }
    }
    const float2* xq = X + il * (int64_t)I * kNbA;
#pragma unroll
    for (int i = 0; i < MAXB; ++i) {
      bl[i] = br[i] = make_float2(0.f, 0.f);
      if (i < I) untangle(xq[(int64_t)i * kNbA + f], xq[(int64_t)i * kNbA + fm], bl[i], br[i]);
      cl[i] = make_float2(al[i].x - ar[i].y, al[i].y + ar[i].x);          // G at f and fm, repacked
      cr[i] = make_float2(al[i].x + ar[i].y, ar[i].x - al[i].y);
    }
#pragma unroll
    for (int o = 0; o < MAXB; ++o) {
      if (o < J) {
        float2 pa = make_float2(0.f, 0.f), qa = pa, pb = pa, qb = pa;
#pragma unroll
        for (int p = 0; p < MAXB; ++p) {
          if (o + p < MAXB) {
            cfma_conj(pa, cl[o + p], bl[p]); cfma(qa, cr[o + p], bl[p]);
            cfma_conj(pb, cl[o + p], br[p]); cfma(qb, cr[o + p], br[p]);
          }
        }
        store(E + (il * 2 * J + o) * (int64_t)kNbA, pa, qa);
        store(E + (il * 2 * J + J + o) * (int64_t)kNbA, pb, qb);
      }
    }
  } else {
#pragma unroll
    for (int pass = 0; pass < 2; ++pass) {
      const float2* bq = (pass == 0 ? H + il * hstride : X + il * (int64_t)I * kNbA);
      const int nbm = pass == 0 ? J : I, nout = pass == 0 ? I : J;
      float2* out = (pass == 0 ? D + il * (int64_t)I * kNbA : E + il * (int64_t)J * kNbA);
#pragma unroll
      for (int i = 0; i < MAXB; ++i) {
        bl[i] = br[i] = make_float2(0.f, 0.f);
        if (i < nbm) untangle(bq[(int64_t)i * kNbA + f], bq[(int64_t)i * kNbA + fm], bl[i], br[i]);
      }
#pragma unroll
      for (int o = 0; o < MAXB; ++o) {
        if (o < nout) {
          float2 sl = make_float2(0.f, 0.f), sr = make_float2(0.f, 0.f);
#pragma unroll
          for (int j = 0; j < MAXB; ++j) {
            if (o + j < MAXB) { cfma_conj(sl, al[o + j], bl[j]); cfma_conj(sr, ar[o + j], br[j]); }   // operands beyond I / nbm are zero
          }
          sl.x *= scale; sl.y *= scale; sr.x *= scale; sr.y *= scale;
          float* pl = reinterpret_cast<float*>(out + (int64_t)o * kNbA);
          pl[f] = sl.x - sr.y; pl[kNbA + f] = sl.y + sr.x;
          if (fm != f) { pl[fm] = sl.x + sr.y; pl[kNbA + fm] = sr.x - sl.y; }
        }
      }
    }
  }
}

// y = (1-mix) x + mix wet; wet[n] = Yt[(il*I + n/kB)*kNbA + kB + n%kB]
__global__ void mix_blocks_kernel(const float* __restrict__ x, const float2* __restrict__ Yt,
                                  const float* __restrict__ mix_p, int mix_stride, float* __restrict__ y, int64_t item0,
                                  int I, int64_t n, int in_chs) {
  const int i = blockIdx.x;
  const int64_t il = blockIdx.y, b = item0 + il;
  const float mix = mix_p[b * mix_stride];
  const float* xl = x + (b * in_chs) * n;
  const float* xr = in_chs == 1 ? xl : xl + n;
  const float2* yt = Yt + (il * I + i) * (int64_t)kNbA + kB;
  for (int m = threadIdx.x; m < kB; m += blockDim.x) {
    const int64_t t = (int64_t)i * kB + m;
    if (t >= n) break;
    const float2 w = yt[m];
    const float a0 = xl[t], a1 = xr[t];
    y[(b * 2 + 0) * n + t] = fmaf(mix, w.x - a0, a0);
    y[(b * 2 + 1) * n + t] = fmaf(mix, w.y - a1, a1);
  }
}

// backward: Gb[(il*I + i)*kNbA + kB + m] = (g_left, g_right)[i kB + m] (not scaled by mix), first half zero
__global__ void g_blocks_kernel(const float* __restrict__ gy, float2* __restrict__ Gb, int64_t item0, int I, int64_t n) {
  const int i = blockIdx.x;
  const int64_t il = blockIdx.y, b = item0 + il;
  const float* gl = gy + (b * 2 + 0) * n;
  const float* gr = gy + (b * 2 + 1) * n;
  float2* out = Gb + (il * I + i) * (int64_t)kNbA;
  for (int m = threadIdx.x; m < kB; m += blockDim.x) {
    const int64_t t = (int64_t)i * kB + m;
    out[m] = make_float2(0.f, 0.f);
    out[kB + m] = t < n ? make_float2(gl[t], gr[t]) : make_float2(0.f, 0.f);
  }
}

// gx[t] = (1-mix) g[t] + mix c[t],  c[t] = Dt[q][t - (q-1) kB] + Dt[q+1][t - q kB], q = t / kB (every sample sits in
// two windows); mono input receives the sum of both channel gradients.
// mix_part[il*I + i] = sum over block i and both channels of x (c - g)  (see g_fft_kernel)
__global__ void finish_dx_blocks_kernel(const float* __restrict__ gy, const float* __restrict__ x,
                                        const float2* __restrict__ Dt, const float* __restrict__ mix_p, int mix_stride,
                                        float* __restrict__ gx, float* __restrict__ mix_part, int64_t item0, int I,
                                        int64_t n, int in_chs) {
  const int i = blockIdx.x;
  const int64_t il = blockIdx.y, b = item0 + il;
  const float mix = mix_p[b * mix_stride];
  const float* xl = x + (b * in_chs) * n;
  const float* xr = in_chs == 1 ? xl : xl + n;
  const float2* d0 = Dt + (il * I + i) * (int64_t)kNbA + kB;
  const float2* d1 = (i + 1 < I) ? Dt + (il * I + i + 1) * (int64_t)kNbA : nullptr;
  float acc = 0.f;
  for (int m = threadIdx.x; m < kB; m += blockDim.x) {
    const int64_t t = (int64_t)i * kB + m;
    if (t >= n) break;
    float2 v = d0[m];
    if (d1) { const float2 u = d1[m]; v.x += u.x; v.y += u.y; }
    const float g0 = gy[(b * 2 + 0) * n + t], g1 = gy[(b * 2 + 1) * n + t];
    const float o0 = fmaf(1.0f - mix, g0, mix * v.x), o1 = fmaf(1.0f - mix, g1, mix * v.y);
    acc = fmaf(xl[t], v.x - g0, fmaf(xr[t], v.y - g1, acc));
    if (in_chs == 1) gx[b * n + t] = o0 + o1;
    else { gx[(b * 2 + 0) * n + t] = o0; gx[(b * 2 + 1) * n + t] = o1; }
  }
  __shared__ float wp[32];
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) wp[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float sum = 0.f;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) sum += wp[w];
    mix_part[il * I + i] = sum;
  }
}

// per (item, block): S0[k] = sum_t (dIR_l f_l + dIR_r f_r) env_k ;  S1[k] = sum_t (...) env_k tt
// part[((item*nbk + b)*12 + k)*2 + {0,1}]
__global__ void ir_grad_pairs_kernel(const float2* __restrict__ Et, const float2* __restrict__ C,
                                     const float* __restrict__ params, float* __restrict__ part, int64_t L,
                                     int64_t leff, int jb, int nbk, int nb, int hop, int P) {
  const int b = blockIdx.x;
  const int64_t il = blockIdx.y;
  __shared__ float rk[kBands];
  __shared__ float red[8][2 * kBands];
  if (threadIdx.x < kBands) rk[threadIdx.x] = band_rate(params, il, threadIdx.x);
  __syncthreads();
  const float step = 1.0f / (float)(L - 1);
  float s0[kBands], s1[kBands];
#pragma unroll
  for (int k = 0; k < kBands; ++k) { s0[k] = 0.f; s1[k] = 0.f; }
  for (int m = threadIdx.x; m < hop; m += blockDim.x) {
    const int64_t t = (int64_t)b * hop + m;
    if (t >= leff) break;
    const float tt = time_axis(t, L, step);
    const float2 gd = Et[ir_slot(il, jb, t)];
    const float gl = gd.x, gr = gd.y;
    const float2* c = C + ((il * kBands) * nbk + b) * (int64_t)nb + m + P;
#pragma unroll
    for (int k = 0; k < kBands; ++k) {
      const float2 v = c[(int64_t)k * nbk * nb];
      const float w = fmaf(gl, v.x, gr * v.y) * expf(rk[k] * tt);
      s0[k] += w;
      s1[k] = fmaf(w, tt, s1[k]);
    }
  }
  block_band_sums(s0, s1, red, (int)(blockDim.x >> 5), threadIdx.x, part + ((il * nbk + b) * kBands) * 2);
}

// one thread per (item, param): gains (0..11), decays (12..23), mix (24).  The dL/dIR partials come from gradient
// spectra that are not scaled by mix (see g_fft_kernel), so the band sums take the factor here.
__global__ void reverb_param_grad_kernel(const float* __restrict__ ir_part, const float* __restrict__ mix_part,
                                         const float* __restrict__ params, float* __restrict__ gparams, int64_t item0,
                                         int64_t items, int nbk, int mix_blocks) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= items * 25) return;
  const int64_t bl = idx / 25;
  const int q = (int)(idx - bl * 25);
  const float* pp = params + (item0 + bl) * 25;
  double s = 0.0;
  if (q < 24) {
    const int k = q % kBands;
    const float* pr = ir_part + (bl * nbk * kBands + k) * 2 + (q < kBands ? 0 : 1);
    for (int i = 0; i < nbk; ++i) s += (double)pr[(int64_t)i * kBands * 2];
    s *= (double)pp[24];
    if (q < kBands) s *= (1.0 / kBands);
    else s *= (double)pp[k] * (-10.0 / kBands);
  } else {
    for (int i = 0; i < mix_blocks; ++i) s += (double)mix_part[bl * mix_blocks + i];
  }
  gparams[(item0 + bl) * 25 + q] = (float)s;
}

// ---- convolution_reverberation: the audio convolution above with an impulse response supplied by the caller ----------
// Forward: ir_pack_kernel puts the caller's taps where the IR synthesis puts its own; x_fft_kernel, partition_mac_kernel
// and ifft_mix_kernel (or the cuFFT pipeline) then run unchanged.  Backward: g_fft_kernel, the correlations and
// ifft_dx_kernel as in the reverb; dL/dIR partition j = mix * first half of IFFT(sum_p G[j+p] conj(X[p])), unpacked into
// the caller's rows by ifft_irtaps_kernel (or irtaps_unpack_kernel after the cuFFT inverse).

// taps t < leff of the planar (bs, ir_chs, L) rows -> (left, right) pairs in the first half of partition slot t / kB
// (a mono IR feeds both channels).  A true-stereo IR (ir_chs 4, rows L->L, L->R, R->L, R->R) fills two partition sets
// per item: set s = gridDim.z index packs rows 2s and 2s + 1 into the slots of (il * 2 + s).
// grid = (ceil(leff / 256), items, 1 or 2 sets)
__global__ void ir_pack_kernel(const float* __restrict__ ir, float2* __restrict__ Hb, int64_t item0, int J, int64_t L,
                               int64_t leff, int ir_chs) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t il = blockIdx.y;
  const int s = blockIdx.z;
  if (t >= leff) return;
  const float* rl = ir + ((item0 + il) * ir_chs + 2 * s) * L;
  const float* rr = ir_chs == 1 ? rl : rl + L;
  Hb[ir_slot(il * gridDim.z + s, J, t)] = make_float2(rl[t], rr[t]);
}

// unit m = (il*sets + s)*J + j: dL/dIR taps [j kB, (j+1) kB) ∩ [0, leff) = mix * first half of IFFT(Epl[m]) (left,
// right), written straight into rows 2s, 2s + 1 of the caller's (bs, ir_chs, L) rows; a mono IR receives the sum of both
// channels.  sets = 2 only for a true-stereo IR.  A null mix is a factor of 1 (a shared IR's summed partitions carry
// their factors already).
__global__ void __launch_bounds__(kFusedThreads, 1)
ifft_irtaps_kernel(const float* __restrict__ Epl, const float* __restrict__ twiddles, const float* __restrict__ mix,
                   float* __restrict__ gir, int64_t item0, int J, int sets, int64_t L, int64_t leff, int ir_chs,
                   int nunits) {
  extern __shared__ __align__(128) float sm[];
  FftSmem s(sm);
  const int t = threadIdx.x;
  s.init(twiddles, t);
  const fft8k::Tables tb = fft8k::carve_tables(s.tabf);
  auto fetch = [&](int it, int m) {
    if (t == 0 && m < nunits) s.load_planar(it, Epl + (int64_t)m * 2 * kNbA);
  };
  fetch(0, blockIdx.x);
  fetch(1, blockIdx.x + gridDim.x);
  int it = 0;
  for (int m = blockIdx.x; m < nunits; m += gridDim.x, ++it) {
    s.wait(it);
    float* gr = s.buf(it);
    const int q = m / J;                           // partition set il * sets + set
    const int64_t il = q / sets, b = item0 + il;
    const int j = m - q * J, set = q - (int)il * sets;
    float xr[16], xi[16];
    fft8192_in_smem<true>(gr, gr + fft8k::kPlaneG, s, tb, t, [&] { fetch(it + 2, m + 2 * gridDim.x); }, [] {}, xr, xi);
    const float mx = mix ? mix[b] : 1.0f;
    float* row = gir + (b * ir_chs + 2 * set) * L;
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const int64_t tau = (int64_t)j * kB + t + 512 * q;
      if (tau < leff) {
        if (ir_chs == 1) row[tau] = mx * (xr[q] + xi[q]);
        else { row[tau] = mx * xr[q]; row[L + tau] = mx * xi[q]; }
      }
    }
  }
}

// dL/dIR taps [t0, L) of the caller's rows: mix * Et (inverse-transformed partitions, pairs in the first half of each
// slot) below leff, 0 from leff on (those taps cannot reach an output).  t0 = leff writes only the zeros.  A null mix is
// a factor of 1.  Partition set s (gridDim.z = 2 for a true-stereo IR) goes to rows 2s, 2s + 1.
// grid = (ceil((L - t0) / 256), items, 1 or 2 sets)
__global__ void irtaps_unpack_kernel(const float2* __restrict__ Et, const float* __restrict__ mix, float* __restrict__ gir,
                                     int64_t item0, int J, int64_t L, int64_t leff, int ir_chs, int64_t t0) {
  const int64_t t = t0 + (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t il = blockIdx.y, b = item0 + il;
  const int s = blockIdx.z;
  if (t >= L) return;
  float2 v = make_float2(0.f, 0.f);
  float mx = 0.f;
  if (t < leff) {
    v = Et[ir_slot(il * gridDim.z + s, J, t)];
    mx = mix ? mix[b] : 1.f;
  }
  float* row = gir + (b * ir_chs + 2 * s) * L;
  if (ir_chs == 1) row[t] = mx * (v.x + v.y);
  else { row[t] = mx * v.x; row[L + t] = mx * v.y; }
}

// dL/dIR of one impulse response shared by the batch: the sum over items b of mix[b] E_b, taken on the partition spectra
// E_b of the es region before any inverse transform (the inverse is linear).  Element by element in fp64 and in absolute
// item order: a product of two floats is exact in fp64, so every element goes through the same sequence of additions
// however the batch is cut into chunks, and the result is the same bits for every chunk size.  Item 0 writes acc instead
// of adding to it (the workspace is never cleared); the chunk that holds the last item writes the sum, rounded to fp32,
// over item 0's slot of Et instead, for the inverse transforms (thread e alone reads and writes element e of every slot).
// Element-wise, so it serves the planar (own FFT) and the interleaved (cuFFT) spectra alike.
// grid = ceil(sets J kNbA / 256), one complex element of the sets * J partitions per thread
__global__ void irgrad_sum_kernel(float2* Et, const float* __restrict__ mix, double2* __restrict__ acc, int64_t item0,
                                  int items, int64_t per_item, bool last) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= per_item) return;
  double2 a = make_double2(0.0, 0.0);
  int il = 0;
  if (item0 != 0) {
    a = acc[e];
  } else {                                         // item 0: written, not added
    const float2 v = Et[e];
    const double m = (double)mix[0];
    a = make_double2(m * (double)v.x, m * (double)v.y);
    il = 1;
  }
  for (; il < items; ++il) {
    const float2 v = Et[il * per_item + e];
    const double m = (double)mix[item0 + il];
    a.x += m * (double)v.x;
    a.y += m * (double)v.y;
  }
  if (last) Et[e] = make_float2((float)a.x, (float)a.y);
  else acc[e] = a;
}

// dL/dmix per item: the per-block partials of ifft_dx_kernel / finish_dx_blocks_kernel summed in block order, in fp64
__global__ void conv_mix_grad_kernel(const float* __restrict__ mix_part, float* __restrict__ gmix, int64_t item0,
                                     int64_t items, int I) {
  const int64_t il = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (il >= items) return;
  double s = 0.0;
  for (int i = 0; i < I; ++i) s += (double)mix_part[il * I + i];
  gmix[item0 + il] = (float)s;
}

// device-resident band spectra H_k: 12 x nb complex (full spectrum of the real taps), scaled by 1/nb;
// built once per (device, taps, sr, nb)
int get_filterbank(const Geom& g, double sr, cudaStream_t st, const float2** out) {
  int dev = 0;
  DASP_CUDA_OK(cudaGetDevice(&dev));
  const bool flat = debug_flat_filterbank();        // test hook: H_k = 1 -> the blocks keep the white noise itself
  FbKey key{dev, flat ? -g.taps : g.taps, g.nb, sr};
  auto it = g_fb.find(key);
  if (it != g_fb.end()) { *out = reinterpret_cast<const float2*>(it->second); return DASP_OK; }
  DASP_REQUIRE(sr / 2.0 > 18000.0, "sample_rate %.1f too low: the filter bank needs 18 kHz < sr/2 (signal.py:84)", sr);
  std::vector<float> taps;
  octave_filterbank((int)g.taps, sr, taps);
  if (flat) {
    taps.assign(taps.size(), 0.f);
    for (int k = 0; k < kBands; ++k) taps[(size_t)k * g.taps] = 1.0f;      // unit impulse at lag 0
  }
  std::vector<float2> padded((size_t)kBands * g.nb, make_float2(0.f, 0.f));
  const float inv = 1.0f / (float)g.nb;
  for (int k = 0; k < kBands; ++k)
    for (int64_t i = 0; i < g.taps; ++i) padded[(size_t)k * g.nb + i].x = taps[(size_t)k * g.taps + i] * inv;
  cufftComplex* d_buf = nullptr;
  void* d_work = nullptr;
  DASP_CUDA_OK(cudaMalloc(&d_buf, sizeof(cufftComplex) * padded.size()));
  DASP_CUDA_OK(cudaMemcpyAsync(d_buf, padded.data(), sizeof(float2) * padded.size(), cudaMemcpyHostToDevice, st));
  PlanVal pv;
  int rc = get_plan(2, g.nb, kBands, g.nb, g.nb, pv);
  if (rc != DASP_OK) return rc;
  DASP_CUDA_OK(cudaMalloc(&d_work, pv.work > 0 ? pv.work : 16));
  if ((rc = exec_c2c(pv, d_work, d_buf, CUFFT_FORWARD, st)) != DASP_OK) return rc;
  DASP_CUDA_OK(cudaStreamSynchronize(st));   // one-off (cache fill): host vector and temp buffers die here
  cudaFree(d_work);
  g_fb[key] = d_buf;
  *out = reinterpret_cast<const float2*>(d_buf);
  return DASP_OK;
}

// half spectrum of the taps on the n1-point grid of the spectral synthesis: 12 x (n1/2+1) complex, scaled sqrt(n1/2)/n1
int get_filterbank_n1(const Geom& g, double sr, cudaStream_t st, const float2** out) {
  int dev = 0;
  DASP_CUDA_OK(cudaGetDevice(&dev));
  const int64_t n1 = g.n1(), n1c = g.n1c();
  const bool flat = debug_flat_filterbank();        // test hook: H_k = 1 -> f_k is the white periodic sequence itself
  FbKey key{dev, flat ? -g.taps : g.taps, -n1, sr};
  auto it = g_fb.find(key);
  if (it != g_fb.end()) { *out = reinterpret_cast<const float2*>(it->second); return DASP_OK; }
  DASP_REQUIRE(sr / 2.0 > 18000.0, "sample_rate %.1f too low: the filter bank needs 18 kHz < sr/2 (signal.py:84)", sr);
  {
    float2 roots[17][16];
    for (int r = 0; r <= 16; ++r)
      for (int m = 0; m < 16; ++m) {
        const double a = (r > 0) ? 2.0 * kPi * (double)(m % r) / (double)r : 0.0;
        roots[r][m] = make_float2((float)cos(a), (float)sin(a));
      }
    DASP_CUDA_OK(cudaMemcpyToSymbolAsync(c_root, roots, sizeof(roots), 0, cudaMemcpyHostToDevice, st));
    DASP_CUDA_OK(cudaStreamSynchronize(st));
  }
  std::vector<float> taps;
  octave_filterbank((int)g.taps, sr, taps);
  if (flat) {
    taps.assign(taps.size(), 0.f);
    for (int k = 0; k < kBands; ++k) taps[(size_t)k * g.taps] = 1.0f;      // unit impulse at lag 0
  }
  std::vector<float> padded((size_t)kBands * n1, 0.f);
  // 1/n1 of the inverse transform and the sqrt(n1/2) of the bins' complex Gaussians (Z ~ CN(0, n1)) are folded in
  const float inv = (float)(sqrt(0.5 * (double)n1) / (double)n1);
  for (int k = 0; k < kBands; ++k)
    for (int64_t i = 0; i < g.taps; ++i) padded[(size_t)k * n1 + i] = taps[(size_t)k * g.taps + i] * inv;
  float* d_in = nullptr;
  cufftComplex* d_out = nullptr;
  void* d_work = nullptr;
  DASP_CUDA_OK(cudaMalloc(&d_in, sizeof(float) * padded.size()));
  DASP_CUDA_OK(cudaMalloc(&d_out, sizeof(cufftComplex) * kBands * n1c));
  DASP_CUDA_OK(cudaMemcpyAsync(d_in, padded.data(), sizeof(float) * padded.size(), cudaMemcpyHostToDevice, st));
  PlanVal pv;
  int rc = get_plan(0, n1, kBands, n1, n1c, pv);
  if (rc != DASP_OK) return rc;
  DASP_CUDA_OK(cudaMalloc(&d_work, pv.work > 0 ? pv.work : 16));
  DASP_CUFFT_OK(cufftSetStream(pv.h, st));
  DASP_CUFFT_OK(cufftSetWorkArea(pv.h, d_work));
  DASP_CUFFT_OK(cufftExecR2C(pv.h, d_in, d_out));
  DASP_CUDA_OK(cudaStreamSynchronize(st));   // one-off cache fill
  cudaFree(d_in);
  cudaFree(d_work);
  g_fb[key] = d_out;
  *out = reinterpret_cast<const float2*>(d_out);
  return DASP_OK;
}

// Appends a launch priority to cfg (at: its attribute array, with room for one more).  The launch then carries the
// priority itself, so a captured graph keeps it per kernel node whatever the priority of the stream it is replayed on.
// prio == nullptr: the stream's priority.
void add_priority(cudaLaunchConfig_t& cfg, cudaLaunchAttribute* at, const int* prio) {
  if (!prio) return;
  at[cfg.numAttrs].id = cudaLaunchAttributePriority;
  at[cfg.numAttrs].val.priority = *prio;
  cfg.attrs = at;
  ++cfg.numAttrs;
}

template <int R>
void launch_spectral(float2* C, const float2* H1, int64_t item0, int64_t items, int nb, const unsigned long long* seed,
                     bool planar, cudaStream_t st, const int* prio) {
  const int threads = 128;
  cudaLaunchConfig_t cfg = {};
  cudaLaunchAttribute at[1];
  cfg.gridDim = dim3((unsigned)((nb / 2 + 1 + threads - 1) / threads), kBands, (unsigned)items);
  cfg.blockDim = dim3(threads, 1, 1);
  cfg.stream = st;
  add_priority(cfg, at, prio);
  if (planar) cudaLaunchKernelEx(&cfg, spectral_gen_kernel<R, true>, C, H1, item0, nb, seed);
  else        cudaLaunchKernelEx(&cfg, spectral_gen_kernel<R, false>, C, H1, item0, nb, seed);
}
bool dispatch_spectral(int R, float2* C, const float2* H1, int64_t item0, int64_t items, int nb,
                       const unsigned long long* seed, bool planar, cudaStream_t st, const int* prio) {
  switch (R) {
#define DASP_R(r) case r: launch_spectral<r>(C, H1, item0, items, nb, seed, planar, st, prio); return true;
    DASP_R(1) DASP_R(2) DASP_R(3) DASP_R(4) DASP_R(5) DASP_R(6) DASP_R(7) DASP_R(8) DASP_R(9) DASP_R(10)
    DASP_R(11) DASP_R(12) DASP_R(13) DASP_R(14) DASP_R(15) DASP_R(16)
#undef DASP_R
    default: return false;       // very long IRs fall back to the time-domain Philox + overlap-save path
  }
}
constexpr int kMaxSpectralR = 16;

// twiddle tables of fft8192.cuh (fp64 on the host, once per device)
std::map<int, float*> g_fft_tab;
int get_fft_tables(cudaStream_t st, const float** out) {
  int dev = 0;
  DASP_CUDA_OK(cudaGetDevice(&dev));
  auto it = g_fft_tab.find(dev);
  if (it == g_fft_tab.end()) {
    std::vector<float> h(fft8k::kTabFloats, 0.f);
    for (int e = 0; e < fft8k::kTabEntries; ++e) {
      int co, so, dup;
      double turns;
      fft8k::table_entry(e, co, so, dup, turns);
      const float c = (float)cos(2.0 * kPi * turns), sn = (float)sin(2.0 * kPi * turns);
      h[co] = c; h[so] = sn;
      if (dup) { h[co + 1] = c; h[so + 1] = sn; }
    }
    float* d = nullptr;
    DASP_CUDA_OK(cudaMalloc(&d, sizeof(float) * h.size()));
    DASP_CUDA_OK(cudaMemcpyAsync(d, h.data(), sizeof(float) * h.size(), cudaMemcpyHostToDevice, st));
    DASP_CUDA_OK(cudaStreamSynchronize(st));   // one-off cache fill (h goes out of scope)
    it = g_fft_tab.emplace(dev, d).first;
  }
  *out = it->second;
  return DASP_OK;
}
// Side streams of the forward's IR synthesis (see dasp_reverb_fwd), created once per device at the greatest stream
// priority.  fork is recorded on the caller's stream before the first synthesis, done[k % 2] after chunk k's synthesis
// on side[k % 2].  Reusing the events across chunks and calls is safe: cudaStreamWaitEvent takes the state of the
// event at the time of the call, and a later record does not change what an earlier wait waits for.
struct SideStreams { cudaStream_t side[2]; cudaEvent_t fork, done[2]; int prio; };
std::map<int, SideStreams> g_side;                  // guarded by g_mu
int get_side_streams(SideStreams** out) {
  int dev = 0;
  DASP_CUDA_OK(cudaGetDevice(&dev));
  auto it = g_side.find(dev);
  if (it == g_side.end()) {
    SideStreams s{};
    int least = 0;
    DASP_CUDA_OK(cudaDeviceGetStreamPriorityRange(&least, &s.prio));
    for (int i = 0; i < 2; ++i) {
      DASP_CUDA_OK(cudaStreamCreateWithPriority(&s.side[i], cudaStreamNonBlocking, s.prio));
      DASP_CUDA_OK(cudaEventCreateWithFlags(&s.done[i], cudaEventDisableTiming));
    }
    DASP_CUDA_OK(cudaEventCreateWithFlags(&s.fork, cudaEventDisableTiming));
    it = g_side.emplace(dev, s).first;
  }
  *out = &it->second;
  return DASP_OK;
}

int configure_fft_kernels();
int launch_ifft_shape(float2* C, const float* tw, const float* params, float2* hs, bool save_f, int64_t items,
                      const Geom& g, int jb, cudaStream_t st, const int* prio) {
  int rc = configure_fft_kernels();
  if (rc != DASP_OK) return rc;
  cudaLaunchConfig_t cfg = {};
  cudaLaunchAttribute at[1];
  cfg.gridDim = dim3((unsigned)g.rpp, (unsigned)items, 1);
  cfg.blockDim = dim3(kFusedThreads, 1, 1);
  cfg.dynamicSmemBytes = kFftSmemBytes;
  cfg.stream = st;
  add_priority(cfg, at, prio);
  cudaLaunchKernelEx(&cfg, ifft_shape_kernel, reinterpret_cast<float*>(C), tw, params, hs, save_f ? 1 : 0, (int)g.L,
                     (int)g.leff, jb, (int)g.rpp);
  DASP_LAUNCH_OK("ifft_shape_kernel");
  return DASP_OK;
}
int g_last_fused = 0;                                // test hook: IR-synthesis path of the last forward chunk
std::map<std::pair<int, int>, int> g_fused_ok;      // (device, R) -> clusters that fit, guarded by g_mu
// cluster synthesis: persistent clusters of R CTAs, as many as the device co-schedules (at most one per item).
// Returns false when the device cannot co-schedule such a cluster (then generator -> ifft_shape_kernel runs), true after
// a launch attempt (check cudaGetLastError).
template <int R>
bool launch_fused(const float2* H1, const float* tw, const float* params, float2* hs, float2* Csave, int64_t item0, int64_t items,
                  int64_t L, int64_t leff, int jb, const unsigned long long* seed, cudaStream_t st, const int* prio) {
  auto kern = ir_synth_cluster_kernel<R>;
  cudaLaunchConfig_t cfg = {};
  cfg.blockDim = dim3(kSynthThreads, 1, 1);
  cfg.dynamicSmemBytes = kSynthSmemBytes;
  cfg.stream = st;
  cudaLaunchAttribute at[2];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = R; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
  cfg.attrs = at;
  cfg.numAttrs = 1;
  int dev = 0;
  cudaGetDevice(&dev);
  auto it = g_fused_ok.find({dev, R});
  if (it == g_fused_ok.end()) {
    int n = 0;
    cfg.gridDim = dim3(R, 1, 1);
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSynthSmemBytes) != cudaSuccess ||
        cudaOccupancyMaxActiveClusters(&n, kern, &cfg) != cudaSuccess) {
      n = 0;
      cudaGetLastError();
    }
    it = g_fused_ok.emplace(std::make_pair(dev, R), n).first;
  }
  if (it->second < 1) return false;
  const int64_t clusters = items < it->second ? items : it->second;
  cfg.gridDim = dim3(R, (unsigned)clusters, 1);
  add_priority(cfg, at, prio);
  cudaLaunchKernelEx(&cfg, kern, H1, tw, params, hs, Csave, item0, (int)items, (int)L, (int)leff, jb, seed);
  return true;
}
bool dispatch_fused(int R, const float2* H1, const float* tw, const float* params, float2* hs, float2* Csave, int64_t item0,
                    int64_t items, int64_t L, int64_t leff, int jb, const unsigned long long* seed, cudaStream_t st,
                    const int* prio) {
  switch (R) {
#define DASP_R(r) case r: return launch_fused<r>(H1, tw, params, hs, Csave, item0, items, L, leff, jb, seed, st, prio);
    DASP_R(1) DASP_R(2) DASP_R(3) DASP_R(4) DASP_R(5) DASP_R(6)
#undef DASP_R
    default: return false;
  }
}

inline size_t align256(size_t v) { return (v + 255) & ~(size_t)255; }

// workspace carve-up shared by the geometry queries and the entry points; extra: the reverb's own region (the filtered
// noise of a chunk when f_save is not kept / the per-partition partials of the 24 band-parameter gradients); acc: the
// fp64 sum of a shared IR's dL/dIR partition spectra (0 bytes unless g.shared)
struct FwdWs { size_t ys, xsp, hsp, extra, cufft, total; };
struct BwdWs { size_t gs, ds, es, extra, mixpart, acc, cufft, total; };

void fwd_layout(const ConvGeom& g, size_t extra_bytes, size_t cufft_work, FwdWs& w) {
  size_t o = 0;
  w.ys = o;  o += align256(sizeof(float2) * (size_t)(g.chunk * g.ib * kNbA));
  // transient homes for what a forward WITHOUT a backward does not keep (null *_save pointers)
  w.xsp = o; o += align256(sizeof(float2) * (size_t)(g.chunk * g.ib * kNbA));
  w.hsp = o; o += align256(sizeof(float2) * (size_t)((g.shared ? 1 : g.chunk) * g.sets * g.jb * kNbA));
  w.extra = o; o += align256(extra_bytes);
  w.cufft = o; o += align256(cufft_work);
  w.total = o;
}
void bwd_layout(const ConvGeom& g, size_t extra_bytes, size_t cufft_work, BwdWs& w) {
  size_t o = 0;
  w.gs = o; o += align256(sizeof(float2) * (size_t)(g.chunk * g.ib * kNbA));
  w.ds = o; o += align256(sizeof(float2) * (size_t)(g.chunk * g.ib * kNbA));
  w.es = o; o += align256(sizeof(float2) * (size_t)(g.chunk * g.sets * g.jb * kNbA));
  w.extra = o; o += align256(extra_bytes);
  w.mixpart = o; o += align256(sizeof(float) * (size_t)(g.chunk * g.ib));
  w.acc = o; o += align256(g.shared ? sizeof(double2) * (size_t)(g.sets * g.jb * kNbA) : 0);
  w.cufft = o; o += align256(cufft_work);
  w.total = o;
}

// cuFFT plans for a full chunk and for the remainder (none without a batch), and both workspace layouts around their
// largest work area.  xi / hj: the block transforms of the convolution's cuFFT pipeline (audio / dL/dx windows, IR /
// dL/dIR partitions).  With synth (the reverb) also blk / pp, its IR synthesis (overlap-save blocks, polyphase), and
// the extra regions.  With g.shared also ir1: the J partitions of the one IR (forward) and of its summed gradient.
// Every IR plan transforms g.sets partition sets of J partitions per IR.
struct Plans { PlanVal xi, hj, blk, pp; };
struct Setup { Plans full, rem; PlanVal ir1; FwdWs fwd; BwdWs bwd; };
int conv_setup(const ConvGeom& g, const Geom* synth, Setup& s) {
  int rc;
  size_t work = 0;
  if (g.shared && g.bs > 0) {
    if ((rc = get_plan(2, kNbA, g.sets * g.jb, kNbA, kNbA, s.ir1)) != DASP_OK) return rc;
    work = s.ir1.work;
  }
  for (int64_t items : {g.bs > 0 ? g.chunk : 0, g.bs % g.chunk}) {
    if (items == 0) continue;
    Plans& p = items == g.chunk ? s.full : s.rem;
    if ((rc = get_plan(2, kNbA, items * g.ib, kNbA, kNbA, p.xi)) != DASP_OK) return rc;
    if ((rc = get_plan(2, kNbA, items * g.sets * g.jb, kNbA, kNbA, p.hj)) != DASP_OK) return rc;
    if (p.xi.work > work) work = p.xi.work;
    if (p.hj.work > work) work = p.hj.work;
    if (synth) {
      if ((rc = get_plan(2, synth->nb, items * kBands * synth->nbk, synth->nb, synth->nb, p.blk)) != DASP_OK) return rc;
      if ((rc = get_plan(2, synth->nb, items * kBands * synth->rpp, synth->nb, synth->nb, p.pp)) != DASP_OK) return rc;
      if (p.blk.work > work) work = p.blk.work;
      if (p.pp.work > work) work = p.pp.work;
    }
  }
  size_t fwd_extra = 0, bwd_extra = 0;
  if (synth) {
    fwd_extra = sizeof(float2) * (size_t)(g.chunk * kBands * synth->pair_c64());
    int64_t nparts = synth->nbk > synth->nparts_pp() ? synth->nbk : synth->nparts_pp();
    if (g.jb > nparts) nparts = g.jb;
    bwd_extra = sizeof(float) * (size_t)(g.chunk * nparts * kBands * 2);
  }
  fwd_layout(g, fwd_extra, work, s.fwd);
  bwd_layout(g, bwd_extra, work, s.bwd);
  return DASP_OK;
}
int check_workspace(const char* what, size_t need, int64_t have) {
  if ((int64_t)need > have) {
    set_error("%s: workspace needs %lld bytes, got %lld", what, (long long)need, (long long)have);
    return DASP_ERR_WORKSPACE;
  }
  return DASP_OK;
}

// the fields dasp_reverb_geom and dasp_conv_geom share
template <class Out>
int put_conv_geometry(const ConvGeom& g, const Geom* synth, Out* out) {
  std::lock_guard<std::mutex> lk(g_mu);
  Setup s{};
  int rc = conv_setup(g, synth, s);
  if (rc != DASP_OK) return rc;
  out->leff = g.leff; out->conv_block = kB; out->x_blocks = g.ib; out->ir_partitions = g.jb; out->chunk_items = g.chunk;
  out->xspec_c64 = g.bs * g.ib * kNbA;
  out->irspec_c64 = (g.shared ? (g.bs > 0 ? 1 : 0) : g.bs) * g.sets * g.jb * kNbA;
  out->fwd_workspace_bytes = (int64_t)s.fwd.total;
  out->bwd_workspace_bytes = (int64_t)s.bwd.total;
  return DASP_OK;
}

// out = conv / corr of packed block spectra, register-cached when both operands have <= 16 blocks
template <bool CORR, bool PLANAR = false, int TS = 0>
void launch_mac(const float2* A, const float2* Bm, float2* Out, int na, int nbm, int bstep, int nout,
                int64_t items, float scale, cudaStream_t st) {
  dim3 grid((kNbA / 2 + 1 + 127) / 128, (unsigned)items);
  const int m = na > nbm ? na : nbm;
  if (m <= 12)      partition_mac_kernel<12, CORR, PLANAR, TS><<<grid, 128, 0, st>>>(A, Bm, Out, na, nbm, nout, scale, bstep);
  else if (m <= 16) partition_mac_kernel<16, CORR, PLANAR, TS><<<grid, 128, 0, st>>>(A, Bm, Out, na, nbm, nout, scale, bstep);
  else              partition_mac_kernel<0, CORR, PLANAR, TS><<<grid, 128, 0, st>>>(A, Bm, Out, na, nbm, nout, scale, bstep);
}

// grid of a persistent FFT kernel: one CTA per SM, at most one per unit of work
unsigned persistent_grid(int64_t units) { return (unsigned)(units < sm_count() ? units : sm_count()); }

// one-off opt-in to the large dynamic shared memory of the FFT kernels (per device, guarded by g_mu)
int configure_fft_kernels() {
  static std::map<int, bool> configured;
  int dev = 0;
  DASP_CUDA_OK(cudaGetDevice(&dev));
  if (!configured[dev]) {
    DASP_CUDA_OK(cudaFuncSetAttribute(ifft_shape_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFftSmemBytes));
    DASP_CUDA_OK(cudaFuncSetAttribute(x_fft_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFftSmemBytes));
    DASP_CUDA_OK(cudaFuncSetAttribute(ifft_mix_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFftSmemBytes));
    DASP_CUDA_OK(cudaFuncSetAttribute(g_fft_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFftSmemBytes));
    DASP_CUDA_OK(cudaFuncSetAttribute(ifft_dx_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFftSmemBytes));
    DASP_CUDA_OK(cudaFuncSetAttribute(ifft_irgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFftSmemBytes));
    DASP_CUDA_OK(cudaFuncSetAttribute(ifft_irtaps_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFftSmemBytes));
    configured[dev] = true;
  }
  return DASP_OK;
}

// ---- the audio convolution of one chunk, forward and backward, for both ops ----
// The own in-shared-memory FFT runs the block transforms (fused with their neighbours) when the rows allow bulk copies:
// n % 4 == 0 and 16-byte aligned rows (b may be null).  dasp_debug_reverb_path(1) pins the cuFFT pipeline (the tests
// compare the two).
bool own_fft_rows(int64_t n, const void* a, const void* b) {
  return debug_reverb_path() != 1 && (n % 4 == 0) && aligned16(a) && (b == nullptr || aligned16(b));
}

// what the backward leaves in the es region for the caller's dL/dIR consumer
enum class IrGrad {
  kNone,     // nothing (a fixed impulse response)
  kPlanar,   // partition spectra, planar, for an own-FFT inverse (own path only)
  kTime,     // partitions after the inverse cuFFT C2C: (left, right) pairs in the first half of each slot
  kSpectra,  // partition spectra as (re, im) pairs, summed over a shared IR's items before the inverse cuFFT
};
// both correlations in one pass over the gradient spectra when the operands fit the register cache (a true-stereo IR,
// sets == 2, caches twice the IR operands: kTsFusedMaxB)
constexpr int kTsFusedMaxB = 16;
bool fused_corr(IrGrad e, int I, int J, int sets) {
  return e == IrGrad::kPlanar && (I > J ? I : J) <= (sets == 2 ? kTsFusedMaxB : 16);
}

// The partitions of an impulse response shared by the batch, transformed in place in hs once before the first chunk,
// filled as conv_fwd_chunk expects them; own: x_fft_kernel with no audio windows, otherwise the J-batch cuFFT C2C.
int conv_shared_ir_spectra(const ConvGeom& g, const PlanVal& ir1, bool own, const float* tw, float2* hs,
                           unsigned char* ws, const FwdWs& w, cudaStream_t st) {
  const int J = (int)g.jb, nparts = g.sets * J;
  if (own) {
    int rc = configure_fft_kernels();
    if (rc != DASP_OK) return rc;
    x_fft_kernel<<<(unsigned)((nparts + kConvRun - 1) / kConvRun), kFusedThreads, kFftSmemBytes, st>>>(
        nullptr, nullptr, hs, tw, 0, (int)g.ib, J, g.n, g.leff, 1, 0, nparts);
    DASP_LAUNCH_OK("x_fft_kernel");
    return DASP_OK;
  }
  return exec_c2c(ir1, ws + w.cufft, hs, CUFFT_FORWARD, st);
}

// y = (1 - mix) x + mix (x * IR), mix of item b at mix[b * mix_stride].  The caller has written IR taps t < leff as
// (left, right) pairs into the first half of partition slot t / kB of hs, and on the cuFFT pipeline zero-filled the
// slots first.  xs / hs receive the window / partition spectra.  own (own_fft_rows of x and hs): x_fft_kernel transforms
// both on the own FFT with the tables tw; otherwise cuFFT C2C does.  h_stride: item stride of hs in complex elements,
// g.sets J kNbA; 0 for one IR shared by the batch, whose partitions conv_shared_ir_spectra has transformed already.
// g.sets == 2 (a true-stereo IR): hs holds set A then set B per IR, and the product is partition_mac_kernel<TS 1>.
int conv_fwd_chunk(const ConvGeom& g, const Plans& pl, bool own, const float* tw, const float* x, int in_chs, float2* xs,
                   float2* hs, int64_t h_stride, const float* mix, int mix_stride, float* y, unsigned char* ws,
                   const FwdWs& w, int64_t item0, int64_t items, cudaStream_t st) {
  float2* ys = (float2*)(ws + w.ys);
  const int I = (int)g.ib, J = (int)g.jb;
  const int nblk = (int)(items * I);
  if (own) {
    int rc = configure_fft_kernels();
    if (rc != DASP_OK) return rc;
    // one work list: the items*I audio windows, then the items*sets*J IR partitions (transformed in place in hs; the
    // zero padding of a partition depends on its index within its set, slot mod J)
    const int nunits = (int)(items * (I + (h_stride != 0 ? g.sets * J : 0)));
    x_fft_kernel<<<(unsigned)((nunits + kConvRun - 1) / kConvRun), kFusedThreads, kFftSmemBytes, st>>>(x, xs, hs, tw, item0, I, J, g.n, g.leff, in_chs, nblk,
                                                                nunits);
    DASP_LAUNCH_OK("x_fft_kernel");
    if (g.sets == 2) launch_mac<false, true, 1>(xs, hs, ys, I, J, h_stride != 0, I, items, 1.0f / (float)kNbA, st);
    else             launch_mac<false, true>(xs, hs, ys, I, J, h_stride != 0, I, items, 1.0f / (float)kNbA, st);
    DASP_LAUNCH_OK("partition_mac_kernel");
    ifft_mix_kernel<<<(unsigned)((nblk + kConvRun - 1) / kConvRun), kFusedThreads, kFftSmemBytes, st>>>(reinterpret_cast<const float*>(ys), tw, x, mix,
                                                                   mix_stride, y, item0, I, g.n, in_chs, nblk);
    DASP_LAUNCH_OK("ifft_mix_kernel");
    return DASP_OK;
  }
  void* cufft = ws + w.cufft;
  int rc;
  if (h_stride != 0 && (rc = exec_c2c(pl.hj, cufft, hs, CUFFT_FORWARD, st)) != DASP_OK) return rc;
  x_blocks_kernel<<<dim3((unsigned)I, (unsigned)items), 256, 0, st>>>(x, xs, item0, I, g.n, in_chs);
  DASP_LAUNCH_OK("x_blocks_kernel");
  if ((rc = exec_c2c(pl.xi, cufft, xs, CUFFT_FORWARD, st)) != DASP_OK) return rc;
  if (g.sets == 2) launch_mac<false, false, 1>(xs, hs, ys, I, J, h_stride != 0, I, items, 1.0f / (float)kNbA, st);
  else             launch_mac<false>(xs, hs, ys, I, J, h_stride != 0, I, items, 1.0f / (float)kNbA, st);
  DASP_LAUNCH_OK("partition_mac_kernel");
  if ((rc = exec_c2c(pl.xi, cufft, ys, CUFFT_INVERSE, st)) != DASP_OK) return rc;
  mix_blocks_kernel<<<dim3((unsigned)I, (unsigned)items), 256, 0, st>>>(x, ys, mix, mix_stride, y, item0, I, g.n, in_chs);
  DASP_LAUNCH_OK("mix_blocks_kernel");
  return DASP_OK;
}

// Backward of conv_fwd_chunk from its saved spectra xs / hs: gx = (1 - mix) g + mix c, c(s) = sum_tau IR(tau) g(s + tau),
// and per block the dL/dmix partials sum x (c - g) in the mixpart region; then the dL/dIR partitions
// E[j] = sum_p G[j+p] conj(X[p]) in the es region, in the form e (kPlanar needs own).  own (own_fft_rows of gy): the G
// transform and ifft_dx_kernel on the own FFT with the tables tw; otherwise the cuFFT pipeline.  Unfused, the dL/dIR
// correlation runs after the dL/dx inverse (the two correlations read the same inputs and write disjoint regions).
// h_stride: item stride of hs as in conv_fwd_chunk (0: one IR shared by the batch).  g.sets == 2 (a true-stereo IR): the
// products of partition_mac_kernel<TS 1 / TS 2>, and es receives 2 J partitions per item, set A then set B.
int conv_bwd_chunk(const ConvGeom& g, const Plans& pl, bool own, IrGrad e, const float* tw, const float* gy,
                   const float* x, int in_chs, const float2* xs, const float2* hs, int64_t h_stride, const float* mix,
                   int mix_stride, float* gx, unsigned char* ws, const BwdWs& w, int64_t item0, int64_t items,
                   cudaStream_t st) {
  float2* gs = (float2*)(ws + w.gs);
  float2* ds = (float2*)(ws + w.ds);
  float2* es = (float2*)(ws + w.es);
  float* mixpart = (float*)(ws + w.mixpart);
  void* cufft = ws + w.cufft;
  const float inv = 1.0f / (float)kNbA;
  const int I = (int)g.ib, J = (int)g.jb;
  const bool fused = fused_corr(e, I, J, g.sets);
  const bool ts = g.sets == 2;
  int rc;
  if (own) {
    if ((rc = configure_fft_kernels()) != DASP_OK) return rc;
    const int nblk = (int)(items * I);
    g_fft_kernel<<<persistent_grid(nblk), kFusedThreads, kFftSmemBytes, st>>>(gy, gs, tw, item0, I, g.n, nblk);
    DASP_LAUNCH_OK("g_fft_kernel");
    if (fused) {
      dim3 mgrid((kNbA / 2 + 1 + 127) / 128, (unsigned)items);
      const bool m12 = (I > J ? I : J) <= 12;
      if (ts && m12)  partition_mac_bwd_kernel<12, true><<<mgrid, 128, 0, st>>>(gs, hs, h_stride, xs, ds, es, I, J, inv);
      else if (ts)    partition_mac_bwd_kernel<kTsFusedMaxB, true><<<mgrid, 128, 0, st>>>(gs, hs, h_stride, xs, ds, es, I, J, inv);
      else if (m12)   partition_mac_bwd_kernel<12><<<mgrid, 128, 0, st>>>(gs, hs, h_stride, xs, ds, es, I, J, inv);
      else            partition_mac_bwd_kernel<16><<<mgrid, 128, 0, st>>>(gs, hs, h_stride, xs, ds, es, I, J, inv);
      DASP_LAUNCH_OK("partition_mac_bwd_kernel");
    } else {
      // dx windows: sum_j conj(H[j]) G[q+j]
      if (ts) launch_mac<true, true, 1>(gs, hs, ds, I, J, h_stride != 0, I, items, inv, st);
      else    launch_mac<true, true>(gs, hs, ds, I, J, h_stride != 0, I, items, inv, st);
      DASP_LAUNCH_OK("partition_mac_kernel<corr>");
    }
    ifft_dx_kernel<<<persistent_grid(items), kFusedThreads, kFftSmemBytes, st>>>(reinterpret_cast<const float*>(ds), tw, gy, x, mix,
                                                                  mix_stride, gx, mixpart, item0, (int)items, I, g.n,
                                                                  in_chs);
    DASP_LAUNCH_OK("ifft_dx_kernel");
  } else {
    g_blocks_kernel<<<dim3((unsigned)I, (unsigned)items), 256, 0, st>>>(gy, gs, item0, I, g.n);
    DASP_LAUNCH_OK("g_blocks_kernel");
    if ((rc = exec_c2c(pl.xi, cufft, gs, CUFFT_FORWARD, st)) != DASP_OK) return rc;
    if (ts) launch_mac<true, false, 1>(gs, hs, ds, I, J, h_stride != 0, I, items, inv, st);
    else    launch_mac<true>(gs, hs, ds, I, J, h_stride != 0, I, items, inv, st);
    DASP_LAUNCH_OK("partition_mac_kernel<corr>");
    if ((rc = exec_c2c(pl.xi, cufft, ds, CUFFT_INVERSE, st)) != DASP_OK) return rc;
    finish_dx_blocks_kernel<<<dim3((unsigned)I, (unsigned)items), 256, 0, st>>>(gy, x, ds, mix, mix_stride, gx, mixpart,
                                                                              item0, I, g.n, in_chs);
    DASP_LAUNCH_OK("finish_dx_blocks_kernel");
  }
  if (e == IrGrad::kPlanar && !fused) {
    // dIR partitions: sum_p conj(X[p]) G[j+p]
    if (ts) launch_mac<true, true, 2>(gs, xs, es, I, I, 1, J, items, inv, st);
    else    launch_mac<true, true>(gs, xs, es, I, I, 1, J, items, inv, st);
    DASP_LAUNCH_OK("partition_mac_kernel<corr>");
  } else if (e == IrGrad::kTime || e == IrGrad::kSpectra) {
    if (ts) launch_mac<true, false, 2>(gs, xs, es, I, I, 1, J, items, inv, st);
    else    launch_mac<true>(gs, xs, es, I, I, 1, J, items, inv, st);
    DASP_LAUNCH_OK("partition_mac_kernel<corr>");
    if (e == IrGrad::kSpectra) return DASP_OK;
    return exec_c2c(pl.hj, cufft, es, CUFFT_INVERSE, st);
  }
  return DASP_OK;
}

}  // namespace

void reverb_shutdown() {
  std::lock_guard<std::mutex> lk(g_mu);
  for (auto& kv : g_plans) cufftDestroy(kv.second.h);
  g_plans.clear();
  for (auto& kv : g_fb) cudaFree(kv.second);
  g_fb.clear();
  for (auto& kv : g_fft_tab) cudaFree(kv.second);
  g_fft_tab.clear();
  for (auto& kv : g_side) {
    for (int i = 0; i < 2; ++i) {
      cudaStreamDestroy(kv.second.side[i]);
      cudaEventDestroy(kv.second.done[i]);
    }
    cudaEventDestroy(kv.second.fork);
  }
  g_side.clear();
}

}  // namespace dasp

using namespace dasp;

extern "C" {

int dasp_debug_reverb_last_path(void) { return g_last_fused; }

// host-side restatement of signal.octave_band_filterbank: writes 12*taps floats (no GPU needed)
int dasp_reverb_filterbank(int64_t taps, double sample_rate, float* out) {
  DASP_REQUIRE(out != nullptr && taps >= 1 && (taps % 2) == 1, "filterbank: taps must be odd and out non-null");
  DASP_REQUIRE(sample_rate / 2.0 > 18000.0, "filterbank: needs 18 kHz < sample_rate/2");
  std::vector<float> v;
  octave_filterbank((int)taps, sample_rate, v);
  for (size_t i = 0; i < v.size(); ++i) out[i] = v[i];
  return DASP_OK;
}

int dasp_reverb_geometry(int64_t bs, int64_t n, int64_t num_samples, int64_t taps, int64_t chunk_items,
                         dasp_reverb_geom* out) {
  DASP_REQUIRE(out != nullptr, "reverb geometry: null out");
  Geom g;
  int rc = make_geom(bs, n, num_samples, taps, chunk_items, g);
  if (rc != DASP_OK) return rc;
  if ((rc = put_conv_geometry(g, &g, out)) != DASP_OK) return rc;
  out->nb = g.nb; out->hop = g.hop; out->nbk = g.nbk; out->rpp = g.rpp;
  out->f_floats = bs * kBands * g.pair_c64() * 2;
  return DASP_OK;
}

int dasp_reverb_fwd(const float* x, int64_t in_chs, const float* params, const float* noise, const uint64_t* seed_dev, float* y,
                    float* f_save, void* xspec_save, void* irspec_save, void* workspace,
                    int64_t workspace_bytes, int64_t bs, int64_t n, int64_t num_samples, int64_t taps,
                    int64_t chunk_items, float sample_rate, void* stream) {
  Geom g;
  int rc = make_geom(bs, n, num_samples, taps, chunk_items, g);
  if (rc != DASP_OK) return rc;
  DASP_REQUIRE(in_chs == 1 || in_chs == 2, "only mono/stereo signals are supported");
  if (bs == 0) return DASP_OK;
  DASP_REQUIRE(x && params && y && workspace, "reverb fwd: null pointer");
  DASP_REQUIRE(noise != nullptr || seed_dev != nullptr, "reverb fwd: device-noise mode needs seed_dev (a device pointer)");
  const unsigned long long* seed = reinterpret_cast<const unsigned long long*>(seed_dev);
  cudaStream_t st = (cudaStream_t)stream;
  std::lock_guard<std::mutex> lk(g_mu);
  const float2 *H = nullptr, *H1 = nullptr;
  const bool spectral = (noise == nullptr) && g.rpp <= kMaxSpectralR;
  if (spectral) { if ((rc = get_filterbank_n1(g, (double)sample_rate, st, &H1)) != DASP_OK) return rc; }
  else          { if ((rc = get_filterbank(g, (double)sample_rate, st, &H)) != DASP_OK) return rc; }
  Setup s{};
  if ((rc = conv_setup(g, &g, s)) != DASP_OK) return rc;
  if ((rc = check_workspace("reverb fwd", s.fwd.total, workspace_bytes)) != DASP_OK) return rc;
  const FwdWs& w = s.fwd;
  unsigned char* base = (unsigned char*)workspace;
  void* ws_cufft = base + w.cufft;
  const int64_t lp = g.L + g.P;
  const int nbk = (int)g.nbk, nb = (int)g.nb, hop = (int)g.hop, P = (int)g.P, I = (int)g.ib, J = (int)g.jb;

  // device-noise IR synthesis (every variant draws the same Philox stream; the two own-FFT ones are bit-identical):
  //   default, nb == 8192: ir_synth_cluster_kernel for R <= 6, generator -> ifft_shape_kernel for 7 <= R <= 16 or
  //     when the device cannot co-schedule the cluster (last path 2);
  //   dasp_debug_reverb_path(2), R <= 8: generator -> ifft_shape_kernel (last path 1);
  //   dasp_debug_reverb_path(1), and any other nb: generator -> batched cuFFT -> shape_ir_pp_kernel (last path 0).
  int synth = 0;
  const bool own_fft = spectral && nb == fft8k::kN && g.L < (int64_t)1 << 31;
  const bool two_kernel_hook = debug_reverb_path() == 2 && g.rpp <= kMaxHookR;
  if (own_fft && debug_reverb_path() != 1) synth = two_kernel_hook ? 1 : 2;
  g_last_fused = synth;
  // Pipeline: chunk k + 1's synthesis runs on a side stream while chunk k's convolution runs on st.  The synthesis holds
  // only the SMs its clusters fit on (17 clusters of 6 = 102 of 132 on an H100 SXM), the convolution fills the rest.
  // Chunk k's synthesis goes to side[k % 2] (the next chunk's clusters are queued behind the running ones and take each
  // slot as it frees), at the greatest priority so that pending clusters are dispatched before convolution CTAs, and
  // st waits for it before chunk k's convolution; the last of these waits joins every side-stream launch back into st,
  // so nothing outlives the call, and under stream capture the fork and join are graph edges.  This needs the chunks'
  // slots disjoint: the synthesis writes only f_save / irspec_save slots (kept when a backward follows; otherwise they
  // share one workspace slot), and neither side uses the shared cuFFT work area (own-FFT synthesis and convolution).
  const bool pipelined = synth != 0 && f_save && irspec_save && own_fft_rows(n, x, irspec_save);
  SideStreams* side = nullptr;
  if (pipelined) {
    if ((rc = get_side_streams(&side)) != DASP_OK) return rc;
    DASP_CUDA_OK(cudaEventRecord(side->fork, st));   // the seed word and the parameters are written on st
    for (int i = 0; i < 2; ++i) DASP_CUDA_OK(cudaStreamWaitEvent(side->side[i], side->fork, 0));
  }
  const int* prio = pipelined ? &side->prio : nullptr;

  for (int64_t item0 = 0, k = 0; item0 < bs; item0 += g.chunk, ++k) {
    const int64_t items = (bs - item0 < g.chunk) ? bs - item0 : g.chunk;
    const Plans& pl = (items == g.chunk) ? s.full : s.rem;
    const cudaStream_t sst = pipelined ? side->side[k & 1] : st;      // the stream of this chunk's synthesis
    // kept for the backward when the caller passes *_save buffers, transient workspace otherwise
    float2* C = f_save ? reinterpret_cast<float2*>(f_save) + item0 * kBands * g.pair_c64()
                       : reinterpret_cast<float2*>(base + w.extra);
    float2* xs = xspec_save ? (float2*)xspec_save + item0 * I * (int64_t)kNbA : (float2*)(base + w.xsp);
    float2* hs = irspec_save ? (float2*)irspec_save + item0 * J * (int64_t)kNbA : (float2*)(base + w.hsp);
    const dim3 gblk((unsigned)nbk, kBands, (unsigned)items);
    const bool own_conv = own_fft_rows(n, x, hs);

    // ---- IR synthesis: taps t < leff land as (left, right) pairs in the first half of partition t / kB of hs ----
    // x_fft_kernel reads nothing else of hs; the cuFFT transform of the partitions reads whole slots, so they are
    // zero-filled first
    if (!own_conv) DASP_CUDA_OK(cudaMemsetAsync(hs, 0, sizeof(float2) * items * J * kNbA, st));
    const float* tw = nullptr;
    if ((synth != 0 || own_conv) && (rc = get_fft_tables(st, &tw)) != DASP_OK) return rc;
    bool clustered = false;
    if (synth == 2 && g.rpp <= kMaxClusterR) {
      clustered = dispatch_fused((int)g.rpp, H1, tw, params + item0 * 25, hs, f_save ? C : nullptr, item0, items, g.L,
                                 g.leff, J, seed, sst, prio);
      if (clustered) DASP_LAUNCH_OK("ir_synth_cluster_kernel");
    }
    if (clustered) {
    } else if (synth != 0) {
      dispatch_spectral((int)g.rpp, C, H1, item0, items, nb, seed, /*planar=*/true, sst, prio);
      DASP_LAUNCH_OK("spectral_gen_kernel");
      if ((rc = launch_ifft_shape(C, tw, params + item0 * 25, hs, f_save != nullptr, items, g, J, sst, prio)) != DASP_OK)
        return rc;
    } else if (spectral) {
      // device noise: draw the filtered spectrum directly, one inverse transform (polyphase layout)
      dispatch_spectral((int)g.rpp, C, H1, item0, items, nb, seed, /*planar=*/false, st, nullptr);
      DASP_LAUNCH_OK("spectral_gen_kernel");
      if ((rc = exec_c2c(pl.pp, ws_cufft, C, CUFFT_INVERSE, st)) != DASP_OK) return rc;
      shape_ir_pp_kernel<<<dim3((unsigned)((g.leff + 255) / 256), (unsigned)items), 256, 0, st>>>(
          C, params + item0 * 25, hs, g.L, g.leff, J, (int)g.rpp, nb);
      DASP_LAUNCH_OK("shape_ir_pp_kernel");
    } else {
      // parity mode (caller's noise tensor) or very long IR: time-domain noise, overlap-save blocks
      if (noise) noise_pairs_layout_kernel<<<gblk, 256, 0, st>>>(noise, C, item0, nbk, nb, hop, lp);
      else       noise_pairs_philox_kernel<<<gblk, 256, 0, st>>>(C, item0, nbk, nb, hop, seed);
      DASP_LAUNCH_OK("reverb noise kernel");
      if ((rc = exec_c2c(pl.blk, ws_cufft, C, CUFFT_FORWARD, st)) != DASP_OK) return rc;
      cmul_filter_pairs_kernel<<<gblk, 256, 0, st>>>(C, H, nbk, nb);
      DASP_LAUNCH_OK("cmul_filter_pairs_kernel");
      if ((rc = exec_c2c(pl.blk, ws_cufft, C, CUFFT_INVERSE, st)) != DASP_OK) return rc;
      shape_ir_pairs_kernel<<<dim3((unsigned)nbk, (unsigned)items), 256, 0, st>>>(C, params + item0 * 25, hs, g.L, g.leff,
                                                                               J, nbk, nb, hop, P);
      DASP_LAUNCH_OK("shape_ir_pairs_kernel");
    }
    if (pipelined) {
      DASP_CUDA_OK(cudaEventRecord(side->done[k & 1], sst));
      DASP_CUDA_OK(cudaStreamWaitEvent(st, side->done[k & 1], 0));
    }
    if ((rc = conv_fwd_chunk(g, pl, own_conv, tw, x, (int)in_chs, xs, hs, J * (int64_t)kNbA, params + 24, 25, y, base,
                             w, item0, items, st)) != DASP_OK)
      return rc;
  }
  return DASP_OK;
}

int dasp_reverb_bwd(const float* gy, const float* x, int64_t in_chs, const float* params,
                    const float* f_save, const void* xspec_save, const void* irspec_save, float* gx, float* gparams,
                    void* workspace, int64_t workspace_bytes, int64_t bs, int64_t n, int64_t num_samples, int64_t taps,
                    int64_t chunk_items, int64_t device_noise, void* stream) {
  Geom g;
  int rc = make_geom(bs, n, num_samples, taps, chunk_items, g);
  if (rc != DASP_OK) return rc;
  DASP_REQUIRE(in_chs == 1 || in_chs == 2, "only mono/stereo signals are supported");
  if (bs == 0) return DASP_OK;
  const bool polyphase = device_noise != 0 && g.rpp <= kMaxSpectralR;   // layout the forward left in f_save
  DASP_REQUIRE(gy && x && params && f_save && xspec_save && irspec_save && gx && gparams && workspace,
               "reverb bwd: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  std::lock_guard<std::mutex> lk(g_mu);
  Setup s{};
  if ((rc = conv_setup(g, &g, s)) != DASP_OK) return rc;
  if ((rc = check_workspace("reverb bwd", s.bwd.total, workspace_bytes)) != DASP_OK) return rc;
  const BwdWs& w = s.bwd;
  unsigned char* base = (unsigned char*)workspace;
  const float2* ws_es = (const float2*)(base + w.es);
  float* ws_irpart = (float*)(base + w.extra);
  const float* ws_mixpart = (const float*)(base + w.mixpart);
  const int nbk = (int)g.nbk, nb = (int)g.nb, hop = (int)g.hop, P = (int)g.P, I = (int)g.ib, J = (int)g.jb;

  for (int64_t item0 = 0; item0 < bs; item0 += g.chunk) {
    const int64_t items = (bs - item0 < g.chunk) ? bs - item0 : g.chunk;
    const Plans& pl = (items == g.chunk) ? s.full : s.rem;
    const float2* C = reinterpret_cast<const float2*>(f_save) + item0 * kBands * g.pair_c64();
    const float2* xs = (const float2*)xspec_save + item0 * I * (int64_t)kNbA;
    const float2* hs = (const float2*)irspec_save + item0 * J * (int64_t)kNbA;

    const bool own_conv = own_fft_rows(n, gy, nullptr);
    // dL/dIR through the band parameters on the own FFT needs the polyphase f_save at nb = 8192
    const bool own_irgrad = own_conv && polyphase && nb == fft8k::kN && g.L < (int64_t)1 << 31;
    const float* tw = nullptr;
    if (own_conv && (rc = get_fft_tables(st, &tw)) != DASP_OK) return rc;
    if ((rc = conv_bwd_chunk(g, pl, own_conv, own_irgrad ? IrGrad::kPlanar : IrGrad::kTime, tw, gy, x, (int)in_chs, xs,
                             hs, J * (int64_t)kNbA, params + 24, 25, gx, base, w, item0, items, st)) != DASP_OK)
      return rc;
    int nparts;
    if (own_irgrad) {
      nparts = J;
      const int nunits = (int)(items * J);
      ifft_irgrad_kernel<<<persistent_grid(nunits), kFusedThreads, kFftSmemBytes, st>>>(reinterpret_cast<const float*>(ws_es), tw, C,
                                                                        params + item0 * 25, ws_irpart, (int)g.L,
                                                                        (int)g.leff, J, (int)g.rpp, nunits);
      DASP_LAUNCH_OK("ifft_irgrad_kernel");
    } else {
      if (polyphase) {
        nparts = (int)g.nparts_pp();
        ir_grad_pp_kernel<<<dim3((unsigned)nparts, (unsigned)items), 256, 0, st>>>(ws_es, C, params + item0 * 25, ws_irpart,
                                                                                  g.L, g.leff, J, (int)g.rpp, nb);
      } else {
        nparts = nbk;
        ir_grad_pairs_kernel<<<dim3((unsigned)nbk, (unsigned)items), 256, 0, st>>>(ws_es, C, params + item0 * 25, ws_irpart,
                                                                                    g.L, g.leff, J, nbk, nb, hop, P);
      }
      DASP_LAUNCH_OK("ir_grad kernel");
    }
    reverb_param_grad_kernel<<<(unsigned)((items * 25 + 127) / 128), 128, 0, st>>>(ws_irpart, ws_mixpart, params, gparams,
                                                                                   item0, items, nparts, I);
    DASP_LAUNCH_OK("reverb_param_grad_kernel");
  }
  return DASP_OK;
}

// ------------------------------------------------------------------ convolution_reverberation
namespace {
int g_conv_last_path[2] = {0, 0};                    // test hook: dispatch of the last conv forward / backward

// The bodies of dasp_conv_* (one IR per item) and dasp_conv_shared_* (one IR for the whole batch).  Shared, the IR's
// partitions are filled and transformed once before the first chunk and every item reads the same spectra (item stride
// 0); the backward sums mix[b] times each item's dL/dIR partition spectra in fp64 (irgrad_sum_kernel) and transforms
// the sum once after the last chunk.  A true-stereo IR (ir_chs 4) is two partition sets per IR (g.sets = 2), carried
// through the same routines.
int conv_op_geometry(bool shared, int sets, int64_t bs, int64_t n, int64_t ir_len, int64_t chunk_items,
                     dasp_conv_geom* out) {
  DASP_REQUIRE(out != nullptr, "conv geometry: null out");
  ConvGeom g;
  int rc = make_conv_geom(bs, n, ir_len, chunk_items, g);
  if (rc != DASP_OK) return rc;
  g.shared = shared;
  g.sets = sets;
  return put_conv_geometry(g, nullptr, out);
}
int ir_sets(int64_t ir_chs) { return ir_chs == 4 ? 2 : 1; }

int conv_op_fwd(bool shared, const float* x, int64_t in_chs, const float* ir, int64_t ir_chs, int64_t ir_len,
                const float* mix, float* y, void* xspec_save, void* irspec_save, void* workspace,
                int64_t workspace_bytes, int64_t bs, int64_t n, int64_t chunk_items, void* stream) {
  ConvGeom g;
  int rc = make_conv_geom(bs, n, ir_len, chunk_items, g);
  if (rc != DASP_OK) return rc;
  g.shared = shared;
  DASP_REQUIRE((in_chs == 1 || in_chs == 2) && (ir_chs == 1 || ir_chs == 2 || ir_chs == 4),
               "conv: only mono/stereo signals and mono/stereo/true-stereo IRs");
  g.sets = ir_sets(ir_chs);
  if (bs == 0) return DASP_OK;
  DASP_REQUIRE(x && ir && mix && y && workspace, "conv fwd: null pointer");
  DASP_REQUIRE((xspec_save == nullptr) == (irspec_save == nullptr), "conv fwd: pass both *_save buffers or neither");
  cudaStream_t st = (cudaStream_t)stream;
  std::lock_guard<std::mutex> lk(g_mu);
  Setup s{};
  if ((rc = conv_setup(g, nullptr, s)) != DASP_OK) return rc;
  if ((rc = check_workspace("conv fwd", s.fwd.total, workspace_bytes)) != DASP_OK) return rc;
  const FwdWs& w = s.fwd;
  unsigned char* base = (unsigned char*)workspace;
  const int I = (int)g.ib, J = (int)g.jb, S = g.sets;
  const int64_t h_stride = shared ? 0 : S * J * (int64_t)kNbA;
  float2* const hs0 = irspec_save ? (float2*)irspec_save : (float2*)(base + w.hsp);
  const float* tw = nullptr;

  // IR taps t < leff of items [item0, item0 + items) into their partition slots; the cuFFT transform of the partitions
  // reads whole slots, x_fft_kernel only the taps ir_pack_kernel writes
  auto fill_ir = [&](float2* hs, bool own, int64_t item0, int64_t items) -> int {
    if (!own) DASP_CUDA_OK(cudaMemsetAsync(hs, 0, sizeof(float2) * items * S * J * kNbA, st));
    ir_pack_kernel<<<dim3((unsigned)((g.leff + 255) / 256), (unsigned)items, (unsigned)S), 256, 0, st>>>(
        ir, hs, item0, J, g.L, g.leff, (int)ir_chs);
    DASP_LAUNCH_OK("ir_pack_kernel");
    return DASP_OK;
  };
  if (shared) {
    const bool own = own_fft_rows(n, x, hs0);
    if ((rc = fill_ir(hs0, own, 0, 1)) != DASP_OK) return rc;
    if (own && (rc = get_fft_tables(st, &tw)) != DASP_OK) return rc;
    if ((rc = conv_shared_ir_spectra(g, s.ir1, own, tw, hs0, base, w, st)) != DASP_OK) return rc;
  }
  for (int64_t item0 = 0; item0 < bs; item0 += g.chunk) {
    const int64_t items = (bs - item0 < g.chunk) ? bs - item0 : g.chunk;
    const Plans& pl = (items == g.chunk) ? s.full : s.rem;
    float2* xs = xspec_save ? (float2*)xspec_save + item0 * I * (int64_t)kNbA : (float2*)(base + w.xsp);
    float2* hs = irspec_save ? hs0 + item0 * h_stride : hs0;
    const bool own_conv = own_fft_rows(n, x, hs);
    g_conv_last_path[0] = (own_conv ? 1 : 0) | (shared ? 2 : 0) | (S == 2 ? 4 : 0);
    if (!shared && (rc = fill_ir(hs, own_conv, item0, items)) != DASP_OK) return rc;
    if (own_conv && (rc = get_fft_tables(st, &tw)) != DASP_OK) return rc;
    if ((rc = conv_fwd_chunk(g, pl, own_conv, tw, x, (int)in_chs, xs, hs, h_stride, mix, 1, y, base, w, item0, items,
                             st)) != DASP_OK)
      return rc;
  }
  return DASP_OK;
}

int conv_op_bwd(bool shared, const float* gy, const float* x, int64_t in_chs, int64_t ir_chs, int64_t ir_len,
                const float* mix, const void* xspec_save, const void* irspec_save, float* gx, float* gir, float* gmix,
                void* workspace, int64_t workspace_bytes, int64_t bs, int64_t n, int64_t chunk_items, void* stream) {
  ConvGeom g;
  int rc = make_conv_geom(bs, n, ir_len, chunk_items, g);
  if (rc != DASP_OK) return rc;
  g.shared = shared;
  DASP_REQUIRE((in_chs == 1 || in_chs == 2) && (ir_chs == 1 || ir_chs == 2 || ir_chs == 4),
               "conv: only mono/stereo signals and mono/stereo/true-stereo IRs");
  g.sets = ir_sets(ir_chs);
  if (bs == 0) return DASP_OK;
  DASP_REQUIRE(gy && x && mix && xspec_save && irspec_save && gx && gmix && workspace, "conv bwd: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  std::lock_guard<std::mutex> lk(g_mu);
  Setup s{};
  if ((rc = conv_setup(g, nullptr, s)) != DASP_OK) return rc;
  if ((rc = check_workspace("conv bwd", s.bwd.total, workspace_bytes)) != DASP_OK) return rc;
  const BwdWs& w = s.bwd;
  unsigned char* base = (unsigned char*)workspace;
  float2* ws_es = (float2*)(base + w.es);
  const float* ws_mixpart = (const float*)(base + w.mixpart);
  double2* ws_acc = (double2*)(base + w.acc);
  const int I = (int)g.ib, J = (int)g.jb, S = g.sets;
  const int64_t h_stride = shared ? 0 : S * J * (int64_t)kNbA;
  const float* tw = nullptr;
  bool own_conv = false;

  // dL/dIR taps of items [item0, item0 + items) from their partitions in the es region (planar spectra, or time-domain
  // pairs after the inverse cuFFT), times mix[b] (a null mix: 1)
  auto ir_taps = [&](IrGrad e, int64_t item0, int64_t items, const float* mx) -> int {
    if (e == IrGrad::kPlanar) {
      const int nunits = (int)(items * S * J);
      ifft_irtaps_kernel<<<persistent_grid(nunits), kFusedThreads, kFftSmemBytes, st>>>(reinterpret_cast<const float*>(ws_es), tw, mx,
                                                                        gir, item0, J, S, g.L, g.leff, (int)ir_chs, nunits);
      DASP_LAUNCH_OK("ifft_irtaps_kernel");
    }
    // taps t0 <= t < L: the zeros from leff on after ifft_irtaps_kernel, every tap after the cuFFT inverse
    const int64_t t0 = e == IrGrad::kPlanar ? g.leff : 0;
    if (g.L > t0) {
      irtaps_unpack_kernel<<<dim3((unsigned)((g.L - t0 + 255) / 256), (unsigned)items, (unsigned)S), 256, 0, st>>>(
          ws_es, mx, gir, item0, J, g.L, g.leff, (int)ir_chs, t0);
      DASP_LAUNCH_OK("irtaps_unpack_kernel");
    }
    return DASP_OK;
  };
  for (int64_t item0 = 0; item0 < bs; item0 += g.chunk) {
    const int64_t items = (bs - item0 < g.chunk) ? bs - item0 : g.chunk;
    const Plans& pl = (items == g.chunk) ? s.full : s.rem;
    const float2* xs = (const float2*)xspec_save + item0 * I * (int64_t)kNbA;
    const float2* hs = (const float2*)irspec_save + item0 * h_stride;
    own_conv = own_fft_rows(n, gy, nullptr);
    const IrGrad e = gir == nullptr ? IrGrad::kNone
                                    : (own_conv ? IrGrad::kPlanar : (shared ? IrGrad::kSpectra : IrGrad::kTime));
    // bit 0: own FFT, bit 1: fused correlations, bit 2: dL/dIR computed, bit 3: one IR shared by the batch, bit 4: a
    // true-stereo IR
    g_conv_last_path[1] = (own_conv ? 1 : 0) | (fused_corr(e, I, J, S) ? 2 : 0) | (gir ? 4 : 0) | (shared ? 8 : 0) |
                          (S == 2 ? 16 : 0);
    if (own_conv && (rc = get_fft_tables(st, &tw)) != DASP_OK) return rc;
    if ((rc = conv_bwd_chunk(g, pl, own_conv, e, tw, gy, x, (int)in_chs, xs, hs, h_stride, mix, 1, gx, base, w, item0,
                             items, st)) != DASP_OK)
      return rc;
    if (e != IrGrad::kNone && shared) {
      const int64_t per_item = S * J * (int64_t)kNbA;
      irgrad_sum_kernel<<<(unsigned)((per_item + 255) / 256), 256, 0, st>>>(ws_es, mix, ws_acc, item0, (int)items,
                                                                            per_item, item0 + items == bs);
      DASP_LAUNCH_OK("irgrad_sum_kernel");
    } else if (e != IrGrad::kNone && (rc = ir_taps(e, item0, items, mix)) != DASP_OK) {
      return rc;
    }
    conv_mix_grad_kernel<<<(unsigned)((items + 127) / 128), 128, 0, st>>>(ws_mixpart, gmix, item0, items, I);
    DASP_LAUNCH_OK("conv_mix_grad_kernel");
  }
  if (shared && gir) {
    // the summed partition spectra, rounded to fp32 in item 0's slots of es: S J inverse transforms for the one IR
    if (!own_conv && (rc = exec_c2c(s.ir1, base + w.cufft, ws_es, CUFFT_INVERSE, st)) != DASP_OK) return rc;
    if ((rc = ir_taps(own_conv ? IrGrad::kPlanar : IrGrad::kTime, 0, 1, nullptr)) != DASP_OK) return rc;
  }
  return DASP_OK;
}
}  // namespace

int dasp_debug_conv_last_path(int which) { return g_conv_last_path[which ? 1 : 0]; }

int dasp_conv_geometry(int64_t bs, int64_t n, int64_t ir_len, int64_t chunk_items, dasp_conv_geom* out) {
  return conv_op_geometry(false, 1, bs, n, ir_len, chunk_items, out);
}

int dasp_conv_ts_geometry(int64_t bs, int64_t n, int64_t ir_len, int64_t chunk_items, dasp_conv_geom* out) {
  return conv_op_geometry(false, 2, bs, n, ir_len, chunk_items, out);
}

int dasp_conv_fwd(const float* x, int64_t in_chs, const float* ir, int64_t ir_chs, int64_t ir_len, const float* mix,
                  float* y, void* xspec_save, void* irspec_save, void* workspace, int64_t workspace_bytes, int64_t bs,
                  int64_t n, int64_t chunk_items, void* stream) {
  return conv_op_fwd(false, x, in_chs, ir, ir_chs, ir_len, mix, y, xspec_save, irspec_save, workspace, workspace_bytes,
                     bs, n, chunk_items, stream);
}

int dasp_conv_bwd(const float* gy, const float* x, int64_t in_chs, int64_t ir_chs, int64_t ir_len, const float* mix,
                  const void* xspec_save, const void* irspec_save, float* gx, float* gir, float* gmix, void* workspace,
                  int64_t workspace_bytes, int64_t bs, int64_t n, int64_t chunk_items, void* stream) {
  return conv_op_bwd(false, gy, x, in_chs, ir_chs, ir_len, mix, xspec_save, irspec_save, gx, gir, gmix, workspace,
                     workspace_bytes, bs, n, chunk_items, stream);
}

int dasp_conv_shared_geometry(int64_t bs, int64_t n, int64_t ir_len, int64_t chunk_items, dasp_conv_geom* out) {
  return conv_op_geometry(true, 1, bs, n, ir_len, chunk_items, out);
}

int dasp_conv_shared_ts_geometry(int64_t bs, int64_t n, int64_t ir_len, int64_t chunk_items, dasp_conv_geom* out) {
  return conv_op_geometry(true, 2, bs, n, ir_len, chunk_items, out);
}

int dasp_conv_shared_fwd(const float* x, int64_t in_chs, const float* ir, int64_t ir_chs, int64_t ir_len,
                         const float* mix, float* y, void* xspec_save, void* irspec_save, void* workspace,
                         int64_t workspace_bytes, int64_t bs, int64_t n, int64_t chunk_items, void* stream) {
  return conv_op_fwd(true, x, in_chs, ir, ir_chs, ir_len, mix, y, xspec_save, irspec_save, workspace, workspace_bytes,
                     bs, n, chunk_items, stream);
}

int dasp_conv_shared_bwd(const float* gy, const float* x, int64_t in_chs, int64_t ir_chs, int64_t ir_len,
                         const float* mix, const void* xspec_save, const void* irspec_save, float* gx, float* gir,
                         float* gmix, void* workspace, int64_t workspace_bytes, int64_t bs, int64_t n,
                         int64_t chunk_items, void* stream) {
  return conv_op_bwd(true, gy, x, in_chs, ir_chs, ir_len, mix, xspec_save, irspec_save, gx, gir, gmix, workspace,
                     workspace_bytes, bs, n, chunk_items, stream);
}

}  // extern "C"
