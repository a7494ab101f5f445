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
// its dL/dIR consumer.  A true-stereo IR (ir_chs 4) is two partition sets per IR (ConvGeom::sets), multiplied by the TS
// variants of the MAC kernels.
//
// convolution_bus (dasp_conv_bus_*) is the same partitioned convolution for S inputs summed into O = 1 or 2 outputs:
// every signal's rows are packed two per transform (bus_fft_kernel, ir_pack_kernel + x_fft_kernel's partition units),
// bus_mac_kernel sums the untangled products over the inputs, and bus_ifft_kernel writes the outputs, dL/dx and dL/dIR.
// multichannel_convolution (dasp_conv_mc_*) is the bus with up to 32 outputs: the outputs and their gradients in
// ceil(M / 2) row pairs per block, and busmc_mac_kernel for the products when M >= 3.
//
// time_varying_convolution_reverberation (dasp_tvconv_*) is the same convolution with K IRs crossfaded along the
// output: the audio windows of a static convolution, the products of the two IRs of each block (tv_mac_kernel), and
// the crossfade in the epilogue of the inverse (tv_ifft_kernel) and in the prologue of the gradient transform
// (tv_fft_kernel).
//
// time_varying_convolution_bus (dasp_tvbus_*) combines the two: the bus's packed window spectra, IR trajectories for
// every source-to-output path, the two IR sets' products per block summed over the sources (tvbus_mac_kernel), and one
// crossfaded inverse per output row and block (tvbus_ifft_kernel).  Its source-side crossfade (dasp_tvbus_in_*) weights
// the input instead, so every sample keeps the IR sets of its emission time: zero-padded transforms of each source's
// weighted blocks (tvbusin_fft_kernel), the products with the IR sets of each input block's interval, overlap-added on
// the spectra (tvbusin_mac_kernel), and the crossfade of dL/dx in the epilogue of its inverse (tvbusin_ifft_kernel).
// time_varying_multichannel_convolution (dasp_tvmc_*, dasp_tvmc_in_*) is that bus with up to 32 outputs: for M >= 3 its
// products are tvmc_mac_kernel's / tvmcin_mac_kernel's, one slice per output pair, input pair or partition set, and
// every transform is an existing kernel's.
//
// The ops whose IR the caller supplies run one host stage per direction (caller_ir_fwd / caller_ir_bwd: checks,
// workspace, IR packing, chunk loop, zeros of the unreachable dL/dIR taps).  One IR for the whole batch
// (dasp_conv_shared_*, dasp_conv_bus_shared_*) is the item stride 0 of the IR spectra: they are transformed once, and
// irgrad_sum_kernel sums the items' dL/dIR spectra in fp64 before one inverse transform.
//
// noise_shaped_impulse_response (dasp_nsir_*) is the IR synthesis without the convolution, with the geometry of the
// reverb at n = L.  Every synthesis kernel is a template on its output sink (PartitionSink: the convolution's partition
// slots; PlanarSink: the caller's (bs, 2, L) rows), and both ops run one host-side synthesis stage: choose_synth (the
// variant and its filter bank, once per call) and synth_chunk (one chunk).  The backward of the IR op packs the planar
// dL/dIR with ir_pack_kernel and runs the reverb's band contraction, ir_grad_chunk, and reverb_param_grad_kernel.
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
#include <type_traits>
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
// the partitioned audio convolution, shared by the reverb, convolution_reverberation and convolution_bus
struct ConvGeom {
  int64_t bs, n, L;
  int64_t leff;                 // min(L, n): the only IR taps that can reach the output
  int64_t ib, jb;               // output/input blocks of kB samples, IR partitions of kB taps
  int64_t chunk;
  bool shared = false;          // one impulse response for the whole batch (the ops whose IR the caller supplies)
  int p = 1;                    // window spectra per block: ceil(S / 2) for the bus
  int sets = 1;                 // partition sets per IR: 2 for a true-stereo IR, ceil(S O / 2) for the bus
  bool has_mix = true;          // a dry/wet mix, and with it the dL/dmix partials region (not the bus)
  bool own_only = false;        // the own FFT only: no cuFFT plans or work area, no dasp_debug_reverb_path(1) (the bus)
  int64_t ex = 0;               // product / gradient spectra per item beyond ib: the crossfaded blocks of the
                                // time-varying convolution, which carry two IRs' products
  int64_t xw = 0;               // window (and dL/dx) spectra per item when not p ib: the source-side crossfade's
  int64_t xwin() const { return xw > 0 ? xw : p * ib; }
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

// Output sinks of the IR synthesis: where tap t (left, right) of chunk item il goes.  The reverb writes the partition
// layout of its audio convolution; noise_shaped_impulse_response writes planar (items, 2, L) rows (ir points at the
// chunk's first item).  Every synthesis variant takes the sink as a template parameter, so both ops run the same
// generator and epilogue arithmetic.
struct PartitionSink {
  float2* Hb; int jb;
  template <class Tap>
  __device__ __forceinline__ void operator()(int64_t il, Tap t, float l, float r) const {
    Hb[ir_slot(il, jb, t)] = make_float2(l, r);
  }
};
struct PlanarSink {
  float* ir; int64_t L;
  template <class Tap>
  __device__ __forceinline__ void operator()(int64_t il, Tap t, float l, float r) const {
    float* row = ir + il * 2 * L;
    row[t] = l;
    row[L + t] = r;
  }
};

// IR[c][t] = (1/12) sum_k gain_k exp(-(10 decay_k + 1) tt(t)) f_c[k][t]  for t < leff, handed to the sink (the reverb:
// (left, right) complex pairs in the first half of partition t / kB; every synthesis variant writes these taps and
// nothing else).
// grid = (nbk, items): CTA (b, item) produces samples [b*hop, (b+1)*hop).
template <class Sink>
__global__ void shape_ir_pairs_kernel(const float2* __restrict__ C, const float* __restrict__ params /* chunk x 25 */,
                                      Sink out, int64_t L, int64_t leff, int nbk, int nb, int hop, int P) {
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
    out(il, t, al, ar);
  }
}

// polyphase layout variant, threads in TIME order (coalesced IR stores; the 12 band loads of a thread are
// issued together).  grid = (ceil(leff / 256), items)
template <class Sink>
__global__ void shape_ir_pp_kernel(const float2* __restrict__ C, const float* __restrict__ params, Sink out, int64_t L,
                                   int64_t leff, int R, int nb) {
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
  out(il, t, al, ar);
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
// the accumulated IR taps tau_q = R (t + 512 q) + c below leff of item il to the sink.  A planar sink stores them R
// floats apart; the R CTAs of an item (one per class c) fill the rest of every 32-byte sector in the same kernel, so the
// partial sectors can meet in L2 instead of costing a packed copy and an unpack pass (DESIGN.md 4.4).
template <class Sink>
__device__ __forceinline__ void store_ir_taps(const Sink& out, int64_t il, int R, int c, int leff, int t,
                                              const float (&accr)[16], const float (&acci)[16]) {
#pragma unroll
  for (int q = 0; q < 16; ++q) {
    const int tau = R * (t + 512 * q) + c;
    if (tau < leff) out(il, tau, accr[q], acci[q]);
  }
}

// Replaces the batched cuFFT C2C + shape_ir_pp_kernel pair: the generator's spectrum is read ONCE (bulk copies
// straight into the planar shared-memory layout of fft8192.cuh, double buffered across the 12 bands), transformed
// in shared memory, and each thread accumulates  gain_k env_k(t) f_k(t) / 12  for its 16 taps in registers.  The
// filtered noise f is written back (over the consumed spectrum block, as (left, right) pairs) only when the
// backward needs it.  grid = (R, items): CTA (c, item) owns polyphase class c, i.e. the IR taps R a + c.
template <class Sink>
__global__ void __launch_bounds__(kFusedThreads, 1)
ifft_shape_kernel(float* __restrict__ Cpl, const float* __restrict__ twiddles, const float* __restrict__ params, Sink out,
                  int save_f, int L, int leff, int R) {
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
  store_ir_taps(out, il, R, c, leff, t, accr, acci);
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
template <int R, class Sink>
__global__ void __launch_bounds__(kSynthThreads, 1)
ir_synth_cluster_kernel(const float2* __restrict__ H1, const float* __restrict__ twiddles, const float* __restrict__ params,
                        Sink out, float2* __restrict__ Csave, int64_t item0, int items, int L, int leff,
                        const unsigned long long* seed) {
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
      store_ir_taps(out, il, R, (int)c, leff, t, accr, acci);
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

// noise_shaped_impulse_response: its [items][24] parameter rows as the reverb's [items][25] rows with a mix of 1, so
// band_gain / band_rate and reverb_param_grad_kernel read them unchanged (the factor 1 keeps every gradient's bits)
__global__ void nsir_params_kernel(const float* __restrict__ p24, float* __restrict__ p25, int64_t items) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= items * 25) return;
  const int64_t row = i / 25;
  const int q = (int)(i - row * 25);
  p25[i] = q < 24 ? p24[row * 24 + q] : 1.0f;
}

// ---- convolution_reverberation: the audio convolution above with an impulse response supplied by the caller ----------
// Forward: ir_pack_kernel puts the caller's taps where the IR synthesis puts its own; x_fft_kernel, partition_mac_kernel
// and ifft_mix_kernel (or the cuFFT pipeline) then run unchanged.  Backward: g_fft_kernel, the correlations and
// ifft_dx_kernel as in the reverb; dL/dIR partition j = mix * first half of IFFT(sum_p G[j+p] conj(X[p])), unpacked into
// the caller's rows by ifft_irtaps_kernel (or irtaps_unpack_kernel after the cuFFT inverse).

// taps t < leff of the planar (bs, rows, L) rows -> (row 2s, row 2s + 1) pairs in the first half of partition slot
// t / kB of set s = gridDim.z index, i.e. of slot (il * sets + s).  An odd last row pairs with itself when odd_self (a
// mono IR of convolution_reverberation feeds both channels), else with 0 (the bus).  A true-stereo IR (rows L->L, L->R,
// R->L, R->R) fills two sets per item.  grid = (ceil(leff / 256), items, sets)
__global__ void ir_pack_kernel(const float* __restrict__ ir, float2* __restrict__ Hb, int64_t item0, int J, int64_t L,
                               int64_t leff, int rows, bool odd_self) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t il = blockIdx.y;
  const int s = blockIdx.z;
  if (t >= leff) return;
  const bool pair = 2 * s + 1 < rows;
  const float* ra = ir + ((item0 + il) * rows + 2 * s) * L;
  const float* rb = pair ? ra + L : ra;
  const float im = rb[t];                          // loaded either way: both loads issue together
  Hb[ir_slot(il * gridDim.z + s, J, t)] = make_float2(ra[t], pair || odd_self ? im : 0.f);
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

// dL/dIR taps [0, leff) of the caller's rows: mix * Et (inverse-transformed partitions, pairs in the first half of each
// slot).  A null mix is a factor of 1.  Partition set s (gridDim.z = 2 for a true-stereo IR) goes to rows 2s, 2s + 1.
// grid = (ceil(leff / 256), items, 1 or 2 sets)
__global__ void irtaps_unpack_kernel(const float2* __restrict__ Et, const float* __restrict__ mix, float* __restrict__ gir,
                                     int64_t item0, int J, int64_t L, int64_t leff, int ir_chs) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t il = blockIdx.y, b = item0 + il;
  const int s = blockIdx.z;
  if (t >= leff) return;
  const float2 v = Et[ir_slot(il * gridDim.z + s, J, t)];
  const float mx = mix ? mix[b] : 1.f;
  float* row = gir + (b * ir_chs + 2 * s) * L;
  if (ir_chs == 1) row[t] = mx * (v.x + v.y);
  else { row[t] = mx * v.x; row[L + t] = mx * v.y; }
}

// dL/dIR of one impulse response shared by the batch: the sum over items b of mix[b] E_b (a null mix: factors of 1),
// taken on the partition spectra E_b of the es region before any inverse transform (the inverse is linear).  Element by
// element in fp64 and in absolute item order: a product of two floats is exact in fp64, so every element goes through
// the same sequence of additions however the batch is cut into chunks, and the result is the same bits for every chunk
// size.  Item 0 writes acc instead of adding to it (the workspace is never cleared); the chunk that holds the last item
// writes the sum, rounded to fp32, over item 0's slot of Et instead, for the inverse transforms (thread e alone reads
// and writes element e of every slot).
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
    const double m = mix ? (double)mix[0] : 1.0;
    a = make_double2(m * (double)v.x, m * (double)v.y);
    il = 1;
  }
  for (; il < items; ++il) {
    const float2 v = Et[il * per_item + e];
    const double m = mix ? (double)mix[item0 + il] : 1.0;
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

// ---- convolution_bus: S input rows, each through its own IR, summed into O = 1 or 2 output rows -----------------
// Every signal of the bus is a group of rows (the S inputs, the O outputs, the S O IR rows s O + o): its rows are packed
// two per complex transform, row 2k as the real and row 2k + 1 as the imaginary part, and an odd last row packs alone
// (imaginary part 0).  So an item has P = ceil(S / 2) window spectra per block, NH = ceil(S O / 2) partition sets
// (a stereo bus: set s = h_s0 + i h_s1; a mono bus: set k = h_2k + i h_2k+1) and one gradient spectrum per block.
// bus_mac_kernel untangles every operand into the spectra of its real rows, so one formula serves both bus widths.

// forward transforms of row pairs, runs of kConvRun units (il, k, i), il < items, k < groups, i < I:
//   out[((il*groups + k)*I + i)*kNbA + f] = FFT of (r_2k + i r_2k+1)[(i-1) kB + m], m < kNbA, zero outside [lo, n), where
//   the rows r are the `rows` rows of item item0 + il in src and lo = 0 (half == 0: the audio windows, as x_fft_kernel)
//   or kB (half == 1: [zeros(kB) | g[i kB, (i+1) kB)], g_fft_kernel's block i); lo = kB for i = 0 either way.
//   Requires n % 4 == 0 and 16-byte aligned rows (bulk copies).
__global__ void __launch_bounds__(kFusedThreads, 1)
bus_fft_kernel(const float* __restrict__ src, float2* __restrict__ out, const float* __restrict__ twiddles, int64_t item0,
               int rows, int groups, int I, int64_t n, int half, int nunits) {
  extern __shared__ __align__(128) float sm[];
  FftSmem s(sm);
  const int t = threadIdx.x;
  s.init(twiddles, t);
  const fft8k::Tables tb = fft8k::carve_tables(s.tabf);
  const int m0 = blockIdx.x * kConvRun;
  const int m1 = nunits - m0 < kConvRun ? nunits : m0 + kConvRun;
  auto fetch = [&](int it, int m) {                // all threads: zero padding; thread 0: the bulk copies
    if (m >= m1) return;
    const int q = m / I, i = m - q * I;            // q = il * groups + k
    const int64_t il = q / groups;
    const int k = q - (int)il * groups;
    const bool two = 2 * k + 1 < rows;
    float* re = s.buf(it);
    float* im = re + fft8k::kPlaneG;
    const int64_t s0 = (int64_t)(i - 1) * kB;
    const int lo = (half || i == 0) ? kB : 0;
    const int64_t rem = n - s0;
    const int hi = rem < kNbA ? (int)rem : kNbA;   // valid window samples are [lo, hi), hi > lo
    for (int e = t; e < lo; e += kFusedThreads) { re[e] = 0.f; im[e] = 0.f; }
    for (int e = hi + t; e < kNbA; e += kFusedThreads) { re[e] = 0.f; im[e] = 0.f; }
    if (!two) for (int e = lo + t; e < hi; e += kFusedThreads) im[e] = 0.f;
    if (t == 0) {
      const float* ra = src + ((item0 + il) * rows + 2 * k) * n + s0;
      uint64_t* bar = &s.full[it & 1];
      mbar_arrive_expect_tx(bar, (two ? 2u : 1u) * (uint32_t)(hi - lo) * 4u);
      for (int o = lo; o < hi; o += 4096) {
        const uint32_t bytes = (uint32_t)((hi - o < 4096 ? hi - o : 4096) * 4);
        tma_load_1d(re + o, ra + o, bytes, bar);
        if (two) tma_load_1d(im + o, ra + n + o, bytes, bar);
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
    float xr[16], xi[16];
    fft8192_in_smem<false>(gr, gr + fft8k::kPlaneG, s, tb, t, [&] { fetch(it + 2, m + 2); }, [] {}, xr, xi);
    float2* o = out + (int64_t)m * kNbA;
#pragma unroll
    for (int q = 0; q < 16; ++q) o[t + 512 * q] = make_float2(xr[q], xi[q]);
  }
}

// The products of the bus on the block spectra, per bin pair (f, kNbA - f) and item.  Every operand is untangled into
// the spectra of its real rows (X_s: input s, H_so: IR row s O + o, G_o: output gradient o), and every result is stored
// packed two real rows per block, planar, scaled by `scale`:
//   BUS_FWD: Y_o[i] = sum_s sum_j X_s[i - j] H_so[j]                       out: I blocks (Y_0 + i Y_1)
//   BUS_DX:  D_s[i] = sum_o sum_j G_o[i + j] conj(H_so[j]),  stored as W_s[i] = D_s[i] + (-1)^f D_s[i + 1]: the inverse
//            of W_s[i] has, in its second half, the second half of D_s[i]'s inverse plus the first half of D_s[i + 1]'s
//            (a circular shift by kB is the factor (-1)^f), i.e. dL/dx_s on samples [i kB, (i+1) kB) with the
//            overlap-add already done                                   out: P I blocks (W_2p + i W_2p+1)
//   BUS_DIR: E_so[j] = sum_i G_o[j + i] conj(X_s[i])                         out: NH J blocks (set k: rows 2k, 2k + 1)
// X: P I blocks per item; H: NH J blocks per IR at item stride hstride (0: one IR for the batch); G: I blocks per item.
// MAXB > 0 caches the block operands of one input in registers (I, J <= MAXB) and loops over the inputs with the
// accumulators held; MAXB == 0 reads every operand from L2.
enum BusMac { BUS_FWD, BUS_DX, BUS_DIR };
// bus_mac_kernel's emit and axpy as functions, for busmc_mac_kernel, at bins (f, fm = kNbA - f) of one thread: real
// rows (a, b) packed planar into block `slot` of Out, scaled; and acc + (-1)^f v (sgn = (-1)^f).  bus_mac_kernel keeps
// its lambdas: calling these from them changes the code nvcc generates for its dL/dx instantiations.
__device__ __forceinline__ void bus_emit(float2* Out, int64_t slot, int f, int fm, float scale, float2 a, float2 b) {
  a.x *= scale; a.y *= scale; b.x *= scale; b.y *= scale;
  float* pl = reinterpret_cast<float*>(Out + slot * kNbA);
  pl[f] = a.x - b.y; pl[kNbA + f] = a.y + b.x;
  if (fm != f) { pl[fm] = a.x + b.y; pl[kNbA + fm] = b.x - a.y; }
}
__device__ __forceinline__ float2 bus_axpy(float sgn, float2 acc, float2 v) {
  return make_float2(fmaf(sgn, v.x, acc.x), fmaf(sgn, v.y, acc.y));
}
template <int MAXB, int MODE, int O>
__global__ void __launch_bounds__(128) bus_mac_kernel(const float2* __restrict__ X, const float2* __restrict__ H,
                                                      int64_t hstride, const float2* __restrict__ G,
                                                      float2* __restrict__ Out, int S, int I, int J, float scale) {
  constexpr int M = MAXB > 0 ? MAXB : 1;
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f > kNbA / 2) return;
  const int fm = (kNbA - f) & (kNbA - 1);
  const int64_t il = blockIdx.y;
  const int P = (S + 1) / 2, NH = (S * O + 1) / 2;
  const float2* x = X + il * (int64_t)P * I * kNbA;
  const float2* h = H + il * hstride;
  const float2* g = G + il * (int64_t)I * kNbA;
  const float2 zero = make_float2(0.f, 0.f);
  auto pair = [&](const float2* base, int64_t slot, float2& a, float2& b) {
    untangle(base[slot * kNbA + f], base[slot * kNbA + fm], a, b);
  };
  // input s at block i
  auto xin = [&](int s, int i) -> float2 {
    float2 a, b;
    pair(x, (int64_t)(s >> 1) * I + i, a, b);
    return (s & 1) ? b : a;
  };
  // IR rows (s, 0) and (s, 1) (O == 2), or row s (O == 1) at partition j
  auto hin = [&](int s, int j, float2& h0, float2& h1) {
    if (O == 2) { pair(h, (int64_t)s * J + j, h0, h1); }
    else { float2 a, b; pair(h, (int64_t)(s >> 1) * J + j, a, b); h0 = (s & 1) ? b : a; h1 = zero; }
  };
  auto gin = [&](int i, float2& g0, float2& g1) { pair(g, i, g0, g1); };
  // packed planar store of real rows (a, b) into block `slot` of Out (item-local index `slot` of the item's blocks)
  auto emit = [&](int64_t slot, float2 a, float2 b) {
    a.x *= scale; a.y *= scale; b.x *= scale; b.y *= scale;
    float* pl = reinterpret_cast<float*>(Out + slot * kNbA);
    pl[f] = a.x - b.y; pl[kNbA + f] = a.y + b.x;
    if (fm != f) { pl[fm] = a.x + b.y; pl[kNbA + fm] = b.x - a.y; }
  };
  const float sgn = (f & 1) ? -1.f : 1.f;
  auto axpy = [&](float2 acc, float2 v) { return make_float2(fmaf(sgn, v.x, acc.x), fmaf(sgn, v.y, acc.y)); };

  if constexpr (MODE == BUS_FWD) {
    const int64_t ob = il * (int64_t)I;
    if constexpr (MAXB > 0) {
      float2 y0[M], y1[M];
#pragma unroll
      for (int o = 0; o < M; ++o) y0[o] = y1[o] = zero;
      for (int s = 0; s < S; ++s) {
        float2 xv[M], h0[M], h1[M];
#pragma unroll
        for (int i = 0; i < M; ++i) {
          xv[i] = h0[i] = h1[i] = zero;                // operands beyond I / J are zero
          if (i < I) xv[i] = xin(s, i);
          if (i < J) hin(s, i, h0[i], h1[i]);
        }
#pragma unroll
        for (int o = 0; o < M; ++o) {
#pragma unroll
          for (int j = 0; j <= o; ++j) {
            cfma(y0[o], xv[o - j], h0[j]);
            if (O == 2) cfma(y1[o], xv[o - j], h1[j]);
          }
        }
      }
#pragma unroll
      for (int o = 0; o < M; ++o)
        if (o < I) emit(ob + o, y0[o], y1[o]);
    } else {
      for (int o = 0; o < I; ++o) {
        float2 y0 = zero, y1 = zero;
        for (int s = 0; s < S; ++s) {
          for (int j = 0; j <= o && j < J; ++j) {
            float2 h0, h1;
            hin(s, j, h0, h1);
            const float2 xv = xin(s, o - j);
            cfma(y0, xv, h0);
            if (O == 2) cfma(y1, xv, h1);
          }
        }
        emit(ob + o, y0, y1);
      }
    }
  } else if constexpr (MODE == BUS_DX) {
    const int64_t ob = il * (int64_t)P * I;
    if constexpr (MAXB > 0) {
      float2 g0[M], g1[M];
#pragma unroll
      for (int i = 0; i < M; ++i) {
        g0[i] = g1[i] = zero;
        if (i < I) gin(i, g0[i], g1[i]);
      }
      for (int p = 0; p < P; ++p) {
        // source 2p: W into wa (folded in place, ascending); source 2p + 1: D in descending order, W emitted with wa
        float2 wa[M], h0[M], h1[M];
#pragma unroll
        for (int j = 0; j < M; ++j) {
          h0[j] = h1[j] = zero;
          if (j < J) hin(2 * p, j, h0[j], h1[j]);
        }
#pragma unroll
        for (int i = 0; i < M; ++i) {
          wa[i] = zero;
#pragma unroll
          for (int j = 0; i + j < M; ++j) {
            cfma_conj(wa[i], g0[i + j], h0[j]);
            if (O == 2) cfma_conj(wa[i], g1[i + j], h1[j]);
          }
        }
#pragma unroll
        for (int i = 0; i + 1 < M; ++i) wa[i] = axpy(wa[i], wa[i + 1]);
        const bool two = 2 * p + 1 < S;
#pragma unroll
        for (int j = 0; j < M; ++j) {
          h0[j] = h1[j] = zero;
          if (two && j < J) hin(2 * p + 1, j, h0[j], h1[j]);
        }
        float2 next = zero;                            // D_b[i + 1]
#pragma unroll
        for (int i = M - 1; i >= 0; --i) {
          float2 d = zero;
#pragma unroll
          for (int j = 0; i + j < M; ++j) {
            cfma_conj(d, g0[i + j], h0[j]);
            if (O == 2) cfma_conj(d, g1[i + j], h1[j]);
          }
          if (i < I) emit(ob + (int64_t)p * I + i, wa[i], axpy(d, next));
          next = d;
        }
      }
    } else {
      for (int p = 0; p < P; ++p) {
        for (int i = 0; i < I; ++i) {
          float2 w[2] = {zero, zero};
          for (int c = 0; c < 2 && 2 * p + c < S; ++c) {
            for (int q = i; q < i + 2 && q < I; ++q) {   // D_s[i] + (-1)^f D_s[i + 1]
              float2 d = zero;
              for (int j = 0; j < J && q + j < I; ++j) {
                float2 g0v, g1v, h0, h1;
                gin(q + j, g0v, g1v);
                hin(2 * p + c, j, h0, h1);
                cfma_conj(d, g0v, h0);
                if (O == 2) cfma_conj(d, g1v, h1);
              }
              w[c] = q == i ? d : axpy(w[c], d);
            }
          }
          emit(ob + (int64_t)p * I + i, w[0], w[1]);
        }
      }
    }
  } else {
    static_assert(MODE == BUS_DIR, "bus_mac_kernel: unknown mode");
    const int64_t ob = il * (int64_t)NH * J;
    if constexpr (MAXB > 0) {
      float2 g0[M], g1[M];
#pragma unroll
      for (int i = 0; i < M; ++i) {
        g0[i] = g1[i] = zero;
        if (i < I) gin(i, g0[i], g1[i]);
      }
      for (int p = 0; p < P; ++p) {
        float2 xa[M], xb[M];
#pragma unroll
        for (int i = 0; i < M; ++i) {
          xa[i] = xb[i] = zero;
          if (i < I) pair(x, (int64_t)p * I + i, xa[i], xb[i]);
        }
        const bool two = 2 * p + 1 < S;
#pragma unroll
        for (int j = 0; j < M; ++j) {
          if (j < J) {
            float2 e00 = zero, e01 = zero, e10 = zero, e11 = zero;   // E_{2p+c, o} = e_co
#pragma unroll
            for (int i = 0; i + j < M; ++i) {
              cfma_conj(e00, g0[j + i], xa[i]);
              cfma_conj(e10, g0[j + i], xb[i]);
              if (O == 2) { cfma_conj(e01, g1[j + i], xa[i]); cfma_conj(e11, g1[j + i], xb[i]); }
            }
            if (O == 2) {
              emit(ob + (int64_t)(2 * p) * J + j, e00, e01);
              if (two) emit(ob + (int64_t)(2 * p + 1) * J + j, e10, e11);
            } else {
              emit(ob + (int64_t)p * J + j, e00, two ? e10 : zero);
            }
          }
        }
      }
    } else {
      for (int p = 0; p < P; ++p) {
        const bool two = 2 * p + 1 < S;
        for (int j = 0; j < J; ++j) {
          float2 e00 = zero, e01 = zero, e10 = zero, e11 = zero;
          for (int i = 0; i + j < I; ++i) {
            float2 g0v, g1v, xa, xb;
            gin(j + i, g0v, g1v);
            pair(x, (int64_t)p * I + i, xa, xb);
            cfma_conj(e00, g0v, xa);
            cfma_conj(e10, g0v, xb);
            if (O == 2) { cfma_conj(e01, g1v, xa); cfma_conj(e11, g1v, xb); }
          }
          if (O == 2) {
            emit(ob + (int64_t)(2 * p) * J + j, e00, e01);
            if (two) emit(ob + (int64_t)(2 * p + 1) * J + j, e10, e11);
          } else {
            emit(ob + (int64_t)p * J + j, e00, two ? e10 : zero);
          }
        }
      }
    }
  }
}

// bus_emit's second row: adds real row b to a block bus_emit stored with b = 0 (the same thread, the same bins), which
// leaves the bits of bus_emit(a, b)
__device__ __forceinline__ void bus_emit_add(float2* Out, int64_t slot, int f, int fm, float scale, float2 b) {
  b.x *= scale; b.y *= scale;
  float* pl = reinterpret_cast<float*>(Out + slot * kNbA);
  pl[f] -= b.y; pl[kNbA + f] += b.x;
  if (fm != f) { pl[fm] += b.y; pl[kNbA + fm] += b.x; }
}

// The bus products for M >= 3 outputs (multichannel_convolution), the operands and results of bus_mac_kernel with the
// outputs in Q = ceil(M / 2) packed pairs: IR row s M + m is row (s M + m) & 1 of partition set (s M + m) >> 1, and
// output / gradient pair q of block i is block q I + i of the item.  One slice of an item per blockIdx.y, the items
// along blockIdx.z, so the slices of an item run next to each other and re-read its spectra from L2:
//   BUS_FWD: slice q < Q:   Y_2q[i], Y_2q+1[i], as the O = 2 body                      out: Q I blocks (Y_2q + i Y_2q+1)
//   BUS_DX:  slice p < P:   W_2p[i], W_2p+1[i] (bus_mac_kernel's), D_s summed over the Q output pairs; source 2p + 1
//                           is added to the stored source 2p (bus_emit_add)            out: P I blocks
//   BUS_DIR: slice k < NH:  E of rows 2k and 2k + 1, each an (s, m)                    out: NH J blocks
// MAXB > 0 caches the blocks of one (input, output pair) in registers (I, J <= MAXB); MAXB == 0 reads from L2.
template <int MAXB, int MODE>
__global__ void __launch_bounds__(128) busmc_mac_kernel(const float2* __restrict__ X, const float2* __restrict__ H,
                                                        int64_t hstride, const float2* __restrict__ G,
                                                        float2* __restrict__ Out, int S, int M, int I, int J,
                                                        float scale) {
  constexpr int MB = MAXB > 0 ? MAXB : 1;
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f > kNbA / 2) return;
  const int fm = (kNbA - f) & (kNbA - 1);
  const int sl = blockIdx.y;
  const int64_t il = blockIdx.z;
  const int P = (S + 1) / 2, Q = (M + 1) / 2, NH = (S * M + 1) / 2;
  const float2* x = X + il * (int64_t)P * I * kNbA;
  const float2* h = H + il * hstride;
  const float2* g = G + il * (int64_t)Q * I * kNbA;
  const float2 zero = make_float2(0.f, 0.f);
  auto pair = [&](const float2* base, int64_t slot, float2& a, float2& b) {
    untangle(base[slot * kNbA + f], base[slot * kNbA + fm], a, b);
  };
  auto pick = [&](const float2* base, int64_t set, int odd) -> float2 {
    float2 a, b;
    pair(base, set, a, b);
    return odd ? b : a;
  };
  // input s at block i; IR row r at partition j; gradient row m at block i
  auto xin = [&](int s, int i) { return pick(x, (int64_t)(s >> 1) * I + i, s & 1); };
  auto hrow = [&](int r, int j) { return pick(h, (int64_t)(r >> 1) * J + j, r & 1); };
  auto grow = [&](int m, int i) { return pick(g, (int64_t)(m >> 1) * I + i, m & 1); };
  // IR rows (s, 2q) and (s, 2q + 1) at partition j, 0 past the last output; one set when s M + 2q is even
  auto hin = [&](int s, int q, int j, float2& h0, float2& h1) {
    const int r = s * M + 2 * q;
    if (2 * q + 1 >= M) { h0 = hrow(r, j); h1 = zero; }
    else if ((r & 1) == 0) pair(h, (int64_t)(r >> 1) * J + j, h0, h1);
    else { h0 = hrow(r, j); h1 = hrow(r + 1, j); }
  };
  auto gin = [&](int q, int i, float2& g0, float2& g1) { pair(g, (int64_t)q * I + i, g0, g1); };
  auto emit = [&](int64_t slot, float2 a, float2 b) { bus_emit(Out, slot, f, fm, scale, a, b); };
  const float sgn = (f & 1) ? -1.f : 1.f;
  auto axpy = [&](float2 acc, float2 v) { return bus_axpy(sgn, acc, v); };

  if constexpr (MODE == BUS_FWD) {
    const int q = sl;
    const int64_t ob = (il * Q + q) * (int64_t)I;
    if constexpr (MAXB > 0) {
      float2 y0[MB], y1[MB];
#pragma unroll
      for (int o = 0; o < MB; ++o) y0[o] = y1[o] = zero;
      for (int s = 0; s < S; ++s) {
        float2 xv[MB], h0[MB], h1[MB];
#pragma unroll
        for (int i = 0; i < MB; ++i) {
          xv[i] = h0[i] = h1[i] = zero;                // operands beyond I / J are zero
          if (i < I) xv[i] = xin(s, i);
          if (i < J) hin(s, q, i, h0[i], h1[i]);
        }
#pragma unroll
        for (int o = 0; o < MB; ++o) {
#pragma unroll
          for (int j = 0; j <= o; ++j) {
            cfma(y0[o], xv[o - j], h0[j]);
            cfma(y1[o], xv[o - j], h1[j]);
          }
        }
      }
#pragma unroll
      for (int o = 0; o < MB; ++o)
        if (o < I) emit(ob + o, y0[o], y1[o]);
    } else {
      for (int o = 0; o < I; ++o) {
        float2 y0 = zero, y1 = zero;
        for (int s = 0; s < S; ++s) {
          for (int j = 0; j <= o && j < J; ++j) {
            float2 h0, h1;
            hin(s, q, j, h0, h1);
            const float2 xv = xin(s, o - j);
            cfma(y0, xv, h0);
            cfma(y1, xv, h1);
          }
        }
        emit(ob + o, y0, y1);
      }
    }
  } else if constexpr (MODE == BUS_DX) {
    const int p = sl;
    const int64_t ob = (il * P + p) * (int64_t)I;
    if constexpr (MAXB > 0) {
      for (int c = 0; c < 2 && 2 * p + c < S; ++c) {
        const int s = 2 * p + c;
        float2 d[MB];                                  // D_s, then W_s folded in place (ascending)
#pragma unroll
        for (int i = 0; i < MB; ++i) d[i] = zero;
        for (int q = 0; q < Q; ++q) {
          float2 g0[MB], g1[MB], h0[MB], h1[MB];
#pragma unroll
          for (int i = 0; i < MB; ++i) {
            g0[i] = g1[i] = h0[i] = h1[i] = zero;
            if (i < I) gin(q, i, g0[i], g1[i]);
            if (i < J) hin(s, q, i, h0[i], h1[i]);
          }
#pragma unroll
          for (int i = 0; i < MB; ++i) {
#pragma unroll
            for (int j = 0; i + j < MB; ++j) {
              cfma_conj(d[i], g0[i + j], h0[j]);
              cfma_conj(d[i], g1[i + j], h1[j]);
            }
          }
        }
#pragma unroll
        for (int i = 0; i + 1 < MB; ++i) d[i] = axpy(d[i], d[i + 1]);
#pragma unroll
        for (int i = 0; i < MB; ++i) {
          if (i < I) {
            if (c == 0) emit(ob + i, d[i], zero);
            else bus_emit_add(Out, ob + i, f, fm, scale, d[i]);
          }
        }
      }
    } else {
      for (int i = 0; i < I; ++i) {
        float2 w[2] = {zero, zero};
        for (int c = 0; c < 2 && 2 * p + c < S; ++c) {
          for (int b = i; b < i + 2 && b < I; ++b) {   // D_s[i] + (-1)^f D_s[i + 1]
            float2 d = zero;
            for (int q = 0; q < Q; ++q) {
              for (int j = 0; j < J && b + j < I; ++j) {
                float2 g0, g1, h0, h1;
                gin(q, b + j, g0, g1);
                hin(2 * p + c, q, j, h0, h1);
                cfma_conj(d, g0, h0);
                cfma_conj(d, g1, h1);
              }
            }
            w[c] = b == i ? d : axpy(w[c], d);
          }
        }
        emit(ob + i, w[0], w[1]);
      }
    }
  } else {
    static_assert(MODE == BUS_DIR, "busmc_mac_kernel: unknown mode");
    const int k = sl;
    const int r0 = 2 * k, r1 = 2 * k + 1;
    const bool two = r1 < S * M;
    const int s0 = r0 / M, m0 = r0 - s0 * M, s1 = r1 / M, m1 = r1 - s1 * M;
    const int64_t ob = (il * NH + k) * (int64_t)J;
    if constexpr (MAXB > 0) {
      // row 2k into ea, then row 2k + 1 with the operands of row 2k out of registers, emitted with ea
      float2 ea[MB], gv[MB], xv[MB];
#pragma unroll
      for (int i = 0; i < MB; ++i) {
        gv[i] = xv[i] = zero;
        if (i < I) { gv[i] = grow(m0, i); xv[i] = xin(s0, i); }
      }
#pragma unroll
      for (int j = 0; j < MB; ++j) {
        ea[j] = zero;
#pragma unroll
        for (int i = 0; i + j < MB; ++i) cfma_conj(ea[j], gv[j + i], xv[i]);
      }
#pragma unroll
      for (int i = 0; i < MB; ++i) {
        gv[i] = xv[i] = zero;
        if (two && i < I) { gv[i] = grow(m1, i); xv[i] = xin(s1, i); }
      }
#pragma unroll
      for (int j = 0; j < MB; ++j) {
        if (j < J) {
          float2 eb = zero;
#pragma unroll
          for (int i = 0; i + j < MB; ++i) cfma_conj(eb, gv[j + i], xv[i]);
          emit(ob + j, ea[j], eb);
        }
      }
    } else {
      for (int j = 0; j < J; ++j) {
        float2 ea = zero, eb = zero;
        for (int i = 0; i + j < I; ++i) {
          cfma_conj(ea, grow(m0, j + i), xin(s0, i));
          if (two) cfma_conj(eb, grow(m1, j + i), xin(s1, i));
        }
        emit(ob + j, ea, eb);
      }
    }
  }
}

// inverse transforms of packed planar block spectra into row pairs, runs of kConvRun units (il, k, q), il < items,
// k < groups, q < nblk: half `half` (0: the first, 1: the second kB outputs) of IFFT(Spl[unit]) is written as samples
// [q kB, (q+1) kB) ∩ [0, lim) of rows 2k (real part) and 2k + 1 (imaginary part, if 2k + 1 < rows) of the `rows` rows
// of length len of item item0 + il in dst.  The bus output and dL/dx (half 1, lim = len = n) and dL/dIR (half 0,
// lim = leff, len = L).
__global__ void __launch_bounds__(kFusedThreads, 1)
bus_ifft_kernel(const float* __restrict__ Spl, const float* __restrict__ twiddles, float* __restrict__ dst, int64_t item0,
                int rows, int groups, int nblk, int64_t len, int64_t lim, int half, int nunits) {
  extern __shared__ __align__(128) float sm[];
  FftSmem s(sm);
  const int t = threadIdx.x;
  s.init(twiddles, t);
  const fft8k::Tables tb = fft8k::carve_tables(s.tabf);
  const int m0 = blockIdx.x * kConvRun;
  const int m1 = nunits - m0 < kConvRun ? nunits : m0 + kConvRun;
  auto fetch = [&](int it, int m) {
    if (t == 0 && m < m1) s.load_planar(it, Spl + (int64_t)m * 2 * kNbA);
  };
  fetch(0, m0);
  fetch(1, m0 + 1);
  int it = 0;
  for (int m = m0; m < m1; ++m, ++it) {
    s.wait(it);
    float* gr = s.buf(it);
    float xr[16], xi[16];
    fft8192_in_smem<true>(gr, gr + fft8k::kPlaneG, s, tb, t, [&] { fetch(it + 2, m + 2); }, [] {}, xr, xi);
    const int u = m / nblk, q = m - u * nblk;      // u = il * groups + k
    const int64_t il = u / groups;
    const int k = u - (int)il * groups;
    const bool two = 2 * k + 1 < rows;
    float* ra = dst + ((item0 + il) * rows + 2 * k) * len;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      const int64_t tg = (int64_t)q * kB + t + 512 * c;
      if (tg < lim) {
        const float vr = half ? xr[c + 8] : xr[c], vi = half ? xi[c + 8] : xi[c];
        ra[tg] = vr;
        if (two) ra[len + tg] = vi;
      }
    }
  }
}

// ---- time_varying_convolution_reverberation: K IRs, IR k anchored at k hop, crossfaded linearly along the output ----
// hop = H kB, so output block i lies in anchor interval k = i / H.  Blocks i < nX = min(I, (K - 1) H) are crossfaded
// between IRs k and k + 1 with a = (t - k hop) / hop; later blocks carry IR K - 1 alone.  An item's product (forward)
// and gradient (backward) spectra are U = I + nX blocks:
//   forward  slot 2i + c (i < nX):  (Y_k,c[i], Y_k+1,c[i]) packed as real + i imag: one inverse gives output channel c
//                                   as (1 - a) real + a imag
//            slot nX + i (i >= nX): (Y_K-1,0[i], Y_K-1,1[i]): one inverse gives both channels, as ifft_mix_kernel
//   backward slot 2i (i < nX):      Ga[i] = FFT of [0 | (1 - a) g block i]  (L + i R)
//            slot 2i + 1:           Gb[i] = FFT of [0 | a g block i]
//            slot nX + i (i >= nX): G[i]  = FFT of [0 | g block i]
// The IR rows of an item are r = k C + c (C = 1 or 2 IR channels; a mono IR feeds both), packed two per partition set
// by ir_pack_kernel: set s = rows (2s, 2s + 1), an odd last row with 0.
__device__ __forceinline__ int tv_slot(int i, int nX) { return i < nX ? 2 * i : nX + i; }
// crossfade weight a of IR k + 1 at sample t of block i (t = i kB + u)
__device__ __forceinline__ float tv_a(int i, int H, int u, int64_t hop) {
  return (float)((int64_t)(i - (i / H) * H) * kB + u) / (float)hop;
}

// gradient transforms, runs of kConvRun units m = il U + s: bus_fft_kernel's half == 1 path (one gradient pair per
// unit) with the crossfade weight applied to the block in shared memory before the transform.  n % 4 == 0 and
// 16-byte aligned rows.
__global__ void __launch_bounds__(kFusedThreads, 1)
tv_fft_kernel(const float* __restrict__ gy, float2* __restrict__ Gb, const float* __restrict__ twiddles, int64_t item0,
              int I, int nX, int H, int64_t hop, int64_t n, int nunits) {
  extern __shared__ __align__(128) float sm[];
  FftSmem s(sm);
  const int t = threadIdx.x;
  s.init(twiddles, t);
  const fft8k::Tables tb = fft8k::carve_tables(s.tabf);
  const int U = I + nX;
  const int m0 = blockIdx.x * kConvRun;
  const int m1 = nunits - m0 < kConvRun ? nunits : m0 + kConvRun;
  auto block = [&](int m, int& i, int& part) {     // part 0: 1 - a, 1: a, 2: no weight
    const int u = m - (m / U) * U;
    if (u < 2 * nX) { i = u >> 1; part = u & 1; }
    else { i = u - nX; part = 2; }
  };
  auto fetch = [&](int it, int m) {                // all threads: zero padding; thread 0: the bulk copies
    if (m >= m1) return;
    const int64_t il = m / U;
    int i, part;
    block(m, i, part);
    float* re = s.buf(it);
    float* im = re + fft8k::kPlaneG;
    const int64_t s0 = (int64_t)i * kB;
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
  fetch(0, m0);
  fetch(1, m0 + 1);
  __syncthreads();
  int it = 0;
  for (int m = m0; m < m1; ++m, ++it) {
    s.wait(it);
    float* gr = s.buf(it);
    float* gi = gr + fft8k::kPlaneG;
    int i, part;
    block(m, i, part);
    if (part < 2) {                                // uniform over the CTA
      for (int e = t; e < kB; e += kFusedThreads) {
        const float a = tv_a(i, H, e, hop);
        const float w = part ? a : 1.0f - a;
        gr[kB + e] *= w;
        gi[kB + e] *= w;
      }
      __syncthreads();
    }
    float xr[16], xi[16];
    fft8192_in_smem<false>(gr, gi, s, tb, t, [&] { fetch(it + 2, m + 2); }, [] {}, xr, xi);
    float2* out = Gb + (int64_t)m * kNbA;
#pragma unroll
    for (int q = 0; q < 16; ++q) out[t + 512 * q] = make_float2(xr[q], xi[q]);
  }
}

// inverse transforms of the product slots, runs of kConvRun units m = il U + s, with ifft_mix_kernel's crop and
// dry/wet mix and the crossfade in the epilogue: y_c = (1 - mix) x_c + mix wet_c on samples [i kB, (i+1) kB) ∩ [0, n).
__global__ void __launch_bounds__(kFusedThreads, 1)
tv_ifft_kernel(const float* __restrict__ Ypl, const float* __restrict__ twiddles, const float* __restrict__ x,
               const float* __restrict__ mix_p, float* __restrict__ y, int64_t item0, int I, int nX, int H, int64_t hop,
               int64_t n, int in_chs, int nunits) {
  extern __shared__ __align__(128) float sm[];
  FftSmem s(sm);
  const int t = threadIdx.x;
  s.init(twiddles, t);
  const fft8k::Tables tb = fft8k::carve_tables(s.tabf);
  const int U = I + nX;
  const int m0 = blockIdx.x * kConvRun;
  const int m1 = nunits - m0 < kConvRun ? nunits : m0 + kConvRun;
  auto fetch = [&](int it, int m) {
    if (t == 0 && m < m1) s.load_planar(it, Ypl + (int64_t)m * 2 * kNbA);
  };
  fetch(0, m0);
  fetch(1, m0 + 1);
  int it = 0;
  for (int m = m0; m < m1; ++m, ++it) {
    s.wait(it);
    float* gr = s.buf(it);
    const int64_t il = m / U, b = item0 + il;
    const int u = m - (int)il * U;
    const bool cross = u < 2 * nX;                 // uniform over the CTA
    const int i = cross ? u >> 1 : u - nX, c = cross ? u & 1 : 0;
    const float mix = mix_p[b];
    const float* xl = x + (b * in_chs) * n;
    const float* xrr = in_chs == 1 ? xl : xl + n;
    float a0[8], a1[8];                            // the dry samples of this thread's 8 outputs
    float xr[16], xi[16];
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
      const int e = t + 512 * q - kB;
      const int64_t tg = (int64_t)i * kB + e;
      if (tg < n) {
        if (cross) {
          const float a = tv_a(i, H, e, hop);
          const float wet = fmaf(a, xi[q], (1.0f - a) * xr[q]);
          const float dry = c ? a1[q - 8] : a0[q - 8];
          y[(b * 2 + c) * n + tg] = fmaf(mix, wet - dry, dry);
        } else {
          y[(b * 2 + 0) * n + tg] = fmaf(mix, xr[q] - a0[q - 8], a0[q - 8]);
          y[(b * 2 + 1) * n + tg] = fmaf(mix, xi[q] - a1[q - 8], a1[q - 8]);
        }
      }
    }
  }
}

// The products of the time-varying convolution per bin pair (f, kNbA - f) and item, every operand untangled into the
// spectra of its real rows (X_c: audio channel c, H_k,c: IR k's channel c, G: the gradient slots), results packed two
// real rows per block, planar, scaled by 1 / kNbA; all operands from L2.
//   TV_FWD: Y_k,c[i] = sum_j X_c[i - j] H_k,c[j] for the IRs of block i          out: U slots per item (see above)
//   TV_DX:  D_c[m] = sum_j Ga_c[m+j] conj(H_k(m+j),c[j]) + Gb_c[m+j] conj(H_k(m+j)+1,c[j])
//                                                                                out: I blocks per item (D_0 + i D_1)
//   TV_DIR: E_k,c[j] = sum_{i in interval k} Ga_c[i] conj(X_c[i-j]) + sum_{i in interval k-1} Gb_c[i] conj(X_c[i-j]),
//           times mix[b] when mix is not null (a shared trajectory's factors are applied by irgrad_sum_kernel); a mono
//           IR row k receives E_k,0 + E_k,1                                     out: sets J blocks per item
// H: sets J partitions per trajectory at item stride hstride (0: one trajectory for the batch).
enum TvMac { TV_FWD, TV_DX, TV_DIR };
template <int MODE, int C>
__global__ void __launch_bounds__(128) tv_mac_kernel(const float2* __restrict__ X, const float2* __restrict__ H,
                                                     int64_t hstride, const float2* __restrict__ G,
                                                     const float* __restrict__ mix, float2* __restrict__ Out,
                                                     int64_t item0, int I, int J, int K, int nX, int Hb, int sets) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f > kNbA / 2) return;
  const int fm = (kNbA - f) & (kNbA - 1);
  const int64_t il = blockIdx.y;
  const int U = I + nX;
  const float2* x = X + il * (int64_t)I * kNbA;
  const float2* h = H + il * hstride;
  const float2* g = G + il * (int64_t)U * kNbA;
  const float2 zero = make_float2(0.f, 0.f);
  auto pair = [&](const float2* base, int64_t slot, float2& a, float2& b) {
    untangle(base[slot * kNbA + f], base[slot * kNbA + fm], a, b);
  };
  auto hin = [&](int k, int j, float2& h0, float2& h1) {     // IR k at partition j, channels 0 and 1
    if (C == 2) { pair(h, (int64_t)k * J + j, h0, h1); }
    else { float2 a, b; pair(h, (int64_t)(k >> 1) * J + j, a, b); h0 = h1 = (k & 1) ? b : a; }
  };
  const float scale = 1.0f / (float)kNbA;
  auto emit = [&](int64_t slot, float2 a, float2 b, float sc) {
    a.x *= sc; a.y *= sc; b.x *= sc; b.y *= sc;
    float* pl = reinterpret_cast<float*>(Out + slot * kNbA);
    pl[f] = a.x - b.y; pl[kNbA + f] = a.y + b.x;
    if (fm != f) { pl[fm] = a.x + b.y; pl[kNbA + fm] = b.x - a.y; }
  };
  auto ival = [&](int i) { const int k = i / Hb; return k < K - 1 ? k : K - 1; };   // anchor interval of block i

  if constexpr (MODE == TV_FWD) {
    for (int o = 0; o < I; ++o) {
      const int k = ival(o);
      const bool cross = o < nX;
      float2 y0 = zero, y1 = zero, z0 = zero, z1 = zero;    // IR k: channels 0, 1; IR k + 1: channels 0, 1
      for (int j = 0; j <= o && j < J; ++j) {
        float2 x0, x1, h0, h1;
        pair(x, o - j, x0, x1);
        hin(k, j, h0, h1);
        cfma(y0, x0, h0);
        cfma(y1, x1, h1);
        if (cross) {
          hin(k + 1, j, h0, h1);
          cfma(z0, x0, h0);
          cfma(z1, x1, h1);
        }
      }
      const int64_t ob = il * (int64_t)U;
      if (cross) { emit(ob + 2 * o, y0, z0, scale); emit(ob + 2 * o + 1, y1, z1, scale); }
      else emit(ob + nX + o, y0, y1, scale);
    }
  } else if constexpr (MODE == TV_DX) {
    for (int m = 0; m < I; ++m) {
      float2 d0 = zero, d1 = zero;
      for (int j = 0; j < J && m + j < I; ++j) {
        const int i = m + j, k = ival(i);
        float2 g0, g1, h0, h1;
        pair(g, tv_slot(i, nX), g0, g1);
        hin(k, j, h0, h1);
        cfma_conj(d0, g0, h0);
        cfma_conj(d1, g1, h1);
        if (i < nX) {
          pair(g, 2 * i + 1, g0, g1);
          hin(k + 1, j, h0, h1);
          cfma_conj(d0, g0, h0);
          cfma_conj(d1, g1, h1);
        }
      }
      emit(il * (int64_t)I + m, d0, d1, scale);
    }
  } else {
    static_assert(MODE == TV_DIR, "tv_mac_kernel: unknown mode");
    const float sc = mix ? mix[item0 + il] * scale : scale;
    // E_k,c[j] over both intervals that carry IR k
    auto ecorr = [&](int k, int j, float2& e0, float2& e1) {
      e0 = e1 = zero;
      for (int part = 0; part < 2; ++part) {       // 0: Ga of interval k, 1: Gb of interval k - 1
        const int kk = k - part;
        if (kk < 0) continue;
        const int lo = kk * Hb, hi = kk == K - 1 ? I : ((kk + 1) * Hb < I ? (kk + 1) * Hb : I);
        for (int i = lo > j ? lo : j; i < hi; ++i) {
          float2 g0, g1, x0, x1;
          pair(g, part ? 2 * i + 1 : tv_slot(i, nX), g0, g1);
          pair(x, i - j, x0, x1);
          cfma_conj(e0, g0, x0);
          cfma_conj(e1, g1, x1);
        }
      }
    };
    const int64_t ob = il * (int64_t)sets * J;
    for (int sI = 0; sI < sets; ++sI) {
      for (int j = 0; j < J; ++j) {
        float2 e0, e1;
        if (C == 2) {
          ecorr(sI, j, e0, e1);
          emit(ob + (int64_t)sI * J + j, e0, e1, sc);
        } else {
          float2 p0, p1, q = zero;
          ecorr(2 * sI, j, p0, p1);
          if (2 * sI + 1 < K) {
            ecorr(2 * sI + 1, j, e0, e1);
            q = make_float2(e0.x + e1.x, e0.y + e1.y);
          }
          emit(ob + (int64_t)sI * J + j, make_float2(p0.x + p1.x, p0.y + p1.y), q, sc);
        }
      }
    }
  }
}

// ---- time_varying_convolution_bus: S sources, each with its own IR trajectory, crossfaded and summed into O outputs --
// The bus's packing (the S inputs in P = ceil(S / 2) window spectra per block, bus_fft_kernel's; the K S O IR rows
// r = (k S + s) O + o in NH = ceil(K S O / 2) partition sets, set q = rows 2q, 2q + 1, an odd last row with 0) on the
// time-varying op's anchor grid (hop = H kB: blocks i < nX = (K - 1) H are crossfaded between IR sets k = i / H and
// k + 1).  Product (forward) and gradient (backward) slots per item:
//   O = 2: U = I + nX, the time-varying op's layout (tv_slot): slot 2i + o (i < nX) holds (Y_k,o[i], Y_k+1,o[i]), slot
//          nX + i (i >= nX) holds (Y_K-1,0[i], Y_K-1,1[i]); the gradient slots are tv_fft_kernel's.
//   O = 1: U = I: slot i holds (Y_k[i], Y_k+1[i]) for i < nX and (Y_K-1[i], 0) after; the gradient slot i is the FFT of
//          [0 | (1 - a) g + i a g] for i < nX and of [0 | g] after (tvbus_gfft_kernel).
// So one inverse transform yields one crossfaded output row (O = 2) or one output block (O = 1).

// gradient transforms of a mono bus, runs of kConvRun units m = il I + i: tv_fft_kernel with one gradient row, whose
// block carries the weight 1 - a in the real and a in the imaginary plane (one transform for both IR sets of the
// block).  n % 4 == 0 and 16-byte aligned rows.
__global__ void __launch_bounds__(kFusedThreads, 1)
tvbus_gfft_kernel(const float* __restrict__ gy, float2* __restrict__ Gb, const float* __restrict__ twiddles,
                  int64_t item0, int I, int nX, int H, int64_t hop, int64_t n, int nunits) {
  extern __shared__ __align__(128) float sm[];
  FftSmem s(sm);
  const int t = threadIdx.x;
  s.init(twiddles, t);
  const fft8k::Tables tb = fft8k::carve_tables(s.tabf);
  const int m0 = blockIdx.x * kConvRun;
  const int m1 = nunits - m0 < kConvRun ? nunits : m0 + kConvRun;
  auto fetch = [&](int it, int m) {                // all threads: zero padding and the im plane; thread 0: the copy
    if (m >= m1) return;
    const int64_t il = m / I;
    const int i = m - (int)il * I;
    float* re = s.buf(it);
    float* im = re + fft8k::kPlaneG;
    const int64_t s0 = (int64_t)i * kB;
    const int64_t rem = n - s0;
    const int len = rem < kB ? (int)rem : kB;
    for (int e = t; e < kB; e += kFusedThreads) re[e] = 0.f;
    for (int e = kB + len + t; e < kNbA; e += kFusedThreads) re[e] = 0.f;
    for (int e = t; e < kNbA; e += kFusedThreads) im[e] = 0.f;
    if (t == 0) {
      uint64_t* bar = &s.full[it & 1];
      mbar_arrive_expect_tx(bar, (uint32_t)len * 4u);
      tma_load_1d(re + kB, gy + (item0 + il) * n + s0, (uint32_t)len * 4u, bar);
    }
  };
  fetch(0, m0);
  fetch(1, m0 + 1);
  __syncthreads();
  int it = 0;
  for (int m = m0; m < m1; ++m, ++it) {
    s.wait(it);
    float* gr = s.buf(it);
    float* gi = gr + fft8k::kPlaneG;
    const int i = m - (m / I) * I;
    if (i < nX) {                                  // uniform over the CTA
      for (int e = t; e < kB; e += kFusedThreads) {
        const float a = tv_a(i, H, e, hop);
        const float v = gr[kB + e];
        gr[kB + e] = (1.0f - a) * v;
        gi[kB + e] = a * v;
      }
      __syncthreads();
    }
    float xr[16], xi[16];
    fft8192_in_smem<false>(gr, gi, s, tb, t, [&] { fetch(it + 2, m + 2); }, [] {}, xr, xi);
    float2* out = Gb + (int64_t)m * kNbA;
#pragma unroll
    for (int q = 0; q < 16; ++q) out[t + 512 * q] = make_float2(xr[q], xi[q]);
  }
}

// inverse transforms of the bus's product slots, runs of kConvRun units m = il U + u, with the crossfade and the crop in
// the epilogue (tv_ifft_kernel without the dry path): a crossfaded slot gives (1 - a) re + a im on samples
// [i kB, (i+1) kB) ∩ [0, n) of output row o (O = 2: o = u & 1; O = 1: the one row); a later slot gives rows 0 and 1 as
// re and im (O = 2) or row 0 as re (O = 1).
__global__ void __launch_bounds__(kFusedThreads, 1)
tvbus_ifft_kernel(const float* __restrict__ Ypl, const float* __restrict__ twiddles, float* __restrict__ y,
                  int64_t item0, int I, int nX, int H, int64_t hop, int64_t n, int O, int nunits) {
  extern __shared__ __align__(128) float sm[];
  FftSmem s(sm);
  const int t = threadIdx.x;
  s.init(twiddles, t);
  const fft8k::Tables tb = fft8k::carve_tables(s.tabf);
  const int U = O == 2 ? I + nX : I;
  const int m0 = blockIdx.x * kConvRun;
  const int m1 = nunits - m0 < kConvRun ? nunits : m0 + kConvRun;
  auto fetch = [&](int it, int m) {
    if (t == 0 && m < m1) s.load_planar(it, Ypl + (int64_t)m * 2 * kNbA);
  };
  fetch(0, m0);
  fetch(1, m0 + 1);
  int it = 0;
  for (int m = m0; m < m1; ++m, ++it) {
    s.wait(it);
    float* gr = s.buf(it);
    const int64_t il = m / U, b = item0 + il;
    const int u = m - (int)il * U;
    const bool cross = O == 2 ? u < 2 * nX : u < nX;                  // uniform over the CTA
    const int i = O == 2 ? (cross ? u >> 1 : u - nX) : u;
    const int o = O == 2 && cross ? u & 1 : 0;
    float xr[16], xi[16];
    fft8192_in_smem<true>(gr, gr + fft8k::kPlaneG, s, tb, t, [&] { fetch(it + 2, m + 2); }, [] {}, xr, xi);
    float* yo = y + (b * O + o) * n;
#pragma unroll
    for (int q = 8; q < 16; ++q) {                 // outputs kB .. 2 kB - 1 of the transform
      const int e = t + 512 * q - kB;
      const int64_t tg = (int64_t)i * kB + e;
      if (tg < n) {
        if (cross) {
          const float a = tv_a(i, H, e, hop);
          yo[tg] = fmaf(a, xi[q], (1.0f - a) * xr[q]);
        } else {
          yo[tg] = xr[q];
          if (O == 2) yo[n + tg] = xi[q];
        }
      }
    }
  }
}

// The products of the time-varying bus per bin pair (f, kNbA - f) and item, every operand untangled into the spectra
// of its real rows (X_s: source s, H_k,s,o: IR row (k S + s) O + o, Ga_o / Gb_o: the gradient of output o weighted
// 1 - a / a, G_o for a block after the last anchor), results packed two real rows per block, planar, scaled by
// 1 / kNbA; all operands from L2.
//   TVB_FWD: Y_k,o[i] = sum_s sum_j X_s[i - j] H_k,s,o[j] for the IR sets of block i        out: U slots (see above)
//   TVB_DX:  D_s[m] = sum_o sum_j Ga_o[m+j] conj(H_k(m+j),s,o[j]) + Gb_o[m+j] conj(H_k(m+j)+1,s,o[j]), stored as
//            bus_mac_kernel's W_s[m] = D_s[m] + (-1)^f D_s[m + 1] (bus_ifft_kernel's half 1 then writes dL/dx_s with
//            the overlap-add done)                                                   out: P I blocks (W_2p + i W_2p+1)
//   TVB_DIR: E_k,s,o[j] = sum_{i in interval k} Ga_o[i] conj(X_s[i-j]) + sum_{i in interval k-1} Gb_o[i] conj(X_s[i-j])
//                                                                                    out: NH J blocks (set q: rows 2q, 2q+1)
// X: P I blocks per item; H: NH J partitions per trajectory set at item stride hstride (0: one set for the batch);
// G: U slots per item.
enum TvBusMac { TVB_FWD, TVB_DX, TVB_DIR };
template <int MODE, int O>
__global__ void __launch_bounds__(128) tvbus_mac_kernel(const float2* __restrict__ X, const float2* __restrict__ H,
                                                        int64_t hstride, const float2* __restrict__ G,
                                                        float2* __restrict__ Out, int S, int I, int J, int K, int nX,
                                                        int Hb) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f > kNbA / 2) return;
  const int fm = (kNbA - f) & (kNbA - 1);
  const int64_t il = blockIdx.y;
  const int P = (S + 1) / 2, U = O == 2 ? I + nX : I;
  const float2* x = X + il * (int64_t)P * I * kNbA;
  const float2* h = H + il * hstride;
  const float2* g = G + il * (int64_t)U * kNbA;
  const float2 zero = make_float2(0.f, 0.f);
  auto pair = [&](const float2* base, int64_t slot, float2& a, float2& b) {
    untangle(base[slot * kNbA + f], base[slot * kNbA + fm], a, b);
  };
  // IR rows (k, s, 0) and (k, s, 1) (O == 2), or row (k, s) (O == 1), at partition j
  auto hin = [&](int k, int s, int j, float2& h0, float2& h1) {
    const int r = k * S + s;
    if (O == 2) { pair(h, (int64_t)r * J + j, h0, h1); }
    else { float2 a, b; pair(h, (int64_t)(r >> 1) * J + j, a, b); h0 = (r & 1) ? b : a; h1 = zero; }
  };
  // the gradient of block i for IR set k(i) (part 0: Ga, or G after the last anchor) or k(i) + 1 (part 1: Gb, i < nX),
  // outputs 0 and 1
  auto gin = [&](int i, int part, float2& g0, float2& g1) {
    if (O == 2) { pair(g, part ? 2 * i + 1 : tv_slot(i, nX), g0, g1); }
    else { float2 a, b; pair(g, i, a, b); g0 = part ? b : a; g1 = zero; }
  };
  const float scale = 1.0f / (float)kNbA;
  auto emit = [&](int64_t slot, float2 a, float2 b) {
    a.x *= scale; a.y *= scale; b.x *= scale; b.y *= scale;
    float* pl = reinterpret_cast<float*>(Out + slot * kNbA);
    pl[f] = a.x - b.y; pl[kNbA + f] = a.y + b.x;
    if (fm != f) { pl[fm] = a.x + b.y; pl[kNbA + fm] = b.x - a.y; }
  };
  auto ival = [&](int i) { const int k = i / Hb; return k < K - 1 ? k : K - 1; };   // anchor interval of block i

  if constexpr (MODE == TVB_FWD) {
    const int64_t ob = il * (int64_t)U;
    for (int o = 0; o < I; ++o) {
      const int k = ival(o);
      const bool cross = o < nX;
      float2 y0 = zero, y1 = zero, z0 = zero, z1 = zero;    // IR set k: outputs 0, 1; IR set k + 1: outputs 0, 1
      for (int p = 0; p < P; ++p) {
        const int nc = 2 * p + 1 < S ? 2 : 1;
        for (int j = 0; j <= o && j < J; ++j) {
          float2 xv[2], h0, h1;
          pair(x, (int64_t)p * I + o - j, xv[0], xv[1]);
          for (int c = 0; c < nc; ++c) {
            hin(k, 2 * p + c, j, h0, h1);
            cfma(y0, xv[c], h0);
            if (O == 2) cfma(y1, xv[c], h1);
            if (cross) {
              hin(k + 1, 2 * p + c, j, h0, h1);
              cfma(z0, xv[c], h0);
              if (O == 2) cfma(z1, xv[c], h1);
            }
          }
        }
      }
      if (O == 2) {
        if (cross) { emit(ob + 2 * o, y0, z0); emit(ob + 2 * o + 1, y1, z1); }
        else emit(ob + nX + o, y0, y1);
      } else {
        emit(ob + o, y0, z0);                      // z0 = 0 after the last anchor
      }
    }
  } else if constexpr (MODE == TVB_DX) {
    // D_2p+c[m], c = 0, 1 (d[1] stays 0 for an odd last source)
    auto dcorr = [&](int p, int m, float2 (&d)[2]) {
      d[0] = d[1] = zero;
      const int nc = 2 * p + 1 < S ? 2 : 1;
      for (int j = 0; j < J && m + j < I; ++j) {
        const int i = m + j, k = ival(i);
        for (int part = 0; part < (i < nX ? 2 : 1); ++part) {
          float2 g0, g1, h0, h1;
          gin(i, part, g0, g1);
          for (int c = 0; c < nc; ++c) {
            hin(k + part, 2 * p + c, j, h0, h1);
            cfma_conj(d[c], g0, h0);
            if (O == 2) cfma_conj(d[c], g1, h1);
          }
        }
      }
    };
    const float sgn = (f & 1) ? -1.f : 1.f;
    const int64_t ob = il * (int64_t)P * I;
    for (int p = 0; p < P; ++p) {
      float2 next[2] = {zero, zero};               // D[m + 1]
      for (int m = I - 1; m >= 0; --m) {
        float2 d[2];
        dcorr(p, m, d);
        emit(ob + (int64_t)p * I + m, make_float2(fmaf(sgn, next[0].x, d[0].x), fmaf(sgn, next[0].y, d[0].y)),
             make_float2(fmaf(sgn, next[1].x, d[1].x), fmaf(sgn, next[1].y, d[1].y)));
        next[0] = d[0]; next[1] = d[1];
      }
    }
  } else {
    static_assert(MODE == TVB_DIR, "tvbus_mac_kernel: unknown mode");
    // e[c][o] = E_k,2p+c,o[j] over both intervals that carry IR set k: each gradient and window-pair spectrum read
    // serves both sources of the pair
    auto ecorr = [&](int k, int p, int j, float2 (&e)[2][2]) {
      e[0][0] = e[0][1] = e[1][0] = e[1][1] = zero;
      for (int part = 0; part < 2; ++part) {       // 0: Ga (G) of interval k, 1: Gb of interval k - 1
        const int kk = k - part;
        if (kk < 0) continue;
        const int lo = kk * Hb, hi = kk == K - 1 ? I : ((kk + 1) * Hb < I ? (kk + 1) * Hb : I);
        for (int i = lo > j ? lo : j; i < hi; ++i) {
          float2 g0, g1, xa, xb;
          gin(i, part, g0, g1);
          pair(x, (int64_t)p * I + i - j, xa, xb);
          cfma_conj(e[0][0], g0, xa);
          cfma_conj(e[1][0], g0, xb);
          if (O == 2) { cfma_conj(e[0][1], g1, xa); cfma_conj(e[1][1], g1, xb); }
        }
      }
    };
    const int NH = (K * S * O + 1) / 2;
    const int64_t ob = il * (int64_t)NH * J;
    float2 e[2][2];
    if (O == 2 || S % 2 == 0) {
      // the sets of sources 2p, 2p + 1: k S + 2p + c (O = 2, rows o = 0, 1) or k S / 2 + p (O = 1, one row each)
      for (int k = 0; k < K; ++k) {
        for (int p = 0; p < P; ++p) {
          for (int j = 0; j < J; ++j) {
            ecorr(k, p, j, e);
            if (O == 2) {
              emit(ob + (int64_t)(k * S + 2 * p) * J + j, e[0][0], e[0][1]);
              if (2 * p + 1 < S) emit(ob + (int64_t)(k * S + 2 * p + 1) * J + j, e[1][0], e[1][1]);
            } else {
              emit(ob + (int64_t)(k * S / 2 + p) * J + j, e[0][0], e[1][0]);
            }
          }
        }
      }
    } else {
      // a mono bus of an odd number of sources: set q holds rows r = 2q, 2q + 1 (r = k S + s), which may belong to two
      // IR sets, so each row is formed on its own
      for (int q = 0; q < NH; ++q) {
        for (int j = 0; j < J; ++j) {
          float2 a, b = zero;
          ecorr((2 * q) / S, ((2 * q) % S) >> 1, j, e);
          a = e[((2 * q) % S) & 1][0];
          if (2 * q + 1 < K * S) {
            ecorr((2 * q + 1) / S, ((2 * q + 1) % S) >> 1, j, e);
            b = e[((2 * q + 1) % S) & 1][0];
          }
          emit(ob + (int64_t)q * J + j, a, b);
        }
      }
    }
  }
}

// ---- time_varying_convolution_bus, source-side crossfade: y_o = sum_k sum_s ((w_k x_s) * h_k,s,o) -------------------
// Every sample is heard through the IR sets of its emission time, its whole tail included.  Input block i lies in one
// anchor interval k = i / H (hop = H kB), where only w_k = 1 - a and w_k+1 = a are nonzero, so its weighted pieces are
// exact zero-padded transforms [0 | u]: no overlap-save window straddles an anchor.  The linear convolution of [0 | u]
// with a partition [h | 0] fills both halves of the circular result, and the first half belongs to the next output
// block, so the overlap-add is done on the spectra: W[m] = Y[m] + (-1)^f Y[m - 1] (a circular shift by kB is the factor
// (-1)^f), and output block m is the second half of W[m]'s inverse.  Window spectra per item, XW = nX S + (I - nX) P
// (nX = (K - 1) H crossfaded blocks, P = ceil(S / 2)):
//   slot i S + s (i < nX):                 FFT of [0 | (1 - a) x_s,i + i a x_s,i]: both IR sets' pieces of one source
//   slot nX S + (i - nX) P + p (i >= nX):  FFT of [0 | x_2p,i + i x_2p+1,i]: two sources, IR set K - 1
// The dL/dx spectra use the same slots.  The product and gradient spectra are one per block, both outputs packed.
__device__ __forceinline__ void tvin_block(int w, int S, int P, int nX, int& i, int& c) {   // slot w -> block, source|pair
  if (w < nX * S) { i = w / S; c = w - i * S; }
  else { const int r = w - nX * S; i = nX + r / P; c = r - (i - nX) * P; }
}

// window transforms of x, runs of kConvRun units m = il XW + w: tvbus_gfft_kernel's weighting prologue on one source's
// block (i < nX), bus_fft_kernel's zero-padded row pair after the last anchor.  n % 4 == 0 and 16-byte aligned rows.
__global__ void __launch_bounds__(kFusedThreads, 1)
tvbusin_fft_kernel(const float* __restrict__ x, float2* __restrict__ Xs, const float* __restrict__ twiddles,
                   int64_t item0, int S, int I, int nX, int H, int64_t hop, int64_t n, int nunits) {
  extern __shared__ __align__(128) float sm[];
  FftSmem s(sm);
  const int t = threadIdx.x;
  s.init(twiddles, t);
  const fft8k::Tables tb = fft8k::carve_tables(s.tabf);
  const int P = (S + 1) / 2, XW = nX * S + (I - nX) * P;
  const int m0 = blockIdx.x * kConvRun;
  const int m1 = nunits - m0 < kConvRun ? nunits : m0 + kConvRun;
  auto fetch = [&](int it, int m) {                // all threads: zero padding; thread 0: the bulk copies
    if (m >= m1) return;
    const int64_t il = m / XW;
    int i, c;
    tvin_block(m - (int)il * XW, S, P, nX, i, c);
    const bool cross = i < nX;
    const bool two = !cross && 2 * c + 1 < S;      // a second source in the imaginary plane
    float* re = s.buf(it);
    float* im = re + fft8k::kPlaneG;
    const int64_t s0 = (int64_t)i * kB;
    const int64_t rem = n - s0;
    const int len = rem < kB ? (int)rem : kB;      // kB for a crossfaded block
    for (int e = t; e < kB; e += kFusedThreads) { re[e] = 0.f; im[e] = 0.f; }
    for (int e = kB + len + t; e < kNbA; e += kFusedThreads) { re[e] = 0.f; im[e] = 0.f; }
    if (!cross && !two) for (int e = kB + t; e < kB + len; e += kFusedThreads) im[e] = 0.f;
    if (t == 0) {
      const float* ra = x + ((item0 + il) * S + (cross ? c : 2 * c)) * n + s0;
      uint64_t* bar = &s.full[it & 1];
      mbar_arrive_expect_tx(bar, (two ? 2u : 1u) * (uint32_t)len * 4u);
      tma_load_1d(re + kB, ra, (uint32_t)len * 4u, bar);
      if (two) tma_load_1d(im + kB, ra + n, (uint32_t)len * 4u, bar);
    }
  };
  fetch(0, m0);
  fetch(1, m0 + 1);
  __syncthreads();
  int it = 0;
  for (int m = m0; m < m1; ++m, ++it) {
    s.wait(it);
    float* gr = s.buf(it);
    float* gi = gr + fft8k::kPlaneG;
    const int w = m - (m / XW) * XW;
    if (w < nX * S) {                              // uniform over the CTA: a crossfaded block, im plane written here
      const int i = w / S;
      for (int e = t; e < kB; e += kFusedThreads) {
        const float a = tv_a(i, H, e, hop);
        const float v = gr[kB + e];
        gr[kB + e] = (1.0f - a) * v;
        gi[kB + e] = a * v;
      }
      __syncthreads();
    }
    float xr[16], xi[16];
    fft8192_in_smem<false>(gr, gi, s, tb, t, [&] { fetch(it + 2, m + 2); }, [] {}, xr, xi);
    float2* out = Xs + (int64_t)m * kNbA;
#pragma unroll
    for (int q = 0; q < 16; ++q) out[t + 512 * q] = make_float2(xr[q], xi[q]);
  }
}

// inverse transforms of the dL/dx spectra, runs of kConvRun units m = il XW + w, second half only: a crossfaded slot
// gives (1 - a) re + a im on samples [i kB, (i+1) kB) of source s, a later slot sources 2p and 2p + 1 as re and im
__global__ void __launch_bounds__(kFusedThreads, 1)
tvbusin_ifft_kernel(const float* __restrict__ Dpl, const float* __restrict__ twiddles, float* __restrict__ gx,
                    int64_t item0, int S, int I, int nX, int H, int64_t hop, int64_t n, int nunits) {
  extern __shared__ __align__(128) float sm[];
  FftSmem s(sm);
  const int t = threadIdx.x;
  s.init(twiddles, t);
  const fft8k::Tables tb = fft8k::carve_tables(s.tabf);
  const int P = (S + 1) / 2, XW = nX * S + (I - nX) * P;
  const int m0 = blockIdx.x * kConvRun;
  const int m1 = nunits - m0 < kConvRun ? nunits : m0 + kConvRun;
  auto fetch = [&](int it, int m) {
    if (t == 0 && m < m1) s.load_planar(it, Dpl + (int64_t)m * 2 * kNbA);
  };
  fetch(0, m0);
  fetch(1, m0 + 1);
  int it = 0;
  for (int m = m0; m < m1; ++m, ++it) {
    s.wait(it);
    float* gr = s.buf(it);
    float xr[16], xi[16];
    fft8192_in_smem<true>(gr, gr + fft8k::kPlaneG, s, tb, t, [&] { fetch(it + 2, m + 2); }, [] {}, xr, xi);
    const int64_t il = m / XW;
    int i, c;
    tvin_block(m - (int)il * XW, S, P, nX, i, c);
    const bool cross = i < nX;                     // uniform over the CTA
    const bool two = !cross && 2 * c + 1 < S;
    float* ra = gx + ((item0 + il) * S + (cross ? c : 2 * c)) * n;
#pragma unroll
    for (int q = 8; q < 16; ++q) {                 // outputs kB .. 2 kB - 1 of the transform
      const int e = t + 512 * q - kB;
      const int64_t tg = (int64_t)i * kB + e;
      if (tg < n) {
        if (cross) {
          const float a = tv_a(i, H, e, hop);
          ra[tg] = fmaf(a, xi[q], (1.0f - a) * xr[q]);
        } else {
          ra[tg] = xr[q];
          if (two) ra[n + tg] = xi[q];
        }
      }
    }
  }
}

// The products of the source-side bus per bin pair (f, kNbA - f) and item, every operand untangled into the spectra of
// its real rows (Za_s / Zb_s: the 1 - a / a pieces of source s in a crossfaded block, Z_s after the last anchor, Za_s
// then; H_k,s,o: IR row (k S + s) O + o; G_o: FFT of [0 | g_o block]), results packed two real rows per block, planar,
// scaled by 1 / kNbA; all operands from L2.  k(i) is the anchor interval of input block i.
//   TVI_FWD: Y_o[m] = sum_s sum_j Za_s[m-j] H_k(m-j),s,o[j] + Zb_s[m-j] H_k(m-j)+1,s,o[j], stored as
//            W_o[m] = Y_o[m] + (-1)^f Y_o[m - 1]                                      out: I blocks (W_0 + i W_1)
//   TVI_DX:  first folds G in place, G_o[q] <- Gt_o[q] = G_o[q] + (-1)^f G_o[q + 1], the spectrum of [g_o,q+1 | g_o,q]
//            (the gradient of Y_o[q]'s whole inverse); then Da_s[i] = sum_o sum_j Gt_o[i+j] conj(H_k(i),s,o[j]) and
//            Db_s[i] the same with IR set k(i) + 1 (i < nX)                           out: XW slots (Da + i Db, or
//            D_2p + i D_2p+1 after the last anchor)
//   TVI_DIR: E_k,s,o[j] = sum_{i in interval k} Gt_o[i+j] conj(Za_s[i]) + sum_{i in interval k-1} Gt_o[i+j] conj(Zb_s[i])
//            (reads the folded G TVI_DX left)                                          out: NH J blocks (set q: rows 2q,
//            2q + 1)
// X: XW slots per item; H: NH J partitions per trajectory set at item stride hstride (0: one set for the batch); G: I
// blocks per item.
enum TvBusInMac { TVI_FWD, TVI_DX, TVI_DIR };
template <int MODE, int O>
__global__ void __launch_bounds__(128) tvbusin_mac_kernel(const float2* __restrict__ X, const float2* __restrict__ H,
                                                          int64_t hstride, float2* G, float2* __restrict__ Out, int S,
                                                          int I, int J, int K, int nX, int Hb) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f > kNbA / 2) return;
  const int fm = (kNbA - f) & (kNbA - 1);
  const int64_t il = blockIdx.y;
  const int P = (S + 1) / 2, XW = nX * S + (I - nX) * P;
  const float2* x = X + il * (int64_t)XW * kNbA;
  const float2* h = H + il * hstride;
  float2* g = G + il * (int64_t)I * kNbA;
  const float2 zero = make_float2(0.f, 0.f);
  auto pair = [&](const float2* base, int64_t slot, float2& a, float2& b) {
    untangle(base[slot * kNbA + f], base[slot * kNbA + fm], a, b);
  };
  // source s of block i: (Za, Zb), or (Z, 0) after the last anchor
  auto xin = [&](int i, int s, float2& za, float2& zb) {
    if (i < nX) { pair(x, (int64_t)i * S + s, za, zb); return; }
    float2 a, b;
    pair(x, (int64_t)nX * S + (int64_t)(i - nX) * P + (s >> 1), a, b);
    za = (s & 1) ? b : a;
    zb = zero;
  };
  // IR rows (k, s, 0) and (k, s, 1) (O == 2), or row (k, s) (O == 1), at partition j
  auto hin = [&](int k, int s, int j, float2& h0, float2& h1) {
    const int r = k * S + s;
    if (O == 2) { pair(h, (int64_t)r * J + j, h0, h1); }
    else { float2 a, b; pair(h, (int64_t)(r >> 1) * J + j, a, b); h0 = (r & 1) ? b : a; h1 = zero; }
  };
  const float scale = 1.0f / (float)kNbA;
  auto emit = [&](int64_t slot, float2 a, float2 b) {
    a.x *= scale; a.y *= scale; b.x *= scale; b.y *= scale;
    float* pl = reinterpret_cast<float*>(Out + slot * kNbA);
    pl[f] = a.x - b.y; pl[kNbA + f] = a.y + b.x;
    if (fm != f) { pl[fm] = a.x + b.y; pl[kNbA + fm] = b.x - a.y; }
  };
  const float sgn = (f & 1) ? -1.f : 1.f;          // (-1)^f, and (-1)^fm: kNbA is even
  auto axpy = [&](float2 acc, float2 v) { return make_float2(fmaf(sgn, v.x, acc.x), fmaf(sgn, v.y, acc.y)); };
  auto ival = [&](int i) { const int k = i / Hb; return k < K - 1 ? k : K - 1; };   // anchor interval of block i

  if constexpr (MODE == TVI_FWD) {
    const int64_t ob = il * (int64_t)I;
    float2 p0 = zero, p1 = zero;                   // Y_0[m - 1], Y_1[m - 1]
    for (int m = 0; m < I; ++m) {
      float2 y0 = zero, y1 = zero;
      for (int j = 0; j <= m && j < J; ++j) {
        const int i = m - j, k = ival(i);
        for (int s = 0; s < S; ++s) {
          float2 za, zb, h0, h1;
          xin(i, s, za, zb);
          hin(k, s, j, h0, h1);
          cfma(y0, za, h0);
          if (O == 2) cfma(y1, za, h1);
          if (i < nX) {
            hin(k + 1, s, j, h0, h1);
            cfma(y0, zb, h0);
            if (O == 2) cfma(y1, zb, h1);
          }
        }
      }
      emit(ob + m, axpy(y0, p0), axpy(y1, p1));
      p0 = y0; p1 = y1;
    }
  } else if constexpr (MODE == TVI_DX) {
    // the fold, in place on this thread's own bins f and fm, which no other thread reads; Gt[I - 1] = G[I - 1]
    for (int q = 0; q + 1 < I; ++q) {
      float2* a = g + (int64_t)q * kNbA;
      const float2* b = a + kNbA;
      a[f] = axpy(a[f], b[f]);
      if (fm != f) a[fm] = axpy(a[fm], b[fm]);
    }
    const int64_t ob = il * (int64_t)XW;
    for (int i = 0; i < I; ++i) {
      const int k = ival(i);
      const bool cross = i < nX;
      for (int p = 0; p < P; ++p) {
        const int nc = 2 * p + 1 < S ? 2 : 1;
        float2 da[2] = {zero, zero}, db[2] = {zero, zero};
        for (int j = 0; j < J && i + j < I; ++j) {
          float2 g0, g1, h0, h1;
          pair(g, i + j, g0, g1);
          for (int c = 0; c < nc; ++c) {
            hin(k, 2 * p + c, j, h0, h1);
            cfma_conj(da[c], g0, h0);
            if (O == 2) cfma_conj(da[c], g1, h1);
            if (cross) {
              hin(k + 1, 2 * p + c, j, h0, h1);
              cfma_conj(db[c], g0, h0);
              if (O == 2) cfma_conj(db[c], g1, h1);
            }
          }
        }
        if (cross) {
          for (int c = 0; c < nc; ++c) emit(ob + (int64_t)i * S + 2 * p + c, da[c], db[c]);
        } else {
          emit(ob + (int64_t)nX * S + (int64_t)(i - nX) * P + p, da[0], da[1]);
        }
      }
    }
  } else {
    static_assert(MODE == TVI_DIR, "tvbusin_mac_kernel: unknown mode");
    // e[o] = E_k,s,o[j] over both intervals that carry IR set k
    auto ecorr = [&](int k, int s, int j, float2 (&e)[2]) {
      e[0] = e[1] = zero;
      for (int part = 0; part < 2; ++part) {       // 0: Za (Z) of interval k, 1: Zb of interval k - 1
        const int kk = k - part;
        if (kk < 0) continue;
        const int lo = kk * Hb, hi = kk == K - 1 ? I : ((kk + 1) * Hb < I ? (kk + 1) * Hb : I);
        for (int i = lo; i < hi && i + j < I; ++i) {
          float2 g0, g1, za, zb;
          pair(g, i + j, g0, g1);
          xin(i, s, za, zb);
          const float2 z = part ? zb : za;
          cfma_conj(e[0], g0, z);
          if (O == 2) cfma_conj(e[1], g1, z);
        }
      }
    };
    const int NH = (K * S * O + 1) / 2;
    const int64_t ob = il * (int64_t)NH * J;
    float2 e[2];
    for (int q = 0; q < NH; ++q) {
      for (int j = 0; j < J; ++j) {
        if (O == 2) {                              // set q: rows (q, o = 0) and (q, o = 1), q = k S + s
          ecorr(q / S, q % S, j, e);
          emit(ob + (int64_t)q * J + j, e[0], e[1]);
        } else {                                   // set q: rows 2q and 2q + 1 (r = k S + s), an odd last row with 0
          ecorr((2 * q) / S, (2 * q) % S, j, e);
          const float2 a = e[0];
          float2 b = zero;
          if (2 * q + 1 < K * S) {
            ecorr((2 * q + 1) / S, (2 * q + 1) % S, j, e);
            b = e[0];
          }
          emit(ob + (int64_t)q * J + j, a, b);
        }
      }
    }
  }
}

// ---- time_varying_multichannel_convolution: the time-varying bus with M >= 3 outputs (Q = ceil(M / 2) output pairs) --
// The IR layout is the bus's: row r = (k S + s) M + m, two rows per partition set (NH = ceil(K S M / 2) sets).
// Output side (tvmc_mac_kernel): the product and gradient slots of an item are tvin_block's layout with (S, P) ->
// (M, Q), U = M nX + Q (I - nX) slots:
//   slot i M + m (i < nX):                (Y_k,m[i], Y_k+1,m[i]); gradient FFT of [0 | (1 - a) g_m,i + i a g_m,i]
//   slot M nX + (i - nX) Q + q (i >= nX): (Y_K-1,2q[i], Y_K-1,2q+1[i]); gradient FFT of [0 | g_2q,i + i g_2q+1,i]
// which are the source-side window spectra of M rows: tvbusin_fft_kernel transforms the gradient into them and
// tvbusin_ifft_kernel gives (1 - a) re + a im on a crossfaded slot, rows 2q and 2q + 1 on a later one.
// Source side (tvmcin_mac_kernel): the windows are tvbusin_fft_kernel's (XW per item), the products and gradients one
// spectrum per block and output pair, pair q of block i at block q I + i of the item (bus_ifft_kernel /
// bus_fft_kernel with rows M, groups Q).
// Both kernels run one slice of an item per blockIdx.y and the items along blockIdx.z, so the slices of an item run
// next to each other and re-read its spectra from L2; all operands from L2, results packed two real rows per block,
// planar, scaled by 1 / kNbA.
//   TVM_FWD: slice q < Q:  Y_k,2q / 2q+1[i] = sum_s sum_j X_s[i - j] H_k,s,m[j] for the IR sets of block i
//                                                                                    out: U slots
//   TVM_DX:  slice p < P:  D_s[i] (s = 2p, 2p + 1) = sum_m sum_j Ga_m[i+j] conj(H_k,s,m[j]) + Gb_m[i+j]
//            conj(H_k+1,s,m[j]), stored as W_s[i] = D_s[i] + (-1)^f D_s[i + 1]   out: P I blocks (bus_ifft_kernel)
//   TVM_DIR: slice h < NH: E_r[j] of rows r = 2h, 2h + 1, each an (k, s, m):
//            sum_{i in interval k} Ga_m[i] conj(X_s[i-j]) + sum_{i in interval k-1} Gb_m[i] conj(X_s[i-j])
//                                                                                    out: NH J blocks
// X: P I blocks per item; H: NH J partitions per trajectory set at item stride hstride (0: one set for the batch);
// G: U slots per item.
enum TvMcMac { TVM_FWD, TVM_DX, TVM_DIR };
template <int MODE>
__global__ void __launch_bounds__(128) tvmc_mac_kernel(const float2* __restrict__ X, const float2* __restrict__ H,
                                                       int64_t hstride, const float2* __restrict__ G,
                                                       float2* __restrict__ Out, int S, int M, int I, int J, int K,
                                                       int nX, int Hb) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f > kNbA / 2) return;
  const int fm = (kNbA - f) & (kNbA - 1);
  const int sl = blockIdx.y;
  const int64_t il = blockIdx.z;
  const int P = (S + 1) / 2, Q = (M + 1) / 2, U = M * nX + Q * (I - nX), NH = (K * S * M + 1) / 2;
  const float2* x = X + il * (int64_t)P * I * kNbA;
  const float2* h = H + il * hstride;
  const float2* g = G + il * (int64_t)U * kNbA;
  const float2 zero = make_float2(0.f, 0.f);
  auto pair = [&](const float2* base, int64_t slot, float2& a, float2& b) {
    untangle(base[slot * kNbA + f], base[slot * kNbA + fm], a, b);
  };
  auto pick = [&](const float2* base, int64_t slot, int odd) -> float2 {
    float2 a, b;
    pair(base, slot, a, b);
    return odd ? b : a;
  };
  // IR rows (k, s, 2q) and (k, s, 2q + 1) at partition j, 0 past the last output; one set when the first row is even
  auto hin = [&](int k, int s, int q, int j, float2& h0, float2& h1) {
    const int r = (k * S + s) * M + 2 * q;
    if (2 * q + 1 >= M) { h0 = pick(h, (int64_t)(r >> 1) * J + j, r & 1); h1 = zero; }
    else if ((r & 1) == 0) pair(h, (int64_t)(r >> 1) * J + j, h0, h1);
    else { h0 = pick(h, (int64_t)(r >> 1) * J + j, 1); h1 = pick(h, (int64_t)((r + 1) >> 1) * J + j, 0); }
  };
  // the gradient of outputs 2q, 2q + 1 at block i: IR set k(i) (ga) and k(i) + 1 (gb, 0 after the last anchor)
  auto gin = [&](int i, int q, float2 (&ga)[2], float2 (&gb)[2]) {
    if (i < nX) {
      pair(g, (int64_t)i * M + 2 * q, ga[0], gb[0]);
      if (2 * q + 1 < M) pair(g, (int64_t)i * M + 2 * q + 1, ga[1], gb[1]);
      else ga[1] = gb[1] = zero;
    } else {
      pair(g, (int64_t)M * nX + (int64_t)(i - nX) * Q + q, ga[0], ga[1]);
      gb[0] = gb[1] = zero;
    }
  };
  auto emit = [&](int64_t slot, float2 a, float2 b) { bus_emit(Out, slot, f, fm, 1.0f / (float)kNbA, a, b); };
  auto ival = [&](int i) { const int k = i / Hb; return k < K - 1 ? k : K - 1; };   // anchor interval of block i

  if constexpr (MODE == TVM_FWD) {
    const int q = sl;
    const int64_t ob = il * (int64_t)U;
    for (int o = 0; o < I; ++o) {
      const int k = ival(o);
      const bool cross = o < nX;
      float2 y0 = zero, y1 = zero, z0 = zero, z1 = zero;    // IR set k: outputs 2q, 2q + 1; IR set k + 1: the same
      for (int p = 0; p < P; ++p) {
        const int nc = 2 * p + 1 < S ? 2 : 1;
        for (int j = 0; j <= o && j < J; ++j) {
          float2 xv[2], h0, h1;
          pair(x, (int64_t)p * I + o - j, xv[0], xv[1]);
#pragma unroll
          for (int c = 0; c < 2; ++c) {
            if (c >= nc) break;
            hin(k, 2 * p + c, q, j, h0, h1);
            cfma(y0, xv[c], h0);
            cfma(y1, xv[c], h1);
            if (cross) {
              hin(k + 1, 2 * p + c, q, j, h0, h1);
              cfma(z0, xv[c], h0);
              cfma(z1, xv[c], h1);
            }
          }
        }
      }
      if (cross) {
        emit(ob + (int64_t)o * M + 2 * q, y0, z0);
        if (2 * q + 1 < M) emit(ob + (int64_t)o * M + 2 * q + 1, y1, z1);
      } else {
        emit(ob + (int64_t)M * nX + (int64_t)(o - nX) * Q + q, y0, y1);
      }
    }
  } else if constexpr (MODE == TVM_DX) {
    const int p = sl;
    const int nc = 2 * p + 1 < S ? 2 : 1;
    const float sgn = (f & 1) ? -1.f : 1.f;
    const int64_t ob = (il * P + p) * (int64_t)I;
    float2 next[2] = {zero, zero};                 // D[m + 1]
    for (int m = I - 1; m >= 0; --m) {
      float2 d[2] = {zero, zero};                  // D_2p+c[m] (d[1] stays 0 for an odd last source)
      for (int j = 0; j < J && m + j < I; ++j) {
        const int i = m + j, k = ival(i);
        for (int q = 0; q < Q; ++q) {
          float2 ga[2], gb[2], h0, h1;
          gin(i, q, ga, gb);
#pragma unroll
          for (int c = 0; c < 2; ++c) {
            if (c >= nc) break;
            hin(k, 2 * p + c, q, j, h0, h1);
            cfma_conj(d[c], ga[0], h0);
            cfma_conj(d[c], ga[1], h1);
            if (i < nX) {
              hin(k + 1, 2 * p + c, q, j, h0, h1);
              cfma_conj(d[c], gb[0], h0);
              cfma_conj(d[c], gb[1], h1);
            }
          }
        }
      }
      emit(ob + m, bus_axpy(sgn, d[0], next[0]), bus_axpy(sgn, d[1], next[1]));
      next[0] = d[0]; next[1] = d[1];
    }
  } else {
    static_assert(MODE == TVM_DIR, "tvmc_mac_kernel: unknown mode");
    // E_r[j] of row r = (k S + s) M + m over both intervals that carry IR set k
    auto ecorr = [&](int r, int j) -> float2 {
      const int k = r / (S * M), sm = r - k * S * M, s = sm / M, m = sm - s * M;
      float2 e = zero;
      for (int part = 0; part < 2; ++part) {       // 0: Ga (G) of interval k, 1: Gb of interval k - 1
        const int kk = k - part;
        if (kk < 0) continue;
        const int lo = kk * Hb, hi = kk == K - 1 ? I : ((kk + 1) * Hb < I ? (kk + 1) * Hb : I);
        for (int i = lo > j ? lo : j; i < hi; ++i) {
          const float2 gv = i < nX ? pick(g, (int64_t)i * M + m, part)
                                   : pick(g, (int64_t)M * nX + (int64_t)(i - nX) * Q + (m >> 1), m & 1);
          cfma_conj(e, gv, pick(x, (int64_t)(s >> 1) * I + i - j, s & 1));
        }
      }
      return e;
    };
    const int r0 = 2 * sl;
    const bool two = r0 + 1 < K * S * M;
    const int64_t ob = (il * NH + sl) * (int64_t)J;
    for (int j = 0; j < J; ++j) emit(ob + j, ecorr(r0, j), two ? ecorr(r0 + 1, j) : zero);
  }
}

// The source-side products with M >= 3 outputs, operands as tvbusin_mac_kernel's (Za_s / Zb_s / Z_s: the window
// slots of source s; G_m: FFT of [0 | g_m block], rows 2q, 2q + 1 in block q I + i of the item), one slice per
// blockIdx.y as tvmc_mac_kernel:
//   TVJ_FOLD: slice q < Q:  folds G of pair q in place, G[i] <- Gt[i] = G[i] + (-1)^f G[i + 1] (tvbusin_mac_kernel's
//                           TVI_DX prologue; each slice and thread owns its blocks and bins)
//   TVJ_FWD:  slice q < Q:  Y_m[i] (m = 2q, 2q + 1) = sum_s sum_j Za_s[i-j] H_k(i-j),s,m[j] + Zb_s[i-j]
//                           H_k(i-j)+1,s,m[j], stored as W_m[i] = Y_m[i] + (-1)^f Y_m[i - 1]   out: Q I blocks
//   TVJ_DX:   slice p < P:  Da_s[i] = sum_m sum_j Gt_m[i+j] conj(H_k(i),s,m[j]), Db_s[i] with IR set k(i) + 1
//                           (i < nX)                                      out: XW slots (tvbusin_ifft_kernel's)
//   TVJ_DIR:  slice h < NH: E_r[j] of rows r = 2h, 2h + 1, each an (k, s, m): sum_{i in interval k} Gt_m[i+j]
//                           conj(Za_s[i]) + sum_{i in interval k-1} Gt_m[i+j] conj(Zb_s[i])     out: NH J blocks
// X: XW slots per item; H: NH J partitions per trajectory set at item stride hstride; G: Q I blocks per item.
enum TvMcInMac { TVJ_FOLD, TVJ_FWD, TVJ_DX, TVJ_DIR };
template <int MODE>
__global__ void __launch_bounds__(128) tvmcin_mac_kernel(const float2* __restrict__ X, const float2* __restrict__ H,
                                                         int64_t hstride, float2* G, float2* __restrict__ Out, int S,
                                                         int M, int I, int J, int K, int nX, int Hb) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f > kNbA / 2) return;
  const int fm = (kNbA - f) & (kNbA - 1);
  const int sl = blockIdx.y;
  const int64_t il = blockIdx.z;
  const int P = (S + 1) / 2, Q = (M + 1) / 2, XW = nX * S + (I - nX) * P, NH = (K * S * M + 1) / 2;
  const float2* x = X + il * (int64_t)XW * kNbA;
  const float2* h = H + il * hstride;
  float2* g = G + il * (int64_t)Q * I * kNbA;
  const float2 zero = make_float2(0.f, 0.f);
  auto pair = [&](const float2* base, int64_t slot, float2& a, float2& b) {
    untangle(base[slot * kNbA + f], base[slot * kNbA + fm], a, b);
  };
  auto pick = [&](const float2* base, int64_t slot, int odd) -> float2 {
    float2 a, b;
    pair(base, slot, a, b);
    return odd ? b : a;
  };
  // source s of block i: (Za, Zb), or (Z, 0) after the last anchor
  auto xin = [&](int i, int s, float2& za, float2& zb) {
    if (i < nX) { pair(x, (int64_t)i * S + s, za, zb); return; }
    za = pick(x, (int64_t)nX * S + (int64_t)(i - nX) * P + (s >> 1), s & 1);
    zb = zero;
  };
  auto hin = [&](int k, int s, int q, int j, float2& h0, float2& h1) {   // as tvmc_mac_kernel's
    const int r = (k * S + s) * M + 2 * q;
    if (2 * q + 1 >= M) { h0 = pick(h, (int64_t)(r >> 1) * J + j, r & 1); h1 = zero; }
    else if ((r & 1) == 0) pair(h, (int64_t)(r >> 1) * J + j, h0, h1);
    else { h0 = pick(h, (int64_t)(r >> 1) * J + j, 1); h1 = pick(h, (int64_t)((r + 1) >> 1) * J + j, 0); }
  };
  auto emit = [&](int64_t slot, float2 a, float2 b) { bus_emit(Out, slot, f, fm, 1.0f / (float)kNbA, a, b); };
  const float sgn = (f & 1) ? -1.f : 1.f;          // (-1)^f, and (-1)^fm: kNbA is even
  auto ival = [&](int i) { const int k = i / Hb; return k < K - 1 ? k : K - 1; };   // anchor interval of block i

  if constexpr (MODE == TVJ_FOLD) {
    float2* gq = g + (int64_t)sl * I * kNbA;
    for (int q = 0; q + 1 < I; ++q) {
      float2* a = gq + (int64_t)q * kNbA;
      const float2* b = a + kNbA;
      a[f] = bus_axpy(sgn, a[f], b[f]);
      if (fm != f) a[fm] = bus_axpy(sgn, a[fm], b[fm]);
    }
  } else if constexpr (MODE == TVJ_FWD) {
    const int q = sl;
    const int64_t ob = (il * Q + q) * (int64_t)I;
    float2 p0 = zero, p1 = zero;                   // Y_2q[m - 1], Y_2q+1[m - 1]
    for (int m = 0; m < I; ++m) {
      float2 y0 = zero, y1 = zero;
      for (int j = 0; j <= m && j < J; ++j) {
        const int i = m - j, k = ival(i);
        for (int s = 0; s < S; ++s) {
          float2 za, zb, h0, h1;
          xin(i, s, za, zb);
          hin(k, s, q, j, h0, h1);
          cfma(y0, za, h0);
          cfma(y1, za, h1);
          if (i < nX) {
            hin(k + 1, s, q, j, h0, h1);
            cfma(y0, zb, h0);
            cfma(y1, zb, h1);
          }
        }
      }
      emit(ob + m, bus_axpy(sgn, y0, p0), bus_axpy(sgn, y1, p1));
      p0 = y0; p1 = y1;
    }
  } else if constexpr (MODE == TVJ_DX) {
    const int p = sl;
    const int nc = 2 * p + 1 < S ? 2 : 1;
    const int64_t ob = il * (int64_t)XW;
    for (int i = 0; i < I; ++i) {
      const int k = ival(i);
      const bool cross = i < nX;
      float2 da[2] = {zero, zero}, db[2] = {zero, zero};
      for (int j = 0; j < J && i + j < I; ++j) {
        for (int q = 0; q < Q; ++q) {
          float2 g0, g1, h0, h1;
          pair(g, (int64_t)q * I + i + j, g0, g1);
#pragma unroll
          for (int c = 0; c < 2; ++c) {
            if (c >= nc) break;
            hin(k, 2 * p + c, q, j, h0, h1);
            cfma_conj(da[c], g0, h0);
            cfma_conj(da[c], g1, h1);
            if (cross) {
              hin(k + 1, 2 * p + c, q, j, h0, h1);
              cfma_conj(db[c], g0, h0);
              cfma_conj(db[c], g1, h1);
            }
          }
        }
      }
      if (cross) {
#pragma unroll
        for (int c = 0; c < 2; ++c) if (c < nc) emit(ob + (int64_t)i * S + 2 * p + c, da[c], db[c]);
      } else {
        emit(ob + (int64_t)nX * S + (int64_t)(i - nX) * P + p, da[0], da[1]);
      }
    }
  } else {
    static_assert(MODE == TVJ_DIR, "tvmcin_mac_kernel: unknown mode");
    // E_r[j] of row r = (k S + s) M + m over both intervals that carry IR set k
    auto ecorr = [&](int r, int j) -> float2 {
      const int k = r / (S * M), sm = r - k * S * M, s = sm / M, m = sm - s * M;
      float2 e = zero;
      for (int part = 0; part < 2; ++part) {       // 0: Za (Z) of interval k, 1: Zb of interval k - 1
        const int kk = k - part;
        if (kk < 0) continue;
        const int lo = kk * Hb, hi = kk == K - 1 ? I : ((kk + 1) * Hb < I ? (kk + 1) * Hb : I);
        for (int i = lo; i < hi && i + j < I; ++i) {
          float2 za, zb;
          xin(i, s, za, zb);
          cfma_conj(e, pick(g, (int64_t)(m >> 1) * I + i + j, m & 1), part ? zb : za);
        }
      }
      return e;
    };
    const int r0 = 2 * sl;
    const bool two = r0 + 1 < K * S * M;
    const int64_t ob = (il * NH + sl) * (int64_t)J;
    for (int j = 0; j < J; ++j) emit(ob + j, ecorr(r0, j), two ? ecorr(r0 + 1, j) : zero);
  }
}

// Device-resident band spectra H_k, built once per (device, taps, sr, grid).  half (the spectral synthesis): the half
// spectrum of the taps on its n1-point grid, 12 x (n1/2+1) complex, scaled sqrt(n1/2)/n1 -- the 1/n1 of the inverse
// transform and the sqrt(n1/2) of the bins' complex Gaussians (Z ~ CN(0, n1)) folded in.  Otherwise the full spectrum on
// the nb-point grid of the overlap-save blocks, 12 x nb complex, scaled 1/nb.
int get_filterbank(const Geom& g, double sr, bool half, cudaStream_t st, const float2** out) {
  int dev = 0;
  DASP_CUDA_OK(cudaGetDevice(&dev));
  const int64_t n = half ? g.n1() : g.nb, nc = half ? g.n1c() : g.nb;
  const bool flat = debug_flat_filterbank();        // test hook: H_k = 1 -> the filtered noise is the white noise itself
  FbKey key{dev, flat ? -g.taps : g.taps, half ? -n : n, sr};
  auto it = g_fb.find(key);
  if (it != g_fb.end()) { *out = reinterpret_cast<const float2*>(it->second); return DASP_OK; }
  DASP_REQUIRE(sr / 2.0 > 18000.0, "sample_rate %.1f too low: the filter bank needs 18 kHz < sr/2 (signal.py:84)", sr);
  if (half) {
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
  const float inv = half ? (float)(sqrt(0.5 * (double)n) / (double)n) : 1.0f / (float)n;
  const int64_t w = half ? 1 : 2;                   // floats per input sample: real (R2C) or complex (in-place C2C)
  std::vector<float> padded((size_t)(kBands * n * w), 0.f);
  for (int k = 0; k < kBands; ++k)
    for (int64_t i = 0; i < g.taps; ++i) padded[(size_t)((k * n + i) * w)] = taps[(size_t)k * g.taps + i] * inv;
  float* d_in = nullptr;
  cufftComplex* d_out = nullptr;
  void* d_work = nullptr;
  DASP_CUDA_OK(cudaMalloc(&d_in, sizeof(float) * padded.size()));
  DASP_CUDA_OK(cudaMemcpyAsync(d_in, padded.data(), sizeof(float) * padded.size(), cudaMemcpyHostToDevice, st));
  if (half) DASP_CUDA_OK(cudaMalloc(&d_out, sizeof(cufftComplex) * kBands * nc));
  else      d_out = reinterpret_cast<cufftComplex*>(d_in);
  PlanVal pv;
  int rc = get_plan(half ? 0 : 2, n, kBands, n, nc, pv);
  if (rc != DASP_OK) return rc;
  DASP_CUDA_OK(cudaMalloc(&d_work, pv.work > 0 ? pv.work : 16));
  DASP_CUFFT_OK(cufftSetStream(pv.h, st));
  DASP_CUFFT_OK(cufftSetWorkArea(pv.h, d_work));
  if (half) DASP_CUFFT_OK(cufftExecR2C(pv.h, d_in, d_out));
  else      DASP_CUFFT_OK(cufftExecC2C(pv.h, d_out, d_out, CUFFT_FORWARD));
  DASP_CUDA_OK(cudaStreamSynchronize(st));   // one-off (cache fill): host vector and temp buffers die here
  if (half) cudaFree(d_in);
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

// the layout of the filtered noise f (f_save): polyphase (the spectral synthesis, device noise up to kMaxSpectralR) or
// overlap-save blocks
bool polyphase_f(const Geom& g, bool device_noise) { return device_noise && g.rpp <= kMaxSpectralR; }

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
// Side stream of the forward's IR synthesis (see dasp_reverb_fwd), created once per device at the greatest stream
// priority.  fork is recorded on the caller's stream before the first synthesis, done after each chunk's synthesis on
// side.  Reusing the events across chunks and calls is safe: cudaStreamWaitEvent takes the state of the event at the
// time of the call, and a later record does not change what an earlier wait waits for.
struct SideStream { cudaStream_t side; cudaEvent_t fork, done; int prio; };
std::map<int, SideStream> g_side;                   // guarded by g_mu
int get_side_stream(SideStream** out) {
  int dev = 0;
  DASP_CUDA_OK(cudaGetDevice(&dev));
  auto it = g_side.find(dev);
  if (it == g_side.end()) {
    SideStream s{};
    int least = 0;
    DASP_CUDA_OK(cudaDeviceGetStreamPriorityRange(&least, &s.prio));
    DASP_CUDA_OK(cudaStreamCreateWithPriority(&s.side, cudaStreamNonBlocking, s.prio));
    DASP_CUDA_OK(cudaEventCreateWithFlags(&s.done, cudaEventDisableTiming));
    DASP_CUDA_OK(cudaEventCreateWithFlags(&s.fork, cudaEventDisableTiming));
    it = g_side.emplace(dev, s).first;
  }
  *out = &it->second;
  return DASP_OK;
}

int configure_fft_kernels();
// generator output -> ifft_shape_kernel for the items of a chunk
template <class Sink>
int launch_ifft_shape(float2* C, const float* tw, const float* params, const Sink& out, bool save_f, int64_t items,
                      const Geom& g, cudaStream_t st, const int* prio) {
  int rc = configure_fft_kernels();
  if (rc != DASP_OK) return rc;
  cudaLaunchConfig_t cfg = {};
  cudaLaunchAttribute at[1];
  cfg.gridDim = dim3((unsigned)g.rpp, (unsigned)items, 1);
  cfg.blockDim = dim3(kFusedThreads, 1, 1);
  cfg.dynamicSmemBytes = kFftSmemBytes;
  cfg.stream = st;
  add_priority(cfg, at, prio);
  cudaLaunchKernelEx(&cfg, ifft_shape_kernel<Sink>, reinterpret_cast<float*>(C), tw, params, out, save_f ? 1 : 0,
                     (int)g.L, (int)g.leff, (int)g.rpp);
  DASP_LAUNCH_OK("ifft_shape_kernel");
  return DASP_OK;
}
int g_last_fused = 0;                                // test hook: IR-synthesis path of the last forward chunk
std::map<std::pair<int, const void*>, int> g_fused_ok;   // (device, kernel) -> clusters that fit, guarded by g_mu
// cluster synthesis: persistent clusters of R CTAs, as many as the device co-schedules (at most one per item).
// Returns false when the device cannot co-schedule such a cluster (then generator -> ifft_shape_kernel runs), true after
// a launch attempt (check cudaGetLastError).
template <int R, class Sink>
bool launch_fused(const float2* H1, const float* tw, const float* params, const Sink& out, float2* Csave, int64_t item0,
                  int64_t items, int64_t L, int64_t leff, const unsigned long long* seed, cudaStream_t st,
                  const int* prio) {
  auto kern = ir_synth_cluster_kernel<R, Sink>;
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
  auto it = g_fused_ok.find({dev, (const void*)kern});
  if (it == g_fused_ok.end()) {
    int n = 0;
    cfg.gridDim = dim3(R, 1, 1);
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSynthSmemBytes) != cudaSuccess ||
        cudaOccupancyMaxActiveClusters(&n, kern, &cfg) != cudaSuccess) {
      n = 0;
      cudaGetLastError();
    }
    it = g_fused_ok.emplace(std::make_pair(dev, (const void*)kern), n).first;
  }
  if (it->second < 1) return false;
  const int64_t clusters = items < it->second ? items : it->second;
  cfg.gridDim = dim3(R, (unsigned)clusters, 1);
  add_priority(cfg, at, prio);
  cudaLaunchKernelEx(&cfg, kern, H1, tw, params, out, Csave, item0, (int)items, (int)L, (int)leff, seed);
  return true;
}
template <class Sink>
bool dispatch_fused(int R, const float2* H1, const float* tw, const float* params, const Sink& out, float2* Csave,
                    int64_t item0, int64_t items, int64_t L, int64_t leff, const unsigned long long* seed,
                    cudaStream_t st, const int* prio) {
  switch (R) {
#define DASP_R(r) case r: return launch_fused<r>(H1, tw, params, out, Csave, item0, items, L, leff, seed, st, prio);
    DASP_R(1) DASP_R(2) DASP_R(3) DASP_R(4) DASP_R(5) DASP_R(6)
#undef DASP_R
    default: return false;
  }
}

inline size_t align256(size_t v) { return (v + 255) & ~(size_t)255; }

// workspace carve-up shared by the geometry queries and the entry points; extra: the reverb's own region (the filtered
// noise of a chunk when f_save is not kept / the per-partition partials of the 24 band-parameter gradients); mixpart:
// the dL/dmix partials (0 bytes without a mix); acc: the fp64 sum of a shared IR's dL/dIR partition spectra (0 bytes
// unless g.shared)
struct FwdWs { size_t ys, xsp, hsp, extra, cufft, total; };
struct BwdWs { size_t gs, ds, es, extra, mixpart, acc, cufft, total; };

void fwd_layout(const ConvGeom& g, size_t extra_bytes, size_t cufft_work, FwdWs& w) {
  size_t o = 0;
  w.ys = o;  o += align256(sizeof(float2) * (size_t)(g.chunk * (g.ib + g.ex) * kNbA));
  // transient homes for what a forward WITHOUT a backward does not keep (null *_save pointers)
  w.xsp = o; o += align256(sizeof(float2) * (size_t)(g.chunk * g.xwin() * kNbA));
  w.hsp = o; o += align256(sizeof(float2) * (size_t)((g.shared ? 1 : g.chunk) * g.sets * g.jb * kNbA));
  w.extra = o; o += align256(extra_bytes);
  w.cufft = o; o += align256(cufft_work);
  w.total = o;
}
void bwd_layout(const ConvGeom& g, size_t extra_bytes, size_t cufft_work, BwdWs& w) {
  size_t o = 0;
  w.gs = o; o += align256(sizeof(float2) * (size_t)(g.chunk * (g.ib + g.ex) * kNbA));
  w.ds = o; o += align256(sizeof(float2) * (size_t)(g.chunk * g.xwin() * kNbA));
  w.es = o; o += align256(sizeof(float2) * (size_t)(g.chunk * g.sets * g.jb * kNbA));
  w.extra = o; o += align256(extra_bytes);
  w.mixpart = o; o += align256(g.has_mix ? sizeof(float) * (size_t)(g.chunk * g.ib) : 0);
  w.acc = o; o += align256(g.shared ? sizeof(double2) * (size_t)(g.sets * g.jb * kNbA) : 0);
  w.cufft = o; o += align256(cufft_work);
  w.total = o;
}

// cuFFT plans for a full chunk and for the remainder (none without a batch), and both workspace layouts around their
// largest work area.  xi / hj: the block transforms of the convolution's cuFFT pipeline (audio / dL/dx windows, IR /
// dL/dIR partitions).  With synth (the reverb) also blk / pp, its IR synthesis (overlap-save blocks, polyphase), and
// the extra regions.  With g.shared also ir1: the J partitions of the one IR (forward) and of its summed gradient.
// Every IR plan transforms g.sets partition sets of J partitions per IR.  g.own_only: no plans and no work area.
struct Plans { PlanVal xi, hj, blk, pp; };
// blk / pp for a chunk of `items`; work: raised to their largest work area
int synth_plans(const Geom& g, int64_t items, Plans& p, size_t& work) {
  int rc;
  if ((rc = get_plan(2, g.nb, items * kBands * g.nbk, g.nb, g.nb, p.blk)) != DASP_OK) return rc;
  if ((rc = get_plan(2, g.nb, items * kBands * g.rpp, g.nb, g.nb, p.pp)) != DASP_OK) return rc;
  if (p.blk.work > work) work = p.blk.work;
  if (p.pp.work > work) work = p.pp.work;
  return DASP_OK;
}
struct Setup { Plans full, rem; PlanVal ir1; FwdWs fwd; BwdWs bwd; };
int conv_setup(const ConvGeom& g, const Geom* synth, Setup& s) {
  int rc;
  size_t work = 0;
  if (g.shared && g.bs > 0 && !g.own_only) {
    if ((rc = get_plan(2, kNbA, g.sets * g.jb, kNbA, kNbA, s.ir1)) != DASP_OK) return rc;
    work = s.ir1.work;
  }
  for (int64_t items : {g.bs > 0 ? g.chunk : 0, g.bs % g.chunk}) {
    if (items == 0 || g.own_only) continue;
    Plans& p = items == g.chunk ? s.full : s.rem;
    if ((rc = get_plan(2, kNbA, items * g.ib, kNbA, kNbA, p.xi)) != DASP_OK) return rc;
    if ((rc = get_plan(2, kNbA, items * g.sets * g.jb, kNbA, kNbA, p.hj)) != DASP_OK) return rc;
    if (p.xi.work > work) work = p.xi.work;
    if (p.hj.work > work) work = p.hj.work;
    if (synth && (rc = synth_plans(*synth, items, p, work)) != DASP_OK) return rc;
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
  out->xspec_c64 = g.bs * g.xwin() * kNbA;
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
// grid of an FFT kernel that gives each CTA a run of kConvRun units
unsigned runs(int64_t units) { return (unsigned)((units + kConvRun - 1) / kConvRun); }

// one-off opt-in to the large dynamic shared memory of the FFT kernels (per device, guarded by g_mu)
int configure_fft_kernels() {
  static std::map<int, bool> configured;
  int dev = 0;
  DASP_CUDA_OK(cudaGetDevice(&dev));
  if (!configured[dev]) {
    DASP_CUDA_OK(cudaFuncSetAttribute(ifft_shape_kernel<PartitionSink>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)kFftSmemBytes));
    DASP_CUDA_OK(cudaFuncSetAttribute(ifft_shape_kernel<PlanarSink>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)kFftSmemBytes));
    DASP_CUDA_OK(cudaFuncSetAttribute(x_fft_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFftSmemBytes));
    DASP_CUDA_OK(cudaFuncSetAttribute(ifft_mix_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFftSmemBytes));
    DASP_CUDA_OK(cudaFuncSetAttribute(g_fft_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFftSmemBytes));
    DASP_CUDA_OK(cudaFuncSetAttribute(ifft_dx_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFftSmemBytes));
    DASP_CUDA_OK(cudaFuncSetAttribute(ifft_irgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFftSmemBytes));
    DASP_CUDA_OK(cudaFuncSetAttribute(ifft_irtaps_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFftSmemBytes));
    DASP_CUDA_OK(cudaFuncSetAttribute(bus_fft_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFftSmemBytes));
    DASP_CUDA_OK(cudaFuncSetAttribute(bus_ifft_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFftSmemBytes));
    DASP_CUDA_OK(cudaFuncSetAttribute(tv_fft_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFftSmemBytes));
    DASP_CUDA_OK(cudaFuncSetAttribute(tv_ifft_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFftSmemBytes));
    DASP_CUDA_OK(cudaFuncSetAttribute(tvbus_gfft_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFftSmemBytes));
    DASP_CUDA_OK(cudaFuncSetAttribute(tvbus_ifft_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFftSmemBytes));
    DASP_CUDA_OK(cudaFuncSetAttribute(tvbusin_fft_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFftSmemBytes));
    DASP_CUDA_OK(cudaFuncSetAttribute(tvbusin_ifft_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFftSmemBytes));
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

// The partitions of `irs` impulse responses in hs (g.sets J per IR), transformed in place on the own FFT: x_fft_kernel
// with no audio windows.  A shared IR's before the first chunk; the bus's per chunk, in a launch of their own.
int ir_partition_spectra(const ConvGeom& g, const float* tw, float2* hs, int64_t irs, cudaStream_t st) {
  int rc = configure_fft_kernels();
  if (rc != DASP_OK) return rc;
  const int nparts = (int)(irs * g.sets * g.jb);
  x_fft_kernel<<<runs(nparts), kFusedThreads, kFftSmemBytes, st>>>(nullptr, nullptr, hs, tw, 0, (int)g.ib, (int)g.jb,
                                                                   g.n, g.leff, 1, 0, nparts);
  DASP_LAUNCH_OK("x_fft_kernel");
  return DASP_OK;
}

// y = (1 - mix) x + mix (x * IR), mix of item b at mix[b * mix_stride].  The caller has written IR taps t < leff as
// (left, right) pairs into the first half of partition slot t / kB of hs, and on the cuFFT pipeline zero-filled the
// slots first.  xs / hs receive the window / partition spectra.  own (own_fft_rows of x and hs): x_fft_kernel transforms
// both on the own FFT with the tables tw; otherwise cuFFT C2C does.  h_stride: item stride of hs in complex elements,
// g.sets J kNbA; 0 for one IR shared by the batch, whose partitions the caller has transformed already.
// g.sets == 2 (a true-stereo IR): hs holds set A then set B per IR, and the product is partition_mac_kernel<TS 1>.
// xs_ready (own only): the caller has already transformed the chunk's windows into xs.
int conv_fwd_chunk(const ConvGeom& g, const Plans& pl, bool own, const float* tw, const float* x, int in_chs, float2* xs,
                   float2* hs, int64_t h_stride, const float* mix, int mix_stride, float* y, unsigned char* ws,
                   const FwdWs& w, int64_t item0, int64_t items, cudaStream_t st, bool xs_ready = false) {
  float2* ys = (float2*)(ws + w.ys);
  const int I = (int)g.ib, J = (int)g.jb;
  const int nblk = (int)(items * I);
  if (own) {
    int rc = configure_fft_kernels();
    if (rc != DASP_OK) return rc;
    // one work list: the items*I audio windows, then the items*sets*J IR partitions (transformed in place in hs; the
    // zero padding of a partition depends on its index within its set, slot mod J)
    const int nwin = xs_ready ? 0 : nblk;
    const int nunits = nwin + (int)(h_stride != 0 ? items * g.sets * J : 0);
    if (nunits > 0) {
      x_fft_kernel<<<runs(nunits), kFusedThreads, kFftSmemBytes, st>>>(x, xs, hs, tw, item0, I, J, g.n, g.leff, in_chs,
                                                                        nwin, nunits);
      DASP_LAUNCH_OK("x_fft_kernel");
    }
    if (g.sets == 2) launch_mac<false, true, 1>(xs, hs, ys, I, J, h_stride != 0, I, items, 1.0f / (float)kNbA, st);
    else             launch_mac<false, true>(xs, hs, ys, I, J, h_stride != 0, I, items, 1.0f / (float)kNbA, st);
    DASP_LAUNCH_OK("partition_mac_kernel");
    ifft_mix_kernel<<<runs(nblk), kFusedThreads, kFftSmemBytes, st>>>(reinterpret_cast<const float*>(ys), tw, x, mix,
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

// ---- the IR synthesis of one chunk and its band contraction, for the reverb and noise_shaped_impulse_response ----
// The variant of a forward call (every variant draws the same Philox stream; the two own-FFT ones are bit-identical):
//   path 2 (default, device noise, nb == 8192): ir_synth_cluster_kernel for R <= kMaxClusterR, generator ->
//     ifft_shape_kernel for larger R or when the device cannot co-schedule the cluster;
//   path 1 (dasp_debug_reverb_path(2), R <= kMaxHookR): generator -> ifft_shape_kernel;
//   path 0: device noise up to kMaxSpectralR (dasp_debug_reverb_path(1), and any other nb): generator -> batched cuFFT
//     -> shape_ir_pp_kernel; the caller's noise tensor (parity mode) or a longer IR: time-domain noise in overlap-save
//     blocks -> C2C -> cmul_filter_pairs_kernel -> inverse C2C -> shape_ir_pairs_kernel.
struct Synth {
  int path;
  bool spectral;                  // polyphase_f: the filtered spectrum is drawn directly (paths 2, 1 and the first 0)
  const float2* H;                // the filter bank of that variant: half spectrum on the n1 grid, or the blocks' spectrum
  const float* tw;                // the FFT tables (paths 2 and 1)
  const float* noise;             // the caller's noise rows of length lp, or null (Philox keyed by *seed)
  const unsigned long long* seed;
  int64_t lp;
};
// L: the true IR length of the noise rows (g.L is 2 for noise_shaped_impulse_response at L = 1)
int choose_synth(const Geom& g, int64_t L, const float* noise, const unsigned long long* seed, double sr,
                 cudaStream_t st, Synth& sy) {
  sy = Synth{0, polyphase_f(g, noise == nullptr), nullptr, nullptr, noise, seed, L + g.P};
  int rc = get_filterbank(g, sr, sy.spectral, st, &sy.H);
  if (rc != DASP_OK) return rc;
  if (sy.spectral && g.nb == fft8k::kN && g.L < (int64_t)1 << 31 && debug_reverb_path() != 1)
    sy.path = debug_reverb_path() == 2 && g.rpp <= kMaxHookR ? 1 : 2;
  if (sy.path != 0 && (rc = get_fft_tables(st, &sy.tw)) != DASP_OK) return rc;
  return DASP_OK;
}

// Taps t < leff of the chunk's items to the sink (the reverb: partition slots; noise_shaped_impulse_response: planar
// rows).  params: the chunk's 25-wide rows; C: its filtered noise, kept for the backward when keep_f; pl / cufft: the
// cuFFT plans and work area of path 0.  st / prio: the stream and launch priority (the reverb's side stream when it
// pipelines, which it does on paths 2 and 1 only: path 0 shares the cuFFT work area with the convolution).
template <class Sink>
int synth_chunk(const Geom& g, const Synth& sy, const Sink& out, const float* params, float2* C, bool keep_f,
                const Plans& pl, void* cufft, int64_t item0, int64_t items, cudaStream_t st, const int* prio) {
  g_last_fused = sy.path;
  const int nbk = (int)g.nbk, nb = (int)g.nb, R = (int)g.rpp;
  int rc;
  if (sy.path != 0) {
    if (sy.path == 2 && g.rpp <= kMaxClusterR &&
        dispatch_fused(R, sy.H, sy.tw, params, out, keep_f ? C : nullptr, item0, items, g.L, g.leff, sy.seed, st, prio)) {
      DASP_LAUNCH_OK("ir_synth_cluster_kernel");
      return DASP_OK;
    }
    dispatch_spectral(R, C, sy.H, item0, items, nb, sy.seed, /*planar=*/true, st, prio);
    DASP_LAUNCH_OK("spectral_gen_kernel");
    return launch_ifft_shape(C, sy.tw, params, out, keep_f, items, g, st, prio);
  }
  if (sy.spectral) {
    // one inverse transform of the drawn spectrum (polyphase layout)
    dispatch_spectral(R, C, sy.H, item0, items, nb, sy.seed, /*planar=*/false, st, nullptr);
    DASP_LAUNCH_OK("spectral_gen_kernel");
    if ((rc = exec_c2c(pl.pp, cufft, C, CUFFT_INVERSE, st)) != DASP_OK) return rc;
    shape_ir_pp_kernel<<<dim3((unsigned)((g.leff + 255) / 256), (unsigned)items), 256, 0, st>>>(C, params, out, g.L,
                                                                                              g.leff, R, nb);
    DASP_LAUNCH_OK("shape_ir_pp_kernel");
    return DASP_OK;
  }
  const dim3 gblk((unsigned)nbk, kBands, (unsigned)items);
  if (sy.noise) noise_pairs_layout_kernel<<<gblk, 256, 0, st>>>(sy.noise, C, item0, nbk, nb, (int)g.hop, sy.lp);
  else          noise_pairs_philox_kernel<<<gblk, 256, 0, st>>>(C, item0, nbk, nb, (int)g.hop, sy.seed);
  DASP_LAUNCH_OK("reverb noise kernel");
  if ((rc = exec_c2c(pl.blk, cufft, C, CUFFT_FORWARD, st)) != DASP_OK) return rc;
  cmul_filter_pairs_kernel<<<gblk, 256, 0, st>>>(C, sy.H, nbk, nb);
  DASP_LAUNCH_OK("cmul_filter_pairs_kernel");
  if ((rc = exec_c2c(pl.blk, cufft, C, CUFFT_INVERSE, st)) != DASP_OK) return rc;
  shape_ir_pairs_kernel<<<dim3((unsigned)nbk, (unsigned)items), 256, 0, st>>>(C, params, out, g.L, g.leff, nbk, nb,
                                                                           (int)g.hop, (int)g.P);
  DASP_LAUNCH_OK("shape_ir_pairs_kernel");
  return DASP_OK;
}

// The band contraction of the backward on the chunk's dL/dIR Et (partition layout) and its filtered noise C (layout
// polyphase_f): nparts partials of the 24 band-parameter gradients per item into part, for reverb_param_grad_kernel
int ir_grad_chunk(const Geom& g, bool polyphase, const float2* Et, const float2* C, const float* params, float* part,
                  int64_t items, cudaStream_t st, int& nparts) {
  const int J = (int)g.jb, nb = (int)g.nb;
  nparts = (int)(polyphase ? g.nparts_pp() : g.nbk);
  if (polyphase) {
    ir_grad_pp_kernel<<<dim3((unsigned)nparts, (unsigned)items), 256, 0, st>>>(Et, C, params, part, g.L, g.leff, J,
                                                                              (int)g.rpp, nb);
  } else {
    ir_grad_pairs_kernel<<<dim3((unsigned)nparts, (unsigned)items), 256, 0, st>>>(Et, C, params, part, g.L, g.leff, J,
                                                                                 nparts, nb, (int)g.hop, (int)g.P);
  }
  DASP_LAUNCH_OK("ir_grad kernel");
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
    cudaStreamDestroy(kv.second.side);
    cudaEventDestroy(kv.second.done);
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
  Synth sy;
  if ((rc = choose_synth(g, g.L, noise, seed, (double)sample_rate, st, sy)) != DASP_OK) return rc;
  Setup s{};
  if ((rc = conv_setup(g, &g, s)) != DASP_OK) return rc;
  if ((rc = check_workspace("reverb fwd", s.fwd.total, workspace_bytes)) != DASP_OK) return rc;
  const FwdWs& w = s.fwd;
  unsigned char* base = (unsigned char*)workspace;
  const int I = (int)g.ib, J = (int)g.jb;

  // Pipeline: chunk k + 1's synthesis runs on a side stream while chunk k's convolution runs on st.  The synthesis holds
  // only the SMs its clusters fit on (17 clusters of 6 = 102 of 132 on an H100 SXM), the convolution fills the rest.
  // Every chunk's synthesis goes to the one side stream, at the greatest priority so that its clusters are dispatched
  // before convolution CTAs, and st waits for it before chunk k's convolution; the last of these waits joins every
  // side-stream launch back into st,
  // so nothing outlives the call, and under stream capture the fork and join are graph edges.  This needs the chunks'
  // slots disjoint: the synthesis writes only f_save / irspec_save slots (kept when a backward follows; otherwise they
  // share one workspace slot), and neither side uses the shared cuFFT work area (own-FFT synthesis and convolution).
  // One side stream, not one per chunk: a cluster launch queued behind a running one stays pending for the whole chunk,
  // and while it was pending the convolution ran at about 12 of the 30 free SMs' worth of its full rate (H100 SXM; the
  // block scheduler appears to hold SMs back for the pending cluster).  With one stream, the next chunk's clusters are
  // launched only when the running chunk ends, and the convolution gets the free SMs (DESIGN.md §0).
  const bool pipelined = sy.path != 0 && f_save && irspec_save && own_fft_rows(n, x, irspec_save);
  SideStream* side = nullptr;
  if (pipelined) {
    if ((rc = get_side_stream(&side)) != DASP_OK) return rc;
    DASP_CUDA_OK(cudaEventRecord(side->fork, st));   // the seed word and the parameters are written on st
    DASP_CUDA_OK(cudaStreamWaitEvent(side->side, side->fork, 0));
  }
  const int* prio = pipelined ? &side->prio : nullptr;
  // The audio windows do not depend on the IR: when every item has its xspec_save slot, the whole batch's windows are
  // transformed on st right after chunk 0's synthesis is launched, so they run on the SMs its clusters leave free
  // instead of waiting behind it.  The chunks' convolutions then transform only their IR partitions.
  const bool windows_first = pipelined && xspec_save != nullptr;

  for (int64_t item0 = 0, k = 0; item0 < bs; item0 += g.chunk, ++k) {
    const int64_t items = (bs - item0 < g.chunk) ? bs - item0 : g.chunk;
    const Plans& pl = (items == g.chunk) ? s.full : s.rem;
    const cudaStream_t sst = pipelined ? side->side : st;      // the stream of this chunk's synthesis
    // kept for the backward when the caller passes *_save buffers, transient workspace otherwise
    float2* C = f_save ? reinterpret_cast<float2*>(f_save) + item0 * kBands * g.pair_c64()
                       : reinterpret_cast<float2*>(base + w.extra);
    float2* xs = xspec_save ? (float2*)xspec_save + item0 * I * (int64_t)kNbA : (float2*)(base + w.xsp);
    float2* hs = irspec_save ? (float2*)irspec_save + item0 * J * (int64_t)kNbA : (float2*)(base + w.hsp);
    const bool own_conv = own_fft_rows(n, x, hs);
    const float* tw = nullptr;
    if (own_conv && (rc = get_fft_tables(st, &tw)) != DASP_OK) return rc;

    // IR taps t < leff land as (left, right) pairs in the first half of partition t / kB of hs.  x_fft_kernel reads
    // nothing else of hs; the cuFFT transform of the partitions reads whole slots, so they are zero-filled first
    if (!own_conv) DASP_CUDA_OK(cudaMemsetAsync(hs, 0, sizeof(float2) * items * J * kNbA, st));
    if ((rc = synth_chunk(g, sy, PartitionSink{hs, J}, params + item0 * 25, C, f_save != nullptr, pl, base + w.cufft,
                          item0, items, sst, prio)) != DASP_OK)
      return rc;
    if (windows_first && k == 0) {
      if ((rc = configure_fft_kernels()) != DASP_OK) return rc;
      const int nwin = (int)(bs * I);
      x_fft_kernel<<<runs(nwin), kFusedThreads, kFftSmemBytes, st>>>(x, (float2*)xspec_save, nullptr, tw, 0, I, J, g.n,
                                                                     g.leff, (int)in_chs, nwin, nwin);
      DASP_LAUNCH_OK("x_fft_kernel");
    }
    if (pipelined) {
      DASP_CUDA_OK(cudaEventRecord(side->done, sst));
      DASP_CUDA_OK(cudaStreamWaitEvent(st, side->done, 0));
    }
    if ((rc = conv_fwd_chunk(g, pl, own_conv, tw, x, (int)in_chs, xs, hs, J * (int64_t)kNbA, params + 24, 25, y, base,
                             w, item0, items, st, windows_first)) != DASP_OK)
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
  const bool polyphase = polyphase_f(g, device_noise != 0);   // the layout the forward left in f_save
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
  const int I = (int)g.ib, J = (int)g.jb;

  for (int64_t item0 = 0; item0 < bs; item0 += g.chunk) {
    const int64_t items = (bs - item0 < g.chunk) ? bs - item0 : g.chunk;
    const Plans& pl = (items == g.chunk) ? s.full : s.rem;
    const float2* C = reinterpret_cast<const float2*>(f_save) + item0 * kBands * g.pair_c64();
    const float2* xs = (const float2*)xspec_save + item0 * I * (int64_t)kNbA;
    const float2* hs = (const float2*)irspec_save + item0 * J * (int64_t)kNbA;

    const bool own_conv = own_fft_rows(n, gy, nullptr);
    // dL/dIR through the band parameters on the own FFT needs the polyphase f_save at nb = 8192
    const bool own_irgrad = own_conv && polyphase && g.nb == fft8k::kN && g.L < (int64_t)1 << 31;
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
    } else if ((rc = ir_grad_chunk(g, polyphase, ws_es, C, params + item0 * 25, ws_irpart, items, st, nparts)) !=
               DASP_OK) {
      return rc;
    }
    reverb_param_grad_kernel<<<(unsigned)((items * 25 + 127) / 128), 128, 0, st>>>(ws_irpart, ws_mixpart, params, gparams,
                                                                                   item0, items, nparts, I);
    DASP_LAUNCH_OK("reverb_param_grad_kernel");
  }
  return DASP_OK;
}

// ------------------------------------------------------------------ convolution_reverberation and convolution_bus
// The ops whose impulse response the caller supplies run one host stage per direction (caller_ir_fwd / caller_ir_bwd):
// the argument checks, the lock, the workspace, the *_save buffers or their transient workspace slots, the IR taps
// packed into their partition slots (ir_pack_kernel), and the chunk loop.  One IR for the whole batch (g.shared) is the
// item stride 0 of the IR spectra: packed and transformed once before the first chunk; in the backward,
// irgrad_sum_kernel sums the items' dL/dIR partition spectra in fp64 (factor mix[b], or 1 without a mix) and the sum is
// transformed once after the last chunk.  dL/dIR taps [leff, L) reach no output and get their zeros from one memset
// after the chunk loop.  The op (ConvOp, BusOp) supplies only its IR rows (ir_rows per item, packed two per partition
// set; kOddSelf: an odd last row pairs with itself, else with 0), its products per chunk (fwd_chunk; bwd_chunk, which
// leaves the dL/dIR partitions in the es region in the form e) and the inverse transform of those partitions into the
// caller's rows (ir_taps, with the factor mix[b] or none).
namespace {
int g_conv_last_path[2] = {0, 0};                    // test hook: dispatch of the last conv forward / backward
int g_bus_last_path[2] = {0, 0};                     // test hook: dispatch of the last bus forward / backward

extern "C++" {
template <class Op>
int caller_ir_fwd(const Op& op, const ConvGeom& g, const float* x, const float* ir, const float* mix, float* y,
                  void* xspec_save, void* irspec_save, void* workspace, int64_t workspace_bytes, void* stream) {
  if (g.bs == 0) return DASP_OK;
  DASP_REQUIRE(x && ir && (mix || !g.has_mix) && y && workspace, "%s: null pointer", Op::kFwd);
  DASP_REQUIRE((xspec_save == nullptr) == (irspec_save == nullptr), "%s: pass both *_save buffers or neither",
               Op::kFwd);
  DASP_REQUIRE(!g.own_only || (g.n % 4 == 0 && aligned16(x)),
               "%s: x needs n %% 4 == 0 and 16-byte aligned rows, got n=%lld", Op::kFwd, (long long)g.n);
  cudaStream_t st = (cudaStream_t)stream;
  std::lock_guard<std::mutex> lk(g_mu);
  Setup s{};
  int rc = conv_setup(g, nullptr, s);
  if (rc != DASP_OK) return rc;
  if ((rc = check_workspace(Op::kFwd, s.fwd.total, workspace_bytes)) != DASP_OK) return rc;
  const FwdWs& w = s.fwd;
  unsigned char* base = (unsigned char*)workspace;
  const int J = (int)g.jb;
  const int64_t h_stride = g.shared ? 0 : g.sets * J * (int64_t)kNbA;
  float2* const hs0 = irspec_save ? (float2*)irspec_save : (float2*)(base + w.hsp);
  const float* tw = nullptr;

  // IR taps t < leff of items [item0, item0 + items) into their partition slots; the cuFFT transform of the partitions
  // reads whole slots, x_fft_kernel only the taps ir_pack_kernel writes
  auto fill_ir = [&](float2* hs, bool own, int64_t item0, int64_t items) -> int {
    if (!own) DASP_CUDA_OK(cudaMemsetAsync(hs, 0, sizeof(float2) * items * g.sets * J * kNbA, st));
    ir_pack_kernel<<<dim3((unsigned)((g.leff + 255) / 256), (unsigned)items, (unsigned)g.sets), 256, 0, st>>>(
        ir, hs, item0, J, g.L, g.leff, op.ir_rows, Op::kOddSelf);
    DASP_LAUNCH_OK("ir_pack_kernel");
    return DASP_OK;
  };
  if (g.shared) {
    const bool own = g.own_only || own_fft_rows(g.n, x, hs0);
    if ((rc = fill_ir(hs0, own, 0, 1)) != DASP_OK) return rc;
    if (own && (rc = get_fft_tables(st, &tw)) != DASP_OK) return rc;
    rc = own ? ir_partition_spectra(g, tw, hs0, 1, st) : exec_c2c(s.ir1, base + w.cufft, hs0, CUFFT_FORWARD, st);
    if (rc != DASP_OK) return rc;
  }
  for (int64_t item0 = 0; item0 < g.bs; item0 += g.chunk) {
    const int64_t items = (g.bs - item0 < g.chunk) ? g.bs - item0 : g.chunk;
    const Plans& pl = (items == g.chunk) ? s.full : s.rem;
    float2* xs = xspec_save ? (float2*)xspec_save + item0 * g.xwin() * (int64_t)kNbA : (float2*)(base + w.xsp);
    float2* hs = irspec_save ? hs0 + item0 * h_stride : hs0;
    const bool own = g.own_only || own_fft_rows(g.n, x, hs);
    if (!g.shared && (rc = fill_ir(hs, own, item0, items)) != DASP_OK) return rc;
    if (own && (rc = get_fft_tables(st, &tw)) != DASP_OK) return rc;
    if ((rc = op.fwd_chunk(g, pl, own, tw, x, mix, xs, hs, h_stride, y, base, w, item0, items, st)) != DASP_OK)
      return rc;
  }
  return DASP_OK;
}

// x and mix (and gmix) only with g.has_mix: the backward needs x for the dL/dmix partials alone
template <class Op>
int caller_ir_bwd(const Op& op, const ConvGeom& g, const float* gy, const float* x, const float* mix,
                  const void* xspec_save, const void* irspec_save, float* gx, float* gir, float* gmix, void* workspace,
                  int64_t workspace_bytes, void* stream) {
  if (g.bs == 0) return DASP_OK;
  DASP_REQUIRE(gy && xspec_save && irspec_save && gx && workspace && (!g.has_mix || (x && mix && gmix)),
               "%s: null pointer", Op::kBwd);
  DASP_REQUIRE(!g.own_only || (g.n % 4 == 0 && aligned16(gy)),
               "%s: gy needs n %% 4 == 0 and 16-byte aligned rows, got n=%lld", Op::kBwd, (long long)g.n);
  cudaStream_t st = (cudaStream_t)stream;
  std::lock_guard<std::mutex> lk(g_mu);
  Setup s{};
  int rc = conv_setup(g, nullptr, s);
  if (rc != DASP_OK) return rc;
  if ((rc = check_workspace(Op::kBwd, s.bwd.total, workspace_bytes)) != DASP_OK) return rc;
  const BwdWs& w = s.bwd;
  unsigned char* base = (unsigned char*)workspace;
  float2* ws_es = (float2*)(base + w.es);
  const float* ws_mixpart = (const float*)(base + w.mixpart);
  double2* ws_acc = (double2*)(base + w.acc);
  const int I = (int)g.ib, J = (int)g.jb;
  const int64_t per_ir = g.sets * J * (int64_t)kNbA;
  const int64_t h_stride = g.shared ? 0 : per_ir;
  const float* tw = nullptr;
  bool own = false;

  for (int64_t item0 = 0; item0 < g.bs; item0 += g.chunk) {
    const int64_t items = (g.bs - item0 < g.chunk) ? g.bs - item0 : g.chunk;
    const Plans& pl = (items == g.chunk) ? s.full : s.rem;
    const float2* xs = (const float2*)xspec_save + item0 * g.xwin() * (int64_t)kNbA;
    const float2* hs = (const float2*)irspec_save + item0 * h_stride;
    own = g.own_only || own_fft_rows(g.n, gy, nullptr);
    const IrGrad e = gir == nullptr ? IrGrad::kNone
                                    : (own ? IrGrad::kPlanar : (g.shared ? IrGrad::kSpectra : IrGrad::kTime));
    if (own && (rc = get_fft_tables(st, &tw)) != DASP_OK) return rc;
    rc = op.bwd_chunk(g, pl, own, e, tw, gy, x, mix, xs, hs, h_stride, gx, base, w, item0, items, st);
    if (rc != DASP_OK) return rc;
    if (e != IrGrad::kNone && g.shared) {
      irgrad_sum_kernel<<<(unsigned)((per_ir + 255) / 256), 256, 0, st>>>(ws_es, mix, ws_acc, item0, (int)items,
                                                                          per_ir, item0 + items == g.bs);
      DASP_LAUNCH_OK("irgrad_sum_kernel");
    } else if (e != IrGrad::kNone && (rc = op.ir_taps(g, own, tw, ws_es, mix, gir, item0, items, st)) != DASP_OK) {
      return rc;
    }
    if (g.has_mix) {
      conv_mix_grad_kernel<<<(unsigned)((items + 127) / 128), 128, 0, st>>>(ws_mixpart, gmix, item0, items, I);
      DASP_LAUNCH_OK("conv_mix_grad_kernel");
    }
  }
  if (!gir) return DASP_OK;
  if (g.shared) {
    // the summed partition spectra, rounded to fp32 in item 0's slots of es: sets J inverse transforms for the one IR
    if (!own && (rc = exec_c2c(s.ir1, base + w.cufft, ws_es, CUFFT_INVERSE, st)) != DASP_OK) return rc;
    if ((rc = op.ir_taps(g, own, tw, ws_es, nullptr, gir, 0, 1, st)) != DASP_OK) return rc;
  }
  if (g.L > g.leff) {
    DASP_CUDA_OK(cudaMemset2DAsync(gir + g.leff, sizeof(float) * g.L, 0, sizeof(float) * (g.L - g.leff),
                                   (size_t)((g.shared ? 1 : g.bs) * op.ir_rows), st));
  }
  return DASP_OK;
}
}  // extern "C++"

// convolution_reverberation: y = (1 - mix) x + mix (x * IR) on conv_fwd_chunk / conv_bwd_chunk.  x is mono or stereo;
// the IR mono (feeding both channels), stereo, or true-stereo (ir_chs 4: two partition sets per IR, g.sets = 2).
struct ConvOp {
  static constexpr const char* kFwd = "conv fwd";
  static constexpr const char* kBwd = "conv bwd";
  static constexpr bool kOddSelf = true;
  int in_chs, ir_rows;
  int fwd_chunk(const ConvGeom& g, const Plans& pl, bool own, const float* tw, const float* x, const float* mix,
                float2* xs, float2* hs, int64_t h_stride, float* y, unsigned char* ws, const FwdWs& w, int64_t item0,
                int64_t items, cudaStream_t st) const {
    g_conv_last_path[0] = (own ? 1 : 0) | (g.shared ? 2 : 0) | (g.sets == 2 ? 4 : 0);
    return conv_fwd_chunk(g, pl, own, tw, x, in_chs, xs, hs, h_stride, mix, 1, y, ws, w, item0, items, st);
  }
  int bwd_chunk(const ConvGeom& g, const Plans& pl, bool own, IrGrad e, const float* tw, const float* gy,
                const float* x, const float* mix, const float2* xs, const float2* hs, int64_t h_stride, float* gx,
                unsigned char* ws, const BwdWs& w, int64_t item0, int64_t items, cudaStream_t st) const {
    // bit 0: own FFT, bit 1: fused correlations, bit 2: dL/dIR computed, bit 3: one IR shared by the batch, bit 4: a
    // true-stereo IR
    g_conv_last_path[1] = (own ? 1 : 0) | (fused_corr(e, (int)g.ib, (int)g.jb, g.sets) ? 2 : 0) |
                          (e != IrGrad::kNone ? 4 : 0) | (g.shared ? 8 : 0) | (g.sets == 2 ? 16 : 0);
    return conv_bwd_chunk(g, pl, own, e, tw, gy, x, in_chs, xs, hs, h_stride, mix, 1, gx, ws, w, item0, items, st);
  }
  // dL/dIR taps [0, leff) of IRs [item0, item0 + items) from their partitions in es: planar spectra (own), or
  // time-domain pairs after the inverse cuFFT
  int ir_taps(const ConvGeom& g, bool own, const float* tw, const float2* es, const float* mix, float* gir,
              int64_t item0, int64_t items, cudaStream_t st) const {
    const int J = (int)g.jb;
    if (own) {
      const int nunits = (int)(items * g.sets * J);
      ifft_irtaps_kernel<<<persistent_grid(nunits), kFusedThreads, kFftSmemBytes, st>>>(
          reinterpret_cast<const float*>(es), tw, mix, gir, item0, J, g.sets, g.L, g.leff, ir_rows, nunits);
      DASP_LAUNCH_OK("ifft_irtaps_kernel");
    } else {
      irtaps_unpack_kernel<<<dim3((unsigned)((g.leff + 255) / 256), (unsigned)items, (unsigned)g.sets), 256, 0, st>>>(
          es, mix, gir, item0, J, g.L, g.leff, ir_rows);
      DASP_LAUNCH_OK("irtaps_unpack_kernel");
    }
    return DASP_OK;
  }
};

// the geometry and argument checks of dasp_conv_* (one IR per item) and dasp_conv_shared_* (one IR for the batch)
int ir_sets(int64_t ir_chs) { return ir_chs == 4 ? 2 : 1; }
int conv_op_geom(bool shared, int sets, int64_t bs, int64_t n, int64_t ir_len, int64_t chunk_items, ConvGeom& g) {
  int rc = make_conv_geom(bs, n, ir_len, chunk_items, g);
  if (rc != DASP_OK) return rc;
  g.shared = shared;
  g.sets = sets;
  return DASP_OK;
}
int conv_op_geometry(bool shared, int sets, int64_t bs, int64_t n, int64_t ir_len, int64_t chunk_items,
                     dasp_conv_geom* out) {
  DASP_REQUIRE(out != nullptr, "conv geometry: null out");
  ConvGeom g;
  int rc = conv_op_geom(shared, sets, bs, n, ir_len, chunk_items, g);
  if (rc != DASP_OK) return rc;
  return put_conv_geometry(g, nullptr, out);
}
int check_conv_chs(int64_t in_chs, int64_t ir_chs) {
  DASP_REQUIRE((in_chs == 1 || in_chs == 2) && (ir_chs == 1 || ir_chs == 2 || ir_chs == 4),
               "conv: only mono/stereo signals and mono/stereo/true-stereo IRs");
  return DASP_OK;
}

int conv_op_fwd(bool shared, const float* x, int64_t in_chs, const float* ir, int64_t ir_chs, int64_t ir_len,
                const float* mix, float* y, void* xspec_save, void* irspec_save, void* workspace,
                int64_t workspace_bytes, int64_t bs, int64_t n, int64_t chunk_items, void* stream) {
  ConvGeom g;
  int rc = conv_op_geom(shared, ir_sets(ir_chs), bs, n, ir_len, chunk_items, g);
  if (rc != DASP_OK || (rc = check_conv_chs(in_chs, ir_chs)) != DASP_OK) return rc;
  return caller_ir_fwd(ConvOp{(int)in_chs, (int)ir_chs}, g, x, ir, mix, y, xspec_save, irspec_save, workspace,
                       workspace_bytes, stream);
}

int conv_op_bwd(bool shared, const float* gy, const float* x, int64_t in_chs, int64_t ir_chs, int64_t ir_len,
                const float* mix, const void* xspec_save, const void* irspec_save, float* gx, float* gir, float* gmix,
                void* workspace, int64_t workspace_bytes, int64_t bs, int64_t n, int64_t chunk_items, void* stream) {
  ConvGeom g;
  int rc = conv_op_geom(shared, ir_sets(ir_chs), bs, n, ir_len, chunk_items, g);
  if (rc != DASP_OK || (rc = check_conv_chs(in_chs, ir_chs)) != DASP_OK) return rc;
  return caller_ir_bwd(ConvOp{(int)in_chs, (int)ir_chs}, g, gy, x, mix, xspec_save, irspec_save, gx, gir, gmix,
                       workspace, workspace_bytes, stream);
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

// ------------------------------------------------------------------ convolution_bus
// y[:, o] = sum_s x[:, s] * h[:, s, o] through the stage above on the own FFT only: P = ceil(S / 2) window spectra per
// block (g.p) and NH = ceil(S O / 2) partition sets per IR (g.sets), no mix.  The row-pair transforms, the products and
// the inverse transforms are the bus kernels; the IR partitions go through x_fft_kernel's partition units.
namespace {
// register-cached products when both operand lists fit (MAXB 12 / 16), else from L2 (templates: C++ linkage)
extern "C++" {
template <int MODE, int O>
void launch_bus_mac_o(const ConvGeom& g, int S, const float2* X, const float2* H, int64_t hstride, const float2* G,
                      float2* Out, int64_t items, cudaStream_t st) {
  dim3 grid((kNbA / 2 + 1 + 127) / 128, (unsigned)items);
  const int I = (int)g.ib, J = (int)g.jb, m = I > J ? I : J;
  const float inv = 1.0f / (float)kNbA;
  if (m <= 12)      bus_mac_kernel<12, MODE, O><<<grid, 128, 0, st>>>(X, H, hstride, G, Out, S, I, J, inv);
  else if (m <= 16) bus_mac_kernel<16, MODE, O><<<grid, 128, 0, st>>>(X, H, hstride, G, Out, S, I, J, inv);
  else              bus_mac_kernel<0, MODE, O><<<grid, 128, 0, st>>>(X, H, hstride, G, Out, S, I, J, inv);
}
// O >= 3 outputs: one slice per output pair (forward), input pair (dL/dx) or partition set (dL/dIR) of each item
template <int MODE>
void launch_busmc_mac(const ConvGeom& g, int S, int O, const float2* X, const float2* H, int64_t hstride,
                      const float2* G, float2* Out, int64_t items, cudaStream_t st) {
  const int slices = MODE == BUS_FWD ? (O + 1) / 2 : (MODE == BUS_DX ? g.p : g.sets);
  dim3 grid((kNbA / 2 + 1 + 127) / 128, (unsigned)slices, (unsigned)items);
  const int I = (int)g.ib, J = (int)g.jb, m = I > J ? I : J;
  const float inv = 1.0f / (float)kNbA;
  if (m <= 12)      busmc_mac_kernel<12, MODE><<<grid, 128, 0, st>>>(X, H, hstride, G, Out, S, O, I, J, inv);
  else if (m <= 16) busmc_mac_kernel<16, MODE><<<grid, 128, 0, st>>>(X, H, hstride, G, Out, S, O, I, J, inv);
  else              busmc_mac_kernel<0, MODE><<<grid, 128, 0, st>>>(X, H, hstride, G, Out, S, O, I, J, inv);
}
template <int MODE>
int launch_bus_mac(const ConvGeom& g, int S, int O, const float2* X, const float2* H, int64_t hstride, const float2* G,
                   float2* Out, int64_t items, cudaStream_t st) {
  if (O == 2)      launch_bus_mac_o<MODE, 2>(g, S, X, H, hstride, G, Out, items, st);
  else if (O == 1) launch_bus_mac_o<MODE, 1>(g, S, X, H, hstride, G, Out, items, st);
  else             launch_busmc_mac<MODE>(g, S, O, X, H, hstride, G, Out, items, st);
  DASP_LAUNCH_OK("bus_mac_kernel");
  return DASP_OK;
}
}  // extern "C++"
bool bus_mac_cached(const ConvGeom& g) { return (g.ib > g.jb ? g.ib : g.jb) <= 16; }

struct BusOp {
  static constexpr const char* kFwd = "conv bus fwd";
  static constexpr const char* kBwd = "conv bus bwd";
  static constexpr bool kOddSelf = false;
  int S, O, ir_rows;                                 // inputs, outputs, IR rows S O
  int fwd_chunk(const ConvGeom& g, const Plans&, bool own, const float* tw, const float* x, const float*, float2* xs,
                float2* hs, int64_t h_stride, float* y, unsigned char* ws, const FwdWs& w, int64_t item0,
                int64_t items, cudaStream_t st) const {
    // bit 0: own FFT, bit 1: one IR shared by the batch, bit 2: register-cached products, bit 3: O >= 3 outputs
    g_bus_last_path[0] = (own ? 1 : 0) | (g.shared ? 2 : 0) | (bus_mac_cached(g) ? 4 : 0) | (O > 2 ? 8 : 0);
    int rc = configure_fft_kernels();
    if (rc != DASP_OK) return rc;
    if (h_stride != 0 && (rc = ir_partition_spectra(g, tw, hs, items, st)) != DASP_OK) return rc;
    float2* ys = (float2*)(ws + w.ys);
    const int I = (int)g.ib, Q = (O + 1) / 2, nwin = (int)(items * g.p * I), nblk = (int)(items * Q * I);
    bus_fft_kernel<<<runs(nwin), kFusedThreads, kFftSmemBytes, st>>>(x, xs, tw, item0, S, g.p, I, g.n, 0, nwin);
    DASP_LAUNCH_OK("bus_fft_kernel");
    if ((rc = launch_bus_mac<BUS_FWD>(g, S, O, xs, hs, h_stride, nullptr, ys, items, st)) != DASP_OK) return rc;
    bus_ifft_kernel<<<runs(nblk), kFusedThreads, kFftSmemBytes, st>>>(reinterpret_cast<const float*>(ys), tw, y, item0,
                                                                      O, Q, I, g.n, g.n, 1, nblk);
    DASP_LAUNCH_OK("bus_ifft_kernel");
    return DASP_OK;
  }
  int bwd_chunk(const ConvGeom& g, const Plans&, bool own, IrGrad e, const float* tw, const float* gy, const float*,
                const float*, const float2* xs, const float2* hs, int64_t h_stride, float* gx, unsigned char* ws,
                const BwdWs& w, int64_t item0, int64_t items, cudaStream_t st) const {
    // bit 0: own FFT, bit 1: register-cached products, bit 2: dL/dIR computed, bit 3: one IR shared by the batch,
    // bit 4: O >= 3 outputs
    g_bus_last_path[1] = (own ? 1 : 0) | (bus_mac_cached(g) ? 2 : 0) | (e != IrGrad::kNone ? 4 : 0) |
                         (g.shared ? 8 : 0) | (O > 2 ? 16 : 0);
    int rc = configure_fft_kernels();
    if (rc != DASP_OK) return rc;
    float2* gs = (float2*)(ws + w.gs);
    float2* ds = (float2*)(ws + w.ds);
    const int I = (int)g.ib, Q = (O + 1) / 2, nblk = (int)(items * Q * I), nwin = (int)(items * g.p * I);
    bus_fft_kernel<<<runs(nblk), kFusedThreads, kFftSmemBytes, st>>>(gy, gs, tw, item0, O, Q, I, g.n, 1, nblk);
    DASP_LAUNCH_OK("bus_fft_kernel");
    if ((rc = launch_bus_mac<BUS_DX>(g, S, O, xs, hs, h_stride, gs, ds, items, st)) != DASP_OK) return rc;
    bus_ifft_kernel<<<runs(nwin), kFusedThreads, kFftSmemBytes, st>>>(reinterpret_cast<const float*>(ds), tw, gx, item0,
                                                                      S, g.p, I, g.n, g.n, 1, nwin);
    DASP_LAUNCH_OK("bus_ifft_kernel");
    if (e == IrGrad::kNone) return DASP_OK;          // a fixed IR: no dL/dIR work at all
    return launch_bus_mac<BUS_DIR>(g, S, O, xs, hs, 0, gs, (float2*)(ws + w.es), items, st);
  }
  // dL/dIR taps [0, leff) of IRs [item0, item0 + items): the first half of the inverse of each partition
  int ir_taps(const ConvGeom& g, bool, const float* tw, const float2* es, const float*, float* gir, int64_t item0,
              int64_t items, cudaStream_t st) const {
    const int J = (int)g.jb, nparts = (int)(items * g.sets * J);
    bus_ifft_kernel<<<runs(nparts), kFusedThreads, kFftSmemBytes, st>>>(reinterpret_cast<const float*>(es), tw, gir,
                                                                        item0, ir_rows, g.sets, J, g.L, g.leff, 0,
                                                                        nparts);
    DASP_LAUNCH_OK("bus_ifft_kernel");
    return DASP_OK;
  }
};

// multichannel_convolution: the bus with up to DASP_CONV_MC_MAX_OUTPUTS outputs, and its own messages
struct McOp : BusOp {
  static constexpr const char* kFwd = "conv mc fwd";
  static constexpr const char* kBwd = "conv mc bwd";
};

// the argument checks of the bus (max_out 2, dasp_conv_bus_*) and of multichannel_convolution (max_out
// DASP_CONV_MC_MAX_OUTPUTS, dasp_conv_mc_*), filling their geometry.  Q = ceil(O / 2) output and gradient spectra per
// block: the Q - 1 beyond the first are g.ex
int make_bus_geom(bool shared, int64_t bs, int64_t n, int64_t L, int64_t S, int64_t O, int max_out, int64_t chunk,
                  ConvGeom& g) {
  const char* what = max_out == 2 ? "conv bus" : "conv mc";
  DASP_REQUIRE(S >= 1 && S <= DASP_CONV_BUS_MAX_INPUTS, "%s: 1 to %d inputs are supported, got %lld", what,
               DASP_CONV_BUS_MAX_INPUTS, (long long)S);
  if (max_out == 2)
    DASP_REQUIRE(O == 1 || O == 2, "conv bus: a mono (1) or stereo (2) bus, got %lld outputs", (long long)O);
  else
    DASP_REQUIRE(O >= 1 && O <= max_out, "%s: 1 to %d outputs are supported, got %lld", what, max_out, (long long)O);
  int rc = make_conv_geom(bs, n, L, chunk, g);
  if (rc != DASP_OK) return rc;
  g.shared = shared;
  g.p = (int)(S + 1) / 2;
  g.sets = (int)(S * O + 1) / 2;
  g.has_mix = false;
  g.own_only = true;
  g.ex = ((O + 1) / 2 - 1) * g.ib;
  return DASP_OK;
}

extern "C++" {
template <class Op>
int conv_bus_fwd(int max_out, bool shared, const float* x, const float* ir, float* y, void* xspec_save,
                 void* irspec_save, void* workspace, int64_t workspace_bytes, int64_t bs, int64_t n, int64_t ir_len,
                 int64_t S, int64_t O, int64_t chunk_items, void* stream) {
  ConvGeom g;
  int rc = make_bus_geom(shared, bs, n, ir_len, S, O, max_out, chunk_items, g);
  if (rc != DASP_OK) return rc;
  Op op{};
  op.S = (int)S; op.O = (int)O; op.ir_rows = (int)(S * O);
  return caller_ir_fwd(op, g, x, ir, nullptr, y, xspec_save, irspec_save, workspace, workspace_bytes, stream);
}

template <class Op>
int conv_bus_bwd(int max_out, bool shared, const float* gy, const void* xspec_save, const void* irspec_save,
                 float* gx, float* gir, void* workspace, int64_t workspace_bytes, int64_t bs, int64_t n,
                 int64_t ir_len, int64_t S, int64_t O, int64_t chunk_items, void* stream) {
  ConvGeom g;
  int rc = make_bus_geom(shared, bs, n, ir_len, S, O, max_out, chunk_items, g);
  if (rc != DASP_OK) return rc;
  Op op{};
  op.S = (int)S; op.O = (int)O; op.ir_rows = (int)(S * O);
  return caller_ir_bwd(op, g, gy, nullptr, nullptr, xspec_save, irspec_save, gx, gir, nullptr, workspace,
                       workspace_bytes, stream);
}
}  // extern "C++"

int conv_bus_geometry(int max_out, int64_t bs, int64_t n, int64_t ir_len, int64_t inputs, int64_t outputs,
                      int64_t shared, int64_t chunk_items, dasp_conv_geom* out) {
  DASP_REQUIRE(out != nullptr, "%s geometry: null out", max_out == 2 ? "conv bus" : "conv mc");
  ConvGeom g;
  int rc = make_bus_geom(shared != 0, bs, n, ir_len, inputs, outputs, max_out, chunk_items, g);
  if (rc != DASP_OK) return rc;
  return put_conv_geometry(g, nullptr, out);
}
}  // namespace

int dasp_debug_conv_bus_last_path(int which) { return g_bus_last_path[which ? 1 : 0]; }

int dasp_conv_bus_geometry(int64_t bs, int64_t n, int64_t ir_len, int64_t inputs, int64_t outputs, int64_t shared,
                           int64_t chunk_items, dasp_conv_geom* out) {
  return conv_bus_geometry(2, bs, n, ir_len, inputs, outputs, shared, chunk_items, out);
}

int dasp_conv_bus_fwd(const float* x, const float* ir, float* y, void* xspec_save, void* irspec_save, void* workspace,
                      int64_t workspace_bytes, int64_t bs, int64_t n, int64_t ir_len, int64_t inputs, int64_t outputs,
                      int64_t chunk_items, void* stream) {
  return conv_bus_fwd<BusOp>(2, false, x, ir, y, xspec_save, irspec_save, workspace, workspace_bytes, bs, n, ir_len,
                             inputs, outputs, chunk_items, stream);
}

int dasp_conv_bus_bwd(const float* gy, const void* xspec_save, const void* irspec_save, float* gx, float* gir,
                      void* workspace, int64_t workspace_bytes, int64_t bs, int64_t n, int64_t ir_len, int64_t inputs,
                      int64_t outputs, int64_t chunk_items, void* stream) {
  return conv_bus_bwd<BusOp>(2, false, gy, xspec_save, irspec_save, gx, gir, workspace, workspace_bytes, bs, n, ir_len,
                             inputs, outputs, chunk_items, stream);
}

int dasp_conv_bus_shared_fwd(const float* x, const float* ir, float* y, void* xspec_save, void* irspec_save,
                             void* workspace, int64_t workspace_bytes, int64_t bs, int64_t n, int64_t ir_len,
                             int64_t inputs, int64_t outputs, int64_t chunk_items, void* stream) {
  return conv_bus_fwd<BusOp>(2, true, x, ir, y, xspec_save, irspec_save, workspace, workspace_bytes, bs, n, ir_len,
                             inputs, outputs, chunk_items, stream);
}

int dasp_conv_bus_shared_bwd(const float* gy, const void* xspec_save, const void* irspec_save, float* gx, float* gir,
                             void* workspace, int64_t workspace_bytes, int64_t bs, int64_t n, int64_t ir_len,
                             int64_t inputs, int64_t outputs, int64_t chunk_items, void* stream) {
  return conv_bus_bwd<BusOp>(2, true, gy, xspec_save, irspec_save, gx, gir, workspace, workspace_bytes, bs, n, ir_len,
                             inputs, outputs, chunk_items, stream);
}

// ------------------------------------------------------------------ multichannel_convolution
// y[:, m] = sum_s x[:, s] * h[:, s, m] for 1 <= M <= DASP_CONV_MC_MAX_OUTPUTS outputs: BusOp with O = M.  M <= 2 runs
// the bus's own products (the same bits as dasp_conv_bus_*), M >= 3 busmc_mac_kernel.
int dasp_conv_mc_geometry(int64_t bs, int64_t n, int64_t ir_len, int64_t inputs, int64_t outputs, int64_t shared,
                          int64_t chunk_items, dasp_conv_geom* out) {
  return conv_bus_geometry(DASP_CONV_MC_MAX_OUTPUTS, bs, n, ir_len, inputs, outputs, shared, chunk_items, out);
}

int dasp_conv_mc_fwd(const float* x, const float* ir, float* y, void* xspec_save, void* irspec_save, void* workspace,
                     int64_t workspace_bytes, int64_t bs, int64_t n, int64_t ir_len, int64_t inputs, int64_t outputs,
                     int64_t chunk_items, void* stream) {
  return conv_bus_fwd<McOp>(DASP_CONV_MC_MAX_OUTPUTS, false, x, ir, y, xspec_save, irspec_save, workspace,
                            workspace_bytes, bs, n, ir_len, inputs, outputs, chunk_items, stream);
}

int dasp_conv_mc_bwd(const float* gy, const void* xspec_save, const void* irspec_save, float* gx, float* gir,
                     void* workspace, int64_t workspace_bytes, int64_t bs, int64_t n, int64_t ir_len, int64_t inputs,
                     int64_t outputs, int64_t chunk_items, void* stream) {
  return conv_bus_bwd<McOp>(DASP_CONV_MC_MAX_OUTPUTS, false, gy, xspec_save, irspec_save, gx, gir, workspace,
                            workspace_bytes, bs, n, ir_len, inputs, outputs, chunk_items, stream);
}

int dasp_conv_mc_shared_fwd(const float* x, const float* ir, float* y, void* xspec_save, void* irspec_save,
                            void* workspace, int64_t workspace_bytes, int64_t bs, int64_t n, int64_t ir_len,
                            int64_t inputs, int64_t outputs, int64_t chunk_items, void* stream) {
  return conv_bus_fwd<McOp>(DASP_CONV_MC_MAX_OUTPUTS, true, x, ir, y, xspec_save, irspec_save, workspace,
                            workspace_bytes, bs, n, ir_len, inputs, outputs, chunk_items, stream);
}

int dasp_conv_mc_shared_bwd(const float* gy, const void* xspec_save, const void* irspec_save, float* gx, float* gir,
                            void* workspace, int64_t workspace_bytes, int64_t bs, int64_t n, int64_t ir_len,
                            int64_t inputs, int64_t outputs, int64_t chunk_items, void* stream) {
  return conv_bus_bwd<McOp>(DASP_CONV_MC_MAX_OUTPUTS, true, gy, xspec_save, irspec_save, gx, gir, workspace,
                            workspace_bytes, bs, n, ir_len, inputs, outputs, chunk_items, stream);
}

// ------------------------------------------------------------------ time_varying_convolution_reverberation
// wet = sum_k w_k(t) (x * h_k)(t), y = (1 - mix) x + mix wet, through the stage above on the own FFT only: the audio
// windows as a static convolution (x_fft_kernel, one spectrum per block, saved the same way), K C IR rows per item
// in ceil(K C / 2) partition sets, and the tv_* kernels for the crossfaded products, their inverse and the weighted
// gradient transforms.  dL/dx and dL/dmix are ifft_dx_kernel's (the weighted correlation D is the gradient of the wet
// signal with respect to x, so sum_t g wet = sum_s x c holds as for a static IR).
namespace {
int g_tv_last_path[2] = {0, 0};                      // test hook: dispatch of the last forward / backward

extern "C++" {
template <int MODE>
int launch_tv_mac(int C, const float2* X, const float2* H, int64_t hstride, const float2* G, const float* mix,
                  float2* Out, int64_t item0, int64_t items, int I, int J, int K, int nX, int Hb, int sets,
                  cudaStream_t st) {
  dim3 grid((kNbA / 2 + 1 + 127) / 128, (unsigned)items);
  if (C == 2) tv_mac_kernel<MODE, 2><<<grid, 128, 0, st>>>(X, H, hstride, G, mix, Out, item0, I, J, K, nX, Hb, sets);
  else        tv_mac_kernel<MODE, 1><<<grid, 128, 0, st>>>(X, H, hstride, G, mix, Out, item0, I, J, K, nX, Hb, sets);
  DASP_LAUNCH_OK("tv_mac_kernel");
  return DASP_OK;
}
}  // extern "C++"

struct TvConvOp {
  static constexpr const char* kFwd = "tvconv fwd";
  static constexpr const char* kBwd = "tvconv bwd";
  static constexpr bool kOddSelf = false;
  int in_chs, C, K, Hb, ir_rows;                     // x channels, IR channels, anchors, hop / kB, IR rows K C
  int fwd_chunk(const ConvGeom& g, const Plans&, bool own, const float* tw, const float* x, const float* mix,
                float2* xs, float2* hs, int64_t h_stride, float* y, unsigned char* ws, const FwdWs& w, int64_t item0,
                int64_t items, cudaStream_t st) const {
    // bit 0: own FFT (always), bit 1: one trajectory shared by the batch, bit 2: crossfaded blocks (K > 1)
    g_tv_last_path[0] = (own ? 1 : 0) | (g.shared ? 2 : 0) | (g.ex > 0 ? 4 : 0);
    int rc = configure_fft_kernels();
    if (rc != DASP_OK) return rc;
    float2* ys = (float2*)(ws + w.ys);
    const int I = (int)g.ib, J = (int)g.jb, nX = (int)g.ex;
    const int nwin = (int)(items * I), nunits = nwin + (int)(h_stride != 0 ? items * g.sets * J : 0);
    x_fft_kernel<<<runs(nunits), kFusedThreads, kFftSmemBytes, st>>>(x, xs, hs, tw, item0, I, J, g.n, g.leff, in_chs,
                                                                      nwin, nunits);
    DASP_LAUNCH_OK("x_fft_kernel");
    if ((rc = launch_tv_mac<TV_FWD>(C, xs, hs, h_stride, nullptr, nullptr, ys, item0, items, I, J, K, nX, Hb, g.sets,
                                    st)) != DASP_OK)
      return rc;
    const int nout = (int)(items * (I + nX));
    tv_ifft_kernel<<<runs(nout), kFusedThreads, kFftSmemBytes, st>>>(reinterpret_cast<const float*>(ys), tw, x, mix, y,
                                                                     item0, I, nX, Hb, (int64_t)Hb * kB, g.n, in_chs,
                                                                     nout);
    DASP_LAUNCH_OK("tv_ifft_kernel");
    return DASP_OK;
  }
  int bwd_chunk(const ConvGeom& g, const Plans&, bool own, IrGrad e, const float* tw, const float* gy, const float* x,
                const float* mix, const float2* xs, const float2* hs, int64_t h_stride, float* gx, unsigned char* ws,
                const BwdWs& w, int64_t item0, int64_t items, cudaStream_t st) const {
    // bit 0: own FFT (always), bit 1: crossfaded blocks (K > 1), bit 2: dL/dIR computed, bit 3: shared trajectory
    g_tv_last_path[1] = (own ? 1 : 0) | (g.ex > 0 ? 2 : 0) | (e != IrGrad::kNone ? 4 : 0) | (g.shared ? 8 : 0);
    int rc = configure_fft_kernels();
    if (rc != DASP_OK) return rc;
    float2* gs = (float2*)(ws + w.gs);
    float2* ds = (float2*)(ws + w.ds);
    const int I = (int)g.ib, J = (int)g.jb, nX = (int)g.ex;
    const int ng = (int)(items * (I + nX));
    tv_fft_kernel<<<runs(ng), kFusedThreads, kFftSmemBytes, st>>>(gy, gs, tw, item0, I, nX, Hb, (int64_t)Hb * kB, g.n,
                                                                  ng);
    DASP_LAUNCH_OK("tv_fft_kernel");
    if ((rc = launch_tv_mac<TV_DX>(C, xs, hs, h_stride, gs, nullptr, ds, item0, items, I, J, K, nX, Hb, g.sets, st)) !=
        DASP_OK)
      return rc;
    ifft_dx_kernel<<<persistent_grid(items), kFusedThreads, kFftSmemBytes, st>>>(
        reinterpret_cast<const float*>(ds), tw, gy, x, mix, 1, gx, (float*)(ws + w.mixpart), item0, (int)items, I, g.n,
        in_chs);
    DASP_LAUNCH_OK("ifft_dx_kernel");
    if (e == IrGrad::kNone) return DASP_OK;          // a fixed trajectory: no dL/dIR work at all
    // per item the factor mix[b] goes into E here; a shared trajectory's is applied by irgrad_sum_kernel
    return launch_tv_mac<TV_DIR>(C, xs, hs, h_stride, gs, g.shared ? nullptr : mix, (float2*)(ws + w.es), item0, items,
                                 I, J, K, nX, Hb, g.sets, st);
  }
  // dL/dIR taps [0, leff) of items [item0, item0 + items): the first half of the inverse of each partition (the factor
  // mix is in the partitions already)
  int ir_taps(const ConvGeom& g, bool, const float* tw, const float2* es, const float*, float* gir, int64_t item0,
              int64_t items, cudaStream_t st) const {
    const int J = (int)g.jb, nparts = (int)(items * g.sets * J);
    bus_ifft_kernel<<<runs(nparts), kFusedThreads, kFftSmemBytes, st>>>(reinterpret_cast<const float*>(es), tw, gir,
                                                                        item0, ir_rows, g.sets, J, g.L, g.leff, 0,
                                                                        nparts);
    DASP_LAUNCH_OK("bus_ifft_kernel");
    return DASP_OK;
  }
};

// the argument checks of dasp_tvconv_*, filling the geometry
int make_tv_geom(bool shared, int64_t bs, int64_t n, int64_t L, int64_t K, int64_t ir_chs, int64_t hop, int64_t chunk,
                 ConvGeom& g) {
  DASP_REQUIRE(K >= 1, "tvconv: K >= 1 impulse responses are needed, got %lld", (long long)K);
  DASP_REQUIRE(ir_chs == 1 || ir_chs == 2, "tvconv: mono or stereo impulse responses only, got %lld channels",
               (long long)ir_chs);
  DASP_REQUIRE(hop > 0 && hop % kB == 0, "tvconv: hop must be a positive multiple of %d, got %lld", kB,
               (long long)hop);
  int rc = make_conv_geom(bs, n, L, chunk, g);
  if (rc != DASP_OK) return rc;
  DASP_REQUIRE(K - 1 <= (n - 1) / hop, "tvconv: anchor %lld at (K - 1) hop is at or after the end of x (n=%lld)",
               (long long)(K - 1), (long long)n);
  g.shared = shared;
  g.sets = (int)((K * ir_chs + 1) / 2);
  g.ex = (K - 1) * (hop / kB);                     // < ib: every crossfaded block is inside x
  g.own_only = true;
  return DASP_OK;
}
TvConvOp tv_op(int64_t in_chs, int64_t ir_chs, int64_t K, int64_t hop) {
  return TvConvOp{(int)in_chs, (int)ir_chs, (int)K, (int)(hop / kB), (int)(K * ir_chs)};
}

int tvconv_fwd(bool shared, const float* x, int64_t in_chs, const float* ir, int64_t ir_chs, int64_t ir_len, int64_t K,
               int64_t hop, const float* mix, float* y, void* xspec_save, void* irspec_save, void* workspace,
               int64_t workspace_bytes, int64_t bs, int64_t n, int64_t chunk_items, void* stream) {
  ConvGeom g;
  int rc = make_tv_geom(shared, bs, n, ir_len, K, ir_chs, hop, chunk_items, g);
  if (rc != DASP_OK) return rc;
  DASP_REQUIRE(in_chs == 1 || in_chs == 2, "tvconv: only mono/stereo signals, got %lld channels", (long long)in_chs);
  return caller_ir_fwd(tv_op(in_chs, ir_chs, K, hop), g, x, ir, mix, y, xspec_save, irspec_save, workspace,
                       workspace_bytes, stream);
}

int tvconv_bwd(bool shared, const float* gy, const float* x, int64_t in_chs, int64_t ir_chs, int64_t ir_len, int64_t K,
               int64_t hop, const float* mix, const void* xspec_save, const void* irspec_save, float* gx, float* gir,
               float* gmix, void* workspace, int64_t workspace_bytes, int64_t bs, int64_t n, int64_t chunk_items,
               void* stream) {
  ConvGeom g;
  int rc = make_tv_geom(shared, bs, n, ir_len, K, ir_chs, hop, chunk_items, g);
  if (rc != DASP_OK) return rc;
  DASP_REQUIRE(in_chs == 1 || in_chs == 2, "tvconv: only mono/stereo signals, got %lld channels", (long long)in_chs);
  return caller_ir_bwd(tv_op(in_chs, ir_chs, K, hop), g, gy, x, mix, xspec_save, irspec_save, gx, gir, gmix, workspace,
                       workspace_bytes, stream);
}
}  // namespace

int dasp_debug_tvconv_last_path(int which) { return g_tv_last_path[which ? 1 : 0]; }

int dasp_tvconv_geometry(int64_t bs, int64_t n, int64_t ir_len, int64_t K, int64_t ir_chs, int64_t hop, int64_t shared,
                         int64_t chunk_items, dasp_conv_geom* out) {
  DASP_REQUIRE(out != nullptr, "tvconv geometry: null out");
  ConvGeom g;
  int rc = make_tv_geom(shared != 0, bs, n, ir_len, K, ir_chs, hop, chunk_items, g);
  if (rc != DASP_OK) return rc;
  return put_conv_geometry(g, nullptr, out);
}

int dasp_tvconv_fwd(const float* x, int64_t in_chs, const float* ir, int64_t ir_chs, int64_t ir_len, int64_t K,
                    int64_t hop, const float* mix, float* y, void* xspec_save, void* irspec_save, void* workspace,
                    int64_t workspace_bytes, int64_t bs, int64_t n, int64_t chunk_items, void* stream) {
  return tvconv_fwd(false, x, in_chs, ir, ir_chs, ir_len, K, hop, mix, y, xspec_save, irspec_save, workspace,
                    workspace_bytes, bs, n, chunk_items, stream);
}

int dasp_tvconv_bwd(const float* gy, const float* x, int64_t in_chs, int64_t ir_chs, int64_t ir_len, int64_t K,
                    int64_t hop, const float* mix, const void* xspec_save, const void* irspec_save, float* gx,
                    float* gir, float* gmix, void* workspace, int64_t workspace_bytes, int64_t bs, int64_t n,
                    int64_t chunk_items, void* stream) {
  return tvconv_bwd(false, gy, x, in_chs, ir_chs, ir_len, K, hop, mix, xspec_save, irspec_save, gx, gir, gmix,
                    workspace, workspace_bytes, bs, n, chunk_items, stream);
}

int dasp_tvconv_shared_fwd(const float* x, int64_t in_chs, const float* ir, int64_t ir_chs, int64_t ir_len, int64_t K,
                           int64_t hop, const float* mix, float* y, void* xspec_save, void* irspec_save,
                           void* workspace, int64_t workspace_bytes, int64_t bs, int64_t n, int64_t chunk_items,
                           void* stream) {
  return tvconv_fwd(true, x, in_chs, ir, ir_chs, ir_len, K, hop, mix, y, xspec_save, irspec_save, workspace,
                    workspace_bytes, bs, n, chunk_items, stream);
}

int dasp_tvconv_shared_bwd(const float* gy, const float* x, int64_t in_chs, int64_t ir_chs, int64_t ir_len, int64_t K,
                           int64_t hop, const float* mix, const void* xspec_save, const void* irspec_save, float* gx,
                           float* gir, float* gmix, void* workspace, int64_t workspace_bytes, int64_t bs, int64_t n,
                           int64_t chunk_items, void* stream) {
  return tvconv_bwd(true, gy, x, in_chs, ir_chs, ir_len, K, hop, mix, xspec_save, irspec_save, gx, gir, gmix,
                    workspace, workspace_bytes, bs, n, chunk_items, stream);
}

// ------------------------------------------------------------------ time_varying_convolution_bus
// y[:, o] = sum_k w_k(t) sum_s (x[:, s] * h[:, k, s, o])(t) through the stage above on the own FFT only: the bus's window
// spectra (bus_fft_kernel, P = ceil(S / 2) per block), the K S O IR rows of a trajectory set in ceil(K S O / 2)
// partition sets, no mix.  The products are tvbus_mac_kernel's; a stereo bus has the time-varying op's slots (its
// inverse tvbus_ifft_kernel, its gradient transforms tv_fft_kernel), a mono bus one slot per block (tvbus_ifft_kernel,
// tvbus_gfft_kernel).  dL/dx and the dL/dIR taps are bus_ifft_kernel's, as for the bus.
namespace {
int g_tvbus_last_path[2] = {0, 0};                   // test hook: dispatch of the last forward / backward

extern "C++" {
template <int MODE>
int launch_tvbus_mac(int O, const float2* X, const float2* H, int64_t hstride, const float2* G, float2* Out,
                     int64_t items, int S, int I, int J, int K, int nX, int Hb, cudaStream_t st) {
  dim3 grid((kNbA / 2 + 1 + 127) / 128, (unsigned)items);
  if (O == 2) tvbus_mac_kernel<MODE, 2><<<grid, 128, 0, st>>>(X, H, hstride, G, Out, S, I, J, K, nX, Hb);
  else        tvbus_mac_kernel<MODE, 1><<<grid, 128, 0, st>>>(X, H, hstride, G, Out, S, I, J, K, nX, Hb);
  DASP_LAUNCH_OK("tvbus_mac_kernel");
  return DASP_OK;
}
}  // extern "C++"

struct TvBusOp {
  static constexpr const char* kFwd = "tvbus fwd";
  static constexpr const char* kBwd = "tvbus bwd";
  static constexpr bool kOddSelf = false;
  int S, O, K, Hb, ir_rows;                          // sources, outputs, anchors, hop / kB, IR rows K S O
  int nx() const { return (K - 1) * Hb; }            // crossfaded blocks (< ib)
  int slots(const ConvGeom& g) const { return (int)g.ib + (int)g.ex; }   // product / gradient slots per item
  int fwd_chunk(const ConvGeom& g, const Plans&, bool own, const float* tw, const float* x, const float*, float2* xs,
                float2* hs, int64_t h_stride, float* y, unsigned char* ws, const FwdWs& w, int64_t item0,
                int64_t items, cudaStream_t st) const {
    // bit 0: own FFT (always), bit 1: one trajectory set shared by the batch, bit 2: crossfaded blocks (K > 1)
    g_tvbus_last_path[0] = (own ? 1 : 0) | (g.shared ? 2 : 0) | (K > 1 ? 4 : 0);
    int rc = configure_fft_kernels();
    if (rc != DASP_OK) return rc;
    if (h_stride != 0 && (rc = ir_partition_spectra(g, tw, hs, items, st)) != DASP_OK) return rc;
    float2* ys = (float2*)(ws + w.ys);
    const int I = (int)g.ib, J = (int)g.jb, nwin = (int)(items * g.p * I), nout = (int)(items * slots(g));
    bus_fft_kernel<<<runs(nwin), kFusedThreads, kFftSmemBytes, st>>>(x, xs, tw, item0, S, g.p, I, g.n, 0, nwin);
    DASP_LAUNCH_OK("bus_fft_kernel");
    if ((rc = launch_tvbus_mac<TVB_FWD>(O, xs, hs, h_stride, nullptr, ys, items, S, I, J, K, nx(), Hb, st)) != DASP_OK)
      return rc;
    tvbus_ifft_kernel<<<runs(nout), kFusedThreads, kFftSmemBytes, st>>>(reinterpret_cast<const float*>(ys), tw, y,
                                                                        item0, I, nx(), Hb, (int64_t)Hb * kB, g.n, O,
                                                                        nout);
    DASP_LAUNCH_OK("tvbus_ifft_kernel");
    return DASP_OK;
  }
  int bwd_chunk(const ConvGeom& g, const Plans&, bool own, IrGrad e, const float* tw, const float* gy, const float*,
                const float*, const float2* xs, const float2* hs, int64_t h_stride, float* gx, unsigned char* ws,
                const BwdWs& w, int64_t item0, int64_t items, cudaStream_t st) const {
    // bit 0: own FFT (always), bit 1: crossfaded blocks (K > 1), bit 2: dL/dIR computed, bit 3: shared trajectory set
    g_tvbus_last_path[1] = (own ? 1 : 0) | (K > 1 ? 2 : 0) | (e != IrGrad::kNone ? 4 : 0) | (g.shared ? 8 : 0);
    int rc = configure_fft_kernels();
    if (rc != DASP_OK) return rc;
    float2* gs = (float2*)(ws + w.gs);
    float2* ds = (float2*)(ws + w.ds);
    const int I = (int)g.ib, J = (int)g.jb, nwin = (int)(items * g.p * I), ng = (int)(items * slots(g));
    const int64_t hop = (int64_t)Hb * kB;
    if (O == 2) {
      tv_fft_kernel<<<runs(ng), kFusedThreads, kFftSmemBytes, st>>>(gy, gs, tw, item0, I, nx(), Hb, hop, g.n, ng);
      DASP_LAUNCH_OK("tv_fft_kernel");
    } else {
      tvbus_gfft_kernel<<<runs(ng), kFusedThreads, kFftSmemBytes, st>>>(gy, gs, tw, item0, I, nx(), Hb, hop, g.n, ng);
      DASP_LAUNCH_OK("tvbus_gfft_kernel");
    }
    if ((rc = launch_tvbus_mac<TVB_DX>(O, xs, hs, h_stride, gs, ds, items, S, I, J, K, nx(), Hb, st)) != DASP_OK)
      return rc;
    bus_ifft_kernel<<<runs(nwin), kFusedThreads, kFftSmemBytes, st>>>(reinterpret_cast<const float*>(ds), tw, gx, item0,
                                                                      S, g.p, I, g.n, g.n, 1, nwin);
    DASP_LAUNCH_OK("bus_ifft_kernel");
    if (e == IrGrad::kNone) return DASP_OK;          // a fixed trajectory set: no dL/dIR work at all
    return launch_tvbus_mac<TVB_DIR>(O, xs, hs, 0, gs, (float2*)(ws + w.es), items, S, I, J, K, nx(), Hb, st);
  }
  // dL/dIR taps [0, leff) of items [item0, item0 + items): the first half of the inverse of each partition
  int ir_taps(const ConvGeom& g, bool, const float* tw, const float2* es, const float*, float* gir, int64_t item0,
              int64_t items, cudaStream_t st) const {
    const int J = (int)g.jb, nparts = (int)(items * g.sets * J);
    bus_ifft_kernel<<<runs(nparts), kFusedThreads, kFftSmemBytes, st>>>(reinterpret_cast<const float*>(es), tw, gir,
                                                                        item0, ir_rows, g.sets, J, g.L, g.leff, 0,
                                                                        nparts);
    DASP_LAUNCH_OK("bus_ifft_kernel");
    return DASP_OK;
  }
};

// the argument checks of dasp_tvbus_* (max_out 2) and of time_varying_multichannel_convolution (max_out
// DASP_CONV_MC_MAX_OUTPUTS, dasp_tvmc_*), filling the geometry of the output-side crossfade: U = O nX + Q (I - nX)
// product / gradient slots per item (Q = ceil(O / 2)), the U - I beyond the first I in g.ex.  That is I + nX for a
// stereo bus and I for a mono bus, which packs both IR sets of a block into one slot.
int make_tvbus_geom(bool shared, int64_t bs, int64_t n, int64_t L, int64_t K, int64_t S, int64_t O, int64_t hop,
                    int max_out, int64_t chunk, ConvGeom& g) {
  const char* what = max_out == 2 ? "tvbus" : "tvmc";
  DASP_REQUIRE(S >= 1 && S <= DASP_CONV_BUS_MAX_INPUTS, "%s: 1 to %d inputs are supported, got %lld", what,
               DASP_CONV_BUS_MAX_INPUTS, (long long)S);
  if (max_out == 2)
    DASP_REQUIRE(O == 1 || O == 2, "tvbus: a mono (1) or stereo (2) bus, got %lld outputs", (long long)O);
  else
    DASP_REQUIRE(O >= 1 && O <= max_out, "%s: 1 to %d outputs are supported, got %lld", what, max_out, (long long)O);
  DASP_REQUIRE(K >= 1, "%s: K >= 1 impulse-response sets are needed, got %lld", what, (long long)K);
  DASP_REQUIRE(hop > 0 && hop % kB == 0, "%s: hop must be a positive multiple of %d, got %lld", what, kB,
               (long long)hop);
  int rc = make_conv_geom(bs, n, L, chunk, g);
  if (rc != DASP_OK) return rc;
  DASP_REQUIRE(K - 1 <= (n - 1) / hop, "%s: anchor %lld at (K - 1) hop is at or after the end of x (n=%lld)", what,
               (long long)(K - 1), (long long)n);
  const int64_t sets = (K * S * O + 1) / 2;
  DASP_REQUIRE(sets <= 65535, "%s: at most 65535 partition sets (K S O / 2) per trajectory set, got %lld", what,
               (long long)sets);
  g.shared = shared;
  g.p = (int)(S + 1) / 2;
  g.sets = (int)sets;
  const int64_t nX = (K - 1) * (hop / kB);
  g.ex = O * nX + (O + 1) / 2 * (g.ib - nX) - g.ib;
  g.has_mix = false;
  g.own_only = true;
  return DASP_OK;
}
TvBusOp tvbus_op(int64_t K, int64_t S, int64_t O, int64_t hop) {
  return TvBusOp{(int)S, (int)O, (int)K, (int)(hop / kB), (int)(K * S * O)};
}

int tvbus_fwd(bool shared, const float* x, const float* ir, float* y, void* xspec_save, void* irspec_save,
              void* workspace, int64_t workspace_bytes, int64_t bs, int64_t n, int64_t ir_len, int64_t K, int64_t S,
              int64_t O, int64_t hop, int64_t chunk_items, void* stream) {
  ConvGeom g;
  int rc = make_tvbus_geom(shared, bs, n, ir_len, K, S, O, hop, 2, chunk_items, g);
  if (rc != DASP_OK) return rc;
  return caller_ir_fwd(tvbus_op(K, S, O, hop), g, x, ir, nullptr, y, xspec_save, irspec_save, workspace,
                       workspace_bytes, stream);
}

int tvbus_bwd(bool shared, const float* gy, const void* xspec_save, const void* irspec_save, float* gx, float* gir,
              void* workspace, int64_t workspace_bytes, int64_t bs, int64_t n, int64_t ir_len, int64_t K, int64_t S,
              int64_t O, int64_t hop, int64_t chunk_items, void* stream) {
  ConvGeom g;
  int rc = make_tvbus_geom(shared, bs, n, ir_len, K, S, O, hop, 2, chunk_items, g);
  if (rc != DASP_OK) return rc;
  return caller_ir_bwd(tvbus_op(K, S, O, hop), g, gy, nullptr, nullptr, xspec_save, irspec_save, gx, gir, nullptr,
                       workspace, workspace_bytes, stream);
}
}  // namespace

int dasp_debug_tvbus_last_path(int which) { return g_tvbus_last_path[which ? 1 : 0]; }

int dasp_tvbus_geometry(int64_t bs, int64_t n, int64_t ir_len, int64_t K, int64_t inputs, int64_t outputs, int64_t hop,
                        int64_t shared, int64_t chunk_items, dasp_conv_geom* out) {
  DASP_REQUIRE(out != nullptr, "tvbus geometry: null out");
  ConvGeom g;
  int rc = make_tvbus_geom(shared != 0, bs, n, ir_len, K, inputs, outputs, hop, 2, chunk_items, g);
  if (rc != DASP_OK) return rc;
  return put_conv_geometry(g, nullptr, out);
}

int dasp_tvbus_fwd(const float* x, const float* ir, float* y, void* xspec_save, void* irspec_save, void* workspace,
                   int64_t workspace_bytes, int64_t bs, int64_t n, int64_t ir_len, int64_t K, int64_t inputs,
                   int64_t outputs, int64_t hop, int64_t chunk_items, void* stream) {
  return tvbus_fwd(false, x, ir, y, xspec_save, irspec_save, workspace, workspace_bytes, bs, n, ir_len, K, inputs,
                   outputs, hop, chunk_items, stream);
}

int dasp_tvbus_bwd(const float* gy, const void* xspec_save, const void* irspec_save, float* gx, float* gir,
                   void* workspace, int64_t workspace_bytes, int64_t bs, int64_t n, int64_t ir_len, int64_t K,
                   int64_t inputs, int64_t outputs, int64_t hop, int64_t chunk_items, void* stream) {
  return tvbus_bwd(false, gy, xspec_save, irspec_save, gx, gir, workspace, workspace_bytes, bs, n, ir_len, K, inputs,
                   outputs, hop, chunk_items, stream);
}

int dasp_tvbus_shared_fwd(const float* x, const float* ir, float* y, void* xspec_save, void* irspec_save,
                          void* workspace, int64_t workspace_bytes, int64_t bs, int64_t n, int64_t ir_len, int64_t K,
                          int64_t inputs, int64_t outputs, int64_t hop, int64_t chunk_items, void* stream) {
  return tvbus_fwd(true, x, ir, y, xspec_save, irspec_save, workspace, workspace_bytes, bs, n, ir_len, K, inputs,
                   outputs, hop, chunk_items, stream);
}

int dasp_tvbus_shared_bwd(const float* gy, const void* xspec_save, const void* irspec_save, float* gx, float* gir,
                          void* workspace, int64_t workspace_bytes, int64_t bs, int64_t n, int64_t ir_len, int64_t K,
                          int64_t inputs, int64_t outputs, int64_t hop, int64_t chunk_items, void* stream) {
  return tvbus_bwd(true, gy, xspec_save, irspec_save, gx, gir, workspace, workspace_bytes, bs, n, ir_len, K, inputs,
                   outputs, hop, chunk_items, stream);
}

// ------------------------------------------------------------------ time_varying_convolution_bus, source-side crossfade
// y[:, o] = sum_k sum_s ((w_k x[:, s]) * h[:, k, s, o]) through the stage above on the own FFT only: the window spectra
// of tvbusin_fft_kernel (XW per item, g.xw), the partition sets and IR packing of dasp_tvbus_*, one product and one
// inverse per block (tvbus_ifft_kernel without crossfaded slots), the static bus's gradient transforms, dL/dx through
// tvbusin_ifft_kernel, and the dL/dIR taps through bus_ifft_kernel.
namespace {
extern "C++" {
template <int MODE>
int launch_tvbusin_mac(int O, const float2* X, const float2* H, int64_t hstride, float2* G, float2* Out,
                       int64_t items, int S, int I, int J, int K, int nX, int Hb, cudaStream_t st) {
  dim3 grid((kNbA / 2 + 1 + 127) / 128, (unsigned)items);
  if (O == 2) tvbusin_mac_kernel<MODE, 2><<<grid, 128, 0, st>>>(X, H, hstride, G, Out, S, I, J, K, nX, Hb);
  else        tvbusin_mac_kernel<MODE, 1><<<grid, 128, 0, st>>>(X, H, hstride, G, Out, S, I, J, K, nX, Hb);
  DASP_LAUNCH_OK("tvbusin_mac_kernel");
  return DASP_OK;
}
}  // extern "C++"

struct TvBusInOp {
  static constexpr const char* kFwd = "tvbus in fwd";
  static constexpr const char* kBwd = "tvbus in bwd";
  static constexpr bool kOddSelf = false;
  int S, O, K, Hb, ir_rows;                          // sources, outputs, anchors, hop / kB, IR rows K S O
  int nx() const { return (K - 1) * Hb; }            // crossfaded blocks (< ib)
  int fwd_chunk(const ConvGeom& g, const Plans&, bool own, const float* tw, const float* x, const float*, float2* xs,
                float2* hs, int64_t h_stride, float* y, unsigned char* ws, const FwdWs& w, int64_t item0,
                int64_t items, cudaStream_t st) const {
    // dasp_tvbus_*'s bits, and bit 3: the source-side crossfade
    g_tvbus_last_path[0] = (own ? 1 : 0) | (g.shared ? 2 : 0) | (K > 1 ? 4 : 0) | 8;
    int rc = configure_fft_kernels();
    if (rc != DASP_OK) return rc;
    if (h_stride != 0 && (rc = ir_partition_spectra(g, tw, hs, items, st)) != DASP_OK) return rc;
    float2* ys = (float2*)(ws + w.ys);
    const int I = (int)g.ib, J = (int)g.jb, nwin = (int)(items * g.xw), nblk = (int)(items * I);
    const int64_t hop = (int64_t)Hb * kB;
    tvbusin_fft_kernel<<<runs(nwin), kFusedThreads, kFftSmemBytes, st>>>(x, xs, tw, item0, S, I, nx(), Hb, hop, g.n,
                                                                         nwin);
    DASP_LAUNCH_OK("tvbusin_fft_kernel");
    if ((rc = launch_tvbusin_mac<TVI_FWD>(O, xs, hs, h_stride, nullptr, ys, items, S, I, J, K, nx(), Hb, st)) != DASP_OK)
      return rc;
    // no crossfaded slots: every inverse is one output block, rows 0 and 1 as re and im
    tvbus_ifft_kernel<<<runs(nblk), kFusedThreads, kFftSmemBytes, st>>>(reinterpret_cast<const float*>(ys), tw, y,
                                                                        item0, I, 0, Hb, hop, g.n, O, nblk);
    DASP_LAUNCH_OK("tvbus_ifft_kernel");
    return DASP_OK;
  }
  int bwd_chunk(const ConvGeom& g, const Plans&, bool own, IrGrad e, const float* tw, const float* gy, const float*,
                const float*, const float2* xs, const float2* hs, int64_t h_stride, float* gx, unsigned char* ws,
                const BwdWs& w, int64_t item0, int64_t items, cudaStream_t st) const {
    // dasp_tvbus_*'s bits, and bit 4: the source-side crossfade
    g_tvbus_last_path[1] = (own ? 1 : 0) | (K > 1 ? 2 : 0) | (e != IrGrad::kNone ? 4 : 0) | (g.shared ? 8 : 0) | 16;
    int rc = configure_fft_kernels();
    if (rc != DASP_OK) return rc;
    float2* gs = (float2*)(ws + w.gs);
    float2* ds = (float2*)(ws + w.ds);
    const int I = (int)g.ib, J = (int)g.jb, nwin = (int)(items * g.xw), nblk = (int)(items * I);
    const int64_t hop = (int64_t)Hb * kB;
    bus_fft_kernel<<<runs(nblk), kFusedThreads, kFftSmemBytes, st>>>(gy, gs, tw, item0, O, 1, I, g.n, 1, nblk);
    DASP_LAUNCH_OK("bus_fft_kernel");
    if ((rc = launch_tvbusin_mac<TVI_DX>(O, xs, hs, h_stride, gs, ds, items, S, I, J, K, nx(), Hb, st)) != DASP_OK)
      return rc;
    tvbusin_ifft_kernel<<<runs(nwin), kFusedThreads, kFftSmemBytes, st>>>(reinterpret_cast<const float*>(ds), tw, gx,
                                                                          item0, S, I, nx(), Hb, hop, g.n, nwin);
    DASP_LAUNCH_OK("tvbusin_ifft_kernel");
    if (e == IrGrad::kNone) return DASP_OK;          // a fixed trajectory set: no dL/dIR work at all
    return launch_tvbusin_mac<TVI_DIR>(O, xs, hs, 0, gs, (float2*)(ws + w.es), items, S, I, J, K, nx(), Hb, st);
  }
  // dL/dIR taps [0, leff) of items [item0, item0 + items): the first half of the inverse of each partition
  int ir_taps(const ConvGeom& g, bool, const float* tw, const float2* es, const float*, float* gir, int64_t item0,
              int64_t items, cudaStream_t st) const {
    const int J = (int)g.jb, nparts = (int)(items * g.sets * J);
    bus_ifft_kernel<<<runs(nparts), kFusedThreads, kFftSmemBytes, st>>>(reinterpret_cast<const float*>(es), tw, gir,
                                                                        item0, ir_rows, g.sets, J, g.L, g.leff, 0,
                                                                        nparts);
    DASP_LAUNCH_OK("bus_ifft_kernel");
    return DASP_OK;
  }
};

// make_tvbus_geom's argument checks; the source-side windows: S per crossfaded block, ceil(S / 2) per later block, and
// one product and gradient spectrum per block and output pair (Q = ceil(O / 2) per block, the Q - 1 beyond the first
// in g.ex)
int make_tvbusin_geom(bool shared, int64_t bs, int64_t n, int64_t L, int64_t K, int64_t S, int64_t O, int64_t hop,
                      int max_out, int64_t chunk, ConvGeom& g) {
  int rc = make_tvbus_geom(shared, bs, n, L, K, S, O, hop, max_out, chunk, g);
  if (rc != DASP_OK) return rc;
  const int64_t nX = (K - 1) * (hop / kB);
  g.ex = ((O + 1) / 2 - 1) * g.ib;
  g.xw = nX * S + (g.ib - nX) * g.p;
  return DASP_OK;
}
TvBusInOp tvbusin_op(int64_t K, int64_t S, int64_t O, int64_t hop) {
  return TvBusInOp{(int)S, (int)O, (int)K, (int)(hop / kB), (int)(K * S * O)};
}

int tvbusin_fwd(bool shared, const float* x, const float* ir, float* y, void* xspec_save, void* irspec_save,
                void* workspace, int64_t workspace_bytes, int64_t bs, int64_t n, int64_t ir_len, int64_t K, int64_t S,
                int64_t O, int64_t hop, int64_t chunk_items, void* stream) {
  ConvGeom g;
  int rc = make_tvbusin_geom(shared, bs, n, ir_len, K, S, O, hop, 2, chunk_items, g);
  if (rc != DASP_OK) return rc;
  return caller_ir_fwd(tvbusin_op(K, S, O, hop), g, x, ir, nullptr, y, xspec_save, irspec_save, workspace,
                       workspace_bytes, stream);
}

int tvbusin_bwd(bool shared, const float* gy, const void* xspec_save, const void* irspec_save, float* gx, float* gir,
                void* workspace, int64_t workspace_bytes, int64_t bs, int64_t n, int64_t ir_len, int64_t K, int64_t S,
                int64_t O, int64_t hop, int64_t chunk_items, void* stream) {
  ConvGeom g;
  int rc = make_tvbusin_geom(shared, bs, n, ir_len, K, S, O, hop, 2, chunk_items, g);
  if (rc != DASP_OK) return rc;
  return caller_ir_bwd(tvbusin_op(K, S, O, hop), g, gy, nullptr, nullptr, xspec_save, irspec_save, gx, gir, nullptr,
                       workspace, workspace_bytes, stream);
}
}  // namespace

int dasp_tvbus_in_geometry(int64_t bs, int64_t n, int64_t ir_len, int64_t K, int64_t inputs, int64_t outputs,
                           int64_t hop, int64_t shared, int64_t chunk_items, dasp_conv_geom* out) {
  DASP_REQUIRE(out != nullptr, "tvbus in geometry: null out");
  ConvGeom g;
  int rc = make_tvbusin_geom(shared != 0, bs, n, ir_len, K, inputs, outputs, hop, 2, chunk_items, g);
  if (rc != DASP_OK) return rc;
  return put_conv_geometry(g, nullptr, out);
}

int dasp_tvbus_in_fwd(const float* x, const float* ir, float* y, void* xspec_save, void* irspec_save, void* workspace,
                      int64_t workspace_bytes, int64_t bs, int64_t n, int64_t ir_len, int64_t K, int64_t inputs,
                      int64_t outputs, int64_t hop, int64_t chunk_items, void* stream) {
  return tvbusin_fwd(false, x, ir, y, xspec_save, irspec_save, workspace, workspace_bytes, bs, n, ir_len, K, inputs,
                     outputs, hop, chunk_items, stream);
}

int dasp_tvbus_in_bwd(const float* gy, const void* xspec_save, const void* irspec_save, float* gx, float* gir,
                      void* workspace, int64_t workspace_bytes, int64_t bs, int64_t n, int64_t ir_len, int64_t K,
                      int64_t inputs, int64_t outputs, int64_t hop, int64_t chunk_items, void* stream) {
  return tvbusin_bwd(false, gy, xspec_save, irspec_save, gx, gir, workspace, workspace_bytes, bs, n, ir_len, K, inputs,
                     outputs, hop, chunk_items, stream);
}

int dasp_tvbus_in_shared_fwd(const float* x, const float* ir, float* y, void* xspec_save, void* irspec_save,
                             void* workspace, int64_t workspace_bytes, int64_t bs, int64_t n, int64_t ir_len,
                             int64_t K, int64_t inputs, int64_t outputs, int64_t hop, int64_t chunk_items,
                             void* stream) {
  return tvbusin_fwd(true, x, ir, y, xspec_save, irspec_save, workspace, workspace_bytes, bs, n, ir_len, K, inputs,
                     outputs, hop, chunk_items, stream);
}

int dasp_tvbus_in_shared_bwd(const float* gy, const void* xspec_save, const void* irspec_save, float* gx, float* gir,
                             void* workspace, int64_t workspace_bytes, int64_t bs, int64_t n, int64_t ir_len,
                             int64_t K, int64_t inputs, int64_t outputs, int64_t hop, int64_t chunk_items,
                             void* stream) {
  return tvbusin_bwd(true, gy, xspec_save, irspec_save, gx, gir, workspace, workspace_bytes, bs, n, ir_len, K, inputs,
                     outputs, hop, chunk_items, stream);
}

// ------------------------------------------------------------------ time_varying_multichannel_convolution
// The time-varying bus with 1 <= M <= DASP_CONV_MC_MAX_OUTPUTS outputs, both crossfades.  M <= 2 runs TvBusOp /
// TvBusInOp unchanged (the bits of dasp_tvbus_* / dasp_tvbus_in_*).  M >= 3, output side: the bus's windows, the
// products of tvmc_mac_kernel in U = M nX + Q (I - nX) slots, whose inverse (tvbusin_ifft_kernel with M rows) crossfades
// each output row of a crossfaded block, and whose gradient slots are tvbusin_fft_kernel's transforms of the M gradient
// rows; dL/dx through bus_ifft_kernel.  Source side: tvbusin_fft_kernel's windows, the products of tvmcin_mac_kernel in
// Q I blocks (inverse bus_ifft_kernel, gradient bus_fft_kernel, rows M, groups Q), dL/dx through tvbusin_ifft_kernel.
// The IR packing, partition transforms, shared-gradient sum and dL/dIR taps are the tv bus's.
namespace {
// the products' grid: `slices` slices (output pairs, input pairs or partition sets) of each item
dim3 tvmc_grid(int slices, int64_t items) {
  return dim3((kNbA / 2 + 1 + 127) / 128, (unsigned)slices, (unsigned)items);
}

struct TvMcOp : TvBusOp {
  static constexpr const char* kFwd = "tvmc fwd";
  static constexpr const char* kBwd = "tvmc bwd";
  int fwd_chunk(const ConvGeom& g, const Plans& pl, bool own, const float* tw, const float* x, const float* mix,
                float2* xs, float2* hs, int64_t h_stride, float* y, unsigned char* ws, const FwdWs& w, int64_t item0,
                int64_t items, cudaStream_t st) const {
    if (O <= 2) return TvBusOp::fwd_chunk(g, pl, own, tw, x, mix, xs, hs, h_stride, y, ws, w, item0, items, st);
    // dasp_tvbus_*'s bits, and bit 4: M >= 3 outputs
    g_tvbus_last_path[0] = (own ? 1 : 0) | (g.shared ? 2 : 0) | (K > 1 ? 4 : 0) | 16;
    int rc = configure_fft_kernels();
    if (rc != DASP_OK) return rc;
    if (h_stride != 0 && (rc = ir_partition_spectra(g, tw, hs, items, st)) != DASP_OK) return rc;
    float2* ys = (float2*)(ws + w.ys);
    const int I = (int)g.ib, J = (int)g.jb, nwin = (int)(items * g.p * I), nout = (int)(items * slots(g));
    const int64_t hop = (int64_t)Hb * kB;
    bus_fft_kernel<<<runs(nwin), kFusedThreads, kFftSmemBytes, st>>>(x, xs, tw, item0, S, g.p, I, g.n, 0, nwin);
    DASP_LAUNCH_OK("bus_fft_kernel");
    tvmc_mac_kernel<TVM_FWD><<<tvmc_grid((O + 1) / 2, items), 128, 0, st>>>(xs, hs, h_stride, nullptr, ys, S,
                                                                                     O, I, J, K, nx(), Hb);
    DASP_LAUNCH_OK("tvmc_mac_kernel");
    tvbusin_ifft_kernel<<<runs(nout), kFusedThreads, kFftSmemBytes, st>>>(reinterpret_cast<const float*>(ys), tw, y,
                                                                          item0, O, I, nx(), Hb, hop, g.n, nout);
    DASP_LAUNCH_OK("tvbusin_ifft_kernel");
    return DASP_OK;
  }
  int bwd_chunk(const ConvGeom& g, const Plans& pl, bool own, IrGrad e, const float* tw, const float* gy,
                const float* x, const float* mix, const float2* xs, const float2* hs, int64_t h_stride, float* gx,
                unsigned char* ws, const BwdWs& w, int64_t item0, int64_t items, cudaStream_t st) const {
    if (O <= 2)
      return TvBusOp::bwd_chunk(g, pl, own, e, tw, gy, x, mix, xs, hs, h_stride, gx, ws, w, item0, items, st);
    // dasp_tvbus_*'s bits, and bit 5: M >= 3 outputs
    g_tvbus_last_path[1] = (own ? 1 : 0) | (K > 1 ? 2 : 0) | (e != IrGrad::kNone ? 4 : 0) | (g.shared ? 8 : 0) | 32;
    int rc = configure_fft_kernels();
    if (rc != DASP_OK) return rc;
    float2* gs = (float2*)(ws + w.gs);
    float2* ds = (float2*)(ws + w.ds);
    const int I = (int)g.ib, J = (int)g.jb, nwin = (int)(items * g.p * I), ng = (int)(items * slots(g));
    const int64_t hop = (int64_t)Hb * kB;
    tvbusin_fft_kernel<<<runs(ng), kFusedThreads, kFftSmemBytes, st>>>(gy, gs, tw, item0, O, I, nx(), Hb, hop, g.n, ng);
    DASP_LAUNCH_OK("tvbusin_fft_kernel");
    tvmc_mac_kernel<TVM_DX><<<tvmc_grid(g.p, items), 128, 0, st>>>(xs, hs, h_stride, gs, ds, S, O, I, J,
                                                                                  K, nx(), Hb);
    DASP_LAUNCH_OK("tvmc_mac_kernel");
    bus_ifft_kernel<<<runs(nwin), kFusedThreads, kFftSmemBytes, st>>>(reinterpret_cast<const float*>(ds), tw, gx, item0,
                                                                      S, g.p, I, g.n, g.n, 1, nwin);
    DASP_LAUNCH_OK("bus_ifft_kernel");
    if (e == IrGrad::kNone) return DASP_OK;          // a fixed trajectory: no dL/dIR work at all
    tvmc_mac_kernel<TVM_DIR><<<tvmc_grid(g.sets, items), 128, 0, st>>>(
        xs, hs, 0, gs, (float2*)(ws + w.es), S, O, I, J, K, nx(), Hb);
    DASP_LAUNCH_OK("tvmc_mac_kernel");
    return DASP_OK;
  }
};

struct TvMcInOp : TvBusInOp {
  static constexpr const char* kFwd = "tvmc in fwd";
  static constexpr const char* kBwd = "tvmc in bwd";
  int fwd_chunk(const ConvGeom& g, const Plans& pl, bool own, const float* tw, const float* x, const float* mix,
                float2* xs, float2* hs, int64_t h_stride, float* y, unsigned char* ws, const FwdWs& w, int64_t item0,
                int64_t items, cudaStream_t st) const {
    if (O <= 2) return TvBusInOp::fwd_chunk(g, pl, own, tw, x, mix, xs, hs, h_stride, y, ws, w, item0, items, st);
    // dasp_tvbus_in_*'s bits, and bit 4: M >= 3 outputs
    g_tvbus_last_path[0] = (own ? 1 : 0) | (g.shared ? 2 : 0) | (K > 1 ? 4 : 0) | 8 | 16;
    int rc = configure_fft_kernels();
    if (rc != DASP_OK) return rc;
    if (h_stride != 0 && (rc = ir_partition_spectra(g, tw, hs, items, st)) != DASP_OK) return rc;
    float2* ys = (float2*)(ws + w.ys);
    const int I = (int)g.ib, J = (int)g.jb, Q = (O + 1) / 2, nwin = (int)(items * g.xw), nblk = (int)(items * Q * I);
    const int64_t hop = (int64_t)Hb * kB;
    tvbusin_fft_kernel<<<runs(nwin), kFusedThreads, kFftSmemBytes, st>>>(x, xs, tw, item0, S, I, nx(), Hb, hop, g.n,
                                                                         nwin);
    DASP_LAUNCH_OK("tvbusin_fft_kernel");
    tvmcin_mac_kernel<TVJ_FWD><<<tvmc_grid(Q, items), 128, 0, st>>>(xs, hs, h_stride, nullptr, ys,
                                                                                       S, O, I, J, K, nx(), Hb);
    DASP_LAUNCH_OK("tvmcin_mac_kernel");
    bus_ifft_kernel<<<runs(nblk), kFusedThreads, kFftSmemBytes, st>>>(reinterpret_cast<const float*>(ys), tw, y, item0,
                                                                      O, Q, I, g.n, g.n, 1, nblk);
    DASP_LAUNCH_OK("bus_ifft_kernel");
    return DASP_OK;
  }
  int bwd_chunk(const ConvGeom& g, const Plans& pl, bool own, IrGrad e, const float* tw, const float* gy,
                const float* x, const float* mix, const float2* xs, const float2* hs, int64_t h_stride, float* gx,
                unsigned char* ws, const BwdWs& w, int64_t item0, int64_t items, cudaStream_t st) const {
    if (O <= 2)
      return TvBusInOp::bwd_chunk(g, pl, own, e, tw, gy, x, mix, xs, hs, h_stride, gx, ws, w, item0, items, st);
    // dasp_tvbus_in_*'s bits, and bit 5: M >= 3 outputs
    g_tvbus_last_path[1] =
        (own ? 1 : 0) | (K > 1 ? 2 : 0) | (e != IrGrad::kNone ? 4 : 0) | (g.shared ? 8 : 0) | 16 | 32;
    int rc = configure_fft_kernels();
    if (rc != DASP_OK) return rc;
    float2* gs = (float2*)(ws + w.gs);
    float2* ds = (float2*)(ws + w.ds);
    const int I = (int)g.ib, J = (int)g.jb, Q = (O + 1) / 2, nwin = (int)(items * g.xw), nblk = (int)(items * Q * I);
    const int64_t hop = (int64_t)Hb * kB;
    bus_fft_kernel<<<runs(nblk), kFusedThreads, kFftSmemBytes, st>>>(gy, gs, tw, item0, O, Q, I, g.n, 1, nblk);
    DASP_LAUNCH_OK("bus_fft_kernel");
    tvmcin_mac_kernel<TVJ_FOLD><<<tvmc_grid(Q, items), 128, 0, st>>>(xs, hs, h_stride, gs, nullptr,
                                                                                         S, O, I, J, K, nx(), Hb);
    DASP_LAUNCH_OK("tvmcin_mac_kernel");
    tvmcin_mac_kernel<TVJ_DX><<<tvmc_grid(g.p, items), 128, 0, st>>>(xs, hs, h_stride, gs, ds, S, O, I,
                                                                                    J, K, nx(), Hb);
    DASP_LAUNCH_OK("tvmcin_mac_kernel");
    tvbusin_ifft_kernel<<<runs(nwin), kFusedThreads, kFftSmemBytes, st>>>(reinterpret_cast<const float*>(ds), tw, gx,
                                                                          item0, S, I, nx(), Hb, hop, g.n, nwin);
    DASP_LAUNCH_OK("tvbusin_ifft_kernel");
    if (e == IrGrad::kNone) return DASP_OK;          // a fixed trajectory: no dL/dIR work at all
    tvmcin_mac_kernel<TVJ_DIR><<<tvmc_grid(g.sets, items), 128, 0, st>>>(
        xs, hs, 0, gs, (float2*)(ws + w.es), S, O, I, J, K, nx(), Hb);
    DASP_LAUNCH_OK("tvmcin_mac_kernel");
    return DASP_OK;
  }
};

extern "C++" {
// input: the source-side crossfade (TvMcInOp), else the output side (TvMcOp)
template <bool INPUT>
int tvmc_geom(bool shared, int64_t bs, int64_t n, int64_t L, int64_t K, int64_t S, int64_t M, int64_t hop,
              int64_t chunk, ConvGeom& g) {
  return INPUT ? make_tvbusin_geom(shared, bs, n, L, K, S, M, hop, DASP_CONV_MC_MAX_OUTPUTS, chunk, g)
               : make_tvbus_geom(shared, bs, n, L, K, S, M, hop, DASP_CONV_MC_MAX_OUTPUTS, chunk, g);
}

template <bool INPUT>
int tvmc_fwd(bool shared, const float* x, const float* ir, float* y, void* xspec_save, void* irspec_save,
             void* workspace, int64_t workspace_bytes, int64_t bs, int64_t n, int64_t ir_len, int64_t K, int64_t S,
             int64_t M, int64_t hop, int64_t chunk_items, void* stream) {
  ConvGeom g;
  int rc = tvmc_geom<INPUT>(shared, bs, n, ir_len, K, S, M, hop, chunk_items, g);
  if (rc != DASP_OK) return rc;
  typename std::conditional<INPUT, TvMcInOp, TvMcOp>::type op{};
  op.S = (int)S; op.O = (int)M; op.K = (int)K; op.Hb = (int)(hop / kB); op.ir_rows = (int)(K * S * M);
  return caller_ir_fwd(op, g, x, ir, nullptr, y, xspec_save, irspec_save, workspace, workspace_bytes, stream);
}

template <bool INPUT>
int tvmc_bwd(bool shared, const float* gy, const void* xspec_save, const void* irspec_save, float* gx, float* gir,
             void* workspace, int64_t workspace_bytes, int64_t bs, int64_t n, int64_t ir_len, int64_t K, int64_t S,
             int64_t M, int64_t hop, int64_t chunk_items, void* stream) {
  ConvGeom g;
  int rc = tvmc_geom<INPUT>(shared, bs, n, ir_len, K, S, M, hop, chunk_items, g);
  if (rc != DASP_OK) return rc;
  typename std::conditional<INPUT, TvMcInOp, TvMcOp>::type op{};
  op.S = (int)S; op.O = (int)M; op.K = (int)K; op.Hb = (int)(hop / kB); op.ir_rows = (int)(K * S * M);
  return caller_ir_bwd(op, g, gy, nullptr, nullptr, xspec_save, irspec_save, gx, gir, nullptr, workspace,
                       workspace_bytes, stream);
}

template <bool INPUT>
int tvmc_geometry(int64_t bs, int64_t n, int64_t ir_len, int64_t K, int64_t inputs, int64_t outputs, int64_t hop,
                  int64_t shared, int64_t chunk_items, dasp_conv_geom* out) {
  DASP_REQUIRE(out != nullptr, "%s geometry: null out", INPUT ? "tvmc in" : "tvmc");
  ConvGeom g;
  int rc = tvmc_geom<INPUT>(shared != 0, bs, n, ir_len, K, inputs, outputs, hop, chunk_items, g);
  if (rc != DASP_OK) return rc;
  return put_conv_geometry(g, nullptr, out);
}
}  // extern "C++"
}  // namespace

int dasp_tvmc_geometry(int64_t bs, int64_t n, int64_t ir_len, int64_t K, int64_t inputs, int64_t outputs, int64_t hop,
                       int64_t shared, int64_t chunk_items, dasp_conv_geom* out) {
  return tvmc_geometry<false>(bs, n, ir_len, K, inputs, outputs, hop, shared, chunk_items, out);
}

int dasp_tvmc_fwd(const float* x, const float* ir, float* y, void* xspec_save, void* irspec_save, void* workspace,
                  int64_t workspace_bytes, int64_t bs, int64_t n, int64_t ir_len, int64_t K, int64_t inputs,
                  int64_t outputs, int64_t hop, int64_t chunk_items, void* stream) {
  return tvmc_fwd<false>(false, x, ir, y, xspec_save, irspec_save, workspace, workspace_bytes, bs, n, ir_len, K,
                         inputs, outputs, hop, chunk_items, stream);
}

int dasp_tvmc_bwd(const float* gy, const void* xspec_save, const void* irspec_save, float* gx, float* gir,
                  void* workspace, int64_t workspace_bytes, int64_t bs, int64_t n, int64_t ir_len, int64_t K,
                  int64_t inputs, int64_t outputs, int64_t hop, int64_t chunk_items, void* stream) {
  return tvmc_bwd<false>(false, gy, xspec_save, irspec_save, gx, gir, workspace, workspace_bytes, bs, n, ir_len, K,
                         inputs, outputs, hop, chunk_items, stream);
}

int dasp_tvmc_shared_fwd(const float* x, const float* ir, float* y, void* xspec_save, void* irspec_save,
                         void* workspace, int64_t workspace_bytes, int64_t bs, int64_t n, int64_t ir_len, int64_t K,
                         int64_t inputs, int64_t outputs, int64_t hop, int64_t chunk_items, void* stream) {
  return tvmc_fwd<false>(true, x, ir, y, xspec_save, irspec_save, workspace, workspace_bytes, bs, n, ir_len, K,
                         inputs, outputs, hop, chunk_items, stream);
}

int dasp_tvmc_shared_bwd(const float* gy, const void* xspec_save, const void* irspec_save, float* gx, float* gir,
                         void* workspace, int64_t workspace_bytes, int64_t bs, int64_t n, int64_t ir_len, int64_t K,
                         int64_t inputs, int64_t outputs, int64_t hop, int64_t chunk_items, void* stream) {
  return tvmc_bwd<false>(true, gy, xspec_save, irspec_save, gx, gir, workspace, workspace_bytes, bs, n, ir_len, K,
                         inputs, outputs, hop, chunk_items, stream);
}

int dasp_tvmc_in_geometry(int64_t bs, int64_t n, int64_t ir_len, int64_t K, int64_t inputs, int64_t outputs,
                          int64_t hop, int64_t shared, int64_t chunk_items, dasp_conv_geom* out) {
  return tvmc_geometry<true>(bs, n, ir_len, K, inputs, outputs, hop, shared, chunk_items, out);
}

int dasp_tvmc_in_fwd(const float* x, const float* ir, float* y, void* xspec_save, void* irspec_save, void* workspace,
                     int64_t workspace_bytes, int64_t bs, int64_t n, int64_t ir_len, int64_t K, int64_t inputs,
                     int64_t outputs, int64_t hop, int64_t chunk_items, void* stream) {
  return tvmc_fwd<true>(false, x, ir, y, xspec_save, irspec_save, workspace, workspace_bytes, bs, n, ir_len, K,
                        inputs, outputs, hop, chunk_items, stream);
}

int dasp_tvmc_in_bwd(const float* gy, const void* xspec_save, const void* irspec_save, float* gx, float* gir,
                     void* workspace, int64_t workspace_bytes, int64_t bs, int64_t n, int64_t ir_len, int64_t K,
                     int64_t inputs, int64_t outputs, int64_t hop, int64_t chunk_items, void* stream) {
  return tvmc_bwd<true>(false, gy, xspec_save, irspec_save, gx, gir, workspace, workspace_bytes, bs, n, ir_len, K,
                        inputs, outputs, hop, chunk_items, stream);
}

int dasp_tvmc_in_shared_fwd(const float* x, const float* ir, float* y, void* xspec_save, void* irspec_save,
                            void* workspace, int64_t workspace_bytes, int64_t bs, int64_t n, int64_t ir_len, int64_t K,
                            int64_t inputs, int64_t outputs, int64_t hop, int64_t chunk_items, void* stream) {
  return tvmc_fwd<true>(true, x, ir, y, xspec_save, irspec_save, workspace, workspace_bytes, bs, n, ir_len, K,
                        inputs, outputs, hop, chunk_items, stream);
}

int dasp_tvmc_in_shared_bwd(const float* gy, const void* xspec_save, const void* irspec_save, float* gx, float* gir,
                            void* workspace, int64_t workspace_bytes, int64_t bs, int64_t n, int64_t ir_len, int64_t K,
                            int64_t inputs, int64_t outputs, int64_t hop, int64_t chunk_items, void* stream) {
  return tvmc_bwd<true>(true, gy, xspec_save, irspec_save, gx, gir, workspace, workspace_bytes, bs, n, ir_len, K,
                        inputs, outputs, hop, chunk_items, stream);
}

// ------------------------------------------------------------------ noise_shaped_impulse_response
// The reverb's IR synthesis with the planar sink: the geometry of the reverb at n = L (leff = L, every tap), the same
// synthesis variants, chunk loop and Philox keys, no convolution.  L = 1 runs the kernels with a time axis of length 2,
// whose tap 0 is 0 like torch.linspace(0, 1, 1); everything that addresses memory (the noise rows, the IR rows) uses
// the true L.  Backward: dL/dIR is time-domain and planar, so ir_pack_kernel puts it where the reverb's inverse
// transform leaves its dL/dIR, and the reverb's band contraction (ir_grad_pp_kernel / ir_grad_pairs_kernel) and
// two-stage sums (reverb_param_grad_kernel) run unchanged on the 25-wide rows of nsir_params_kernel.
namespace {
int make_nsir_geom(int64_t bs, int64_t L, int64_t taps, int64_t chunk, Geom& g) {
  DASP_REQUIRE(L >= 1, "impulse response: bad num_samples=%lld", (long long)L);
  return make_geom(bs, L, L < 2 ? 2 : L, taps, chunk, g);
}

// workspace: fwd = 25-wide parameter rows, the filtered noise of a chunk when f_save is not kept, the cuFFT work area;
// bwd = the parameter rows, their 25-wide gradients, dL/dIR in the partition layout, the band-gradient partials
struct NsirWs { size_t p25, f, cufft, fwd_total, g25, et, part, bwd_total; Plans full, rem; };
int64_t nsir_nparts(const Geom& g) { return g.nbk > g.nparts_pp() ? g.nbk : g.nparts_pp(); }
int nsir_setup(const Geom& g, NsirWs& w) {
  int rc;
  size_t work = 0;
  for (int64_t items : {g.bs > 0 ? g.chunk : 0, g.bs % g.chunk}) {
    if (items == 0) continue;
    if ((rc = synth_plans(g, items, items == g.chunk ? w.full : w.rem, work)) != DASP_OK) return rc;
  }
  size_t o = 0;
  w.p25 = o;  o += align256(sizeof(float) * (size_t)(g.chunk * 25));
  w.f = o;    o += align256(sizeof(float2) * (size_t)(g.chunk * kBands * g.pair_c64()));
  w.cufft = o; o += align256(work);
  w.fwd_total = o;
  o = w.p25 + align256(sizeof(float) * (size_t)(g.chunk * 25));
  w.g25 = o;  o += align256(sizeof(float) * (size_t)(g.chunk * 25));
  w.et = o;   o += align256(sizeof(float2) * (size_t)(g.chunk * g.jb * kNbA));
  w.part = o; o += align256(sizeof(float) * (size_t)(g.chunk * nsir_nparts(g) * kBands * 2));
  w.bwd_total = o;
  return DASP_OK;
}
}  // namespace

int dasp_nsir_geometry(int64_t bs, int64_t num_samples, int64_t taps, int64_t chunk_items, dasp_reverb_geom* out) {
  DASP_REQUIRE(out != nullptr, "impulse response geometry: null out");
  Geom g;
  int rc = make_nsir_geom(bs, num_samples, taps, chunk_items, g);
  if (rc != DASP_OK) return rc;
  std::lock_guard<std::mutex> lk(g_mu);
  NsirWs w{};
  if ((rc = nsir_setup(g, w)) != DASP_OK) return rc;
  out->nb = g.nb; out->hop = g.hop; out->nbk = g.nbk; out->leff = g.leff; out->rpp = g.rpp;
  out->conv_block = kB; out->x_blocks = 0; out->ir_partitions = g.jb; out->chunk_items = g.chunk;
  out->f_floats = bs * kBands * g.pair_c64() * 2;
  out->xspec_c64 = 0; out->irspec_c64 = 0;
  out->fwd_workspace_bytes = (int64_t)w.fwd_total;
  out->bwd_workspace_bytes = (int64_t)w.bwd_total;
  return DASP_OK;
}

int dasp_nsir_fwd(const float* params, const float* noise, const uint64_t* seed_dev, float* ir_out, float* f_save,
                  void* workspace, int64_t workspace_bytes, int64_t bs, int64_t num_samples, int64_t taps,
                  int64_t chunk_items, float sample_rate, void* stream) {
  Geom g;
  int rc = make_nsir_geom(bs, num_samples, taps, chunk_items, g);
  if (rc != DASP_OK) return rc;
  if (bs == 0) return DASP_OK;
  DASP_REQUIRE(params && ir_out && workspace, "impulse response fwd: null pointer");
  DASP_REQUIRE(noise != nullptr || seed_dev != nullptr,
               "impulse response fwd: device-noise mode needs seed_dev (a device pointer)");
  const unsigned long long* seed = reinterpret_cast<const unsigned long long*>(seed_dev);
  cudaStream_t st = (cudaStream_t)stream;
  std::lock_guard<std::mutex> lk(g_mu);
  Synth sy;
  if ((rc = choose_synth(g, num_samples, noise, seed, (double)sample_rate, st, sy)) != DASP_OK) return rc;
  NsirWs w{};
  if ((rc = nsir_setup(g, w)) != DASP_OK) return rc;
  if ((rc = check_workspace("impulse response fwd", w.fwd_total, workspace_bytes)) != DASP_OK) return rc;
  unsigned char* base = (unsigned char*)workspace;
  float* p25 = (float*)(base + w.p25);

  for (int64_t item0 = 0; item0 < bs; item0 += g.chunk) {
    const int64_t items = (bs - item0 < g.chunk) ? bs - item0 : g.chunk;
    const Plans& pl = (items == g.chunk) ? w.full : w.rem;
    float2* C = f_save ? reinterpret_cast<float2*>(f_save) + item0 * kBands * g.pair_c64()
                       : reinterpret_cast<float2*>(base + w.f);
    nsir_params_kernel<<<(unsigned)((items * 25 + 255) / 256), 256, 0, st>>>(params + item0 * 24, p25, items);
    DASP_LAUNCH_OK("nsir_params_kernel");
    if ((rc = synth_chunk(g, sy, PlanarSink{ir_out + item0 * 2 * num_samples, num_samples}, p25, C, f_save != nullptr,
                          pl, base + w.cufft, item0, items, st, nullptr)) != DASP_OK)
      return rc;
  }
  return DASP_OK;
}

int dasp_nsir_bwd(const float* gir, const float* params, const float* f_save, float* gparams, void* workspace,
                  int64_t workspace_bytes, int64_t bs, int64_t num_samples, int64_t taps, int64_t chunk_items,
                  int64_t device_noise, void* stream) {
  Geom g;
  int rc = make_nsir_geom(bs, num_samples, taps, chunk_items, g);
  if (rc != DASP_OK) return rc;
  if (bs == 0) return DASP_OK;
  DASP_REQUIRE(gir && params && f_save && gparams && workspace, "impulse response bwd: null pointer");
  const bool polyphase = polyphase_f(g, device_noise != 0);   // the layout the forward left in f_save
  cudaStream_t st = (cudaStream_t)stream;
  std::lock_guard<std::mutex> lk(g_mu);
  NsirWs w{};
  if ((rc = nsir_setup(g, w)) != DASP_OK) return rc;
  if ((rc = check_workspace("impulse response bwd", w.bwd_total, workspace_bytes)) != DASP_OK) return rc;
  unsigned char* base = (unsigned char*)workspace;
  float* p25 = (float*)(base + w.p25);
  float* g25 = (float*)(base + w.g25);
  float2* et = (float2*)(base + w.et);
  float* part = (float*)(base + w.part);
  const int J = (int)g.jb;

  for (int64_t item0 = 0; item0 < bs; item0 += g.chunk) {
    const int64_t items = (bs - item0 < g.chunk) ? bs - item0 : g.chunk;
    const float2* C = reinterpret_cast<const float2*>(f_save) + item0 * kBands * g.pair_c64();
    nsir_params_kernel<<<(unsigned)((items * 25 + 255) / 256), 256, 0, st>>>(params + item0 * 24, p25, items);
    DASP_LAUNCH_OK("nsir_params_kernel");
    ir_pack_kernel<<<dim3((unsigned)((g.leff + 255) / 256), (unsigned)items, 1), 256, 0, st>>>(
        gir, et, item0, J, num_samples, g.leff, 2, false);
    DASP_LAUNCH_OK("ir_pack_kernel");
    int nparts;
    if ((rc = ir_grad_chunk(g, polyphase, et, C, p25, part, items, st, nparts)) != DASP_OK) return rc;
    // mix_blocks 0: the mix column of g25 is 0 and is not copied out
    reverb_param_grad_kernel<<<(unsigned)((items * 25 + 127) / 128), 128, 0, st>>>(part, nullptr, p25, g25, 0, items,
                                                                                   nparts, 0);
    DASP_LAUNCH_OK("reverb_param_grad_kernel");
    DASP_CUDA_OK(cudaMemcpy2DAsync(gparams + item0 * 24, 24 * sizeof(float), g25, 25 * sizeof(float),
                                   24 * sizeof(float), (size_t)items, cudaMemcpyDeviceToDevice, st));
  }
  return DASP_OK;
}

}  // extern "C"
