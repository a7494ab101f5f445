/* dasp_b200.h -- C ABI of libdasp_b200.so: the H100 (sm_90a) kernels behind
 * dasp_pytorch.functional's batched audio-processor hot path.
 *
 * The reference (csteinmetz1/dasp-pytorch @ c9ae0126) is pure Python and has no FFI of its
 * own; each entry point below replaces the arithmetic of one reference function and is what
 * a ctypes/cffi binding inside that function would call (INTEGRATION.md shows the binding).
 *
 * Conventions
 *   - every pointer is a DEVICE pointer to contiguous fp32 (unless stated), owned by the
 *     caller; the library never allocates tensors -- scratch comes in through `ws`
 *     arguments sized by the matching *_workspace_* query;
 *   - audio tensors are (batch, channels, samples) row-major, exactly the reference's
 *     tensor contract (README.md:38);
 *   - `stream` is a cudaStream_t; all work is enqueued on it, nothing synchronises -- with ONE documented
 *     exception: the first call on a device for a new (taps, sample_rate, geometry) builds library-owned caches
 *     (cuFFT plans, filter-bank spectra, FFT twiddle tables: cudaMalloc + one cudaStreamSynchronize; for the
 *     reverb forward also a side stream at the greatest priority and two events).  Warm the shapes up once
 *     before capturing a CUDA graph -- the first call should not be under capture; later calls are pure enqueues.
 *     dasp_reverb_fwd with f_save and irspec_save (a backward follows) runs each chunk's IR synthesis on that side
 *     stream, forked from `stream` by an event recorded on it at the start of the call and joined back into it
 *     before the call returns (event waits, which stream capture turns into graph edges), so the caller still sees
 *     one stream;
 *   - return value 0 = ok, negative = error (see DASP_ERR_*); the message is available
 *     from dasp_last_error() (thread-local).  No exception crosses this boundary;
 *   - reentrant from several host threads as long as they use distinct streams.
 */
#ifndef DASP_B200_H_
#define DASP_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DASP_ABI_VERSION 2

#define DASP_OK 0
#define DASP_ERR_INVALID (-1)   /* bad shape / null pointer / misalignment        */
#define DASP_ERR_CUDA (-2)      /* CUDA runtime call or kernel launch failed      */
#define DASP_ERR_CUFFT (-3)     /* cuFFT call failed                              */
#define DASP_ERR_WORKSPACE (-4) /* caller workspace smaller than *_workspace_*()  */

/* ---- library ---------------------------------------------------------------------- */
int dasp_abi_version(void);
const char* dasp_last_error(void);
/* compiled-for architecture as an integer (900 for sm_90a) */
int dasp_compiled_arch(void);
/* frees cached cuFFT plans and device-side filter-bank spectra */
void dasp_shutdown(void);
/* The dasp_debug_* entry points are TEST HOOKS: process-global switches, not thread-safe, not for production
 * callers (they exist so that every kernel variant can be pinned against the oracle at small sizes). */
/* test hook: pin the warps-per-row variant of the scan kernels (1, 2, 3, 4, 8, 16; 0 = automatic choice; a kernel
 * family without the requested variant keeps its automatic choice) */
void dasp_debug_force_warps(int warps);
/* test hook: pin the number of x / dL/dy stages per warp of the EQ backward (1 or 2; 0 = automatic) */
void dasp_debug_eq_bwd_stages(int stages);
/* test hook: pin the number of load stages per warp of the EQ forward (1 or 2; 0 = automatic) */
void dasp_debug_eq_fwd_stages(int stages);
/* test hook: 1 = the EQ kernels use (row A, row B) pair coefficient tables even when both rows of every pair belong
 * to one item (even channel counts); 0 = automatic (pair tables only where a pair straddles two items) */
void dasp_debug_eq_pair_tables(int on);
/* test hook, IR synthesis of the device-noise reverb (all variants draw the same Philox stream and must agree):
   0 = automatic (block FFT of 8192 points: one warp-specialised thread-block-cluster kernel for polyphase factors
   R <= 6, generator -> fused in-shared-memory inverse FFT + shaping kernel otherwise),
   1 = generator -> batched cuFFT -> shaping kernel,
   2 = generator -> fused in-shared-memory inverse FFT + shaping kernel for R <= 8 */
void dasp_debug_reverb_path(int path);
/* test hook: variant used by the last chunk of the most recent dasp_reverb_fwd: 0 = cuFFT pipeline, 1 = generator +
   fused FFT/shaping kernel selected by dasp_debug_reverb_path(2), 2 = the default own-FFT synthesis (cluster kernel
   or generator + fused FFT/shaping kernel) */
int dasp_debug_reverb_last_path(void);

/* test hook: 1 = the IR synthesis uses unit-impulse filters, so the f_save buffer of dasp_reverb_fwd returns the white
   noise itself (used to rebuild a reference-style noise tensor): the periodic sequences w_k of the spectral generator
   (polyphase layout), or, on the overlap-save path (caller's noise, or device noise with a polyphase factor > 16), the
   noise blocks C[((item*12 + k)*nbk + b)*nb + m] = noise[b*hop + m] */
void dasp_debug_reverb_flat_filterbank(int on);

/* ---- Processor.denormalize_param_dict on the device      (reference modules.py:13-14, 70-91) ------
 * out[r][c] = lo[c] + p01[r][c] * span[c].  The reference's range check (ValueError when a value leaves [0, 1])
 * cannot raise from the device: an offending element becomes NaN and bit 0 of *flag (device int, may be NULL)
 * is set; the host reads the flag whenever it can afford to (modules.Processor does so outside graph capture). */
int dasp_denormalize(const float* p01, const float* lo /* [cols] */, const float* span /* [cols] */, float* out,
                     int* flag, int64_t rows, int64_t cols, void* stream);

/* ---- gain: y = x * 10^(gain_db/20)            (reference functional.py:10-29) ------ */
int dasp_gain_fwd(const float* x, const float* gain_db /* [bs] */, float* y, int64_t bs, int64_t chs,
                  int64_t n, void* stream);
int dasp_gain_bwd(const float* gy, const float* x, const float* gain_db, float* gx,
                  float* g_gain_db /* [bs] */, float* ws, int64_t ws_floats, int64_t bs, int64_t chs,
                  int64_t n, void* stream);

/* ---- distortion: y = tanh(x * 10^(drive_db/20))   (reference functional.py:65-78) --
 * rows = bs*chs; one drive value per row (the reference's drive_db.view(bs, chs, -1)). */
int dasp_distortion_fwd(const float* x, const float* drive_db /* [rows] */, float* y, int64_t rows,
                        int64_t n, void* stream);
int dasp_distortion_bwd(const float* gy, const float* x, const float* drive_db, float* gx,
                        float* g_drive_db /* [rows] */, float* ws, int64_t ws_floats, int64_t rows,
                        int64_t n, void* stream);
/* floats of scratch the two *_bwd calls above need (rows = bs for gain with n = chs*N) */
int64_t dasp_pointwise_bwd_workspace_floats(int64_t rows, int64_t n);

/* ---- stereo_widener / stereo_panner / stereo_bus      (reference functional.py:580-604, 607-636, 32-62) --
 * widener: x, y (bs, 2, n), width [bs].   panner: x (bs, tracks, n), pan [bs*tracks], y (bs, 2, tracks, n).
 * bus: x (bs, 2, tracks, n), send_db [bs*tracks], y (bs, 2, n).
 * ws: dasp_stereo_bwd_workspace_floats(rows, n) floats with rows = bs (widener), bs*tracks (panner),
 * bs*2*tracks (bus). */
int64_t dasp_stereo_bwd_workspace_floats(int64_t rows, int64_t n);
int dasp_widener_fwd(const float* x, const float* width, float* y, int64_t bs, int64_t n, void* stream);
int dasp_widener_bwd(const float* gy, const float* x, const float* width, float* gx, float* g_width, float* ws,
                     int64_t ws_floats, int64_t bs, int64_t n, void* stream);
int dasp_panner_fwd(const float* x, const float* pan, float* y, int64_t bs, int64_t tracks, int64_t n, void* stream);
int dasp_panner_bwd(const float* gy, const float* x, const float* pan, float* gx, float* g_pan, float* ws,
                    int64_t ws_floats, int64_t bs, int64_t tracks, int64_t n, void* stream);
int dasp_bus_fwd(const float* x, const float* send_db, float* y, int64_t bs, int64_t tracks, int64_t n, void* stream);
int dasp_bus_bwd(const float* gy, const float* x, const float* send_db, float* gx, float* g_send_db, float* ws,
                 int64_t ws_floats, int64_t bs, int64_t tracks, int64_t n, void* stream);

/* ---- compressor / expander            (reference functional.py:275-399; :402-403 stub) --
 * kind: 0 = compressor (reference semantics: attack-only smoothing, release_ms unused),
 *       1 = downward expander (new op, same signature; the reference only stubs it).
 * Parameters are [bs] arrays.  `ckpt` (fwd: optional out, bwd: in) holds the smoother state at
 * every tile boundary: bs * ceil(n / dasp_dynamics_tile_len(bs, chs)) floats; pass NULL in the
 * forward when no backward will follow.  gparams is [bs][6] in signature order
 * (threshold, ratio, attack, release(=0), knee, makeup).  g_scratch (bs*n floats) is only
 * needed when lookahead > 0. */
int64_t dasp_dynamics_tile_len(int64_t bs, int64_t chs);
int dasp_dynamics_fwd(int kind, const float* x, const float* threshold_db, const float* ratio,
                      const float* attack_ms, const float* knee_db, const float* makeup_db, float* y,
                      float* ckpt, int64_t bs, int64_t chs, int64_t n, float sample_rate, float eps,
                      int64_t lookahead, void* stream);
int dasp_dynamics_bwd(int kind, const float* gy, const float* x, const float* threshold_db,
                      const float* ratio, const float* attack_ms, const float* knee_db,
                      const float* makeup_db, const float* ckpt, float* gx, float* gparams,
                      float* g_scratch, int64_t bs, int64_t chs, int64_t n, float sample_rate, float eps,
                      int64_t lookahead, void* stream);
/* External side chain: the gain is computed from a key (bs, key_chs, n) instead of from x (ducking, de-essing with an
 * EQ'd copy of x, gating one track from another).  side = the sum of the key_chs key channels (fp64, rounded once),
 * then the same level, static curve, attack smoother and makeup; y[b,c,t] = x[b,c,t-lookahead] * G[b,t] (the key is
 * not delayed).  1 <= key_chs <= 32 and 2 * chs + key_chs <= 76: the backward streams x, dL/dy -> dL/dx and
 * key -> dL/dkey through three shared-memory stages, which hold 76 tiles of the smallest (224-sample) geometry in
 * 200 KB.  Other combinations return -1 before any CUDA call, and the tile-length query returns 0 for them.
 * ckpt holds bs * ceil(n / dasp_dynamics_sidechain_tile_len(bs, chs, key_chs)) floats.  Backward: gx = gy * G with no
 * detector term (shifted by the look-ahead); gkey (bs, key_chs, n) receives dL/dside, so all its key_chs rows of an
 * item are equal; gkey may be NULL, which writes no key gradient.  gparams and g_scratch as above. */
int64_t dasp_dynamics_sidechain_tile_len(int64_t bs, int64_t chs, int64_t key_chs);
int dasp_dynamics_sidechain_fwd(int kind, const float* x, const float* key, int64_t key_chs,
                                const float* threshold_db, const float* ratio, const float* attack_ms,
                                const float* knee_db, const float* makeup_db, float* y, float* ckpt, int64_t bs,
                                int64_t chs, int64_t n, float sample_rate, float eps, int64_t lookahead, void* stream);
int dasp_dynamics_sidechain_bwd(int kind, const float* gy, const float* x, const float* key, int64_t key_chs,
                                const float* threshold_db, const float* ratio, const float* attack_ms,
                                const float* knee_db, const float* makeup_db, const float* ckpt, float* gx,
                                float* gkey /* may be NULL */, float* gparams, float* g_scratch, int64_t bs,
                                int64_t chs, int64_t n, float sample_rate, float eps, int64_t lookahead,
                                void* stream);
/* The gain curve on its own: the detector of dasp_dynamics_fwd on x (bs, chs, n), 1 <= chs <= 32, and no audio path.
 * g (bs, 1, n) receives G[b,t] = 10^((s + M) / 20), or s + M in dB when db != 0 (s: the smoothed static curve,
 * M: makeup).  The tiles are dasp_dynamics_fwd's for the same (bs, chs), so G is bit-identical to the gain that
 * dasp_dynamics_fwd multiplies into x[b,c,t-lookahead], and ckpt holds bs * ceil(n / dasp_dynamics_tile_len(bs, chs))
 * floats (NULL in the forward when no backward will follow).  Backward: gg (bs, 1, n) is dL/dg (dL/d(dB) when db);
 * gside (bs, 1, n) receives dL/dside, the gradient every channel of x gets, which is 0 where |side| < eps; gparams as
 * above.  Bad shapes and channel counts return -1 before any CUDA call. */
int dasp_dynamics_gain_fwd(int kind, const float* x, int64_t chs, const float* threshold_db, const float* ratio,
                           const float* attack_ms, const float* knee_db, const float* makeup_db, float* g, float* ckpt,
                           int64_t bs, int64_t n, float sample_rate, float eps, int db, void* stream);
int dasp_dynamics_gain_bwd(int kind, const float* gg, const float* x, const float* threshold_db, const float* ratio,
                           const float* attack_ms, const float* knee_db, const float* makeup_db, const float* ckpt,
                           float* gside, float* gparams, int64_t bs, int64_t chs, int64_t n, float sample_rate,
                           float eps, int db, void* stream);

/* ---- parametric_eq: six cascaded biquads   (reference functional.py:118-272 with
 *      signal.biquad signal.py:242-306 and signal.sosfilt_via_fsm signal.py:136-166) ------
 * params is [bs][18] = (gain_dB, cutoff_Hz, Q) for low shelf, band0..band3, high shelf, i.e. the
 * 18 tensors of the reference signature stacked in order; the same filter is applied to every
 * channel of an item (signal.py:157-158).  Rows (item, channel) are processed in pairs; ckpt (fwd: optional out,
 * bwd: in) holds the section states of a pair at every tile boundary: dasp_eq_ckpt_floats(bs, chs, n) floats
 * (tiles of dasp_eq_tile_len() samples).  gparams is [bs][18]; ws needs dasp_eq_bwd_workspace_floats(bs, chs)
 * floats. */
int64_t dasp_eq_tile_len(int64_t rows);
int64_t dasp_eq_ckpt_floats(int64_t bs, int64_t chs, int64_t n);
int64_t dasp_eq_bwd_workspace_floats(int64_t bs, int64_t chs);
int dasp_eq_fwd(const float* x, const float* params, float* y, float* ckpt, int64_t bs, int64_t chs,
                int64_t n, float sample_rate, void* stream);
int dasp_eq_bwd(const float* gy, const float* x, const float* params, const float* ckpt, float* gx,
                float* gparams, float* ws, int64_t ws_floats, int64_t bs, int64_t chs, int64_t n,
                float sample_rate, void* stream);

/* ---- parametric_eq_frequency_response: the EQ's transfer function on a caller's frequency grid
 *      (reference signal.fft_sosfreqz signal.py:14-32, on any grid instead of rfft bins) ----------------------------
 * params is [bs][18] as for dasp_eq_fwd; freqs_hz is [nfreq] frequencies in Hz (any finite value: H is periodic in
 * sample_rate).  h is (bs, nfreq) complex, interleaved (re, im):
 *   h[b][f] = prod_k H_k(exp(j 2 pi freqs_hz[f] / sample_rate)),  the six sections dasp_eq_fwd runs,
 * evaluated in fp32 in the sigma form of the recursion with coefficients designed in fp64.  Backward: gh is the
 * gradient (dL/dRe h, dL/dIm h) in the same layout, gparams [bs][18] receives
 *   dL/dtheta = sum_f Re(conj(gh[b][f]) dh[b][f]/dtheta)
 * (per-item sums in fp64, fixed order: two backward calls give the same bits).  Both recompute what they need from
 * params and freqs_hz; ws is dasp_eq_response_workspace_floats(bs, nfreq) floats (8-byte aligned) for either
 * direction.  bs = 0, and a forward with nfreq = 0, return 0 without touching the device; a backward with nfreq = 0
 * only zeroes gparams on `stream`. */
int64_t dasp_eq_response_workspace_floats(int64_t bs, int64_t nfreq);
int dasp_eq_response_fwd(const float* params, const double* freqs_hz, float* h, float* ws, int64_t ws_floats,
                         int64_t bs, int64_t nfreq, float sample_rate, void* stream);
int dasp_eq_response_bwd(const float* gh, const float* params, const double* freqs_hz, float* gparams, float* ws,
                         int64_t ws_floats, int64_t bs, int64_t nfreq, float sample_rate, void* stream);

/* ---- noise_shaped_reverberation         (reference functional.py:406-577, filter bank
 *      signal.octave_band_filterbank signal.py:42-92) --------------------------------------
 * params is [bs][25] = 12 band gains, 12 band decays, mix (signature order).  x is (bs, in_chs, n)
 * with in_chs 1 or 2; y is always (bs, 2, n) (mono is duplicated, functional.py:493-495).
 * noise: NULL -> white noise is generated on the device (Philox4x32-10, keyed by the 64-bit value the kernels read
 *        from the DEVICE pointer `seed_dev` when they run -- so a captured CUDA graph draws fresh noise on every
 *        replay as long as the caller's graph also refreshes that word, as torch's graph-safe generator does);
 *        else the (bs*2, 12, num_samples + taps - 1) tensor the reference would have drawn
 *        (functional.py:547-548) -- the parity-test entry.
 * Buffers kept for the backward (pass NULL for all three when no backward follows):
 *   f_save  geom.f_floats floats (band-filtered noise blocks, left/right channel interleaved as complex pairs),
 *   xspec_save  geom.xspec_c64 complex64, irspec_save  geom.irspec_c64 complex64 (block spectra).
 *   The wet signal is not kept: the backward forms dL/dmix from x and the gradient it propagates to x.
 * workspace: geom.fwd_workspace_bytes / geom.bwd_workspace_bytes bytes of device memory. */
typedef struct dasp_reverb_geom {
  int64_t nb, hop, nbk;       /* IR synthesis, overlap-save path: block length, hop, blocks per band signal */
  int64_t leff;               /* min(num_samples, n): IR taps that can reach the n output samples */
  int64_t rpp;                /* IR synthesis, spectral path: polyphase factor (n1 = rpp * nb >= leff + taps - 1) */
  int64_t conv_block;         /* audio convolution: partition / hop length (its FFT length is twice that) */
  int64_t x_blocks;           /* ceil(n / conv_block) */
  int64_t ir_partitions;      /* ceil(leff / conv_block) */
  int64_t chunk_items;        /* items processed per pass */
  int64_t f_floats, xspec_c64, irspec_c64;  /* sizes of the buffers kept for the backward */
  int64_t fwd_workspace_bytes, bwd_workspace_bytes;
} dasp_reverb_geom;
int dasp_reverb_geometry(int64_t bs, int64_t n, int64_t num_samples, int64_t taps, int64_t chunk_items,
                         dasp_reverb_geom* out);
int dasp_reverb_fwd(const float* x, int64_t in_chs, const float* params, const float* noise, const uint64_t* seed_dev,
                    float* y, float* f_save, void* xspec_save, void* irspec_save,
                    void* workspace, int64_t workspace_bytes, int64_t bs, int64_t n, int64_t num_samples,
                    int64_t taps, int64_t chunk_items, float sample_rate, void* stream);
int dasp_reverb_bwd(const float* gy, const float* x, int64_t in_chs, const float* params,
                    const float* f_save, const void* xspec_save,
                    const void* irspec_save, float* gx, float* gparams, void* workspace,
                    int64_t workspace_bytes, int64_t bs, int64_t n, int64_t num_samples, int64_t taps,
                    int64_t chunk_items, int64_t device_noise /* 1 iff the forward ran with noise == NULL */,
                    void* stream);
/* host-only: the 12 x taps fp32 filter bank (scipy.signal.firwin restated; no GPU needed) */
int dasp_reverb_filterbank(int64_t taps, double sample_rate, float* out);

/* ---- noise_shaped_impulse_response: the reverb's IR synthesis on its own      (reference functional.py:547-567) ----
 * params is [bs][24] = 12 band gains, 12 band decays (the reverb's first 24); ir_out is (bs, 2, num_samples):
 *   IR[b][c][t] = (1/12) sum_k gain_k exp(-(10 decay_k + 1) tt(t)) f[b][c][k][t],  tt = torch.linspace(0, 1, L)
 * for every t < num_samples (num_samples >= 1; tt = 0 at num_samples 1).  noise / seed_dev as in dasp_reverb_fwd; the
 * synthesis variants, their test hooks (dasp_debug_reverb_path, dasp_debug_reverb_last_path,
 * dasp_debug_reverb_flat_filterbank) and the Philox keys are the reverb's, with leff = num_samples.  So with the same
 * seed word the taps are the bits the reverb convolves when n >= num_samples.
 * The geometry is the reverb's struct: leff = num_samples, rpp and f_floats as dasp_reverb_geometry at n = num_samples
 * (num_samples >= 2), x_blocks = xspec_c64 = irspec_c64 = 0.  f_save (geom.f_floats floats, or NULL when no backward
 * follows) keeps the band-filtered noise for the backward.  Backward: gir is dL/dIR (bs, 2, num_samples), gparams
 * [bs][24]; device_noise is 1 iff the forward ran with noise == NULL.  workspace: geom.fwd_workspace_bytes /
 * geom.bwd_workspace_bytes.  A geometry query with bs = 0 needs no GPU. */
int dasp_nsir_geometry(int64_t bs, int64_t num_samples, int64_t taps, int64_t chunk_items, dasp_reverb_geom* out);
int dasp_nsir_fwd(const float* params, const float* noise, const uint64_t* seed_dev, float* ir_out,
                  float* f_save /* may be NULL */, void* workspace, int64_t workspace_bytes, int64_t bs,
                  int64_t num_samples, int64_t taps, int64_t chunk_items, float sample_rate, void* stream);
int dasp_nsir_bwd(const float* gir, const float* params, const float* f_save, float* gparams, void* workspace,
                  int64_t workspace_bytes, int64_t bs, int64_t num_samples, int64_t taps, int64_t chunk_items,
                  int64_t device_noise, void* stream);

/* ---- convolution_reverberation: the reverb's apply stage with a caller-supplied impulse response
 *      (reference functional.py:569-575: y = (1 - mix) x + mix (x * IR), causal, cropped to n) --------------
 * x is (bs, in_chs, n), ir is (bs, ir_chs, ir_len) with in_chs 1 or 2 and ir_chs 1, 2 or 4 (mono is used for both
 * channels; 4 is a true-stereo IR, see below), mix is [bs]; y is always (bs, 2, n).  Any ir_len >= 1; only the first leff = min(ir_len, n) taps reach the output.
 * The convolution is the reverb's: uniformly partitioned overlap-save on conv_block-sample partitions.
 * Buffers kept for the backward (pass NULL for both when no backward follows):
 *   xspec_save  geom.xspec_c64 complex64 (audio block spectra), irspec_save  geom.irspec_c64 complex64 (IR partitions).
 * Backward: gx is (bs, in_chs, n) (mono receives the sum of both channel gradients), gmix [bs], gir (bs, ir_chs, ir_len)
 * or NULL, which skips all dL/dIR work; a mono IR receives the sum of both channel gradients and taps >= leff get 0.
 * workspace: geom.fwd_workspace_bytes / geom.bwd_workspace_bytes bytes of device memory.  A geometry query with
 * bs = 0 needs no GPU (its workspace sizes then leave out the cuFFT work area). */
typedef struct dasp_conv_geom {
  int64_t leff;               /* min(ir_len, n): IR taps that can reach the n output samples */
  int64_t conv_block;         /* partition / hop length (its FFT length is twice that) */
  int64_t x_blocks;           /* ceil(n / conv_block) */
  int64_t ir_partitions;      /* ceil(leff / conv_block) */
  int64_t chunk_items;        /* items processed per pass */
  int64_t xspec_c64, irspec_c64;  /* sizes of the buffers kept for the backward */
  int64_t fwd_workspace_bytes, bwd_workspace_bytes;
} dasp_conv_geom;
int dasp_conv_geometry(int64_t bs, int64_t n, int64_t ir_len, int64_t chunk_items, dasp_conv_geom* out);
int dasp_conv_fwd(const float* x, int64_t in_chs, const float* ir, int64_t ir_chs, int64_t ir_len, const float* mix,
                  float* y, void* xspec_save, void* irspec_save, void* workspace, int64_t workspace_bytes, int64_t bs,
                  int64_t n, int64_t chunk_items, void* stream);
int dasp_conv_bwd(const float* gy, const float* x, int64_t in_chs, int64_t ir_chs, int64_t ir_len, const float* mix,
                  const void* xspec_save, const void* irspec_save, float* gx, float* gir /* may be NULL */, float* gmix,
                  void* workspace, int64_t workspace_bytes, int64_t bs, int64_t n, int64_t chunk_items, void* stream);
/* One impulse response for the whole batch: the same argument lists, with ir (fwd) and gir (bwd) pointing at ONE
 * (ir_chs, ir_len) IR that applies to every item.  Its partitions are transformed once per call instead of once per
 * item, and gir receives the sum over the items of each item's dL/dIR (fp64, in item order: the same bits for every
 * chunk_items).  The geometry is the same struct: irspec_c64 is one IR's (0 at bs = 0), and the workspace sizes include
 * the fp64 gradient sum of the backward. */
int dasp_conv_shared_geometry(int64_t bs, int64_t n, int64_t ir_len, int64_t chunk_items, dasp_conv_geom* out);
int dasp_conv_shared_fwd(const float* x, int64_t in_chs, const float* ir, int64_t ir_chs, int64_t ir_len,
                         const float* mix, float* y, void* xspec_save, void* irspec_save, void* workspace,
                         int64_t workspace_bytes, int64_t bs, int64_t n, int64_t chunk_items, void* stream);
int dasp_conv_shared_bwd(const float* gy, const float* x, int64_t in_chs, int64_t ir_chs, int64_t ir_len,
                         const float* mix, const void* xspec_save, const void* irspec_save, float* gx,
                         float* gir /* may be NULL */, float* gmix, void* workspace, int64_t workspace_bytes, int64_t bs,
                         int64_t n, int64_t chunk_items, void* stream);
/* True-stereo IR: ir_chs = 4 in all four dasp_conv[_shared]_fwd / _bwd calls above.  Rows are input-major, row 2 i + o
 * is the path from input channel i to output channel o (L->L, L->R, R->L, R->R):
 *   wet_L = x_L * h0 + x_R * h2,  wet_R = x_L * h1 + x_R * h3,  y = (1 - mix) x + mix wet.
 * gir is (bs, 4, ir_len) (shared: (4, ir_len)).  Its buffers are larger than a mono/stereo IR's (irspec_save, the IR
 * partition regions of both workspaces and the shared backward's fp64 sum hold two partition sets per IR), so size them
 * with these two queries; ir_partitions is still ceil(leff / conv_block), the partitions of one set, and irspec_c64 is
 * 2 * ir_partitions * 2 * conv_block per IR. */
int dasp_conv_ts_geometry(int64_t bs, int64_t n, int64_t ir_len, int64_t chunk_items, dasp_conv_geom* out);
int dasp_conv_shared_ts_geometry(int64_t bs, int64_t n, int64_t ir_len, int64_t chunk_items, dasp_conv_geom* out);
/* test hook: dispatch of the most recent call.  which = 0: dasp_conv_fwd / dasp_conv_shared_fwd, bit 0 = own
   in-shared-memory FFT, clear = cuFFT pipeline (dasp_debug_reverb_path(1), n % 4 != 0, rows not 16-byte aligned),
   bit 1 = shared IR, bit 2 = true-stereo IR.  which = 1: dasp_conv_bwd / dasp_conv_shared_bwd, bit 0 = own FFT,
   bit 1 = fused correlation kernel, bit 2 = dL/dIR computed, bit 3 = shared IR, bit 4 = true-stereo IR */
int dasp_debug_conv_last_path(int which);

/* ---- convolution_bus: S input rows, each through its own impulse responses, summed into a mono or stereo bus ------
 * x is (bs, S, n), ir is (bs, S, O, ir_len) (or ONE (S, O, ir_len) IR set for the whole batch: the *_shared_* entry
 * points), y is (bs, O, n), with 1 <= S <= DASP_CONV_BUS_MAX_INPUTS inputs and O = 1 or 2 outputs:
 *   y[b, o] = sum_s (x[b, s] * ir[b, s, o])[:n]   (* the causal convolution, as convolution_reverberation's wet signal)
 * There is no dry/wet mix: inputs and outputs differ in number, so no dry signal is defined.
 * The convolution is convolution_reverberation's (conv_block-sample partitions, the same FFT), with the rows of every
 * signal packed two per transform: ceil(S / 2) window spectra per block, ceil(S O / 2) partition sets per IR.
 * n % 4 == 0 and 16-byte aligned x / gy rows are required (the transforms bulk-copy them).
 * Buffers kept for the backward (NULL for both when no backward follows): xspec_save geom.xspec_c64 and irspec_save
 * geom.irspec_c64 complex64.  Backward: gx (bs, S, n); gir (bs, S, O, ir_len) (shared: (S, O, ir_len), the sum over
 * the items in fp64 in item order, the same bits for every chunk_items), or NULL, which skips all dL/dIR work; taps
 * >= leff = min(ir_len, n) get 0.  Workspace sizes come from dasp_conv_bus_geometry (shared != 0 for the shared entry
 * points), which needs no GPU.  Bad S, O or shapes are rejected before any CUDA call. */
#define DASP_CONV_BUS_MAX_INPUTS 32
int dasp_conv_bus_geometry(int64_t bs, int64_t n, int64_t ir_len, int64_t inputs, int64_t outputs, int64_t shared,
                           int64_t chunk_items, dasp_conv_geom* out);
int dasp_conv_bus_fwd(const float* x, const float* ir, float* y, void* xspec_save, void* irspec_save, void* workspace,
                      int64_t workspace_bytes, int64_t bs, int64_t n, int64_t ir_len, int64_t inputs, int64_t outputs,
                      int64_t chunk_items, void* stream);
int dasp_conv_bus_bwd(const float* gy, const void* xspec_save, const void* irspec_save, float* gx,
                      float* gir /* may be NULL */, void* workspace, int64_t workspace_bytes, int64_t bs, int64_t n,
                      int64_t ir_len, int64_t inputs, int64_t outputs, int64_t chunk_items, void* stream);
int dasp_conv_bus_shared_fwd(const float* x, const float* ir, float* y, void* xspec_save, void* irspec_save,
                             void* workspace, int64_t workspace_bytes, int64_t bs, int64_t n, int64_t ir_len,
                             int64_t inputs, int64_t outputs, int64_t chunk_items, void* stream);
int dasp_conv_bus_shared_bwd(const float* gy, const void* xspec_save, const void* irspec_save, float* gx,
                             float* gir /* may be NULL */, void* workspace, int64_t workspace_bytes, int64_t bs,
                             int64_t n, int64_t ir_len, int64_t inputs, int64_t outputs, int64_t chunk_items,
                             void* stream);
/* ---- multichannel_convolution: S input rows through an S x M impulse-response matrix into M output rows -----------
 * The bus with 1 <= M <= DASP_CONV_MC_MAX_OUTPUTS outputs (microphone arrays, ambisonics, multichannel beds):
 *   y[b, m] = sum_s (x[b, s] * ir[b, s, m])[:n]
 * The arguments, shapes, rules and rejections are dasp_conv_bus_*'s with outputs = M.  The IR rows s M + m are packed two
 * per partition set (ceil(S M / 2) sets), the outputs and their gradients two per transform (ceil(M / 2) spectra per
 * block), so xspec_c64 and irspec_c64 come from dasp_conv_mc_geometry, which needs no GPU.  M <= 2 gives the bits of
 * dasp_conv_bus_*. */
#define DASP_CONV_MC_MAX_OUTPUTS 32
int dasp_conv_mc_geometry(int64_t bs, int64_t n, int64_t ir_len, int64_t inputs, int64_t outputs, int64_t shared,
                          int64_t chunk_items, dasp_conv_geom* out);
int dasp_conv_mc_fwd(const float* x, const float* ir, float* y, void* xspec_save, void* irspec_save, void* workspace,
                     int64_t workspace_bytes, int64_t bs, int64_t n, int64_t ir_len, int64_t inputs, int64_t outputs,
                     int64_t chunk_items, void* stream);
int dasp_conv_mc_bwd(const float* gy, const void* xspec_save, const void* irspec_save, float* gx,
                     float* gir /* may be NULL */, void* workspace, int64_t workspace_bytes, int64_t bs, int64_t n,
                     int64_t ir_len, int64_t inputs, int64_t outputs, int64_t chunk_items, void* stream);
int dasp_conv_mc_shared_fwd(const float* x, const float* ir, float* y, void* xspec_save, void* irspec_save,
                            void* workspace, int64_t workspace_bytes, int64_t bs, int64_t n, int64_t ir_len,
                            int64_t inputs, int64_t outputs, int64_t chunk_items, void* stream);
int dasp_conv_mc_shared_bwd(const float* gy, const void* xspec_save, const void* irspec_save, float* gx,
                            float* gir /* may be NULL */, void* workspace, int64_t workspace_bytes, int64_t bs,
                            int64_t n, int64_t ir_len, int64_t inputs, int64_t outputs, int64_t chunk_items,
                            void* stream);

/* test hook: dispatch of the most recent dasp_conv_bus_* or dasp_conv_mc_* call.  which = 0 (forward): bit 0 = own
   in-shared-memory FFT (always), bit 1 = shared IR, bit 2 = register-cached products, bit 3 = M >= 3 outputs
   (dasp_conv_mc_*).  which = 1 (backward): bit 0 = own FFT (always), bit 1 = register-cached products, bit 2 = dL/dIR
   computed, bit 3 = shared IR, bit 4 = M >= 3 outputs */
int dasp_debug_conv_bus_last_path(int which);

/* ---- time_varying_convolution_reverberation: a trajectory of K impulse responses crossfaded along the output -------
 * x is (bs, in_chs, n) with in_chs 1 or 2, ir is (bs, K, ir_chs, ir_len) with ir_chs 1 or 2 (or ONE (K, ir_chs, ir_len)
 * trajectory for the whole batch: the *_shared_* entry points), mix has bs elements, y is (bs, 2, n).  IR k belongs to
 * the anchor time k hop, hop a positive multiple of conv_block (4096) with (K - 1) hop < n:
 *   wet(t) = sum_k w_k(t) (x * h_k)(t),  y = (1 - mix) x + mix wet  (* as convolution_reverberation's wet signal)
 *   k hop <= t < (k+1) hop, k < K - 1:  a = (t - k hop) / hop,  w_k = 1 - a,  w_k+1 = a;   t >= (K-1) hop:  w_K-1 = 1
 * A mono x or IR is used for both channels.  The audio windows are transformed once per block, as for one static IR;
 * a block between two anchors takes the products of its two IRs, each packed with its other channel or its
 * neighbour so that one inverse transform carries two real rows.  n % 4 == 0 and 16-byte aligned x / gy rows are
 * required.  Buffers kept for the backward (NULL for both when no backward follows): xspec_save geom.xspec_c64 and
 * irspec_save geom.irspec_c64 complex64.  Backward: gx (bs, in_chs, n), gmix (bs,), gir (bs, K, ir_chs, ir_len)
 * (shared: (K, ir_chs, ir_len), the sum over the items in fp64 in item order, the same bits for every chunk_items), or
 * NULL, which skips all dL/dIR work; a mono IR receives the sum of both channel gradients; taps >= leff =
 * min(ir_len, n) get 0.  Workspace sizes come from dasp_tvconv_geometry (shared != 0 for the shared entry points),
 * which needs no GPU.  Bad K, hop, channel counts or shapes are rejected before any CUDA call. */
int dasp_tvconv_geometry(int64_t bs, int64_t n, int64_t ir_len, int64_t K, int64_t ir_chs, int64_t hop, int64_t shared,
                         int64_t chunk_items, dasp_conv_geom* out);
int dasp_tvconv_fwd(const float* x, int64_t in_chs, const float* ir, int64_t ir_chs, int64_t ir_len, int64_t K,
                    int64_t hop, const float* mix, float* y, void* xspec_save, void* irspec_save, void* workspace,
                    int64_t workspace_bytes, int64_t bs, int64_t n, int64_t chunk_items, void* stream);
int dasp_tvconv_bwd(const float* gy, const float* x, int64_t in_chs, int64_t ir_chs, int64_t ir_len, int64_t K,
                    int64_t hop, const float* mix, const void* xspec_save, const void* irspec_save, float* gx,
                    float* gir /* may be NULL */, float* gmix, void* workspace, int64_t workspace_bytes, int64_t bs,
                    int64_t n, int64_t chunk_items, void* stream);
int dasp_tvconv_shared_fwd(const float* x, int64_t in_chs, const float* ir, int64_t ir_chs, int64_t ir_len, int64_t K,
                           int64_t hop, const float* mix, float* y, void* xspec_save, void* irspec_save,
                           void* workspace, int64_t workspace_bytes, int64_t bs, int64_t n, int64_t chunk_items,
                           void* stream);
int dasp_tvconv_shared_bwd(const float* gy, const float* x, int64_t in_chs, int64_t ir_chs, int64_t ir_len, int64_t K,
                           int64_t hop, const float* mix, const void* xspec_save, const void* irspec_save, float* gx,
                           float* gir /* may be NULL */, float* gmix, void* workspace, int64_t workspace_bytes,
                           int64_t bs, int64_t n, int64_t chunk_items, void* stream);
/* test hook: dispatch of the most recent call.  which = 0 (forward): bit 0 = own in-shared-memory FFT (always),
   bit 1 = shared trajectory, bit 2 = crossfaded blocks (K > 1).  which = 1 (backward): bit 0 = own FFT (always),
   bit 1 = crossfaded blocks, bit 2 = dL/dIR computed, bit 3 = shared trajectory */
int dasp_debug_tvconv_last_path(int which);

/* ---- time_varying_convolution_bus: S moving sources, each with its own IR trajectory, summed into one bus ----------
 * x is (bs, inputs, n) with 1 <= inputs (S) <= DASP_CONV_BUS_MAX_INPUTS, ir is (bs, K, S, outputs, ir_len) with outputs
 * (O) 1 or 2 (or ONE (K, S, O, ir_len) trajectory set for the whole batch: the *_shared_* entry points), y is
 * (bs, O, n).  ir[:, k] is a complete convolution_bus IR set, the scene at the anchor time k hop; hop is a positive
 * multiple of conv_block (4096) with (K - 1) hop < n:
 *   y[:, o](t) = sum_k w_k(t) sum_s (x[:, s] * h[:, k, s, o])(t)   (* and w_k as in dasp_tvconv_*; no dry/wet mix)
 * The rows of every signal are packed two per transform as for the bus: ceil(S / 2) window transforms per block, one
 * product per IR set and block summed over the sources, and one inverse transform per output row and crossfaded block
 * (a stereo bus) or per block (a mono bus).  n % 4 == 0 and 16-byte aligned x / gy rows are required.  Buffers kept for
 * the backward (NULL for both when no backward follows): xspec_save geom.xspec_c64 and irspec_save geom.irspec_c64
 * complex64.  Backward: gx (bs, S, n), gir (bs, K, S, O, ir_len) (shared: (K, S, O, ir_len), the sum over the items in
 * fp64 in item order, the same bits for every chunk_items), or NULL, which skips all dL/dIR work; taps >= leff =
 * min(ir_len, n) get 0.  Workspace sizes come from dasp_tvbus_geometry (shared != 0 for the shared entry points), which
 * needs no GPU.  Bad S, O, K, hop or shapes, null pointers and unaligned rows are rejected before any CUDA call. */
int dasp_tvbus_geometry(int64_t bs, int64_t n, int64_t ir_len, int64_t K, int64_t inputs, int64_t outputs, int64_t hop,
                        int64_t shared, int64_t chunk_items, dasp_conv_geom* out);
int dasp_tvbus_fwd(const float* x, const float* ir, float* y, void* xspec_save, void* irspec_save, void* workspace,
                   int64_t workspace_bytes, int64_t bs, int64_t n, int64_t ir_len, int64_t K, int64_t inputs,
                   int64_t outputs, int64_t hop, int64_t chunk_items, void* stream);
int dasp_tvbus_bwd(const float* gy, const void* xspec_save, const void* irspec_save, float* gx,
                   float* gir /* may be NULL */, void* workspace, int64_t workspace_bytes, int64_t bs, int64_t n,
                   int64_t ir_len, int64_t K, int64_t inputs, int64_t outputs, int64_t hop, int64_t chunk_items,
                   void* stream);
int dasp_tvbus_shared_fwd(const float* x, const float* ir, float* y, void* xspec_save, void* irspec_save,
                          void* workspace, int64_t workspace_bytes, int64_t bs, int64_t n, int64_t ir_len, int64_t K,
                          int64_t inputs, int64_t outputs, int64_t hop, int64_t chunk_items, void* stream);
int dasp_tvbus_shared_bwd(const float* gy, const void* xspec_save, const void* irspec_save, float* gx,
                          float* gir /* may be NULL */, void* workspace, int64_t workspace_bytes, int64_t bs, int64_t n,
                          int64_t ir_len, int64_t K, int64_t inputs, int64_t outputs, int64_t hop, int64_t chunk_items,
                          void* stream);
/* ---- the same bus with a source-side crossfade: every emitted sample keeps the IR set of its emission time --------
 *   y[:, o](t) = sum_k sum_s ((w_k x[:, s]) * h[:, k, s, o])(t)
 * The arguments, shapes, rules and rejections are dasp_tvbus_*'s.  The window spectra are zero-padded transforms of
 * each source's weighted blocks: S per crossfaded block ((K - 1) hop / conv_block blocks), ceil(S / 2) per later block,
 * so geom.xspec_c64 comes from dasp_tvbus_in_geometry; one product and one inverse transform per output block. */
int dasp_tvbus_in_geometry(int64_t bs, int64_t n, int64_t ir_len, int64_t K, int64_t inputs, int64_t outputs,
                           int64_t hop, int64_t shared, int64_t chunk_items, dasp_conv_geom* out);
int dasp_tvbus_in_fwd(const float* x, const float* ir, float* y, void* xspec_save, void* irspec_save, void* workspace,
                      int64_t workspace_bytes, int64_t bs, int64_t n, int64_t ir_len, int64_t K, int64_t inputs,
                      int64_t outputs, int64_t hop, int64_t chunk_items, void* stream);
int dasp_tvbus_in_bwd(const float* gy, const void* xspec_save, const void* irspec_save, float* gx,
                      float* gir /* may be NULL */, void* workspace, int64_t workspace_bytes, int64_t bs, int64_t n,
                      int64_t ir_len, int64_t K, int64_t inputs, int64_t outputs, int64_t hop, int64_t chunk_items,
                      void* stream);
int dasp_tvbus_in_shared_fwd(const float* x, const float* ir, float* y, void* xspec_save, void* irspec_save,
                             void* workspace, int64_t workspace_bytes, int64_t bs, int64_t n, int64_t ir_len,
                             int64_t K, int64_t inputs, int64_t outputs, int64_t hop, int64_t chunk_items,
                             void* stream);
int dasp_tvbus_in_shared_bwd(const float* gy, const void* xspec_save, const void* irspec_save, float* gx,
                             float* gir /* may be NULL */, void* workspace, int64_t workspace_bytes, int64_t bs,
                             int64_t n, int64_t ir_len, int64_t K, int64_t inputs, int64_t outputs, int64_t hop,
                             int64_t chunk_items, void* stream);
/* ---- time_varying_multichannel_convolution: the time-varying bus with up to 32 outputs ----------------------------
 * dasp_tvbus_* and dasp_tvbus_in_* with 1 <= outputs (M) <= DASP_CONV_MC_MAX_OUTPUTS (moving talkers recorded by a
 * microphone array, ambisonic scenes and multichannel beds with moving objects):
 *   dasp_tvmc_*:     y[:, m](t) = sum_k w_k(t) sum_s (x[:, s] * h[:, k, s, m])(t)
 *   dasp_tvmc_in_*:  y[:, m](t) = sum_k sum_s ((w_k x[:, s]) * h[:, k, s, m])(t)
 * The arguments, shapes, rules and rejections are dasp_tvbus_*'s with outputs = M; at most 65535 partition sets
 * ceil(K S M / 2) per trajectory set (K <= 127 at S = M = 32).  M <= 2 gives the bits of dasp_tvbus_* /
 * dasp_tvbus_in_*.  With nX = (K - 1) hop / conv_block crossfaded blocks, I = ceil(n / conv_block) blocks,
 * J = ceil(min(ir_len, n) / conv_block) partitions, P = ceil(S / 2) and Q = ceil(M / 2), per item:
 *   dasp_tvmc_*:     xspec_c64 = P I 8192, product / gradient slots U = M nX + Q (I - nX)
 *   dasp_tvmc_in_*:  xspec_c64 = (S nX + P (I - nX)) 8192, product / gradient spectra Q I
 *   both:            irspec_c64 = ceil(K S M / 2) J 8192 (one trajectory set for the shared entry points)
 * The geometry queries return these sizes and the workspaces and need no GPU. */
int dasp_tvmc_geometry(int64_t bs, int64_t n, int64_t ir_len, int64_t K, int64_t inputs, int64_t outputs, int64_t hop,
                       int64_t shared, int64_t chunk_items, dasp_conv_geom* out);
int dasp_tvmc_fwd(const float* x, const float* ir, float* y, void* xspec_save, void* irspec_save, void* workspace,
                  int64_t workspace_bytes, int64_t bs, int64_t n, int64_t ir_len, int64_t K, int64_t inputs,
                  int64_t outputs, int64_t hop, int64_t chunk_items, void* stream);
int dasp_tvmc_bwd(const float* gy, const void* xspec_save, const void* irspec_save, float* gx,
                  float* gir /* may be NULL */, void* workspace, int64_t workspace_bytes, int64_t bs, int64_t n,
                  int64_t ir_len, int64_t K, int64_t inputs, int64_t outputs, int64_t hop, int64_t chunk_items,
                  void* stream);
int dasp_tvmc_shared_fwd(const float* x, const float* ir, float* y, void* xspec_save, void* irspec_save,
                         void* workspace, int64_t workspace_bytes, int64_t bs, int64_t n, int64_t ir_len, int64_t K,
                         int64_t inputs, int64_t outputs, int64_t hop, int64_t chunk_items, void* stream);
int dasp_tvmc_shared_bwd(const float* gy, const void* xspec_save, const void* irspec_save, float* gx,
                         float* gir /* may be NULL */, void* workspace, int64_t workspace_bytes, int64_t bs, int64_t n,
                         int64_t ir_len, int64_t K, int64_t inputs, int64_t outputs, int64_t hop, int64_t chunk_items,
                         void* stream);
int dasp_tvmc_in_geometry(int64_t bs, int64_t n, int64_t ir_len, int64_t K, int64_t inputs, int64_t outputs,
                          int64_t hop, int64_t shared, int64_t chunk_items, dasp_conv_geom* out);
int dasp_tvmc_in_fwd(const float* x, const float* ir, float* y, void* xspec_save, void* irspec_save, void* workspace,
                     int64_t workspace_bytes, int64_t bs, int64_t n, int64_t ir_len, int64_t K, int64_t inputs,
                     int64_t outputs, int64_t hop, int64_t chunk_items, void* stream);
int dasp_tvmc_in_bwd(const float* gy, const void* xspec_save, const void* irspec_save, float* gx,
                     float* gir /* may be NULL */, void* workspace, int64_t workspace_bytes, int64_t bs, int64_t n,
                     int64_t ir_len, int64_t K, int64_t inputs, int64_t outputs, int64_t hop, int64_t chunk_items,
                     void* stream);
int dasp_tvmc_in_shared_fwd(const float* x, const float* ir, float* y, void* xspec_save, void* irspec_save,
                            void* workspace, int64_t workspace_bytes, int64_t bs, int64_t n, int64_t ir_len, int64_t K,
                            int64_t inputs, int64_t outputs, int64_t hop, int64_t chunk_items, void* stream);
int dasp_tvmc_in_shared_bwd(const float* gy, const void* xspec_save, const void* irspec_save, float* gx,
                            float* gir /* may be NULL */, void* workspace, int64_t workspace_bytes, int64_t bs,
                            int64_t n, int64_t ir_len, int64_t K, int64_t inputs, int64_t outputs, int64_t hop,
                            int64_t chunk_items, void* stream);

/* test hook: dispatch of the most recent dasp_tvbus_*, dasp_tvbus_in_*, dasp_tvmc_* or dasp_tvmc_in_* call.  which = 0
   (forward): bit 0 = own in-shared-memory FFT (always), bit 1 = shared trajectory set, bit 2 = crossfaded blocks
   (K > 1), bit 3 = source-side crossfade (dasp_tvbus_in_*, dasp_tvmc_in_*), bit 4 = M >= 3 outputs.  which = 1
   (backward): bit 0 = own FFT (always), bit 1 = crossfaded blocks, bit 2 = dL/dIR computed, bit 3 = shared trajectory
   set, bit 4 = source-side crossfade, bit 5 = M >= 3 outputs */
int dasp_debug_tvbus_last_path(int which);

#ifdef __cplusplus
}
#endif
#endif /* DASP_B200_H_ */
