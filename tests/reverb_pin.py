"""Pin the device-noise reverb to the fp64 oracle.

The default reverb draws its noise on the device, so the oracle cannot be handed the same noise directly.  The test
hook ``dasp_debug_reverb_flat_filterbank`` makes every band filter a unit impulse, and then the band-filtered noise the
forward keeps for the backward (``f_save``) is the white noise itself, in one of two layouts:

* polyphase (spectral generator, polyphase factor R = rpp <= 16): per (item, band) R blocks of nb complex samples,
  block b element a = w[R a + b] of the periodic white sequence w of length n1 = R nb (real = left, imag = right).
  The forward filters it circularly, f[t] = sum_m h[m] w[(t - m) mod n1], so the reference-style noise tensor
  noise[s] = w[(s - P) mod n1] (P = taps - 1, symmetric FIRs) makes the reference's valid correlation produce the same
  f for every t < leff.
* overlap-save (time-domain Philox generator, R > 16): per (item, band) nbk blocks of nb samples, block b element m =
  noise[b hop + m]; the blocks overlap by nb - hop samples and the forward's f[t] is the reference's correlation of
  exactly that noise.

In both layouts the chunk of items c starts at complex offset  c * chunk * 12 * pair_c64,  pair_c64 = max(nbk, R) nb,
while inside a chunk an (item, band) pair takes R nb (polyphase) or nbk nb (overlap-save) samples.

Everything except ``white_sequences`` / ``pin`` runs on the CPU (tests/test_reverb_pin_host.py checks the algebra).
"""
import math
from types import SimpleNamespace

import numpy as np
import torch

import oracle
from helpers import SR, param_grad_err, peak_err

TOL = 1e-4                  # SURVEY.md 8c: max(1e-4, error of the reference's own fp32 run)
MAX_SPECTRAL_R = 16         # polyphase factors the spectral generator is instantiated for
OS_ROUNDING = 1e-4          # overlap-save layout: N(0, 1) samples after an fp32 FFT round trip of nb points


def default_case(R):
    """(n, L) whose device-noise call at 1023 taps has polyphase factor R (1 <= R <= 16, nb = 8192).  R % 3 picks
    L = N, L < N or L > N; n % 4 == 0, so the own-FFT convolution runs; the audio block count ceil(n / 4096) grows
    with R through the <= 12, <= 16 and > 16 instantiations of the partition multiply-accumulate."""
    leff = R * 8192 - 1024 - 256 * (R % 4)
    if R % 3 == 0:
        return leff, leff
    if R % 3 == 1:
        return leff + 4000, leff
    return leff, leff + 3001


def geometry(bs, n, L, taps, chunk):
    """dasp_reverb_geometry as a namespace (nb, hop, nbk, leff, rpp, chunk_items, x_blocks, ...).  bs = 0 needs no GPU."""
    from dasp_pytorch_b200 import _abi
    g = _abi.ReverbGeom()
    _abi.check(_abi.lib().dasp_reverb_geometry(bs, n, L, taps, chunk, g), "dasp_reverb_geometry")
    return SimpleNamespace(**{name: int(getattr(g, name)) for name, _ in _abi.ReverbGeom._fields_})


def polyphase(geom):
    """True when the device-noise forward leaves the spectral generator's polyphase layout in f_save."""
    return geom.rpp <= MAX_SPECTRAL_R


def pair_c64(geom):
    return max(geom.nbk, geom.rpp) * geom.nb


def item_blocks(fsave, item, geom):
    """The 12 band blocks of one item in f_save (flat float32 tensor), as a (12, blocks, nb) complex tensor:
    blocks = rpp (polyphase) or nbk (overlap-save)."""
    blocks = geom.rpp if polyphase(geom) else geom.nbk
    c, il = divmod(item, geom.chunk_items)
    start = c * geom.chunk_items * 12 * pair_c64(geom) + il * 12 * blocks * geom.nb       # complex samples
    flat = fsave[2 * start: 2 * (start + 12 * blocks * geom.nb)]
    return torch.view_as_complex(flat.reshape(12, blocks, geom.nb, 2).contiguous())


def unpack(blocks, geom):
    """(12, blocks, nb) complex -> (12, length) complex white sequences (real = left, imag = right).
    polyphase: w of length n1 = R nb; overlap-save: noise[0 : (nbk - 1) hop + nb], after checking that the samples
    the overlapping blocks share agree (the generator addresses them by absolute position; the blocks then pass
    through a forward and an inverse transform even with unit-impulse filters, so they agree to OS_ROUNDING)."""
    if polyphase(geom):
        return blocks.permute(0, 2, 1).reshape(blocks.shape[0], -1)          # [k, b, a] -> w[R a + b]
    hop, nb = geom.hop, geom.nb
    gap = (blocks[:, 1:, : nb - hop] - blocks[:, :-1, hop:]).abs().max() if blocks.shape[1] > 1 else 0.0
    assert float(gap) < OS_ROUNDING, ("overlapping blocks disagree", float(gap))
    return torch.cat([blocks[:, :-1, :hop].reshape(blocks.shape[0], -1), blocks[:, -1]], dim=1)


def reference_noise(seqs, geom, L, taps):
    """(items, 12, length) complex white sequences -> the (items*2, 12, L + P) float64 tensor the reference draws."""
    P = taps - 1
    items, length = seqs.shape[0], seqs.shape[-1]
    if polyphase(geom):
        idx = (torch.arange(L + P) - P) % length
        s = seqs[:, :, idx]
    else:
        assert length >= geom.leff + P, (length, geom.leff, P)
        s = torch.zeros(items, 12, L + P, dtype=seqs.dtype)                  # samples >= leff + P never reach y
        m = min(length, L + P)
        s[:, :, :m] = seqs[:, :, :m]
    return torch.stack([s.real, s.imag], 1).reshape(items * 2, 12, L + P).double()


def white_sequences(x, params, L, taps, seed, path=0, chunk=None, items=None):
    """Run the device-noise forward once with unit-impulse filters (x, params on the GPU) and return
    (geometry, last path, {item: (12, length) complex sequence on the CPU}) for `items` (default: all)."""
    import dasp_pytorch_b200 as D
    from dasp_pytorch_b200 import _abi, functional as F
    lib = _abi.lib()
    bs, _, n = x.shape
    old_chunk = F.REVERB_CHUNK_ITEMS
    if chunk is not None:
        F.REVERB_CHUNK_ITEMS = chunk
    lib.dasp_debug_reverb_path(path)
    lib.dasp_debug_reverb_flat_filterbank(1)
    try:
        torch.manual_seed(seed)
        xq = x.detach().clone().requires_grad_(True)
        y = D.noise_shaped_reverberation(xq, SR, *params, num_samples=L, num_bandpass_taps=taps)
        used = lib.dasp_debug_reverb_last_path()
        geom = geometry(bs, n, L, taps, F.reverb_chunk_items(x.device))
        fsave = y.grad_fn.saved_tensors[3]
        assert fsave.numel() == bs * 12 * pair_c64(geom) * 2
        out = {i: unpack(item_blocks(fsave, i, geom), geom).cpu() for i in (range(bs) if items is None else items)}
    finally:
        lib.dasp_debug_reverb_flat_filterbank(0)
        lib.dasp_debug_reverb_path(0)
        F.REVERB_CHUNK_ITEMS = old_chunk
    return geom, used, out


def _grads(fn, x, params, dtype, device):
    """y, dx, [dparam] of loss = sum(y^2): per-item gradients that do not depend on the batch size."""
    xx = torch.as_tensor(x).to(device=device, dtype=dtype).clone().requires_grad_(True)
    pp = [torch.as_tensor(p).to(device=device, dtype=dtype).clone().requires_grad_(True) for p in params]
    y = fn(xx, pp)
    y.pow(2).sum().backward()
    return y.detach(), xx.grad.detach(), torch.stack([p.grad.detach() for p in pp], 1)


def pin(device, x, params, L, taps, seed, path=0, chunk=None, items=None, expect_path=None):
    """Pin one device-noise call against the fp64 oracle.

    x (bs, chs, n) and params (25 tensors of bs) on the CPU.  Runs the default call (test hook `path`, chunk size
    `chunk`) with torch.manual_seed(seed), and for `items` (default: all) compares y, dL/dx and the 25 parameter
    gradients with oracle.noise_shaped_reverberation fed the noise read back under the unit-impulse hook.  Returns
    (geometry, {item: white sequence}, {"y"|"dx"|"dp": per-item errors})."""
    import dasp_pytorch_b200 as D
    from dasp_pytorch_b200 import _abi, functional as F
    lib = _abi.lib()
    bs = x.shape[0]
    items = list(range(bs)) if items is None else list(items)
    xg = x.to(device)
    pg = [p.to(device) for p in params]
    geom, used_flat, seqs = white_sequences(xg, pg, L, taps, seed, path, chunk, items)
    if expect_path is not None:
        assert used_flat == expect_path, (used_flat, expect_path)
    noise = reference_noise(torch.stack([seqs[i] for i in items]), geom, L, taps)
    kw = dict(num_samples=L, num_bandpass_taps=taps)

    def run_default(xx, p):
        torch.manual_seed(seed)
        return D.noise_shaped_reverberation(xx, SR, *p, **kw)

    old_chunk = F.REVERB_CHUNK_ITEMS
    if chunk is not None:
        F.REVERB_CHUNK_ITEMS = chunk
    lib.dasp_debug_reverb_path(path)
    try:
        y, dx, dp = _grads(run_default, xg, pg, torch.float32, device)
        used = lib.dasp_debug_reverb_last_path()
    finally:
        lib.dasp_debug_reverb_path(0)
        F.REVERB_CHUNK_ITEMS = old_chunk
    assert used == used_flat, (used, used_flat)
    sel = torch.tensor(items)
    got = [t.index_select(0, sel.to(t.device)).cpu().double() for t in (y, dx, dp)]
    del y, dx, dp
    xs, ps = x[sel], [p[sel] for p in params]

    def run_oracle(dtype):
        return _grads(lambda xx, p: oracle.noise_shaped_reverberation(xx, SR, *p, noise=noise.to(dtype), method="fft", **kw),
                      xs, ps, dtype, "cpu")

    ref = run_oracle(torch.float64)
    errs = {"y": peak_err(got[0], ref[0]), "dx": peak_err(got[1], ref[1]),
            "dp": param_grad_err(list(got[2].T), list(ref[2].T))}
    if max(float(e.max()) for e in errs.values()) >= TOL:
        # the rule of SURVEY.md 8c: where the reference's own fp32 run is further off than 1e-4, that is the bound
        r32 = [t.double() for t in run_oracle(torch.float32)]
        bound = {"y": peak_err(r32[0], ref[0]), "dx": peak_err(r32[1], ref[1]),
                 "dp": param_grad_err(list(r32[2].T), list(ref[2].T))}
    else:
        bound = {k: torch.zeros_like(e) for k, e in errs.items()}
    for k, e in errs.items():
        lim = bound[k].clamp_min(TOL)
        assert bool((e < lim).all()), (k, items, e.tolist(), lim.tolist())
    return geom, seqs, errs


# ---------------------------------------------------------------------------------------------- statistics
# Bounds follow from the sample size: every statistic below is (asymptotically) normal or chi-square under the
# hypothesis "independent N(0, 1) samples", and each test allows a total false-alarm probability ALPHA over all the
# statistics it checks (Bonferroni), so a fixed seed passes by a wide margin unless the generator is wrong.
ALPHA = 1e-6


def _z(count, alpha=ALPHA):
    from scipy import stats
    return float(stats.norm.isf(alpha / (2 * count)))


def check_marginals(rows):
    """rows: (m, length) float64, each supposedly i.i.d. N(0, 1): mean, variance, excess kurtosis, Kolmogorov-Smirnov."""
    from scipy import stats
    m, n = rows.shape
    z = _z(4 * m)
    mean = rows.mean(1)
    var = rows.var(1)
    kurt = ((rows - mean[:, None]) ** 4).mean(1) / var ** 2 - 3.0
    assert np.abs(mean).max() < z / math.sqrt(n), np.abs(mean).max()
    assert np.abs(var - 1.0).max() < z * math.sqrt(2.0 / n), np.abs(var - 1.0).max()
    assert np.abs(kurt).max() < z * math.sqrt(24.0 / n), np.abs(kurt).max()
    pks = min(stats.kstest(r, "norm").pvalue for r in rows)
    assert pks > ALPHA / (4 * m), pks


def check_white(rows):
    """rows: (m, length) float64 i.i.d. N(0, 1) sequences.  Their DFT bins are then independent: |X_j|^2 / length is
    Exp(1) at 0 < j < length/2 and chi-square(1) at the real bins j = 0 and length/2 (same mean, twice the variance).
    The periodogram averaged over the m rows must lie inside those chi-square bounds bin by bin and, for a sharper
    test of the shape, averaged over 64 frequency bands."""
    from scipy import stats
    m, n = rows.shape
    pgram = (np.abs(np.fft.rfft(rows, axis=1)) ** 2 / n).mean(0)
    real_bins = [0] + ([n // 2] if n % 2 == 0 else [])
    inner = np.ones(pgram.shape[0], dtype=bool)
    inner[real_bins] = False
    groups = 64
    tests = inner.sum() + len(real_bins) + groups
    a = ALPHA / (2 * tests)
    lo, hi = stats.chi2.ppf(a, 2 * m) / (2 * m), stats.chi2.isf(a, 2 * m) / (2 * m)
    p = pgram[inner]
    assert lo < p.min() and p.max() < hi, (p.min(), p.max(), lo, hi)
    lo1, hi1 = stats.chi2.ppf(a, m) / m, stats.chi2.isf(a, m) / m
    for j in real_bins:
        assert lo1 < pgram[j] < hi1, (j, pgram[j], lo1, hi1)
    per = p.shape[0] // groups
    band = p[: per * groups].reshape(groups, per).mean(1)
    dof = 2 * m * per
    glo, ghi = stats.chi2.ppf(a, dof) / dof, stats.chi2.isf(a, dof) / dof
    assert glo < band.min() and band.max() < ghi, (band.min(), band.max(), glo, ghi)


def check_independent(pairs, length):
    """pairs: list of (label, a, b) float64 sequences of `length` samples, supposedly independent white N(0, 1).
    The circular cross-correlation at EVERY lag, sum_t a[t] b[(t + d) mod length] / length, is N(0, 1/length) for
    such a pair (so a copy, a shifted copy or a partial reuse of the other's stream shows up at its lag).
    Returns the largest |correlation| over all pairs and lags, in units of 1/sqrt(length)."""
    lag0, peak = [], []
    for s in range(0, len(pairs), 32):
        a = np.stack([p[1] for p in pairs[s: s + 32]])
        b = np.stack([p[2] for p in pairs[s: s + 32]])
        a = (a - a.mean(1, keepdims=True)) / a.std(1, keepdims=True)
        b = (b - b.mean(1, keepdims=True)) / b.std(1, keepdims=True)
        xc = np.fft.irfft(np.conj(np.fft.rfft(a, axis=1)) * np.fft.rfft(b, axis=1), n=length, axis=1) / length
        lag0.append(np.abs(xc[:, 0]))
        peak.append(np.abs(xc).max(1))
    lag0, peak = np.concatenate(lag0), np.concatenate(peak)
    b0 = _z(len(pairs)) / math.sqrt(length)                   # the plain correlation coefficient
    worst = int(lag0.argmax())
    assert lag0[worst] < b0, (pairs[worst][0], float(lag0[worst]), b0)
    bound = _z(len(pairs) * length) / math.sqrt(length)      # any lag
    worst = int(peak.argmax())
    assert peak[worst] < bound, (pairs[worst][0], float(peak[worst]), bound)
    return float(peak.max() * math.sqrt(length))


def channel_rows(seq):
    """(12, length) complex -> (24, length) float64 rows: band k left, band k right."""
    s = seq.numpy()
    return np.concatenate([s.real, s.imag]).astype(np.float64)


def independence_pairs(seqs, chunk):
    """The pairs whose independence the generator promises, for a dict {item: (12, length) complex}:
    left vs right of a band, neighbouring bands, neighbouring items, the last item of a chunk vs the first of the next,
    item 0 vs the first item of every chunk."""
    items = sorted(seqs)
    get = {i: seqs[i].numpy() for i in items}
    pairs = []
    for i in items:
        s = get[i]
        pairs += [(f"item {i} band {k} L/R", s[k].real, s[k].imag) for k in range(12)]
        pairs += [(f"item {i} bands {k},{k + 1} {c}", getattr(s[k], c), getattr(s[k + 1], c))
                  for k in range(11) for c in ("real", "imag")]
    firsts = [i for i in items if i % chunk == 0]
    cross = [(i, i + 1) for i in items if i + 1 in get]
    cross += [(i, j) for i in items for j in items if (j % chunk == 0 and i == j - 1)]
    cross += [(items[0], j) for j in firsts if j != items[0]]
    for i, j in sorted(set(cross)):
        pairs += [(f"items {i},{j} band {k} {c}", getattr(get[i][k], c), getattr(get[j][k], c))
                  for k in range(12) for c in ("real", "imag")]
    return pairs
