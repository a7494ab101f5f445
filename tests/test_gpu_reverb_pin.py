"""The device-noise reverb pinned to the fp64 oracle on every path it dispatches to, and the statistics of its noise.

Each pin (tests/reverb_pin.py) reads the white noise of the call back under the unit-impulse filter-bank hook, rebuilds
the reference-style noise tensor from it and requires y, dL/dx and all 25 parameter gradients of the DEFAULT call with
the same seed to equal oracle.noise_shaped_reverberation(noise=...) in fp64, per item, to 1e-4 (or the reference's own
fp32 error where that is larger, SURVEY.md 8c).  Because the pins take the noise from the GPU itself, the generator's
statistics are checked separately: a stream reused across items, bands, channels or chunks would pass every pin."""
import numpy as np
import pytest
import torch

import reverb_pin as rp
from helpers import SR

pytestmark = pytest.mark.gpu
TAPS = 1023


def _params01(bs, seed):
    g = torch.Generator().manual_seed(seed)
    p = torch.rand(bs, 25, generator=g)
    return [p[:, i].clone() for i in range(25)]


def _audio(bs, chs, n, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(bs, chs, n, generator=g) * 2 - 1


def _corner(kind, bs):
    p = _params01(bs, 61)
    if kind == "gains0":
        for k in range(12):
            p[k] = torch.zeros(bs)
    elif kind == "decay0_1":                                     # item 0: every decay 0, item 1: every decay 1
        for k in range(12, 24):
            p[k] = torch.tensor([0.0, 1.0])
    elif kind == "mix0_1":                                       # item 0: dry only (IR gradients vanish), item 1: wet only
        p[24] = torch.tensor([0.0, 1.0])
    return p


# (id, n, L, taps, path hook, expected last path, polyphase factor, bs, channels, parameter corner)
#   path hook: 0 automatic, 1 generator -> cuFFT -> shape_ir_pp_kernel, 2 cluster kernel
#   last path: 2 generator + ifft_shape_kernel, 1 cluster kernel, 0 cuFFT / overlap-save
CASES = (
    [(f"default-R{R}", *rp.default_case(R), TAPS, 0, 2, R, 2, 2, None) for R in range(1, 17)]
    + [(f"cluster-R{R}", *rp.default_case(R), TAPS, 2, 1, R, 2, 2, None) for R in range(1, 9)]
    + [(f"cufft-R{R}", *rp.default_case(R), TAPS, 1, 0, R, 2, 2, None) for R in (2, 4, 7, 8)]
    + [("taps2047-R1", 12000, 14001, 2047, 0, 0, 1, 2, 2, None),             # nb = 16384
       ("taps2047-R3", 44000, 44000, 2047, 0, 0, 3, 2, 2, None),
       ("taps4095-R1", 26000, 24000, 4095, 0, 0, 1, 2, 2, None),             # nb = 32768
       ("n-odd", 30001, 20000, TAPS, 0, 2, 3, 2, 2, None),                   # cuFFT convolution + ir_grad_pp_kernel
       ("mono", 20000, 26000, TAPS, 0, 2, 3, 2, 1, None),
       ("time-domain-R17", 132000, 132000, TAPS, 0, 0, 17, 1, 2, None),      # Philox overlap-save fallback
       # the four cases of the first pinned test
       ("legacy-6000-4000-255", 6000, 4000, 255, 0, 2, 1, 2, 2, None),
       ("legacy-48000-48000", 48000, 48000, TAPS, 0, 2, 6, 2, 2, None),
       ("legacy-48000-96000", 48000, 96000, TAPS, 0, 2, 6, 2, 2, None),
       ("legacy-70000-66000", 70000, 66000, TAPS, 0, 2, 9, 2, 2, None)]
    + [(f"corner-{kind}", *rp.default_case(6), TAPS, 0, 2, 6, 2, 2, kind) for kind in ("gains0", "decay0_1", "mix0_1")]
)


@pytest.mark.parametrize("case,n,L,taps,path,expect,R,bs,chs,corner", CASES, ids=[c[0] for c in CASES])
def test_reverb_device_noise_pinned_to_oracle(cuda_device, case, n, L, taps, path, expect, R, bs, chs, corner):
    x = _audio(bs, chs, n, seed=n + L + chs)
    params = _params01(bs, 5 + R) if corner is None else _corner(corner, bs)
    geom, seqs, errs = rp.pin(cuda_device, x, params, L, taps, seed=1000 + R, path=path, expect_path=expect)
    assert geom.rpp == R, (geom.rpp, R)
    assert rp.polyphase(geom) == (R <= rp.MAX_SPECTRAL_R)
    if taps == 2047:
        assert geom.nb == 16384
    elif taps == 4095:
        assert geom.nb == 32768
    else:
        assert geom.nb == 8192
    # the sequences are unit-variance white noise (the full checks are below): a flat filter bank really was used
    s = torch.stack(list(seqs.values()))
    assert abs(float(s.real.std()) - 1.0) < 0.02 and abs(float(s.imag.std()) - 1.0) < 0.02
    print(f"PIN {case}: y {errs['y'].max():.2e} dx {errs['dx'].max():.2e} dparams {errs['dp'].max():.2e}")


# spectral generator at R = 1, 6, 9, 16 and the time-domain generator (R = 17); four items in chunks of two
STAT_CASES = [(f"spectral-R{R}", *rp.default_case(R)) for R in (1, 6, 9, 16)] + [("time-domain-R17", 132000, 132000)]


@pytest.mark.parametrize("case,n,L", STAT_CASES, ids=[c[0] for c in STAT_CASES])
def test_reverb_noise_statistics(cuda_device, case, n, L):
    """per (item, band, channel): N(0, 1) marginals; together: a flat periodogram; pairwise: no correlation at any lag
    between the channels of a band, neighbouring bands, neighbouring items, the items on either side of a chunk
    boundary, item 0 and the first item of every chunk, and one item under two seeds"""
    bs, chunk = 4, 2
    x = torch.zeros(bs, 2, n, device=cuda_device)
    p = [q.to(cuda_device) for q in _params01(bs, 9)]
    geom, _, seqs = rp.white_sequences(x, p, L, TAPS, seed=21, chunk=chunk)
    _, _, other = rp.white_sequences(x, p, L, TAPS, seed=22, chunk=chunk)
    assert rp.polyphase(geom) == case.startswith("spectral")
    rows = np.concatenate([rp.channel_rows(seqs[i]) for i in range(bs)])
    rp.check_marginals(rows)
    rp.check_white(rows)
    pairs = rp.independence_pairs(seqs, chunk)
    pairs += [(f"item {i} band {k} {c} seeds 21/22", getattr(seqs[i][k].numpy(), c), getattr(other[i][k].numpy(), c))
              for i in range(bs) for k in range(12) for c in ("real", "imag")]
    peak = rp.check_independent(pairs, rows.shape[1])
    print(f"STATS {case}: {rows.shape[0]} rows x {rows.shape[1]}, {len(pairs)} pairs, largest |xcorr| {peak:.2f}/sqrt(n)")


@pytest.mark.parametrize("case,n,L,big", [("spectral-R6", *rp.default_case(6), 300),
                                          ("time-domain-R17", 132000, 132000, 10)])
def test_reverb_noise_keyed_by_item(cuda_device, case, n, L, big):
    """item i's noise is the same whatever the batch size and the chunk size: the Philox counter is keyed by the
    global item index.  The spectral generator's sequences are compared bit for bit; the time-domain blocks pass through
    a batched cuFFT round trip, whose kernel may depend on the batch size, so they are compared to its rounding."""
    from dasp_pytorch_b200 import functional as F
    auto = F.reverb_chunk_items(cuda_device)
    runs = {}
    for bs, chunk in ((3, None), (3, 1), (big, None), (big, 7)):
        x = torch.zeros(bs, 2, n, device=cuda_device)
        p = [q.to(cuda_device) for q in _params01(bs, 4)]
        keep = [0, 1, 2] if bs == 3 else sorted({0, 1, 2, 6, 7, bs - 1} | {i for i in (auto - 1, auto) if i < bs})
        runs[(bs, chunk)] = rp.white_sequences(x, p, L, TAPS, seed=31, chunk=chunk, items=keep)[2]
    ref = runs[(3, None)]
    for key, got in runs.items():
        for i, s in got.items():
            want = ref[i] if i in ref else runs[(big, None)][i]
            if case.startswith("spectral"):
                assert torch.equal(s, want), (case, key, i)
            else:
                assert float((s - want).abs().max()) < rp.OS_ROUNDING, (case, key, i)


def test_reverb_benchmark_batch_pinned(cuda_device):
    """bench.py's batch (1024 x 2 x 48000, IR 96000, 1023 taps) with the automatic chunk: the default forward and
    backward of the whole batch, pinned to the oracle on item 0, both sides of every chunk boundary, the last item
    and two random ones, whose noise must also be independent of each other's"""
    from dasp_pytorch_b200 import functional as F
    bs, n, L = 1024, 48000, 96000
    chunk = F.reverb_chunk_items(cuda_device)
    g = torch.Generator().manual_seed(1024)
    items = {0, bs - 1} | {i for c in range(chunk, bs, chunk) for i in (c - 1, c)}
    items |= set(torch.randint(1, bs - 1, (2,), generator=g).tolist())
    x = _audio(bs, 2, n, seed=77)
    params = _params01(bs, 78)
    geom, seqs, errs = rp.pin(cuda_device, x, params, L, TAPS, seed=2024, items=sorted(items), expect_path=2)
    assert (geom.chunk_items, geom.rpp, geom.nbk) == (chunk, 6, 7)
    rp.check_marginals(np.concatenate([rp.channel_rows(s) for s in seqs.values()]))
    pairs = rp.independence_pairs(seqs, chunk)
    peak = rp.check_independent(pairs, geom.rpp * geom.nb)
    print(f"PIN bench batch (chunk {chunk}, items {sorted(items)}): y {errs['y'].max():.2e} dx {errs['dx'].max():.2e} "
          f"dparams {errs['dp'].max():.2e}; {len(pairs)} pairs, largest |xcorr| {peak:.2f}/sqrt(n)")
