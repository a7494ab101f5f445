"""CPU checks of the index algebra behind the device-noise reverb pins (tests/reverb_pin.py), at a small block size:
read back from a synthetic f_save laid out like the kernels' (chunk stride max(nbk, R) nb, in-chunk stride R nb or nbk nb),
the rebuilt reference-style noise must make the reference's valid correlation equal to what the kernels compute, and
the statistical checks must accept white noise and reject the generator faults they exist to catch."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import reverb_pin as rp


def small_geometry(bs, n, L, taps, nb, chunk):
    """make_geom (csrc/reverb.cu) with a free block length nb"""
    P = taps - 1
    discard = ((P + 3) // 4) * 4
    hop = nb - discard
    leff = min(L, n)
    return SimpleNamespace(nb=nb, hop=hop, nbk=-(-leff // hop), leff=leff, rpp=-(-(leff + P) // nb),
                           chunk_items=min(chunk, bs))


def symmetric_bank(rng, taps):
    h = rng.standard_normal((12, taps))
    return h + h[:, ::-1]


def valid_correlation(noise, h):
    """the reference's conv1d (functional.py:551-556): f[t] = sum_j h[j] noise[t + j]"""
    taps = h.shape[-1]
    out = noise.shape[-1] - taps + 1
    return sum(h[..., j, None] * noise[..., j: j + out] for j in range(taps))


def fake_fsave(geom, bs, blocks_of):
    """f_save with the kernels' chunked layout; unused slots hold NaN so a wrong offset cannot go unnoticed"""
    pair = rp.pair_c64(geom)
    buf = np.full(bs * 12 * pair, np.nan + 1j * np.nan, dtype=np.complex64)
    per = (geom.rpp if rp.polyphase(geom) else geom.nbk) * geom.nb
    for i in range(bs):
        c, il = divmod(i, geom.chunk_items)
        start = c * geom.chunk_items * 12 * pair + il * 12 * per
        buf[start: start + 12 * per] = blocks_of(i).reshape(-1)
    return torch.view_as_real(torch.from_numpy(buf)).reshape(-1)


@pytest.mark.parametrize("R", range(1, 17))
@pytest.mark.parametrize("order", ["L<N", "L>N"])
def test_polyphase_index_algebra(R, order):
    """circular filtering of the periodic w (what the spectral generator computes) equals the reference's valid
    correlation of the noise rebuilt from f_save, for every t < leff"""
    rng = np.random.default_rng(R)
    nb, taps, bs, chunk = 64, 9, 5, 2
    P = taps - 1
    leff = R * nb - P - (R % 5)
    n, L = (leff + 7, leff) if order == "L<N" else (leff, leff + 11)
    g = small_geometry(bs, n, L, taps, nb, chunk)
    assert g.rpp == R and rp.polyphase(g)
    n1 = R * nb
    w = (rng.standard_normal((bs, 12, n1)) + 1j * rng.standard_normal((bs, 12, n1))).astype(np.complex64)
    # polyphase layout: block b, element a holds w[R a + b]
    fs = fake_fsave(g, bs, lambda i: w[i].reshape(12, nb, R).transpose(0, 2, 1))
    seqs = torch.stack([rp.unpack(rp.item_blocks(fs, i, g), g) for i in range(bs)])
    assert np.array_equal(seqs.numpy(), w)
    noise = rp.reference_noise(seqs, g, L, taps).numpy().reshape(bs, 2, 12, L + P)
    h = symmetric_bank(rng, taps)
    hpad = np.zeros((12, n1))
    hpad[:, :taps] = h
    wd = w.astype(np.complex128)
    circ = np.fft.ifft(np.fft.fft(wd, axis=-1) * np.fft.fft(hpad, axis=-1), axis=-1)      # sum_m h[m] w[(t-m) mod n1]
    ref = valid_correlation(noise, h)                                                     # (bs, 2, 12, L)
    np.testing.assert_allclose(ref[:, 0, :, :leff], circ.real[..., :leff], atol=1e-9)
    np.testing.assert_allclose(ref[:, 1, :, :leff], circ.imag[..., :leff], atol=1e-9)


@pytest.mark.parametrize("n,L", [(400, 300), (300, 520), (700, 700)])
def test_overlap_save_unpacking(n, L):
    """blocks C[b, m] = noise[b hop + m] (the time-domain generator under the unit-impulse hook) unpack to the noise;
    and the overlap-save filtering of those blocks, f[b hop + m] = (h circ C_b)[m + P], equals the reference's valid
    correlation of the rebuilt noise"""
    rng = np.random.default_rng(n + L)
    nb, taps, bs, chunk = 64, 15, 5, 3
    P = taps - 1
    g = small_geometry(bs, n, L, taps, nb, chunk)
    g.rpp = rp.MAX_SPECTRAL_R + 1                          # the layout the device path uses beyond R = 16
    assert not rp.polyphase(g)
    span = (g.nbk - 1) * g.hop + nb
    assert span >= g.leff + P
    src = (rng.standard_normal((bs, 12, span)) + 1j * rng.standard_normal((bs, 12, span))).astype(np.complex64)
    blocks = np.stack([src[:, :, b * g.hop: b * g.hop + nb] for b in range(g.nbk)], 2)   # (bs, 12, nbk, nb)
    fs = fake_fsave(g, bs, lambda i: blocks[i])
    seqs = torch.stack([rp.unpack(rp.item_blocks(fs, i, g), g) for i in range(bs)])
    assert np.array_equal(seqs.numpy(), src)
    noise = rp.reference_noise(seqs, g, L, taps).numpy().reshape(bs, 2, 12, L + P)
    h = symmetric_bank(rng, taps)
    hpad = np.zeros((12, 1, nb))
    hpad[:, 0, :taps] = h
    filt = np.fft.ifft(np.fft.fft(blocks.astype(np.complex128), axis=-1) * np.fft.fft(hpad, axis=-1), axis=-1)
    f = np.concatenate([filt[:, :, b, P: P + g.hop] for b in range(g.nbk)], -1)[..., : g.leff]
    ref = valid_correlation(noise, h)
    np.testing.assert_allclose(ref[:, 0, :, : g.leff], f.real, atol=1e-9)
    np.testing.assert_allclose(ref[:, 1, :, : g.leff], f.imag, atol=1e-9)
    # samples shared by neighbouring blocks must agree, or the helper refuses the buffer
    blocks[1, 3, 1, 0] += 1.0
    with pytest.raises(AssertionError, match="overlapping"):
        rp.unpack(rp.item_blocks(fake_fsave(g, bs, lambda i: blocks[i]), 1, g), g)


def test_matrix_geometry():
    """the library's geometry for the cases of tests/test_gpu_reverb_pin.py: the polyphase factor each one is meant to
    reach, and the audio block counts that select the three partition multiply-accumulate instantiations"""
    from dasp_pytorch_b200 import build
    build.build()
    classes, orders = set(), set()
    for R in range(1, 17):
        n, L = rp.default_case(R)
        g = rp.geometry(0, n, L, 1023, 0)
        assert (g.nb, g.rpp) == (8192, R) and n % 4 == 0, (R, g)
        classes.add(12 if g.x_blocks <= 12 else (16 if g.x_blocks <= 16 else 0))
        orders.add((L > n) - (L < n))
    assert classes == {12, 16, 0} and orders == {-1, 0, 1}
    assert rp.geometry(0, 12000, 14001, 2047, 0).nb == 16384
    assert rp.geometry(0, 44000, 44000, 2047, 0).rpp == 3
    assert rp.geometry(0, 26000, 24000, 4095, 0).nb == 32768
    assert rp.geometry(0, 132000, 132000, 1023, 0).rpp > rp.MAX_SPECTRAL_R
    bench = rp.geometry(0, 48000, 96000, 1023, 0)
    assert (bench.rpp, bench.nbk) == (6, 7)          # chunk stride 12 * 7 nb != in-chunk stride 6 nb


def test_statistics_accept_white_noise():
    rng = np.random.default_rng(0)
    rows = rng.standard_normal((24, 16384))
    rp.check_marginals(rows)
    rp.check_white(rows)
    pairs = [(f"{i}", rows[i], rows[i + 1]) for i in range(23)]
    rp.check_independent(pairs, rows.shape[1])


def test_statistics_reject_generator_faults():
    rng = np.random.default_rng(1)
    n = 16384
    rows = rng.standard_normal((24, n))
    with pytest.raises(AssertionError):
        rp.check_marginals(rows * 1.05)                                   # variance 10 % off
    with pytest.raises(AssertionError):
        rp.check_marginals(np.sign(rows) * np.sqrt(np.abs(rows)) * 1.48)  # not Gaussian
    with pytest.raises(AssertionError):
        rp.check_white(rows + 0.3 * np.roll(rows, 1, axis=1))            # coloured
    with pytest.raises(AssertionError):
        shifted = np.roll(rows[0], 777)
        rp.check_independent([("shifted copy", rows[0], shifted)], n)    # a reused stream at an offset
    with pytest.raises(AssertionError):
        part = rows[1].copy()
        part[: n // 8] = rows[0][: n // 8]
        rp.check_independent([("shared start", rows[0], part)], n)      # one eighth of the stream reused
