"""CPU checks of convolution_reverberation: the library's geometry query, input validation before any launch, and the
fp64 oracle of tests/conv_oracle.py held to the reference goldens through the reverb it is the apply stage of."""
import numpy as np
import pytest
import torch

import conv_oracle
import oracle
from conftest import load_golden, rel_peak_err
from helpers import SR

KB, NFFT = 4096, 8192


@pytest.fixture(scope="module")
def lib():
    from dasp_pytorch_b200 import _abi, build
    build.build()
    return _abi.lib()


def _align(v):
    return (v + 255) // 256 * 256


# (n, L, leff, ir_partitions)
GEOMS = [
    (48000, 30000, 30000, 8),          # L < n
    (48000, 48000, 48000, 12),         # L = n
    (48000, 96000, 48000, 12),         # L > n: taps >= n reach no output
    (48000, 1, 1, 1),                  # a single tap
    (48000, 8191, 8191, 2),            # k * 4096 - 1
    (48000, 8192, 8192, 2),            # k * 4096
    (48000, 8193, 8193, 3),            # k * 4096 + 1
    (1001, 500, 500, 1),
    (70000, 66000, 66000, 17),
]


@pytest.mark.parametrize("n,L,leff,J", GEOMS)
def test_conv_geometry_without_gpu(lib, n, L, leff, J):
    from dasp_pytorch_b200 import _abi
    g = _abi.ConvGeom()
    assert lib.dasp_conv_geometry(0, n, L, 7, g) == 0
    I = -(-n // KB)
    assert (g.leff, g.conv_block, g.x_blocks, g.ir_partitions) == (leff, KB, I, J)
    assert g.chunk_items == 1 and g.xspec_c64 == 0 and g.irspec_c64 == 0
    # one item per pass without a batch, and no cuFFT work area is planned without a GPU
    assert g.fwd_workspace_bytes == 2 * _align(8 * I * NFFT) + _align(8 * J * NFFT)
    assert g.bwd_workspace_bytes == 2 * _align(8 * I * NFFT) + _align(8 * J * NFFT) + _align(4 * I)


# (n, L, taps): L > n, L < n, I = 18 and J = 17, 2047 taps (nb = 16384), a short signal, polyphase factor 19 > 16
@pytest.mark.parametrize("n,L,taps", [(48000, 96000, 1023), (48000, 30000, 1023), (70000, 66000, 1023),
                                      (48000, 48000, 2047), (1001, 500, 31), (200000, 150000, 1023)])
def test_reverb_geometry_workspace_without_gpu(lib, n, L, taps):
    """the reverb's workspace is the convolution's plus its own region: the filtered noise of a chunk in the forward,
    the per-partition partials of the 24 band-parameter gradients in the backward"""
    from dasp_pytorch_b200 import _abi
    g = _abi.ReverbGeom()
    assert lib.dasp_reverb_geometry(0, n, L, taps, 7, g) == 0
    I, J = -(-n // KB), -(-min(L, n) // KB)
    assert (g.leff, g.x_blocks, g.ir_partitions, g.chunk_items) == (min(L, n), I, J, 1)
    conv = 2 * _align(8 * I * NFFT) + _align(8 * J * NFFT)
    pair_c64 = max(g.nbk, g.rpp) * g.nb
    assert g.fwd_workspace_bytes == conv + _align(8 * 12 * pair_c64)
    assert g.bwd_workspace_bytes == conv + _align(4 * 24 * max(g.nbk, -(-g.nb // 256), J)) + _align(4 * I)


def test_conv_geometry_rejects_bad_shapes(lib):
    from dasp_pytorch_b200 import _abi
    g = _abi.ConvGeom()
    assert lib.dasp_conv_geometry(0, 48000, 0, 1, g) == -1 and b"ir_len" in lib.dasp_last_error()
    assert lib.dasp_conv_geometry(0, 0, 10, 1, g) == -1
    assert lib.dasp_conv_geometry(0, 10, 10, 1, None) == -1


def _call(x=None, ir=None, mix=None):
    import dasp_pytorch_b200 as D
    x = torch.zeros(2, 2, 64) if x is None else x
    ir = torch.zeros(2, 2, 16) if ir is None else ir
    mix = torch.zeros(2) if mix is None else mix
    return D.convolution_reverberation(x, SR, ir, mix)


def test_conv_validation_before_any_launch():
    from dasp_pytorch_b200.functional import DaspError
    with pytest.raises(DaspError):                                  # CPU tensors: no CPU path
        _call()
    with pytest.raises(DaspError):
        _call(x=torch.zeros(2, 2, 64, dtype=torch.int32))
    for kw in (dict(x=torch.zeros(2, 3, 64)), dict(ir=torch.zeros(2, 3, 16)),      # 3 channels
               dict(ir=torch.zeros(3, 2, 16)),                                     # batch mismatch
               dict(mix=torch.zeros(3)),                                           # wrong mix count
               dict(x=torch.zeros(2, 64)), dict(ir=torch.zeros(2, 16)),            # ranks
               dict(ir=torch.zeros(2, 2, 0))):
        with pytest.raises(ValueError):
            _call(**kw)


def test_conv_exported():
    import dasp_pytorch_b200 as D
    assert "convolution_reverberation" in D.functional.__all__
    assert D.convolution_reverberation is D.functional.convolution_reverberation


@pytest.mark.parametrize("tag", ["st", "mono"])
@pytest.mark.parametrize("method", ["fft", "direct"])
def test_conv_oracle_is_the_reverb_apply_stage(tag, method):
    """the reverb oracle's IR through conv_oracle.convolution_reverberation gives the reference goldens"""
    g = load_golden("reverb.npz")
    L, taps, seed = int(g["L"]), int(g["taps"]), int(g[f"{tag}_seed"])
    x = torch.as_tensor(g[f"{tag}_x"]).double()
    bs = x.shape[0]
    p64 = [torch.as_tensor(g[f"{tag}_p01"]).double()[:, i] for i in range(25)]
    noise = oracle.reverb_noise(bs, L, taps, seed)
    ir = conv_oracle.reverb_ir(SR, p64, noise, L, taps)
    y = conv_oracle.convolution_reverberation(x, SR, ir, p64[24], method=method)
    assert rel_peak_err(y, g[f"{tag}_y64"]).max() < 1e-9
    ref = oracle.noise_shaped_reverberation(x, SR, *p64, num_samples=L, num_bandpass_taps=taps, noise=noise)
    assert rel_peak_err(y, ref).max() < 1e-12


def test_conv_oracle_mono_ir_and_short_ir():
    """a mono IR equals its stereo duplicate; an IR longer than x only contributes its first n taps"""
    gen = torch.Generator().manual_seed(3)
    x = torch.rand(2, 1, 300, generator=gen, dtype=torch.float64) - 0.5
    ir = torch.rand(2, 1, 500, generator=gen, dtype=torch.float64) - 0.5
    mix = torch.tensor([0.3, 0.8], dtype=torch.float64)
    a = conv_oracle.convolution_reverberation(x, SR, ir, mix)
    b = conv_oracle.convolution_reverberation(x, SR, ir.repeat(1, 2, 1), mix, method="direct")
    c = conv_oracle.convolution_reverberation(x, SR, ir[..., :300], mix)
    assert np.abs((a - b).numpy()).max() < 1e-12 and np.abs((a - c).numpy()).max() < 1e-12
