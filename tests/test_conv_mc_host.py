"""CPU checks of multichannel_convolution: the bus oracle (tests/conv_bus_oracle.py) at M >= 3 outputs against its
direct form and its output-pair composition, the geometry query without a GPU, the entry points at bs = 0, and the
shapes, channel counts and devices the op and the entry points reject before any launch."""
import pytest
import torch

import conv_bus_oracle
from helpers import SR

KB, NFFT = 4096, 8192


@pytest.fixture(scope="module")
def lib():
    from dasp_pytorch_b200 import _abi, build
    build.build()
    return _abi.lib()


def _rand(gen, *shape):
    return torch.rand(*shape, generator=gen, dtype=torch.float64) * 2 - 1


def _rel(a, b):
    return float((a - b).abs().max() / b.abs().max())


def _align(v):
    return (v + 255) // 256 * 256


@pytest.mark.parametrize("M", [3, 4, 5, 8, 32])
def test_mc_oracle_direct_fft_and_output_pairs_agree(M):
    """the oracle states any M: its direct and FFT forms agree, and it is the concatenation of its output-pair calls"""
    gen = torch.Generator().manual_seed(M)
    S = 3
    x, h = _rand(gen, 2, S, 600), _rand(gen, 2, S, M, 700)
    y = conv_bus_oracle.convolution_bus(x, SR, h)
    assert y.shape == (2, M, 600)
    assert _rel(y, conv_bus_oracle.convolution_bus(x, SR, h, method="direct")) < 1e-12
    pairs = torch.cat([conv_bus_oracle.convolution_bus(x, SR, h[:, :, q:q + 2], method="direct")
                       for q in range(0, M, 2)], 1)
    assert _rel(y, pairs) < 1e-12


# (n, L, S, M, leff, ir_partitions)
GEOMS = [(48000, 48000, 4, 8, 48000, 12), (48000, 96000, 3, 5, 48000, 12), (48000, 1, 1, 3, 1, 1),
         (6000, 4097, 5, 7, 4097, 2), (70000, 66000, 16, 4, 66000, 17), (1001, 500, 2, 16, 500, 1),
         (48000, 30000, 32, 32, 30000, 8), (20000, 9000, 3, 1, 9000, 3), (20000, 9000, 5, 2, 9000, 3)]


def _check_mc_geometry(lib, n, L, S, M, leff, J, shared):
    """the bus's sizes with Q = ceil(M / 2) output and gradient spectra per block: ceil(S / 2) window spectra per block,
    ceil(S M / 2) partition sets; a shared IR adds the fp64 sum of its dL/dIR spectra to the backward workspace"""
    from dasp_pytorch_b200 import _abi
    I, P, Q, NH = -(-n // KB), (S + 1) // 2, (M + 1) // 2, (S * M + 1) // 2
    for bs, chunk in ((0, 7), (10, 4)):
        g = _abi.ConvGeom()
        assert lib.dasp_conv_mc_geometry(bs, n, L, S, M, shared, chunk, g) == 0
        c = g.chunk_items
        assert (g.leff, g.conv_block, g.x_blocks, g.ir_partitions) == (leff, KB, I, J)
        assert c == (1 if bs == 0 else 4)
        assert g.xspec_c64 == bs * P * I * NFFT
        assert g.irspec_c64 == (min(bs, 1) if shared else bs) * NH * J * NFFT
        blk = 8 * NFFT
        fwd = _align(blk * c * Q * I) + _align(blk * c * P * I) + _align(blk * (1 if shared else c) * NH * J)
        bwd = (_align(blk * c * Q * I) + _align(blk * c * P * I) + _align(blk * c * NH * J)
               + (_align(16 * NFFT * NH * J) if shared else 0))
        assert (g.fwd_workspace_bytes, g.bwd_workspace_bytes) == (fwd, bwd)


@pytest.mark.parametrize("shared", [0, 1], ids=["item", "shared"])
@pytest.mark.parametrize("n,L,S,M,leff,J", GEOMS)
def test_mc_geometry_without_gpu(lib, n, L, S, M, leff, J, shared):
    _check_mc_geometry(lib, n, L, S, M, leff, J, shared)


@pytest.mark.parametrize("shared", [0, 1])
@pytest.mark.parametrize("S,M", [(3, 1), (5, 2), (16, 2)])
def test_mc_geometry_is_the_bus_geometry_up_to_two_outputs(lib, S, M, shared):
    from dasp_pytorch_b200 import _abi
    a, b = _abi.ConvGeom(), _abi.ConvGeom()
    assert lib.dasp_conv_mc_geometry(6, 50000, 30000, S, M, shared, 4, a) == 0
    assert lib.dasp_conv_bus_geometry(6, 50000, 30000, S, M, shared, 4, b) == 0
    assert [getattr(a, f) for f, _ in a._fields_] == [getattr(b, f) for f, _ in b._fields_]


@pytest.mark.parametrize("S,M", [(0, 4), (33, 4), (4, 0), (4, 33), (-1, 4), (4, -2)])
def test_mc_entry_points_reject_bad_channels(lib, S, M):
    from dasp_pytorch_b200 import _abi
    g = _abi.ConvGeom()
    assert lib.dasp_conv_mc_geometry(0, 4096, 100, S, M, 0, 4, g) != 0
    for fn in (lib.dasp_conv_mc_fwd, lib.dasp_conv_mc_shared_fwd, lib.dasp_conv_mc_bwd, lib.dasp_conv_mc_shared_bwd):
        assert fn(None, None, None, None, None, None, 0, 0, 4096, 100, S, M, 4, None) != 0


def test_mc_geometry_rejects_a_null_out(lib):
    assert lib.dasp_conv_mc_geometry(2, 4096, 100, 3, 4, 0, 4, None) != 0


def test_mc_entry_points_at_batch_zero(lib):
    """an empty batch is a no-op (null pointers accepted); bad lengths are still rejected"""
    for fn in (lib.dasp_conv_mc_fwd, lib.dasp_conv_mc_shared_fwd, lib.dasp_conv_mc_bwd, lib.dasp_conv_mc_shared_bwd):
        assert fn(None, None, None, None, None, None, 0, 0, 4096, 100, 3, 8, 4, None) == 0
        assert fn(None, None, None, None, None, None, 0, 0, 0, 100, 3, 8, 4, None) != 0
        assert fn(None, None, None, None, None, None, 0, 0, 4096, 0, 3, 8, 4, None) != 0
        assert fn(None, None, None, None, None, None, 0, -1, 4096, 100, 3, 8, 4, None) != 0


def test_mc_entry_points_reject_unaligned_rows_and_null_pointers_before_any_launch(lib):
    """n % 4 != 0 (the Python op pads those rows), misaligned rows and null pointers fail before any CUDA call"""
    for fn in (lib.dasp_conv_mc_fwd, lib.dasp_conv_mc_shared_fwd):
        assert fn(16, 16, 16, None, None, 16, 1 << 20, 2, 1001, 100, 3, 8, 4, None) != 0
        assert fn(20, 16, 16, None, None, 16, 1 << 20, 2, 1000, 100, 3, 8, 4, None) != 0
        assert fn(None, None, None, None, None, None, 1 << 20, 2, 1000, 100, 3, 8, 4, None) != 0
        assert fn(16, 16, None, None, None, 16, 1 << 20, 2, 1000, 100, 3, 8, 4, None) != 0
        assert fn(16, 16, 16, 16, None, 16, 1 << 20, 2, 1000, 100, 3, 8, 4, None) != 0   # one *_save buffer
    for fn in (lib.dasp_conv_mc_bwd, lib.dasp_conv_mc_shared_bwd):
        assert fn(16, 16, 16, 16, None, 16, 1 << 20, 2, 1001, 100, 3, 8, 4, None) != 0
        assert fn(20, 16, 16, 16, None, 16, 1 << 20, 2, 1000, 100, 3, 8, 4, None) != 0
        assert fn(None, None, None, None, None, None, 1 << 20, 2, 1000, 100, 3, 8, 4, None) != 0
        assert fn(16, None, 16, 16, None, 16, 1 << 20, 2, 1000, 100, 3, 8, 4, None) != 0


def test_bus_entry_points_still_reject_three_outputs(lib):
    from dasp_pytorch_b200 import _abi
    assert lib.dasp_conv_bus_geometry(0, 4096, 100, 4, 3, 0, 4, _abi.ConvGeom()) != 0
    for fn in (lib.dasp_conv_bus_fwd, lib.dasp_conv_bus_shared_fwd, lib.dasp_conv_bus_bwd, lib.dasp_conv_bus_shared_bwd):
        assert fn(None, None, None, None, None, None, 0, 0, 4096, 100, 4, 3, 4, None) != 0


def _call(x=None, ir=None):
    import dasp_pytorch_b200 as D
    x = torch.zeros(2, 3, 64) if x is None else x
    ir = torch.zeros(2, 3, 8, 16) if ir is None else ir
    return D.multichannel_convolution(x, SR, ir)


@pytest.mark.parametrize("x,ir,msg", [
    (torch.zeros(2, 64), None, "x must be"),
    (None, torch.zeros(2, 3, 16), "impulse_response must be"),
    (torch.zeros(2, 0, 64), torch.zeros(2, 0, 8, 16), "multichannel_convolution: 1 to 32 input channels"),
    (torch.zeros(2, 33, 64), torch.zeros(2, 33, 8, 16), "multichannel_convolution: 1 to 32 input channels"),
    (None, torch.zeros(2, 4, 8, 16), "4 input rows, x has 3"),
    (None, torch.zeros(2, 3, 0, 16), "1 to 32 output channels are supported, got 0"),
    (None, torch.zeros(2, 3, 33, 16), "1 to 32 output channels are supported, got 33"),
    (None, torch.zeros(3, 3, 8, 16), "batch 3, x has batch 2"),
    (None, torch.zeros(2, 3, 8, 0), "at least one tap"),
    (torch.zeros(2, 3, 0), None, "at least one sample"),
])
def test_mc_shape_validation(x, ir, msg):
    with pytest.raises(ValueError, match=msg):
        _call(x, ir)


def test_bus_still_rejects_three_outputs():
    import dasp_pytorch_b200 as D
    with pytest.raises(ValueError, match="mono \\(1\\) or stereo \\(2\\) bus is supported, got 3 outputs"):
        D.convolution_bus(torch.zeros(2, 3, 64), SR, torch.zeros(2, 3, 3, 16))


def test_mc_rejects_cpu_tensors():
    from dasp_pytorch_b200._abi import DaspError
    import dasp_pytorch_b200 as D
    with pytest.raises(DaspError, match="no CPU path"):
        _call()
    assert D.CONV_MC_MAX_OUTPUTS == 32 and "multichannel_convolution" in D.functional.__all__
    assert D.multichannel_convolution is D.functional.multichannel_convolution
