"""CPU checks of convolution_bus: its fp64 oracle (tests/conv_bus_oracle.py) against the true-stereo oracle and against
its own single-source composition, the geometry query without a GPU, the entry points at bs = 0, and the shapes,
channel counts and devices the op and the entry points reject before any launch."""
import pytest
import torch

import conv_bus_oracle
import conv_oracle
import conv_ts_oracle
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


@pytest.mark.parametrize("method", ["fft", "direct"])
def test_bus_oracle_methods_agree(method):
    gen = torch.Generator().manual_seed(5)
    x, h = _rand(gen, 2, 5, 700), _rand(gen, 2, 5, 2, 900)
    a = conv_bus_oracle.convolution_bus(x, SR, h, method=method)
    b = conv_bus_oracle.convolution_bus(x, SR, h, method="direct" if method == "fft" else "fft")
    assert a.shape == (2, 2, 700) and _rel(a, b) < 1e-12


@pytest.mark.parametrize("method", ["fft", "direct"])
def test_bus_oracle_is_the_true_stereo_oracle_at_two_inputs(method):
    """S = 2, O = 2 is convolution_reverberation with the (bs, 4, L) true-stereo IR at mix 1; S = 1, O = 2 is the
    stereo IR with a mono x"""
    gen = torch.Generator().manual_seed(7)
    x, h = _rand(gen, 3, 2, 600), _rand(gen, 3, 2, 2, 800)
    ones = torch.ones(3, dtype=torch.float64)
    ts = conv_ts_oracle.convolution_reverberation(x, SR, h.reshape(3, 4, 800), ones, method=method)
    assert _rel(conv_bus_oracle.convolution_bus(x, SR, h, method=method), ts) < 1e-12
    st = conv_oracle.convolution_reverberation(x[:, :1], SR, h[:, 0], ones, method=method)
    assert _rel(conv_bus_oracle.convolution_bus(x[:, :1], SR, h[:, :1], method=method), st) < 1e-12


@pytest.mark.parametrize("S,O", [(3, 1), (5, 2), (16, 2)])
def test_bus_oracle_is_the_sum_of_single_sources(S, O):
    gen = torch.Generator().manual_seed(S * 10 + O)
    x, h = _rand(gen, 2, S, 500), _rand(gen, 1, S, O, 300)
    y = conv_bus_oracle.convolution_bus(x, SR, h)
    parts = sum(conv_bus_oracle.convolution_bus(x[:, s:s + 1], SR, h[:, s:s + 1], method="direct") for s in range(S))
    assert y.shape == (2, O, 500) and _rel(y, parts) < 1e-12


# (n, L, S, O, leff, ir_partitions)
GEOMS = [(48000, 48000, 8, 2, 48000, 12), (48000, 96000, 3, 1, 48000, 12), (48000, 1, 1, 2, 1, 1),
         (6000, 4097, 5, 1, 4097, 2), (70000, 66000, 16, 2, 66000, 17), (1001, 500, 2, 2, 500, 1)]


def _check_bus_geometry(lib, n, L, S, O, leff, J, shared):
    """the sizes follow from the pair packing: ceil(S / 2) window spectra per block, ceil(S O / 2) partition sets; a
    shared IR adds the fp64 sum of its dL/dIR spectra to the backward workspace"""
    from dasp_pytorch_b200 import _abi
    I, P, NH = -(-n // KB), (S + 1) // 2, (S * O + 1) // 2
    for bs, chunk in ((0, 7), (10, 4)):
        g = _abi.ConvGeom()
        assert lib.dasp_conv_bus_geometry(bs, n, L, S, O, shared, chunk, g) == 0
        c = g.chunk_items
        assert (g.leff, g.conv_block, g.x_blocks, g.ir_partitions) == (leff, KB, I, J)
        assert c == (1 if bs == 0 else 4)
        assert g.xspec_c64 == bs * P * I * NFFT
        assert g.irspec_c64 == (min(bs, 1) if shared else bs) * NH * J * NFFT
        blk = 8 * NFFT
        fwd = _align(blk * c * I) + _align(blk * c * P * I) + _align(blk * (1 if shared else c) * NH * J)
        bwd = (_align(blk * c * I) + _align(blk * c * P * I) + _align(blk * c * NH * J)
               + (_align(16 * NFFT * NH * J) if shared else 0))
        assert (g.fwd_workspace_bytes, g.bwd_workspace_bytes) == (fwd, bwd)


@pytest.mark.parametrize("shared", [0])
@pytest.mark.parametrize("n,L,S,O,leff,J", GEOMS)
def test_bus_geometry_without_gpu(lib, n, L, S, O, leff, J, shared):
    """one IR set per item"""
    _check_bus_geometry(lib, n, L, S, O, leff, J, shared)


@pytest.mark.parametrize("n,L,S,O,leff,J", GEOMS)
def test_bus_shared_geometry_without_gpu(lib, n, L, S, O, leff, J):
    """one IR set for the batch: its partition spectra once, and no per-item factors in the backward workspace (the
    fp64 sum of a shared IR's gradient takes a null factor as 1)"""
    _check_bus_geometry(lib, n, L, S, O, leff, J, 1)


def test_bus_memory_at_1024_items_of_8_inputs(lib):
    """bs = 1024, S = 8, 48000 samples, IR 48000, stereo bus: the workspaces are bounded by the chunk (two items per SM
    of an H100, 264, the default), the saved spectra grow with the batch"""
    from dasp_pytorch_b200 import _abi
    g = _abi.ConvGeom()
    assert lib.dasp_conv_bus_geometry(1024, 48000, 48000, 8, 2, 0, 264, g) == 0
    saved = 8 * (g.xspec_c64 + g.irspec_c64)
    assert saved == 8 * 1024 * (4 * 12 + 8 * 12) * NFFT            # 9.7 GB: (P I + NH J) blocks of 64 KB per item
    assert g.fwd_workspace_bytes == g.bwd_workspace_bytes == 264 * (12 + 48 + 96) * 8 * NFFT      # 2.7 GB


@pytest.mark.parametrize("S,O", [(0, 2), (33, 2), (4, 0), (4, 3)])
def test_bus_entry_points_reject_bad_channels(lib, S, O):
    from dasp_pytorch_b200 import _abi
    g = _abi.ConvGeom()
    assert lib.dasp_conv_bus_geometry(0, 4096, 100, S, O, 0, 4, g) != 0
    for fn in (lib.dasp_conv_bus_fwd, lib.dasp_conv_bus_shared_fwd):
        assert fn(None, None, None, None, None, None, 0, 0, 4096, 100, S, O, 4, None) != 0
    for fn in (lib.dasp_conv_bus_bwd, lib.dasp_conv_bus_shared_bwd):
        assert fn(None, None, None, None, None, None, 0, 0, 4096, 100, S, O, 4, None) != 0


def test_bus_entry_points_at_batch_zero(lib):
    """an empty batch is a no-op (null pointers accepted); bad lengths are still rejected"""
    for fn in (lib.dasp_conv_bus_fwd, lib.dasp_conv_bus_shared_fwd, lib.dasp_conv_bus_bwd, lib.dasp_conv_bus_shared_bwd):
        assert fn(None, None, None, None, None, None, 0, 0, 4096, 100, 3, 2, 4, None) == 0
        assert fn(None, None, None, None, None, None, 0, 0, 0, 100, 3, 2, 4, None) != 0
        assert fn(None, None, None, None, None, None, 0, 0, 4096, 0, 3, 2, 4, None) != 0


def test_bus_entry_points_reject_unaligned_rows_before_any_launch(lib):
    """n % 4 != 0 (the Python op pads those rows) and null pointers fail before any CUDA call"""
    for fn in (lib.dasp_conv_bus_fwd, lib.dasp_conv_bus_shared_fwd):
        assert fn(16, 16, 16, None, None, 16, 1 << 20, 2, 1001, 100, 3, 2, 4, None) != 0
        assert fn(None, None, None, None, None, None, 1 << 20, 2, 1000, 100, 3, 2, 4, None) != 0
    for fn in (lib.dasp_conv_bus_bwd, lib.dasp_conv_bus_shared_bwd):
        assert fn(16, 16, 16, 16, None, 16, 1 << 20, 2, 1001, 100, 3, 2, 4, None) != 0
        assert fn(None, None, None, None, None, None, 1 << 20, 2, 1000, 100, 3, 2, 4, None) != 0


def _call(x=None, ir=None):
    import dasp_pytorch_b200 as D
    x = torch.zeros(2, 3, 64) if x is None else x
    ir = torch.zeros(2, 3, 2, 16) if ir is None else ir
    return D.convolution_bus(x, SR, ir)


@pytest.mark.parametrize("x,ir,msg", [
    (torch.zeros(2, 64), None, "x must be"),
    (None, torch.zeros(2, 3, 16), "impulse_response must be"),
    (torch.zeros(2, 0, 64), torch.zeros(2, 0, 2, 16), "1 to 32 input channels"),
    (torch.zeros(2, 33, 64), torch.zeros(2, 33, 2, 16), "1 to 32 input channels"),
    (None, torch.zeros(2, 4, 2, 16), "4 input rows, x has 3"),
    (None, torch.zeros(2, 3, 3, 16), "mono \\(1\\) or stereo \\(2\\) bus"),
    (None, torch.zeros(3, 3, 2, 16), "batch 3, x has batch 2"),
    (None, torch.zeros(2, 3, 2, 0), "at least one tap"),
    (torch.zeros(2, 3, 0), None, "at least one sample"),
])
def test_bus_shape_validation(x, ir, msg):
    with pytest.raises(ValueError, match=msg):
        _call(x, ir)


def test_bus_rejects_cpu_tensors():
    from dasp_pytorch_b200._abi import DaspError
    import dasp_pytorch_b200 as D
    with pytest.raises(DaspError, match="no CPU path"):
        _call()
    assert D.CONV_BUS_MAX_INPUTS == 32 and "convolution_bus" in D.functional.__all__
