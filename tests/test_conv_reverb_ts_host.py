"""CPU checks of convolution_reverberation with a true-stereo (four-channel) impulse response: the identities that tie
its fp64 oracle (tests/conv_ts_oracle.py) to the stereo one (tests/conv_oracle.py), the two true-stereo geometry
queries, and the shapes the op and the entry points accept and reject before any launch."""
import pytest
import torch

import conv_oracle
import conv_ts_oracle
from helpers import SR
from test_conv_reverb_host import GEOMS, KB, NFFT, _align, _call


@pytest.fixture(scope="module")
def lib():
    from dasp_pytorch_b200 import _abi, build
    build.build()
    return _abi.lib()


def _rand(gen, *shape):
    return torch.rand(*shape, generator=gen, dtype=torch.float64) * 2 - 1


def _rel(a, b):
    return float((a - b).abs().max() / b.abs().max())


@pytest.mark.parametrize("method", ["fft", "direct"])
@pytest.mark.parametrize("in_chs", [2, 1])
def test_ts_oracle_diagonal_ir_is_the_stereo_ir(method, in_chs):
    """(hL, 0, 0, hR) is the stereo IR (hL, hR)"""
    gen = torch.Generator().manual_seed(61 + in_chs)
    x, h, mix = _rand(gen, 3, in_chs, 700), _rand(gen, 3, 2, 900), torch.rand(3, generator=gen, dtype=torch.float64)
    z = torch.zeros_like(h[:, :1])
    ts = torch.cat([h[:, :1], z, z, h[:, 1:]], dim=1)
    a = conv_ts_oracle.convolution_reverberation(x, SR, ts, mix, method=method)
    b = conv_oracle.convolution_reverberation(x, SR, h, mix, method=method)
    assert _rel(a, b) < 1e-12


@pytest.mark.parametrize("in_chs", [2, 1])
def test_ts_oracle_is_the_two_call_composition(in_chs):
    """a true-stereo call equals the left input through (LL, LR) plus the right input through (RL, RR), each at mix 1,
    blended with the dry signal; fft equals direct"""
    gen = torch.Generator().manual_seed(67 + in_chs)
    bs, n, L = 3, 800, 1500
    x, ir, mix = _rand(gen, bs, in_chs, n), _rand(gen, bs, 4, L), torch.rand(bs, generator=gen, dtype=torch.float64)
    y = conv_ts_oracle.convolution_reverberation(x, SR, ir, mix)
    x2 = x.repeat(1, 2, 1) if in_chs == 1 else x
    one = torch.ones(bs, dtype=torch.float64)
    wet = (conv_oracle.convolution_reverberation(x2[:, 0:1], SR, ir[:, 0:2], one)
           + conv_oracle.convolution_reverberation(x2[:, 1:2], SR, ir[:, 2:4], one))
    m = mix.reshape(bs, 1, 1)
    assert _rel(y, (1 - m) * x2 + m * wet) < 1e-12
    assert _rel(y, conv_ts_oracle.convolution_reverberation(x, SR, ir, mix, method="direct")) < 1e-12


def test_ts_oracle_expanded_ir_gradient_is_the_item_sum():
    gen = torch.Generator().manual_seed(71)
    bs, n, L = 4, 700, 900
    x, ir, mix, w = _rand(gen, bs, 2, n), _rand(gen, 1, 4, L), torch.rand(bs, generator=gen, dtype=torch.float64), \
        _rand(gen, bs, 2, n)
    h = ir.clone().requires_grad_(True)
    (conv_ts_oracle.convolution_reverberation(x, SR, h.expand(bs, -1, -1), mix) * w).sum().backward()
    total = torch.zeros_like(ir)
    for b in range(bs):
        hb = ir.clone().requires_grad_(True)
        (conv_ts_oracle.convolution_reverberation(x[b:b + 1], SR, hb, mix[b:b + 1]) * w[b:b + 1]).sum().backward()
        total += hb.grad
    assert h.grad.shape == (1, 4, L)
    assert _rel(h.grad, total) < 1e-12
    assert float(h.grad[..., n:].abs().max() / total.abs().max()) < 1e-12      # taps >= n reach no output


@pytest.mark.parametrize("n,L,leff,J", GEOMS)
def test_ts_geometry_without_gpu(lib, n, L, leff, J):
    """bs = 0 needs no GPU; ir_partitions is still J per set, the IR regions hold both sets (2 J partitions)"""
    from dasp_pytorch_b200 import _abi
    I = -(-n // KB)
    for fn, shared in ((lib.dasp_conv_ts_geometry, False), (lib.dasp_conv_shared_ts_geometry, True)):
        g = _abi.ConvGeom()
        assert fn(0, n, L, 7, g) == 0
        assert (g.leff, g.conv_block, g.x_blocks, g.ir_partitions, g.chunk_items) == (leff, KB, I, J, 1)
        assert g.xspec_c64 == 0 and g.irspec_c64 == 0
        assert g.fwd_workspace_bytes == 2 * _align(8 * I * NFFT) + _align(8 * 2 * J * NFFT)
        acc = _align(16 * 2 * J * NFFT) if shared else 0
        assert g.bwd_workspace_bytes == 2 * _align(8 * I * NFFT) + _align(8 * 2 * J * NFFT) + _align(4 * I) + acc


def test_ts_geometry_rejects_bad_shapes(lib):
    from dasp_pytorch_b200 import _abi
    g = _abi.ConvGeom()
    for fn in (lib.dasp_conv_ts_geometry, lib.dasp_conv_shared_ts_geometry):
        assert fn(0, 48000, 0, 1, g) == -1 and b"ir_len" in lib.dasp_last_error()
        assert fn(0, 0, 10, 1, g) == -1
        assert fn(0, 10, 10, 1, None) == -1


def test_ts_entry_points_at_bs0(lib):
    """ir_chs = 4 is accepted and launches nothing at bs = 0; 3 and 5 are still rejected"""
    for fwd, bwd in ((lib.dasp_conv_fwd, lib.dasp_conv_bwd), (lib.dasp_conv_shared_fwd, lib.dasp_conv_shared_bwd)):
        for ir_chs, rc in ((4, 0), (3, -1), (5, -1)):
            assert fwd(None, 2, None, ir_chs, 100, None, None, None, None, None, 0, 0, 1000, 1, None) == rc
            assert bwd(None, None, 1, ir_chs, 100, None, None, None, None, None, None, None, 0, 0, 1000, 1, None) == rc


def test_ts_ir_reaches_the_cuda_check():
    """a four-channel IR, per item or shared, is accepted: on CPU tensors it fails only for want of a GPU"""
    from dasp_pytorch_b200.functional import DaspError
    for kw in (dict(ir=torch.zeros(2, 4, 16)), dict(ir=torch.zeros(1, 4, 16)),
               dict(x=torch.zeros(2, 1, 64), ir=torch.zeros(2, 4, 16))):
        with pytest.raises(DaspError):
            _call(**kw)


@pytest.mark.parametrize("chs", [3, 5])
def test_ts_other_channel_counts_are_rejected(chs):
    for ir in (torch.zeros(2, chs, 16), torch.zeros(1, chs, 16)):
        with pytest.raises(ValueError):
            _call(ir=ir)
