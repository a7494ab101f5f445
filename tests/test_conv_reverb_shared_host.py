"""CPU checks of convolution_reverberation with one impulse response shared by the batch: the shared geometry query,
the shapes the op now accepts and still rejects before any launch, and the fp64 oracle's summed IR gradient."""
import pytest
import torch

import conv_oracle
from helpers import SR
from test_conv_reverb_host import GEOMS, KB, NFFT, _align, _call


@pytest.fixture(scope="module")
def lib():
    from dasp_pytorch_b200 import _abi, build
    build.build()
    return _abi.lib()


@pytest.mark.parametrize("n,L,leff,J", GEOMS)
def test_conv_shared_geometry_without_gpu(lib, n, L, leff, J):
    """bs = 0 needs no GPU; the forward's IR slot holds one IR, the backward adds the fp64 sum of its J partitions"""
    from dasp_pytorch_b200 import _abi
    g, ref = _abi.ConvGeom(), _abi.ConvGeom()
    assert lib.dasp_conv_shared_geometry(0, n, L, 7, g) == 0
    assert lib.dasp_conv_geometry(0, n, L, 7, ref) == 0
    I = -(-n // KB)
    assert (g.leff, g.conv_block, g.x_blocks, g.ir_partitions, g.chunk_items) == (leff, KB, I, J, 1)
    assert g.xspec_c64 == 0 and g.irspec_c64 == 0
    assert g.fwd_workspace_bytes == 2 * _align(8 * I * NFFT) + _align(8 * J * NFFT) == ref.fwd_workspace_bytes
    assert g.bwd_workspace_bytes == (2 * _align(8 * I * NFFT) + _align(8 * J * NFFT) + _align(4 * I)
                                     + _align(16 * J * NFFT))
    assert g.bwd_workspace_bytes - ref.bwd_workspace_bytes == _align(16 * J * NFFT)


def test_conv_shared_geometry_rejects_bad_shapes(lib):
    from dasp_pytorch_b200 import _abi
    g = _abi.ConvGeom()
    assert lib.dasp_conv_shared_geometry(0, 48000, 0, 1, g) == -1 and b"ir_len" in lib.dasp_last_error()
    assert lib.dasp_conv_shared_geometry(0, 0, 10, 1, g) == -1
    assert lib.dasp_conv_shared_geometry(-1, 10, 10, 1, g) == -1
    assert lib.dasp_conv_shared_geometry(0, 10, 10, 1, None) == -1


def test_conv_shared_entry_points_need_nothing_at_bs0(lib):
    """like the per-item entry points, bs = 0 launches nothing, and bad channel counts are rejected first"""
    assert lib.dasp_conv_shared_fwd(None, 2, None, 2, 100, None, None, None, None, None, 0, 0, 1000, 1, None) == 0
    assert lib.dasp_conv_shared_bwd(None, None, 2, 2, 100, None, None, None, None, None, None, None, 0, 0, 1000, 1,
                                    None) == 0
    assert lib.dasp_conv_shared_fwd(None, 3, None, 2, 100, None, None, None, None, None, 0, 0, 1000, 1, None) == -1
    assert lib.dasp_conv_shared_bwd(None, None, 2, 3, 100, None, None, None, None, None, None, None, 0, 0, 1000, 1,
                                    None) == -1


def test_conv_shared_ir_reaches_the_cuda_check():
    """an IR of batch 1 against x of batch 2 is accepted now: on CPU tensors it fails only for want of a GPU"""
    from dasp_pytorch_b200.functional import DaspError
    for ir in (torch.zeros(1, 2, 16), torch.zeros(1, 1, 16)):
        with pytest.raises(DaspError):
            _call(ir=ir)
        with pytest.raises(DaspError):
            _call(ir=ir, mix=torch.zeros(1))


def test_conv_shared_still_rejects_other_shapes():
    for kw in (dict(ir=torch.zeros(3, 2, 16)),                                     # batch 3 against 2
               dict(ir=torch.zeros(1, 3, 16)),                                     # 3 channels
               dict(ir=torch.zeros(1, 2, 0)),                                      # no taps
               dict(ir=torch.zeros(1, 16)),                                        # rank
               dict(ir=torch.zeros(1, 2, 16), mix=torch.zeros(3)),                 # wrong mix count
               dict(x=torch.zeros(0, 2, 64), ir=torch.zeros(1, 2, 16), mix=torch.zeros(1))):   # batch 1 against 0
        with pytest.raises(ValueError):
            _call(**kw)


@pytest.mark.parametrize("in_chs,ir_chs", [(2, 2), (1, 2), (2, 1), (1, 1)])
def test_conv_oracle_expanded_ir_gradient_is_the_item_sum(in_chs, ir_chs):
    """the fp64 oracle with ir.expand(bs, -1, -1) gives the shared IR the sum of the per-item IR gradients"""
    gen = torch.Generator().manual_seed(29 + in_chs + 2 * ir_chs)
    bs, n, L = 4, 700, 900
    x = torch.rand(bs, in_chs, n, generator=gen, dtype=torch.float64) * 2 - 1
    ir = torch.rand(1, ir_chs, L, generator=gen, dtype=torch.float64) * 2 - 1
    mix = torch.rand(bs, generator=gen, dtype=torch.float64)
    w = torch.rand(bs, 2, n, generator=gen, dtype=torch.float64) * 2 - 1
    h = ir.clone().requires_grad_(True)
    (conv_oracle.convolution_reverberation(x, SR, h.expand(bs, -1, -1), mix) * w).sum().backward()
    total = torch.zeros_like(ir)
    for b in range(bs):
        hb = ir.clone().requires_grad_(True)
        (conv_oracle.convolution_reverberation(x[b:b + 1], SR, hb, mix[b:b + 1]) * w[b:b + 1]).sum().backward()
        total += hb.grad
    assert h.grad.shape == (1, ir_chs, L)
    assert float((h.grad - total).abs().max() / total.abs().max()) < 1e-12
    assert float(h.grad[..., n:].abs().max() / total.abs().max()) < 1e-12      # taps >= n reach no output
