"""The reverb's forward reads only the IR taps its synthesis wrote.

The IR-partition transform bulk-copies the first half of each partition slot and pads in shared memory (taps >= leff
and the second half), so the slots are never zero-filled beforehand.  Whatever the partition buffer held before the
call, NaN included, must therefore leave y and the saved spectra unchanged."""
import pytest
import torch

from dasp_pytorch_b200 import _abi
from helpers import SR

pytestmark = pytest.mark.gpu
TAPS = 1023


def _geom(bs, n, L, chunk):
    g = _abi.ReverbGeom()
    _abi.check(_abi.lib().dasp_reverb_geometry(bs, n, L, TAPS, chunk, g), "dasp_reverb_geometry")
    return g


# leff = 30001: last of 8 partitions holds 1329 taps (an odd count); leff = n = 20000: last of 5 holds 3616 taps
@pytest.mark.parametrize("n,L,in_chs", [(48000, 30001, 2), (20000, 26000, 2), (20000, 26000, 1)])
def test_reverb_fwd_ignores_prior_partition_contents(cuda_device, n, L, in_chs):
    lib = _abi.lib()
    dev = cuda_device
    bs, chunk = 3, 2                                            # two chunks: per-chunk offsets into irspec_save
    g = _geom(bs, n, L, chunk)
    assert g.leff % g.conv_block != 0
    gen = torch.Generator().manual_seed(5)
    x = (torch.rand(bs, in_chs, n, generator=gen) * 2 - 1).to(dev)
    params = torch.rand(bs, 25, generator=gen).to(dev)
    seed = torch.tensor([1234], dtype=torch.int64, device=dev)

    def run(fill, keep):
        y = torch.empty(bs, 2, n, device=dev)
        ws = torch.empty(g.fwd_workspace_bytes, dtype=torch.uint8, device=dev)
        ws.view(torch.float32)[: g.fwd_workspace_bytes // 4].fill_(fill)
        fsave = xspec = irspec = None
        if keep:
            fsave = torch.empty(g.f_floats, device=dev)
            xspec = torch.empty(g.xspec_c64, dtype=torch.complex64, device=dev)
            irspec = torch.empty(g.irspec_c64, dtype=torch.complex64, device=dev)
            irspec.view(torch.float32).fill_(fill)
        _abi.check(lib.dasp_reverb_fwd(_abi.ptr(x), in_chs, _abi.ptr(params), None, _abi.ptr(seed), _abi.ptr(y),
                                       _abi.ptr(fsave), _abi.ptr(xspec), _abi.ptr(irspec), _abi.ptr(ws), ws.numel(), bs,
                                       n, L, TAPS, chunk, float(SR), _abi.stream_ptr(dev)), "dasp_reverb_fwd")
        torch.cuda.synchronize(dev)
        assert lib.dasp_debug_reverb_last_path() == 2               # generator + ifft_shape_kernel, own convolution
        return y, irspec

    y0, h0 = run(0.0, True)
    y1, h1 = run(float("nan"), True)
    y2, _ = run(float("nan"), False)                                # transient partition buffer in the workspace
    assert torch.isfinite(y0).all() and torch.isfinite(torch.view_as_real(h0)).all()
    assert torch.equal(y0, y1) and torch.equal(y0, y2)
    assert torch.equal(torch.view_as_real(h0), torch.view_as_real(h1))
