"""The reverb forward overlaps chunk k's audio convolution with chunk k + 1's IR synthesis (side streams forked from and
joined back to the caller's stream) when a backward follows, i.e. when f_save and irspec_save keep every chunk's slots.
Every unit writes fixed addresses keyed by the absolute item index, so the pipelined forward, the serial one (no saved
buffers) and a single chunk agree bit for bit, and so do the gradients."""
from types import SimpleNamespace

import pytest
import torch

import reverb_pin as rp
from dasp_pytorch_b200 import _abi
from helpers import SR

pytestmark = pytest.mark.gpu
TAPS = 1023


def _fwd_bwd(dev, x, params, L, chunk, save=True, fill=float("nan")):
    """raw forward (with f_save / xspec_save / irspec_save prefilled with `fill` when save, without them otherwise) and,
    when save, the backward; returns (last path, y, f_save, X spectra, IR spectra, dL/dx, dL/dparams, geometry)"""
    lib = _abi.lib()
    bs, in_chs, n = x.shape
    g = _abi.ReverbGeom()
    _abi.check(lib.dasp_reverb_geometry(bs, n, L, TAPS, chunk, g), "dasp_reverb_geometry")
    seed = torch.tensor([2468], dtype=torch.int64, device=dev)
    y = torch.full((bs, 2, n), fill, device=dev)
    fsave = xspec = irspec = None
    if save:
        fsave = torch.full((g.f_floats,), fill, device=dev)
        xspec = torch.full((g.xspec_c64 * 2,), fill, device=dev)
        irspec = torch.full((g.irspec_c64 * 2,), fill, device=dev)
    ws = torch.full((g.fwd_workspace_bytes // 4 + 1,), fill, device=dev)
    _abi.check(lib.dasp_reverb_fwd(_abi.ptr(x), in_chs, _abi.ptr(params), None, _abi.ptr(seed), _abi.ptr(y),
                                   _abi.ptr(fsave), _abi.ptr(xspec), _abi.ptr(irspec), _abi.ptr(ws), ws.numel() * 4,
                                   bs, n, L, TAPS, chunk, float(SR), _abi.stream_ptr(dev)), "dasp_reverb_fwd")
    used = lib.dasp_debug_reverb_last_path()
    gx = gp = None
    if save:
        gy = torch.cos(torch.arange(bs * 2 * n, device=dev, dtype=torch.float32) * 0.003).reshape(bs, 2, n)
        gx = torch.empty_like(x)
        gp = torch.empty_like(params)
        wsb = torch.full((g.bwd_workspace_bytes // 4 + 1,), fill, device=dev)
        _abi.check(lib.dasp_reverb_bwd(_abi.ptr(gy), _abi.ptr(x), in_chs, _abi.ptr(params), _abi.ptr(fsave),
                                       _abi.ptr(xspec), _abi.ptr(irspec), _abi.ptr(gx), _abi.ptr(gp), _abi.ptr(wsb),
                                       wsb.numel() * 4, bs, n, L, TAPS, chunk, 1, _abi.stream_ptr(dev)), "dasp_reverb_bwd")
    torch.cuda.synchronize(dev)
    return used, y, fsave, xspec, irspec, gx, gp, g


@pytest.mark.parametrize("in_chs", [1, 2])
@pytest.mark.parametrize("R", [6, 9])          # 6: ir_synth_cluster_kernel; 9: spectral_gen_kernel -> ifft_shape_kernel
def test_pipelined_forward_matches_serial_and_one_chunk(cuda_device, R, in_chs):
    dev = cuda_device
    n, L = rp.default_case(R)
    bs = 7
    gen = torch.Generator().manual_seed(700 + R + in_chs)
    x = (torch.rand(bs, in_chs, n, generator=gen) * 2 - 1).to(dev)
    params = torch.rand(bs, 25, generator=gen).to(dev)

    used, y1, _, _, _, gx1, gp1, g = _fwd_bwd(dev, x, params, L, bs)        # one chunk
    assert g.rpp == R and g.nb == 8192 and used == 2
    for chunk in (2, 3):                                                     # 4 and 3 chunks, remainder chunks of 1
        used, y, fsave, xspec, irspec, gx, gp, g = _fwd_bwd(dev, x, params, L, chunk)
        assert used == 2
        # every element the backward reads was written, over a NaN prefill
        geom = SimpleNamespace(rpp=g.rpp, nbk=g.nbk, nb=g.nb, chunk_items=g.chunk_items)
        for i in range(bs):
            assert torch.isfinite(torch.view_as_real(rp.item_blocks(fsave, i, geom))).all(), (chunk, i)
        assert torch.isfinite(xspec).all() and torch.isfinite(irspec).all(), chunk
        assert torch.equal(y, y1), chunk
        assert torch.equal(gx, gx1) and torch.equal(gp, gp1), chunk
        used, y_serial, *_ = _fwd_bwd(dev, x, params, L, chunk, save=False)  # no saved buffers: serial order
        assert used == 2
        assert torch.equal(y_serial, y1), chunk


def _reverb_step(D, x, p, L):
    xx = x.detach().requires_grad_(True)
    pp = [q.detach().requires_grad_(True) for q in p]
    y = D.noise_shaped_reverberation(xx, SR, *pp, num_samples=L, num_bandpass_taps=TAPS)
    grads = torch.autograd.grad(y.square().sum(), [xx, *pp])
    return y.detach(), grads[0], torch.stack(grads[1:], 1)


def test_fork_waits_for_work_queued_on_the_callers_stream(cuda_device, monkeypatch):
    """The parameters come from a copy queued behind a long kernel on a non-default current stream; the side streams
    must not start the synthesis before it."""
    import dasp_pytorch_b200 as D
    from dasp_pytorch_b200 import functional as F
    dev = cuda_device
    n, L = rp.default_case(6)
    bs = 6
    gen = torch.Generator().manual_seed(31)
    x = (torch.rand(bs, 2, n, generator=gen) * 2 - 1).to(dev)
    src = torch.rand(25, bs, generator=gen).to(dev)
    monkeypatch.setattr(F, "REVERB_CHUNK_ITEMS", 2)
    s = torch.cuda.Stream(dev)
    s.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(s):
        p = torch.zeros(25, bs, device=dev)
        torch.manual_seed(17)
        torch.cuda.synchronize(dev)
        ref = _reverb_step(D, x, list(src), L)
        torch.cuda._sleep(200_000_000)              # ~0.1 s on the stream, then the parameters are written
        p.copy_(src)
        torch.manual_seed(17)
        got = _reverb_step(D, x, list(p), L)
    torch.cuda.synchronize(dev)
    assert _abi.lib().dasp_debug_reverb_last_path() == 2
    for a, b in zip(got, ref):
        assert torch.equal(a, b)


def test_captured_fwd_bwd_matches_eager(cuda_device):
    """A captured forward + backward over three chunks (pipelined inside the graph) replays what the eager call
    computes after the same manual_seed, and draws new noise on the next replay."""
    import dasp_pytorch_b200 as D
    from dasp_pytorch_b200 import functional as F
    dev = cuda_device
    n, L = rp.default_case(6)
    bs = 6
    gen = torch.Generator().manual_seed(12)
    x = (torch.rand(bs, 2, n, generator=gen) * 2 - 1).to(dev)
    p = [q.to(dev) for q in torch.rand(25, bs, generator=gen)]
    old_chunk = F.REVERB_CHUNK_ITEMS
    F.REVERB_CHUNK_ITEMS = 2
    try:
        torch.manual_seed(8)
        eager = _reverb_step(D, x, p, L)
        assert _abi.lib().dasp_debug_reverb_last_path() == 2
        side = torch.cuda.Stream(dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            _reverb_step(D, x, p, L)
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize(dev)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out = _reverb_step(D, x, p, L)
        torch.manual_seed(8)
        graph.replay()
        torch.cuda.synchronize(dev)
        replay1 = [t.clone() for t in out]
        graph.replay()
        torch.cuda.synchronize(dev)
    finally:
        F.REVERB_CHUNK_ITEMS = old_chunk
    for a, b in zip(replay1, eager):
        assert torch.isfinite(a).all()
        assert torch.equal(a, b)
    assert not torch.equal(out[0], replay1[0])
