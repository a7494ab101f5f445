"""The default device-noise IR synthesis for R <= 8 (ir_synth_cluster_kernel: persistent clusters of R CTAs, generator
and inverse FFT in one kernel) against the two-kernel synthesis (spectral_gen_kernel -> ifft_shape_kernel, selected with
dasp_debug_reverb_path(2)).  Both draw the same spectrum and run the same transform and epilogue, so the IR partitions,
the saved filtered noise f, y and the gradients must agree bit for bit.

Each case uses two chunks whose first holds more items than the device co-schedules clusters of R CTAs (so clusters
loop over items) and whose second holds 7, with leff % 4096 != 0."""
from types import SimpleNamespace

import pytest
import torch

import reverb_pin as rp
from dasp_pytorch_b200 import _abi
from helpers import SR

pytestmark = pytest.mark.gpu
TAPS = 1023


def _run(dev, x, params, L, chunk, path, fill):
    """raw forward + backward with f_save and the workspaces prefilled with `fill`; returns
    (last path, y, IR partition spectra, f_save, dL/dx, dL/dparams, geometry)"""
    lib = _abi.lib()
    bs, in_chs, n = x.shape
    g = _abi.ReverbGeom()
    _abi.check(lib.dasp_reverb_geometry(bs, n, L, TAPS, chunk, g), "dasp_reverb_geometry")
    seed = torch.tensor([4321], dtype=torch.int64, device=dev)
    y = torch.empty(bs, 2, n, device=dev)
    fsave = torch.full((g.f_floats,), fill, device=dev)
    xspec = torch.empty(g.xspec_c64, dtype=torch.complex64, device=dev)
    irspec = torch.empty(g.irspec_c64, dtype=torch.complex64, device=dev)
    ws = torch.full((g.fwd_workspace_bytes // 4,), fill, device=dev)
    lib.dasp_debug_reverb_path(path)
    try:
        _abi.check(lib.dasp_reverb_fwd(_abi.ptr(x), in_chs, _abi.ptr(params), None, _abi.ptr(seed), _abi.ptr(y),
                                       _abi.ptr(fsave), _abi.ptr(xspec), _abi.ptr(irspec), _abi.ptr(ws), ws.numel() * 4,
                                       bs, n, L, TAPS, chunk, float(SR), _abi.stream_ptr(dev)), "dasp_reverb_fwd")
        used = lib.dasp_debug_reverb_last_path()
    finally:
        lib.dasp_debug_reverb_path(0)
    gy = torch.sin(torch.arange(bs * 2 * n, device=dev, dtype=torch.float32) * 0.01).reshape(bs, 2, n)
    gx = torch.empty_like(x)
    gp = torch.empty_like(params)
    wsb = torch.full((g.bwd_workspace_bytes // 4 + 1,), fill, device=dev)
    _abi.check(lib.dasp_reverb_bwd(_abi.ptr(gy), _abi.ptr(x), in_chs, _abi.ptr(params), _abi.ptr(fsave), _abi.ptr(xspec),
                                   _abi.ptr(irspec), _abi.ptr(gx), _abi.ptr(gp), _abi.ptr(wsb), wsb.numel() * 4, bs, n, L,
                                   TAPS, chunk, 1, _abi.stream_ptr(dev)), "dasp_reverb_bwd")
    torch.cuda.synchronize(dev)
    return used, y, torch.view_as_real(irspec), fsave, gx, gp, g


@pytest.mark.parametrize("in_chs", [1, 2])
@pytest.mark.parametrize("R", range(1, 7))
def test_cluster_synthesis_matches_two_kernel_path(cuda_device, R, in_chs):
    dev = cuda_device
    n, L = rp.default_case(R)
    chunk = 140 // R + 5                      # more items than the H100 co-schedules clusters of R CTAs
    bs = chunk + 7
    gen = torch.Generator().manual_seed(100 + R)
    x = (torch.rand(bs, in_chs, n, generator=gen) * 2 - 1).to(dev)
    params = torch.rand(bs, 25, generator=gen).to(dev)

    used0, y0, h0, f0, gx0, gp0, g = _run(dev, x, params, L, chunk, 0, float("nan"))
    used1, y1, h1, f1, gx1, gp1, _ = _run(dev, x, params, L, chunk, 2, 0.0)
    assert g.rpp == R and g.nb == 8192 and g.leff % g.conv_block != 0
    assert (used0, used1) == (2, 1)
    # every slot of the polyphase f layout the backward reads was written, over a NaN prefill
    geom = SimpleNamespace(rpp=g.rpp, nbk=g.nbk, nb=g.nb, chunk_items=g.chunk_items)
    for i in range(bs):
        assert torch.isfinite(torch.view_as_real(rp.item_blocks(f0, i, geom))).all(), i
        assert torch.equal(rp.item_blocks(f0, i, geom), rp.item_blocks(f1, i, geom)), i
    assert torch.isfinite(y0).all() and torch.isfinite(gx0).all() and torch.isfinite(gp0).all()
    assert torch.equal(h0, h1)
    assert torch.equal(y0, y1)
    assert torch.equal(gx0, gx1) and torch.equal(gp0, gp1)


def test_cluster_synthesis_graph_replay_matches_eager(cuda_device):
    import dasp_pytorch_b200 as D
    from dasp_pytorch_b200 import functional as F
    dev = cuda_device
    n, L = rp.default_case(6)
    bs = 3
    gen = torch.Generator().manual_seed(9)
    x = (torch.rand(bs, 2, n, generator=gen) * 2 - 1).to(dev)
    p = [q.to(dev) for q in torch.rand(25, bs, generator=gen)]

    def f():
        return D.noise_shaped_reverberation(x, SR, *p, num_samples=L, num_bandpass_taps=TAPS)

    old_chunk = F.REVERB_CHUNK_ITEMS
    F.REVERB_CHUNK_ITEMS = 2                  # two chunks inside the graph
    try:
        torch.manual_seed(5)
        y_eager = f()
        assert _abi.lib().dasp_debug_reverb_last_path() == 2
        side = torch.cuda.Stream(dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            f()
        torch.cuda.current_stream(dev).wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            y_graph = f()
        torch.manual_seed(5)
        graph.replay()
        torch.cuda.synchronize(dev)
    finally:
        F.REVERB_CHUNK_ITEMS = old_chunk
    assert torch.isfinite(y_eager).all()
    assert torch.equal(y_graph, y_eager)
