"""convolution_reverberation with a true-stereo (four-channel) impulse response on the GPU: pinned to the fp64 oracle
per item and shared over the batch, the own FFT against the cuFFT pipeline, a diagonal IR against the stereo path, the
same bits for every chunk size, blind to stale buffers, a fixed IR, CUDA-graph replay and mix 0.  Every case asserts the
path bits it reached (dasp_debug_conv_last_path: bit 2 of the forward and bit 4 of the backward mark a true-stereo IR)."""
import pytest
import torch

import conv_ts_oracle
from helpers import SR, peak_err
from test_gpu_conv_reverb import BOUND, SHAPES, _errs, _gpu, _inputs, _lib

pytestmark = pytest.mark.gpu
KB, NFFT = 4096, 8192


def _bits(n, L, shared, ir_grad=True, own=None):
    """expected (forward, backward) path bits of a true-stereo call"""
    I, J = -(-n // KB), -(-min(n, L) // KB)
    own = n % 4 == 0 if own is None else own
    fused = own and ir_grad and max(I, J) <= 16
    sh = 1 if shared else 0
    return ((1 if own else 0) | 2 * sh | 4,
            (1 if own else 0) | (2 if fused else 0) | (4 if ir_grad else 0) | 8 * sh | 16)


def _ts_inputs(bs, in_chs, n, L, seed, shared):
    x, ir, mix, w = _inputs(bs, in_chs, 4, n, L, seed)
    return x, (ir[:1] if shared else ir), mix, w


def _ref(x, ir, mix, w):
    bs = x.shape[0]
    xx = x.clone().requires_grad_(True)
    hh = ir.clone().requires_grad_(True)
    mm = mix.clone().requires_grad_(True)
    y = conv_ts_oracle.convolution_reverberation(xx, SR, hh.expand(bs, -1, -1), mm)
    (y * w).sum().backward()
    return y.detach(), xx.grad, hh.grad, mm.grad


def _path():
    lib = _lib()
    return lib.dasp_debug_conv_last_path(0), lib.dasp_debug_conv_last_path(1)


@pytest.mark.parametrize("shared", [False, True], ids=["item", "shared"])
@pytest.mark.parametrize("in_chs", [2, 1], ids=["x2", "x1"])
@pytest.mark.parametrize("n,L", SHAPES, ids=[f"{n}-{L}" for n, L in SHAPES])
def test_conv_ts_pinned_to_oracle(cuda_device, monkeypatch, n, L, in_chs, shared):
    """bs 3 in chunks of 2, mix 0 / 1 / random: y, dL/dx, dL/dIR (all four channels) and dL/dmix within 1e-4 of the fp64
    oracle; I = 18 runs the generic MAC and the unfused correlations, n = 1001 the cuFFT pipeline"""
    from dasp_pytorch_b200 import functional as F
    monkeypatch.setattr(F, "REVERB_CHUNK_ITEMS", 2)
    x, ir, mix, w = _ts_inputs(3, in_chs, n, L, seed=n + L + 10 * in_chs + 4 + shared, shared=shared)
    got = _gpu(x, ir, mix, w, cuda_device)
    assert _path() == _bits(n, L, shared)
    assert got[2].shape == ir.shape and got[1].shape == (3, in_chs, n)
    if L > n:
        assert bool((got[2][..., n:] == 0).all())              # taps >= n reach no output
    if not shared:
        assert float(got[2][0].abs().max()) == 0.0              # mix 0
    errs = _errs(got, _ref(x, ir, mix, w))
    for k, e in errs.items():
        assert float(e.max()) < BOUND, (k, e)
    print(f"TS {n}-{L} x{in_chs} {'shared' if shared else 'item'}: "
          + " ".join(f"{k} {float(e.max()):.2e}" for k, e in errs.items()))


@pytest.mark.parametrize("n,L,in_chs,shared", [(48000, 30001, 2, False), (20000, 26000, 1, False),
                                               (70000, 66000, 2, False), (48000, 30001, 2, True)])
def test_conv_ts_cufft_path_agrees_with_default(cuda_device, n, L, in_chs, shared):
    x, ir, mix, w = _ts_inputs(3, in_chs, n, L, seed=73, shared=shared)
    lib = _lib()
    own = _gpu(x, ir, mix, w, cuda_device)
    assert _path() == _bits(n, L, shared)
    lib.dasp_debug_reverb_path(1)
    try:
        cu = _gpu(x, ir, mix, w, cuda_device)
        assert _path() == _bits(n, L, shared, own=False)
    finally:
        lib.dasp_debug_reverb_path(0)
    # dL/dmix sums 2n products that largely cancel, so its rounding relative to its value is larger than the others'
    for a, b, tol in zip(own, cu, (1e-5, 1e-5, 1e-5, BOUND)):
        assert float(peak_err(a, b).max()) < tol
    assert torch.equal(cu[2][..., min(n, L):], torch.zeros_like(cu[2][..., min(n, L):]))


@pytest.mark.parametrize("n,L,in_chs,shared", [(48000, 48000, 2, False), (48000, 96000, 1, False),
                                               (70000, 66000, 2, False), (1001, 500, 2, False),
                                               (20000, 30001, 2, True)])
def test_conv_ts_diagonal_ir_matches_the_stereo_path(cuda_device, n, L, in_chs, shared):
    """(hL, 0, 0, hR) against today's stereo call with (hL, hR): y and dL/dx within 1e-6, dL/dIR channels 0 and 3
    against the stereo call's channels 0 and 1 within 1e-6 of their peak, and dL/dmix within 1e-5 (it sums 2n products
    that largely cancel, so the last-bit differences of the two products' dL/dx windows weigh more in it; up to 3.7e-6
    seen on an H100)"""
    x, h, mix, w = _inputs(3, in_chs, 2, n, L, seed=79)
    if shared:
        h = h[:1]
    z = torch.zeros_like(h[:, :1])
    ts = _gpu(x, torch.cat([h[:, :1], z, z, h[:, 1:]], dim=1), mix, w, cuda_device)
    assert _path() == _bits(n, L, shared)
    st = _gpu(x, h, mix, w, cuda_device)
    assert _lib().dasp_debug_conv_last_path(0) & 4 == 0 and _lib().dasp_debug_conv_last_path(1) & 16 == 0
    for i, tol in ((0, 1e-6), (1, 1e-6), (3, 1e-5)):
        assert float(peak_err(ts[i], st[i]).max()) < tol, i
    scale = st[2].abs().amax().clamp_min(1e-30)
    for c_ts, c_st in ((0, 0), (3, 1)):
        assert float((ts[2][:, c_ts] - st[2][:, c_st]).abs().max() / scale) < 1e-6, c_ts


@pytest.mark.parametrize("n,L,in_chs", [(20000, 30001, 2), (48000, 30001, 1), (20001, 26000, 2)])
def test_conv_ts_shared_chunking_and_runs_are_bit_identical(cuda_device, monkeypatch, n, L, in_chs):
    from dasp_pytorch_b200 import functional as F
    x, ir, mix, w = _ts_inputs(5, in_chs, n, L, seed=83, shared=True)
    runs = []
    for chunk in (1, 2, 0, 0):
        monkeypatch.setattr(F, "REVERB_CHUNK_ITEMS", chunk)
        runs.append(_gpu(x, ir, mix, w, cuda_device))
        assert _path() == _bits(n, L, True)
    for other in runs[1:]:
        for a, b in zip(runs[0], other):
            assert torch.equal(a, b)


def test_conv_ts_geometry_with_a_batch(cuda_device):
    """irspec_c64 holds 2 J partitions per IR (one IR when shared)"""
    from dasp_pytorch_b200 import _abi
    lib = _lib()
    bs, n, L, chunk = 5, 48000, 96000, 2
    J = 12
    for fn, per in ((lib.dasp_conv_ts_geometry, bs), (lib.dasp_conv_shared_ts_geometry, 1)):
        g = _abi.ConvGeom()
        _abi.check(fn(bs, n, L, chunk, g), "ts geometry")
        assert g.ir_partitions == J and g.irspec_c64 == per * 2 * J * NFFT


@pytest.mark.parametrize("n,L,in_chs,shared", [(48000, 30001, 2, False), (20000, 26000, 1, True),
                                               (20001, 26000, 2, False), (20001, 26000, 1, True)])
def test_conv_ts_ignores_prior_buffer_contents(cuda_device, n, L, in_chs, shared):
    """NaN in both workspaces, in irspec_save (set B's slots included) and in the outputs reaches no result"""
    from dasp_pytorch_b200 import _abi
    lib, dev = _lib(), cuda_device
    bs, chunk = 3, 2
    g = _abi.ConvGeom()
    _abi.check((lib.dasp_conv_shared_ts_geometry if shared else lib.dasp_conv_ts_geometry)(bs, n, L, chunk, g), "geom")
    assert g.leff % g.conv_block != 0
    fwd, bwd = (lib.dasp_conv_shared_fwd, lib.dasp_conv_shared_bwd) if shared else (lib.dasp_conv_fwd, lib.dasp_conv_bwd)
    x, ir, mix, w = _ts_inputs(bs, in_chs, n, L, seed=89, shared=shared)
    x, ir, mix, gy = (t.float().to(dev).contiguous() for t in (x, ir, mix, w))

    def filled(numel, dtype, fill):
        t = torch.empty(numel, dtype=dtype, device=dev)
        t.view(torch.float32).fill_(fill)
        return t

    def run(fill, keep=True):
        y = filled(bs * 2 * n, torch.float32, fill)
        ws = filled(g.fwd_workspace_bytes // 4, torch.float32, fill)
        xs = filled(g.xspec_c64, torch.complex64, fill) if keep else None
        hs = filled(g.irspec_c64, torch.complex64, fill) if keep else None
        _abi.check(fwd(_abi.ptr(x), in_chs, _abi.ptr(ir), 4, L, _abi.ptr(mix), _abi.ptr(y), _abi.ptr(xs), _abi.ptr(hs),
                       _abi.ptr(ws), g.fwd_workspace_bytes, bs, n, chunk, _abi.stream_ptr(dev)), "fwd")
        assert lib.dasp_debug_conv_last_path(0) == _bits(n, L, shared)[0]
        if not keep:
            torch.cuda.synchronize(dev)
            return (y,)
        wsb = filled(g.bwd_workspace_bytes // 4, torch.float32, fill)
        gx, gir, gmix = (filled(k, torch.float32, fill) for k in (bs * in_chs * n, ir.numel(), bs))
        _abi.check(bwd(_abi.ptr(gy), _abi.ptr(x), in_chs, 4, L, _abi.ptr(mix), _abi.ptr(xs), _abi.ptr(hs), _abi.ptr(gx),
                       _abi.ptr(gir), _abi.ptr(gmix), _abi.ptr(wsb), g.bwd_workspace_bytes, bs, n, chunk,
                       _abi.stream_ptr(dev)), "bwd")
        assert lib.dasp_debug_conv_last_path(1) == _bits(n, L, shared)[1]
        torch.cuda.synchronize(dev)
        return y, gx, gir, gmix

    clean = run(0.0)
    for t in clean:
        assert torch.isfinite(t).all()
    for a, b in zip(clean, run(float("nan"))):
        assert torch.equal(a, b)
    assert torch.equal(clean[0], run(float("nan"), keep=False)[0])


@pytest.mark.parametrize("n,L,shared", [(48000, 96000, False), (70000, 66000, False), (20001, 26000, False),
                                        (48000, 96000, True)])
def test_conv_ts_fixed_ir_skips_ir_gradient(cuda_device, n, L, shared):
    x, ir, mix, w = _ts_inputs(3, 2, n, L, seed=97, shared=shared)
    full = _gpu(x, ir, mix, w, cuda_device)
    assert _path()[1] == _bits(n, L, shared)[1]
    skip = _gpu(x, ir, mix, w, cuda_device, ir_grad=False)
    assert _path()[1] == _bits(n, L, shared, ir_grad=False)[1]
    assert skip[2] is None
    assert torch.equal(skip[0], full[0]) and torch.equal(skip[1], full[1]) and torch.equal(skip[3], full[3])


@pytest.mark.parametrize("shared", [False, True], ids=["item", "shared"])
def test_conv_ts_cuda_graph_replay_matches_eager(cuda_device, shared):
    import dasp_pytorch_b200 as D
    dev = cuda_device
    x, ir, mix, w = (t.float().to(dev) for t in _ts_inputs(3, 2, 48000, 48000, seed=101, shared=shared))
    ir = ir.clone()
    for t in (x, ir, mix):
        t.requires_grad_(True)

    def step():                                        # returns no tensor that keeps the autograd graph alive
        y = D.convolution_reverberation(x, SR, ir, mix)
        return (y.detach(),) + torch.autograd.grad((y * w).sum(), (x, ir, mix))

    eager = [t.clone() for t in step()]
    assert _path() == _bits(48000, 48000, shared)
    s = torch.cuda.Stream(dev)
    s.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(s):
        for _ in range(2):
            step()
    torch.cuda.current_stream(dev).wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static = step()
    graph.replay()
    torch.cuda.synchronize(dev)
    assert static[2].shape == ir.shape
    for a, b in zip(static, eager):
        assert torch.equal(a, b)


@pytest.mark.parametrize("n,L", [(48000, 30001), (20001, 26000)])
@pytest.mark.parametrize("shared", [False, True], ids=["item", "shared"])
def test_conv_ts_mix0_gives_a_zero_ir_gradient(cuda_device, n, L, shared):
    x, ir, _, w = _ts_inputs(3, 2, n, L, seed=103, shared=shared)
    got = _gpu(x, ir, torch.zeros(3, dtype=torch.float64), w, cuda_device)
    assert _path() == _bits(n, L, shared)
    assert torch.equal(got[2], torch.zeros_like(got[2]))
    assert torch.equal(got[0], x.float().expand(3, 2, n) if x.shape[1] == 2 else x.float().repeat(1, 2, 1))
