"""convolution_reverberation with one impulse response for the whole batch, on the GPU: pinned to the fp64 oracle with
the IR expanded over the batch, equal to today's per-item path with that expansion (bit for bit on the own FFT), the
same bits for every chunk size and run, blind to stale workspace contents, and CUDA-graph safe.  Every case asserts the
path bits it reached (dasp_debug_conv_last_path: bit 1 of the forward and bit 3 of the backward mark the shared IR)."""
import pytest
import torch

import conv_oracle
from helpers import SR, peak_err
from test_gpu_conv_reverb import BOUND, CHANS, SHAPES, _errs, _gpu, _inputs, _lib

pytestmark = pytest.mark.gpu
KB, NFFT = 4096, 8192


def _align(v):
    return (v + 255) // 256 * 256


def _ref_shared(x, ir1, mix, w):
    """fp64 oracle of the shared IR: the oracle with ir1 expanded over the batch, gradient summed by autograd"""
    bs = x.shape[0]
    xx = x.clone().requires_grad_(True)
    hh = ir1.clone().requires_grad_(True)
    mm = mix.clone().requires_grad_(True)
    y = conv_oracle.convolution_reverberation(xx, SR, hh.expand(bs, -1, -1), mm)
    (y * w).sum().backward()
    return y.detach(), xx.grad, hh.grad, mm.grad


def _bits(n, L, ir_grad=True):
    """expected (forward, backward) path bits of a shared call on the own FFT (n % 4 == 0) or the cuFFT pipeline"""
    I, J = -(-n // KB), -(-min(n, L) // KB)
    own = n % 4 == 0
    fused = own and ir_grad and max(I, J) <= 16
    return (1 if own else 0) | 2, (1 if own else 0) | (2 if fused else 0) | (4 if ir_grad else 0) | 8


def _rel_ir(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30))


@pytest.mark.parametrize("in_chs,ir_chs", CHANS, ids=[f"x{a}-ir{b}" for a, b in CHANS])
@pytest.mark.parametrize("n,L", SHAPES, ids=[f"{n}-{L}" for n, L in SHAPES])
def test_conv_shared_pinned_to_oracle_and_per_item_path(cuda_device, monkeypatch, n, L, in_chs, ir_chs):
    """bs 3 in chunks of 2 (a full chunk and a remainder), mix 0 / 1 / random: y, dL/dx, dL/dmix and the summed dL/dIR
    within 1e-4 of the fp64 oracle; against the same call with the IR expanded to a per-item copy, y, dL/dx and dL/dmix
    are the same bits on the own FFT (the IR spectra come from the same kernel and taps) and within 1e-5 on cuFFT"""
    from dasp_pytorch_b200 import functional as F
    monkeypatch.setattr(F, "REVERB_CHUNK_ITEMS", 2)
    x, ir, mix, w = _inputs(3, in_chs, ir_chs, n, L, seed=n + L + 10 * in_chs + ir_chs + 1)
    ir1 = ir[:1]
    got = _gpu(x, ir1, mix, w, cuda_device)
    lib = _lib()
    assert (lib.dasp_debug_conv_last_path(0), lib.dasp_debug_conv_last_path(1)) == _bits(n, L)
    assert got[2].shape == (1, ir_chs, L) and got[1].shape == (3, in_chs, n)
    if L > n:
        assert bool((got[2][..., n:] == 0).all())              # taps >= n reach no output
    errs = _errs(got, _ref_shared(x, ir1, mix, w))
    for k, e in errs.items():
        assert float(e.max()) < BOUND, (k, e)

    per = _gpu(x, ir1.expand(3, -1, -1).contiguous(), mix, w, cuda_device)
    assert lib.dasp_debug_conv_last_path(0) & 2 == 0 and lib.dasp_debug_conv_last_path(1) & 8 == 0
    if n % 4 == 0:
        for i in (0, 1, 3):
            assert torch.equal(got[i], per[i]), i
    else:
        for i, tol in ((0, 1e-5), (1, 1e-5), (3, BOUND)):   # dL/dmix sums 2n largely cancelling products
            assert float(peak_err(got[i], per[i]).max()) < tol, i
    e_sum = _rel_ir(got[2], per[2].double().sum(0, keepdim=True))
    assert e_sum < 1e-5
    print(f"SHARED {n}-{L} x{in_chs} ir{ir_chs}: " + " ".join(f"{k} {float(e.max()):.2e}" for k, e in errs.items())
          + f" dir-vs-expanded {e_sum:.2e}")


def test_conv_shared_geometry_with_a_batch(cuda_device):
    """irspec_c64 is one IR's J partitions; the forward keeps one IR slot, the backward adds the fp64 sum"""
    from dasp_pytorch_b200 import _abi
    lib = _lib()
    bs, n, L, chunk = 5, 48000, 96000, 2
    I, J = -(-n // KB), 12
    g, ref = _abi.ConvGeom(), _abi.ConvGeom()
    _abi.check(lib.dasp_conv_shared_geometry(bs, n, L, chunk, g), "dasp_conv_shared_geometry")
    _abi.check(lib.dasp_conv_geometry(bs, n, L, chunk, ref), "dasp_conv_geometry")
    assert (g.leff, g.x_blocks, g.ir_partitions, g.chunk_items) == (n, I, J, chunk)
    assert g.xspec_c64 == bs * I * NFFT == ref.xspec_c64 and g.irspec_c64 == J * NFFT
    fwd = 2 * _align(8 * chunk * I * NFFT)
    bwd = 2 * _align(8 * chunk * I * NFFT) + _align(8 * chunk * J * NFFT) + _align(4 * chunk * I)
    cufft_ref = ref.fwd_workspace_bytes - fwd - _align(8 * chunk * J * NFFT)
    cufft = g.fwd_workspace_bytes - fwd - _align(8 * J * NFFT)
    assert cufft >= cufft_ref >= 0
    assert g.bwd_workspace_bytes == bwd + _align(16 * J * NFFT) + cufft


@pytest.mark.parametrize("n,L,in_chs,ir_chs", [(20000, 30001, 2, 1), (48000, 30001, 1, 2), (20001, 26000, 2, 2)])
def test_conv_shared_chunking_and_runs_are_bit_identical(cuda_device, monkeypatch, n, L, in_chs, ir_chs):
    """chunks of 1, 2 and the automatic size, and a repeated run, give the same bits for all four outputs (the fp64
    item sum sees the same additions whatever the chunking), on the own FFT and on cuFFT (n % 4 != 0)"""
    from dasp_pytorch_b200 import functional as F
    x, ir, mix, w = _inputs(5, in_chs, ir_chs, n, L, seed=31)
    runs = []
    for chunk in (1, 2, 0, 0):
        monkeypatch.setattr(F, "REVERB_CHUNK_ITEMS", chunk)
        runs.append(_gpu(x, ir[:1], mix, w, cuda_device))
        assert (_lib().dasp_debug_conv_last_path(0), _lib().dasp_debug_conv_last_path(1)) == _bits(n, L)
    for other in runs[1:]:
        for a, b in zip(runs[0], other):
            assert torch.equal(a, b)


def test_conv_shared_large_batch_pinned_to_oracle(cuda_device, monkeypatch):
    """more items than one automatic chunk holds (two per SM), at a short n: pinned to the oracle, and the same bits
    as chunks of 7"""
    from dasp_pytorch_b200 import functional as F
    bs = F.reverb_chunk_items(cuda_device) + 5
    n, L = 8000, 5000
    x, ir, mix, w = _inputs(bs, 2, 2, n, L, seed=37)
    ir1 = ir[:1]
    got = _gpu(x, ir1, mix, w, cuda_device)
    assert (_lib().dasp_debug_conv_last_path(0), _lib().dasp_debug_conv_last_path(1)) == _bits(n, L)
    errs = _errs(got, _ref_shared(x, ir1, mix, w))
    for k, e in errs.items():
        assert float(e.max()) < BOUND, (k, e)
    monkeypatch.setattr(F, "REVERB_CHUNK_ITEMS", 7)
    for a, b in zip(got, _gpu(x, ir1, mix, w, cuda_device)):
        assert torch.equal(a, b)
    print(f"SHARED bs {bs}: " + " ".join(f"{k} {float(e.max()):.2e}" for k, e in errs.items()))


@pytest.mark.parametrize("n,L,in_chs,ir_chs", [(48000, 30001, 2, 2), (20000, 26000, 1, 1), (20001, 26000, 2, 1)])
def test_conv_shared_ignores_prior_workspace_contents(cuda_device, n, L, in_chs, ir_chs):
    """NaN in both workspaces, in irspec_save and in the output buffers reaches no output: every element read is
    written first, and item 0 writes the gradient sum rather than adding to it"""
    from dasp_pytorch_b200 import _abi
    lib, dev = _lib(), cuda_device
    bs, chunk = 3, 2
    g = _abi.ConvGeom()
    _abi.check(lib.dasp_conv_shared_geometry(bs, n, L, chunk, g), "dasp_conv_shared_geometry")
    assert g.leff % g.conv_block != 0
    x, ir, mix, w = _inputs(bs, in_chs, ir_chs, n, L, seed=41)
    x, ir1, mix, gy = (t.float().to(dev).contiguous() for t in (x, ir[:1], mix, w))

    def filled(numel, dtype, fill):
        t = torch.empty(numel, dtype=dtype, device=dev)
        t.view(torch.float32).fill_(fill)
        return t

    def run(fill, keep=True):
        y = filled(bs * 2 * n, torch.float32, fill)
        ws = filled(g.fwd_workspace_bytes // 4, torch.float32, fill)
        xs = filled(g.xspec_c64, torch.complex64, fill) if keep else None
        hs = filled(g.irspec_c64, torch.complex64, fill) if keep else None
        _abi.check(lib.dasp_conv_shared_fwd(_abi.ptr(x), in_chs, _abi.ptr(ir1), ir_chs, L, _abi.ptr(mix), _abi.ptr(y),
                                            _abi.ptr(xs), _abi.ptr(hs), _abi.ptr(ws), g.fwd_workspace_bytes, bs, n,
                                            chunk, _abi.stream_ptr(dev)), "dasp_conv_shared_fwd")
        assert lib.dasp_debug_conv_last_path(0) == _bits(n, L)[0]
        if not keep:
            torch.cuda.synchronize(dev)
            return (y,)
        wsb = filled(g.bwd_workspace_bytes // 4, torch.float32, fill)
        gx, gir, gmix = (filled(k, torch.float32, fill) for k in (bs * in_chs * n, ir_chs * L, bs))
        _abi.check(lib.dasp_conv_shared_bwd(_abi.ptr(gy), _abi.ptr(x), in_chs, ir_chs, L, _abi.ptr(mix), _abi.ptr(xs),
                                            _abi.ptr(hs), _abi.ptr(gx), _abi.ptr(gir), _abi.ptr(gmix), _abi.ptr(wsb),
                                            g.bwd_workspace_bytes, bs, n, chunk, _abi.stream_ptr(dev)),
                   "dasp_conv_shared_bwd")
        assert lib.dasp_debug_conv_last_path(1) == _bits(n, L)[1]
        torch.cuda.synchronize(dev)
        return y, gx, gir, gmix

    clean = run(0.0)
    for t in clean:
        assert torch.isfinite(t).all()
    for a, b in zip(clean, run(float("nan"))):
        assert torch.equal(a, b)
    assert torch.equal(clean[0], run(float("nan"), keep=False)[0])


@pytest.mark.parametrize("n,L", [(48000, 96000), (70000, 66000), (20001, 26000)])
def test_conv_shared_fixed_ir_skips_ir_gradient(cuda_device, n, L):
    x, ir, mix, w = _inputs(3, 2, 2, n, L, seed=43)
    full = _gpu(x, ir[:1], mix, w, cuda_device)
    assert _lib().dasp_debug_conv_last_path(1) == _bits(n, L)[1]
    skip = _gpu(x, ir[:1], mix, w, cuda_device, ir_grad=False)
    assert _lib().dasp_debug_conv_last_path(1) == _bits(n, L, ir_grad=False)[1]
    assert skip[2] is None
    assert torch.equal(skip[0], full[0]) and torch.equal(skip[1], full[1]) and torch.equal(skip[3], full[3])


def test_conv_shared_cuda_graph_replay_matches_eager(cuda_device):
    import dasp_pytorch_b200 as D
    dev = cuda_device
    x, ir, mix, w = (t.float().to(dev) for t in _inputs(3, 2, 2, 48000, 48000, seed=47))
    ir = ir[:1].clone()
    for t in (x, ir, mix):
        t.requires_grad_(True)

    def step():                                        # returns no tensor that keeps the autograd graph alive
        y = D.convolution_reverberation(x, SR, ir, mix)
        return (y.detach(),) + torch.autograd.grad((y * w).sum(), (x, ir, mix))

    eager = [t.clone() for t in step()]
    assert _lib().dasp_debug_conv_last_path(1) & 8
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
    assert static[2].shape == (1, 2, 48000)
    for a, b in zip(static, eager):
        assert torch.equal(a, b)


def test_conv_batch_of_one_takes_the_per_item_path(cuda_device):
    x, ir, mix, w = _inputs(3, 2, 2, 48000, 30000, seed=53)
    got = _gpu(x[:1], ir[:1], mix[:1], w[:1], cuda_device)
    lib = _lib()
    assert lib.dasp_debug_conv_last_path(0) == 1 and lib.dasp_debug_conv_last_path(1) == 1 | 2 | 4
    assert got[2].shape == (1, 2, 30000)
