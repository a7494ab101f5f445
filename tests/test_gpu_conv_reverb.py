"""convolution_reverberation on the GPU, pinned to the fp64 oracle (tests/conv_oracle.py) per item with the SURVEY.md 8c
metric: y, dL/dx, dL/dIR (relative to the item's largest fp64 IR gradient) and dL/dmix within 1e-4, on every path the
convolution dispatches to; plus the path-independence, workspace, skip, chunking and graph-capture properties."""
import pytest
import torch

import conv_oracle
import oracle
from helpers import SR, peak_err

pytestmark = pytest.mark.gpu
BOUND = 1e-4

# (n, L): L < n, = n, > n, a single tap, one partition, k * 4096 + 1, I = 18 (generic MAC, unfused correlations),
# n % 4 != 0 (cuFFT pipeline)
SHAPES = [(48000, 48000), (48000, 96000), (48000, 1), (4096, 4096), (6000, 4097), (20000, 30001), (70000, 66000),
          (1001, 500)]
CHANS = [(2, 2), (1, 2), (2, 1), (1, 1)]               # (x channels, IR channels)


def _inputs(bs, in_chs, ir_chs, n, L, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(bs, in_chs, n, generator=g, dtype=torch.float64) * 2 - 1
    ir = (torch.rand(bs, ir_chs, L, generator=g, dtype=torch.float64) * 2 - 1) * torch.exp(
        -torch.arange(L, dtype=torch.float64) / max(L / 4, 1.0))
    mix = torch.rand(bs, generator=g, dtype=torch.float64)
    mix[0], mix[1] = 0.0, 1.0                            # item 0 dry only, item 1 wet only, item 2 random
    w = torch.rand(bs, 2, n, generator=g, dtype=torch.float64) * 2 - 1     # loss = sum(w y)
    return x, ir, mix, w


def _run(fn, x, ir, mix, w, device, dtype, ir_grad=True):
    xx = x.to(device=device, dtype=dtype).requires_grad_(True)
    hh = ir.to(device=device, dtype=dtype).requires_grad_(ir_grad)
    mm = mix.to(device=device, dtype=dtype).requires_grad_(True)
    y = fn(xx, SR, hh, mm)
    (y * w.to(device=device, dtype=dtype)).sum().backward()
    return (y.detach().cpu(), xx.grad.cpu(), None if hh.grad is None else hh.grad.cpu(), mm.grad.cpu())


def _gpu(x, ir, mix, w, dev, **kw):
    import dasp_pytorch_b200 as D
    return _run(D.convolution_reverberation, x, ir, mix, w, dev, torch.float32, **kw)


def _ref(x, ir, mix, w):
    return _run(conv_oracle.convolution_reverberation, x, ir, mix, w, "cpu", torch.float64)


def _errs(got, ref):
    y, dx, dir_, dm = got
    ry, rdx, rdir, rdm = ref
    e_ir = (dir_.double() - rdir).reshape(len(rdir), -1).abs().amax(1)
    scale = rdir.reshape(len(rdir), -1).abs().amax(1)
    e_ir = torch.where(scale > 0, e_ir / scale.clamp_min(1e-300), e_ir)      # mix 0: the gradient must be exactly 0
    e_m = (dm.double() - rdm).abs() / rdm.abs().clamp_min(1e-30)
    return {"y": peak_err(y, ry), "dx": peak_err(dx, rdx), "dir": e_ir, "dmix": e_m}


def _lib():
    from dasp_pytorch_b200 import _abi
    return _abi.lib()


@pytest.mark.parametrize("in_chs,ir_chs", CHANS, ids=[f"x{a}-ir{b}" for a, b in CHANS])
@pytest.mark.parametrize("n,L", SHAPES, ids=[f"{n}-{L}" for n, L in SHAPES])
def test_conv_reverb_pinned_to_oracle(cuda_device, monkeypatch, n, L, in_chs, ir_chs):
    from dasp_pytorch_b200 import functional as F
    monkeypatch.setattr(F, "REVERB_CHUNK_ITEMS", 2)          # bs 3: a full chunk and a remainder
    x, ir, mix, w = _inputs(3, in_chs, ir_chs, n, L, seed=n + L + 10 * in_chs + ir_chs)
    got = _gpu(x, ir, mix, w, cuda_device)
    I, J = -(-n // 4096), -(-min(n, L) // 4096)
    own = n % 4 == 0
    assert _lib().dasp_debug_conv_last_path(0) == (1 if own else 0)
    assert _lib().dasp_debug_conv_last_path(1) == (1 if own else 0) | (2 if own and max(I, J) <= 16 else 0) | 4
    errs = _errs(got, _ref(x, ir, mix, w))
    assert got[2].shape == (3, ir_chs, L) and got[1].shape == (3, in_chs, n)
    if L > n:
        assert bool((got[2][..., n:] == 0).all())              # taps >= n reach no output
    assert float(got[2][0].abs().max()) == 0.0                  # mix 0
    for k, e in errs.items():
        assert float(e.max()) < BOUND, (k, e)
    print(f"CONV {n}-{L} x{in_chs} ir{ir_chs}: " + " ".join(f"{k} {float(e.max()):.2e}" for k, e in errs.items()))


@pytest.mark.parametrize("n,L,in_chs,ir_chs", [(48000, 30001, 2, 2), (20000, 26000, 1, 1), (70000, 66000, 2, 1)])
def test_conv_cufft_path_agrees_with_default(cuda_device, n, L, in_chs, ir_chs):
    x, ir, mix, w = _inputs(3, in_chs, ir_chs, n, L, seed=7)
    lib = _lib()
    own = _gpu(x, ir, mix, w, cuda_device)
    assert lib.dasp_debug_conv_last_path(0) == 1 and lib.dasp_debug_conv_last_path(1) & 1
    lib.dasp_debug_reverb_path(1)
    try:
        cu = _gpu(x, ir, mix, w, cuda_device)
        assert lib.dasp_debug_conv_last_path(0) == 0 and lib.dasp_debug_conv_last_path(1) == 4
    finally:
        lib.dasp_debug_reverb_path(0)
    # dL/dmix sums 2n products that largely cancel, so its rounding relative to its value is larger than the others'
    for a, b, tol in zip(own, cu, (1e-5, 1e-5, 1e-5, BOUND)):
        assert float(peak_err(a, b).max()) < tol
    assert torch.equal(cu[2][..., min(n, L):], torch.zeros_like(cu[2][..., min(n, L):]))


@pytest.mark.parametrize("n,L,in_chs,ir_chs", [(48000, 30001, 2, 2), (20000, 26000, 1, 1), (20000, 26000, 2, 1)])
def test_conv_fwd_ignores_prior_workspace_contents(cuda_device, n, L, in_chs, ir_chs):
    """the partition slots are never zero-filled: NaN in the workspace and in irspec_save must not reach y or the spectra"""
    from dasp_pytorch_b200 import _abi
    lib, dev = _lib(), cuda_device
    bs, chunk = 3, 2
    g = _abi.ConvGeom()
    _abi.check(lib.dasp_conv_geometry(bs, n, L, chunk, g), "dasp_conv_geometry")
    assert g.leff % g.conv_block != 0
    x, ir, mix, _ = _inputs(bs, in_chs, ir_chs, n, L, seed=5)
    x, ir, mix = (t.float().to(dev).contiguous() for t in (x, ir, mix))

    def run(fill, keep):
        y = torch.empty(bs, 2, n, device=dev)
        ws = torch.empty(g.fwd_workspace_bytes, dtype=torch.uint8, device=dev)
        ws.view(torch.float32)[: g.fwd_workspace_bytes // 4].fill_(fill)
        xs = hs = None
        if keep:
            xs = torch.empty(g.xspec_c64, dtype=torch.complex64, device=dev)
            hs = torch.empty(g.irspec_c64, dtype=torch.complex64, device=dev)
            hs.view(torch.float32).fill_(fill)
        _abi.check(lib.dasp_conv_fwd(_abi.ptr(x), in_chs, _abi.ptr(ir), ir_chs, L, _abi.ptr(mix), _abi.ptr(y),
                                     _abi.ptr(xs), _abi.ptr(hs), _abi.ptr(ws), ws.numel(), bs, n, chunk,
                                     _abi.stream_ptr(dev)), "dasp_conv_fwd")
        torch.cuda.synchronize(dev)
        assert lib.dasp_debug_conv_last_path(0) == 1
        return y, xs, hs

    y0, x0, h0 = run(0.0, True)
    y1, x1, h1 = run(float("nan"), True)
    y2, _, _ = run(float("nan"), False)
    assert torch.isfinite(y0).all() and torch.isfinite(torch.view_as_real(h0)).all()
    assert torch.equal(y0, y1) and torch.equal(y0, y2)
    assert torch.equal(torch.view_as_real(h0), torch.view_as_real(h1))
    assert torch.equal(torch.view_as_real(x0), torch.view_as_real(x1))


@pytest.mark.parametrize("n,L", [(48000, 96000), (70000, 66000)])
def test_conv_fixed_ir_skips_ir_gradient(cuda_device, n, L):
    x, ir, mix, w = _inputs(3, 2, 2, n, L, seed=11)
    full = _gpu(x, ir, mix, w, cuda_device)
    assert _lib().dasp_debug_conv_last_path(1) & 4
    skip = _gpu(x, ir, mix, w, cuda_device, ir_grad=False)
    assert _lib().dasp_debug_conv_last_path(1) == 1            # own FFT, dL/dx windows only
    assert skip[2] is None
    assert torch.equal(skip[0], full[0]) and torch.equal(skip[1], full[1]) and torch.equal(skip[3], full[3])


def test_conv_chunking_is_bit_identical(cuda_device, monkeypatch):
    from dasp_pytorch_b200 import functional as F
    x, ir, mix, w = _inputs(5, 2, 1, 20000, 30001, seed=13)
    runs = []
    for chunk in (1, 2, 0):
        monkeypatch.setattr(F, "REVERB_CHUNK_ITEMS", chunk)
        runs.append(_gpu(x, ir, mix, w, cuda_device))
    for other in runs[1:]:
        for a, b in zip(runs[0], other):
            assert torch.equal(a, b)


def test_conv_cuda_graph_replay_matches_eager(cuda_device):
    import dasp_pytorch_b200 as D
    dev = cuda_device
    x, ir, mix, w = (t.float().to(dev) for t in _inputs(3, 2, 2, 48000, 48000, seed=17))
    x.requires_grad_(True)
    ir.requires_grad_(True)
    mix.requires_grad_(True)

    def step():                                        # returns no tensor that keeps the autograd graph alive
        y = D.convolution_reverberation(x, SR, ir, mix)
        return (y.detach(),) + torch.autograd.grad((y * w).sum(), (x, ir, mix))

    eager = [t.clone() for t in step()]
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
    for a, b in zip(static, eager):
        assert torch.equal(a, b)


def test_conv_composes_with_the_reverb(cuda_device):
    """noise_shaped_reverberation with a noise tensor N and convolution_reverberation with the oracle's IR from N are
    both the oracle's reverb"""
    import dasp_pytorch_b200 as D
    bs, n, L, taps = 2, 6000, 4000, 255
    gen = torch.Generator().manual_seed(19)
    x = torch.rand(bs, 2, n, generator=gen, dtype=torch.float64) * 2 - 1
    p = [q.clone() for q in torch.rand(bs, 25, generator=gen, dtype=torch.float64).unbind(1)]
    noise = oracle.reverb_noise(bs, L, taps, seed=23)
    ref = oracle.noise_shaped_reverberation(x, SR, *p, num_samples=L, num_bandpass_taps=taps, noise=noise)
    ir = conv_oracle.reverb_ir(SR, p, noise, L, taps)
    f = lambda t: t.float().to(cuda_device)
    y_rev = D.noise_shaped_reverberation(f(x), SR, *[f(q) for q in p], num_samples=L, num_bandpass_taps=taps,
                                         noise=f(noise)).cpu()
    y_conv = D.convolution_reverberation(f(x), SR, f(ir), f(p[24])).cpu()
    assert float(peak_err(y_rev, ref).max()) < BOUND
    assert float(peak_err(y_conv, ref).max()) < BOUND
