"""convolution_bus on the GPU: y, dL/dx and dL/dIR pinned to the fp64 oracle (tests/conv_bus_oracle.py) per item for
1 to 16 inputs, mono and stereo buses, per-item and shared IRs, every length class and several chunks; the identities
with convolution_reverberation and with the op's own single-source calls; the same bits for every chunk size, a fixed IR,
stale buffers, CUDA-graph replay and bf16.  Every case asserts the path bits it reached (dasp_debug_conv_bus_last_path)."""
import pytest
import torch

import conv_bus_oracle
from helpers import SR, peak_err

pytestmark = pytest.mark.gpu
BOUND = 1e-4
KB = 4096

# (n, L): L < n, L = n at a partition multiple, L > n, n % 4 = 1, 2, 3 (padded rows; L > n there too), I = 18 / J = 17
# (products from L2)
SHAPES = [(48000, 30000), (8192, 8192), (6000, 9001), (20001, 12000), (7002, 7002), (9003, 20000), (70000, 66000)]
SO = [(1, 1), (1, 2), (2, 1), (2, 2), (3, 1), (3, 2), (5, 1), (5, 2), (8, 1), (8, 2), (16, 1), (16, 2)]
CASES = [(S, O, *SHAPES[(3 * i + sh) % len(SHAPES)], bool(sh)) for i, (S, O) in enumerate(SO) for sh in (0, 1)]
CASES += [(3, 2, 70000, 66000, False), (16, 1, 70000, 66000, True)]


def _lib():
    from dasp_pytorch_b200 import _abi
    return _abi.lib()


def _bits(n, L, shared, ir_grad=True):
    """expected (forward, backward) path bits"""
    I, J = -(-n // KB), -(-min(n, L) // KB)
    cached = max(I, J) <= 16
    return (1 | (2 if shared else 0) | (4 if cached else 0),
            1 | (2 if cached else 0) | (4 if ir_grad else 0) | (8 if shared else 0))


def _path():
    lib = _lib()
    return lib.dasp_debug_conv_bus_last_path(0), lib.dasp_debug_conv_bus_last_path(1)


def _inputs(bs, S, O, n, L, seed, shared):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(bs, S, n, generator=g, dtype=torch.float64) * 2 - 1
    ir = (torch.rand(1 if shared else bs, S, O, L, generator=g, dtype=torch.float64) * 2 - 1) * torch.exp(
        -torch.arange(L, dtype=torch.float64) / max(L / 4, 1.0))
    w = torch.rand(bs, O, n, generator=g, dtype=torch.float64) * 2 - 1          # loss = sum(w y)
    return x, ir, w


def _run(fn, x, ir, w, device, dtype, ir_grad=True):
    xx = x.to(device=device, dtype=dtype).requires_grad_(True)
    hh = ir.to(device=device, dtype=dtype).requires_grad_(ir_grad)
    y = fn(xx, hh)
    (y * w.to(device=device, dtype=dtype)).sum().backward()
    return y.detach().cpu(), xx.grad.cpu(), None if hh.grad is None else hh.grad.cpu()


def _gpu(x, ir, w, dev, **kw):
    import dasp_pytorch_b200 as D
    return _run(lambda a, h: D.convolution_bus(a, SR, h), x, ir, w, dev, torch.float32, **kw)


def _ref(x, ir, w):
    return _run(lambda a, h: conv_bus_oracle.convolution_bus(a, SR, h), x, ir, w, "cpu", torch.float64)


def _errs(got, ref):
    e_ir = (got[2].double() - ref[2]).reshape(len(ref[2]), -1).abs().amax(1) / ref[2].reshape(
        len(ref[2]), -1).abs().amax(1)
    return {"y": peak_err(got[0], ref[0]), "dx": peak_err(got[1], ref[1]), "dir": e_ir}


@pytest.mark.parametrize("S,O,n,L,shared", CASES, ids=[f"S{c[0]}-O{c[1]}-{c[2]}-{c[3]}-{'sh' if c[4] else 'it'}"
                                                         for c in CASES])
def test_bus_pinned_to_oracle(cuda_device, monkeypatch, S, O, n, L, shared):
    """bs 3 in chunks of 2: y, dL/dx and dL/dIR (relative to the item's, or the shared IR's, largest fp64 gradient)
    within 1e-4 of the fp64 oracle; taps >= n get exactly 0"""
    from dasp_pytorch_b200 import functional as F
    monkeypatch.setattr(F, "REVERB_CHUNK_ITEMS", 2)
    x, ir, w = _inputs(3, S, O, n, L, seed=S * 100 + O * 10 + n % 97 + shared, shared=shared)
    got = _gpu(x, ir, w, cuda_device)
    assert _path() == _bits(n, L, shared)
    assert got[0].shape == (3, O, n) and got[1].shape == x.shape and got[2].shape == ir.shape
    if L > n:
        assert bool((got[2][..., n:] == 0).all())
    errs = _errs(got, _ref(x, ir, w))
    for k, e in errs.items():
        assert float(e.max()) < BOUND, (k, e)
    print(f"bus S{S} O{O} {n}-{L} {'shared' if shared else 'item'}: "
          + " ".join(f"{k} {float(e.max()):.2e}" for k, e in errs.items()))


def _rel(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max())


@pytest.mark.parametrize("n,L", [(48000, 30000), (20001, 26000)])
@pytest.mark.parametrize("shared", [False, True], ids=["item", "shared"])
def test_bus_identities_with_convolution_reverberation(cuda_device, n, L, shared):
    """(1) S = 2, O = 2 is the true-stereo convolution_reverberation at mix 1; (2) S = 1, O = 2 the stereo one with a mono
    x.  Different kernels (and the dry term mix (wet - x) + x), so they agree to fp32 rounding"""
    import dasp_pytorch_b200 as D
    dev = cuda_device
    bs = 3
    ones = torch.ones(bs, device=dev)
    worst = {}
    for S in (2, 1):
        x, ir, w = _inputs(bs, S, 2, n, L, seed=17 + S + shared, shared=shared)
        bus = _gpu(x, ir, w, dev)
        assert _path() == _bits(n, L, shared)
        conv_ir = ir.reshape(ir.shape[0], 4, L) if S == 2 else ir[:, 0]
        ref = _run(lambda a, h: D.convolution_reverberation(a, SR, h, ones), x, conv_ir, w, dev, torch.float32)
        for k, a, b in zip(("y", "dx", "dir"), bus, ref):
            worst[(S, k)] = _rel(a.reshape(b.shape), b)
            assert worst[(S, k)] < 1e-5, (S, k, worst[(S, k)])
    print(f"identities {n}-{L} {'shared' if shared else 'item'}: " + " ".join(f"S{s} {k} {e:.1e}" for (s, k), e in
                                                                           worst.items()))


@pytest.mark.parametrize("S,O,shared", [(5, 2, False), (8, 1, True), (16, 2, False)])
def test_bus_is_the_sum_of_its_single_source_calls(cuda_device, S, O, shared):
    """(3) the bus of S inputs equals the sum of the S one-input buses, gradients included, to fp32 rounding"""
    dev = cuda_device
    n, L = 30000, 20000
    x, ir, w = _inputs(2, S, O, n, L, seed=31 + S, shared=shared)
    bus = _gpu(x, ir, w, dev)
    assert _path() == _bits(n, L, shared)
    parts = [_gpu(x[:, s:s + 1], ir[:, s:s + 1], w, dev) for s in range(S)]
    y = sum(p[0].double() for p in parts)
    assert _rel(bus[0], y) < 1e-5
    assert _rel(bus[1], torch.cat([p[1] for p in parts], 1)) < 1e-5
    assert _rel(bus[2], torch.cat([p[2] for p in parts], 1)) < 1e-5


@pytest.mark.parametrize("O", [1, 2])
def test_bus_shared_ir_gradient_same_bits_for_every_chunk(cuda_device, monkeypatch, O):
    from dasp_pytorch_b200 import functional as F
    x, ir, w = _inputs(5, 5, O, 20000, 15000, seed=41 + O, shared=True)
    runs = []
    for chunk in (1, 2, 5, 2):
        monkeypatch.setattr(F, "REVERB_CHUNK_ITEMS", chunk)
        runs.append(_gpu(x, ir, w, cuda_device))
        assert _path() == _bits(20000, 15000, True)
    for r in runs[1:]:
        assert torch.equal(r[2], runs[0][2])
        assert torch.equal(r[0], runs[0][0]) and torch.equal(r[1], runs[0][1])


@pytest.mark.parametrize("shared", [False, True], ids=["item", "shared"])
def test_bus_fixed_ir_skips_the_ir_gradient(cuda_device, shared):
    x, ir, w = _inputs(3, 3, 2, 20000, 15000, seed=43, shared=shared)
    full = _gpu(x, ir, w, cuda_device)
    fixed = _gpu(x, ir, w, cuda_device, ir_grad=False)
    assert _path() == _bits(20000, 15000, shared, ir_grad=False)
    assert fixed[2] is None
    assert torch.equal(fixed[0], full[0]) and torch.equal(fixed[1], full[1])


@pytest.mark.parametrize("S,O,shared", [(3, 1, False), (5, 2, True)])
def test_bus_ignores_prior_buffer_contents(cuda_device, S, O, shared):
    """NaN in both workspaces, the saved spectra and the outputs reaches no result"""
    from dasp_pytorch_b200 import _abi
    lib, dev = _lib(), cuda_device
    bs, n, L, chunk = 3, 20000, 15001, 2
    g = _abi.ConvGeom()
    _abi.check(lib.dasp_conv_bus_geometry(bs, n, L, S, O, int(shared), chunk, g), "geom")
    fwd, bwd = ((lib.dasp_conv_bus_shared_fwd, lib.dasp_conv_bus_shared_bwd) if shared
                else (lib.dasp_conv_bus_fwd, lib.dasp_conv_bus_bwd))
    x, ir, w = _inputs(bs, S, O, n, L, seed=47, shared=shared)
    x, ir, gy = (t.float().to(dev).contiguous() for t in (x, ir, w))

    def filled(numel, dtype, fill):
        t = torch.empty(numel, dtype=dtype, device=dev)
        t.view(torch.float32).fill_(fill)
        return t

    def run(fill):
        y = filled(bs * O * n, torch.float32, fill)
        ws = filled(g.fwd_workspace_bytes // 4, torch.float32, fill)
        xs, hs = filled(g.xspec_c64, torch.complex64, fill), filled(g.irspec_c64, torch.complex64, fill)
        _abi.check(fwd(_abi.ptr(x), _abi.ptr(ir), _abi.ptr(y), _abi.ptr(xs), _abi.ptr(hs), _abi.ptr(ws),
                       g.fwd_workspace_bytes, bs, n, L, S, O, chunk, _abi.stream_ptr(dev)), "fwd")
        gx = filled(bs * S * n, torch.float32, fill)
        gir = filled(ir.numel(), torch.float32, fill)
        wb = filled(g.bwd_workspace_bytes // 4, torch.float32, fill)
        _abi.check(bwd(_abi.ptr(gy), _abi.ptr(xs), _abi.ptr(hs), _abi.ptr(gx), _abi.ptr(gir), _abi.ptr(wb),
                       g.bwd_workspace_bytes, bs, n, L, S, O, chunk, _abi.stream_ptr(dev)), "bwd")
        assert _path() == _bits(n, L, shared)
        torch.cuda.synchronize(dev)
        return y, gx, gir

    clean, dirty = run(0.0), run(float("nan"))
    for a, b in zip(clean, dirty):
        assert bool(torch.isfinite(b).all())
        assert torch.equal(a, b)


@pytest.mark.parametrize("shared", [False, True], ids=["item", "shared"])
def test_bus_cuda_graph_replay_matches_eager(cuda_device, shared):
    import dasp_pytorch_b200 as D
    dev = cuda_device
    x, ir, w = (t.float().to(dev) for t in _inputs(3, 6, 2, 48000, 48000, seed=53, shared=shared))
    x.requires_grad_(True)
    ir.requires_grad_(True)

    def step():
        y = D.convolution_bus(x, SR, ir)
        return (y.detach(),) + torch.autograd.grad((y * w).sum(), (x, ir))

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
    for a, b in zip(static, eager):
        assert torch.equal(a, b)


def test_bus_bf16_is_the_rounded_fp32_result(cuda_device):
    import dasp_pytorch_b200 as D
    dev = cuda_device
    x, ir, _ = _inputs(2, 5, 2, 10000, 7000, seed=59, shared=False)
    xb, hb = x.to(dev, torch.bfloat16), ir.to(dev, torch.bfloat16)
    y = D.convolution_bus(xb, SR, hb)
    assert y.dtype == torch.bfloat16
    assert torch.equal(y, D.convolution_bus(xb.float(), SR, hb.float()).to(torch.bfloat16))
