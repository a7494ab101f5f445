"""multichannel_convolution on the GPU: y, dL/dx and dL/dIR pinned to the fp64 oracle (tests/conv_bus_oracle.py, run in
fp64 on the device) per item for 1 to 16 inputs and 3 to 32 outputs, per-item and shared matrices, every length class,
the L2 path and a minute of audio; M <= 2 bit for bit convolution_bus; the identities with the output-pair
convolution_bus calls and with the op's own single-source calls; the same bits for every chunk size, a fixed IR, stale
buffers, CUDA-graph replay and bf16.  Every case asserts the path bits it reached (dasp_debug_conv_bus_last_path)."""
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
# (S, M, shape index, shared): every S in {1, 2, 3, 5, 8, 16} and every M in {3, 4, 5, 7, 8, 16, 32}, both IR kinds and
# every length class; the L2 cases keep S M small for the oracle's memory
CASES = [(1, 3, 0, False), (1, 32, 1, True), (2, 3, 2, True), (2, 4, 3, False), (3, 5, 4, False), (3, 8, 5, True),
         (5, 7, 0, True), (5, 4, 2, False), (8, 8, 3, False), (8, 16, 4, True), (16, 3, 5, False), (16, 32, 2, True),
         (2, 8, 6, False), (3, 5, 6, True), (1, 7, 6, False), (16, 5, 1, False), (1, 16, 3, True), (5, 32, 4, False),
         (8, 7, 1, True), (2, 16, 0, False), (3, 4, 5, True), (16, 8, 0, True)]
CASES = [(S, M, *SHAPES[i], shared) for S, M, i, shared in CASES]


def _ids(c):
    return f"S{c[0]}-M{c[1]}-{c[2]}-{c[3]}-{'sh' if c[4] else 'it'}"


def _lib():
    from dasp_pytorch_b200 import _abi
    return _abi.lib()


def _bits(n, L, shared, M, ir_grad=True):
    """expected (forward, backward) path bits"""
    I, J = -(-n // KB), -(-min(n, L) // KB)
    cached, mc = max(I, J) <= 16, M > 2
    return (1 | (2 if shared else 0) | (4 if cached else 0) | (8 if mc else 0),
            1 | (2 if cached else 0) | (4 if ir_grad else 0) | (8 if shared else 0) | (16 if mc else 0))


def _path():
    lib = _lib()
    return lib.dasp_debug_conv_bus_last_path(0), lib.dasp_debug_conv_bus_last_path(1)


def _inputs(bs, S, M, n, L, seed, shared):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(bs, S, n, generator=g, dtype=torch.float64) * 2 - 1
    ir = (torch.rand(1 if shared else bs, S, M, L, generator=g, dtype=torch.float64) * 2 - 1) * torch.exp(
        -torch.arange(L, dtype=torch.float64) / max(L / 4, 1.0))
    w = torch.rand(bs, M, n, generator=g, dtype=torch.float64) * 2 - 1          # loss = sum(w y)
    return x, ir, w


def _run(fn, x, ir, w, device, dtype, ir_grad=True):
    xx = x.to(device=device, dtype=dtype).requires_grad_(True)
    hh = ir.to(device=device, dtype=dtype).requires_grad_(ir_grad)
    y = fn(xx, hh)
    (y * w.to(device=device, dtype=dtype)).sum().backward()
    return y.detach().cpu(), xx.grad.cpu(), None if hh.grad is None else hh.grad.cpu()


def _gpu(x, ir, w, dev, **kw):
    import dasp_pytorch_b200 as D
    return _run(lambda a, h: D.multichannel_convolution(a, SR, h), x, ir, w, dev, torch.float32, **kw)


def _bus(x, ir, w, dev, **kw):
    import dasp_pytorch_b200 as D
    return _run(lambda a, h: D.convolution_bus(a, SR, h), x, ir, w, dev, torch.float32, **kw)


def _ref(x, ir, w, dev):
    """the oracle in fp64 on the device (cuFFT in double precision, no project kernel)"""
    return _run(lambda a, h: conv_bus_oracle.convolution_bus(a, SR, h), x, ir, w, dev, torch.float64)


def _check(got, ref, label):
    """y and dL/dx per item; dL/dIR per item (or the shared matrix) on its own largest fp64 gradient"""
    errs = {k: peak_err(a, b) for k, a, b in zip(("y", "dx", "dir"), got, ref)}
    for k, e in errs.items():
        assert float(e.max()) < BOUND, (label, k, e)
    print(f"{label}: " + " ".join(f"{k} {float(e.max()):.2e}" for k, e in errs.items()))


@pytest.mark.parametrize("S,M,n,L,shared", CASES, ids=[_ids(c) for c in CASES])
def test_mc_pinned_to_oracle(cuda_device, monkeypatch, S, M, n, L, shared):
    """bs 3 in chunks of 2: y, dL/dx and dL/dIR within 1e-4 of the fp64 oracle; taps >= n get exactly 0"""
    from dasp_pytorch_b200 import functional as F
    monkeypatch.setattr(F, "REVERB_CHUNK_ITEMS", 2)
    x, ir, w = _inputs(3, S, M, n, L, seed=S * 100 + M * 7 + n % 97 + shared, shared=shared)
    got = _gpu(x, ir, w, cuda_device)
    assert _path() == _bits(n, L, shared, M)
    assert got[0].shape == (3, M, n) and got[1].shape == x.shape and got[2].shape == ir.shape
    if L > n:
        assert bool((got[2][..., n:] == 0).all())
    _check(got, _ref(x, ir, w, cuda_device), _ids((S, M, n, L, shared)))


def test_mc_pinned_to_oracle_on_a_minute_of_audio(cuda_device):
    """60 s at 48 kHz, two sources, an 8-microphone array, two-second impulse responses"""
    n, L = 60 * 48000, 96000
    x, ir, w = _inputs(1, 2, 8, n, L, seed=61, shared=False)
    got = _gpu(x, ir, w, cuda_device)
    assert _path() == _bits(n, L, False, 8)
    _check(got, _ref(x, ir, w, cuda_device), "60 s S2 M8")


@pytest.mark.parametrize("shared", [False, True], ids=["item", "shared"])
@pytest.mark.parametrize("S,M,n,L", [(3, 1, 20000, 15000), (5, 2, 48000, 30000), (2, 2, 70000, 66000),
                                     (4, 1, 9003, 20000)])
def test_mc_up_to_two_outputs_is_the_bus_bit_for_bit(cuda_device, S, M, n, L, shared):
    x, ir, w = _inputs(3, S, M, n, L, seed=19 + S + M + shared, shared=shared)
    mc = _gpu(x, ir, w, cuda_device)
    bits = _path()
    assert bits == _bits(n, L, shared, M)
    bus = _bus(x, ir, w, cuda_device)
    assert _path() == bits
    for a, b in zip(mc, bus):
        assert torch.equal(a, b)


def _rel(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max())


@pytest.mark.parametrize("shared", [False, True], ids=["item", "shared"])
@pytest.mark.parametrize("S,M", [(1, 3), (2, 4), (3, 5), (4, 7), (2, 8), (5, 16), (3, 32)])
def test_mc_is_the_output_pair_bus_calls(cuda_device, S, M, shared):
    """(2) the concatenation of the ceil(M / 2) convolution_bus calls on the output pairs, gradients summed over the
    calls by autograd, to 1e-5 of the peak"""
    dev = cuda_device
    n, L = 30000, 20000
    x, ir, w = _inputs(2, S, M, n, L, seed=23 + S * M + shared, shared=shared)
    mc = _gpu(x, ir, w, dev)
    assert _path() == _bits(n, L, shared, M)

    def pairs(a, h):
        import dasp_pytorch_b200 as D
        return torch.cat([D.convolution_bus(a, SR, h[:, :, q:q + 2]) for q in range(0, M, 2)], 1)

    ref = _run(pairs, x, ir, w, dev, torch.float32)
    for k, a, b in zip(("y", "dx", "dir"), mc, ref):
        assert _rel(a, b) < 1e-5, (k, _rel(a, b))


@pytest.mark.parametrize("S,M,shared", [(5, 4, False), (8, 3, True), (3, 16, False)])
def test_mc_is_the_sum_of_its_single_source_calls(cuda_device, S, M, shared):
    """(3) S inputs equal the sum of the S one-input calls, gradients included, to fp32 rounding"""
    dev = cuda_device
    n, L = 30000, 20000
    x, ir, w = _inputs(2, S, M, n, L, seed=31 + S + M, shared=shared)
    mc = _gpu(x, ir, w, dev)
    assert _path() == _bits(n, L, shared, M)
    parts = [_gpu(x[:, s:s + 1], ir[:, s:s + 1], w, dev) for s in range(S)]
    assert _rel(mc[0], sum(p[0].double() for p in parts)) < 1e-5
    assert _rel(mc[1], torch.cat([p[1] for p in parts], 1)) < 1e-5
    assert _rel(mc[2], torch.cat([p[2] for p in parts], 1)) < 1e-5


@pytest.mark.parametrize("M", [3, 8])
def test_mc_shared_ir_gradient_same_bits_for_every_chunk(cuda_device, monkeypatch, M):
    from dasp_pytorch_b200 import functional as F
    x, ir, w = _inputs(5, 5, M, 20000, 15000, seed=41 + M, shared=True)
    runs = []
    for chunk in (1, 2, 5, 2):
        monkeypatch.setattr(F, "REVERB_CHUNK_ITEMS", chunk)
        runs.append(_gpu(x, ir, w, cuda_device))
        assert _path() == _bits(20000, 15000, True, M)
    for r in runs[1:]:
        assert torch.equal(r[2], runs[0][2])
        assert torch.equal(r[0], runs[0][0]) and torch.equal(r[1], runs[0][1])


@pytest.mark.parametrize("shared", [False, True], ids=["item", "shared"])
@pytest.mark.parametrize("n,L", [(20000, 15000), (70000, 66000)])
def test_mc_fixed_ir_skips_the_ir_gradient(cuda_device, shared, n, L):
    x, ir, w = _inputs(3, 3, 6, n, L, seed=43, shared=shared)
    full = _gpu(x, ir, w, cuda_device)
    fixed = _gpu(x, ir, w, cuda_device, ir_grad=False)
    assert _path() == _bits(n, L, shared, 6, ir_grad=False)
    assert fixed[2] is None
    assert torch.equal(fixed[0], full[0]) and torch.equal(fixed[1], full[1])


@pytest.mark.parametrize("S,M,shared,n,L", [(3, 5, False, 20000, 15001), (5, 8, True, 20000, 15001),
                                            (2, 3, False, 70000, 66000)])
def test_mc_ignores_prior_buffer_contents(cuda_device, S, M, shared, n, L):
    """NaN in both workspaces, the saved spectra and the outputs reaches no result"""
    from dasp_pytorch_b200 import _abi
    lib, dev = _lib(), cuda_device
    bs, chunk = 3, 2
    g = _abi.ConvGeom()
    _abi.check(lib.dasp_conv_mc_geometry(bs, n, L, S, M, int(shared), chunk, g), "geom")
    fwd, bwd = ((lib.dasp_conv_mc_shared_fwd, lib.dasp_conv_mc_shared_bwd) if shared
                else (lib.dasp_conv_mc_fwd, lib.dasp_conv_mc_bwd))
    x, ir, w = _inputs(bs, S, M, n, L, seed=47, shared=shared)
    x, ir, gy = (t.float().to(dev).contiguous() for t in (x, ir, w))

    def filled(numel, dtype, fill):
        t = torch.empty(numel, dtype=dtype, device=dev)
        t.view(torch.float32).fill_(fill)
        return t

    def run(fill):
        y = filled(bs * M * n, torch.float32, fill)
        ws = filled(g.fwd_workspace_bytes // 4, torch.float32, fill)
        xs, hs = filled(g.xspec_c64, torch.complex64, fill), filled(g.irspec_c64, torch.complex64, fill)
        _abi.check(fwd(_abi.ptr(x), _abi.ptr(ir), _abi.ptr(y), _abi.ptr(xs), _abi.ptr(hs), _abi.ptr(ws),
                       g.fwd_workspace_bytes, bs, n, L, S, M, chunk, _abi.stream_ptr(dev)), "fwd")
        gx = filled(bs * S * n, torch.float32, fill)
        gir = filled(ir.numel(), torch.float32, fill)
        wb = filled(g.bwd_workspace_bytes // 4, torch.float32, fill)
        _abi.check(bwd(_abi.ptr(gy), _abi.ptr(xs), _abi.ptr(hs), _abi.ptr(gx), _abi.ptr(gir), _abi.ptr(wb),
                       g.bwd_workspace_bytes, bs, n, L, S, M, chunk, _abi.stream_ptr(dev)), "bwd")
        assert _path() == _bits(n, L, shared, M)
        torch.cuda.synchronize(dev)
        return y, gx, gir

    clean, dirty = run(0.0), run(float("nan"))
    for a, b in zip(clean, dirty):
        assert bool(torch.isfinite(b).all())
        assert torch.equal(a, b)


@pytest.mark.parametrize("shared", [False, True], ids=["item", "shared"])
def test_mc_cuda_graph_replay_matches_eager(cuda_device, shared):
    import dasp_pytorch_b200 as D
    dev = cuda_device
    x, ir, w = (t.float().to(dev) for t in _inputs(3, 4, 8, 48000, 48000, seed=53, shared=shared))
    x.requires_grad_(True)
    ir.requires_grad_(True)

    def step():
        y = D.multichannel_convolution(x, SR, ir)
        return (y.detach(),) + torch.autograd.grad((y * w).sum(), (x, ir))

    eager = [t.clone() for t in step()]
    assert _path() == _bits(48000, 48000, shared, 8)
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


def test_mc_bf16_is_the_rounded_fp32_result(cuda_device):
    import dasp_pytorch_b200 as D
    dev = cuda_device
    x, ir, _ = _inputs(2, 5, 7, 10001, 7000, seed=59, shared=False)
    xb, hb = x.to(dev, torch.bfloat16), ir.to(dev, torch.bfloat16)
    y = D.multichannel_convolution(xb, SR, hb)
    assert _path()[0] == _bits(10001, 7000, False, 7)[0]
    assert y.dtype == torch.bfloat16 and y.shape == (2, 7, 10001)
    assert torch.equal(y, D.multichannel_convolution(xb.float(), SR, hb.float()).to(torch.bfloat16))
