"""time_varying_convolution_bus with crossfade="input" (the source-side crossfade) on the GPU: y, dL/dx and dL/dIR
pinned to the fp64 oracle (tests/tv_bus_input_oracle.py, run in fp64 on the device's cuFFT) for 1 to 32 sources, mono
and stereo buses, per-item and shared trajectory sets, K from 1 to 15, anchor spacings of 1, 3 and 8 partitions, IRs
shorter than, longer than and as long as x, padded rows, more than 16 blocks or partitions and a minute of audio; the
identities with convolution_bus, the sum of single-source calls, the segment composition and the emission-time
response; the same bits for every chunk size, a fixed set, stale buffers, CUDA-graph replay, bf16, and
crossfade="output" against the default.  Every case asserts the path bits it reached (dasp_debug_tvbus_last_path)."""
import pytest
import torch

import tv_bus_input_oracle
import tv_bus_oracle
from helpers import SR, peak_err

pytestmark = pytest.mark.gpu
BOUND = 1e-4
KB = 4096

# (S, O, shared, K, hop, n, L)
CASES = [
    (1, 2, False, 1, KB, 20000, 9000),             # K = 1, one source
    (2, 1, True, 2, KB, 9001, 3000),               # n % 4 = 1, L < hop
    (3, 2, False, 5, 3 * KB, 60002, 15000),        # n % 4 = 2, L > hop
    (5, 1, True, 5, 3 * KB, 50003, 60000),         # n % 4 = 3, L >= n
    (8, 2, True, 15, KB, 70000, 66000),            # I = 18, J = 17
    (32, 1, False, 2, 8 * KB, 40000, 5000),
    (32, 2, True, 2, KB, 12000, 3000),
    (3, 1, False, 15, KB, 61540, 20000),
    (2, 2, False, 3, 8 * KB, 100000, 40000),
    (8, 1, True, 1, KB, 5000, 100),
    (5, 2, False, 5, 8 * KB, 140000, 30000),
    (1, 1, True, 15, KB, 70001, 70001),            # L = n, n % 4 = 1
]


def _ids(c):
    return f"S{c[0]}-O{c[1]}-{'sh' if c[2] else 'it'}-K{c[3]}-hop{c[4] // KB}-{c[5]}-{c[6]}"


def _lib():
    from dasp_pytorch_b200 import _abi
    return _abi.lib()


def _bits(K, shared, ir_grad=True):
    """expected (forward, backward) path bits: the output-side op's, and the source-side bit of each direction"""
    cross = K > 1
    return (1 | (2 if shared else 0) | (4 if cross else 0) | 8,
            1 | (2 if cross else 0) | (4 if ir_grad else 0) | (8 if shared else 0) | 16)


def _path():
    lib = _lib()
    return lib.dasp_debug_tvbus_last_path(0), lib.dasp_debug_tvbus_last_path(1)


def _inputs(bs, S, O, K, n, L, seed, shared):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(bs, S, n, generator=g, dtype=torch.float64) * 2 - 1
    ir = (torch.rand(1 if shared else bs, K, S, O, L, generator=g, dtype=torch.float64) * 2 - 1) * torch.exp(
        -torch.arange(L, dtype=torch.float64) / max(L / 4, 1.0))
    w = torch.rand(bs, O, n, generator=g, dtype=torch.float64) * 2 - 1          # loss = sum(w y)
    return x, ir, w


def _run(fn, x, ir, w, device, dtype, ir_grad=True):
    xx = x.to(device=device, dtype=dtype).requires_grad_(True)
    hh = ir.to(device=device, dtype=dtype).requires_grad_(ir_grad)
    y = fn(xx, hh)
    (y * w.to(device=device, dtype=dtype)).sum().backward()
    return (y.detach().cpu(), xx.grad.cpu(), None if hh.grad is None else hh.grad.cpu())


def _gpu(x, ir, w, hop, dev, **kw):
    import dasp_pytorch_b200 as D
    return _run(lambda a, h: D.time_varying_convolution_bus(a, SR, h, hop, crossfade="input"), x, ir, w, dev,
                torch.float32, **kw)


def _ref(x, ir, w, hop, dev):
    return _run(lambda a, h: tv_bus_input_oracle.time_varying_convolution_bus(a, SR, h, hop), x, ir, w, dev,
                torch.float64)


def _check(got, ref, label):
    """y and dL/dx per item; dL/dIR per item (or the shared set) on its own largest fp64 gradient"""
    errs = {k: peak_err(a, b) for k, a, b in zip(("y", "dx", "dir"), got, ref)}
    for k, e in errs.items():
        assert float(e.max()) < BOUND, (label, k, e)
    print(f"{label}: " + " ".join(f"{k} {float(e.max()):.2e}" for k, e in errs.items()))


@pytest.mark.parametrize("S,O,shared,K,hop,n,L", CASES, ids=[_ids(c) for c in CASES])
def test_tv_bus_input_pinned_to_oracle(cuda_device, monkeypatch, S, O, shared, K, hop, n, L):
    """bs 3 in chunks of 2: y, dL/dx and dL/dIR within 1e-4 of the fp64 oracle; taps >= n get exactly 0"""
    from dasp_pytorch_b200 import functional as F
    monkeypatch.setattr(F, "REVERB_CHUNK_ITEMS", 2)
    x, ir, w = _inputs(3, S, O, K, n, L, seed=K * 100 + n % 97 + S + 40 * O + shared, shared=shared)
    got = _gpu(x, ir, w, hop, cuda_device)
    assert _path() == _bits(K, shared)
    assert got[0].shape == (3, O, n) and got[1].shape == x.shape and got[2].shape == ir.shape
    if L > n:
        assert bool((got[2][..., n:] == 0).all())
    _check(got, _ref(x, ir, w, hop, cuda_device), _ids((S, O, shared, K, hop, n, L)))


def test_tv_bus_input_pinned_to_oracle_on_a_minute_of_audio(cuda_device):
    """60 s at 48 kHz, four sources, 15 anchors 48 partitions apart, one-second stereo IRs"""
    n, L, K, hop = 60 * 48000, 48000, 15, 48 * KB
    x, ir, w = _inputs(1, 4, 2, K, n, L, seed=61, shared=False)
    got = _gpu(x, ir, w, hop, cuda_device)
    assert _path() == _bits(K, False)
    _check(got, _ref(x, ir, w, hop, cuda_device), "60 s")


def _rel(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max())


@pytest.mark.parametrize("shared", [False, True], ids=["item", "shared"])
@pytest.mark.parametrize("S,O", [(3, 2), (4, 1)])
def test_tv_bus_input_identities(cuda_device, shared, S, O):
    """(1) K = 1 is convolution_bus(x, sr, h[:, 0]); (2) K equal sets are that set's static bus, and the K sets'
    gradients sum to the static one; (3) the sum of S single-source calls; (4) the segment composition
    sum_k convolution_bus(w_k x, sr, h[:, k]) in torch, gradients included.  Different kernels or summation orders, so
    they agree to fp32 rounding"""
    import dasp_pytorch_b200 as D
    dev = cuda_device
    n, L, hop, K = 60000, 20000, 3 * KB, 4
    worst = {}

    def bus(x, h, w):
        return _run(lambda a, hh: D.convolution_bus(a, SR, hh), x, h, w, dev, torch.float32)

    x, ir, w = _inputs(3, S, O, 1, n, L, seed=71 + shared + S, shared=shared)
    tv = _gpu(x, ir, w, hop, dev)
    assert _path() == _bits(1, shared)
    ref = bus(x, ir[:, 0], w)
    for k, a, b in zip(("y", "dx", "dir"), tv, ref):
        worst[("K1", k)] = _rel(a.reshape(b.shape), b)

    tv = _gpu(x, ir.expand(-1, K, -1, -1, -1).contiguous(), w, hop, dev)
    assert _path() == _bits(K, shared)
    for k, a, b in zip(("y", "dx", "dir"), (tv[0], tv[1], tv[2].sum(1)), ref):
        worst[("equal", k)] = _rel(a, b)

    _, irk, _ = _inputs(3, S, O, K, n, L, seed=73 + shared + S, shared=shared)
    tv = _gpu(x, irk, w, hop, dev)
    parts = [_gpu(x[:, s:s + 1], irk[:, :, s:s + 1], w, hop, dev) for s in range(S)]
    worst[("sum", "y")] = _rel(tv[0], sum(p[0] for p in parts))
    worst[("sum", "dx")] = _rel(tv[1], torch.cat([p[1] for p in parts], 1))
    worst[("sum", "dir")] = _rel(tv[2], torch.cat([p[2] for p in parts], 2))

    wk = tv_bus_oracle.hat_weights(K, hop, n, torch.float32, dev)
    comp = _run(lambda a, hh: sum(D.convolution_bus(wk[k] * a, SR, hh[:, k]) for k in range(K)), x, irk, w, dev,
                torch.float32)
    for k, a, b in zip(("y", "dx", "dir"), tv, comp):
        worst[("segments", k)] = _rel(a, b)
    for key, e in worst.items():
        assert e < 1e-5, (key, e)
    print(f"identities S{S} O{O} {'shared' if shared else 'item'}: worst "
          + " ".join(f"{a}-{b} {e:.1e}" for (a, b), e in worst.items()))


@pytest.mark.parametrize("O", [1, 2])
def test_tv_bus_input_keeps_the_emission_time_ir_over_the_whole_tail(cuda_device, O):
    """a unit impulse on source 1 of 3 at tau between anchors 1 and 2 (weight a) gives (1 - a) h_1 + a h_2 over its
    whole tail, which runs past anchors 2 to 4 (L > 3 hop), and nothing before tau"""
    import dasp_pytorch_b200 as D
    dev = cuda_device
    n, L, K, hop, tau = 40000, 15000, 5, KB, 5000
    g = torch.Generator().manual_seed(101 + O)
    h = torch.rand(1, K, 3, O, L, generator=g) * 2 - 1
    x = torch.zeros(1, 3, n)
    x[0, 1, tau] = 1
    y = D.time_varying_convolution_bus(x.to(dev), SR, h.to(dev), hop, crossfade="input").cpu()
    assert _path()[0] == _bits(K, False)[0]
    k, a = tau // hop, (tau % hop) / hop
    want = (1 - a) * h[0, k, 1] + a * h[0, k + 1, 1]
    assert float(y[0, :, :tau].abs().max()) < 1e-6
    assert _rel(y[0, :, tau:tau + L], want) < 1e-5


@pytest.mark.parametrize("shared", [False, True], ids=["item", "shared"])
@pytest.mark.parametrize("O", [1, 2])
def test_tv_bus_input_same_bits_for_every_chunk(cuda_device, monkeypatch, shared, O):
    from dasp_pytorch_b200 import functional as F
    x, ir, w = _inputs(5, 3, O, 5, 40000, 15000, seed=81 + shared + O, shared=shared)
    runs = []
    for chunk in (1, 2, 5, 3):
        monkeypatch.setattr(F, "REVERB_CHUNK_ITEMS", chunk)
        runs.append(_gpu(x, ir, w, 2 * KB, cuda_device))
        assert _path() == _bits(5, shared)
    for r in runs[1:]:
        for a, b in zip(r, runs[0]):
            assert torch.equal(a, b)


@pytest.mark.parametrize("shared", [False, True], ids=["item", "shared"])
@pytest.mark.parametrize("O", [1, 2])
def test_tv_bus_input_fixed_set_skips_the_ir_gradient(cuda_device, shared, O):
    x, ir, w = _inputs(3, 3, O, 3, 30000, 15000, seed=83 + O, shared=shared)
    full = _gpu(x, ir, w, KB, cuda_device)
    fixed = _gpu(x, ir, w, KB, cuda_device, ir_grad=False)
    assert _path() == _bits(3, shared, ir_grad=False)
    assert fixed[2] is None
    for i in (0, 1):
        assert torch.equal(fixed[i], full[i])


@pytest.mark.parametrize("shared", [False, True], ids=["item", "shared"])
@pytest.mark.parametrize("O", [1, 2])
def test_tv_bus_input_ignores_prior_buffer_contents(cuda_device, shared, O):
    """NaN in both workspaces, the saved spectra and the outputs reaches no result"""
    from dasp_pytorch_b200 import _abi
    lib, dev = _lib(), cuda_device
    bs, n, L, K, S, hop, chunk = 3, 40000, 15001, 5, 3, 2 * KB, 2
    g = _abi.ConvGeom()
    _abi.check(lib.dasp_tvbus_in_geometry(bs, n, L, K, S, O, hop, int(shared), chunk, g), "geom")
    fwd, bwd = ((lib.dasp_tvbus_in_shared_fwd, lib.dasp_tvbus_in_shared_bwd) if shared
                else (lib.dasp_tvbus_in_fwd, lib.dasp_tvbus_in_bwd))
    x, ir, w = _inputs(bs, S, O, K, n, L, seed=87 + O, shared=shared)
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
                       g.fwd_workspace_bytes, bs, n, L, K, S, O, hop, chunk, _abi.stream_ptr(dev)), "fwd")
        gx = filled(bs * S * n, torch.float32, fill)
        gir = filled(ir.numel(), torch.float32, fill)
        wb = filled(g.bwd_workspace_bytes // 4, torch.float32, fill)
        _abi.check(bwd(_abi.ptr(gy), _abi.ptr(xs), _abi.ptr(hs), _abi.ptr(gx), _abi.ptr(gir), _abi.ptr(wb),
                       g.bwd_workspace_bytes, bs, n, L, K, S, O, hop, chunk, _abi.stream_ptr(dev)), "bwd")
        assert _path() == _bits(K, shared)
        torch.cuda.synchronize(dev)
        return y, gx, gir

    clean, dirty = run(0.0), run(float("nan"))
    for a, b in zip(clean, dirty):
        assert bool(torch.isfinite(b).all())
        assert torch.equal(a, b)


@pytest.mark.parametrize("shared", [False, True], ids=["item", "shared"])
def test_tv_bus_input_cuda_graph_replay_matches_eager(cuda_device, shared):
    import dasp_pytorch_b200 as D
    dev = cuda_device
    x, ir, w = (t.float().to(dev) for t in _inputs(3, 3, 2, 5, 48000, 20000, seed=91, shared=shared))
    for t in (x, ir):
        t.requires_grad_(True)

    def step():
        y = D.time_varying_convolution_bus(x, SR, ir, 2 * KB, crossfade="input")
        return (y.detach(),) + torch.autograd.grad((y * w).sum(), (x, ir))

    eager = [t.clone() for t in step()]
    assert _path() == _bits(5, shared)
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


def test_tv_bus_input_bf16_is_the_rounded_fp32_result(cuda_device):
    import dasp_pytorch_b200 as D
    dev = cuda_device
    x, ir, _ = _inputs(2, 3, 2, 3, 20000, 7000, seed=97, shared=False)
    xb, hb = x.to(dev, torch.bfloat16), ir.to(dev, torch.bfloat16)
    y = D.time_varying_convolution_bus(xb, SR, hb, KB, crossfade="input")
    assert _path()[0] == _bits(3, False)[0]
    assert y.dtype == torch.bfloat16
    ref = D.time_varying_convolution_bus(xb.float(), SR, hb.float(), KB, crossfade="input").to(torch.bfloat16)
    assert torch.equal(y, ref)


@pytest.mark.parametrize("shared", [False, True], ids=["item", "shared"])
def test_tv_bus_output_crossfade_is_the_default(cuda_device, shared):
    """crossfade="output" gives the same bits as omitting the keyword, and the output-side path bits"""
    import dasp_pytorch_b200 as D
    dev = cuda_device
    x, ir, w = _inputs(3, 3, 2, 4, 30000, 12000, seed=99 + shared, shared=shared)
    default = _run(lambda a, h: D.time_varying_convolution_bus(a, SR, h, KB), x, ir, w, dev, torch.float32)
    paths = _path()
    named = _run(lambda a, h: D.time_varying_convolution_bus(a, SR, h, KB, crossfade="output"), x, ir, w, dev,
                 torch.float32)
    assert _path() == paths and paths[0] & 8 == 0 and paths[1] & 16 == 0
    for a, b in zip(default, named):
        assert torch.equal(a, b)
