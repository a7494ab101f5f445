"""time_varying_multichannel_convolution on the GPU, both crossfades: y, dL/dx and dL/dIR pinned to the fp64 oracles
(tests/tv_bus_oracle.py, tests/tv_bus_input_oracle.py, run in fp64 on the device's cuFFT) for 1 to 16 sources, 3 to 32
outputs, per-item and shared trajectories, K from 1 to 15, IRs shorter and longer than x, padded rows, more than 16
blocks and a minute of audio; M <= 2 bit for bit time_varying_convolution_bus; the identities with the output-pair
time_varying_convolution_bus calls, multichannel_convolution, the single-source calls, the last anchor (output side),
the segment composition and the emission-time response (source side); the same bits for every chunk size, a fixed
trajectory, stale buffers, CUDA-graph replay and bf16.  Every case asserts the path bits it reached
(dasp_debug_tvbus_last_path)."""
import pytest
import torch

import tv_bus_input_oracle
import tv_bus_oracle
from helpers import SR, peak_err

pytestmark = pytest.mark.gpu
BOUND = 1e-4
KB = 4096
ORACLES = {"output": tv_bus_oracle, "input": tv_bus_input_oracle}
XF = ["output", "input"]

# (S, M, shared, K, hop, n, L): every S in {1, 2, 3, 5, 8, 16}, every M in {3, 4, 5, 7, 8, 16, 32}, K in {1, 2, 3, 15},
# L < n and L > n, n % 4 = 1, 2, 3, and I = 18 / J = 17
CASES = [
    (1, 3, False, 1, KB, 20000, 9000),             # K = 1, one source
    (2, 4, True, 2, KB, 9001, 3000),               # n % 4 = 1, L < hop
    (3, 5, False, 3, 3 * KB, 60002, 15000),        # n % 4 = 2, L > hop
    (5, 7, True, 3, 3 * KB, 50003, 60000),         # n % 4 = 3, L > n
    (8, 8, True, 15, KB, 70000, 66000),            # I = 18, J = 17
    (16, 3, False, 2, 8 * KB, 40000, 5000),
    (2, 16, True, 2, KB, 12000, 3000),
    (3, 32, False, 15, KB, 61540, 8000),
    (5, 4, False, 2, 2 * KB, 30001, 12000),
    (16, 32, True, 2, KB, 9000, 2000),
    (1, 5, True, 15, KB, 70001, 70001),            # L = n, n % 4 = 1
    (8, 7, False, 3, 2 * KB, 30000, 20000),
]


def _ids(c):
    return f"S{c[0]}-M{c[1]}-{'sh' if c[2] else 'it'}-K{c[3]}-hop{c[4] // KB}-{c[5]}-{c[6]}"


def _lib():
    from dasp_pytorch_b200 import _abi
    return _abi.lib()


def _bits(crossfade, K, shared, M, ir_grad=True):
    """expected (forward, backward) path bits: dasp_tvbus_*'s, the source-side bits, and the M >= 3 bits"""
    cross, src, mc = K > 1, crossfade == "input", M > 2
    return (1 | (2 if shared else 0) | (4 if cross else 0) | (8 if src else 0) | (16 if mc else 0),
            1 | (2 if cross else 0) | (4 if ir_grad else 0) | (8 if shared else 0) | (16 if src else 0)
            | (32 if mc else 0))


def _path():
    lib = _lib()
    return lib.dasp_debug_tvbus_last_path(0), lib.dasp_debug_tvbus_last_path(1)


def _inputs(bs, S, M, K, n, L, seed, shared):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(bs, S, n, generator=g, dtype=torch.float64) * 2 - 1
    ir = (torch.rand(1 if shared else bs, K, S, M, L, generator=g, dtype=torch.float64) * 2 - 1) * torch.exp(
        -torch.arange(L, dtype=torch.float64) / max(L / 4, 1.0))
    w = torch.rand(bs, M, n, generator=g, dtype=torch.float64) * 2 - 1          # loss = sum(w y)
    return x, ir, w


def _run(fn, x, ir, w, device, dtype, ir_grad=True):
    xx = x.to(device=device, dtype=dtype).requires_grad_(True)
    hh = ir.to(device=device, dtype=dtype).requires_grad_(ir_grad)
    y = fn(xx, hh)
    (y * w.to(device=device, dtype=dtype)).sum().backward()
    return (y.detach().cpu(), xx.grad.cpu(), None if hh.grad is None else hh.grad.cpu())


def _gpu(x, ir, w, hop, dev, crossfade, **kw):
    import dasp_pytorch_b200 as D
    return _run(lambda a, h: D.time_varying_multichannel_convolution(a, SR, h, hop, crossfade=crossfade), x, ir, w,
                dev, torch.float32, **kw)


def _tvbus(x, ir, w, hop, dev, crossfade, **kw):
    import dasp_pytorch_b200 as D
    return _run(lambda a, h: D.time_varying_convolution_bus(a, SR, h, hop, crossfade=crossfade), x, ir, w, dev,
                torch.float32, **kw)


def _ref(x, ir, w, hop, dev, crossfade):
    oracle = ORACLES[crossfade]
    return _run(lambda a, h: oracle.time_varying_convolution_bus(a, SR, h, hop), x, ir, w, dev, torch.float64)


def _check(got, ref, label):
    """y and dL/dx per item; dL/dIR per item (or the shared trajectory) on its own largest fp64 gradient"""
    errs = {k: peak_err(a, b) for k, a, b in zip(("y", "dx", "dir"), got, ref)}
    for k, e in errs.items():
        assert float(e.max()) < BOUND, (label, k, e)
    print(f"{label}: " + " ".join(f"{k} {float(e.max()):.2e}" for k, e in errs.items()))


def _rel(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max())


@pytest.mark.parametrize("crossfade", XF)
@pytest.mark.parametrize("S,M,shared,K,hop,n,L", CASES, ids=[_ids(c) for c in CASES])
def test_tv_mc_pinned_to_oracle(cuda_device, monkeypatch, crossfade, S, M, shared, K, hop, n, L):
    """bs 3 in chunks of 2: y, dL/dx and dL/dIR within 1e-4 of the fp64 oracle; taps >= n get exactly 0"""
    from dasp_pytorch_b200 import functional as F
    monkeypatch.setattr(F, "REVERB_CHUNK_ITEMS", 2)
    x, ir, w = _inputs(3, S, M, K, n, L, seed=K * 100 + n % 97 + S + 40 * M + shared, shared=shared)
    got = _gpu(x, ir, w, hop, cuda_device, crossfade)
    assert _path() == _bits(crossfade, K, shared, M)
    assert got[0].shape == (3, M, n) and got[1].shape == x.shape and got[2].shape == ir.shape
    if L > n:
        assert bool((got[2][..., n:] == 0).all())
    _check(got, _ref(x, ir, w, hop, cuda_device, crossfade), f"{crossfade} {_ids((S, M, shared, K, hop, n, L))}")


@pytest.mark.parametrize("crossfade", XF)
def test_tv_mc_pinned_to_oracle_on_a_minute_of_audio(cuda_device, crossfade):
    """60 s at 48 kHz, two talkers at a 4-microphone array, 15 anchors 48 partitions apart, one-second IRs"""
    n, L, K, hop = 60 * 48000, 48000, 15, 48 * KB
    x, ir, w = _inputs(1, 2, 4, K, n, L, seed=61, shared=False)
    got = _gpu(x, ir, w, hop, cuda_device, crossfade)
    assert _path() == _bits(crossfade, K, False, 4)
    _check(got, _ref(x, ir, w, hop, cuda_device, crossfade), f"60 s {crossfade}")


@pytest.mark.parametrize("crossfade", XF)
@pytest.mark.parametrize("ir_grad", [True, False], ids=["irgrad", "fixed"])
@pytest.mark.parametrize("shared", [False, True], ids=["item", "shared"])
@pytest.mark.parametrize("S,M,K,n,L", [(3, 1, 3, 20000, 15000), (5, 2, 4, 48000, 30000), (2, 2, 15, 70000, 66000)])
def test_tv_mc_up_to_two_outputs_is_the_tv_bus_bit_for_bit(cuda_device, crossfade, ir_grad, shared, S, M, K, n, L):
    x, ir, w = _inputs(3, S, M, K, n, L, seed=19 + S + M + shared, shared=shared)
    mc = _gpu(x, ir, w, KB, cuda_device, crossfade, ir_grad=ir_grad)
    bits = _path()
    assert bits == _bits(crossfade, K, shared, M, ir_grad)
    bus = _tvbus(x, ir, w, KB, cuda_device, crossfade, ir_grad=ir_grad)
    assert _path() == bits
    for a, b in zip(mc, bus):
        assert (a is None and b is None) or torch.equal(a, b)


@pytest.mark.parametrize("crossfade", XF)
@pytest.mark.parametrize("shared", [False, True], ids=["item", "shared"])
@pytest.mark.parametrize("S,M,K", [(1, 3, 3), (2, 4, 2), (3, 5, 4), (4, 8, 3), (2, 32, 2)])
def test_tv_mc_is_the_output_pair_tv_bus_calls(cuda_device, crossfade, shared, S, M, K):
    """the concatenation of the ceil(M / 2) time_varying_convolution_bus calls on the output pairs, gradients summed
    over the calls by autograd, to 1e-5 of the peak"""
    import dasp_pytorch_b200 as D
    dev, n, L, hop = cuda_device, 30000, 20000, 2 * KB
    x, ir, w = _inputs(2, S, M, K, n, L, seed=23 + S * M + shared, shared=shared)
    mc = _gpu(x, ir, w, hop, dev, crossfade)
    assert _path() == _bits(crossfade, K, shared, M)

    def pairs(a, h):
        return torch.cat([D.time_varying_convolution_bus(a, SR, h[:, :, :, q:q + 2], hop, crossfade=crossfade)
                          for q in range(0, M, 2)], 1)

    ref = _run(pairs, x, ir, w, dev, torch.float32)
    for k, a, b in zip(("y", "dx", "dir"), mc, ref):
        assert _rel(a, b) < 1e-5, (k, _rel(a, b))


@pytest.mark.parametrize("crossfade", XF)
@pytest.mark.parametrize("shared", [False, True], ids=["item", "shared"])
def test_tv_mc_with_one_or_equal_matrices_is_multichannel_convolution(cuda_device, crossfade, shared):
    import dasp_pytorch_b200 as D
    dev, S, M, n, L = cuda_device, 3, 6, 40000, 15000
    x, ir, w = _inputs(2, S, M, 1, n, L, seed=29 + shared, shared=shared)
    ref = _run(lambda a, h: D.multichannel_convolution(a, SR, h[:, 0]), x, ir, w, dev, torch.float32)
    one = _gpu(x, ir, w, KB, dev, crossfade)
    assert _path() == _bits(crossfade, 1, shared, M)
    for a, b in zip(one[:2], ref[:2]):
        assert _rel(a, b) < 1e-5
    eq = ir.expand(-1, 4, -1, -1, -1).contiguous()
    four = _gpu(x, eq, w, 2 * KB, dev, crossfade)
    assert _path() == _bits(crossfade, 4, shared, M)
    assert _rel(four[0], ref[0]) < 1e-5 and _rel(four[1], ref[1]) < 1e-5
    assert _rel(four[2].sum(1, keepdim=True), ref[2]) < 1e-5


@pytest.mark.parametrize("crossfade", XF)
@pytest.mark.parametrize("S,M,shared", [(5, 4, False), (3, 7, True)])
def test_tv_mc_is_the_sum_of_its_single_source_calls(cuda_device, crossfade, S, M, shared):
    dev, n, L, K = cuda_device, 30000, 20000, 3
    x, ir, w = _inputs(2, S, M, K, n, L, seed=31 + S + M, shared=shared)
    mc = _gpu(x, ir, w, 2 * KB, dev, crossfade)
    assert _path() == _bits(crossfade, K, shared, M)
    parts = [_gpu(x[:, s:s + 1], ir[:, :, s:s + 1], w, 2 * KB, dev, crossfade) for s in range(S)]
    assert _rel(mc[0], sum(p[0].double() for p in parts)) < 1e-5
    assert _rel(mc[1], torch.cat([p[1] for p in parts], 1)) < 1e-5
    assert _rel(mc[2], torch.cat([p[2] for p in parts], 2)) < 1e-5


def test_tv_mc_output_side_after_the_last_anchor_is_multichannel_convolution(cuda_device):
    import dasp_pytorch_b200 as D
    dev, S, M, K, hop, n, L = cuda_device, 3, 5, 4, 2 * KB, 40000, 9000
    x, ir, _ = _inputs(2, S, M, K, n, L, seed=37, shared=False)
    xf, hf = x.float().to(dev), ir.float().to(dev)
    y = D.time_varying_multichannel_convolution(xf, SR, hf, hop)
    assert _path()[0] == _bits("output", K, False, M)[0]
    ref = D.multichannel_convolution(xf, SR, hf[:, K - 1])
    t0 = (K - 1) * hop
    assert _rel(y[..., t0:].cpu(), ref[..., t0:].cpu()) < 1e-5


def test_tv_mc_input_side_is_the_segment_composition(cuda_device):
    """sum_k multichannel_convolution(w_k x, h[:, k]), gradients included"""
    import dasp_pytorch_b200 as D
    dev, S, M, K, hop, n, L = cuda_device, 3, 6, 4, 2 * KB, 40000, 15000
    x, ir, w = _inputs(2, S, M, K, n, L, seed=41, shared=False)
    got = _gpu(x, ir, w, hop, dev, "input")
    assert _path() == _bits("input", K, False, M)
    wk = tv_bus_oracle.hat_weights(K, hop, n, torch.float32, dev)
    ref = _run(lambda a, h: sum(D.multichannel_convolution(wk[k] * a, SR, h[:, k]) for k in range(K)), x, ir, w, dev,
               torch.float32)
    for k, a, b in zip(("y", "dx", "dir"), got, ref):
        assert _rel(a, b) < 1e-5, (k, _rel(a, b))


def test_tv_mc_input_side_keeps_the_emission_time_ir_over_the_whole_tail(cuda_device):
    """a unit impulse on source 1 at tau between anchors 1 and 2 (weight a) gives (1 - a) h_1 + a h_2 on every
    output, also past the later anchors (L > hop)"""
    import dasp_pytorch_b200 as D
    dev, K, hop, n, L, M = cuda_device, 4, KB, 20000, 9000, 5
    tau = hop + 1229
    x = torch.zeros(1, 2, n, device=dev)
    x[0, 1, tau] = 1
    _, ir, _ = _inputs(1, 2, M, K, n, L, seed=43, shared=False)
    h = ir.float().to(dev)
    y = D.time_varying_multichannel_convolution(x, SR, h, hop, crossfade="input")
    assert _path()[0] == _bits("input", K, False, M)[0]
    a = 1229 / hop
    want = (1 - a) * h[0, 1, 1] + a * h[0, 2, 1]
    assert float(y[0, :, :tau].abs().max()) < 1e-6
    assert _rel(y[0, :, tau:tau + L].cpu(), want.cpu()) < 1e-5


@pytest.mark.parametrize("crossfade", XF)
def test_tv_mc_same_bits_for_every_chunk(cuda_device, monkeypatch, crossfade):
    """per-item and shared trajectories; the shared gradient is the fp64 item sum in item order"""
    from dasp_pytorch_b200 import functional as F
    for shared in (False, True):
        x, ir, w = _inputs(5, 3, 5, 3, 20000, 15000, seed=47 + shared, shared=shared)
        runs = []
        for chunk in (1, 2, 5, 2):
            monkeypatch.setattr(F, "REVERB_CHUNK_ITEMS", chunk)
            runs.append(_gpu(x, ir, w, KB, cuda_device, crossfade))
            assert _path() == _bits(crossfade, 3, shared, 5)
        for r in runs[1:]:
            for a, b in zip(r, runs[0]):
                assert torch.equal(a, b)


@pytest.mark.parametrize("crossfade", XF)
@pytest.mark.parametrize("shared", [False, True], ids=["item", "shared"])
def test_tv_mc_fixed_ir_skips_the_ir_gradient(cuda_device, crossfade, shared):
    x, ir, w = _inputs(3, 3, 6, 3, 40000, 30000, seed=53, shared=shared)
    full = _gpu(x, ir, w, 2 * KB, cuda_device, crossfade)
    fixed = _gpu(x, ir, w, 2 * KB, cuda_device, crossfade, ir_grad=False)
    assert _path() == _bits(crossfade, 3, shared, 6, ir_grad=False)
    assert fixed[2] is None
    assert torch.equal(fixed[0], full[0]) and torch.equal(fixed[1], full[1])


@pytest.mark.parametrize("crossfade", XF)
@pytest.mark.parametrize("S,M,shared,K,n,L", [(3, 5, False, 3, 20000, 15001), (5, 8, True, 2, 20000, 15001),
                                              (2, 3, False, 15, 70000, 66000)])
def test_tv_mc_ignores_prior_buffer_contents(cuda_device, crossfade, S, M, shared, K, n, L):
    """NaN in both workspaces, the saved spectra and the outputs reaches no result"""
    from dasp_pytorch_b200 import _abi
    lib, dev = _lib(), cuda_device
    bs, chunk, hop = 3, 2, KB
    p = "dasp_tvmc" if crossfade == "output" else "dasp_tvmc_in"
    g = _abi.ConvGeom()
    _abi.check(getattr(lib, f"{p}_geometry")(bs, n, L, K, S, M, hop, int(shared), chunk, g), "geom")
    kind = f"{p}_shared" if shared else p
    fwd, bwd = getattr(lib, f"{kind}_fwd"), getattr(lib, f"{kind}_bwd")
    x, ir, w = _inputs(bs, S, M, K, n, L, seed=59, shared=shared)
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
                       g.fwd_workspace_bytes, bs, n, L, K, S, M, hop, chunk, _abi.stream_ptr(dev)), "fwd")
        gx = filled(bs * S * n, torch.float32, fill)
        gir = filled(ir.numel(), torch.float32, fill)
        wb = filled(g.bwd_workspace_bytes // 4, torch.float32, fill)
        _abi.check(bwd(_abi.ptr(gy), _abi.ptr(xs), _abi.ptr(hs), _abi.ptr(gx), _abi.ptr(gir), _abi.ptr(wb),
                       g.bwd_workspace_bytes, bs, n, L, K, S, M, hop, chunk, _abi.stream_ptr(dev)), "bwd")
        assert _path() == _bits(crossfade, K, shared, M)
        torch.cuda.synchronize(dev)
        return y, gx, gir

    clean, dirty = run(0.0), run(float("nan"))
    for a, b in zip(clean, dirty):
        assert bool(torch.isfinite(b).all())
        assert torch.equal(a, b)


@pytest.mark.parametrize("crossfade", XF)
@pytest.mark.parametrize("shared", [False, True], ids=["item", "shared"])
def test_tv_mc_cuda_graph_replay_matches_eager(cuda_device, crossfade, shared):
    import dasp_pytorch_b200 as D
    dev, K, hop = cuda_device, 3, 4 * KB
    x, ir, w = (t.float().to(dev) for t in _inputs(3, 4, 8, K, 48000, 24000, seed=67, shared=shared))
    x.requires_grad_(True)
    ir.requires_grad_(True)

    def step():
        y = D.time_varying_multichannel_convolution(x, SR, ir, hop, crossfade=crossfade)
        return (y.detach(),) + torch.autograd.grad((y * w).sum(), (x, ir))

    eager = [t.clone() for t in step()]
    assert _path() == _bits(crossfade, K, shared, 8)
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


@pytest.mark.parametrize("crossfade", XF)
def test_tv_mc_bf16_is_the_rounded_fp32_result(cuda_device, crossfade):
    import dasp_pytorch_b200 as D
    dev = cuda_device
    x, ir, _ = _inputs(2, 5, 7, 3, 10001, 7000, seed=71, shared=False)
    xb, hb = x.to(dev, torch.bfloat16), ir.to(dev, torch.bfloat16)
    y = D.time_varying_multichannel_convolution(xb, SR, hb, KB, crossfade=crossfade)
    assert _path()[0] == _bits(crossfade, 3, False, 7)[0]
    assert y.dtype == torch.bfloat16 and y.shape == (2, 7, 10001)
    ref = D.time_varying_multichannel_convolution(xb.float(), SR, hb.float(), KB, crossfade=crossfade)
    assert torch.equal(y, ref.to(torch.bfloat16))
