"""time_varying_convolution_reverberation on the GPU: y, dL/dx, dL/dIR and dL/dmix pinned to the fp64 oracle
(tests/tv_conv_oracle.py) for mono and stereo x and IRs, per-item and shared trajectories, K from 1 to 15, anchor
spacings of 1, 3 and 8 partitions, IRs shorter than, longer than and as long as x, padded rows, the L2-sized products and
a minute of audio; the identities with convolution_reverberation; the same bits for every chunk size, a fixed
trajectory, stale buffers, CUDA-graph replay and bf16.  Every case asserts the path bits it reached
(dasp_debug_tvconv_last_path)."""
import pytest
import torch

import tv_conv_oracle
from helpers import SR, peak_err

pytestmark = pytest.mark.gpu
BOUND = 1e-4
KB = 4096

# (in_chs, ir_chs, shared, K, hop, n, L)
CASES = [
    (2, 2, False, 1, KB, 20000, 9000),              # K = 1
    (1, 2, True, 2, KB, 9001, 3000),                # n % 4 = 1, L < hop
    (2, 1, False, 5, 3 * KB, 60002, 15000),         # n % 4 = 2, L > hop
    (1, 1, True, 5, 3 * KB, 50003, 60000),          # n % 4 = 3, L >= n
    (2, 2, True, 15, KB, 70000, 66000),             # I = 18, J = 17
    (2, 1, True, 2, 8 * KB, 40000, 5000),
    (1, 2, False, 15, KB, 61540, 20000),
    (2, 2, False, 3, 8 * KB, 100000, 40000),
    (1, 1, False, 2, KB, 8192, 8192),
    (2, 1, True, 1, KB, 5000, 100),
    (1, 2, True, 5, 8 * KB, 140000, 30000),
    (2, 2, False, 5, 3 * KB, 70001, 70001),         # L = n, n % 4 = 1
]


def _ids(c):
    return f"x{c[0]}-h{c[1]}-{'sh' if c[2] else 'it'}-K{c[3]}-hop{c[4] // KB}-{c[5]}-{c[6]}"


def _lib():
    from dasp_pytorch_b200 import _abi
    return _abi.lib()


def _bits(K, shared, ir_grad=True):
    """expected (forward, backward) path bits"""
    cross = K > 1
    return (1 | (2 if shared else 0) | (4 if cross else 0),
            1 | (2 if cross else 0) | (4 if ir_grad else 0) | (8 if shared else 0))


def _path():
    lib = _lib()
    return lib.dasp_debug_tvconv_last_path(0), lib.dasp_debug_tvconv_last_path(1)


def _inputs(bs, in_chs, ir_chs, K, n, L, seed, shared):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(bs, in_chs, n, generator=g, dtype=torch.float64) * 2 - 1
    ir = (torch.rand(1 if shared else bs, K, ir_chs, L, generator=g, dtype=torch.float64) * 2 - 1) * torch.exp(
        -torch.arange(L, dtype=torch.float64) / max(L / 4, 1.0))
    mix = torch.rand(bs, generator=g, dtype=torch.float64)
    w = torch.rand(bs, 2, n, generator=g, dtype=torch.float64) * 2 - 1          # loss = sum(w y)
    return x, ir, mix, w


def _run(fn, x, ir, mix, w, device, dtype, ir_grad=True):
    xx = x.to(device=device, dtype=dtype).requires_grad_(True)
    hh = ir.to(device=device, dtype=dtype).requires_grad_(ir_grad)
    mm = mix.to(device=device, dtype=dtype).requires_grad_(True)
    y = fn(xx, hh, mm)
    (y * w.to(device=device, dtype=dtype)).sum().backward()
    return (y.detach().cpu(), xx.grad.cpu(), None if hh.grad is None else hh.grad.cpu(), mm.grad.cpu())


def _gpu(x, ir, mix, w, hop, dev, **kw):
    import dasp_pytorch_b200 as D
    return _run(lambda a, h, m: D.time_varying_convolution_reverberation(a, SR, h, hop, m), x, ir, mix, w, dev,
                torch.float32, **kw)


def _ref(x, ir, mix, w, hop):
    return _run(lambda a, h, m: tv_conv_oracle.time_varying_convolution_reverberation(a, SR, h, hop, m), x, ir, mix,
                w, "cpu", torch.float64)


def _errs(got, ref):
    """y and dL/dx per item; dL/dIR per item (or the shared trajectory) on its own largest fp64 gradient; dL/dmix on the
    largest fp64 dL/dmix"""
    return {"y": peak_err(got[0], ref[0]), "dx": peak_err(got[1], ref[1]), "dir": peak_err(got[2], ref[2]),
            "dmix": (got[3].double() - ref[3]).abs().max() / ref[3].abs().max()}


def _check(got, ref, label):
    errs = _errs(got, ref)
    for k, e in errs.items():
        assert float(e.max()) < BOUND, (label, k, e)
    print(f"{label}: " + " ".join(f"{k} {float(e.max()):.2e}" for k, e in errs.items()))


@pytest.mark.parametrize("in_chs,ir_chs,shared,K,hop,n,L", CASES, ids=[_ids(c) for c in CASES])
def test_tv_pinned_to_oracle(cuda_device, monkeypatch, in_chs, ir_chs, shared, K, hop, n, L):
    """bs 3 in chunks of 2: y, dL/dx, dL/dIR and dL/dmix within 1e-4 of the fp64 oracle; taps >= n get exactly 0"""
    from dasp_pytorch_b200 import functional as F
    monkeypatch.setattr(F, "REVERB_CHUNK_ITEMS", 2)
    x, ir, mix, w = _inputs(3, in_chs, ir_chs, K, n, L, seed=K * 100 + n % 97 + in_chs + 4 * ir_chs + shared,
                            shared=shared)
    got = _gpu(x, ir, mix, w, hop, cuda_device)
    assert _path() == _bits(K, shared)
    assert got[0].shape == (3, 2, n) and got[1].shape == x.shape and got[2].shape == ir.shape
    if L > n:
        assert bool((got[2][..., n:] == 0).all())
    _check(got, _ref(x, ir, mix, w, hop), _ids((in_chs, ir_chs, shared, K, hop, n, L)))


def test_tv_pinned_to_oracle_on_a_minute_of_audio(cuda_device):
    """60 s at 48 kHz, 15 anchors 48 partitions apart, a one-second stereo trajectory"""
    n, L, K, hop = 60 * 48000, 48000, 15, 48 * KB
    x, ir, mix, w = _inputs(1, 2, 2, K, n, L, seed=61, shared=False)
    got = _gpu(x, ir, mix, w, hop, cuda_device)
    assert _path() == _bits(K, False)
    _check(got, _ref(x, ir, mix, w, hop), "60 s")


def _rel(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max())


@pytest.mark.parametrize("shared", [False, True], ids=["item", "shared"])
@pytest.mark.parametrize("in_chs,ir_chs", [(2, 2), (1, 1)])
def test_tv_identities_with_convolution_reverberation(cuda_device, shared, in_chs, ir_chs):
    """(1) K = 1 is convolution_reverberation(x, sr, h[:, 0], mix); (2) K equal IRs are that IR's static convolution,
    and the K IR gradients sum to the static one; (3) after the last anchor the output is the static convolution with
    h_K-1.  Different kernels, so they agree to fp32 rounding"""
    import dasp_pytorch_b200 as D
    dev = cuda_device
    n, L, hop = 60000, 20000, 3 * KB
    worst = {}

    def conv(x, h, mix, w):
        return _run(lambda a, hh, m: D.convolution_reverberation(a, SR, hh, m), x, h, mix, w, dev, torch.float32)

    x, ir, mix, w = _inputs(3, in_chs, ir_chs, 1, n, L, seed=71 + shared, shared=shared)
    tv = _gpu(x, ir, mix, w, hop, dev)
    assert _path() == _bits(1, shared)
    ref = conv(x, ir[:, 0], mix, w)
    for k, a, b in zip(("y", "dx", "dir", "dmix"), tv, ref):
        worst[("K1", k)] = _rel(a.reshape(b.shape), b)

    K = 4
    tv = _gpu(x, ir.expand(-1, K, -1, -1).contiguous(), mix, w, hop, dev)
    assert _path() == _bits(K, shared)
    for k, a, b in zip(("y", "dx", "dir", "dmix"), (tv[0], tv[1], tv[2].sum(1), tv[3]), ref):
        worst[("equal", k)] = _rel(a, b)

    _, ir4, _, _ = _inputs(3, in_chs, ir_chs, K, n, L, seed=73 + shared, shared=shared)
    tv = _gpu(x, ir4, mix, w, hop, dev)
    last = conv(x, ir4[:, K - 1], mix, w)
    worst[("last", "y")] = _rel(tv[0][..., (K - 1) * hop:], last[0][..., (K - 1) * hop:])
    for key, e in worst.items():
        assert e < 1e-5, (key, e)
    print(f"identities x{in_chs} h{ir_chs} {'shared' if shared else 'item'}: worst "
          + " ".join(f"{a}-{b} {e:.1e}" for (a, b), e in worst.items()))


@pytest.mark.parametrize("shared", [False, True], ids=["item", "shared"])
def test_tv_same_bits_for_every_chunk(cuda_device, monkeypatch, shared):
    from dasp_pytorch_b200 import functional as F
    x, ir, mix, w = _inputs(5, 2, 2, 5, 40000, 15000, seed=81 + shared, shared=shared)
    runs = []
    for chunk in (1, 2, 5, 3):
        monkeypatch.setattr(F, "REVERB_CHUNK_ITEMS", chunk)
        runs.append(_gpu(x, ir, mix, w, 2 * KB, cuda_device))
        assert _path() == _bits(5, shared)
    for r in runs[1:]:
        for a, b in zip(r, runs[0]):
            assert torch.equal(a, b)


@pytest.mark.parametrize("shared", [False, True], ids=["item", "shared"])
def test_tv_fixed_trajectory_skips_the_ir_gradient(cuda_device, shared):
    x, ir, mix, w = _inputs(3, 2, 1, 3, 30000, 15000, seed=83, shared=shared)
    full = _gpu(x, ir, mix, w, KB, cuda_device)
    fixed = _gpu(x, ir, mix, w, KB, cuda_device, ir_grad=False)
    assert _path() == _bits(3, shared, ir_grad=False)
    assert fixed[2] is None
    for i in (0, 1, 3):
        assert torch.equal(fixed[i], full[i])


@pytest.mark.parametrize("shared", [False, True], ids=["item", "shared"])
def test_tv_ignores_prior_buffer_contents(cuda_device, shared):
    """NaN in both workspaces, the saved spectra and the outputs reaches no result"""
    from dasp_pytorch_b200 import _abi
    lib, dev = _lib(), cuda_device
    bs, n, L, K, C, hop, chunk = 3, 40000, 15001, 5, 2, 2 * KB, 2
    g = _abi.ConvGeom()
    _abi.check(lib.dasp_tvconv_geometry(bs, n, L, K, C, hop, int(shared), chunk, g), "geom")
    fwd, bwd = ((lib.dasp_tvconv_shared_fwd, lib.dasp_tvconv_shared_bwd) if shared
                else (lib.dasp_tvconv_fwd, lib.dasp_tvconv_bwd))
    x, ir, mix, w = _inputs(bs, 2, C, K, n, L, seed=87, shared=shared)
    x, ir, mix, gy = (t.float().to(dev).contiguous() for t in (x, ir, mix, w))

    def filled(numel, dtype, fill):
        t = torch.empty(numel, dtype=dtype, device=dev)
        t.view(torch.float32).fill_(fill)
        return t

    def run(fill):
        y = filled(bs * 2 * n, torch.float32, fill)
        ws = filled(g.fwd_workspace_bytes // 4, torch.float32, fill)
        xs, hs = filled(g.xspec_c64, torch.complex64, fill), filled(g.irspec_c64, torch.complex64, fill)
        _abi.check(fwd(_abi.ptr(x), 2, _abi.ptr(ir), C, L, K, hop, _abi.ptr(mix), _abi.ptr(y), _abi.ptr(xs),
                       _abi.ptr(hs), _abi.ptr(ws), g.fwd_workspace_bytes, bs, n, chunk, _abi.stream_ptr(dev)), "fwd")
        gx = filled(bs * 2 * n, torch.float32, fill)
        gir = filled(ir.numel(), torch.float32, fill)
        gmix = filled(bs, torch.float32, fill)
        wb = filled(g.bwd_workspace_bytes // 4, torch.float32, fill)
        _abi.check(bwd(_abi.ptr(gy), _abi.ptr(x), 2, C, L, K, hop, _abi.ptr(mix), _abi.ptr(xs), _abi.ptr(hs),
                       _abi.ptr(gx), _abi.ptr(gir), _abi.ptr(gmix), _abi.ptr(wb), g.bwd_workspace_bytes, bs, n, chunk,
                       _abi.stream_ptr(dev)), "bwd")
        assert _path() == _bits(K, shared)
        torch.cuda.synchronize(dev)
        return y, gx, gir, gmix

    clean, dirty = run(0.0), run(float("nan"))
    for a, b in zip(clean, dirty):
        assert bool(torch.isfinite(b).all())
        assert torch.equal(a, b)


@pytest.mark.parametrize("shared", [False, True], ids=["item", "shared"])
def test_tv_cuda_graph_replay_matches_eager(cuda_device, shared):
    import dasp_pytorch_b200 as D
    dev = cuda_device
    x, ir, mix, w = (t.float().to(dev) for t in _inputs(3, 2, 2, 5, 48000, 20000, seed=91, shared=shared))
    for t in (x, ir, mix):
        t.requires_grad_(True)

    def step():
        y = D.time_varying_convolution_reverberation(x, SR, ir, 2 * KB, mix)
        return (y.detach(),) + torch.autograd.grad((y * w).sum(), (x, ir, mix))

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


def test_tv_bf16_is_the_rounded_fp32_result(cuda_device):
    import dasp_pytorch_b200 as D
    dev = cuda_device
    x, ir, mix, _ = _inputs(2, 2, 2, 3, 20000, 7000, seed=97, shared=False)
    xb, hb, mb = x.to(dev, torch.bfloat16), ir.to(dev, torch.bfloat16), mix.to(dev, torch.bfloat16)
    y = D.time_varying_convolution_reverberation(xb, SR, hb, KB, mb)
    assert _path()[0] == _bits(3, False)[0]
    assert y.dtype == torch.bfloat16
    ref = D.time_varying_convolution_reverberation(xb.float(), SR, hb.float(), KB, mb.float()).to(torch.bfloat16)
    assert torch.equal(y, ref)
