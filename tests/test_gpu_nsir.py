"""noise_shaped_impulse_response on the GPU: the IR and its 24 parameter gradients pinned per item to the fp64 oracle
(tests/conv_oracle.reverb_ir, the IR synthesis of the reference reverb) with the SURVEY.md 8c rule, with the caller's
noise and, through the unit-impulse filter hook (tests/reverb_pin.py), with the device noise of every synthesis path;
composed with convolution_reverberation it is the reverb, bit for bit; plus chunking, seeding, graph capture,
broadcasting, empty batches, bf16 parameters, no saved state for fixed parameters, and a short fit of the decays."""
from types import SimpleNamespace

import pytest
import torch

import conv_oracle
import oracle
import reverb_pin
from helpers import SR, param_grad_err, peak_err

pytestmark = pytest.mark.gpu
TOL = 1e-4


def _lib():
    from dasp_pytorch_b200 import _abi
    return _abi.lib()


def _params(bs, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.rand(bs, generator=g) for _ in range(24)]


def _weights(bs, L, seed):
    g = torch.Generator().manual_seed(seed + 1)
    return torch.rand(bs, 2, L, generator=g, dtype=torch.float64) * 2 - 1


def _gpu(dev, params, L, taps, w, noise=None):
    """IR and the 24 gradients of sum(w IR) on the GPU (fp32)"""
    import dasp_pytorch_b200 as D
    pp = [p.to(dev).clone().requires_grad_(True) for p in params]
    ir = D.noise_shaped_impulse_response(SR, *pp, num_samples=L, num_bandpass_taps=taps,
                                         noise=None if noise is None else noise.to(dev))
    (ir * w.to(dev, torch.float32)).sum().backward()
    return ir.detach().cpu().double(), torch.stack([p.grad.cpu() for p in pp], 1).double()


def _oracle(params, noise, L, taps, w, dtype):
    pp = [p.to(dtype).clone().requires_grad_(True) for p in params]
    ir = conv_oracle.reverb_ir(SR, pp, noise.to(dtype), L, taps, dtype=dtype)
    (ir * w.to(dtype)).sum().backward()
    return ir.detach().double(), torch.stack([p.grad for p in pp], 1).double()


def _pin(got, params, noise, L, taps, w):
    """per-item errors of IR and gradients against fp64, bounded by max(TOL, the reference's own fp32 error)"""
    ref = _oracle(params, noise, L, taps, w, torch.float64)
    errs = {"ir": peak_err(got[0], ref[0]), "dp": param_grad_err(list(got[1].T), list(ref[1].T))}
    if max(float(e.max()) for e in errs.values()) >= TOL:
        r32 = _oracle(params, noise, L, taps, w, torch.float32)
        bound = {"ir": peak_err(r32[0], ref[0]), "dp": param_grad_err(list(r32[1].T), list(ref[1].T))}
    else:
        bound = {k: torch.zeros_like(e) for k, e in errs.items()}
    for k, e in errs.items():
        assert bool((e < bound[k].clamp_min(TOL)).all()), (k, e.tolist(), bound[k].tolist())
    return errs


# L: one sample (the reference's one-point linspace is t = 0), L < taps, k * 4096, k * 4096 + 1, 48000, 96000
@pytest.mark.parametrize("taps", [1023, 31])
@pytest.mark.parametrize("L", [1, 500, 8192, 8193, 48000, 96000])
def test_nsir_parity_pinned_to_oracle(cuda_device, monkeypatch, L, taps):
    from dasp_pytorch_b200 import functional as F
    monkeypatch.setattr(F, "REVERB_CHUNK_ITEMS", 2)          # bs 3: a full chunk and a remainder
    bs = 3
    params = _params(bs, seed=L + taps)
    noise = torch.randn(bs * 2, 12, L + taps - 1, generator=torch.Generator().manual_seed(L), dtype=torch.float64)
    w = _weights(bs, L, L + taps)
    got = _gpu(cuda_device, params, L, taps, w, noise=noise.float())
    assert got[0].shape == (bs, 2, L)
    errs = _pin(got, params, noise.float().double(), L, taps, w)
    if L == 1:                                               # t = 0: the decays have no effect
        assert bool((got[1][:, 12:] == 0).all())
    print(f"NSIR parity L={L} taps={taps}: " + " ".join(f"{k} {float(e.max()):.2e}" for k, e in errs.items()))


def _geometry(bs, L, taps, chunk):
    from dasp_pytorch_b200 import _abi
    g = _abi.ReverbGeom()
    _abi.check(_lib().dasp_nsir_geometry(bs, L, taps, chunk, g), "dasp_nsir_geometry")
    return SimpleNamespace(**{name: int(getattr(g, name)) for name, _ in _abi.ReverbGeom._fields_})


# (L, taps, hook, expected dasp_debug_reverb_last_path, chunk): R = 6 cluster kernel, R = 12 generator +
# ifft_shape_kernel (one item per chunk: Philox keyed by the global item), hook 2, hook 1 (cuFFT), 2047 taps (nb =
# 16384, cuFFT polyphase), R = 17 (time-domain Philox, overlap-save)
PATHS = [(48000, 1023, 0, 2, None), (96000, 1023, 0, 2, 1), (48000, 1023, 2, 1, None), (48000, 1023, 1, 0, None),
         (30000, 2047, 0, 0, None), (132000, 1023, 0, 0, None)]


@pytest.mark.parametrize("L,taps,hook,expect,chunk", PATHS, ids=[f"{p[0]}-{p[1]}-hook{p[2]}" for p in PATHS])
def test_nsir_device_noise_pinned_on_every_path(cuda_device, monkeypatch, L, taps, hook, expect, chunk):
    from dasp_pytorch_b200 import functional as F
    import dasp_pytorch_b200 as D
    if chunk is not None:
        monkeypatch.setattr(F, "REVERB_CHUNK_ITEMS", chunk)
    lib = _lib()
    bs, seed = 2, 100 + L
    params = _params(bs, seed)
    geom = _geometry(bs, L, taps, F.reverb_chunk_items(cuda_device))
    assert geom.f_floats == bs * 12 * reverb_pin.pair_c64(geom) * 2
    r = reverb_pin.geometry(bs, L, L, taps, F.reverb_chunk_items(cuda_device))        # the reverb at n = L
    assert (r.rpp, r.nbk, r.f_floats) == (geom.rpp, geom.nbk, geom.f_floats)
    lib.dasp_debug_reverb_path(hook)
    try:
        lib.dasp_debug_reverb_flat_filterbank(1)
        try:
            torch.manual_seed(seed)
            pp = [p.to(cuda_device).requires_grad_(True) for p in params]
            ir = D.noise_shaped_impulse_response(SR, *pp, num_samples=L, num_bandpass_taps=taps)
            assert lib.dasp_debug_reverb_last_path() == expect
            fsave = ir.grad_fn.saved_tensors[1]
            assert fsave.numel() == geom.f_floats
            seqs = torch.stack([reverb_pin.unpack(reverb_pin.item_blocks(fsave, i, geom), geom).cpu() for i in range(bs)])
        finally:
            lib.dasp_debug_reverb_flat_filterbank(0)
        noise = reverb_pin.reference_noise(seqs, geom, L, taps)
        w = _weights(bs, L, seed)
        torch.manual_seed(seed)
        got = _gpu(cuda_device, params, L, taps, w)
        assert lib.dasp_debug_reverb_last_path() == expect
    finally:
        lib.dasp_debug_reverb_path(0)
    errs = _pin(got, params, noise, L, taps, w)
    print(f"NSIR device L={L} taps={taps} hook={hook}: " + " ".join(f"{k} {float(e.max()):.2e}" for k, e in errs.items()))


# (n, L, x channels, hook): cluster synthesis (R 6), n > L, R 12 (generator + ifft_shape_kernel), mono x, the cuFFT
# synthesis (hook 1), n % 4 != 0 (cuFFT convolution)
COMPOSE = [(48000, 48000, 2, 0), (60000, 40000, 2, 0), (96000, 96000, 2, 0), (48000, 30000, 1, 0), (48000, 48000, 2, 1),
           (48001, 40000, 2, 0)]


@pytest.mark.parametrize("n,L,chs,hook", COMPOSE, ids=[f"{c[0]}-{c[1]}-x{c[2]}-hook{c[3]}" for c in COMPOSE])
def test_nsir_composes_to_the_reverb_bit_for_bit(cuda_device, n, L, chs, hook):
    import dasp_pytorch_b200 as D
    lib = _lib()
    bs = 3
    g = torch.Generator().manual_seed(n + L)
    x = (torch.rand(bs, chs, n, generator=g) * 2 - 1).to(cuda_device)
    params = [p.to(cuda_device) for p in _params(bs, n)]
    mix = torch.rand(bs, generator=g).to(cuda_device)
    lib.dasp_debug_reverb_path(hook)
    try:
        torch.manual_seed(5)
        ir = D.noise_shaped_impulse_response(SR, *params, num_samples=L)
        y1 = D.convolution_reverberation(x, SR, ir, mix)
        torch.manual_seed(5)
        y2 = D.noise_shaped_reverberation(x, SR, *params, mix, num_samples=L)
    finally:
        lib.dasp_debug_reverb_path(0)
    assert torch.equal(y1, y2), float((y1 - y2).abs().max())


# parity mode: n >= L and n < L (the device noise of the two ops differs there by design: different polyphase factor)
@pytest.mark.parametrize("n,L", [(20000, 16000), (12000, 20000)])
def test_nsir_composition_gradients_pinned_to_oracle(cuda_device, n, L):
    import dasp_pytorch_b200 as D
    bs, taps = 2, 1023
    g = torch.Generator().manual_seed(n)
    x = torch.rand(bs, 2, n, generator=g, dtype=torch.float64) * 2 - 1
    params = [p.double() for p in _params(bs, n)] + [torch.rand(bs, generator=g, dtype=torch.float64)]
    noise = torch.randn(bs * 2, 12, L + taps - 1, generator=g, dtype=torch.float64).float().double()
    w = torch.rand(bs, 2, n, generator=g, dtype=torch.float64) * 2 - 1

    def run(fn, dev, dtype):
        xx = x.to(dev, dtype).requires_grad_(True)
        pp = [p.to(dev, dtype).requires_grad_(True) for p in params]
        y = fn(xx, pp, noise.to(dev, dtype))
        (y * w.to(dev, dtype)).sum().backward()
        return y.detach().cpu().double(), xx.grad.cpu().double(), torch.stack([p.grad.cpu() for p in pp], 1).double()

    def gpu(xx, pp, nz):
        ir = D.noise_shaped_impulse_response(SR, *pp[:24], num_samples=L, num_bandpass_taps=taps, noise=nz)
        return D.convolution_reverberation(xx, SR, ir, pp[24])

    def ref(xx, pp, nz):
        return oracle.noise_shaped_reverberation(xx, SR, *pp, num_samples=L, num_bandpass_taps=taps, noise=nz,
                                                 method="fft")

    got = run(gpu, cuda_device, torch.float32)
    r64 = run(ref, "cpu", torch.float64)
    errs = {"y": peak_err(got[0], r64[0]), "dx": peak_err(got[1], r64[1]),
            "dp": param_grad_err(list(got[2].T), list(r64[2].T))}
    for k, e in errs.items():
        assert float(e.max()) < TOL, (k, e.tolist())


def _ir(dev, params, L=20000, taps=1023, seed=None, **kw):
    import dasp_pytorch_b200 as D
    if seed is not None:
        torch.manual_seed(seed)
    return D.noise_shaped_impulse_response(SR, *params, num_samples=L, num_bandpass_taps=taps, **kw)


def test_nsir_chunking_does_not_change_a_bit(cuda_device, monkeypatch):
    from dasp_pytorch_b200 import functional as F
    bs, L = 5, 40000
    params = _params(bs, 9)
    w = _weights(bs, L, 9)
    out = []
    for chunk in (0, 1, 2):
        monkeypatch.setattr(F, "REVERB_CHUNK_ITEMS", chunk)
        torch.manual_seed(21)
        out.append(_gpu(cuda_device, params, L, 1023, w))
    for a in out[1:]:
        assert torch.equal(a[0], out[0][0]) and torch.equal(a[1], out[0][1])


def test_nsir_seeding(cuda_device):
    params = [p.to(cuda_device) for p in _params(2, 4)]
    a, b, c = _ir(cuda_device, params, seed=1), _ir(cuda_device, params, seed=1), _ir(cuda_device, params, seed=2)
    assert torch.equal(a, b)
    assert float((a - c).abs().max()) > 1e-3 * float(a.abs().max())
    # one item's IR does not depend on the others (Philox is keyed on the global item index)
    d = _ir(cuda_device, [p[:1] for p in params], seed=1)
    assert torch.equal(d[0], a[0])


def test_nsir_graph_replay(cuda_device):
    bs, L = 3, 30000
    p = torch.rand(bs, 24, device=cuda_device).requires_grad_(True)
    w = torch.rand(bs, 2, L, device=cuda_device)
    from dasp_pytorch_b200 import functional as F

    def step():
        ir = F.noise_shaped_impulse_response_packed(SR, p, num_samples=L)
        (ir * w).sum().backward()
        return ir

    def eager(seed):
        p.grad = None
        torch.manual_seed(seed)
        ir = step()
        return ir.detach().clone(), p.grad.clone()

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            eager(0)
    torch.cuda.current_stream().wait_stream(side)
    ref = eager(11)
    p.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        irs = step()
    outs = []
    for seed in (11, None):
        with torch.no_grad():
            p.grad.zero_()
        if seed is not None:
            torch.manual_seed(seed)
        graph.replay()
        torch.cuda.synchronize()
        outs.append((irs.detach().clone(), p.grad.clone()))
    for a, b in zip(outs[0], ref):
        assert torch.equal(a, b)
    assert float((outs[1][0] - outs[0][0]).abs().max()) > 1e-3 * float(outs[0][0].abs().max())


def test_nsir_broadcast_parameters(cuda_device):
    bs = 3
    full = [p.to(cuda_device) for p in _params(bs, 6)]
    mixed = [p if k % 2 else p[:1].reshape(1, 1) for k, p in enumerate(full)]       # every other one broadcast
    expanded = [p if k % 2 else p[:1].expand(bs) for k, p in enumerate(full)]
    pm = [p.clone().requires_grad_(True) for p in mixed]
    a = _ir(cuda_device, pm, seed=3)
    b = _ir(cuda_device, expanded, seed=3)
    assert a.shape == (bs, 2, 20000) and torch.equal(a, b)
    a.sum().backward()
    assert all(p.grad.shape == p.shape for p in pm)
    packed = torch.stack([p.reshape(-1).expand(bs) for p in mixed], 1)
    from dasp_pytorch_b200 import functional as F
    torch.manual_seed(3)
    assert torch.equal(F.noise_shaped_impulse_response_packed(SR, packed, num_samples=20000), a)


def test_nsir_empty_batch(cuda_device):
    params = [torch.zeros(0, device=cuda_device, requires_grad=True) for _ in range(24)]
    ir = _ir(cuda_device, params, seed=1)
    assert ir.shape == (0, 2, 20000)
    ir.sum().backward()
    assert all(p.grad.shape == (0,) for p in params)


def test_nsir_bf16_parameters(cuda_device):
    params = [p.to(cuda_device, torch.bfloat16).requires_grad_(True) for p in _params(2, 8)]
    ir = _ir(cuda_device, params, seed=4)
    assert ir.dtype == torch.bfloat16
    ref = _ir(cuda_device, [p.detach().float() for p in params], seed=4)
    assert torch.equal(ir, ref.to(torch.bfloat16))
    ir.float().sum().backward()
    assert all(p.grad.dtype == torch.bfloat16 and torch.isfinite(p.grad.float()).all() for p in params)
    assert _ir(cuda_device, [p.detach().double() for p in params], seed=4).dtype == torch.float64


def test_nsir_fixed_parameters_keep_nothing(cuda_device):
    params = [p.to(cuda_device) for p in _params(2, 10)]
    ir = _ir(cuda_device, params, seed=4)
    assert ir.grad_fn is None and not ir.requires_grad
    pg = [p.clone().requires_grad_(k == 3) for k, p in enumerate(params)]
    ir2 = _ir(cuda_device, pg, seed=4)
    assert torch.equal(ir, ir2.detach())
    assert ir2.grad_fn is not None
    # the no-grad forward keeps no f_save: its allocations are the output and the workspace only
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    ir3 = _ir(cuda_device, params, L=96000, seed=4)
    kept = torch.cuda.memory_allocated() - base
    assert kept == ir3.numel() * 4, kept


def _edc(ir):
    """energy-decay curve in dB: 10 log10 of the backward-integrated energy, normalised to its start"""
    e = torch.flip(torch.cumsum(torch.flip(ir.pow(2), [-1]), -1), [-1])
    return 10 * torch.log10(e / e[..., :1] + 1e-12)


def test_nsir_fit_recovers_decays(cuda_device):
    """IR estimation in miniature: with fixed caller noise, Adam on the 24 parameters fits the per-band energy-decay
    curves of a target room and recovers its 12 decays.  Item k of a batch of 12 isolates band k (its gain row is the
    k-th unit vector times 12, a constant), the 12 decays are one broadcast element each, and the loss is the squared
    difference of the items' energy-decay curves; the curves do not depend on the gains, so their gradient is ~0."""
    import dasp_pytorch_b200 as D
    L, taps, steps = 24000, 255, 200
    g = torch.Generator().manual_seed(0)
    noise = torch.randn(2, 12, L + taps - 1, generator=g).repeat(12, 1, 1).to(cuda_device)
    target = torch.rand(12, generator=g) * 0.6 + 0.2
    unit = torch.eye(12, device=cuda_device) * 12.0

    def edcs(gains, decays):
        ir = D.noise_shaped_impulse_response(SR, *gains, *decays, num_samples=L, num_bandpass_taps=taps, noise=noise)
        return _edc(ir)[..., : L // 2]

    fixed_gains = [unit[:, j] for j in range(12)]
    with torch.no_grad():
        ref = edcs(fixed_gains, [t.reshape(1).to(cuda_device) for t in target])
        start = edcs(fixed_gains, [torch.full((1,), 0.5, device=cuda_device)] * 12)
    gains = [unit[:, j].clone().requires_grad_(True) for j in range(12)]
    decays = [torch.full((1,), 0.5, device=cuda_device, requires_grad=True) for _ in range(12)]
    opt = torch.optim.Adam(gains + decays, lr=0.03)
    for i in range(steps):
        for group in opt.param_groups:
            group["lr"] = 0.03 * (1 - i / steps)
        opt.zero_grad()
        loss = (edcs(gains, decays) - ref).pow(2).mean()
        loss.backward()
        opt.step()
    got = torch.cat([d.detach().cpu() for d in decays])
    assert float(loss) < 1e-3 * float((start - ref).pow(2).mean()), (float(loss), float((start - ref).pow(2).mean()))
    assert float((got - target).abs().max()) < 0.01, (got.tolist(), target.tolist())
