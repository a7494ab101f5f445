"""Every op at the sample rates of high-resolution sessions (44.1 to 192 kHz), held to the fp64 oracle.

At 192 kHz a 20 Hz shelf has its poles within 3e-5 of the unit circle and a 100 ms attack has alpha = 1 - 1.1e-4: the
filters' state decays over hundreds of thousands of samples and the coefficients carry their information in their
distance from 1.  The EQ runs a fixed corner grid (20 Hz low shelf, 80 Hz band 0, band 3 and the high shelf at
sr/2 - 1000, Q 0.1 / 0.707 / 6, +-20 dB, and both low sections at +-20 dB with Q 6) at the automatic warp count and at forced W = 1 and 16, forward and backward,
to the strict 1e-4 of test_gpu_eq._check(strict=True); its frequency response runs the same corners.  The compressor,
expander and compressor_gain run attack 5 and 100 ms at 176.4 and 192 kHz; the reverb and noise_shaped_impulse_response
run at 96 kHz with the caller's noise, where the octave filter bank changes with the rate.

Arbiter: the oracle on CUDA fp64 tensors (tests/long_oracle.py), with the frequency-sampling grid extended past the
slowest pole.  The loss is <y, r> with a fixed random cotangent r.  Every pin prints a "PIN <case>:" line.
"""
import functools

import pytest
import torch

import conv_oracle
import dyn_gain_oracle
import long_oracle as lo
import oracle
from eq_response_oracle import log_grid, parametric_eq_response
from test_gpu_dynamics_pin import forced_warps

pytestmark = pytest.mark.gpu
TOL = 1e-4
EQ_RATES = [44100, 48000, 96000, 176400, 192000]
EQ_N = 1 << 17


def _D():
    import dasp_pytorch_b200 as D
    return D


def eq_corner_params(sr):
    """one item per (Q, gain): every section at that Q, the gain alternating in sign from section to section; and one
    item per gain with the 20 Hz shelf and the 80 Hz band both at that gain and Q 6, the worst-conditioned cascade"""
    hi = sr // 2 - 1000
    freqs = [20.0, 80.0, 4000.0, 10000.0, float(hi), float(hi)]
    items = [(q, [g if k % 2 == 0 else -g for k in range(6)]) for q in (0.1, 0.707, 6.0) for g in (-20.0, 20.0)]
    items += [(6.0, [g, g, -g, g, -g, g]) for g in (-20.0, 20.0)]
    params = [[] for _ in range(18)]
    for q, gains in items:
        for k in range(6):
            params[3 * k].append(gains[k])
            params[3 * k + 1].append(freqs[k])
            params[3 * k + 2].append(q)
    return [torch.tensor(p, dtype=torch.float32) for p in params]


def _eq_inputs(sr, chs=2, n=EQ_N):
    params = eq_corner_params(sr)
    bs = params[0].numel()
    g = torch.Generator().manual_seed(sr)
    x = torch.rand(bs, chs, n, generator=g) * 2 - 1
    r = torch.randn(bs, chs, n, generator=g)
    return x, params, r


@functools.lru_cache(maxsize=1)           # the cases run rate by rate: keep one rate's fp64 reference
def _eq_ref(sr, device):
    x, params, r = _eq_inputs(sr)
    tail = lo.eq_tail(sr, params)
    ref = lo.vjp(lambda xx, pp: oracle.parametric_eq(xx, sr, *pp, fsm_tail=tail), x, params, r, device, group=2)
    return ref, tail


@pytest.mark.parametrize("w", [0, 1, 16], ids=["Wauto", "W1", "W16"])
@pytest.mark.parametrize("sr", EQ_RATES)
def test_eq_corners(cuda_device, sr, w):
    """W = 16 exists for the forward only; the backward keeps its own choice there"""
    x, params, r = _eq_inputs(sr)
    lo.need_memory(24 * x.numel() * 8, cuda_device)
    ref, tail = _eq_ref(sr, cuda_device)
    with forced_warps(w):
        got = lo.gpu(lambda xx, pp: _D().parametric_eq(xx, sr, *pp), x, params, r, cuda_device)
    lo.pin(f"eq-{sr}Hz-W{w or 'auto'}-tail{tail}", got, ref)


@pytest.mark.parametrize("sr", EQ_RATES)
def test_eq_response_corners(cuda_device, sr):
    """the response per bin against the fp64 product of the designed sections, on a log grid from 10 Hz to sr/2"""
    params = eq_corner_params(sr)
    f = log_grid(sr, n=2048)
    h = _D().parametric_eq_frequency_response(sr, *[p.to(cuda_device) for p in params], frequencies=f).cpu()
    ref = parametric_eq_response(sr, *[p.double() for p in params], frequencies=f)
    err = (h.to(torch.complex128) - ref).abs() / ref.abs()
    print(f"PIN eq_response-{sr}Hz: per-bin {float(err.max()):.2e}")
    assert float(err.max()) <= 5e-5


def _dyn_inputs(kind, n, seed):
    g = torch.Generator().manual_seed(seed)
    bs = 4
    x = (torch.rand(bs, 2, n, generator=g) * 2 - 1) * (0.05 + 0.95 * torch.rand(bs, 1, 1, generator=g))
    side = x.sum(1).abs().median(1).values
    params = [(20 * torch.log10(side) + torch.rand(bs, generator=g) * 12 - 6).float(),
              1.0 + torch.rand(bs, generator=g) * (19.0 if kind == "comp" else 3.0),
              torch.tensor([5.0, 100.0, 5.0, 100.0]),
              torch.full((bs,), 50.0),
              0.6 + 11.4 * torch.rand(bs, generator=g),
              12.0 * torch.rand(bs, generator=g)]
    return x, params, torch.randn(bs, 2, n, generator=g)


@pytest.mark.parametrize("w", [1, 16])
@pytest.mark.parametrize("sr", [176400, 192000])
@pytest.mark.parametrize("kind", ["comp", "exp"])
def test_dynamics_high_rates(cuda_device, kind, sr, w):
    """attack 5 and 100 ms: alpha up to 1 - 1.1e-4 through the power tables and the tile-to-tile carry"""
    n = 3 * sr // 2 + (0 if w == 16 else 1)
    x, params, r = _dyn_inputs(kind, n, seed=sr + w)
    tail = lo.dyn_tail(sr, 100.0)
    orc = oracle.compressor if kind == "comp" else oracle.expander
    ref = lo.vjp(lambda xx, pp: orc(xx, sr, *pp, fsm_tail=tail), x, params, r, cuda_device)
    fn = _D().compressor if kind == "comp" else _D().expander
    with forced_warps(w):
        got = lo.gpu(lambda xx, pp: fn(xx, sr, *pp), x, params, r, cuda_device)
    assert got[2][3] is None and ref[2][3] is None
    lo.pin(f"{kind}-{sr}Hz-W{w}", got, ref)


@pytest.mark.parametrize("db", [False, True])
@pytest.mark.parametrize("sr", [176400, 192000])
def test_compressor_gain_high_rates(cuda_device, sr, db):
    n = 3 * sr // 2
    x, params, _ = _dyn_inputs("comp", n, seed=sr + db)
    r = torch.randn(x.shape[0], 1, n, generator=torch.Generator().manual_seed(sr))
    tail = lo.dyn_tail(sr, 100.0)
    ref = lo.vjp(lambda xx, pp: dyn_gain_oracle.compressor_gain(xx, sr, *pp, fsm_tail=tail, db=db), x, params, r,
                 cuda_device)
    got = lo.gpu(lambda xx, pp: _D().compressor_gain(xx, sr, *pp, db=db), x, params, r, cuda_device)
    lo.pin(f"compressor_gain-{sr}Hz-db{db}", got, ref)


def _reverb_params(bs, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.rand(bs, generator=g) for _ in range(25)]


@pytest.mark.parametrize("n,L", [(96000, 96000), (200001, 48000)])
def test_reverb_96k_parity(cuda_device, n, L):
    """the reverb with the caller's noise: the 1023-tap octave filter bank designed at 96 kHz"""
    sr, taps, bs = 96000, 1023, 3
    g = torch.Generator().manual_seed(n + L)
    x = torch.rand(bs, 2, n, generator=g) * 2 - 1
    noise = torch.randn(bs * 2, 12, L + taps - 1, generator=g)
    params = _reverb_params(bs, n)
    r = torch.randn(bs, 2, n, generator=g)
    nd = noise.to(cuda_device)
    ref = lo.vjp(lambda xx, pp: oracle.noise_shaped_reverberation(xx, sr, *pp, num_samples=L, num_bandpass_taps=taps,
                                                                  noise=nd), x, params, r, cuda_device)
    got = lo.gpu(lambda xx, pp: _D().noise_shaped_reverberation(xx, sr, *pp, num_samples=L, num_bandpass_taps=taps,
                                                               noise=nd), x, params, r, cuda_device)
    lo.pin(f"reverb-96kHz-n{n}-L{L}", got, ref)


@pytest.mark.parametrize("L", [96000, 192001])
def test_nsir_96k_parity(cuda_device, L):
    sr, taps, bs = 96000, 1023, 3
    g = torch.Generator().manual_seed(L)
    noise = torch.randn(bs * 2, 12, L + taps - 1, generator=g)
    params = _reverb_params(bs, L)[:24]
    r = torch.randn(bs, 2, L, generator=g)
    nd = noise.to(cuda_device)
    ref = lo.param_vjp(lambda pp: conv_oracle.reverb_ir(sr, pp, nd, L, taps), params, r, cuda_device)
    got = lo.param_vjp(lambda pp: _D().noise_shaped_impulse_response(sr, *pp, num_samples=L, num_bandpass_taps=taps,
                                                                    noise=nd), params, r, cuda_device, torch.float32)
    lo.pin(f"nsir-96kHz-L{L}", got, ref, names=("ir", None))
