"""fp64 restatement of convolution_reverberation for the tests, and the impulse response the reverb oracle builds.

``convolution_reverberation`` is the apply stage of the reference's reverb (functional.py:569-575) with the IR given;
``reverb_ir`` is the IR synthesis of ``oracle.noise_shaped_reverberation`` (functional.py:547-567).  Composed, they
equal ``oracle.noise_shaped_reverberation`` (tests/test_conv_reverb_host.py checks it on the reference goldens), which
is what ties this oracle to the reference."""
import math

import torch

import oracle


def convolution_reverberation(x, sample_rate, ir, mix, method: str = "fft"):
    """x (bs, 1|2, n), ir (bs, 1|2, L), mix (bs elements) -> (bs, 2, n); mono x or IR is used for both channels."""
    bs, chs, n = x.shape
    if chs == 1:
        x = x.repeat(1, 2, 1)
    if ir.shape[1] == 1:
        ir = ir.repeat(1, 2, 1)
    L = ir.shape[-1]
    mix = mix.reshape(bs, 1, 1)
    if method == "direct":
        xp = torch.nn.functional.pad(x, (L - 1, 0)).reshape(1, bs * 2, n + L - 1)
        wet = torch.nn.functional.conv1d(xp, torch.flip(ir, dims=[-1]).reshape(bs * 2, 1, L), groups=bs * 2)
        wet = wet.reshape(bs, 2, n)
    else:
        m = 1 << math.ceil(math.log2(n + L - 1))
        wet = torch.fft.irfft(torch.fft.rfft(x, m) * torch.fft.rfft(ir, m), m)[..., :n]
    return (1.0 - mix) * x + mix * wet


def reverb_ir(sample_rate, params, noise, num_samples, num_bandpass_taps, dtype=torch.float64):
    """(bs, 2, num_samples) IR of oracle.noise_shaped_reverberation for its 25 parameters and noise tensor"""
    bs = params[0].numel()
    gains = torch.stack([p.reshape(bs) for p in params[0:12]], dim=1).reshape(bs, 1, 12, 1).to(dtype)
    decays = torch.stack([p.reshape(bs) for p in params[12:24]], dim=1).reshape(bs, 1, 12, 1).to(dtype)
    fb = oracle.octave_filterbank(num_bandpass_taps, sample_rate).to(dtype)
    m = 1 << math.ceil(math.log2(noise.shape[-1] + num_bandpass_taps - 1))
    full = torch.fft.irfft(torch.fft.rfft(noise.to(dtype), m) * torch.fft.rfft(torch.flip(fb, dims=[-1]), m), m)
    shaped = full[..., num_bandpass_taps - 1: noise.shape[-1]].reshape(bs, 2, 12, num_samples)
    t = torch.linspace(0, 1, steps=num_samples, dtype=torch.float32).to(dtype)
    env = torch.exp(-(decays * 10.0 + 1.0) * t.reshape(1, 1, 1, -1))
    return (shaped * env * gains).mean(dim=2)
