"""fp64 restatement of time_varying_convolution_reverberation for the tests, written from its definition: the K static
convolutions of x with the trajectory's IRs, weighted by the linear crossfade between neighbouring anchors.  Independent
of tests/conv_oracle.py (tests/test_tv_conv_host.py ties the two together at K = 1 and for K equal IRs)."""
import math

import torch


def crossfade_weights(K, hop, n, dtype=torch.float64):
    """(K, n) weights w_k(t): 1 - a and a between anchors k and k + 1, a = (t - k hop) / hop; 1 for IR K - 1 after its
    anchor"""
    t = torch.arange(n, dtype=dtype)
    w = torch.zeros(K, n, dtype=dtype)
    for k in range(K - 1):
        seg = (t >= k * hop) & (t < (k + 1) * hop)
        a = (t[seg] - k * hop) / hop
        w[k, seg] += 1 - a
        w[k + 1, seg] += a
    w[K - 1, t >= (K - 1) * hop] = 1
    return w


def static_wet(x, h, method):
    """(x * h)[:n] per item and channel: x (bs, 2, n), h (bs, 2, L)"""
    bs, _, n = x.shape
    L = h.shape[-1]
    if method == "direct":
        xp = torch.nn.functional.pad(x, (L - 1, 0)).reshape(1, bs * 2, n + L - 1)
        return torch.nn.functional.conv1d(xp, torch.flip(h, dims=[-1]).reshape(bs * 2, 1, L), groups=bs * 2).reshape(
            bs, 2, n)
    m = 1 << math.ceil(math.log2(n + L - 1))
    return torch.fft.irfft(torch.fft.rfft(x, m) * torch.fft.rfft(h, m), m)[..., :n]


def time_varying_convolution_reverberation(x, sample_rate, ir, hop, mix, method: str = "fft"):
    """x (bs, 1|2, n), ir (bs | 1, K, 1|2, L), mix (bs elements) -> (bs, 2, n)"""
    bs, _, n = x.shape
    x = x.expand(bs, 2, n)
    K = ir.shape[1]
    ir = ir.expand(bs, K, 2, ir.shape[-1])
    w = crossfade_weights(K, hop, n, x.dtype)
    wet = sum(w[k] * static_wet(x, ir[:, k], method) for k in range(K))
    mix = mix.reshape(bs, 1, 1)
    return (1.0 - mix) * x + mix * wet
