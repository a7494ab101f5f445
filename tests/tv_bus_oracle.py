"""fp64 restatement of time_varying_convolution_bus for the tests, written from its definition: the K static bus
mixes of the sources with the trajectory's IR sets, weighted by the linear crossfade between neighbouring anchors (as
hat functions of the anchor times).  Independent of tests/conv_bus_oracle.py and tests/tv_conv_oracle.py
(tests/test_tv_bus_host.py ties it to both)."""
import math

import torch


def hat_weights(K, hop, n, dtype=torch.float64, device="cpu"):
    """(K, n) weights: w_k(t) = max(0, 1 - |t - k hop| / hop), and w_K-1(t) = 1 from its anchor on"""
    t = torch.arange(n, dtype=dtype, device=device)
    w = torch.stack([(1 - (t - k * hop).abs() / hop).clamp_min(0) for k in range(K)])
    w[K - 1, t >= (K - 1) * hop] = 1
    return w


def static_bus(x, h, method):
    """sum_s (x[:, s] * h[:, s, o])[:n]: x (bs, S, n), h (bs, S, O, L) -> (bs, O, n)"""
    bs, S, n = x.shape
    O, L = h.shape[2], h.shape[3]
    if method == "direct":
        w = torch.flip(h, dims=[-1]).transpose(1, 2).reshape(bs * O, S, L)
        xp = torch.nn.functional.pad(x, (L - 1, 0)).reshape(1, bs * S, n + L - 1)
        return torch.nn.functional.conv1d(xp, w, groups=bs).reshape(bs, O, n)
    m = 1 << math.ceil(math.log2(n + L - 1))
    X, Hf = torch.fft.rfft(x, m), torch.fft.rfft(h, m)
    return torch.fft.irfft((X[:, :, None] * Hf).sum(1), m)[..., :n]


def time_varying_convolution_bus(x, sample_rate, ir, hop, method: str = "fft"):
    """x (bs, S, n), ir (bs | 1, K, S, O, L) -> (bs, O, n), on x's device"""
    bs, _, n = x.shape
    K = ir.shape[1]
    ir = ir.expand(bs, -1, -1, -1, -1)
    w = hat_weights(K, hop, n, x.dtype, x.device)
    return sum(w[k] * static_bus(x, ir[:, k], method) for k in range(K))
