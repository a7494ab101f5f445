"""fp64 restatement of time_varying_convolution_bus with crossfade="input" for the tests, written from its definition:
the K static bus mixes of the weighted sources w_k x with the trajectory's IR sets, every weight a hat function of the
anchor times.  Every emitted sample therefore keeps the IR sets of its emission time over its whole tail.  Reuses only
the weights of tests/tv_bus_oracle.py and has its own static bus (tests/test_tv_bus_input_host.py ties it to the static
bus oracle)."""
import math

import torch

from tv_bus_oracle import hat_weights


def static_bus(x, h, method):
    """sum_s (x[:, s] * h[:, s, o])[:n]: x (bs, S, n), h (bs, S, O, L) -> (bs, O, n)"""
    bs, S, n = x.shape
    O, L = h.shape[2], h.shape[3]
    if method == "direct":
        w = torch.flip(h, dims=[-1]).transpose(1, 2).reshape(bs * O, S, L)
        xp = torch.nn.functional.pad(x, (L - 1, 0)).reshape(1, bs * S, n + L - 1)
        return torch.nn.functional.conv1d(xp, w, groups=bs).reshape(bs, O, n)
    m = 1 << math.ceil(math.log2(n + L - 1))
    return torch.fft.irfft(torch.einsum("bsf,bsof->bof", torch.fft.rfft(x, m), torch.fft.rfft(h, m)), m)[..., :n]


def time_varying_convolution_bus(x, sample_rate, ir, hop, method: str = "fft"):
    """x (bs, S, n), ir (bs | 1, K, S, O, L) -> (bs, O, n) = sum_k static_bus(w_k x, h[:, k]), on x's device"""
    bs, _, n = x.shape
    K = ir.shape[1]
    ir = ir.expand(bs, -1, -1, -1, -1)
    w = hat_weights(K, hop, n, x.dtype, x.device)
    return sum(static_bus(w[k] * x, ir[:, k], method) for k in range(K))
