"""fp64 restatement of convolution_bus for the tests: y[:, o] = sum_s (x[:, s] * h[:, s, o])[:n], `*` the causal
convolution cropped to n.  Written from the definition, independently of tests/conv_oracle.py and tests/conv_ts_oracle.py
(tests/test_conv_bus_host.py ties it to the true-stereo oracle at S = 2)."""
import math

import torch


def convolution_bus(x, sample_rate, ir, method: str = "fft"):
    """x (bs, S, n), ir (bs | 1, S, O, L) -> (bs, O, n)"""
    bs, S, n = x.shape
    ir = ir.expand(bs, -1, -1, -1)
    L = ir.shape[-1]
    if method == "direct":
        # y[b, o, t] = sum_s sum_tau h[b, s, o, tau] x[b, s, t - tau]: one conv1d over the S input channels per item
        O = ir.shape[2]
        w = torch.flip(ir, dims=[-1]).transpose(1, 2).reshape(bs * O, S, L)
        xp = torch.nn.functional.pad(x, (L - 1, 0)).reshape(1, bs * S, n + L - 1)
        return torch.nn.functional.conv1d(xp, w, groups=bs).reshape(bs, O, n)
    m = 1 << math.ceil(math.log2(n + L - 1))
    return torch.fft.irfft(torch.einsum("bsf,bsof->bof", torch.fft.rfft(x, m), torch.fft.rfft(ir, m)), m)[..., :n]
