"""CPU oracle of parametric_eq_frequency_response.  TEST INFRASTRUCTURE ONLY.

The response of the six sections ``oracle.eq_sections`` designs (the reference's ``signal.biquad`` calls,
functional.py:211-265), evaluated directly as prod_k B_k(z^-1) / A_k(z^-1) at z = exp(j 2 pi f / sample_rate) in the
caller's dtype: complex64 for fp32 parameters, complex128 for fp64.  With fp64 parameters it is the arbiter, and
forward- and reverse-mode autograd through it give the reference gradients.  It is pinned to the reference's own
``signal.fft_sosfreqz`` by ``tests/golden/eq_response.npz`` (tests/test_eq_response_host.py).
"""
import math

import torch

import oracle


def parametric_eq_response(sample_rate, *params, frequencies):
    """(bs, F) complex response of the 18 EQ parameters (signature order) at ``frequencies`` (Hz, 1-D)"""
    params = [p if torch.is_tensor(p) else torch.as_tensor(p) for p in params]
    sos = oracle.eq_sections(sample_rate, params)                          # (bs, 6, 6) [b0 b1 b2 1 a1 a2]
    f = torch.as_tensor(frequencies).to(sos.dtype).reshape(1, -1)
    zi = torch.exp(-1j * (2.0 * math.pi / sample_rate) * f)                 # z^-1
    zi2 = zi * zi
    h = None
    for k in range(sos.shape[1]):
        b0, b1, b2, _, a1, a2 = (sos[:, k, i, None] for i in range(6))
        hk = (b0 + b1 * zi + b2 * zi2) / (1.0 + a1 * zi + a2 * zi2)
        h = hk if h is None else h * hk
    return h


def log_grid(sample_rate, n=512, lo=10.0, dtype=torch.float64):
    """n frequencies from lo to sample_rate / 2, evenly spaced in log frequency"""
    return torch.logspace(math.log10(lo), math.log10(sample_rate / 2), n, dtype=dtype)
