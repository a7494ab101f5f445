"""CPU checks of parametric_eq_frequency_response: its signature and exports, input validation before any launch, the
oracle against the reference's own fft_sosfreqz (tests/golden/eq_response.npz), and the C ABI's empty calls, which
need no device."""
import ctypes
import inspect

import numpy as np
import pytest
import torch

from eq_response_oracle import parametric_eq_response
from helpers import SR
from param_grad_pin import EQ_NAMES


@pytest.fixture(scope="module")
def lib():
    from dasp_pytorch_b200 import _abi, build
    build.build()
    return _abi.lib()


def test_eq_response_signature_and_exports():
    import dasp_pytorch_b200 as D
    ps = list(inspect.signature(D.parametric_eq_frequency_response).parameters)
    assert ps == ["sample_rate", *EQ_NAMES, "frequencies"]
    assert list(inspect.signature(D.parametric_eq).parameters)[2:] == EQ_NAMES       # parametric_eq's names and order
    assert list(inspect.signature(D.parametric_eq_frequency_response_packed).parameters) == [
        "sample_rate", "params", "frequencies"]
    assert list(inspect.signature(D.ParametricEQ.frequency_response).parameters) == [
        "self", "param_tensor", "frequencies"]
    for name in ("parametric_eq_frequency_response", "parametric_eq_frequency_response_packed"):
        assert name in D.functional.__all__ and getattr(D, name) is getattr(D.functional, name)


def _call(bs=2, sr=SR, freqs=None, counts=None, device="cpu"):
    import dasp_pytorch_b200 as D
    counts = counts or [bs] * 18
    ps = [torch.full((c,), 1000.0, device=device) for c in counts]
    f = torch.linspace(0, sr / 2, 9) if freqs is None else freqs
    return D.parametric_eq_frequency_response(sr, *ps, frequencies=f)


def test_eq_response_validation_before_any_launch():
    import dasp_pytorch_b200 as D
    from dasp_pytorch_b200.functional import DaspError
    for kw in (dict(counts=[2] * 17 + [3]),                                  # element counts 2 and 3
               dict(freqs=torch.zeros(2, 4)),                                # 2-D frequencies
               dict(freqs=torch.zeros(4, requires_grad=True)),               # frequencies that want a gradient
               dict(sr=0), dict(sr=-44100)):
        with pytest.raises(ValueError):
            _call(**kw)
    with pytest.raises(DaspError):                                           # valid, but CPU tensors: no CPU path
        _call()
    with pytest.raises(DaspError):
        _call(counts=[1] * 18)
    with pytest.raises(DaspError):                                           # plain numbers have no CUDA device
        D.parametric_eq_frequency_response(SR, *([1000.0] * 18), frequencies=torch.zeros(3))
    for bad in (torch.zeros(2, 17), torch.zeros(18), torch.zeros(2, 18, 1)):
        with pytest.raises(ValueError):
            D.parametric_eq_frequency_response_packed(SR, bad, torch.zeros(3))
    with pytest.raises(ValueError):
        D.parametric_eq_frequency_response_packed(SR, torch.zeros(2, 18), torch.zeros(3, 1))
    with pytest.raises(ValueError):
        D.parametric_eq_frequency_response_packed(0, torch.zeros(2, 18), torch.zeros(3))
    with pytest.raises(DaspError):
        D.parametric_eq_frequency_response_packed(SR, torch.zeros(2, 18), torch.zeros(3))
    with pytest.raises(DaspError):
        D.ParametricEQ(SR).frequency_response(torch.full((2, 18), 0.5), torch.zeros(3))


def _golden():
    from conftest import load_golden
    z = load_golden("eq_response.npz")
    return z, [torch.from_numpy(p) for p in z["params"]], float(z["sample_rate"])


@pytest.mark.parametrize("n_fft", [4096, 131072])
def test_oracle_matches_reference_fft_sosfreqz(n_fft):
    """the fixture keeps a subset of each rfft grid's bins (bins_<n_fft>): all of the low ones, a subsample above"""
    z, params, sr = _golden()
    bins = torch.from_numpy(z[f"bins_{n_fft}"])
    f = torch.fft.rfftfreq(n_fft, 1 / sr, dtype=torch.float64)[bins]
    h64 = parametric_eq_response(sr, *[p.double() for p in params], frequencies=f)
    ref64 = torch.from_numpy(z[f"h64_{n_fft}"])
    assert h64.dtype == torch.complex128 and h64.shape == ref64.shape
    err = ((h64 - ref64).abs() / ref64.abs()).amax()
    assert err <= 1e-8, float(err)
    # the reference's fp32 values: its own fp32 level, measured against fp64.  Above 1 kHz the median bin is ~1e-7 off;
    # next to the low shelves fp32 loses up to percents (1 + a1 + a2 ~ 1e-5), which is why most stored bins sit there.
    # The oracle in fp32 (direct form too) is at the same level.
    upper = f > 1000.0
    ref32 = torch.from_numpy(z[f"h32_{n_fft}"]).to(torch.complex128)
    e_ref = (ref32 - ref64).abs() / ref64.abs()
    assert float(e_ref[:, upper].median()) <= 1e-5 and float(e_ref.amax()) <= 1.0
    h32 = parametric_eq_response(sr, *params, frequencies=f.float())
    assert h32.dtype == torch.complex64
    e_orc = (h32.to(torch.complex128) - ref64).abs() / ref64.abs()
    assert float(e_orc[:, upper].median()) <= 1e-5


def test_oracle_gradient_modes_agree():
    """forward- and reverse-mode AD through the oracle give the same parameter gradients"""
    import torch.autograd.forward_ad as fwAD
    _, params, sr = _golden()
    f = torch.tensor([0.0, 20.0, 100.0, 1000.0, 9000.0, sr / 2], dtype=torch.float64)
    pp = [p.double() for p in params]
    c = torch.randn(pp[0].shape[0], f.numel(), dtype=torch.complex128, generator=torch.Generator().manual_seed(1))
    for j in (1, 5, 13, 17):
        with fwAD.dual_level():
            dual = [fwAD.make_dual(p, torch.ones_like(p)) if i == j else p for i, p in enumerate(pp)]
            tan = fwAD.unpack_dual(parametric_eq_response(sr, *dual, frequencies=f)).tangent
        fwd = (c.conj() * tan).real.sum(1)
        q = [p.clone().requires_grad_(i == j) for i, p in enumerate(pp)]
        h = parametric_eq_response(sr, *q, frequencies=f)
        (g,) = torch.autograd.grad(h, q[j], grad_outputs=c)
        assert torch.allclose(fwd, g, rtol=1e-10, atol=0), j


def test_abi_empty_calls_without_gpu(lib):
    n = lib.dasp_eq_response_workspace_floats(0, 100)
    assert n >= 0
    assert lib.dasp_eq_response_workspace_floats(4, 0) >= 0
    # bs = 0 in both directions, nfreq = 0 in the forward: no device is touched
    assert lib.dasp_eq_response_fwd(None, None, None, None, 0, 0, 100, ctypes.c_float(SR), None) == 0
    assert lib.dasp_eq_response_bwd(None, None, None, None, None, 0, 0, 100, ctypes.c_float(SR), None) == 0
    assert lib.dasp_eq_response_fwd(None, None, None, None, 0, 4, 0, ctypes.c_float(SR), None) == 0
    assert lib.dasp_eq_response_fwd(None, None, None, None, 0, -1, 4, ctypes.c_float(SR), None) == -1


def test_workspace_grows_with_the_problem(lib):
    """the query needs no device, and covers the vs table, the coefficients and the parameter-gradient sums"""
    for bs, nf in ((1, 1), (1, 65537), (64, 65537), (1024, 65537), (1024, 512)):
        n = lib.dasp_eq_response_workspace_floats(bs, nf)
        assert n >= 2 * nf + 60 * bs
        assert n % 2 == 0
