"""CPU-only checks of compressor_gain / expander_gain: the signatures, validation before any launch, the test oracle
against oracle.compressor / oracle.expander, the C entry points' argument checks and the kernels in the library."""
import inspect
import os
import re
import shutil
import subprocess

import pytest
import torch

import dyn_gain_oracle as go
import oracle
from helpers import COMP_RANGES, SR, denorm

COMP = ["x", "sample_rate", "threshold_db", "ratio", "attack_ms", "release_ms", "knee_db", "makeup_gain_db", "eps"]


def test_gain_signatures():
    import dasp_pytorch_b200 as D
    for fn in (D.compressor_gain, D.expander_gain):
        p = inspect.signature(fn).parameters
        assert list(p) == COMP + ["db"]
        assert p["eps"].default == 1e-8
        assert p["db"].kind is inspect.Parameter.KEYWORD_ONLY and p["db"].default is False
    p = inspect.signature(D.functional.dynamics_gain_packed).parameters
    assert list(p) == ["kind", "x", "sample_rate", "params", "eps", "db"]
    assert p["db"].kind is inspect.Parameter.KEYWORD_ONLY and p["db"].default is False
    for cls in (D.Compressor, D.Expander):
        p = inspect.signature(cls.gain_curve).parameters
        assert list(p) == ["self", "x", "param_tensor", "db"] and p["db"].kind is inspect.Parameter.KEYWORD_ONLY
    assert {"compressor_gain", "expander_gain"} <= set(D.functional.__all__)


def _args(bs=2):
    p = torch.zeros(bs)
    return (44100, p - 20, p + 4, p + 10, p + 50, p + 6, p)


@pytest.mark.parametrize("fn", ["compressor_gain", "expander_gain", "packed"])
def test_functional_rejects_bad_input_before_any_launch(fn):
    """rank, channel count and parameter counts are checked before the CUDA-only check of x, so this runs without a
    GPU"""
    import dasp_pytorch_b200 as D
    from dasp_pytorch_b200._abi import DaspError

    def call(x, args=None, params=None):
        if fn == "packed":
            return D.functional.dynamics_gain_packed(0, x, 44100, torch.zeros(2, 6) if params is None else params)
        return getattr(D, fn)(x, *(args or _args()))

    with pytest.raises(ValueError, match=r"shape \(batch, channels, samples\)"):
        call(torch.zeros(2, 64))
    with pytest.raises(ValueError, match="1 to 32 channels"):
        call(torch.zeros(2, 33, 64))
    with pytest.raises(ValueError, match="1 to 32 channels"):
        call(torch.zeros(2, 0, 64))
    if fn == "packed":
        with pytest.raises(ValueError, match=r"expected a \(2, 6\) parameter tensor"):
            call(torch.zeros(2, 2, 64), params=torch.zeros(2, 5))
        with pytest.raises(ValueError, match=r"expected a \(2, 6\) parameter tensor"):
            call(torch.zeros(2, 2, 64), params=torch.zeros(3, 6))
    else:
        for i, name in enumerate(["threshold_db", "ratio", "attack_ms", "release_ms", "knee_db", "makeup_gain_db"]):
            args = list(_args())
            args[1 + i] = torch.zeros(3)
            with pytest.raises(RuntimeError, match=f"{name}: expected 2 element"):
                call(torch.zeros(2, 2, 64), args)
        args = list(_args())
        args[1:] = [torch.zeros(1) for _ in args[1:]]                       # one element broadcasts
        with pytest.raises(DaspError, match="only runs on CUDA"):
            call(torch.zeros(2, 2, 64), args)
    with pytest.raises(DaspError, match="only runs on CUDA"):           # valid input: x's own device check
        call(torch.zeros(2, 32, 64))


def test_gain_curve_rejects_cpu_parameters():
    import dasp_pytorch_b200 as D
    from dasp_pytorch_b200._abi import DaspError
    for cls in (D.Compressor, D.Expander):
        with pytest.raises(DaspError, match="gain_curve: param_tensor must be a CUDA tensor"):
            cls(44100).gain_curve(torch.zeros(2, 2, 64), torch.rand(2, 6))


@pytest.mark.parametrize("la", [0, 1, 37, 1499])
@pytest.mark.parametrize("kind", ["comp", "exp"])
def test_oracle_delay_times_gain_is_the_processor(kind, la):
    """delay(x, la) * gain(x) is oracle.compressor / oracle.expander with look-ahead la: the same values and the same
    gradients to x and the parameters, to fp64 rounding; the dB curve is 20 log10 of the linear one"""
    g = torch.Generator().manual_seed(11 + la)
    bs, chs, n = 3, 3, 1500
    x = (torch.rand(bs, chs, n, generator=g, dtype=torch.float64) * 2 - 1) * 0.5
    params = [p.double() for p in denorm(torch.rand(bs, 6, generator=g).clamp(min=0.05), COMP_RANGES)]
    r = torch.randn(bs, chs, n, generator=g, dtype=torch.float64)
    proc, gain = (oracle.compressor, go.compressor_gain) if kind == "comp" else (oracle.expander, go.expander_gain)

    xa = x.clone().requires_grad_(True)
    pa = [p.clone().requires_grad_(True) for p in params]
    ya = proc(xa, SR, *pa, lookahead_samples=la, fsm_tail=1 << 16)
    (ya * r).sum().backward()

    xb = x.clone().requires_grad_(True)
    pb = [p.clone().requires_grad_(True) for p in params]
    gb = gain(xb, SR, *pb, fsm_tail=1 << 16)
    assert gb.shape == (bs, 1, n)
    yb = go.delay(xb, la) * gb
    (yb * r).sum().backward()

    torch.testing.assert_close(yb, ya, rtol=1e-13, atol=1e-15)
    torch.testing.assert_close(xb.grad, xa.grad, rtol=1e-10, atol=1e-12)
    for a, b in zip(pa, pb):
        assert (a.grad is None) == (b.grad is None)
        if a.grad is not None:
            torch.testing.assert_close(b.grad, a.grad, rtol=1e-10, atol=1e-12)
    gdb = gain(x, SR, *params, fsm_tail=1 << 16, db=True)
    torch.testing.assert_close(gdb, 20 * torch.log10(gb.detach()), rtol=1e-12, atol=1e-11)
    rec = gain(x, SR, *params, smoother="recursion")
    torch.testing.assert_close(gb.detach(), rec, rtol=1e-9, atol=1e-12)    # the enlarged grid is the true recursion


@pytest.fixture(scope="module")
def lib():
    from dasp_pytorch_b200 import build, _abi
    build.build()
    return _abi.lib()


def test_c_entry_points_reject_bad_shapes_without_gpu(lib):
    """-1 with a message, before any CUDA call"""
    fake = 256                                   # never dereferenced: validation returns first
    ps = [fake] * 5
    for bs, chs, n, what in ((4, 0, 1000, b"bad shape"), (4, 33, 1000, b"at most 32 channels"),
                             (-1, 2, 1000, b"bad shape"), (4, 2, -5, b"bad shape")):
        rc = lib.dasp_dynamics_gain_fwd(0, fake, chs, *ps, fake, fake, bs, n, 44100.0, 1e-8, 0, None)
        assert rc == -1 and what in lib.dasp_last_error(), (chs, lib.dasp_last_error())
        rc = lib.dasp_dynamics_gain_bwd(1, fake, fake, *ps, fake, fake, fake, bs, chs, n, 44100.0, 1e-8, 1, None)
        assert rc == -1 and what in lib.dasp_last_error(), (chs, lib.dasp_last_error())
    rc = lib.dasp_dynamics_gain_fwd(0, None, 2, *ps, fake, fake, 4, 1000, 44100.0, 1e-8, 0, None)
    assert rc == -1 and b"null x" in lib.dasp_last_error()
    rc = lib.dasp_dynamics_gain_fwd(2, fake, 2, *ps, fake, fake, 4, 1000, 44100.0, 1e-8, 0, None)
    assert rc == -1 and b"kind must be" in lib.dasp_last_error()
    rc = lib.dasp_dynamics_gain_fwd(0, fake, 2, *ps, None, fake, 4, 1000, 44100.0, 1e-8, 0, None)
    assert rc == -1 and b"null g" in lib.dasp_last_error()
    rc = lib.dasp_dynamics_gain_bwd(0, fake, fake, *ps, fake, fake, None, 4, 2, 1000, 44100.0, 1e-8, 0, None)
    assert rc == -1 and b"null gparams" in lib.dasp_last_error()
    # nothing to do: no launch, no CUDA call
    assert lib.dasp_dynamics_gain_fwd(0, None, 2, None, None, None, None, None, None, None, 0, 1000, 44100.0, 1e-8, 0,
                                      None) == 0
    assert lib.dasp_dynamics_gain_bwd(0, None, None, None, None, None, None, None, None, None, None, 0, 2, 1000,
                                      44100.0, 1e-8, 0, None) == 0


def test_library_has_the_gain_kernels_with_tma(lib):
    """curve x W {1, 2, 4, 8, 16}, forward and backward: 20 kernels, each streaming with UBLKCP"""
    from dasp_pytorch_b200 import _abi
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", _abi.LIB_PATH], capture_output=True, text=True).stdout
    found = {}
    for body in re.split(r"\n\s*Function : ", sass):
        m = re.match(r"\S*dynamics_gain_(fwd|bwd)_kernelILNS0_5CurveE(\d)ELi(\d+)EE", body)
        if m:
            found[m.groups()] = "UBLKCP" in body
    want = {(d, c, str(w)) for d in ("fwd", "bwd") for c in "01" for w in (1, 2, 4, 8, 16)}
    assert set(found) == want, sorted(set(found) ^ want)
    assert all(found.values())
