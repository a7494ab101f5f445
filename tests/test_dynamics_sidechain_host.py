"""CPU-only checks of the compressor / expander side chain (key): the test oracle reduces to the pinned one, the
functional layer and the C entry points reject bad keys before any launch, and the library carries the new kernels."""
import os
import re
import shutil
import subprocess

import pytest
import torch

import dyn_sidechain_oracle as sco
import oracle
from helpers import COMP_RANGES, SR, denorm


def test_sidechain_signatures():
    """compressor / expander keep the reference's parameters (Processor.process_normalized dispatches by name); the
    side-chain functions take the same ones plus a required keyword-only sidechain, and dynamics_packed an optional
    one"""
    import inspect
    import dasp_pytorch_b200 as D
    sig = lambda f: list(inspect.signature(f).parameters)
    comp = ["x", "sample_rate", "threshold_db", "ratio", "attack_ms", "release_ms", "knee_db", "makeup_gain_db", "eps",
            "lookahead_samples"]
    assert sig(D.compressor) == comp and sig(D.expander) == comp
    assert sig(D.sidechain_compressor) == comp + ["sidechain"] and sig(D.sidechain_expander) == comp + ["sidechain"]
    for fn, default in ((D.sidechain_compressor, inspect.Parameter.empty), (D.sidechain_expander, inspect.Parameter.empty),
                        (D.functional.dynamics_packed, None)):
        p = inspect.signature(fn).parameters
        assert p["eps"].default == 1e-8 and p["lookahead_samples"].default == 0
        assert p["sidechain"].kind is inspect.Parameter.KEYWORD_ONLY and p["sidechain"].default is default
    for cls in (D.Compressor, D.Expander):
        assert list(inspect.signature(cls.process_normalized).parameters) == ["self", "x", "param_tensor", "sidechain"]


def test_process_normalized_by_name_routes_the_key():
    """the by-name path (here: parameters on the CPU) calls the side-chain function, which accepts the key and
    then refuses the CPU tensors like every op (a TypeError would mean sidechain went to compressor())"""
    import dasp_pytorch_b200 as D
    from dasp_pytorch_b200._abi import DaspError
    for cls in (D.Compressor, D.Expander):
        with pytest.raises(DaspError, match="sidechain is on cpu"):
            cls(44100).process_normalized(torch.zeros(2, 2, 64), torch.rand(2, 6), sidechain=torch.zeros(2, 1, 64))


@pytest.fixture(scope="module")
def lib():
    from dasp_pytorch_b200 import build, _abi
    build.build()
    return _abi.lib()


@pytest.mark.parametrize("la", [0, 37])
@pytest.mark.parametrize("kind", ["comp", "exp"])
def test_oracle_sidechain_x_is_the_plain_oracle(kind, la):
    """sidechain=x: the same y, and dL/dx of the keyed op (gain path) plus dL/dkey (detector path) is the plain
    oracle's dL/dx; the parameter gradients are the same"""
    g = torch.Generator().manual_seed(5)
    bs, chs, n = 3, 2, 1500
    x = (torch.rand(bs, chs, n, generator=g, dtype=torch.float64) * 2 - 1) * 0.5
    params = [p.double() for p in denorm(torch.rand(bs, 6, generator=g).clamp(min=0.05), COMP_RANGES)]
    r = torch.randn(bs, chs, n, generator=g, dtype=torch.float64)
    plain, keyed = (oracle.compressor, sco.compressor) if kind == "comp" else (oracle.expander, sco.expander)

    xa = x.clone().requires_grad_(True)
    pa = [p.clone().requires_grad_(True) for p in params]
    ya = plain(xa, SR, *pa, lookahead_samples=la, fsm_tail=1 << 16)
    (ya * r).sum().backward()

    xb = x.clone().requires_grad_(True)
    kb = x.clone().requires_grad_(True)
    pb = [p.clone().requires_grad_(True) for p in params]
    yb = keyed(xb, SR, *pb, lookahead_samples=la, fsm_tail=1 << 16, sidechain=kb)
    (yb * r).sum().backward()

    assert torch.equal(ya, yb)
    torch.testing.assert_close(xb.grad + kb.grad, xa.grad, rtol=1e-12, atol=1e-12)
    assert torch.equal(kb.grad[:, 0], kb.grad[:, 1])              # every key channel gets the same dL/dside
    for a, b in zip(pa, pb):
        assert (a.grad is None) == (b.grad is None)
        if a.grad is not None:
            torch.testing.assert_close(b.grad, a.grad, rtol=1e-12, atol=1e-12)


def _args(bs=2):
    p = torch.zeros(bs)
    return (44100, p - 20, p + 4, p + 10, p + 50, p + 6, p)


@pytest.mark.parametrize("fn", ["sidechain_compressor", "sidechain_expander", "packed"])
def test_functional_rejects_bad_keys_before_any_launch(fn):
    """shape, channel count and device are checked before the CUDA-only check of x, so this runs without a GPU"""
    import dasp_pytorch_b200 as D
    from dasp_pytorch_b200._abi import DaspError
    x = torch.zeros(2, 2, 64)

    def call(key, xx=x):
        if fn == "packed":
            return D.functional.dynamics_packed(0, xx, 44100, torch.zeros(2, 6), sidechain=key)
        return getattr(D, fn)(xx, *_args(), sidechain=key)

    with pytest.raises(ValueError, match="batch and length"):
        call(torch.zeros(3, 1, 64))
    with pytest.raises(ValueError, match="batch and length"):
        call(torch.zeros(2, 1, 63))
    with pytest.raises(ValueError, match="key channels are supported"):
        call(torch.zeros(2, 0, 64))
    with pytest.raises(ValueError, match="key channels are supported"):
        call(torch.zeros(2, 33, 64))
    with pytest.raises(ValueError, match="exceeds 76"):
        call(torch.zeros(2, 13, 64), torch.zeros(2, 32, 64))
    with pytest.raises(ValueError, match=r"shape \(batch, key_channels, samples\)"):
        call(torch.zeros(2, 64))
    with pytest.raises(DaspError, match="sidechain is on meta but x is on cpu"):
        call(torch.zeros(2, 1, 64, device="meta"))
    with pytest.raises(DaspError, match="only runs on CUDA"):           # a valid key: x's own check
        call(torch.zeros(2, 1, 64))


def test_c_entry_points_reject_bad_key_channels_without_gpu(lib):
    """-1 with a message, before any CUDA call; the tile-length query returns 0 for the same combinations"""
    fake = 256                                   # never dereferenced: validation returns first
    ps = [fake] * 5
    for chs, kc, what in ((2, 0, b"key channels"), (2, 33, b"key channels"), (32, 13, b"exceeds 76"),
                          (30, 17, b"exceeds 76")):
        assert lib.dasp_dynamics_sidechain_tile_len(4, chs, kc) == 0
        rc = lib.dasp_dynamics_sidechain_fwd(0, fake, fake, kc, *ps, fake, fake, 4, chs, 1000, 44100.0, 1e-8, 0, None)
        assert rc == -1 and what in lib.dasp_last_error(), (chs, kc, lib.dasp_last_error())
        rc = lib.dasp_dynamics_sidechain_bwd(1, fake, fake, fake, kc, *ps, fake, fake, None, fake, None, 4, chs, 1000,
                                             44100.0, 1e-8, 0, None)
        assert rc == -1 and what in lib.dasp_last_error(), (chs, kc, lib.dasp_last_error())
    rc = lib.dasp_dynamics_sidechain_fwd(0, fake, None, 1, *ps, fake, fake, 4, 2, 1000, 44100.0, 1e-8, 0, None)
    assert rc == -1 and b"null key" in lib.dasp_last_error()


def test_library_has_the_sidechain_kernels_with_tma(lib):
    """curve x W {1, 2, 4, 8, 16} x look-ahead, forward and backward: 40 kernels, each streaming with UBLKCP"""
    from dasp_pytorch_b200 import _abi
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", _abi.LIB_PATH], capture_output=True, text=True).stdout
    bodies = re.split(r"\n\s*Function : ", sass)
    sc = {}
    for body in bodies:
        m = re.match(r"\S*dynamics_sc_(fwd|bwd)_kernelILNS0_5CurveE(\d)ELi(\d+)ELb(\d)E", body)
        if m:
            sc[m.groups()] = "UBLKCP" in body
    want = {(d, c, str(w), la) for d in ("fwd", "bwd") for c in "01" for w in (1, 2, 4, 8, 16) for la in "01"}
    assert set(sc) == want, sorted(set(sc) ^ want)
    assert all(sc.values())
