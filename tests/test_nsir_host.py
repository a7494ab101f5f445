"""CPU checks of noise_shaped_impulse_response: its signature, input validation before any launch, the library's bs = 0
geometry against the reverb's at n = L, and the kernels the library must contain."""
import inspect
import os
import re
import shutil
import subprocess

import pytest
import torch

from helpers import SR

KB, NFFT = 4096, 8192
NAMES = [f"band{k}_gain" for k in range(12)] + [f"band{k}_decay" for k in range(12)]


@pytest.fixture(scope="module")
def lib():
    from dasp_pytorch_b200 import _abi, build
    build.build()
    return _abi.lib()


def _align(v):
    return (v + 255) // 256 * 256


def test_nsir_signature_and_exports():
    import dasp_pytorch_b200 as D
    sig = inspect.signature(D.noise_shaped_impulse_response)
    ps = list(sig.parameters.values())
    assert [p.name for p in ps] == ["sample_rate", *NAMES, "num_samples", "num_bandpass_taps", "noise"]
    assert sig.parameters["num_samples"].default == 65536 and sig.parameters["num_bandpass_taps"].default == 1023
    assert sig.parameters["noise"].kind is inspect.Parameter.KEYWORD_ONLY and sig.parameters["noise"].default is None
    # the reverb's first 24 parameters, in its order, without mix
    rev = list(inspect.signature(D.noise_shaped_reverberation).parameters)
    assert rev[2:26] == NAMES
    sigp = inspect.signature(D.noise_shaped_impulse_response_packed)
    assert list(sigp.parameters) == ["sample_rate", "params", "num_samples", "num_bandpass_taps", "noise"]
    for name in ("noise_shaped_impulse_response", "noise_shaped_impulse_response_packed"):
        assert name in D.functional.__all__ and getattr(D, name) is getattr(D.functional, name)


def _call(bs=2, sr=SR, L=64, taps=31, noise=None, counts=None, device="cpu", dtype=torch.float32):
    import dasp_pytorch_b200 as D
    counts = counts or [bs] * 24
    ps = [torch.full((c,), 0.5, dtype=dtype, device=device) for c in counts]
    return D.noise_shaped_impulse_response(sr, *ps, num_samples=L, num_bandpass_taps=taps, noise=noise)


def test_nsir_validation_before_any_launch():
    import dasp_pytorch_b200 as D
    from dasp_pytorch_b200.functional import DaspError
    for kw in (dict(taps=30), dict(taps=0), dict(L=0), dict(sr=32000),
               dict(counts=[2] * 23 + [3]),                                   # parameter counts 2 and 3
               dict(noise=torch.zeros(4, 12, 64 + 31)),                       # one sample short
               dict(noise=torch.zeros(2, 12, 64 + 30))):                      # rows of one item
        with pytest.raises(ValueError):
            _call(**kw)
    with pytest.raises(DaspError):                                            # valid, but CPU tensors: no CPU path
        _call()
    with pytest.raises(DaspError):
        _call(counts=[1] * 24)
    with pytest.raises(DaspError):                                            # plain numbers have no CUDA device
        D.noise_shaped_impulse_response(SR, *([0.5] * 24), num_samples=64, num_bandpass_taps=31)
    for bad in (torch.zeros(2, 25), torch.zeros(24), torch.zeros(2, 24, 1)):
        with pytest.raises(ValueError):
            D.noise_shaped_impulse_response_packed(SR, bad, num_samples=64, num_bandpass_taps=31)
    with pytest.raises(ValueError):
        D.noise_shaped_impulse_response_packed(SR, torch.zeros(2, 24), num_samples=64, num_bandpass_taps=33 - 1)
    with pytest.raises(DaspError):
        D.noise_shaped_impulse_response_packed(SR, torch.zeros(2, 24), num_samples=64, num_bandpass_taps=31)


# (L, taps): one tap, L < taps, k * 4096, k * 4096 + 1, 48000, 96000 (R = 12), 2047 taps (nb = 16384), R > 16
GEOMS = [(1, 1023), (500, 1023), (8192, 1023), (8193, 31), (48000, 1023), (96000, 1023), (48000, 2047),
         (150000, 1023)]


@pytest.mark.parametrize("L,taps", GEOMS)
def test_nsir_geometry_without_gpu(lib, L, taps):
    from dasp_pytorch_b200 import _abi
    g = _abi.ReverbGeom()
    assert lib.dasp_nsir_geometry(0, L, taps, 7, g) == 0
    J = -(-L // KB)
    assert (g.leff, g.conv_block, g.x_blocks, g.ir_partitions, g.chunk_items) == (L, KB, 0, J, 1)
    assert g.f_floats == 0 and g.xspec_c64 == 0 and g.irspec_c64 == 0
    nb = g.nb
    assert g.rpp == -(-(L + taps - 1) // nb)
    if L >= 2:                                       # the reverb at n = L synthesises the same taps the same way
        r = _abi.ReverbGeom()
        assert lib.dasp_reverb_geometry(0, L, L, taps, 7, r) == 0
        assert (g.nb, g.hop, g.nbk, g.leff, g.rpp) == (r.nb, r.hop, r.nbk, r.leff, r.rpp)
    pair_c64 = max(g.nbk, g.rpp) * nb
    # one item per pass without a batch, and no cuFFT work area is planned without a GPU
    assert g.fwd_workspace_bytes == _align(4 * 25) + _align(8 * 12 * pair_c64)
    assert g.bwd_workspace_bytes == 2 * _align(4 * 25) + _align(8 * J * NFFT) + _align(4 * 24 * max(g.nbk, -(-nb // 256)))


def test_nsir_geometry_rejects_bad_shapes(lib):
    from dasp_pytorch_b200 import _abi
    g = _abi.ReverbGeom()
    assert lib.dasp_nsir_geometry(0, 0, 1023, 1, g) == -1
    assert lib.dasp_nsir_geometry(0, 100, 1024, 1, g) == -1 and b"odd" in lib.dasp_last_error()
    assert lib.dasp_nsir_geometry(-1, 100, 1023, 1, g) == -1
    assert lib.dasp_nsir_geometry(0, 100, 1023, 1, None) == -1


def test_ir_synthesis_kernels_in_library(lib):
    from dasp_pytorch_b200 import _abi
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not installed")
    out = subprocess.run([cuobjdump, "-symbols", _abi.LIB_PATH], capture_output=True, text=True).stdout
    entries = set(re.findall(r"STO_ENTRY\s+(\S+)", out))
    def has(pat):
        return any(re.search(pat, e) for e in entries)
    # every IR-synthesis kernel in both instantiations: the reverb's partition sink and the IR op's planar sink
    for sink in ("13PartitionSink", "10PlanarSink"):
        for r in range(1, 7):
            assert has(rf"\dir_synth_cluster_kernelILi{r}ENS0_{sink}EE"), (r, sink)
        for name in ("ifft_shape_kernel", "shape_ir_pp_kernel", "shape_ir_pairs_kernel"):
            assert has(rf"\d{name}INS0_{sink}EE"), (name, sink)
    for name in ("nsir_params_kernel", "ir_pack_kernel", "ir_grad_pp_kernel", "ir_grad_pairs_kernel",
                 "reverb_param_grad_kernel"):
        assert has(rf"\d{name}E"), name
