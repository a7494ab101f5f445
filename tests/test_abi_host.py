"""CPU-only checks of the C-ABI library: it loads, exports every symbol include/dasp_b200.h declares, the
host-side filter-bank design equals scipy's firwin, and the product path refuses to run without CUDA."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from conftest import ROOT, load_golden


@pytest.fixture(scope="module")
def lib():
    from dasp_pytorch_b200 import build, _abi
    build.build()
    return _abi.lib()


def test_header_symbols_exported(lib):
    from dasp_pytorch_b200 import _abi
    hdr = open(os.path.join(ROOT, "include", "dasp_b200.h")).read()
    declared = set(re.findall(r"\b(dasp_[a-z0-9_]+)\s*\(", hdr))
    assert declared, "no declarations parsed"
    for name in sorted(declared):
        assert hasattr(lib, name), f"{name} declared in include/dasp_b200.h but not exported"
    assert declared == set(_abi.exported_symbols()), declared ^ set(_abi.exported_symbols())
    assert lib.dasp_abi_version() == _abi.ABI_VERSION == 2 and lib.dasp_compiled_arch() == 900


def test_sm90a_sass_and_tma(lib):
    """the shared library carries sm_90a SASS with TMA bulk copies (UBLKCP) in the recurrence kernels"""
    import shutil
    import subprocess
    from dasp_pytorch_b200 import _abi
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    out = subprocess.run([cuobjdump, "-lelf", _abi.LIB_PATH], capture_output=True, text=True).stdout
    assert "sm_90a" in out
    assert "sm_52" not in out and "sm_100" not in out         # sm_90a only: no multi-arch fat binary
    sass = subprocess.run([cuobjdump, "-sass", _abi.LIB_PATH], capture_output=True, text=True).stdout
    assert "UBLKCP" in sass and "SYNCS" in sass               # cp.async.bulk + mbarrier in the scan kernels


def test_eq_kernel_instantiations(lib):
    """the library holds exactly the EQ kernels the dispatch can launch (tests/test_gpu_eq_variants.py pins and
    profiles each of them)"""
    from dasp_pytorch_b200 import _abi
    from helpers import EQ_INSTANTIATIONS, eq_kernel_instantiations
    got = eq_kernel_instantiations(_abi.LIB_PATH)
    if got is None:
        pytest.skip("cuobjdump not available")
    assert got == EQ_INSTANTIATIONS, (sorted(got - EQ_INSTANTIATIONS), sorted(EQ_INSTANTIATIONS - got))


@pytest.mark.parametrize("taps,sr", [(1023, 44100.0), (255, 44100.0), (1023, 48000.0), (511, 96000.0)])
def test_filterbank_matches_scipy(lib, taps, sr):
    import oracle
    out = np.zeros((12, taps), dtype=np.float32)
    rc = lib.dasp_reverb_filterbank(taps, sr, out.ctypes.data_as(ctypes.POINTER(ctypes.c_float)))
    assert rc == 0
    ref = oracle.octave_filterbank(taps, sr).numpy()
    assert np.abs(out - ref).max() <= 2e-7 * np.abs(ref).max()
    if (taps, sr) == (255, 44100.0):
        assert np.abs(out - load_golden("reverb.npz")["filterbank"]).max() <= 2e-7 * np.abs(ref).max()


def test_error_reporting_without_gpu(lib):
    rc = lib.dasp_reverb_filterbank(1024, 44100.0, None)
    assert rc == -1 and b"odd" in lib.dasp_last_error()
    rc = lib.dasp_reverb_filterbank(1023, 16000.0, np.zeros(12 * 1023, np.float32).ctypes.data_as(ctypes.POINTER(ctypes.c_float)))
    assert rc == -1


def test_no_cpu_fallback():
    import dasp_pytorch_b200 as D
    x = torch.zeros(2, 2, 64)
    p = torch.zeros(2)
    for call in (lambda: D.gain(x, 44100, p), lambda: D.distortion(x, 44100, torch.zeros(4)),
                 lambda: D.compressor(x, 44100, p, p + 2, p + 10, p + 10, p + 1, p),
                 lambda: D.parametric_eq(x, 44100, *([p + 1] * 18)),
                 lambda: D.noise_shaped_reverberation(x, 44100, *([p] * 25), num_samples=256, num_bandpass_taps=31)):
        with pytest.raises(D.functional.DaspError):
            call()


def test_product_does_not_import_oracle():
    """only tests/, __graft_entry__.smoke() and bench.py may touch oracle/"""
    pkg = os.path.join(ROOT, "dasp_pytorch_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(import|from)\s+oracle\b", src, re.M), f
