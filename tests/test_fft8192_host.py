"""Host emulation of the in-shared-memory 8192-point FFT (csrc/fft8192.cuh): the same pass functions the fused
reverb kernel runs, with the CTA's 512 threads looped over sequentially.
Pins the index mathematics / twiddle tables of both transform directions without a GPU."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_fft8192_passes_against_fp64_reference(tmp_path):
    exe = str(tmp_path / "fft8192_host_check")
    subprocess.run(["g++", "-O2", "-std=c++17", "-I", os.path.join(ROOT, "dasp_pytorch_b200", "csrc"),
                    os.path.join(ROOT, "tools", "probe", "fft8192_host_check.cpp"), "-o", exe], check=True)
    out = subprocess.run([exe], capture_output=True, text=True)
    sys.stdout.write(out.stdout)
    assert out.returncode == 0, out.stdout + out.stderr
    errs = dict(line.split() for line in out.stdout.strip().splitlines())
    assert float(errs["inverse_rel_err"]) < 1e-6 and float(errs["forward_rel_err"]) < 1e-6
