#!/usr/bin/env python
"""Run seeded forward + backward calls of the reverbs through two builds of the library and compare every result byte
for byte.

    python tools/lib_bitcmp.py LIB_A LIB_B --out DIR

A build is chosen when the package loads it (DASP_LIB_PATH), so each library runs in a process of its own and saves
what its calls computed to DIR/a/<case>.npy and DIR/b/<case>.npy; then the files are compared.  The cases reach the
paths bench.py does not: the cuFFT pipeline and the two-kernel IR synthesis (dasp_debug_reverb_path 1 and 2), R = 9
(two-kernel synthesis by default) and R = 17 (time-domain overlap-save), parity mode with a noise tensor, 2047 taps
(nb = 16384: cuFFT polyphase synthesis), n % 4 != 0 (cuFFT convolution), mono input, and convolution_reverberation with
per-item and shared impulse responses.  Refactors that must keep the bits use it; it needs a CUDA device.  Exit code 1
on any difference.
"""
from __future__ import annotations

import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SR = 44100

# name: (kind, bs, in_chs, n, L or ir_len, taps | ir_chs, debug path | shared IR, parity noise)
CASES = {
    "reverb_cluster_R6": ("reverb", 3, 2, 48000, 96000, 1023, 0, False),
    "reverb_two_kernel_R6": ("reverb", 3, 2, 48000, 96000, 1023, 2, False),
    "reverb_cufft_R6": ("reverb", 3, 2, 48000, 96000, 1023, 1, False),
    "reverb_R9": ("reverb", 2, 2, 72000, 70000, 1023, 0, False),
    "reverb_R17": ("reverb", 2, 2, 132000, 132000, 1023, 0, False),
    "reverb_parity": ("reverb", 2, 2, 24000, 20000, 1023, 0, True),
    "reverb_taps2047": ("reverb", 2, 2, 48000, 30000, 2047, 0, False),
    "reverb_n_odd": ("reverb", 2, 2, 48001, 40000, 1023, 0, False),
    "reverb_mono": ("reverb", 3, 1, 48000, 40000, 1023, 0, False),
    "conv_item": ("conv", 3, 2, 48000, 30000, 2, False, False),
    "conv_item_mono_ir": ("conv", 3, 1, 48000, 50000, 1, False, False),
    "conv_item_n_odd": ("conv", 3, 2, 48001, 30000, 2, False, False),
    "conv_shared": ("conv", 4, 2, 48000, 30000, 2, True, False),
    "conv_shared_n_odd": ("conv", 4, 1, 48003, 20000, 1, True, False),
}


def run_cases(out_dir):
    """the cases on cuda:0 with the library the package loads; one .npy per result"""
    sys.path.insert(0, ROOT)
    import torch

    import dasp_pytorch_b200 as D
    from dasp_pytorch_b200 import _abi

    lib = _abi.lib()
    dev = torch.device("cuda:0")
    os.makedirs(out_dir, exist_ok=True)
    for ci, (name, (kind, bs, in_chs, n, L, c5, c6, parity)) in enumerate(CASES.items()):
        g = torch.Generator().manual_seed(1000 + ci)
        x = ((torch.rand(bs, in_chs, n, generator=g) * 2 - 1) * 0.5).to(dev).requires_grad_(True)
        gy = (torch.rand(bs, 2, n, generator=g) * 2 - 1).to(dev)
        res = {}
        if kind == "reverb":
            taps, path = c5, c6
            params = torch.rand(bs, 25, generator=g).to(dev).requires_grad_(True)
            noise = torch.randn(bs * 2, 12, L + taps - 1, generator=g).to(dev) if parity else None
            torch.manual_seed(77 + ci)                 # the device-noise key is drawn from torch's CUDA generator
            lib.dasp_debug_reverb_path(path)
            try:
                y = D.functional.noise_shaped_reverberation_packed(x, SR, params, num_samples=L, num_bandpass_taps=taps,
                                                                   noise=noise)
                res["last_path"] = np.array([lib.dasp_debug_reverb_last_path()], dtype=np.int32)
                y.backward(gy)
            finally:
                lib.dasp_debug_reverb_path(0)
            res["params_grad"] = params.grad
        else:
            ir_chs, shared = c5, c6
            ir = (torch.randn(1 if shared else bs, ir_chs, L, generator=g) * 0.05).to(dev).requires_grad_(True)
            mix = torch.rand(bs, generator=g).to(dev).requires_grad_(True)
            y = D.functional.convolution_reverberation(x, SR, ir, mix)
            res["last_path_fwd"] = np.array([lib.dasp_debug_conv_last_path(0)], dtype=np.int32)
            y.backward(gy)
            res["last_path_bwd"] = np.array([lib.dasp_debug_conv_last_path(1)], dtype=np.int32)
            res["ir_grad"], res["mix_grad"] = ir.grad, mix.grad
        torch.cuda.synchronize(dev)
        res["y"], res["x_grad"] = y, x.grad
        for k, v in res.items():
            a = v.detach().cpu().numpy() if torch.is_tensor(v) else v
            np.save(os.path.join(out_dir, f"{name}.{k}.npy"), a)
        print(f"{name}: done", flush=True)


def main():
    if len(sys.argv) >= 3 and sys.argv[1] == "--run":
        run_cases(sys.argv[2])
        return 0
    if len(sys.argv) != 5 or sys.argv[3] != "--out":
        print(__doc__)
        return 2
    lib_a, lib_b, out = sys.argv[1], sys.argv[2], sys.argv[4]
    for tag, path in (("a", lib_a), ("b", lib_b)):
        env = dict(os.environ, DASP_LIB_PATH=os.path.abspath(path))
        subprocess.run([sys.executable, os.path.abspath(__file__), "--run", os.path.join(out, tag)], env=env, check=True)
    files = sorted(os.listdir(os.path.join(out, "a")))
    differ = [f for f in files
              if not os.path.exists(os.path.join(out, "b", f))
              or open(os.path.join(out, "a", f), "rb").read() != open(os.path.join(out, "b", f), "rb").read()]
    missing = sorted(set(os.listdir(os.path.join(out, "b"))) - set(files))
    print(json.dumps({"files": len(files), "differ": differ, "only_in_b": missing}))
    return 1 if differ or missing else 0


if __name__ == "__main__":
    sys.exit(main())
