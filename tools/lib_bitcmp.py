#!/usr/bin/env python
"""Run seeded forward + backward calls of the reverbs, convolution_bus and the compressor / expander through two builds of
the library and compare every result byte for byte.

    python tools/lib_bitcmp.py LIB_A LIB_B --out DIR

A build is chosen when the package loads it (DASP_LIB_PATH), so each library runs in a process of its own and saves
what its calls computed to DIR/a/<case>.npy and DIR/b/<case>.npy; then the files are compared.  The cases reach the
paths bench.py does not: the cuFFT pipeline and the two-kernel IR synthesis (dasp_debug_reverb_path 1 and 2), R = 9
(two-kernel synthesis by default) and R = 17 (time-domain overlap-save), parity mode with a noise tensor, 2047 taps
(nb = 16384: cuFFT polyphase synthesis), n % 4 != 0 (cuFFT convolution), mono input, a forward without a backward (the
filtered noise and the spectra in the workspace), several chunks and a remainder (the forward's synthesis runs on its
side stream), and convolution_reverberation with per-item and shared impulse responses: stereo, mono and true-stereo
(per item on both pipelines, shared, and shared over several chunks with mono x), and a fixed IR (no dL/dIR).  The
convolution_bus cases cover a mono bus per item, a stereo bus with a shared IR over several chunks, n % 4 != 0 (the
padded rows) and a fixed IR.  Every convolution case saves its last-path hooks.  The
noise_shaped_impulse_response cases run the same synthesis paths with the planar sink (the cluster kernel, hooks 2 and
1, R = 12, R = 17, parity noise, 2047 taps, L = 1, chunks, a forward without a backward) and save the IR, dL/dparams
and the last path.  The dynamics cases run both curves at every warps-per-item W the library can be
pinned to (dasp_debug_force_warps), at lengths where that W fits: without a key mono (the generic channel loop), stereo
(the stereo kernels), stereo through the generic loop (DASP_DYN_GENERIC=1) and a look-ahead; with a key a mono key, a
stereo key, a look-ahead and a key that needs no gradient.  Refactors that must keep the bits use it; it needs a CUDA
device.  Exit code 1 on any difference.
"""
from __future__ import annotations

import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SR = 44100

# name: (kind, bs, in_chs, n, L or ir_len, taps | ir_chs, debug path | shared IR, parity noise[, options]); options:
# "grad": False (a forward only), "chunk": items per pass (REVERB_CHUNK_ITEMS), "ir_grad": False (a fixed IR).  A bus
# case reads in_chs as its S inputs and ir_chs as its O outputs.
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
    "reverb_fwd_only": ("reverb", 3, 2, 48000, 96000, 1023, 0, False, {"grad": False}),
    "reverb_chunks": ("reverb", 5, 2, 48000, 96000, 1023, 0, False, {"chunk": 2}),
    "conv_ts_item": ("conv", 3, 2, 48000, 30000, 4, False, False),
    "conv_ts_item_n_odd": ("conv", 3, 2, 48001, 30000, 4, False, False),
    "conv_ts_shared": ("conv", 4, 2, 48000, 50000, 4, True, False),
    "conv_ts_shared_chunks_mono_x": ("conv", 5, 1, 48000, 30000, 4, True, False, {"chunk": 2}),
    "conv_fixed_ir": ("conv", 3, 2, 48000, 30000, 2, False, False, {"ir_grad": False}),
    "bus_S3_O1_item": ("bus", 3, 3, 48000, 30000, 1, False, False),
    "bus_S8_O2_shared_chunks": ("bus", 5, 8, 48000, 50000, 2, True, False, {"chunk": 2}),
    "bus_S5_O2_n_odd": ("bus", 3, 5, 48003, 20000, 2, False, False),
    "bus_fixed_ir": ("bus", 3, 4, 48000, 30000, 2, False, False, {"ir_grad": False}),
}

# noise_shaped_impulse_response: name: (bs, L, taps, debug path, parity noise, options as above)
NSIR_CASES = {
    "nsir_cluster_R6": (3, 48000, 1023, 0, False, {}),
    "nsir_two_kernel_R6": (3, 48000, 1023, 2, False, {}),
    "nsir_cufft_R6": (3, 48000, 1023, 1, False, {}),
    "nsir_R12": (2, 96000, 1023, 0, False, {}),
    "nsir_R17": (2, 132000, 1023, 0, False, {}),
    "nsir_parity": (2, 20000, 1023, 0, True, {}),
    "nsir_taps2047": (2, 30000, 2047, 0, False, {}),
    "nsir_L1": (3, 1, 1023, 0, False, {}),
    "nsir_fwd_only": (3, 48000, 1023, 0, False, {"grad": False}),
    "nsir_chunks": (5, 48000, 1023, 0, False, {"chunk": 2}),
}

# dynamics: name: (x channels, key channels (0: no key), look-ahead, DASP_DYN_GENERIC, key gradient); each runs for
# curve x W {1, 2, 4, 8, 16}.  2C + K <= 4 keeps every forced W; the look-ahead cases take an n % 4 != 0 (cooperative
# copies instead of TMA)
DYN_E = 7
DYN_CASES = {
    "mono": (1, 0, False, False, False),
    "stereo": (2, 0, False, False, False),
    "stereo_generic": (2, 0, False, True, False),
    "lookahead": (2, 0, True, False, False),
    "key_mono": (1, 1, False, False, True),
    "key_stereo": (1, 2, False, False, True),
    "key_lookahead": (1, 1, True, False, True),
    "key_fixed": (1, 1, False, False, False),
}


def run_cases(out_dir):
    """the cases on cuda:0 with the library the package loads; one .npy per result"""
    sys.path.insert(0, ROOT)
    import torch

    import dasp_pytorch_b200 as D
    from dasp_pytorch_b200 import _abi

    lib = _abi.lib()
    dev = torch.device("cuda:0")
    chunk0 = D.functional.REVERB_CHUNK_ITEMS
    os.makedirs(out_dir, exist_ok=True)
    for ci, (name, (kind, bs, in_chs, n, L, c5, c6, parity, *opt)) in enumerate(CASES.items()):
        opt = opt[0] if opt else {}
        grad = opt.get("grad", True)
        g = torch.Generator().manual_seed(1000 + ci)
        x = ((torch.rand(bs, in_chs, n, generator=g) * 2 - 1) * 0.5).to(dev).requires_grad_(grad)
        gy = (torch.rand(bs, c5 if kind == "bus" else 2, n, generator=g) * 2 - 1).to(dev)
        res = {}
        if kind == "reverb":
            taps, path = c5, c6
            params = torch.rand(bs, 25, generator=g).to(dev).requires_grad_(grad)
            noise = torch.randn(bs * 2, 12, L + taps - 1, generator=g).to(dev) if parity else None
            torch.manual_seed(77 + ci)                 # the device-noise key is drawn from torch's CUDA generator
            lib.dasp_debug_reverb_path(path)
            D.functional.REVERB_CHUNK_ITEMS = opt.get("chunk", chunk0)
            try:
                y = D.functional.noise_shaped_reverberation_packed(x, SR, params, num_samples=L, num_bandpass_taps=taps,
                                                                   noise=noise)
                res["last_path"] = np.array([lib.dasp_debug_reverb_last_path()], dtype=np.int32)
                if grad:
                    y.backward(gy)
            finally:
                lib.dasp_debug_reverb_path(0)
                D.functional.REVERB_CHUNK_ITEMS = chunk0
            if grad:
                res["params_grad"] = params.grad
        else:
            shared, ir_grad = c6, opt.get("ir_grad", True)
            bus = kind == "bus"
            shape = (in_chs, c5, L) if bus else (c5, L)
            ir = (torch.randn(1 if shared else bs, *shape, generator=g) * 0.05).to(dev).requires_grad_(ir_grad)
            hook = lib.dasp_debug_conv_bus_last_path if bus else lib.dasp_debug_conv_last_path
            D.functional.REVERB_CHUNK_ITEMS = opt.get("chunk", chunk0)
            try:
                if bus:
                    y = D.functional.convolution_bus(x, SR, ir)
                else:
                    mix = torch.rand(bs, generator=g).to(dev).requires_grad_(True)
                    y = D.functional.convolution_reverberation(x, SR, ir, mix)
                res["last_path_fwd"] = np.array([hook(0)], dtype=np.int32)
                y.backward(gy)
                res["last_path_bwd"] = np.array([hook(1)], dtype=np.int32)
            finally:
                D.functional.REVERB_CHUNK_ITEMS = chunk0
            if ir_grad:
                res["ir_grad"] = ir.grad
            if not bus:
                res["mix_grad"] = mix.grad
        torch.cuda.synchronize(dev)
        res["y"] = y
        if grad:
            res["x_grad"] = x.grad
        save(out_dir, name, res)
    run_nsir_cases(out_dir)
    run_dynamics_cases(out_dir)


def save(out_dir, name, res):
    """one .npy per result of case `name` (tensors or numpy arrays)"""
    import torch

    for k, v in res.items():
        a = v.detach().cpu().numpy() if torch.is_tensor(v) else v
        np.save(os.path.join(out_dir, f"{name}.{k}.npy"), a)
    print(f"{name}: done", flush=True)


def run_nsir_cases(out_dir):
    """the noise_shaped_impulse_response cases: the IR, dL/dparams and the last synthesis path of each"""
    import torch

    import dasp_pytorch_b200 as D
    from dasp_pytorch_b200 import _abi

    lib = _abi.lib()
    dev = torch.device("cuda:0")
    chunk0 = D.functional.REVERB_CHUNK_ITEMS
    for ci, (name, (bs, L, taps, path, parity, opt)) in enumerate(NSIR_CASES.items()):
        grad = opt.get("grad", True)
        g = torch.Generator().manual_seed(3000 + ci)
        params = torch.rand(bs, 24, generator=g).to(dev).requires_grad_(grad)
        gir = torch.randn(bs, 2, L, generator=g).to(dev)
        noise = torch.randn(bs * 2, 12, L + taps - 1, generator=g).to(dev) if parity else None
        torch.manual_seed(177 + ci)
        lib.dasp_debug_reverb_path(path)
        D.functional.REVERB_CHUNK_ITEMS = opt.get("chunk", chunk0)
        try:
            ir = D.functional.noise_shaped_impulse_response_packed(SR, params, num_samples=L, num_bandpass_taps=taps,
                                                                   noise=noise)
            res = {"ir": ir, "last_path": np.array([lib.dasp_debug_reverb_last_path()], dtype=np.int32)}
            if grad:
                ir.backward(gir)
                res["params_grad"] = params.grad
        finally:
            lib.dasp_debug_reverb_path(0)
            D.functional.REVERB_CHUNK_ITEMS = chunk0
        torch.cuda.synchronize(dev)
        save(out_dir, name, res)


def run_dynamics_cases(out_dir):
    """the dynamics cases: y, dL/dx, dL/dkey and the five parameter gradients of each"""
    import torch

    import dasp_pytorch_b200 as D
    from dasp_pytorch_b200 import _abi

    lib = _abi.lib()
    dev = torch.device("cuda:0")
    ci = 0
    for curve in ("comp", "exp"):
        for w in (1, 2, 4, 8, 16):
            for case, (chs, kc, la, generic, key_grad) in DYN_CASES.items():
                name = f"dyn_{curve}_W{w}_{case}"
                ci += 1
                g = torch.Generator().manual_seed(5000 + ci)
                bs, T = 3, w * 32 * DYN_E
                n = 2 * T + (37 if la else 36)
                x = ((torch.rand(bs, chs, n, generator=g) * 2 - 1) * 0.5).to(dev).requires_grad_(True)
                gy = torch.randn(bs, chs, n, generator=g).to(dev)
                key = None
                if kc:
                    key = ((torch.rand(bs, kc, n, generator=g) * 2 - 1) * 0.5).to(dev).requires_grad_(key_grad)
                u = [torch.rand(bs, generator=g) for _ in range(6)]
                ratio = 1.5 + 4 * u[1] if curve == "comp" else 1.2 + 1.3 * u[1]
                ps = [(-35 + 25 * u[0]), ratio, 1 + 20 * u[2], 50 + 100 * u[3], 1 + 10 * u[4], -3 + 6 * u[5]]
                ps = [p.to(dev).requires_grad_(True) for p in ps]
                lookahead = T + T // 2 + 5 if la else 0
                if generic:
                    os.environ["DASP_DYN_GENERIC"] = "1"
                lib.dasp_debug_force_warps(w)
                try:
                    tile = (lib.dasp_dynamics_sidechain_tile_len(bs, chs, kc) if kc
                            else lib.dasp_dynamics_tile_len(bs, chs))
                    assert tile == T, (name, tile, T)
                    if kc:
                        fn = D.functional.sidechain_compressor if curve == "comp" else D.functional.sidechain_expander
                        y = fn(x, SR, *ps, lookahead_samples=lookahead, sidechain=key)
                    else:
                        fn = D.functional.compressor if curve == "comp" else D.functional.expander
                        y = fn(x, SR, *ps, lookahead_samples=lookahead)
                    y.backward(gy)
                    torch.cuda.synchronize(dev)
                finally:
                    lib.dasp_debug_force_warps(0)
                    os.environ.pop("DASP_DYN_GENERIC", None)
                res = {"y": y, "x_grad": x.grad}
                if key_grad:
                    res["key_grad"] = key.grad
                for pn, i in (("threshold", 0), ("ratio", 1), ("attack", 2), ("knee", 4), ("makeup", 5)):
                    res[f"{pn}_grad"] = ps[i].grad
                assert ps[3].grad is None                          # release_ms receives no gradient
                for k, v in res.items():
                    np.save(os.path.join(out_dir, f"{name}.{k}.npy"), v.detach().cpu().numpy())
    print(f"dynamics: {ci} cases done", flush=True)


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
