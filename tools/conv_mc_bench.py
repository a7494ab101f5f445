"""Time multichannel_convolution (S sources through an S x M IR matrix) against what a caller does without it, on the same
GPU.

    python tools/conv_mc_bench.py [--steps 10] [--warmup 2] [--geometry a b] [--out FILE.json]

Two geometries: (a) 256 x 4 x 48000 with L 48000 and M in {4, 8, 16}; (b) speech arrays at 16 kHz, 256 x 2 x 64000 with
L 8000 and M in {4, 8} (J = 2, so the window transforms the op saves are a larger share of the work).  For each M it
times, with CUDA events over --steps calls after --warmup, the forward alone, forward + backward with gradients to x and
the IR, and forward + backward with a fixed IR, for:
  mc            multichannel_convolution(x, sr, ir), ir (batch, S, M, L): one matrix per item;
  mc shared     the same with one matrix (1, S, M, L) for the batch;
  composition   ceil(M / 2) convolution_bus calls on the output pairs ir[:, :, 2q:2q+2], concatenated in torch (autograd
                sums their dL/dx);
  torch.fft     rfft / irfft at the next power of two >= n + L - 1 with the source sum in the spectrum (fp32, autograd).
Next to each time it records torch.cuda.max_memory_allocated above the inputs.  It prints the card name, power limit and
SM clock it ran on (the clock read right after the timed calls), and the per-item transform counts of the op and the
composition as they follow from the code (counted, not measured).  Development aid; bench.py is the benchmark."""
import argparse
import json
import math
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import dasp_pytorch_b200 as D  # noqa: E402
from conv_bench import time_ms  # noqa: E402
from profile_step import card  # noqa: E402

KB = 4096
# name: (batch, S, n, L, sample rate, [M])
GEOMETRIES = {"a": (256, 4, 48000, 48000, 48000, [4, 8, 16]), "b": (256, 2, 64000, 8000, 16000, [4, 8])}


def sm_clock(dev):
    """(current, max) SM clock in MHz from a read-only nvidia-smi query, or None"""
    try:
        out = subprocess.run(["nvidia-smi", f"--id={dev.index or 0}", "--query-gpu=clocks.sm,clocks.max.sm",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout
        cur, mx = (float(v) for v in out.strip().splitlines()[0].split(","))
        return cur, mx
    except Exception:
        return None


def composition(x, sample_rate, ir):
    M = ir.shape[2]
    return torch.cat([D.convolution_bus(x, sample_rate, ir[:, :, q:q + 2]) for q in range(0, M, 2)], 1)


def torch_fft_mc(x, sample_rate, ir):
    n, L = x.shape[-1], ir.shape[-1]
    m = 1 << math.ceil(math.log2(n + L - 1))
    return torch.fft.irfft(torch.einsum("bsf,bsmf->bmf", torch.fft.rfft(x, m), torch.fft.rfft(ir, m)), m)[..., :n]


def transform_counts(S, M, n, L):
    """8192-point transforms per item (a shared matrix's partitions: per call), counted from the code"""
    I, J, P, Q, NH = -(-n // KB), -(-min(n, L) // KB), (S + 1) // 2, (M + 1) // 2, (S * M + 1) // 2
    return {"op": {"window": P * I, "partition": NH * J, "inverse": Q * I, "grad": Q * I, "dx_inverse": P * I,
                   "dir_inverse": NH * J, "saved_window_spectra": P * I},
            "composition": {"window": Q * P * I, "partition": NH * J, "inverse": Q * I, "grad": Q * I,
                            "dx_inverse": Q * P * I, "dir_inverse": NH * J, "saved_window_spectra": Q * P * I}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--geometry", nargs="+", default=["a", "b"], choices=sorted(GEOMETRIES))
    ap.add_argument("--out", help="also write the results as JSON to this file")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    name, limit = card(dev)
    print(f"card: {name}, power limit: {limit if limit is not None else 'unknown'} W", flush=True)
    g = torch.Generator(device=dev).manual_seed(0)
    rows, counts, clocks = [], {}, []
    for geo in args.geometry:
        bs, S, n, L, sr, Ms = GEOMETRIES[geo]
        for M in Ms:
            counts[f"{geo} M{M}"] = transform_counts(S, M, n, L)
            print(f"({geo}) S {S} M {M}: transforms per item (counted, not measured): {counts[f'{geo} M{M}']}",
                  flush=True)
            x = torch.rand(bs, S, n, device=dev, generator=g) * 2 - 1
            w = torch.rand(bs, M, n, device=dev, generator=g)
            ir = (torch.rand(bs, S, M, L, device=dev, generator=g) * 2 - 1) * 0.01
            for impl, fn, h in (("mc", D.multichannel_convolution, ir), ("mc shared", D.multichannel_convolution, ir[:1]),
                                ("composition", composition, ir), ("composition shared", composition, ir[:1]),
                                ("torch.fft", torch_fft_mc, ir)):
                def fwd():
                    with torch.no_grad():
                        fn(x, sr, h)

                def fwd_bwd(ir_grad):
                    xx = x.detach().requires_grad_(True)
                    hh = h.detach().requires_grad_(ir_grad)
                    y = fn(xx, sr, hh)
                    torch.autograd.grad((y * w).sum(), (xx, hh) if ir_grad else (xx,))

                for mode, call in (("fwd", fwd), ("fwd+bwd", lambda: fwd_bwd(True)),
                                   ("fwd+bwd, fixed IR", lambda: fwd_bwd(False))):
                    torch.cuda.synchronize()
                    torch.cuda.empty_cache()
                    base = torch.cuda.memory_allocated()
                    torch.cuda.reset_peak_memory_stats()
                    ms = time_ms(call, args.steps, args.warmup)
                    clk = sm_clock(dev)
                    clocks.append(clk)
                    peak = (torch.cuda.max_memory_allocated() - base) / 2**20
                    rows.append({"geometry": geo, "S": S, "M": M, "impl": impl, "mode": mode, "ms": round(ms, 3),
                                 "peak_mib": round(peak, 1), "sm_clock_mhz": clk[0] if clk else None})
                    print(f"({geo}) {bs} x {S} x {n}, L {L}, M {M}: {impl:18s} {mode:18s} {ms:8.2f} ms  "
                          f"peak {peak:8.1f} MiB above the inputs  SM clock {clk[0] if clk else '?'} MHz", flush=True)
            del x, w, ir
            torch.cuda.empty_cache()
    known = [c for c in clocks if c]
    if known:
        print(f"SM clock after the timed calls: {min(c[0] for c in known):.0f}-{max(c[0] for c in known):.0f} MHz "
              f"(max {known[0][1]:.0f} MHz)", flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"card": name, "power_limit_w": limit, "steps": args.steps, "transform_counts": counts,
                       "results": rows}, f, indent=1)


if __name__ == "__main__":
    main()
