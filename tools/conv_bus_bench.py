"""Time convolution_bus (S inputs summed into a stereo bus) against what a caller does without it, on the same GPU.

    python tools/conv_bus_bench.py [--batch 256] [--n 48000] [--ir 48000] [--inputs 4 8 16] [--steps 20] [--warmup 3]
                                   [--out FILE.json]

For each S it times, with CUDA events over --steps calls after --warmup, the forward alone, forward + backward with
gradients to x and the IR, and forward + backward with a fixed IR, for:
  bus          convolution_bus(x, sr, ir), ir (batch, S, 2, L): one IR set per item;
  bus shared   the same with one set (1, S, 2, L) for the batch;
  composition  x viewed as (batch S, 1, n), one convolution_reverberation call per source at mix 1 (a shared set is
               expanded per source), the result viewed as (batch, S, 2, n) and summed over S in torch;
  torch.fft    rfft / irfft at the next power of two >= n + L - 1 with the source sum in the spectrum (fp32, autograd).
Next to each time it records torch.cuda.max_memory_allocated above the inputs.  It prints the card name and power limit
it ran on, and the per-item transform counts of the fused op and the composition as they follow from the code (counted,
not measured).  Development aid; bench.py is the benchmark."""
import argparse
import json
import math
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import dasp_pytorch_b200 as D  # noqa: E402
from conv_bench import time_ms  # noqa: E402
from profile_step import card  # noqa: E402

KB = 4096


def composition(x, sample_rate, ir):
    bs, S, n = x.shape
    ir = ir.expand(bs, -1, -1, -1).reshape(bs * S, 2, ir.shape[-1])
    one = torch.ones(bs * S, device=x.device)
    return D.convolution_reverberation(x.reshape(bs * S, 1, n), sample_rate, ir, one).view(bs, S, 2, n).sum(1)


def torch_fft_bus(x, sample_rate, ir):
    n, L = x.shape[-1], ir.shape[-1]
    m = 1 << math.ceil(math.log2(n + L - 1))
    return torch.fft.irfft(torch.einsum("bsf,bsof->bof", torch.fft.rfft(x, m), torch.fft.rfft(ir, m)), m)[..., :n]


def transform_counts(S, n, L):
    """8192-point transforms per item (a shared IR's partitions: per call), stereo bus, counted from the code"""
    I, J, P = -(-n // KB), -(-min(n, L) // KB), (S + 1) // 2
    return {"fused": {"window": P * I, "partition": S * J, "inverse": I, "grad": I, "dx_inverse": P * I,
                      "dir_inverse": S * J},
            "composition": {"window": S * I, "partition": S * J, "inverse": S * I, "grad": S * I,
                            "dx_inverse": S * I, "dir_inverse": S * J}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--n", type=int, default=48000)
    ap.add_argument("--ir", type=int, default=48000)
    ap.add_argument("--inputs", type=int, nargs="+", default=[4, 8, 16])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", help="also write the results as JSON to this file")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    name, limit = card(dev)
    print(f"card: {name}, power limit: {limit if limit is not None else 'unknown'} W", flush=True)
    bs, n, L = args.batch, args.n, args.ir
    g = torch.Generator(device=dev).manual_seed(0)
    rows, counts = [], {}
    for S in args.inputs:
        counts[S] = transform_counts(S, n, L)
        print(f"S {S}: transforms per item (counted, not measured): {counts[S]}", flush=True)
        x = torch.rand(bs, S, n, device=dev, generator=g) * 2 - 1
        w = torch.rand(bs, 2, n, device=dev, generator=g)
        ir = (torch.rand(bs, S, 2, L, device=dev, generator=g) * 2 - 1) * 0.01
        for impl, fn, h in (("bus", D.convolution_bus, ir), ("bus shared", D.convolution_bus, ir[:1]),
                            ("composition", composition, ir), ("composition shared", composition, ir[:1]),
                            ("torch.fft", torch_fft_bus, ir)):
            def fwd():
                with torch.no_grad():
                    fn(x, 44100, h)

            def fwd_bwd(ir_grad):
                xx = x.detach().requires_grad_(True)
                hh = h.detach().requires_grad_(ir_grad)
                y = fn(xx, 44100, hh)
                torch.autograd.grad((y * w).sum(), (xx, hh) if ir_grad else (xx,))

            for mode, call in (("fwd", fwd), ("fwd+bwd", lambda: fwd_bwd(True)),
                               ("fwd+bwd, fixed IR", lambda: fwd_bwd(False))):
                torch.cuda.synchronize()
                torch.cuda.empty_cache()
                base = torch.cuda.memory_allocated()
                torch.cuda.reset_peak_memory_stats()
                ms = time_ms(call, args.steps, args.warmup)
                peak = (torch.cuda.max_memory_allocated() - base) / 2**20
                rows.append({"S": S, "impl": impl, "mode": mode, "ms": round(ms, 3), "peak_mib": round(peak, 1)})
                print(f"batch {bs} x {S} x {n}, IR {L}: {impl:18s} {mode:18s} {ms:8.2f} ms  peak {peak:8.1f} MiB "
                      "above the inputs", flush=True)
        del x, w, ir
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"card": name, "power_limit_w": limit, "batch": bs, "n": n, "ir": L, "steps": args.steps,
                       "transform_counts": counts, "results": rows}, f, indent=1)


if __name__ == "__main__":
    main()
