"""Time convolution_reverberation next to a torch.fft FFT convolution on the same GPU.

    python tools/conv_bench.py [--batch 1024] [--n 48000] [--steps 20] [--warmup 3] [--out FILE.json]

For IR lengths 48000 and 96000 at batch x 2 x n (stereo x and IR, one mix per item) it times, with CUDA events after
warm-up: the forward alone, forward + backward with gradients to x, IR and mix, and forward + backward with a fixed IR
(gradients to x and mix only).  The comparison is the same arithmetic in torch.fft: rfft / irfft at the next power of two
>= n + L - 1 (2^17 for both lengths), fp32, with autograd.  Prints the card name and power limit it ran on: both belong
beside any number it produces.  Development aid; bench.py is the benchmark."""
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
from profile_step import card  # noqa: E402


def torch_fft_conv(x, sample_rate, ir, mix):
    n, L = x.shape[-1], ir.shape[-1]
    m = 1 << math.ceil(math.log2(n + L - 1))
    wet = torch.fft.irfft(torch.fft.rfft(x, m) * torch.fft.rfft(ir, m), m)[..., :n]
    mix = mix.reshape(-1, 1, 1)
    return (1.0 - mix) * x + mix * wet


def time_ms(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--n", type=int, default=48000)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", help="also write the results as JSON to this file")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    name, limit = card(dev)
    print(f"card: {name}, power limit: {limit if limit is not None else 'unknown'} W", flush=True)
    bs, n = args.batch, args.n
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.rand(bs, 2, n, device=dev, generator=g) * 2 - 1
    w = torch.rand(bs, 2, n, device=dev, generator=g)
    mix = torch.rand(bs, device=dev, generator=g)
    rows = []
    for L in (48000, 96000):
        ir = (torch.rand(bs, 2, L, device=dev, generator=g) * 2 - 1) * 0.01
        for impl, fn in (("dasp", D.convolution_reverberation), ("torch.fft", torch_fft_conv)):
            def fwd():
                with torch.no_grad():
                    fn(x, 44100, ir, mix)

            def fwd_bwd(ir_grad):
                xx = x.detach().requires_grad_(True)
                hh = ir.detach().requires_grad_(ir_grad)
                mm = mix.detach().requires_grad_(True)
                y = fn(xx, 44100, hh, mm)
                torch.autograd.grad((y * w).sum(), (xx, hh, mm) if ir_grad else (xx, mm))

            for mode, call in (("fwd", fwd), ("fwd+bwd", lambda: fwd_bwd(True)),
                               ("fwd+bwd, fixed IR", lambda: fwd_bwd(False))):
                ms = time_ms(call, args.steps, args.warmup)
                rows.append({"L": L, "impl": impl, "mode": mode, "ms": round(ms, 3)})
                print(f"batch {bs} x 2 x {n}, IR {L}: {impl:9s} {mode:18s} {ms:8.2f} ms", flush=True)
        del ir
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"card": name, "power_limit_w": limit, "batch": bs, "n": n, "steps": args.steps,
                       "results": rows}, f, indent=1)


if __name__ == "__main__":
    main()
