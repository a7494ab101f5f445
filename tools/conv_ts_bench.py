"""Time convolution_reverberation with a TRUE-STEREO (four-channel) impulse response, four ways, on the same GPU.

    python tools/conv_ts_bench.py [--batch 1024] [--n 48000] [--steps 20] [--warmup 3] [--out FILE.json]

For IR lengths 48000 and 96000 at batch x 2 x n (stereo x, a (L->L, L->R, R->L, R->R) IR, one mix per item) it times,
with CUDA events after warm-up, the forward alone, forward + backward with gradients to x, the IR and mix, and forward +
backward with a fixed IR, for:
  ts         convolution_reverberation(x, sr, ir, mix) with ir of shape (batch, 4, L): one call;
  ts shared  the same with one IR of shape (1, 4, L) for the whole batch;
  two calls  what a caller does without the feature: the left channel through (L->L, L->R) and the right channel through
             (R->L, R->R), each a stereo-IR call at mix 1, then the sum blended with the dry signal in torch;
  torch.fft  the same arithmetic in torch.fft (rfft / irfft at the next power of two >= n + L - 1, fp32, autograd).
Next to each time it records torch.cuda.max_memory_allocated over the timed calls.  Prints the card name and power limit
it ran on: both belong beside any number it produces.  Development aid; bench.py is the benchmark."""
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


def two_calls(x, sample_rate, ir, mix):
    one = torch.ones_like(mix)
    wet = (D.convolution_reverberation(x[:, 0:1], sample_rate, ir[:, 0:2], one)
           + D.convolution_reverberation(x[:, 1:2], sample_rate, ir[:, 2:4], one))
    m = mix.reshape(-1, 1, 1)
    return (1.0 - m) * x + m * wet


def torch_fft_ts(x, sample_rate, ir, mix):
    n, L = x.shape[-1], ir.shape[-1]
    m = 1 << math.ceil(math.log2(n + L - 1))
    xs, hs = torch.fft.rfft(x, m), torch.fft.rfft(ir, m)
    wet = torch.fft.irfft(xs[:, 0:1] * hs[:, 0:2] + xs[:, 1:2] * hs[:, 2:4], m)[..., :n]
    mix = mix.reshape(-1, 1, 1)
    return (1.0 - mix) * x + mix * wet


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
        ir = (torch.rand(bs, 4, L, device=dev, generator=g) * 2 - 1) * 0.01
        for impl, fn, h in (("ts", D.convolution_reverberation, ir), ("ts shared", D.convolution_reverberation, ir[:1]),
                            ("two calls", two_calls, ir), ("torch.fft", torch_fft_ts, ir)):
            def fwd():
                with torch.no_grad():
                    fn(x, 44100, h, mix)

            def fwd_bwd(ir_grad):
                xx = x.detach().requires_grad_(True)
                hh = h.detach().requires_grad_(ir_grad)
                mm = mix.detach().requires_grad_(True)
                y = fn(xx, 44100, hh, mm)
                torch.autograd.grad((y * w).sum(), (xx, hh, mm) if ir_grad else (xx, mm))

            for mode, call in (("fwd", fwd), ("fwd+bwd", lambda: fwd_bwd(True)),
                               ("fwd+bwd, fixed IR", lambda: fwd_bwd(False))):
                torch.cuda.synchronize()
                torch.cuda.empty_cache()
                base = torch.cuda.memory_allocated()
                torch.cuda.reset_peak_memory_stats()
                ms = time_ms(call, args.steps, args.warmup)
                peak = (torch.cuda.max_memory_allocated() - base) / 2**20
                rows.append({"L": L, "impl": impl, "mode": mode, "ms": round(ms, 3), "peak_mib": round(peak, 1)})
                print(f"batch {bs} x 2 x {n}, IR {L}: {impl:9s} {mode:18s} {ms:8.2f} ms  peak {peak:8.1f} MiB "
                      "above the inputs", flush=True)
        del ir
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"card": name, "power_limit_w": limit, "batch": bs, "n": n, "steps": args.steps,
                       "results": rows}, f, indent=1)


if __name__ == "__main__":
    main()
