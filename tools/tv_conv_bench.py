"""Time time_varying_convolution_reverberation against what a caller does without it, on the same GPU.

    python tools/tv_conv_bench.py [--batch 256] [--n 480000] [--ir 48000] [--hop 32768] [--irs 15] [--steps 20]
                                  [--warmup 3] [--out FILE.json]

It times, with CUDA events over --steps calls after --warmup, the forward alone, forward + backward with gradients to
x, the IRs and mix, and forward + backward with a fixed trajectory, for:
  tv              time_varying_convolution_reverberation(x, sr, ir, hop, mix), ir (batch, K, 2, L);
  tv shared       the same with one trajectory (1, K, 2, L) for the batch;
  full-length     K convolution_reverberation calls at mix 1 over the whole of x, one per IR, weighted and summed in torch;
  cropped         the same on the output segment each IR reaches (two anchor intervals, plus L - 1 samples of input
                  history), overlap-added in torch;
  torch.fft       rfft / irfft at the next power of two >= n + L - 1, one product and inverse per IR (fp32, autograd).
Next to each time it records torch.cuda.max_memory_allocated above the inputs; an implementation that runs out of
memory is reported as such.  It prints the card name, power limit and SM clock (maximum, and the current clock read
right after the timed calls) it ran on, and the per-item transform counts of the op and of the full-length composition
as they follow from the code (counted, not measured).  Development aid; bench.py is the benchmark."""
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

KB = 4096
SR = 48000


def card(dev):
    """name, power limit (W), maximum and current SM clock (MHz) of the device, from read-only nvidia-smi queries"""
    info = {"name": torch.cuda.get_device_name(dev), "power_limit_w": None, "sm_clock_max_mhz": None,
            "sm_clock_mhz": None}
    try:
        out = subprocess.run(["nvidia-smi", f"--id={dev.index or 0}", "--query-gpu=power.limit,clocks.max.sm,clocks.sm",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout
        lim, cmax, cur = (float(v) for v in out.strip().splitlines()[0].split(","))
        info.update(power_limit_w=lim, sm_clock_max_mhz=cmax, sm_clock_mhz=cur)
    except Exception:
        pass
    return info


def weights(K, hop, n, dev):
    """(K, n) crossfade weights of the op's definition"""
    t = torch.arange(n, device=dev, dtype=torch.float32)
    w = torch.zeros(K, n, device=dev)
    for k in range(K - 1):
        seg = (t >= k * hop) & (t < (k + 1) * hop)
        a = (t[seg] - k * hop) / hop
        w[k, seg] += 1 - a
        w[k + 1, seg] += a
    w[K - 1, (K - 1) * hop:] = 1
    return w


def full_length(x, ir, hop, mix, w):
    bs, K = x.shape[0], ir.shape[1]
    one = torch.ones(bs, device=x.device)
    wet = sum(w[k] * D.convolution_reverberation(x, SR, ir[:, k], one) for k in range(K))
    m = mix.reshape(-1, 1, 1)
    return (1 - m) * x + m * wet


def cropped(x, ir, hop, mix, w):
    bs, _, n = x.shape
    K, L = ir.shape[1], ir.shape[-1]
    one = torch.ones(bs, device=x.device)
    parts = []
    for k in range(K):
        s0, s1 = max(0, (k - 1) * hop), (n if k == K - 1 else min(n, (k + 1) * hop))
        c0 = max(0, s0 - (L - 1))
        seg = D.convolution_reverberation(x[..., c0:s1], SR, ir[:, k], one)[..., s0 - c0:]
        parts.append(torch.nn.functional.pad(w[k, s0:s1] * seg, (s0, n - s1)))
    m = mix.reshape(-1, 1, 1)
    return (1 - m) * x + m * sum(parts)


def torch_fft(x, ir, hop, mix, w):
    n, L, K = x.shape[-1], ir.shape[-1], ir.shape[1]
    mm = 1 << math.ceil(math.log2(n + L - 1))
    X = torch.fft.rfft(x, mm)
    wet = sum(w[k] * torch.fft.irfft(X * torch.fft.rfft(ir[:, k], mm), mm)[..., :n] for k in range(K))
    m = mix.reshape(-1, 1, 1)
    return (1 - m) * x + m * wet


def transform_counts(K, hop, n, L):
    """8192-point transforms per item, stereo x and trajectory (a shared trajectory's partitions: per call), counted
    from the code"""
    I, J = -(-n // KB), -(-min(n, L) // KB)
    nX = (K - 1) * hop // KB
    return {"tv": {"window": I, "partition": K * J, "inverse": I + nX, "grad": I + nX, "dx_inverse": I,
                   "dir_inverse": K * J},
            "full-length": {"window": K * I, "partition": K * J, "inverse": K * I, "grad": K * I, "dx_inverse": K * I,
                            "dir_inverse": K * J}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--n", type=int, default=480000)
    ap.add_argument("--ir", type=int, default=48000)
    ap.add_argument("--hop", type=int, default=32768)
    ap.add_argument("--irs", type=int, default=15)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", help="also write the results as JSON to this file")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    bs, n, L, hop, K = args.batch, args.n, args.ir, args.hop, args.irs
    counts = transform_counts(K, hop, n, L)
    print(f"transforms per item (counted, not measured): {counts}", flush=True)
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.rand(bs, 2, n, device=dev, generator=g) * 2 - 1
    gw = torch.rand(bs, 2, n, device=dev, generator=g)
    ir = (torch.rand(bs, K, 2, L, device=dev, generator=g) * 2 - 1) * 0.01
    mix = torch.rand(bs, device=dev, generator=g)
    w = weights(K, hop, n, dev)
    tv = lambda x, h, hop, m, w: D.time_varying_convolution_reverberation(x, SR, h, hop, m)
    rows = []
    for impl, fn, h in (("tv", tv, ir), ("tv shared", tv, ir[:1]), ("full-length", full_length, ir),
                        ("cropped", cropped, ir), ("torch.fft", torch_fft, ir)):
        def fwd():
            with torch.no_grad():
                fn(x, h, hop, mix, w)

        def fwd_bwd(ir_grad):
            xx, mm = x.detach().requires_grad_(True), mix.detach().requires_grad_(True)
            hh = h.detach().requires_grad_(ir_grad)
            y = fn(xx, hh, hop, mm, w)
            torch.autograd.grad((y * gw).sum(), (xx, hh, mm) if ir_grad else (xx, mm))

        for mode, call in (("fwd", fwd), ("fwd+bwd", lambda: fwd_bwd(True)),
                           ("fwd+bwd, fixed IR", lambda: fwd_bwd(False))):
            torch.cuda.synchronize()
            torch.cuda.empty_cache()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            try:
                ms = round(time_ms(call, args.steps, args.warmup), 3)
                peak = round((torch.cuda.max_memory_allocated() - base) / 2**30, 2)
            except torch.cuda.OutOfMemoryError:
                ms = peak = "out of memory"
            clock = card(dev)["sm_clock_mhz"]
            rows.append({"impl": impl, "mode": mode, "ms": ms, "peak_gib": peak, "sm_clock_mhz_after": clock})
            print(f"batch {bs} x 2 x {n}, K {K} x 2 x {L}, hop {hop}: {impl:12s} {mode:18s} {ms} ms  peak {peak} GiB "
                  f"above the inputs (SM clock after: {clock} MHz)", flush=True)
    info = card(dev)
    print(f"card: {info['name']}, power limit: {info['power_limit_w']} W, max SM clock: {info['sm_clock_max_mhz']} MHz",
          flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"card": info, "batch": bs, "n": n, "ir": L, "hop": hop, "irs": K, "steps": args.steps,
                       "transform_counts": counts, "results": rows}, f, indent=1)


if __name__ == "__main__":
    main()
