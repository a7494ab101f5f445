"""Time time_varying_multichannel_convolution against what a caller does without it, on the same GPU.

    python tools/tv_mc_bench.py [--batch 16] [--sources 4] [--outputs 8] [--n 480000] [--ir 48000] [--hop 32768]
                                [--irs 15] [--crossfade output|input] [--steps 10] [--warmup 3] [--out FILE.json]

It times, with CUDA events over --steps calls after --warmup, the forward alone, forward + backward with gradients to
x and the IRs, and forward + backward with a fixed trajectory, for:
  tv mc              time_varying_multichannel_convolution(x, sr, ir, hop, crossfade=...), ir (batch, K, S, M, L);
  tv mc shared       the same with one trajectory (1, K, S, M, L) for the batch;
  tv bus pairs       the Q = ceil(M / 2) time_varying_convolution_bus calls on the output pairs, concatenated in torch
                     (autograd sums their Q copies of dL/dx);
  tv bus pairs shared  the same with the shared trajectory;
  torch.fft          rfft / irfft at the next power of two >= n + L - 1 of x (output side) or of every weighted source
                     (input side), one product per IR set summed over the sources (fp32, autograd).
Next to each time it records torch.cuda.max_memory_allocated above the inputs; an implementation that runs out of
memory is reported as such.  It prints the card name, power limit and SM clock, and the per-item transform counts of
the op and of the composition as they follow from the code (counted, not measured).  The timing, clock and weight
helpers are tools/tv_bus_bench.py's.  Development aid; bench.py is the benchmark."""
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
from tv_bus_bench import card, time_ms, weights  # noqa: E402

KB = 4096
SR = 48000


def transform_counts(K, S, M, hop, n, L):
    """8192-point transforms per item (a shared trajectory's partitions: per call), counted from the code, for the op
    and for the output-pair composition, both crossfades"""
    I, J = -(-n // KB), -(-min(n, L) // KB)
    nX = (K - 1) * hop // KB
    P, Q, NH = (S + 1) // 2, (M + 1) // 2, (K * S * M + 1) // 2
    XW = nX * S + (I - nX) * P
    out = {"window": P * I, "partition": NH * J, "inverse": M * nX + Q * (I - nX), "grad": M * nX + Q * (I - nX),
           "dx_inverse": P * I, "dir_inverse": NH * J, "kept_spectra": P * I + NH * J}
    inp = {"window": XW, "partition": NH * J, "inverse": Q * I, "grad": Q * I, "dx_inverse": XW,
           "dir_inverse": NH * J, "kept_spectra": XW + NH * J}
    # one time_varying_convolution_bus call per output pair (the last one mono when M is odd)
    pairs = {}
    for name, mc, win in (("output", out, P * I), ("input", inp, XW)):
        per = {k: 0 for k in mc}
        for q in range(Q):
            O = 2 if 2 * q + 1 < M else 1
            nh = (K * S * O + 1) // 2
            u = (I + nX if O == 2 else I) if name == "output" else I
            for k, v in (("window", win), ("partition", nh * J), ("inverse", u), ("grad", u), ("dx_inverse", win),
                         ("dir_inverse", nh * J), ("kept_spectra", win + nh * J)):
                per[k] += v
        pairs[name] = per
    return {"tv mc output": out, "tv bus pairs output": pairs["output"], "tv mc input": inp,
            "tv bus pairs input": pairs["input"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--sources", type=int, default=4)
    ap.add_argument("--outputs", type=int, default=8)
    ap.add_argument("--n", type=int, default=480000)
    ap.add_argument("--ir", type=int, default=48000)
    ap.add_argument("--hop", type=int, default=32768)
    ap.add_argument("--irs", type=int, default=15)
    ap.add_argument("--crossfade", choices=("output", "input"), default="output")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--no-fft", action="store_true", help="skip the torch.fft rows")
    ap.add_argument("--out", help="also write the results as JSON to this file")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    bs, S, M, n, L, hop, K, xf = (args.batch, args.sources, args.outputs, args.n, args.ir, args.hop, args.irs,
                                  args.crossfade)
    counts = transform_counts(K, S, M, hop, n, L)
    print(f"transforms per item (counted, not measured): {counts}", flush=True)
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.rand(bs, S, n, device=dev, generator=g) * 2 - 1
    gw = torch.rand(bs, M, n, device=dev, generator=g)
    ir = (torch.rand(bs, K, S, M, L, device=dev, generator=g) * 2 - 1) * 0.01
    w = weights(K, hop, n, dev)

    def tv_mc(xx, h):
        return D.time_varying_multichannel_convolution(xx, SR, h, hop, crossfade=xf)

    def pairs(xx, h):
        return torch.cat([D.time_varying_convolution_bus(xx, SR, h[:, :, :, q:q + 2], hop, crossfade=xf)
                          for q in range(0, M, 2)], 1)

    def torch_fft(xx, h):
        mm = 1 << math.ceil(math.log2(n + L - 1))
        if xf == "output":
            X = torch.fft.rfft(xx, mm)[:, :, None]
            return sum(w[k] * torch.fft.irfft((X * torch.fft.rfft(h[:, k], mm)).sum(1), mm)[..., :n]
                       for k in range(K))
        return torch.fft.irfft(sum((torch.fft.rfft(w[k] * xx, mm)[:, :, None] * torch.fft.rfft(h[:, k], mm)).sum(1)
                                   for k in range(K)), mm)[..., :n]

    impls = [("tv mc", tv_mc, ir), ("tv mc shared", tv_mc, ir[:1]), ("tv bus pairs", pairs, ir),
             ("tv bus pairs shared", pairs, ir[:1])]
    if not args.no_fft:
        impls.append(("torch.fft", torch_fft, ir))

    def fwd_bwd(fn, h, ir_grad):
        xx, hh = x.detach().requires_grad_(True), h.detach().requires_grad_(ir_grad)
        y = fn(xx, hh)
        torch.autograd.grad((y * gw).sum(), (xx, hh) if ir_grad else (xx,))

    rows = []
    for impl, fn, h in impls:
        def fwd():
            with torch.no_grad():
                fn(x, h)

        for mode, call in (("fwd", fwd), ("fwd+bwd", lambda: fwd_bwd(fn, h, True)),
                           ("fwd+bwd, fixed IR", lambda: fwd_bwd(fn, h, False))):
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
            print(f"{xf} batch {bs} x {S} x {n}, K {K} x {S} x {M} x {L}, hop {hop}: {impl:20s} {mode:18s} {ms} ms  "
                  f"peak {peak} GiB above the inputs (SM clock after: {clock} MHz)", flush=True)
    info = card(dev)
    print(f"card: {info['name']}, power limit: {info['power_limit_w']} W, max SM clock: {info['sm_clock_max_mhz']} MHz",
          flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"card": info, "crossfade": xf, "batch": bs, "sources": S, "outputs": M, "n": n, "ir": L,
                       "hop": hop, "irs": K, "steps": args.steps, "transform_counts": counts, "results": rows}, f,
                      indent=1)


if __name__ == "__main__":
    main()
