"""Time time_varying_convolution_bus with crossfade="input" against what a caller does without it, on the same GPU.

    python tools/tv_bus_input_bench.py [--batch 64] [--sources 4] [--outputs 2] [--n 480000] [--ir 48000]
                                       [--hop 32768] [--irs 15] [--steps 10] [--warmup 3] [--kernels] [--out FILE.json]

It times, with CUDA events over --steps calls after --warmup, the forward alone, forward + backward with gradients to
x and the IRs, and forward + backward with a fixed trajectory set, for:
  tv bus in          time_varying_convolution_bus(x, sr, ir, hop, crossfade="input"), ir (batch, K, S, O, L);
  tv bus in shared   the same with one set (1, K, S, O, L) for the batch;
  segments           the segment composition: the K weighted segments (w_k x)[(k-1) hop : (k+1) hop] (the last one to
                     the end of x), each zero-padded to hold its L - 1 tail, go as batch K items through one
                     convolution_bus call and are overlap-added in torch;
  segments shared    the same with the shared set expanded over the batch;
  torch.fft          rfft / irfft at the next power of two >= n + L - 1 of every weighted source, one product per IR
                     set summed over the sources (fp32, autograd);
  tv bus out         the output-side op on the same inputs: a different result, timed for the cost comparison.
Next to each time it records torch.cuda.max_memory_allocated above the inputs; an implementation that runs out of
memory is reported as such.  It prints the card name, power limit and SM clock, and the per-item transform counts of
the op as they follow from the code (counted, not measured).  --kernels then records one fwd+bwd of the op and of the
segment composition under torch.profiler (a separate pass) and prints the summed device time of every kernel.  The
timing, clock and weight helpers are tools/tv_bus_bench.py's.  Development aid; bench.py is the benchmark."""
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
from tv_bus_bench import card, kernel_times, time_ms, weights  # noqa: E402

KB = 4096
SR = 48000


def tv_bus_in(x, ir, hop, w):
    return D.time_varying_convolution_bus(x, SR, ir, hop, crossfade="input")


def tv_bus_out(x, ir, hop, w):
    return D.time_varying_convolution_bus(x, SR, ir, hop)


def segments(x, ir, hop, w):
    bs, S, n = x.shape
    K, L = ir.shape[1], ir.shape[-1]
    ir = ir.expand(bs, -1, -1, -1, -1)
    starts = [max(0, (k - 1) * hop) for k in range(K)]
    ends = [min(n, (k + 1) * hop) if k < K - 1 else n for k in range(K)]
    seg = max(e - s for s, e in zip(starts, ends)) + L - 1
    xs = torch.stack([torch.nn.functional.pad((w[k, s:e] * x[..., s:e]), (0, seg - (e - s)))
                      for k, (s, e) in enumerate(zip(starts, ends))])                    # (K, bs, S, seg)
    ys = D.convolution_bus(xs.reshape(K * bs, S, seg), SR, ir.transpose(0, 1).reshape(K * bs, S, -1, L))
    ys = ys.reshape(K, bs, -1, seg)
    y = x.new_zeros(bs, ys.shape[2], n + seg)
    for k, s in enumerate(starts):
        y = y + torch.nn.functional.pad(ys[k], (s, n - s))
    return y[..., :n]


def torch_fft(x, ir, hop, w):
    n, L, K = x.shape[-1], ir.shape[-1], ir.shape[1]
    mm = 1 << math.ceil(math.log2(n + L - 1))
    return torch.fft.irfft(sum((torch.fft.rfft(w[k] * x, mm)[:, :, None] * torch.fft.rfft(ir[:, k], mm)).sum(1)
                               for k in range(K)), mm)[..., :n]


def transform_counts(K, S, O, hop, n, L):
    """8192-point transforms per item (a shared set's partitions: per call), counted from the code"""
    I, J = -(-n // KB), -(-min(n, L) // KB)
    nX = (K - 1) * hop // KB
    P, NH = (S + 1) // 2, (K * S * O + 1) // 2
    XW = nX * S + (I - nX) * P
    U = I + nX if O == 2 else I
    return {"tv bus in": {"window": XW, "partition": NH * J, "inverse": I, "grad": I, "dx_inverse": XW,
                          "dir_inverse": NH * J, "kept_spectra": XW + NH * J},
            "tv bus out": {"window": P * I, "partition": NH * J, "inverse": U, "grad": U, "dx_inverse": P * I,
                           "dir_inverse": NH * J, "kept_spectra": P * I + NH * J}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--sources", type=int, default=4)
    ap.add_argument("--outputs", type=int, default=2)
    ap.add_argument("--n", type=int, default=480000)
    ap.add_argument("--ir", type=int, default=48000)
    ap.add_argument("--hop", type=int, default=32768)
    ap.add_argument("--irs", type=int, default=15)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--kernels", action="store_true", help="also print per-kernel device times of one fwd+bwd")
    ap.add_argument("--out", help="also write the results as JSON to this file")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    bs, S, O, n, L, hop, K = args.batch, args.sources, args.outputs, args.n, args.ir, args.hop, args.irs
    counts = transform_counts(K, S, O, hop, n, L)
    print(f"transforms per item (counted, not measured): {counts}", flush=True)
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.rand(bs, S, n, device=dev, generator=g) * 2 - 1
    gw = torch.rand(bs, O, n, device=dev, generator=g)
    ir = (torch.rand(bs, K, S, O, L, device=dev, generator=g) * 2 - 1) * 0.01
    w = weights(K, hop, n, dev)
    impls = (("tv bus in", tv_bus_in, ir), ("tv bus in shared", tv_bus_in, ir[:1]), ("segments", segments, ir),
             ("segments shared", segments, ir[:1]), ("torch.fft", torch_fft, ir), ("tv bus out", tv_bus_out, ir))

    def fwd_bwd(fn, h, ir_grad):
        xx, hh = x.detach().requires_grad_(True), h.detach().requires_grad_(ir_grad)
        y = fn(xx, hh, hop, w)
        torch.autograd.grad((y * gw).sum(), (xx, hh) if ir_grad else (xx,))

    rows = []
    for impl, fn, h in impls:
        def fwd():
            with torch.no_grad():
                fn(x, h, hop, w)

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
            print(f"batch {bs} x {S} x {n}, K {K} x {S} x {O} x {L}, hop {hop}: {impl:18s} {mode:18s} {ms} ms  "
                  f"peak {peak} GiB above the inputs (SM clock after: {clock} MHz)", flush=True)
    kernels = {}
    if args.kernels:
        torch.cuda.empty_cache()
        for impl, fn, h in impls[:4]:
            kernels[impl] = {k: round(v, 3) for k, v in kernel_times(lambda: fwd_bwd(fn, h, True)).items()}
            print(f"kernels, one fwd+bwd of {impl}: {kernels[impl]}", flush=True)
    info = card(dev)
    print(f"card: {info['name']}, power limit: {info['power_limit_w']} W, max SM clock: {info['sm_clock_max_mhz']} MHz",
          flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"card": info, "batch": bs, "sources": S, "outputs": O, "n": n, "ir": L, "hop": hop, "irs": K,
                       "steps": args.steps, "transform_counts": counts, "results": rows, "kernels": kernels}, f,
                      indent=1)


if __name__ == "__main__":
    main()
