"""Time time_varying_convolution_bus against what a caller does without it, on the same GPU.

    python tools/tv_bus_bench.py [--batch 64] [--sources 4] [--outputs 2] [--n 480000] [--ir 48000] [--hop 32768]
                                 [--irs 15] [--steps 10] [--warmup 3] [--kernels] [--out FILE.json]

It times, with CUDA events over --steps calls after --warmup, the forward alone, forward + backward with gradients to
x and the IRs, and forward + backward with a fixed trajectory set, for:
  tv bus          time_varying_convolution_bus(x, sr, ir, hop), x (batch, S, n), ir (batch, K, S, O, L);
  tv bus shared   the same with one set (1, K, S, O, L) for the batch;
  composition     S time_varying_convolution_reverberation calls at mix 1, one per source (mono x, the source's
                  trajectory h[:, :, s] as its IR), summed in torch (a mono bus takes channel 0 of a mono-IR call);
  composition shared   the same with the shared set;
  torch.fft       rfft / irfft at the next power of two >= n + L - 1: one product per IR set summed over the sources,
                  one inverse per set and output, weighted and summed (fp32, autograd).
Next to each time it records torch.cuda.max_memory_allocated above the inputs; an implementation that runs out of
memory is reported as such.  It prints the card name, power limit and SM clock (maximum, and the current clock read
right after the timed calls), and the per-item transform counts of the op and of the composition as they follow from
the code (counted, not measured).  --kernels then records one fwd+bwd of the op and of the composition under
torch.profiler (a separate pass, after the timings) and prints the summed device time of every kernel.  Development
aid; bench.py is the benchmark."""
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
from tv_conv_bench import card, weights  # noqa: E402

KB = 4096
SR = 48000


def tv_bus(x, ir, hop, w):
    return D.time_varying_convolution_bus(x, SR, ir, hop)


def composition(x, ir, hop, w):
    bs, S, _ = x.shape
    O = ir.shape[3]
    one = torch.ones(bs, device=x.device)
    return sum(D.time_varying_convolution_reverberation(x[:, s:s + 1], SR, ir[:, :, s], hop, one)[:, :O]
               for s in range(S))


def torch_fft(x, ir, hop, w):
    n, L, K = x.shape[-1], ir.shape[-1], ir.shape[1]
    mm = 1 << math.ceil(math.log2(n + L - 1))
    X = torch.fft.rfft(x, mm)[:, :, None]
    return sum(w[k] * torch.fft.irfft((X * torch.fft.rfft(ir[:, k], mm)).sum(1), mm)[..., :n] for k in range(K))


def transform_counts(K, S, O, hop, n, L):
    """8192-point transforms per item (a shared set's partitions: per call), counted from the code"""
    I, J = -(-n // KB), -(-min(n, L) // KB)
    nX = (K - 1) * hop // KB
    P, NH = (S + 1) // 2, (K * S * O + 1) // 2
    U = I + nX if O == 2 else I
    return {"tv bus": {"window": P * I, "partition": NH * J, "inverse": U, "grad": U, "dx_inverse": P * I,
                       "dir_inverse": NH * J},
            # one call per source: mono x, a stereo (O = 2) or mono (O = 1) trajectory in ceil(K O / 2) sets
            "composition": {"window": S * I, "partition": S * ((K * O + 1) // 2) * J, "inverse": S * (I + nX),
                            "grad": S * (I + nX), "dx_inverse": S * I, "dir_inverse": S * ((K * O + 1) // 2) * J}}


def kernel_times(call):
    """{kernel name: summed device ms} of one call under torch.profiler"""
    from torch.profiler import ProfilerActivity, profile
    call()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call()
        torch.cuda.synchronize()
    out = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            name = e.name.replace("(anonymous namespace)::", "").replace("void ", "").replace("dasp::", "")
            name = name.split("(")[0]
            out[name] = out.get(name, 0.0) + e.device_time_total / 1000.0
    return dict(sorted(out.items(), key=lambda kv: -kv[1]))


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
    impls = (("tv bus", tv_bus, ir), ("tv bus shared", tv_bus, ir[:1]), ("composition", composition, ir),
             ("composition shared", composition, ir[:1]), ("torch.fft", torch_fft, ir))

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
