"""Time parametric_eq_frequency_response on one GPU next to the two ways of getting the EQ's response without it.

    python tools/eq_response_bench.py [--batch 1024] [--steps 20] [--warmup 3] [--out FILE.json]

Workloads, at --batch items drawn over the ParametricEQ ranges (44.1 kHz): the rfftfreq grid of n_fft = 131072 (65537
bins, the reference's grid for 48000-sample audio), that of n_fft = 8192, and a 512-point log grid from 10 Hz to sr/2.
Each is timed forward alone and forward + backward (loss sum(w * view_as_real(H)), gradients to the (bs, 18)
parameters), against
  (a) the reference's fft_sosfreqz restated in torch: fp32 rfft of each section's b and a, divided and multiplied,
      with autograd (the sections designed with torch ops from the same parameters); on the log grid it is read off
      the n_fft = 131072 grid, which is what that route can do;
  (b) the impulse route: a unit impulse through this package's parametric_eq at 65536 samples, then torch.fft.rfft
      (one grid only; timed once and listed under every workload).
Also prints the bytes-based floor of the forward: 8 bytes written per (item, bin) at the data sheet's 3.35 TB/s
(H100 SXM HBM3), computed, not measured, and each time's share of it.

Prints the card, its power limit and its maximum SM clock (read-only nvidia-smi query): they belong beside every number
it produces.  Development aid; bench.py is the benchmark."""
import argparse
import json
import math
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import dasp_pytorch_b200 as D  # noqa: E402

SR = 44100
HBM_BPS = 3.35e12


def card(dev):
    name, limit, clock = torch.cuda.get_device_name(dev), None, None
    try:
        out = subprocess.run(["nvidia-smi", f"--id={dev.index or 0}", "--query-gpu=power.limit,clocks.max.sm",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout
        a, b = out.strip().splitlines()[0].split(",")
        limit, clock = float(a), float(b)
    except Exception:
        pass
    return name, limit, clock


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


def sections(sr, p):
    """(bs, 6, 6) RBJ sections [b0 b1 b2 1 a1 a2] from the (bs, 18) parameters, with torch ops (fp32, autograd)"""
    rows = []
    for k in range(6):
        g, fc, q = p[:, 3 * k], p[:, 3 * k + 1], p[:, 3 * k + 2]
        A = torch.pow(10.0, g / 40.0)
        w0 = 2 * math.pi * fc / sr
        alpha = torch.sin(w0) / (2 * q)
        cw = torch.cos(w0)
        if k in (1, 2, 3, 4):
            b = (1 + alpha * A, -2 * cw, 1 - alpha * A)
            a = (1 + alpha / A, -2 * cw, 1 - alpha / A)
        else:
            s = 1.0 if k == 0 else -1.0
            r = 2 * torch.sqrt(A) * alpha
            b = (A * ((A + 1) - s * (A - 1) * cw + r), s * 2 * A * ((A - 1) - s * (A + 1) * cw),
                 A * ((A + 1) - s * (A - 1) * cw - r))
            a = ((A + 1) + s * (A - 1) * cw + r, -s * 2 * ((A - 1) + s * (A + 1) * cw),
                 (A + 1) + s * (A - 1) * cw - r)
        rows.append(torch.stack([t / a[0] for t in (*b, *a)], -1))
    return torch.stack(rows, 1)


def fft_sosfreqz(sos, n_fft):
    """the reference's signal.fft_sosfreqz (signal.py:14-32) in torch"""
    h = None
    for k in range(sos.shape[1]):
        hk = torch.fft.rfft(sos[:, k, :3], n_fft) / torch.fft.rfft(sos[:, k, 3:], n_fft)
        h = hk if h is None else h * hk
    return h


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", help="also write the results as JSON to this file")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    name, limit, clock = card(dev)
    print(f"card: {name}, power limit: {limit} W, max SM clock: {clock} MHz", flush=True)
    bs = args.batch
    g = torch.Generator(device=dev).manual_seed(0)
    lo = torch.tensor([r[0] for r in D.ParametricEQ(SR).param_ranges.values()], device=dev)
    hi = torch.tensor([r[1] for r in D.ParametricEQ(SR).param_ranges.values()], device=dev)
    p = lo + (hi - lo) * torch.rand(bs, 18, device=dev, generator=g)
    rows = []

    def report(what, ms, floor_ms=None):
        share = f"  floor {floor_ms:.3f} ms = {100 * floor_ms / ms:5.1f} % of this" if floor_ms else ""
        rows.append({"case": what, "ms": round(ms, 4), "floor_ms": None if floor_ms is None else round(floor_ms, 4)})
        print(f"{what:64s} {ms:9.3f} ms{share}", flush=True)

    # (b) the impulse route, one grid: rfft of parametric_eq(unit impulse, 65536)
    n_imp = 65536
    x = torch.zeros(bs, 1, n_imp, device=dev)
    x[:, :, 0] = 1.0

    def impulse(grad):
        pp = p.detach().requires_grad_(grad)
        h = torch.fft.rfft(D.functional.parametric_eq_packed(x, SR, pp)[:, 0])
        if grad:
            torch.autograd.grad(torch.view_as_real(h).sum(), pp)

    imp = {}
    for grad in (False, True):
        with torch.set_grad_enabled(grad):
            imp[grad] = time_ms(lambda: impulse(grad), args.steps, args.warmup)
    del x
    torch.cuda.empty_cache()

    grids = {"rfft n_fft 131072 (65537 bins)": (torch.fft.rfftfreq(131072, 1 / SR, dtype=torch.float64), 131072),
             "rfft n_fft 8192 (4097 bins)": (torch.fft.rfftfreq(8192, 1 / SR, dtype=torch.float64), 8192),
             "log grid 10 Hz..sr/2 (512 points)": (torch.logspace(1, math.log10(SR / 2), 512, dtype=torch.float64),
                                                   131072)}
    for gname, (f, n_ref) in grids.items():
        f = f.to(dev)
        nf = f.numel()
        w = torch.rand(bs, nf, 2, device=dev, generator=g)
        floor = bs * nf * 8 / HBM_BPS * 1e3
        pick = None
        if nf != n_ref // 2 + 1:        # the reference's route reads a log grid off its rfft grid (nearest bin)
            pick = torch.round(f * n_ref / SR).long()

        def op(grad):
            pp = p.detach().requires_grad_(grad)
            h = D.parametric_eq_frequency_response_packed(SR, pp, f)
            if grad:
                torch.autograd.grad((torch.view_as_real(h) * w).sum(), pp)

        def ref(grad):
            pp = p.detach().requires_grad_(grad)
            h = fft_sosfreqz(sections(SR, pp), n_ref)
            if pick is not None:
                h = h[:, pick]
            if grad:
                torch.autograd.grad((torch.view_as_real(h) * w).sum(), pp)

        for grad in (False, True):
            mode = "fwd+bwd" if grad else "fwd"
            with torch.set_grad_enabled(grad):
                report(f"op, {gname}: {mode}", time_ms(lambda: op(grad), args.steps, args.warmup),
                       floor if not grad else None)
                report(f"(a) torch fft_sosfreqz, {gname}: {mode}", time_ms(lambda: ref(grad), args.steps,
                                                                            args.warmup))
                report(f"(b) impulse through parametric_eq + rfft (65536): {mode}", imp[grad])
        del w
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as fh:
            json.dump({"card": name, "power_limit_w": limit, "max_sm_clock_mhz": clock, "batch": bs,
                       "steps": args.steps, "results": rows}, fh, indent=1)


if __name__ == "__main__":
    main()
