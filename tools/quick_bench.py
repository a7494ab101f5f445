"""Per-op device timings at the BASELINE config sizes (CUDA events, L2 flushed between iterations).
Development aid; bench.py is the contract benchmark."""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import dasp_pytorch_b200 as D  # noqa: E402

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
from helpers import COMP_RANGES, SR, denorm, eq_ranges  # noqa: E402

PEAK = 3350.0       # GB/s, H100 SXM data-sheet HBM3 bandwidth


def timeit(fn, iters=10, warmup=3, flush=None):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        if flush is not None:
            flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ops", default="dist,gain,comp,eq,reverb")
    ap.add_argument("--bs", type=int, default=0)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    torch.manual_seed(0)
    out = {}

    def report(name, bs, chs, n, f_ms, fb_ms):
        e = bs * chs * n
        b_ms = fb_ms - f_ms
        out[name] = dict(shape=[bs, chs, n], fwd_ms=f_ms, fwdbwd_ms=fb_ms,
                         fwd_frac=8 * e / (f_ms * 1e-3) / 1e9 / PEAK, bwd_frac=12 * e / (max(b_ms, 1e-6) * 1e-3) / 1e9 / PEAK,
                         fwdbwd_frac=20 * e / (fb_ms * 1e-3) / 1e9 / PEAK, gsamples_per_s=e / (fb_ms * 1e-3) / 1e9)
        print(name, json.dumps(out[name]), flush=True)

    def run(name, bs, chs, n, make):
        x = (torch.rand(bs, chs, n, device=dev) * 2 - 1).requires_grad_(True)
        fn = make(x)
        with torch.no_grad():
            f_ms = timeit(lambda: fn(x.detach()), flush=flush)
        gy = torch.rand(bs, chs, n, device=dev)

        def fb():
            y = fn(x)
            y.backward(gy)
            x.grad = None
        fb_ms = timeit(fb, flush=flush)
        report(name, bs, chs, n, f_ms, fb_ms)

    ops = args.ops.split(",")
    if "dist" in ops:
        bs = args.bs or 1024
        d = (torch.rand(bs * 2, device=dev) * 24).requires_grad_(True)
        run("distortion", bs, 2, 48000, lambda x: (lambda xx: D.distortion(xx, SR, d)))
    if "gain" in ops:
        bs = args.bs or 1024
        d = (torch.rand(bs, device=dev) * 24).requires_grad_(True)
        run("gain", bs, 2, 48000, lambda x: (lambda xx: D.gain(xx, SR, d)))
    if "comp" in ops:
        for bs in ([args.bs] if args.bs else [512, 1024]):
            p = [q.to(dev).requires_grad_(True) for q in denorm(torch.rand(bs, 6).clamp(min=0.05), COMP_RANGES)]
            run(f"compressor_bs{bs}", bs, 2, 48000, lambda x: (lambda xx: D.compressor(xx, SR, *p)))
    if "eq" in ops:
        for bs in ([args.bs] if args.bs else [256, 1024]):
            p = [q.to(dev).requires_grad_(True) for q in denorm(torch.rand(bs, 18), eq_ranges())]
            run(f"parametric_eq_bs{bs}", bs, 2, 48000, lambda x: (lambda xx: D.parametric_eq(xx, SR, *p)))
    if "reverb" in ops:
        # BASELINE config 4: 256 x 2 x 48000, IR 96000, 1023 taps, device noise.  Algorithmic bytes (DESIGN.md 4.4):
        # fwd 2*2N*4 + 2*2Leff*4, bwd 3*2N*4 + 2Leff*4 + 2*2Leff*4 + 2*12*Leff*4 per item (Leff = min(L, N))
        bs, n, L = (args.bs or 256), 48000, 96000
        leff = min(L, n)
        p = [torch.rand(bs, device=dev).requires_grad_(True) for _ in range(25)]
        x = (torch.rand(bs, 2, n, device=dev) * 2 - 1).requires_grad_(True)
        fn = lambda xx: D.noise_shaped_reverberation(xx, SR, *p, num_samples=L, num_bandpass_taps=1023)
        with torch.no_grad():
            f_ms = timeit(lambda: fn(x.detach()), flush=flush)
        gy = torch.rand(bs, 2, n, device=dev)

        def fb():
            fn(x).backward(gy)
            x.grad = None
        fb_ms = timeit(fb, flush=flush)
        fwd_b = bs * (2 * 2 * n * 4 + 2 * 2 * leff * 4)
        bwd_b = bs * (3 * 2 * n * 4 + 2 * leff * 4 + 2 * 2 * leff * 4 + 2 * 12 * leff * 4)
        out["reverb_bs%d" % bs] = dict(shape=[bs, 2, n], ir=L, fwd_ms=f_ms, fwdbwd_ms=fb_ms,
                                       fwd_frac=fwd_b / (f_ms * 1e-3) / 1e9 / PEAK,
                                       bwd_frac=bwd_b / ((fb_ms - f_ms) * 1e-3) / 1e9 / PEAK,
                                       gsamples_per_s=bs * 2 * n / (fb_ms * 1e-3) / 1e9)
        print("reverb_bs%d" % bs, json.dumps(out["reverb_bs%d" % bs]), flush=True)
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
