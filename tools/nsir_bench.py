"""Time noise_shaped_impulse_response on one GPU, next to the same IR built in torch, and its composition with
convolution_reverberation next to noise_shaped_reverberation.

    python tools/nsir_bench.py [--batch 1024] [--torch-batch 64] [--steps 10] [--warmup 2] [--out FILE.json]

* IR op at L = 65536 and 96000 (1023 taps, device noise): forward alone, forward + backward (loss sum(w IR), gradients
  to the 24 parameters) and the peak memory of each, at --batch items.
* The reference's synthesis in torch on the same GPU (functional.py:547-567: randn, grouped conv1d with the 12 FIRs,
  envelope, band mean), forward only, at --torch-batch items and scaled to --batch (the scale is printed): its
  activations do not fit at 1024 items.
* At --batch x 2 x 48000 with L = 48000: IR op + convolution_reverberation against noise_shaped_reverberation, forward
  and forward + backward (gradients to x and the 25 parameters): what handing the IR through HBM costs.

Prints the card, its power limit and its maximum SM clock (read-only nvidia-smi query): they belong beside every number
it produces.  Development aid; bench.py is the benchmark."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import dasp_pytorch_b200 as D  # noqa: E402
import oracle  # noqa: E402

SR, TAPS = 44100, 1023


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
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps, (torch.cuda.max_memory_allocated() - base) / 2**30


def torch_ir(params, L, fb):
    """the reference's IR synthesis in torch (fp32, GPU): randn, grouped conv1d with the 12 FIRs, envelope, mean"""
    bs = params.shape[0]
    noise = torch.randn(bs * 2, 12, L + TAPS - 1, device=params.device)
    f = torch.nn.functional.conv1d(noise, fb.unsqueeze(1), groups=12)                 # (bs*2, 12, L)
    f = f.reshape(bs, 2, 12, L)
    t = torch.linspace(0, 1, L, device=params.device)
    env = torch.exp(-(params[:, 12:].reshape(bs, 1, 12, 1) * 10.0 + 1.0) * t)
    return (f * env * params[:, :12].reshape(bs, 1, 12, 1)).mean(2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--torch-batch", type=int, default=64)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", help="also write the results as JSON to this file")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    name, limit, clock = card(dev)
    print(f"card: {name}, power limit: {limit} W, max SM clock: {clock} MHz", flush=True)
    bs = args.batch
    g = torch.Generator(device=dev).manual_seed(0)
    rows = []

    def report(what, ms, gib, extra=""):
        rows.append({"case": what, "ms": round(ms, 3), "peak_gib": round(gib, 2)})
        print(f"{what:58s} {ms:9.2f} ms  peak {gib:6.2f} GiB {extra}", flush=True)

    p = torch.rand(bs, 24, device=dev, generator=g)
    for L in (65536, 96000):
        w = torch.rand(bs, 2, L, device=dev, generator=g)

        def fwd():
            with torch.no_grad():
                D.noise_shaped_impulse_response_packed(SR, p, num_samples=L)

        def fwd_bwd():
            pp = p.detach().requires_grad_(True)
            ir = D.noise_shaped_impulse_response_packed(SR, pp, num_samples=L)
            torch.autograd.grad((ir * w).sum(), pp)

        report(f"IR op, {bs} items, L {L}: fwd", *time_ms(fwd, args.steps, args.warmup))
        report(f"IR op, {bs} items, L {L}: fwd+bwd", *time_ms(fwd_bwd, args.steps, args.warmup))
        del w
        torch.cuda.empty_cache()

        tb = args.torch_batch
        fb = oracle.octave_filterbank(TAPS, SR).to(dev, torch.float32)
        pt = p[:tb]

        def torch_fwd():
            with torch.no_grad():
                torch_ir(pt, L, fb)

        ms, gib = time_ms(torch_fwd, max(1, args.steps // 5), 1)
        report(f"torch conv1d IR, L {L}: fwd, {tb} items x {bs / tb:g}", ms * bs / tb, gib,
               f"(measured {ms:.2f} ms at {tb} items)")
        torch.cuda.empty_cache()

    n = L = 48000
    x = torch.rand(bs, 2, n, device=dev, generator=g) * 2 - 1
    w = torch.rand(bs, 2, n, device=dev, generator=g)
    p25 = torch.rand(bs, 25, device=dev, generator=g)

    def composed(grad):
        xx = x.detach().requires_grad_(grad)
        pp = p25.detach().requires_grad_(grad)
        ir = D.noise_shaped_impulse_response_packed(SR, pp[:, :24], num_samples=L)
        y = D.convolution_reverberation(xx, SR, ir, pp[:, 24])
        if grad:
            torch.autograd.grad((y * w).sum(), (xx, pp))

    def reverb(grad):
        xx = x.detach().requires_grad_(grad)
        pp = p25.detach().requires_grad_(grad)
        y = D.functional.noise_shaped_reverberation_packed(xx, SR, pp, num_samples=L)
        if grad:
            torch.autograd.grad((y * w).sum(), (xx, pp))

    for grad in (False, True):
        mode = "fwd+bwd" if grad else "fwd"
        with torch.set_grad_enabled(grad):
            for _ in range(2):                        # alternate the two, twice
                report(f"IR op + convolution_reverberation, {bs}x2x{n}, L {L}: {mode}",
                       *time_ms(lambda: composed(grad), args.steps, args.warmup))
                report(f"noise_shaped_reverberation, {bs}x2x{n}, L {L}: {mode}",
                       *time_ms(lambda: reverb(grad), args.steps, args.warmup))
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"card": name, "power_limit_w": limit, "max_sm_clock_mhz": clock, "batch": bs,
                       "steps": args.steps, "results": rows}, f, indent=1)


if __name__ == "__main__":
    main()
