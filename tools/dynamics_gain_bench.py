"""Time compressor_gain (linear and dB) against the compressor and a torch restatement.

    python tools/dynamics_gain_bench.py [--batch 512] [--chs 2] [--n 48000] [--steps 20] [--warmup 3] [--out FILE.json]

At batch x chs x n it times, with CUDA events after warm-up, the forward alone and forward + backward with gradients to
x and the five parameters, for:
  gain       compressor_gain(x, ...): the gain curve G (bs, 1, n);
  gain-db    compressor_gain(x, ..., db=True): the same curve in dB;
  compressor compressor(x, ...) on the same x, which computes the same G and multiplies it into x;
  torch      G in torch on the GPU, what a caller writes without the op: the fp64 test oracle's restatement
             (tests/dyn_gain_oracle.py) run in fp32, with its frequency-sampling smoother.
The backward is driven with torch.autograd.grad and a fixed cotangent, so no loss kernels are timed.  For the kernel
paths it also records the time of each C-ABI call and its algorithmic HBM bytes as a fraction of the 3.35 TB/s
data-sheet bandwidth of the H100 SXM: the gain op reads C and writes 1 float per frame forward, reads C + 1 and writes 1
backward; the compressor moves 2C forward and 3C backward.  Prints the card name and power limit it ran on: both belong
beside any number it produces.  Development aid; bench.py is the benchmark."""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import dasp_pytorch_b200 as D  # noqa: E402
from dasp_pytorch_b200 import functional as F  # noqa: E402
from conv_bench import time_ms  # noqa: E402
from profile_step import card  # noqa: E402
import dyn_gain_oracle as go  # noqa: E402

HBM_BPS = 3.35e12
SR = 44100


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--chs", type=int, default=2)
    ap.add_argument("--n", type=int, default=48000)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", help="also write the results as JSON to this file")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    name, limit = card(dev)
    print(f"card: {name}, power limit: {limit if limit is not None else 'unknown'} W", flush=True)
    bs, C, n = args.batch, args.chs, args.n
    g = torch.Generator(device=dev).manual_seed(0)
    x = (torch.rand(bs, C, n, device=dev, generator=g) * 2 - 1) * 0.5
    u = torch.rand(bs, 6, device=dev, generator=g)
    params = [-60 + 60 * u[:, 0], 1 + 19 * u[:, 1], 5 + 95 * u[:, 2], 5 + 95 * u[:, 3], 12 * u[:, 4], 12 * u[:, 5]]
    impls = [("gain", lambda xx, pp: D.compressor_gain(xx, SR, *pp)),
             ("gain-db", lambda xx, pp: D.compressor_gain(xx, SR, *pp, db=True)),
             ("compressor", lambda xx, pp: D.compressor(xx, SR, *pp)),
             ("torch", lambda xx, pp: go.compressor_gain(xx, SR, *pp))]
    # algorithmic bytes per frame of each C-ABI call
    bpf = {"dyn_gain_fwd": (C + 1) * 4, "dyn_gain_bwd": (C + 2) * 4, "comp_fwd": 2 * C * 4, "comp_bwd": 3 * C * 4}
    rows = []
    for impl, fn in impls:
        gy = torch.randn((bs, C, n) if impl == "compressor" else (bs, 1, n), device=dev, generator=g)

        def fwd():
            with torch.no_grad():
                fn(x, params)

        def fwd_bwd():
            xx = x.detach().requires_grad_(True)
            pp = [p.detach().requires_grad_(True) for p in params]
            y = fn(xx, pp)
            torch.autograd.grad(y, [xx] + pp[:3] + pp[4:], grad_outputs=gy)

        for mode, call in (("fwd", fwd), ("fwd+bwd", fwd_bwd)):
            torch.cuda.synchronize()
            ms = time_ms(call, args.steps, args.warmup)
            row = {"impl": impl, "mode": mode, "ms": round(ms, 4)}
            line = f"{bs} x {C} x {n}: {impl:10s} {mode:8s} {ms:8.3f} ms"
            if impl != "torch":
                # per C-ABI call: events around each kernel launch, over a separate set of steps
                F.STAGE_TIMING = []
                for _ in range(args.steps):
                    call()
                torch.cuda.synchronize()
                per = {}
                for stage, a, b in F.STAGE_TIMING:
                    per.setdefault(stage, []).append(a.elapsed_time(b))
                F.STAGE_TIMING = None
                for stage, ts in sorted(per.items()):
                    t = sum(ts) / len(ts)
                    frac = bpf[stage] * bs * n / (t * 1e-3) / HBM_BPS
                    row[stage] = {"ms": round(t, 4), "bytes": bpf[stage] * bs * n, "hbm_fraction": round(frac, 3)}
                    line += f"  {stage} {t:.3f} ms ({frac:.2f} of 3.35 TB/s)"
            rows.append(row)
            print(line, flush=True)
        del gy
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"card": name, "power_limit_w": limit, "batch": bs, "chs": C, "n": n, "steps": args.steps,
                       "results": rows}, f, indent=1)


if __name__ == "__main__":
    main()
