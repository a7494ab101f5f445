"""Time the compressor with an external side chain (key) against the plain compressor and a torch restatement.

    python tools/sidechain_bench.py [--batch 512] [--chs 2] [--n 48000] [--steps 20] [--warmup 3] [--out FILE.json]

At batch x chs x n with a mono and a stereo key it times, with CUDA events after warm-up, the forward alone, forward +
backward with gradients to x, the key and the five parameters, and forward + backward with a fixed key, for:
  plain      compressor(x, ...): the detector on x itself (no key; the floor);
  sidechain  sidechain_compressor(x, ..., sidechain=key);
  torch      the same arithmetic in torch on the GPU, what a caller writes without the feature: the fp64 test oracle's
             restatement (tests/dyn_sidechain_oracle.py) run in fp32, with its frequency-sampling smoother.
The backward is driven with torch.autograd.grad and a fixed cotangent, so no loss kernels are timed.  For the two
kernel paths it also records the time of each C-ABI call (forward, backward) and its algorithmic HBM bytes:
(2C + K) * 4 B per frame forward, (3C + 2K) * 4 backward, (3C + K) * 4 with a fixed key (C = chs, K = key channels;
the plain compressor is the K = 0, x-as-key case: 2C forward, 3C backward), as a fraction of the 3.35 TB/s data-sheet
bandwidth of the H100 SXM.  Prints the card name and power limit it ran on: both belong beside any number it produces.
Development aid; bench.py is the benchmark."""
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
import dyn_sidechain_oracle as sco  # noqa: E402

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
    gy = torch.randn(bs, C, n, device=dev, generator=g)
    u = torch.rand(bs, 6, device=dev, generator=g)
    params = [-60 + 60 * u[:, 0], 1 + 19 * u[:, 1], 5 + 95 * u[:, 2], 5 + 95 * u[:, 3], 12 * u[:, 4], 12 * u[:, 5]]
    rows = []
    for K in (1, 2):
        key = (torch.rand(bs, K, n, device=dev, generator=g) * 2 - 1) * 0.5
        impls = [("sidechain", lambda xx, kk, pp: D.sidechain_compressor(xx, SR, *pp, sidechain=kk)),
                 ("torch", lambda xx, kk, pp: sco.compressor(xx, SR, *pp, sidechain=kk))]
        if K == 1:
            impls.insert(0, ("plain", lambda xx, kk, pp: D.compressor(xx, SR, *pp)))
        for impl, fn in impls:
            def fwd():
                with torch.no_grad():
                    fn(x, key, params)

            def fwd_bwd(key_grad):
                xx = x.detach().requires_grad_(True)
                kk = key.detach().requires_grad_(key_grad)
                pp = [p.detach().requires_grad_(True) for p in params]
                y = fn(xx, kk, pp)
                leaves = [xx] + ([kk] if key_grad and impl != "plain" else []) + pp[:3] + pp[4:]
                torch.autograd.grad(y, leaves, grad_outputs=gy)

            modes = [("fwd", fwd), ("fwd+bwd", lambda: fwd_bwd(True))]
            if impl != "plain":
                modes.append(("fwd+bwd, fixed key", lambda: fwd_bwd(False)))
            for mode, call in modes:
                torch.cuda.synchronize()
                ms = time_ms(call, args.steps, args.warmup)
                row = {"K": K, "impl": impl, "mode": mode, "ms": round(ms, 4)}
                line = f"{bs} x {C} x {n}, key {K}: {impl:9s} {mode:18s} {ms:8.3f} ms"
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
                    kk = 0 if impl == "plain" else K
                    fixed = mode.endswith("fixed key")
                    bpf = {"fwd": (2 * C + kk) * 4, "bwd": (3 * C + (kk if fixed else 2 * kk)) * 4}
                    for stage, ts in sorted(per.items()):
                        d = "bwd" if stage.endswith("bwd") else "fwd"
                        t = sum(ts) / len(ts)
                        frac = bpf[d] * bs * n / (t * 1e-3) / HBM_BPS
                        row[stage] = {"ms": round(t, 4), "bytes": bpf[d] * bs * n, "hbm_fraction": round(frac, 3)}
                        line += f"  {stage} {t:.3f} ms ({frac:.2f} of 3.35 TB/s)"
                rows.append(row)
                print(line, flush=True)
        del key
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"card": name, "power_limit_w": limit, "batch": bs, "chs": C, "n": n, "steps": args.steps,
                       "results": rows}, f, indent=1)


if __name__ == "__main__":
    main()
