"""Per-kernel device time of bench.py's chain step (eq -> compressor -> reverb -> distortion, fwd + bwd), eager.

    python tools/profile_step.py OUT_DIR [--batch 1024] [--steps 3] [--warmup 3]

Runs a few eager steps of the benchmark's workload under torch.profiler (CUDA activities) and writes OUT_DIR/kernels.md
and OUT_DIR/kernels.json: per kernel the launches, total and per-step device time, and for the reverb's kernels the HBM
bytes per item that the code moves at this geometry (derived from dasp_reverb_geometry, not measured) with the
bandwidth that implies.  Prints the card name and power limit it ran on: both belong beside any number it produces.
Development aid; bench.py is the benchmark."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
import dasp_pytorch_b200 as D  # noqa: E402
from dasp_pytorch_b200 import _abi  # noqa: E402


def card(dev):
    """(name, power limit in W or None) of the device; the limit from a read-only nvidia-smi query"""
    name, limit = torch.cuda.get_device_name(dev), None
    try:
        out = subprocess.run(["nvidia-smi", f"--id={dev.index or 0}", "--query-gpu=power.limit",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout
        limit = float(out.strip().splitlines()[0])
    except Exception:
        pass
    return name, limit


def reverb_bytes_per_item(n, in_chs=2):
    """HBM bytes per stereo item of each reverb kernel at the benchmark's geometry, counted from the code:
    c8 = one complex64 block spectrum slot (2 kB points), a = one audio row of n floats"""
    g = _abi.ReverbGeom()
    _abi.check(_abi.lib().dasp_reverb_geometry(0, n, bench.IR_LEN, bench.TAPS, 1, g), "dasp_reverb_geometry")
    I, J, kB, leff = g.x_blocks, g.ir_partitions, g.conv_block, g.leff
    c8, a, f = 2 * kB * 8, n * 4, 12 * g.rpp * g.nb * 8                 # f: the 12 bands' polyphase spectra
    return {
        "spectral_gen_kernel": f,                                         # generator spectrum written
        "ifft_shape_kernel": 2 * f + leff * 8,                            # spectrum read, f written, IR taps written
        "ir_synth_cluster_kernel": f + leff * 8,                          # f written, IR taps written
        "x_fft_kernel": 2 * in_chs * a + J * kB * 8 + (I + J) * c8,       # windows (each sample twice), taps, spectra
        "partition_mac_kernel": (I + J) * c8 + I * c8,                    # X, H read; Y written
        "ifft_mix_kernel": I * c8 + in_chs * a + 2 * a,                   # Y, x read; y written
        "g_fft_kernel": 2 * a + I * c8,                                   # dL/dy read; G written
        "partition_mac_bwd_kernel": (2 * I + J) * c8 + (I + J) * c8,      # G, H, X read; D, E written
        "ifft_dx_kernel": I * c8 + 2 * a + in_chs * a + in_chs * a,       # D, dL/dy, x read; dL/dx written
        "ifft_irgrad_kernel": J * c8 + 12 * leff * 8,                     # E and the f taps read
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--batch", type=int, default=bench.GLOBAL_BATCH)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    name, limit = card(dev)
    print(f"card: {name}, power limit: {limit if limit is not None else 'unknown'} W", flush=True)

    torch.manual_seed(1000)
    step = bench.Step(D, dev, args.batch, seed=1000)
    for _ in range(args.warmup):
        step.eager()
    torch.cuda.synchronize()
    acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
    with torch.profiler.profile(activities=acts) as prof:
        for _ in range(args.steps):
            step.eager()
        torch.cuda.synchronize()

    rows = {}
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        # "void dasp::(anonymous namespace)::partition_mac_kernel<12, false, true>(...)" -> "partition_mac_kernel"
        short = e.name.replace("(anonymous namespace)::", "").removeprefix("void ")
        key = short.split("(")[0].split("<")[0].split("::")[-1].strip() or e.name
        r = rows.setdefault(key, {"kernel": key, "launches": 0, "us": 0.0})
        r["launches"] += 1
        r["us"] += e.time_range.elapsed_us()
    model = reverb_bytes_per_item(bench.N_SAMPLES)
    total_us = sum(r["us"] for r in rows.values())
    table = sorted(rows.values(), key=lambda r: -r["us"])
    for r in table:
        r["ms_per_step"] = r["us"] / 1e3 / args.steps
        r["share"] = r["us"] / total_us
        if r["kernel"] in model:
            r["mb_per_item"] = model[r["kernel"]] / 1e6
            r["gb_per_s"] = model[r["kernel"]] * args.batch * args.steps / (r["us"] * 1e-6) / 1e9

    os.makedirs(args.out_dir, exist_ok=True)
    head = (f"Per-kernel device time, {args.steps} eager steps of bench.py's chain at batch {args.batch} x 2 x "
            f"{bench.N_SAMPLES} (IR {bench.IR_LEN}, {bench.TAPS} taps), torch.profiler.\n"
            f"Card: {name}, power limit {limit if limit is not None else 'unknown'} W.  "
            f"Sum of kernel time per step: {total_us / 1e3 / args.steps:.2f} ms.\n"
            "MB/item: HBM bytes the reverb kernel moves per stereo item, counted from the code (not measured).\n")
    lines = [head, "| kernel | launches/step | ms/step | share | MB/item | GB/s |", "|---|---:|---:|---:|---:|---:|"]
    for r in table:
        mb = f"{r['mb_per_item']:.2f}" if "mb_per_item" in r else ""
        bw = f"{r['gb_per_s']:.0f}" if "gb_per_s" in r else ""
        lines.append(f"| {r['kernel'][:60]} | {r['launches'] / args.steps:g} | {r['ms_per_step']:.3f} | "
                     f"{100 * r['share']:.1f} % | {mb} | {bw} |")
    text = "\n".join(lines) + "\n"
    with open(os.path.join(args.out_dir, "kernels.md"), "w") as fh:
        fh.write(text)
    with open(os.path.join(args.out_dir, "kernels.json"), "w") as fh:
        json.dump({"card": name, "power_limit_w": limit, "batch": args.batch, "steps": args.steps,
                   "kernels": table}, fh, indent=1)
    print(text, flush=True)


if __name__ == "__main__":
    main()
