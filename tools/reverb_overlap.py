"""Where the reverb forward's time goes when the IR synthesis of chunk k + 1 overlaps the convolution of chunk k.

    python tools/reverb_overlap.py OUT_DIR [--batch 1024] [--steps 3] [--warmup 3] [--baseline OTHER_OUT_DIR/overlap.json]

Traces bench.py's chain step (eq -> compressor -> reverb -> distortion, fwd + bwd) under torch.profiler (CUDA
activities), once run eagerly and once as replays of the captured step, and reports per reverb forward call:
  * span: first synthesis kernel's start to the last ifft_mix_kernel's end, against the sum of the call's kernel times;
  * overlap: convolution kernel time (x_fft_kernel, partition_mac_kernel, ifft_mix_kernel) that ran while a synthesis
    kernel was running;
  * each synthesis launch's duration.  The profiler sees kernels, not clusters: a cluster slot lost to a convolution CTA
    shows up as a longer synthesis.  --baseline puts the durations of an earlier run (e.g. the serial forward) beside.
Writes OUT_DIR/overlap.json and OUT_DIR/overlap.md and prints the card name and power limit it ran on.  Development aid;
bench.py is the benchmark."""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import bench  # noqa: E402
import dasp_pytorch_b200 as D  # noqa: E402
from dasp_pytorch_b200 import functional as F  # noqa: E402
from profile_step import card  # noqa: E402

SYNTH = ("ir_synth_cluster_kernel", "spectral_gen_kernel", "ifft_shape_kernel")
CHUNK_START = ("ir_synth_cluster_kernel", "spectral_gen_kernel")       # one launch per chunk on either path
CONV = ("x_fft_kernel", "partition_mac_kernel", "ifft_mix_kernel")


def short_name(name):
    short = name.replace("(anonymous namespace)::", "").removeprefix("void ")
    return short.split("(")[0].split("<")[0].split("::")[-1].strip() or name


def kernels(prof):
    """(name, start us, end us) of every CUDA kernel in the trace, by start"""
    out = []
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        out.append((short_name(e.name), e.time_range.start, e.time_range.end))
    return sorted(out, key=lambda k: k[1])


def forward_calls(ks, chunks):
    """the reverb forward calls in the trace: from a chunk's first synthesis launch until `chunks` ifft_mix_kernels"""
    calls, cur, mixes = [], None, 0
    for k in ks:
        if cur is None:
            if k[0] in CHUNK_START:
                cur, mixes = [], 0
            else:
                continue
        if k[0] in SYNTH or k[0] in CONV:
            cur.append(k)
        if k[0] == "ifft_mix_kernel":
            mixes += 1
            if mixes == chunks:
                calls.append(cur)
                cur = None
    return calls


def overlap(a0, a1, ivs):
    """length of [a0, a1) covered by the union of the intervals ivs (sorted by start)"""
    cov, reach = 0.0, a0
    for b0, b1 in ivs:
        lo, hi = max(b0, reach), min(b1, a1)
        if hi > lo:
            cov += hi - lo
            reach = hi
    return cov


def summarise(call):
    synth = [(s, e) for n, s, e in call if n in SYNTH]
    conv = [(n, s, e) for n, s, e in call if n in CONV]
    t0 = min(s for s, _ in synth)
    t1 = max(e for n, _, e in conv if n == "ifft_mix_kernel")
    return {
        "span_ms": (t1 - t0) / 1e3,
        "kernel_sum_ms": sum(e - s for _, s, e in call) / 1e3,
        "synth_ms": sum(e - s for s, e in synth) / 1e3,
        "conv_ms": sum(e - s for _, s, e in conv) / 1e3,
        "conv_overlapped_ms": sum(overlap(s, e, synth) for _, s, e in conv) / 1e3,
        "synth_launch_ms": [round((e - s) / 1e3, 4) for n, s, e in call if n in SYNTH],
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--batch", type=int, default=bench.GLOBAL_BATCH)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--baseline", help="overlap.json of an earlier run, for the synthesis launch durations")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    name, limit = card(dev)
    print(f"card: {name}, power limit: {limit if limit is not None else 'unknown'} W", flush=True)
    chunk = F.reverb_chunk_items(dev)
    chunks = (args.batch + chunk - 1) // chunk

    torch.manual_seed(1000)
    step = bench.Step(D, dev, args.batch, seed=1000)
    for _ in range(args.warmup):
        step.eager()
    step.capture(warm=2)
    for _ in range(args.warmup):
        step.replay()
    torch.cuda.synchronize()
    acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
    result = {"card": name, "power_limit_w": limit, "batch": args.batch, "chunk_items": chunk, "modes": {}}
    for mode, run in (("eager", step.eager), ("graph", step.replay)):
        with torch.profiler.profile(activities=acts) as prof:
            for _ in range(args.steps):
                run()
            torch.cuda.synchronize()
        calls = [summarise(c) for c in forward_calls(kernels(prof), chunks)]
        result["modes"][mode] = calls

    base = None
    if args.baseline:
        with open(args.baseline) as fh:
            base = json.load(fh)
    lines = [f"Reverb forward, bench.py's chain at batch {args.batch} ({chunks} chunks of {chunk} items), "
             f"torch.profiler.  Card: {name}, power limit {limit if limit is not None else 'unknown'} W.", "",
             "| mode | call | span ms | kernel sum ms | synthesis ms | convolution ms | convolution under synthesis ms |",
             "|---|---:|---:|---:|---:|---:|---:|"]
    for mode, calls in result["modes"].items():
        for i, c in enumerate(calls):
            lines.append(f"| {mode} | {i} | {c['span_ms']:.3f} | {c['kernel_sum_ms']:.3f} | {c['synth_ms']:.3f} | "
                         f"{c['conv_ms']:.3f} | {c['conv_overlapped_ms']:.3f} |")
    lines += ["", "Synthesis launch durations (ms)" + (", this run / baseline" if base else "") + ":"]
    for mode, calls in result["modes"].items():
        for i, c in enumerate(calls):
            row = c["synth_launch_ms"]
            if base and mode in base["modes"] and i < len(base["modes"][mode]):
                ref = base["modes"][mode][i]["synth_launch_ms"]
                row = [f"{a:.3f}/{b:.3f}" for a, b in zip(row, ref)]
            lines.append(f"- {mode} call {i}: {row}")
    text = "\n".join(lines) + "\n"
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, "overlap.json"), "w") as fh:
        json.dump(result, fh, indent=1)
    with open(os.path.join(args.out_dir, "overlap.md"), "w") as fh:
        fh.write(text)
    print(text, flush=True)


if __name__ == "__main__":
    main()
