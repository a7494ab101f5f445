"""Where the reverb forward's time goes when its IR synthesis overlaps the audio convolution.

    python tools/reverb_overlap.py OUT_DIR [--batch 1024] [--steps 3] [--warmup 3] [--baseline OTHER_OUT_DIR/overlap.json]

Traces bench.py's chain step (eq -> compressor -> reverb -> distortion, fwd + bwd) under torch.profiler (CUDA
activities), once run eagerly and once as replays of the captured step, and reports per reverb forward call:
  * span: first kernel's start to the last ifft_mix_kernel's end, against the sum of the call's kernel times;
  * overlap: convolution kernel time (x_fft_kernel, partition_mac_kernel, ifft_mix_kernel) that ran while a synthesis
    kernel was running;
  * a work-conserving lower bound on the span: the synthesis's SM time on the SMs its clusters hold plus the
    convolution's SM time at the full-GPU rate, over the device's SMs;
  * idle SM time under chunk 0's synthesis (on the SMs outside its clusters) and after the last synthesis ends;
  * each synthesis launch's duration.  The profiler sees kernels, not clusters: a cluster slot lost to a convolution CTA
    shows up as a longer synthesis.  --baseline puts the durations of an earlier run (e.g. the serial forward) beside.

The bound and the idle times need the rates of the kernels when each runs alone: the tool also traces forwards without
a backward (no saved buffers: synthesis and convolution run in turn on one stream) on the same geometry.  A kernel's
SM time is its CTAs times that run's SM time per CTA of the kernel (duration x SMs / CTAs); idle time in an interval is
the SMs free in it times its length, less the SM time of the convolution CTAs that ran in it (a kernel that straddles
an edge counts pro rata).  It is an estimate from the trace: it can go below zero when convolution CTAs take cluster
slots.  Writes OUT_DIR/overlap.json and OUT_DIR/overlap.md and prints the card name and power limit it ran on.
Development aid; bench.py is the benchmark."""
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
CLUSTER = "ir_synth_cluster_kernel"                                     # one CTA per SM: its grid is the SMs it holds
CONV = ("x_fft_kernel", "partition_mac_kernel", "ifft_mix_kernel")


def short_name(name):
    short = name.replace("(anonymous namespace)::", "").removeprefix("void ")
    return short.split("(")[0].split("<")[0].split("::")[-1].strip() or name


def kernels(prof, path):
    """(name, start us, end us, CTAs) of every CUDA kernel in the trace, by start (from the exported trace, which
    carries the grids)"""
    prof.export_chrome_trace(path)
    with open(path) as fh:
        events = json.load(fh)["traceEvents"]
    out = []
    for e in events:
        if e.get("cat") != "kernel":
            continue
        gx, gy, gz = e.get("args", {}).get("grid", [1, 1, 1])
        out.append((short_name(e["name"]), float(e["ts"]), float(e["ts"]) + float(e["dur"]), gx * gy * gz))
    return sorted(out, key=lambda k: k[1])


def forward_calls(ks):
    """the reverb forward calls in the trace: each a maximal run of synthesis and convolution kernels (the chain runs
    no other kernel between a forward's first and last)"""
    calls, cur = [], []
    for k in ks:
        if k[0] in SYNTH or k[0] in CONV:
            cur.append(k)
        elif cur:
            calls.append(cur)
            cur = []
    if cur:
        calls.append(cur)
    return [c for c in calls if any(k[0] == "ifft_mix_kernel" for k in c) and any(k[0] in SYNTH for k in c)]


def overlap(a0, a1, ivs):
    """length of [a0, a1) covered by the union of the intervals ivs (sorted by start)"""
    cov, reach = 0.0, a0
    for b0, b1 in ivs:
        lo, hi = max(b0, reach), min(b1, a1)
        if hi > lo:
            cov += hi - lo
            reach = hi
    return cov


def cta_rates(calls, sms):
    """SM us per CTA of each convolution kernel, from calls whose kernels ran one at a time"""
    tot = {}
    for call in calls:
        for n, s, e, ctas in call:
            if n in CONV:
                t = tot.setdefault(n, [0.0, 0])
                t[0] += (e - s) * sms
                t[1] += ctas
    return {n: us / ctas for n, (us, ctas) in tot.items()}


def conv_work_in(conv, rates, a0, a1):
    """SM us of the convolution kernels' CTAs that ran in [a0, a1), each kernel pro rata to its time inside"""
    w = 0.0
    for n, s, e, ctas in conv:
        inside = max(0.0, min(e, a1) - max(s, a0))
        if inside > 0:
            w += ctas * rates[n] * inside / (e - s)
    return w


def summarise(call, sms, rates, bound_ms):
    synth = [(s, e) for n, s, e, _ in call if n in SYNTH]
    starts = [(s, e) for n, s, e, _ in call if n in CHUNK_START]
    conv = [k for k in call if k[0] in CONV]
    cluster_sms = max([c for n, _, _, c in call if n == CLUSTER], default=0)
    t0 = min(s for _, s, _, _ in call)
    t1 = max(e for n, _, e, _ in conv if n == "ifft_mix_kernel")
    c0s, c0e = starts[0]
    last = max(e for _, e in synth)
    return {
        "span_ms": (t1 - t0) / 1e3,
        "bound_ms": bound_ms,
        "kernel_sum_ms": sum(e - s for _, s, e, _ in call) / 1e3,
        "synth_ms": sum(e - s for s, e in synth) / 1e3,
        "conv_ms": sum(e - s for _, s, e, _ in conv) / 1e3,
        "conv_overlapped_ms": sum(overlap(s, e, synth) for _, s, e, _ in conv) / 1e3,
        "chunks": len(starts),
        "cluster_sms": cluster_sms,
        "chunk0_ms": (c0e - c0s) / 1e3,
        "chunk0_idle_sm_ms": ((sms - cluster_sms) * (c0e - c0s) - conv_work_in(conv, rates, c0s, c0e)) / 1e3,
        "tail_ms": (t1 - last) / 1e3,
        "tail_idle_sm_ms": (sms * (t1 - last) - conv_work_in(conv, rates, last, t1)) / 1e3,
        "synth_launch_ms": [round((e - s) / 1e3, 4) for n, s, e, _ in call if n in SYNTH],
    }


def serial_reference(dev, bs, steps, sms, path):
    """forwards without a backward (synthesis and convolution in turn, every kernel alone on the device): the SM time
    per CTA of each convolution kernel, and the bound from the call's synthesis and convolution kernel times"""
    gen = torch.Generator().manual_seed(1001)
    x = (torch.rand(bs, 2, bench.N_SAMPLES, generator=gen) * 2 - 1).to(dev)
    p = torch.rand(bs, 25, generator=gen).to(dev)
    run = lambda: F.noise_shaped_reverberation_packed(x, bench.SR, p, num_samples=bench.IR_LEN,
                                                      num_bandpass_taps=bench.TAPS)
    with torch.no_grad():
        run()
        torch.cuda.synchronize()
        acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
        with torch.profiler.profile(activities=acts) as prof:
            for _ in range(steps):
                run()
            torch.cuda.synchronize()
    calls = forward_calls(kernels(prof, path))
    rates = cta_rates(calls, sms)
    synth = [sum(e - s for n, s, e, _ in c if n in SYNTH) for c in calls]
    conv = [sum(e - s for n, s, e, _ in c if n in CONV) for c in calls]
    cluster_sms = max([k[3] for c in calls for k in c if k[0] == CLUSTER], default=sms)
    synth_ms, conv_ms = sum(synth) / len(calls) / 1e3, sum(conv) / len(calls) / 1e3
    return rates, {"synth_ms": synth_ms, "conv_ms": conv_ms, "cluster_sms": cluster_sms,
                   "bound_ms": (synth_ms * cluster_sms + conv_ms * sms) / sms}


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
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    os.makedirs(args.out_dir, exist_ok=True)
    trace = lambda tag: os.path.join(args.out_dir, f"overlap_{tag}.pt.trace.json")

    rates, serial = serial_reference(dev, args.batch, args.steps, sms, trace("serial"))
    torch.manual_seed(1000)
    step = bench.Step(D, dev, args.batch, seed=1000)
    for _ in range(args.warmup):
        step.eager()
    step.capture(warm=2)
    for _ in range(args.warmup):
        step.replay()
    torch.cuda.synchronize()
    acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
    result = {"card": name, "power_limit_w": limit, "batch": args.batch, "chunk_items": chunk, "sms": sms,
              "serial": serial, "modes": {}}
    for mode, run in (("eager", step.eager), ("graph", step.replay)):
        with torch.profiler.profile(activities=acts) as prof:
            for _ in range(args.steps):
                run()
            torch.cuda.synchronize()
        calls = [summarise(c, sms, rates, serial["bound_ms"]) for c in forward_calls(kernels(prof, trace(mode)))]
        result["modes"][mode] = calls

    base = None
    if args.baseline:
        with open(args.baseline) as fh:
            base = json.load(fh)
    chunks = {c["chunks"] for calls in result["modes"].values() for c in calls}
    lines = [f"Reverb forward, bench.py's chain at batch {args.batch} (chunks per call: "
             f"{', '.join(map(str, sorted(chunks)))}; chunk_items {chunk}), torch.profiler.  Card: {name}, power limit "
             f"{limit if limit is not None else 'unknown'} W, {sms} SMs.", "",
             f"Serial forward (no backward, same geometry): synthesis {serial['synth_ms']:.3f} ms on "
             f"{serial['cluster_sms']} SMs, convolution {serial['conv_ms']:.3f} ms on {sms}: work-conserving bound "
             f"{serial['bound_ms']:.3f} ms.", "",
             "| mode | call | span ms | bound ms | kernel sum ms | synthesis ms | convolution ms | convolution under "
             "synthesis ms | chunk 0 ms | idle under chunk 0 SM·ms | after last synthesis ms | idle after it SM·ms |",
             "|---|---:|---:|---:|---:|---:|---:|---:|---:|---:|---:|---:|"]
    for mode, calls in result["modes"].items():
        for i, c in enumerate(calls):
            lines.append(f"| {mode} | {i} | {c['span_ms']:.3f} | {c['bound_ms']:.3f} | {c['kernel_sum_ms']:.3f} | "
                         f"{c['synth_ms']:.3f} | {c['conv_ms']:.3f} | {c['conv_overlapped_ms']:.3f} | "
                         f"{c['chunk0_ms']:.3f} | {c['chunk0_idle_sm_ms']:.1f} | {c['tail_ms']:.3f} | "
                         f"{c['tail_idle_sm_ms']:.1f} |")
    lines += ["", "Synthesis launch durations (ms)" + (", this run / baseline" if base else "") + ":"]
    for mode, calls in result["modes"].items():
        for i, c in enumerate(calls):
            row = c["synth_launch_ms"]
            if base and mode in base["modes"] and i < len(base["modes"][mode]):
                ref = base["modes"][mode][i]["synth_launch_ms"]
                row = [f"{a:.3f}/{b:.3f}" for a, b in zip(row, ref)]
            lines.append(f"- {mode} call {i}: {row}")
    text = "\n".join(lines) + "\n"
    with open(os.path.join(args.out_dir, "overlap.json"), "w") as fh:
        json.dump(result, fh, indent=1)
    with open(os.path.join(args.out_dir, "overlap.md"), "w") as fh:
        fh.write(text)
    print(text, flush=True)


if __name__ == "__main__":
    main()
