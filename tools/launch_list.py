"""What one call of every public op puts on the device, as text that two versions of the package can be diffed on.

For each op, its packed twin and the processors' packed paths, at a small seeded size, with and without gradients
(with: the parameters, the audio and the IR require one, and a backward follows the forward), one warmed-up call is
recorded with torch.profiler: the name and count of every kernel, memcpy and memset on the device, the count of
every CUDA runtime and driver call on the host (launches, copies, synchronisations), and the number and bytes of the
caching allocator's allocations.  Identical output means identical device work.

``--host-out`` also writes the median host time per call (the enqueue, without a synchronise) of the same cases
without the profiler; that file differs run to run.  Development aid: needs a CUDA device.

    python tools/launch_list.py --out launches.txt --host-out host_us.json
"""
import argparse
import json
import os
import statistics
import sys
import time
from collections import Counter

import torch
from torch.autograd import DeviceType
from torch.profiler import ProfilerActivity, profile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import dasp_pytorch_b200 as D  # noqa: E402
from dasp_pytorch_b200 import functional as F  # noqa: E402

SR = 48000
BS, N = 2, 4096


def _t(g, *shape, lo=-1.0, hi=1.0):
    return (torch.rand(*shape, generator=g) * (hi - lo) + lo).cuda()


def _leaf(t, grad):
    return t.detach().requires_grad_(grad)


def _eq_params(g):
    cols = []
    for lo, hi in ((20, 2000), (80, 2000), (2000, 8000), (8000, 12000), (12000, 20000), (4000, 20000)):
        cols += [_t(g, BS, lo=-12, hi=12), _t(g, BS, lo=lo, hi=hi), _t(g, BS, lo=0.5, hi=2.0)]
    return cols


def _dyn_params(g):
    return [_t(g, BS, lo=-30, hi=-10), _t(g, BS, lo=2, hi=8), _t(g, BS, lo=5, hi=20), _t(g, BS, lo=20, hi=80),
            _t(g, BS, lo=1, hi=6), _t(g, BS, lo=0, hi=3)]


def cases():
    """name -> function(grad) that makes the seeded inputs and returns the forward call on them"""
    c = {}

    def setup(grad, *shapes, params=None, packed=False):
        g = torch.Generator().manual_seed(1)
        xs = [_leaf(_t(g, *s), grad) for s in shapes]
        ps = params(g) if params else []
        ps = [_leaf(torch.stack(ps, dim=1), grad)] if packed else [_leaf(p, grad) for p in ps]
        return xs, ps

    rev = lambda g: [_t(g, BS, lo=0, hi=1) for _ in range(25)]                    # noqa: E731
    L, TAPS = 4096, 255

    def pointwise(grad, fn, shape, n_params):
        (x, p), _ = setup(grad, shape, (n_params,))
        return lambda: fn(x, SR, p)
    for name, fn, shape, n_params in (("gain", F.gain, (BS, 2, N), BS),
                                      ("distortion", F.distortion, (BS, 2, N), BS * 2),
                                      ("stereo_widener", F.stereo_widener, (BS, 2, N), BS),
                                      ("stereo_panner", F.stereo_panner, (BS, 3, N), BS * 3),
                                      ("stereo_bus", F.stereo_bus, (BS, 2, 3, N), BS * 3)):
        c[name] = lambda grad, fn=fn, shape=shape, n_params=n_params: pointwise(grad, fn, shape, n_params)

    def eq(grad, packed):
        (x,), ps = setup(grad, (BS, 2, N), params=_eq_params, packed=packed)
        return lambda: (F.parametric_eq_packed if packed else F.parametric_eq)(x, SR, *ps)
    c["parametric_eq"] = lambda grad: eq(grad, False)
    c["parametric_eq_packed"] = lambda grad: eq(grad, True)

    def dyn(grad, kind, packed, key=False, la=0):
        shapes = [(BS, 2, N), (BS, 3, N)] if key else [(BS, 2, N)]
        xs, ps = setup(grad, *shapes, params=_dyn_params, packed=packed)
        kw = {"sidechain": xs[1]} if key else {}
        if packed:
            return lambda: F.dynamics_packed(kind, xs[0], SR, ps[0], 1e-8, la, **kw)
        fn = [[F.compressor, F.expander], [F.sidechain_compressor, F.sidechain_expander]][key][kind]
        return lambda: fn(xs[0], SR, *ps, 1e-8, la, **kw)
    for kind, name in ((0, "compressor"), (1, "expander")):
        c[name] = lambda grad, kind=kind: dyn(grad, kind, False)
        c[f"{name}_lookahead"] = lambda grad, kind=kind: dyn(grad, kind, False, la=64)
        c[f"sidechain_{name}"] = lambda grad, kind=kind: dyn(grad, kind, False, key=True)
        c[f"dynamics_packed_{kind}"] = lambda grad, kind=kind: dyn(grad, kind, True)
        c[f"dynamics_packed_{kind}_sidechain"] = lambda grad, kind=kind: dyn(grad, kind, True, key=True, la=16)

    def dyn_gain(grad, kind, packed, db):
        (x,), ps = setup(grad, (BS, 3, N), params=_dyn_params, packed=packed)
        if packed:
            return lambda: F.dynamics_gain_packed(kind, x, SR, ps[0], db=db)
        return lambda: (F.compressor_gain, F.expander_gain)[kind](x, SR, *ps, db=db)
    for kind, name in ((0, "compressor_gain"), (1, "expander_gain")):
        c[name] = lambda grad, kind=kind: dyn_gain(grad, kind, False, False)
        c[f"{name}_db"] = lambda grad, kind=kind: dyn_gain(grad, kind, False, True)
        c[f"dynamics_gain_packed_{kind}"] = lambda grad, kind=kind: dyn_gain(grad, kind, True, kind == 1)

    def reverb(grad, packed, chs, noise):
        (x,), ps = setup(grad, (BS, chs, N), params=rev, packed=packed)
        kw = dict(num_samples=L, num_bandpass_taps=TAPS)
        if noise:
            kw["noise"] = torch.randn(BS * 2, 12, L + TAPS - 1, generator=torch.Generator().manual_seed(3)).cuda()
        if packed:
            return lambda: F.noise_shaped_reverberation_packed(x, SR, ps[0], **kw)
        return lambda: F.noise_shaped_reverberation(x, SR, *ps, **kw)
    c["noise_shaped_reverberation"] = lambda grad: reverb(grad, False, 2, False)
    c["noise_shaped_reverberation_mono_noise"] = lambda grad: reverb(grad, False, 1, True)
    c["noise_shaped_reverberation_packed"] = lambda grad: reverb(grad, True, 2, False)

    def nsir(grad, packed, noise):
        _, ps = setup(grad, params=lambda g: rev(g)[:24], packed=packed)
        kw = dict(num_samples=L, num_bandpass_taps=TAPS)
        if noise:
            kw["noise"] = torch.randn(BS * 2, 12, L + TAPS - 1, generator=torch.Generator().manual_seed(3)).cuda()
        if packed:
            return lambda: F.noise_shaped_impulse_response_packed(SR, ps[0], **kw)
        return lambda: F.noise_shaped_impulse_response(SR, *ps, **kw)
    c["noise_shaped_impulse_response"] = lambda grad: nsir(grad, False, False)
    c["noise_shaped_impulse_response_noise"] = lambda grad: nsir(grad, False, True)
    c["noise_shaped_impulse_response_packed"] = lambda grad: nsir(grad, True, False)

    def eq_response(grad, packed):
        _, ps = setup(grad, params=_eq_params, packed=packed)
        f = torch.linspace(0, SR / 2, 257, dtype=torch.float64)
        if packed:
            return lambda: F.parametric_eq_frequency_response_packed(SR, ps[0], f)
        return lambda: F.parametric_eq_frequency_response(SR, *ps, f)
    c["parametric_eq_frequency_response"] = lambda grad: eq_response(grad, False)
    c["parametric_eq_frequency_response_packed"] = lambda grad: eq_response(grad, True)

    def conv(grad, x_chs, ir_bs, ir_chs):
        (x, ir, mix), _ = setup(grad, (BS, x_chs, N), (ir_bs, ir_chs, 3000), (BS,))
        return lambda: F.convolution_reverberation(x, SR, ir, mix)
    c["convolution_reverberation"] = lambda grad: conv(grad, 2, BS, 2)
    c["convolution_reverberation_shared_mono"] = lambda grad: conv(grad, 1, 1, 1)
    c["convolution_reverberation_true_stereo"] = lambda grad: conv(grad, 2, BS, 4)

    def bus(grad, n, ir_bs, O):
        (x, ir), _ = setup(grad, (BS, 3, n), (ir_bs, 3, O, 3000))
        return lambda: F.convolution_bus(x, SR, ir)
    c["convolution_bus"] = lambda grad: bus(grad, N, BS, 2)
    c["convolution_bus_shared_padded"] = lambda grad: bus(grad, N + 2, 1, 1)

    def processor(grad, name, method="process_normalized", **kw):
        proc = getattr(D, name)(SR)
        g = torch.Generator().manual_seed(4)
        p = _leaf(_t(g, BS, proc.num_params, lo=0.05, hi=0.95), grad)
        x = _leaf(_t(g, BS, 2, N), grad)
        if method == "frequency_response":
            f = torch.linspace(0, SR / 2, 129)
            return lambda: proc.frequency_response(p, f)
        return lambda: getattr(proc, method)(x, p, **kw)
    for name in ("ParametricEQ", "Compressor", "Expander", "Gain"):
        c[f"{name}.process_normalized"] = lambda grad, name=name: processor(grad, name)
    c["Compressor.process_normalized_sidechain"] = lambda grad: processor(
        grad, "Compressor", sidechain=torch.ones(BS, 1, N, device="cuda"))
    c["ParametricEQ.frequency_response"] = lambda grad: processor(grad, "ParametricEQ", "frequency_response")
    c["Expander.gain_curve"] = lambda grad: processor(grad, "Expander", "gain_curve", db=True)
    return c


def run(call, grad):
    torch.manual_seed(0)
    out = call()
    if grad:
        torch.autograd.backward(out, torch.ones_like(out))


def record(fn, grad):
    call = fn(grad)
    run(call, grad)                                      # warm-up: module loads, plans, allocator pools
    torch.cuda.synchronize()
    stats0 = torch.cuda.memory_stats()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        run(call, grad)
        torch.cuda.synchronize()
    stats1 = torch.cuda.memory_stats()
    dev, api = Counter(), Counter()
    for e in prof.events():
        if e.device_type == DeviceType.CUDA:
            dev[e.name] += 1
        elif e.name.startswith("cuda") or (e.name.startswith("cu") and e.name[2:3].isupper()):
            api[e.name] += 1
    allocs = {k: stats1[k] - stats0[k] for k in ("allocation.all.allocated", "allocated_bytes.all.allocated")}
    return dev, api, allocs


def host_us(fn, grad, reps=25):
    call = fn(grad)
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        torch.manual_seed(0)
        t0 = time.perf_counter()
        out = call()
        ts.append(time.perf_counter() - t0)
        if grad:
            torch.autograd.backward(out, torch.ones_like(out))
    torch.cuda.synchronize()
    return statistics.median(ts) * 1e6


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="the launch list (text)")
    ap.add_argument("--host-out", help="median host microseconds per forward call (JSON)")
    args = ap.parse_args()
    lines, host = [], {}
    for name, fn in cases().items():
        for grad in (False, True):
            tag = f"{name} grad={int(grad)}"
            dev, api, allocs = record(fn, grad)
            lines.append(tag)
            lines += [f"  device {k} x{v}" for k, v in sorted(dev.items())]
            lines += [f"  host {k} x{v}" for k, v in sorted(api.items())]
            lines.append(f"  allocations {allocs['allocation.all.allocated']} bytes "
                         f"{allocs['allocated_bytes.all.allocated']}")
            if args.host_out:
                host[tag] = round(host_us(fn, grad), 1)
    with open(args.out, "w") as f:
        f.write("\n".join(lines) + "\n")
    if args.host_out:
        with open(args.host_out, "w") as f:
            json.dump(host, f, indent=1)
    print(f"{len(lines)} lines, {sum(1 for ln in lines if not ln.startswith(' '))} cases -> {args.out}")


if __name__ == "__main__":
    main()
