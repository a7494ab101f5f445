"""Every op on rows that are not 16-byte aligned, at lengths n % 4 == 0, pinned to the fp64 oracles.

Each streaming kernel takes its fast path (TMA bulk copies or 128-bit vector accesses) only when n % 4 == 0 and every
row pointer is 16-byte aligned, and its fallback (cooperative or scalar copies) otherwise; the forward decides on
(x, y), the backward on (dL/dy, x, dL/dx).  Contiguous tensors with a storage offset reach the kernels unchanged
(``clip[:, :, 1:]`` of a mono clip, ``flat[k:k + numel].view(...)``, the gradient slices ``torch.cat`` hands back), so
every case here offsets x, dL/dy or both (and the side-chain key and the impulse response on their own) by 4, 8 or 12
bytes at lengths where the last tile is full (a multiple of the op's tile), one past it (+ 4) and shorter than a tile.

Arbiters: the fp64 oracle of each op at the tolerances of the file that pins it, and the aligned run of the same
inputs.  The EQ and dynamics fallbacks only change how tiles are copied, so all their outputs must match the aligned
run bit for bit; the pointwise and stereo fallbacks do the same per-element FMAs, so y and dL/dx match bit for bit while
their parameter gradients add per-thread partial sums in another order.  The reverbs' convolution runs on cuFFT
instead of the in-shared-memory FFT wherever the rows it reads are offset, forward and backward deciding separately:
an offset x saves cuFFT spectra that an own-FFT backward reads, an offset dL/dy the other way round (asserted through
dasp_debug_conv_last_path).  Every pin prints its errors ("PIN <case>: ...").
"""
import math
import re

import pytest
import torch

import conv_oracle
import conv_ts_oracle
import dyn_sidechain_oracle
import oracle
import reverb_pin
from helpers import COMP_RANGES, SR, denorm, eq_ranges, param_grad_err, peak_err

pytestmark = pytest.mark.gpu
PLACEMENTS = {"x": {"x": 1}, "gy": {"gy": 2}, "both": {"x": 3, "gy": 3}}
LENGTHS = ("tiles", "tiles+4", "short")


def _lib():
    from dasp_pytorch_b200 import _abi
    return _abi.lib()


def offset_copy(t, k):
    """a contiguous copy of t whose data_ptr() % 16 == 4 k (k = 0: an aligned copy)"""
    buf = torch.empty(t.numel() + 4, dtype=t.dtype, device=t.device)
    s = (k - buf.data_ptr() % 16 // 4) % 4
    out = buf[s: s + t.numel()].view(t.shape)
    out.copy_(t)
    assert out.is_contiguous() and out.data_ptr() % 16 == 4 * k, (out.data_ptr() % 16, k)
    return out


class Op:
    """one op: its inputs (CPU fp64; `rows` are the audio-shaped tensors that may be offset, `grad` the inputs that get
    a gradient), GPU and oracle functions of a dict of inputs, tolerances, and the outputs that must match the aligned
    run bit for bit"""

    def __init__(self, name, inputs, grad, gpu, ref, tol, exact, rows=("x",), pgrad="item"):
        self.name, self.inputs, self.grad, self.gpu, self.ref = name, inputs, grad, gpu, ref
        self.tol, self.exact, self.rows, self.pgrad = tol, exact, rows, pgrad


def run(op, gy, device, dtype, offsets=None, keep=None):
    """{"y": y, name: dL/dname} for L = <y, gy> by torch.autograd.grad; offsets: {tensor name | "gy": k}.  keep: a
    list that holds on to the device outputs, so that the next run's outputs cannot be handed the same memory (an
    element a kernel failed to write would then still hold the right value)"""
    offsets = offsets or {}
    t = {}
    for k, v in op.inputs.items():
        v = v.to(device=device, dtype=dtype)
        if offsets is not None and device != "cpu" and k in op.rows:
            v = offset_copy(v, offsets.get(k, 0))
        t[k] = v.detach().requires_grad_(k in op.grad)
    g = gy.to(device=device, dtype=dtype)
    if device != "cpu":
        g = offset_copy(g, offsets.get("gy", 0))
    y = op.gpu(t) if device != "cpu" else op.ref(t)
    grads = torch.autograd.grad(y, [t[k] for k in op.grad], grad_outputs=g)
    if keep is not None:
        keep += [y, *grads]
    return {"y": y.detach().cpu(), **{k: d.detach().cpu() for k, d in zip(op.grad, grads)}}


def errors(op, got, ref):
    """per-item errors: audio-shaped outputs by peak_err, the parameter gradients together (param_grad_err per item,
    or relative to the largest gradient over the batch for single-parameter ops)"""
    errs = {k: peak_err(got[k], ref[k]) for k in ["y"] + [k for k in op.grad if k in op.rows or k == "ir"]}
    ps = [k for k in op.grad if k not in errs]
    if ps:
        if op.pgrad == "item":
            errs["dp"] = param_grad_err([got[k] for k in ps], [ref[k] for k in ps])
        else:
            g, r = (torch.cat([d[k].double().reshape(-1) for k in ps]) for d in (got, ref))
            errs["dp"] = (g - r).abs().amax(0, keepdim=True) / r.abs().max()
    return errs


def pin(case, op, got, ref):
    errs = errors(op, got, ref)
    print(f"PIN {case}: " + " ".join(f"{k} {float(e.max()):.2e}" for k, e in errs.items()))
    for k, e in errs.items():
        assert bool((e < op.tol.get(k, op.tol["dp"])).all()), (case, k, e)


def check_op(op, gy, device, placements=PLACEMENTS, after=None):
    """pin the aligned run and every offset placement to the oracle; hold the exact outputs to the aligned run"""
    ref = run(op, gy, "cpu", torch.float64)
    keep = []
    base = run(op, gy, device, torch.float32, keep=keep)
    if after:
        after("aligned", {})
    pin(f"{op.name}-aligned", op, base, ref)
    for pname, offs in placements.items():
        got = run(op, gy, device, torch.float32, offs, keep)
        if after:
            after(pname, offs)
        pin(f"{op.name}-{pname}", op, got, ref)
        for k in op.exact:
            assert torch.equal(got[k], base[k]), (op.name, pname, k, float((got[k] - base[k]).abs().max()))


def _length(kind, tile):
    return {"tiles": 2 * tile, "tiles+4": 2 * tile + 4, "short": 8}[kind]


# ------------------------------------------------------------------ pointwise and stereo
PW_TOL = {"y": 1e-5, "x": 1e-5, "dp": 1e-4}           # tests/test_gpu_pointwise.py, tests/test_gpu_stereo.py


def _pointwise_ops(n, g):
    import dasp_pytorch_b200 as D
    bs, chs = 2, 2
    x = torch.rand(bs, chs, n, generator=g, dtype=torch.float64) * 2 - 1
    gain = torch.rand(bs, generator=g, dtype=torch.float64) * 48 - 24
    drive = torch.rand(bs * chs, generator=g, dtype=torch.float64) * 24
    return [Op("gain", {"x": x, "p": gain}, ("x", "p"), lambda t: D.gain(t["x"], SR, t["p"]),
               lambda t: oracle.gain(t["x"], SR, t["p"]), PW_TOL, ("y", "x"), pgrad="batch"),
            Op("distortion", {"x": x, "p": drive}, ("x", "p"), lambda t: D.distortion(t["x"], SR, t["p"]),
               lambda t: oracle.distortion(t["x"], SR, t["p"]), PW_TOL, ("y", "x"), pgrad="batch")]


def _stereo_ops(n, g):
    import dasp_pytorch_b200 as D
    r = lambda *s: torch.rand(*s, generator=g, dtype=torch.float64)
    ops = []
    for name, x, p in (("widener", r(3, 2, n) * 2 - 1, r(3)), ("panner", r(2, 3, n) * 2 - 1, r(2, 3) * 0.9 + 0.05),
                       ("bus", r(2, 2, 4, n) * 2 - 1, r(2, 4, 1) * 30 - 24)):
        fg, fo = getattr(D, f"stereo_{name}"), getattr(oracle, f"stereo_{name}")
        ops.append(Op(name, {"x": x, "p": p}, ("x", "p"), lambda t, fg=fg: fg(t["x"], SR, t["p"]),
                      lambda t, fo=fo: fo(t["x"], SR, t["p"]), PW_TOL, ("y", "x"), pgrad="batch"))
    return ops


def _cotangent(op, g):
    with torch.no_grad():
        y = op.ref({k: v for k, v in op.inputs.items()})
    return torch.randn(y.shape, generator=g, dtype=torch.float64)


@pytest.mark.parametrize("length", LENGTHS)
@pytest.mark.parametrize("family", ["pointwise", "stereo"])
def test_pointwise_and_stereo(cuda_device, family, length):
    """tile 4096 samples per row (pointwise), 2048 (stereo)"""
    tile = 4096 if family == "pointwise" else 2048
    n = _length(length, tile)
    g = torch.Generator().manual_seed(n + len(family))
    for op in (_pointwise_ops if family == "pointwise" else _stereo_ops)(n, g):
        op.name = f"{op.name}-n{n}"
        check_op(op, _cotangent(op, g), cuda_device)


_VEC_PAT = re.compile(r"(pointwise_fwd_kernel|pointwise_bwd_kernel|widener_kernel|panner_kernel|bus_fwd_kernel|"
                      r"bus_bwd_kernel)<([^>]*)>")


def _vec_flags(prof):
    """{(kernel, backward?): {VEC flags launched}} from a profiler trace"""
    out = {}
    for e in prof.events():
        m = _VEC_PAT.search(e.name)
        if not m:
            continue
        args = [a.strip() for a in m[2].split(",")]
        kern = m[1]
        if kern.startswith("pointwise"):
            key, vec = (kern, None), args[1]
        elif kern.startswith("bus"):
            key, vec = (kern, None), args[0]
        else:
            key, vec = (kern, args[1]), args[0]
        out.setdefault(key, set()).add(vec)
    return out


@pytest.mark.parametrize("where", ["x", "gy"])
def test_pointwise_and_stereo_run_the_scalar_kernels(cuda_device, where):
    """the profiler sees the <..., false> (scalar) instantiation of every pointwise and stereo kernel when x (forward
    and backward) or only dL/dy (backward) is offset, and the vector one elsewhere"""
    from torch.profiler import ProfilerActivity, profile
    n = 4096
    g = torch.Generator().manual_seed(5)
    ops = _pointwise_ops(n, g) + _stereo_ops(n, g)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for op in ops:
            run(op, _cotangent(op, g), cuda_device, torch.float32, PLACEMENTS[where])
        torch.cuda.synchronize()
    flags = _vec_flags(prof)
    fwd = {("pointwise_fwd_kernel", None), ("widener_kernel", "false"), ("panner_kernel", "false"),
           ("bus_fwd_kernel", None)}
    bwd = {("pointwise_bwd_kernel", None), ("widener_kernel", "true"), ("panner_kernel", "true"), ("bus_bwd_kernel", None)}
    assert set(flags) == fwd | bwd, sorted(flags)
    print(f"VEC flags with {where} offset: {sorted(flags.items())}")
    for k in bwd:
        assert flags[k] == {"false"}, (k, flags[k])
    for k in fwd:
        assert flags[k] == ({"false"} if where == "x" else {"true"}), (k, flags[k])


# ------------------------------------------------------------------ parametric EQ
def _eq_op(bs, chs, n, g):
    import dasp_pytorch_b200 as D
    x = torch.rand(bs, chs, n, generator=g, dtype=torch.float64) * 2 - 1
    p = denorm(torch.rand(bs, 18, generator=g), eq_ranges(), torch.float64)
    inputs = {"x": x, **{f"p{i}": q for i, q in enumerate(p)}}
    names = [f"p{i}" for i in range(18)]
    return Op(f"eq-{chs}ch-n{n}", inputs, ("x", *names), lambda t: D.parametric_eq(t["x"], SR, *[t[k] for k in names]),
              lambda t: oracle.parametric_eq(t["x"], SR, *[t[k] for k in names], fsm_tail=1 << 16),
              {"y": 1e-4, "x": 1e-4, "dp": 1e-4}, ("y", "x", *names))


@pytest.mark.parametrize("length", LENGTHS)
@pytest.mark.parametrize("chs", [2, 3])
def test_parametric_eq(cuda_device, chs, length):
    """tile dasp_eq_tile_len(); float tables at 2 channels, pair tables at 3 (tests/test_gpu_eq.py: strict 1e-4)"""
    n = _length(length, int(_lib().dasp_eq_tile_len(6)))
    g = torch.Generator().manual_seed(n + chs)
    op = _eq_op(3, chs, n, g)
    check_op(op, _cotangent(op, g), cuda_device)


# ------------------------------------------------------------------ compressor / expander, with and without a key
DYN_TOL = {"y": 1e-4, "x": 1e-4, "key": 1e-4, "dp": 1e-4}          # tests/test_gpu_dynamics_pin.py
DYN_NAMES = ("threshold", "ratio", "attack", "release", "knee", "makeup")


def _dyn_op(kind, bs, chs, n, g, key_chs=0):
    import dasp_pytorch_b200 as D
    level = 0.05 + 0.95 * torch.rand(bs, 1, 1, generator=g, dtype=torch.float64)
    x = (torch.rand(bs, chs, n, generator=g, dtype=torch.float64) * 2 - 1) * level
    p01 = torch.rand(bs, 6, generator=g)
    p01[:, 4] = p01[:, 4].clamp(min=0.05)                  # knee > 0
    p = denorm(p01, COMP_RANGES, torch.float64)
    if kind == "exp":
        p[1] = 1.0 + 3.0 * p01[:, 1].double()              # expansion ratios up to 4 (larger ones underflow in fp32)
    tail = max(1 << 16, 1 << int(12.6 * SR * float(p[2].max()) * 1e-3).bit_length())   # alias-free smoother
    inputs = {"x": x, **dict(zip(DYN_NAMES, p))}
    grad = ["x"] + [k for k in DYN_NAMES if k != "release"]
    rows = ("x",)
    if key_chs:
        inputs["key"] = torch.rand(bs, key_chs, n, generator=g, dtype=torch.float64) * 2 - 1
        grad.insert(1, "key")
        rows = ("x", "key")
        gpu_fn = getattr(D, "sidechain_compressor" if kind == "comp" else "sidechain_expander")
        ref_fn = getattr(dyn_sidechain_oracle, "compressor" if kind == "comp" else "expander")
        gpu = lambda t: gpu_fn(t["x"], SR, *[t[k] for k in DYN_NAMES], sidechain=t["key"])
        ref = lambda t: ref_fn(t["x"], SR, *[t[k] for k in DYN_NAMES], fsm_tail=tail, sidechain=t["key"])
    else:
        gpu_fn = D.compressor if kind == "comp" else D.expander
        ref_fn = oracle.compressor if kind == "comp" else oracle.expander
        gpu = lambda t: gpu_fn(t["x"], SR, *[t[k] for k in DYN_NAMES])
        ref = lambda t: ref_fn(t["x"], SR, *[t[k] for k in DYN_NAMES], fsm_tail=tail)
    name = f"{kind}{'-key' + str(key_chs) if key_chs else ''}-{chs}ch-n{n}"
    return Op(name, inputs, tuple(grad), gpu, ref, DYN_TOL, ("y", *grad), rows=rows)


@pytest.mark.parametrize("length", LENGTHS)
@pytest.mark.parametrize("kind,chs,key_chs", [("comp", 2, 0), ("exp", 1, 0), ("comp", 2, 1), ("exp", 1, 3)])
def test_dynamics(cuda_device, kind, chs, key_chs, length):
    """tile dasp_dynamics_tile_len(bs, chs) / dasp_dynamics_sidechain_tile_len(bs, chs, K); the key is offset on its own
    too, and together with x and dL/dy"""
    bs = 2
    lib = _lib()
    tile = int(lib.dasp_dynamics_sidechain_tile_len(bs, chs, key_chs) if key_chs else lib.dasp_dynamics_tile_len(bs, chs))
    n = _length(length, tile)
    g = torch.Generator().manual_seed(n + 10 * chs + key_chs)
    op = _dyn_op(kind, bs, chs, n, g, key_chs)
    placements = dict(PLACEMENTS)
    if key_chs:
        placements.update({"key": {"key": 1}, "all": {"x": 2, "gy": 1, "key": 3}})
    check_op(op, _cotangent(op, g), cuda_device, placements)


# ------------------------------------------------------------------ reverbs
REV_TOL = {"y": 1e-4, "x": 1e-4, "ir": 1e-4, "dp": 1e-4}          # tests/test_gpu_conv_reverb*.py, reverb_pin.py


def _expect_paths(n):
    """after(placement, offsets): the convolution ran on the own FFT exactly where its rows were aligned"""
    def after(pname, offs):
        lib = _lib()
        own_fwd = n % 4 == 0 and not offs.get("x")
        own_bwd = n % 4 == 0 and not offs.get("gy")
        assert (lib.dasp_debug_conv_last_path(0) & 1) == own_fwd, (pname, lib.dasp_debug_conv_last_path(0))
        assert (lib.dasp_debug_conv_last_path(1) & 1) == own_bwd, (pname, lib.dasp_debug_conv_last_path(1))
    return after


def _conv_op(ir_kind, ir_grad, n, L, g):
    import dasp_pytorch_b200 as D
    bs = 3
    ir_bs, ir_chs = {"item": (bs, 2), "shared": (1, 2), "ts": (bs, 4)}[ir_kind]
    x = torch.rand(bs, 2, n, generator=g, dtype=torch.float64) * 2 - 1
    ir = (torch.rand(ir_bs, ir_chs, L, generator=g, dtype=torch.float64) * 2 - 1) * torch.exp(
        -torch.arange(L, dtype=torch.float64) / (L / 4))
    mix = 0.2 + 0.7 * torch.rand(bs, generator=g, dtype=torch.float64)
    fo = conv_ts_oracle if ir_chs == 4 else conv_oracle
    ref = lambda t: fo.convolution_reverberation(t["x"], SR, t["ir"].expand(bs, -1, -1), t["mix"])
    grad = ("x", "ir", "mix") if ir_grad else ("x", "mix")
    return Op(f"conv-{ir_kind}-{'irgrad' if ir_grad else 'fixed'}-n{n}-L{L}", {"x": x, "ir": ir, "mix": mix}, grad,
              lambda t: D.convolution_reverberation(t["x"], SR, t["ir"], t["mix"]), ref, REV_TOL, (), rows=("x", "ir"),
              pgrad="batch")


@pytest.mark.parametrize("length", LENGTHS)
@pytest.mark.parametrize("ir_kind", ["item", "shared", "ts"])
def test_convolution_reverberation(cuda_device, monkeypatch, ir_kind, length):
    """convolution block 4096; one IR per item, one IR shared by the batch, true-stereo IRs, each with and without an
    IR gradient; the IR offset on its own.  Each offset side switches its own direction to cuFFT"""
    from dasp_pytorch_b200 import functional as F
    monkeypatch.setattr(F, "REVERB_CHUNK_ITEMS", 2)          # bs 3: a full chunk and a remainder
    n = _length(length, 4096)
    L = 5000
    placements = dict(PLACEMENTS, ir={"ir": 1}, all={"x": 1, "gy": 2, "ir": 3})
    for ir_grad in (True, False):
        g = torch.Generator().manual_seed(n + len(ir_kind) + ir_grad)
        op = _conv_op(ir_kind, ir_grad, n, L, g)
        check_op(op, _cotangent(op, g), cuda_device, placements, after=_expect_paths(n))


def _reverb_op(n, L, taps, noise=None, seed=None):
    import dasp_pytorch_b200 as D
    bs = 2
    g = torch.Generator().manual_seed(n + L)
    x = torch.rand(bs, 2, n, generator=g, dtype=torch.float64) * 2 - 1
    p = torch.rand(bs, 25, generator=g, dtype=torch.float64)
    names = [f"p{i}" for i in range(25)]
    inputs = {"x": x, **{k: p[:, i].clone() for i, k in enumerate(names)}}
    kw = dict(num_samples=L, num_bandpass_taps=taps)

    def gpu(t):
        if noise is None:
            torch.manual_seed(seed)
            return D.noise_shaped_reverberation(t["x"], SR, *[t[k] for k in names], **kw)
        return D.noise_shaped_reverberation(t["x"], SR, *[t[k] for k in names], noise=noise.to(t["x"]), **kw)

    def ref(t):
        return oracle.noise_shaped_reverberation(t["x"], SR, *[t[k] for k in names], noise=ref_noise[0].to(t["x"].dtype),
                                                 method="fft", **kw)
    ref_noise = [noise]
    op = Op(f"reverb-{'caller' if noise is not None else 'device'}-noise-n{n}-L{L}", inputs, ("x", *names), gpu, ref,
            REV_TOL, ())
    return op, g, ref_noise


@pytest.mark.parametrize("length", LENGTHS)
@pytest.mark.parametrize("noise_from", ["caller", "device"])
def test_noise_shaped_reverberation(cuda_device, noise_from, length):
    """caller's noise: the oracle with the same tensor; device noise: the oracle with the noise read back through the
    unit-impulse filter bank hook (reverb_pin.white_sequences), at L = 6912, 1023 taps (one 8192-point polyphase block,
    so the backward's dL/dIR runs on the own FFT whenever dL/dy is aligned)"""
    n = _length(length, 4096)
    L, taps, seed = 6912, 1023, 17
    if noise_from == "caller":
        op, g, _ = _reverb_op(n, L, taps, noise=oracle.reverb_noise(2, L, taps, seed=seed))
    else:
        op, g, ref_noise = _reverb_op(n, L, taps, seed=seed)
        x = op.inputs["x"].float().to(cuda_device)
        p = [op.inputs[f"p{i}"].float().to(cuda_device) for i in range(25)]
        geom, used, seqs = reverb_pin.white_sequences(x, p, L, taps, seed)
        assert geom.nb == 8192 and reverb_pin.polyphase(geom) and used == 2, (geom, used)
        ref_noise[0] = reverb_pin.reference_noise(torch.stack([seqs[i] for i in range(2)]), geom, L, taps)
    synth = 0 if noise_from == "caller" else 2          # time-domain noise on cuFFT / the own-FFT synthesis

    def after(pname, offs):
        assert _lib().dasp_debug_reverb_last_path() == synth, pname
    check_op(op, _cotangent(op, g), cuda_device, after=after)


# ------------------------------------------------------------------ a realistic composition
def test_offset_clip_through_a_chain(cuda_device):
    """a mono clip sliced as clip[:, :, 1:] (n % 4 == 0, 4 bytes past alignment) through parametric_eq -> compressor ->
    convolution_reverberation; the loss joins this chain's output with a second, odd-length chain's through torch.cat,
    so the reverb's backward receives an offset view of dL/dy.  Equals the same chains on aligned copies with a loss
    that hands back aligned gradients"""
    import dasp_pytorch_b200 as D
    n1, n2, L = 4001, 8192, 3000
    g = torch.Generator().manual_seed(77)
    clip1 = (torch.rand(1, 1, n1, generator=g) * 2 - 1).to(cuda_device)
    clip2 = (torch.rand(1, 1, n2 + 1, generator=g) * 2 - 1).to(cuda_device)
    eq = [q.to(cuda_device) for q in denorm(torch.rand(1, 18, generator=g), eq_ranges())]
    comp = [q.to(cuda_device) for q in denorm(torch.rand(1, 6, generator=g).clamp(min=0.05), COMP_RANGES)]
    ir = ((torch.rand(1, 2, L, generator=g) * 2 - 1) * torch.exp(-torch.arange(L) / 750.0)).to(cuda_device)
    mix = torch.tensor([0.6], device=cuda_device)
    r = torch.randn(1, 1, 2 * (n1 + n2), generator=g).to(cuda_device)

    def chains(x2, joined):
        leaves = [t.detach().clone().requires_grad_(True) for t in [*eq, *comp[:3], *comp[4:], ir, mix]]
        e, c, (h, m) = leaves[:18], leaves[18:23], leaves[23:]
        x2 = x2.detach().requires_grad_(True)
        seen = []

        def chain(x):
            y = D.parametric_eq(x, SR, *e)
            y = D.compressor(y, SR, *c[:3], comp[3], *c[3:])
            return D.convolution_reverberation(y, SR, h, m)
        y1, y2 = chain(clip1), chain(x2)
        y2.register_hook(lambda gy: seen.append(gy.data_ptr() % 16))
        if joined:
            loss = (torch.cat([y1.reshape(1, 1, -1), y2.reshape(1, 1, -1)], dim=-1) * r).sum()
        else:
            loss = (y1 * r[..., : 2 * n1].reshape(1, 2, n1)).sum() + (y2 * r[..., 2 * n1:].reshape(1, 2, n2)).sum()
        grads = torch.autograd.grad(loss, [x2, *leaves])
        return [y2.detach()] + list(grads), seen

    x2 = clip2[:, :, 1:]
    assert x2.is_contiguous() and x2.data_ptr() % 16 == 4
    got, seen = chains(x2, joined=True)
    assert seen == [8], seen                               # 2 n1 floats into the joined gradient
    ref, seen = chains(x2.clone(), joined=False)
    assert seen == [0], seen
    names = ["y", "dx"] + [f"eq{i}" for i in range(18)] + ["comp"] * 5 + ["ir", "mix"]
    for name, a, b in zip(names, got, ref):
        e = float((a - b).abs().max() / b.abs().max())
        print(f"PIN chain {name}: {e:.2e}")
        assert e < 1e-4, (name, e)
