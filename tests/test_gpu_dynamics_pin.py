"""Pin every compressor / expander kernel variant to the fp64 oracle.

dynamics.cu instantiates its forward and backward for curve {Compress, Expand} x warps per item W {1, 2, 4, 8, 16} x
channel path {generic channel loop, stereo registers ST (chs == 2, no look-ahead), look-ahead LA}: 30 kernels each
way.  A forced W (dasp_debug_force_warps) that does not fit shared memory is silently halved by pick_warps, so every
case asserts the W it covers through dasp_dynamics_tile_len (= W * 32 * E, E = 7 samples per thread).
DASP_DYN_GENERIC=1 sends stereo through the generic loop; it is read at every launch.  n % 4 == 0 streams the tiles
with TMA, any other n with cooperative copies.

Arbiter: the fp64 oracle on an enlarged frequency-sampling grid (fsm_tail), which equals the true recursion and stays
differentiable.  Tolerances are fixed, per item in the SURVEY.md 8c metric: TOL for y and dL/dx, PGRAD_TOL for the
five parameter gradients.  The loss is <y, r> with a fixed random cotangent r, so dL/dy does not shrink with y.
Every pin prints its errors ("PIN <case>: ...").
"""
import contextlib
import re

import pytest
import torch

import oracle
from helpers import COMP_RANGES, SR, denorm, param_grad_err, peak_err

pytestmark = pytest.mark.gpu
TOL = 1e-4
PGRAD_TOL = 1e-4
E = 7                                   # samples per thread per tile (dynamics.cu kE)
WARPS = (1, 2, 4, 8, 16)
KINDS = ("comp", "exp")
EXP_RATIO_MAX = 4.0                     # larger expansion ratios underflow the gain in fp32


def _fns(kind):
    import dasp_pytorch_b200 as D
    return (D.compressor, oracle.compressor) if kind == "comp" else (D.expander, oracle.expander)


def _lib():
    from dasp_pytorch_b200 import _abi
    return _abi.lib()


def tile_len(bs, chs):
    return int(_lib().dasp_dynamics_tile_len(bs, chs))


@contextlib.contextmanager
def forced_warps(w):
    _lib().dasp_debug_force_warps(w)
    try:
        yield
    finally:
        _lib().dasp_debug_force_warps(0)


def expected_warps(bs, chs, sms):
    """pick_warps restated: fill 16 warps per SM, one 16-warp CTA per item when bs <= SMs, then halve W until three
    backward stages (x and dL/dy per channel) fit in 96 KB (200 KB at W = 16)."""
    w = 1
    while w < 8 and bs * w < 16 * sms:
        w *= 2
    if w == 8 and bs <= sms:
        w = 16
    while w > 1 and 3 * 2 * chs * w * 32 * E * 4 + 512 > (200 if w == 16 else 96) * 1024:
        w //= 2
    return w


def _params(kind, bs, g):
    p01 = torch.rand(bs, 6, generator=g)
    p01[:, 4] = p01[:, 4].clamp(min=0.05)        # knee > 0 (W == 0 gives NaN grads in the reference too)
    params = denorm(p01, COMP_RANGES)
    if kind == "exp":
        params[1] = 1.0 + (EXP_RATIO_MAX - 1.0) * p01[:, 1]
    return params


def _inputs(kind, bs, chs, n, seed):
    g = torch.Generator().manual_seed(seed)
    level = 0.05 + 0.95 * torch.rand(bs, 1, 1, generator=g)
    x = (torch.rand(bs, chs, n, generator=g) * 2 - 1) * level
    return x, _params(kind, bs, g), torch.randn(bs, chs, n, generator=g)


def _run(fn, x, params, r, device, dtype):
    """y, dL/dx, [dL/dparam] for L = <y, r>"""
    xx = x.to(device=device, dtype=dtype).clone().requires_grad_(True)
    pp = [p.to(device=device, dtype=dtype).clone().requires_grad_(True) for p in params]
    y = fn(xx, pp)
    (y * r.to(device=device, dtype=dtype)).sum().backward()
    return y.detach().cpu(), xx.grad.detach().cpu(), [None if p.grad is None else p.grad.detach().cpu() for p in pp]


def fsm_tail(sample_rate, attack_ms_max):
    """grid extension past n that makes the oracle's smoother alias-free: alpha^tail < 1e-12 at the longest attack"""
    need = int(12.6 * sample_rate * attack_ms_max * 1e-3) + 1
    return max(1 << 16, 1 << (need - 1).bit_length())


def gpu_run(kind, x, params, r, device, sample_rate=SR, eps=1e-8, la=0):
    gpu, _ = _fns(kind)
    return _run(lambda xx, pp: gpu(xx, sample_rate, *pp, eps=eps, lookahead_samples=la), x, params, r, device,
                torch.float32)


def pin(case, kind, x, params, r, device, sample_rate=SR, eps=1e-8, la=0, got=None):
    """run (or take) the GPU result and hold it to the fp64 oracle; returns (gpu result, per-item errors)"""
    _, orc = _fns(kind)
    got = got or gpu_run(kind, x, params, r, device, sample_rate, eps, la)
    y, dx, dp = got
    tail = fsm_tail(sample_rate, float(params[2].max()))
    kw = dict(eps=eps, lookahead_samples=la)
    y64, dx64, dp64 = _run(lambda xx, pp: orc(xx, sample_rate, *pp, fsm_tail=tail, **kw), x, params, r, "cpu",
                           torch.float64)
    yt = orc(x.double(), sample_rate, *[p.double() for p in params], smoother="recursion", **kw)
    assert (peak_err(y64, yt) < 1e-9).all()                       # the enlarged grid is the true recursion
    assert dp[3] is None and dp64[3] is None                      # release_ms: no gradient
    for t in [y, dx] + [d for d in dp if d is not None]:
        assert torch.isfinite(t).all(), case
    errs = {"y": peak_err(y, y64), "dx": peak_err(dx, dx64), "dp": param_grad_err(dp, dp64)}
    print(f"PIN {case}: y {errs['y'].max():.2e} dx {errs['dx'].max():.2e} dparams {errs['dp'].max():.2e}")
    assert (errs["y"] < TOL).all(), (case, errs["y"])
    assert (errs["dx"] < TOL).all(), (case, errs["dx"])
    assert (errs["dp"] < PGRAD_TOL).all(), (case, errs["dp"])
    return got, errs


# ------------------------------------------------------------------ 1. instantiation matrix
def _matrix():
    """per (kind, W): ST (and generic stereo on the same input), generic mono, generic 3-ch where W fits, each with
    and without a look-ahead between one and two tiles; the pipeline alternates along the list so that TMA and
    cooperative copies both meet every (kind, W) and every look-ahead kernel"""
    cases = []
    for k, kind in enumerate(KINDS):
        for w in WARPS:
            paths = [("ST+gen2", False), ("gen1", False)] + ([("gen3", False)] if w <= 4 else [])
            paths += [("gen1", True), ("gen2", True)] + ([("gen3", True)] if w <= 4 else [])
            for i, (path, la) in enumerate(paths):
                pipe = ("tma", "coop")[(i + k) % 2]
                cases.append(pytest.param(kind, w, path, la, pipe,
                                          id=f"{kind}-W{w}-{path}-{'la1.5T' if la else 'la0'}-{pipe}"))
    return cases


@pytest.mark.parametrize("kind,w,path,la,pipe", _matrix())
def test_instantiation_matrix(cuda_device, monkeypatch, kind, w, path, la, pipe):
    bs, T = 3, w * 32 * E
    chs = int(path[-1])
    n = 3 * T + (36 if pipe == "tma" else 37)
    la = T + T // 2 + 5 if la else 0
    x, params, r = _inputs(kind, bs, chs, n, seed=100 * w + chs + la)
    case = f"{kind}-W{w}-{path}-la{la}-n{n}"
    with forced_warps(w):
        assert tile_len(bs, chs) == T
        with monkeypatch.context() as m:
            if path == "gen2":
                m.setenv("DASP_DYN_GENERIC", "1")
            got, _ = pin(case, kind, x, params, r, cuda_device, la=la)
        if path == "ST+gen2":
            with monkeypatch.context() as m:
                m.setenv("DASP_DYN_GENERIC", "1")
                gen = pin(case + "-generic", kind, x, params, r, cuda_device)[0]
            # same fp32 side-chain sum, scan and apply: bit-identical y (dG is accumulated in another fma order, so
            # the gradients are only held to the oracle)
            assert torch.equal(got[0], gen[0])


def test_every_instantiation_is_launched(cuda_device, monkeypatch):
    """the kernels the profiler sees: all 30 (curve, W, LA, ST) instantiations, forward and backward"""
    from torch.profiler import ProfilerActivity, profile
    bs, chs = 3, 2
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for kind in KINDS:
            for w in WARPS:
                T = w * 32 * E
                x, params, r = _inputs(kind, bs, chs, 2 * T + 1, seed=w)
                for path in ("ST", "generic", "LA"):
                    with forced_warps(w), monkeypatch.context() as m:
                        assert tile_len(bs, chs) == T
                        if path == "generic":
                            m.setenv("DASP_DYN_GENERIC", "1")
                        gpu_run(kind, x, params, r, cuda_device, la=T + 1 if path == "LA" else 0)
        torch.cuda.synchronize()
    names = {e.name for e in prof.events() if "dynamics_" in e.name}
    pat = re.compile(r"dynamics_(fwd|bwd)_kernel<(.+?), (\d+), (true|false), (true|false)>")
    seen = set()
    for name in names:
        mt = pat.search(name)
        if mt:
            curve = "comp" if ("Compress" in mt[2] or mt[2].endswith("0")) else "exp"
            seen.add((mt[1], curve, int(mt[3]), mt[4] == "true", mt[5] == "true"))
    want = {(d, k, w, la, st) for d in ("fwd", "bwd") for k in KINDS for w in WARPS
            for la, st in ((False, True), (False, False), (True, False))}
    assert want <= seen, (sorted(want - seen), sorted(names))
    assert any("dynamics_lookahead_fixup_kernel" in s for s in names)


# ------------------------------------------------------------------ 2. look-ahead edges
LA_EDGES = {"1": lambda T, n: 1, "T-1": lambda T, n: T - 1, "T": lambda T, n: T, "T+1": lambda T, n: T + 1,
            "3T+5": lambda T, n: 3 * T + 5, "n-1": lambda T, n: n - 1, "n": lambda T, n: n, "n+1": lambda T, n: n + 1,
            "2n-1": lambda T, n: 2 * n - 1}


@pytest.mark.parametrize("la_name", list(LA_EDGES))
@pytest.mark.parametrize("chs", [1, 2])
@pytest.mark.parametrize("w", [1, 16])
@pytest.mark.parametrize("kind", KINDS)
def test_lookahead_edges(cuda_device, kind, w, chs, la_name):
    """delays that cross tile boundaries, reach the last samples, and reach past n (silence).  Mono runs a ragged
    n on the cooperative copies, stereo a ragged n on TMA.  dL/dx includes the fix-up kernel's direct term
    gy[m+la] G[m+la] and the first la samples, which only see it"""
    bs, T = 3, w * 32 * E
    n = 4 * T + (13 if chs == 1 else 12)
    la = LA_EDGES[la_name](T, n)
    x, params, r = _inputs(kind, bs, chs, n, seed=7 * la + chs)
    case = f"{kind}-W{w}-{chs}ch-la{la_name}={la}-n{n}"
    with forced_warps(w):
        assert tile_len(bs, chs) == T
        if la < n:
            pin(case, kind, x, params, r, cuda_device, la=la)
            return
        y, dx, dp = gpu_run(kind, x, params, r, cuda_device, la=la)
    _, orc = _fns(kind)
    y64 = orc(x.double(), SR, *[p.double() for p in params], lookahead_samples=la)
    assert float(y64.abs().max()) == 0.0
    assert float(y.abs().max()) == 0.0, case
    for t in [dx] + [d for d in dp if d is not None]:
        assert torch.isfinite(t).all() and float(t.abs().max()) == 0.0, case
    print(f"PIN {case}: y, dL/dx and dparams exactly 0")


# ------------------------------------------------------------------ 3. gain-curve regions, silence, eps
REGION_ITEMS = [(t, k, rr) for t in (-60.0, 0.0) for k in (0.05, 12.0) for rr in ("one", "max")]


def _sweep(n, seed, reverse):
    """side chain sweeping -100 -> 0 dBFS with random signs and stretches of exact digital zero (start, inside,
    end: the backward's first tile is the partial last one)"""
    g = torch.Generator().manual_seed(seed)
    lv = torch.linspace(-100.0, 0.0, n, dtype=torch.float64)
    s = 10.0 ** (lv / 20.0) * (torch.randint(0, 2, (n,), generator=g) * 2 - 1)
    if reverse:
        s = s.flip(0)
    for a, b in ((0, 150), (n // 7, n // 7 + 400), (n // 2, n // 2 + 300), (n - 200, n)):
        s[a:b] = 0
    return s.float()


@pytest.mark.parametrize("eps", [1e-8, 1e-3])
@pytest.mark.parametrize("w,chs", [(1, 1), (16, 2)])
@pytest.mark.parametrize("kind", KINDS)
def test_gain_curve_regions(cuda_device, kind, w, chs, eps):
    """one item per (threshold -60 / 0 dB, knee 0.05 / 12 dB, ratio 1 / range max); each side chain crosses
    below-knee, knee and above-knee.  eps = 1e-3 (-60 dBFS) puts part of every sweep under the |side| >= eps gate
    of dL/dx.  Stereo halves sum exactly, so fp32 and fp64 see the same side chain"""
    bs = len(REGION_ITEMS)
    n = 12000 if w == 16 else 12001
    rmax = 20.0 if kind == "comp" else EXP_RATIO_MAX
    g = torch.Generator().manual_seed(31)
    side = torch.stack([_sweep(n, i, reverse=i % 2 == 1) for i in range(bs)])
    x = (side / chs).unsqueeze(1).expand(bs, chs, n).contiguous()
    params = [torch.tensor([it[0] for it in REGION_ITEMS]),
              torch.tensor([1.0 if it[2] == "one" else rmax for it in REGION_ITEMS]),
              5.0 + 95.0 * torch.rand(bs, generator=g),
              torch.full((bs,), 50.0),
              torch.tensor([it[1] for it in REGION_ITEMS]),
              12.0 * torch.rand(bs, generator=g)]
    r = torch.randn(bs, chs, n, generator=g)
    with forced_warps(w):
        assert tile_len(bs, chs) == w * 32 * E
        pin(f"{kind}-W{w}-{chs}ch-eps{eps:g}", kind, x, params, r, cuda_device, eps=eps)


@pytest.mark.parametrize("kind", KINDS)
def test_silent_item_among_loud_ones(cuda_device, kind):
    """an all-zero item: y exactly 0, no NaN anywhere, exactly zero parameter gradients, dL/dx = r G from the
    oracle; its neighbours are bit-identical to a run without it (same forced W)"""
    x, params, r = _inputs(kind, 4, 2, 5000, seed=41)
    x[2] = 0
    keep = [0, 1, 3]
    with forced_warps(4):
        assert tile_len(4, 2) == tile_len(3, 2) == 4 * 32 * E
        (y, dx, dp), _ = pin(f"{kind}-silent-item", kind, x, params, r, cuda_device)
        y3, dx3, dp3 = gpu_run(kind, x[keep], [p[keep] for p in params], r[keep], cuda_device)
    assert float(y[2].abs().max()) == 0.0
    assert all(float(d[2]) == 0.0 for d in dp if d is not None)
    assert torch.equal(y[keep], y3) and torch.equal(dx[keep], dx3)
    assert all(torch.equal(a[keep], b) for a, b in zip(dp, dp3) if a is not None)


# ------------------------------------------------------------------ 4. sample rates
@pytest.mark.parametrize("w", [1, 16])
@pytest.mark.parametrize("sample_rate", [16000, 22050, 48000, 96000])
@pytest.mark.parametrize("kind", KINDS)
def test_sample_rates(cuda_device, kind, sample_rate, w):
    """attack 5 and 100 ms: alpha from 0.973 (16 kHz, 5 ms) to 0.99977 (96 kHz, 100 ms) through the power tables
    a^(E 2^k), a^(32E), a^(E lane) and the tile-to-tile carry"""
    bs, chs = 2, 2
    n = 3 * 3584 + (100 if w == 16 else 101)
    x, params, r = _inputs(kind, bs, chs, n, seed=sample_rate + w)
    params[2] = torch.tensor([5.0, 100.0])
    with forced_warps(w):
        assert tile_len(bs, chs) == w * 32 * E
        pin(f"{kind}-{sample_rate}Hz-W{w}", kind, x, params, r, cuda_device, sample_rate=sample_rate)


# ------------------------------------------------------------------ 5. wide channel counts
WIDE = {4: 4, 5: 2, 8: 2, 19: 1, 32: 1}     # W that pick_warps leaves for 3 items (at most one item per SM)


@pytest.mark.parametrize("chs", sorted(WIDE))
@pytest.mark.parametrize("kind", KINDS)
def test_wide_channel_counts(cuda_device, kind, chs):
    """automatic W shrinks with the channel count; from 19 channels up the one-warp backward needs more than 96 KB
    (172 544 B at 32 channels) and runs on the 200 KB opt-in"""
    bs = 3
    sms = torch.cuda.get_device_properties(cuda_device).multi_processor_count
    assert expected_warps(bs, chs, sms) == WIDE[chs]
    assert tile_len(bs, chs) == WIDE[chs] * 32 * E
    n = 4000 if chs % 2 == 0 else 4001
    x, params, r = _inputs(kind, bs, chs, n, seed=chs)
    pin(f"{kind}-{chs}ch-W{WIDE[chs]}", kind, x, params, r, cuda_device)


@pytest.mark.parametrize("kind", KINDS)
def test_cancelling_channels(cuda_device, kind):
    """channels that cancel to a side chain about 80 dB below the loudest channel: a running fp32 sum keeps the loud
    channels' rounding error, a large share of the side chain there, and dL/dx carries 1/side.  The threshold puts
    the side chain where the curve has a slope (above the knee for the compressor, below it for the expander)"""
    bs, chs, n = 3, 4, 6000
    x, params, r = _inputs(kind, bs, chs, n, seed=77)
    x[:, 1] = -x[:, 0] + 3e-3 * x[:, 0]
    x[:, 2] *= 30.0
    x[:, 3] = -x[:, 2]
    params[0] = torch.full((bs,), -60.0 if kind == "comp" else -20.0)
    assert tile_len(bs, chs) == 4 * 32 * E
    pin(f"{kind}-cancelling-4ch", kind, x, params, r, cuda_device)


def test_too_many_channels_raises(cuda_device):
    import dasp_pytorch_b200 as D
    from dasp_pytorch_b200._abi import DaspError
    assert tile_len(3, 33) == 0
    x = torch.rand(3, 33, 500, device=cuda_device)
    p = [torch.full((3,), v, device=cuda_device) for v in (-20.0, 4.0, 10.0, 50.0, 6.0, 3.0)]
    for fn in (D.compressor, D.expander):
        with pytest.raises(DaspError):
            fn(x, SR, *p)
        with pytest.raises(DaspError):
            fn(x.clone().requires_grad_(True), SR, *p)


# ------------------------------------------------------------------ 6. automatic geometry by batch size
@pytest.mark.parametrize("which,kind,n", [("sm", "comp", 3000), ("sm+1", "exp", 3001), ("4sm-1", "comp", 3001),
                                          ("4sm", "exp", 3000)])
def test_automatic_warps_by_batch_size(cuda_device, which, kind, n):
    """the batch sizes where the automatic W changes (132 SMs: 16, 8, 8, 4); 512 items run at W = 8"""
    sms = torch.cuda.get_device_properties(cuda_device).multi_processor_count
    bs = {"sm": sms, "sm+1": sms + 1, "4sm-1": 4 * sms - 1, "4sm": 4 * sms}[which]
    w = {"sm": 16, "sm+1": 8, "4sm-1": 8, "4sm": 4}[which]
    assert expected_warps(bs, 2, sms) == w
    assert tile_len(bs, 2) == w * 32 * E
    x, params, r = _inputs(kind, bs, 2, n, seed=bs)
    pin(f"{kind}-bs{bs}-W{w}", kind, x, params, r, cuda_device)


# ------------------------------------------------------------------ 7. packed path and entry contract
def test_expander_process_normalized(cuda_device):
    """Expander.process_normalized == expander() on the denormalised columns, and both meet the oracle; the release
    column gets exactly zero gradient"""
    import dasp_pytorch_b200 as D
    bs, n = 5, 6001
    g = torch.Generator().manual_seed(3)
    x = torch.rand(bs, 2, n, generator=g) * 2 - 1
    p01 = torch.rand(bs, 6, generator=g)
    p01[:, 4] = p01[:, 4].clamp(min=0.05)
    r = torch.randn(bs, 2, n, generator=g)
    ranges = list(COMP_RANGES)
    ranges[1] = (1.0, EXP_RATIO_MAX)
    proc = D.Expander(SR)
    assert list(proc.param_ranges.values()) == ranges
    xd = x.to(cuda_device).requires_grad_(True)
    pd = p01.to(cuda_device).requires_grad_(True)
    y = proc.process_normalized(xd, pd)
    (y * r.to(cuda_device)).sum().backward()
    assert float(pd.grad[:, 3].abs().max()) == 0.0
    cols = denorm(p01, ranges)
    y_fn = D.expander(xd.detach(), SR, *[c.to(cuda_device) for c in cols])
    assert peak_err(y.detach().cpu(), y_fn.cpu()).max() < 1e-5
    # d/d(p01) = span * d/d(physical)
    dp = [None if i == 3 else pd.grad[:, i].cpu() / (hi - lo) for i, (lo, hi) in enumerate(ranges)]
    pin("exp-process_normalized", "exp", x, cols, r, cuda_device, got=(y.detach().cpu(), xd.grad.cpu(), dp))


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16, torch.float64])
@pytest.mark.parametrize("kind", KINDS)
def test_other_dtypes(cuda_device, kind, dtype):
    """fp16 / bf16 / fp64 inputs run in fp32 and come back in their own dtype; a gradient reaches a low-precision x"""
    fn, _ = _fns(kind)
    x, params, _ = _inputs(kind, 3, 2, 3001, seed=9)
    p = [q.to(cuda_device) for q in params]
    xd = x.to(device=cuda_device, dtype=dtype).requires_grad_(True)
    y = fn(xd, SR, *p, lookahead_samples=5)
    assert y.dtype == dtype
    assert torch.equal(y, fn(xd.detach().float(), SR, *p, lookahead_samples=5).to(dtype))
    y.float().pow(2).sum().backward()
    assert xd.grad.dtype == dtype and torch.isfinite(xd.grad).all() and float(xd.grad.abs().max()) > 0


@pytest.mark.parametrize("la", [0, 5])
@pytest.mark.parametrize("bs,n", [(3, 0), (0, 100)])
@pytest.mark.parametrize("kind", KINDS)
def test_empty_shapes(cuda_device, kind, bs, n, la):
    """n = 0 or bs = 0 with requires_grad: empty dL/dx and zero parameter gradients, not an error"""
    fn, _ = _fns(kind)
    x = torch.zeros(bs, 2, n, device=cuda_device, requires_grad=True)
    p = [torch.full((bs,), v, device=cuda_device, requires_grad=True) for v in (-20.0, 2.0, 10.0, 50.0, 6.0, 3.0)]
    y = fn(x, SR, *p, lookahead_samples=la)
    assert y.shape == (bs, 2, n)
    y.sum().backward()
    assert x.grad.shape == (bs, 2, n)
    assert p[3].grad is None
    for q in p[:3] + p[4:]:
        assert q.grad.shape == (bs,) and float(q.grad.abs().sum()) == 0.0


@pytest.mark.parametrize("la", [0, 33])
@pytest.mark.parametrize("kind", KINDS)
def test_repeat_calls_bit_identical(cuda_device, kind, la):
    x, params, r = _inputs(kind, 4, 2, 9001, seed=12)
    a = gpu_run(kind, x, params, r, cuda_device, la=la)
    b = gpu_run(kind, x, params, r, cuda_device, la=la)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    assert all(torch.equal(u, v) for u, v in zip(a[2], b[2]) if u is not None)


# ------------------------------------------------------------------ 8. graph capture with look-ahead
def test_lookahead_graph_capture(cuda_device):
    """compressor forward + backward with lookahead_samples = 33 (g_scratch and the fix-up kernel inside the graph):
    a replay equals the eager step bit for bit, before and after new values in the captured input"""
    import dasp_pytorch_b200 as D
    x0, params, r = _inputs("comp", 4, 2, 8192, seed=13)
    x = x0.to(cuda_device).requires_grad_(True)
    p = [q.to(cuda_device).requires_grad_(True) for q in params]
    rd = r.to(cuda_device)
    leaves = [x] + p[:3] + p[4:]

    def step():
        y = D.compressor(x, SR, *p, lookahead_samples=33)
        (y * rd).sum().backward()
        return y

    def eager():
        for t in leaves:
            t.grad = None
        y = step()
        return [y.detach().clone()] + [t.grad.clone() for t in leaves]

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            eager()
    torch.cuda.current_stream().wait_stream(side)
    refs = [eager()]
    with torch.no_grad():
        x.mul_(0.5)
    refs.append(eager())
    with torch.no_grad():
        x.mul_(2.0)

    for t in leaves:
        t.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ys = step()
    for k, ref in enumerate(refs):
        if k == 1:
            with torch.no_grad():
                x.mul_(0.5)
        graph.replay()
        torch.cuda.synchronize()
        got = [ys] + [t.grad for t in leaves]
        assert all(torch.equal(a, b) for a, b in zip(got, ref)), k
