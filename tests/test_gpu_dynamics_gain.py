"""Pin compressor_gain / expander_gain to the fp64 oracle, and hold them bit for bit to the gain the compressor and
expander apply.

dynamics.cu instantiates the gain kernels for curve {Compress, Expand} x warps per item W {1, 2, 4, 8, 16}, forward and
backward; the dB output is a runtime flag of the same kernels.  A forced W that does not fit shared memory for the
compressor's backward (2C tile buffers per stage) is halved by pick_warps exactly as for the compressor, so each case
derives the W it covers from dasp_dynamics_tile_len.  Values: linear G to 1e-4 relative per item, the dB curve to 1e-3
dB absolute.  Gradients: dL/dx to 1e-4 relative per item, each of the five parameters to 1e-4 on its own scale
(tests/param_grad_pin.py's owned-parameter method).  Every pin prints its errors ("PIN <case>: ...").
"""
import re

import pytest
import torch

import dyn_gain_oracle as go
import param_grad_pin as pg
from helpers import SR, param_grad_err, peak_err
from test_gpu_dynamics_pin import E, KINDS, WARPS, forced_warps, fsm_tail, tile_len
from test_gpu_param_grads import _run_launched

pytestmark = pytest.mark.gpu
TOL = 1e-4
DB_TOL = 1e-3
CHANNELS = (1, 2, 3, 8, 32)


def _D():
    import dasp_pytorch_b200 as D
    return D


def _gpu_fn(kind):
    D = _D()
    return D.compressor_gain if kind == "comp" else D.expander_gain


def _orc_fn(kind):
    return go.compressor_gain if kind == "comp" else go.expander_gain


def fitted_warps(w, chs):
    """the W pick_warps keeps of a forced w: halved until three stages of the compressor backward's 2C buffers fit in
    96 KB (200 KB at W = 16)"""
    while w > 1 and 3 * 2 * chs * w * 32 * E * 4 + 512 > (200 if w == 16 else 96) * 1024:
        w //= 2
    return w


def _matrix():
    """every (kind, C, W) a forced W reaches for C in CHANNELS, alternating TMA and cooperative copies"""
    cases = sorted({(kind, c, fitted_warps(w, c)) for kind in KINDS for c in CHANNELS for w in WARPS})
    return [pytest.param(k, c, w, ("tma", "coop")[i % 2], id=f"{k}-C{c}-W{w}-{('tma', 'coop')[i % 2]}")
            for i, (k, c, w) in enumerate(cases)]


def _inputs(kind, bs, chs, n, seed):
    """x, the six parameters with the threshold within 6 dB of each item's median side-chain level (so that no owned
    column is zero), and the owners"""
    x, params, own = pg.dyn_inputs(kind, bs, chs, n, seed)
    side = x.sum(1).abs().median(1).values
    g = torch.Generator().manual_seed(seed + 99)
    params[0] = (20 * torch.log10(side) + torch.rand(bs, generator=g) * 12 - 6).float()
    return x, params, own


def _oracle(kind, params, eps, db):
    tail = fsm_tail(SR, float(params[2].max()))
    return lambda xx, pp, s: _orc_fn(kind)(xx, SR, *pp, eps=eps, db=db, fsm_tail=tail)


def pin(case, kind, x, params, own, device, db, eps=1e-8, db_tol=DB_TOL):
    """GPU gain, dL/dx and the owned parameter gradients against the fp64 oracle; returns (GPU result, value error)"""
    orc = _oracle(kind, params, eps, db)
    v = pg.owned_columns(orc, x, params, own)
    c, r, zero = pg.cotangent(v, x)
    y64, dx64, _ = pg.vjp(orc, x, params, c, torch.float64)
    fn = _gpu_fn(kind)
    y, dx, dp = pg.gpu_grads(lambda xx, pp: fn(xx, SR, *pp, eps=eps, db=db), x, params, c, device)
    assert y.shape == (x.shape[0], 1, x.shape[2]) and dp[3] is None
    for t in [y, dx] + [d for d in dp if d is not None]:
        assert torch.isfinite(t).all(), case
    verr = (y.double() - y64).reshape(x.shape[0], -1).abs().amax(1) if db else peak_err(y, y64)
    dxerr = peak_err(dx, dx64)
    print(f"PIN {case}: {'dB abs' if db else 'G rel'} {verr.max():.2e} dx {dxerr.max():.2e}")
    assert (verr < (db_tol if db else TOL)).all(), (case, verr)
    assert (dxerr < TOL).all(), (case, dxerr)
    assert torch.equal(dx, dx[:, :1].expand_as(dx))                    # every channel gets the same dL/dside
    pg.check(case, pg.DYN_NAMES, own, pg.owned(dp, own), r, zero)
    return (y, dx, dp), verr


# ------------------------------------------------------------------ 1. values and gradients, every kernel and C
@pytest.mark.parametrize("kind,chs,w,pipe", _matrix())
def test_gain_matrix(cuda_device, kind, chs, w, pipe):
    bs, T = 5, w * 32 * E
    n = 3 * T + (36 if pipe == "tma" else 37)
    x, params, own = _inputs(kind, bs, chs, n, seed=100 * chs + w)
    with forced_warps(w):
        assert tile_len(bs, chs) == T
        for db in (False, True):
            pin(f"{kind}-C{chs}-W{w}-{pipe}-{'db' if db else 'lin'}", kind, x, params, own, cuda_device, db)


_GAIN_PAT = re.compile(r"dynamics_gain_(fwd|bwd)_kernel<(.+?), (\d+)>")


def _gain_launched(names):
    """{(direction, curve, W)} of the gain kernels among the launched kernel names"""
    out = set()
    for m in map(_GAIN_PAT.search, names):
        if m:
            out.add((m[1], "comp" if ("Compress" in m[2] or m[2].endswith("0")) else "exp", int(m[3])))
    return out


@pytest.mark.parametrize("db", [False, True])
@pytest.mark.parametrize("w", WARPS)
@pytest.mark.parametrize("kind", KINDS)
def test_every_gain_kernel_is_launched(cuda_device, kind, w, db):
    """the profiler sees exactly the forward and backward gain kernel of (curve, W), linear and dB"""
    bs, n = 4, 2 * w * 32 * E + 12
    g = torch.Generator().manual_seed(w)
    x = ((torch.rand(bs, 1, n, generator=g) * 2 - 1) * 0.5).to(cuda_device).requires_grad_(True)
    p = [t.to(cuda_device) for t in pg.dyn_inputs(kind, bs, 1, n, seed=w)[1]]
    fn = _gpu_fn(kind)

    def call():
        y = fn(x, SR, *p, db=db)
        (gx,) = torch.autograd.grad(y.sum(), x)
        torch.cuda.synchronize()
        return gx

    with forced_warps(w):
        assert tile_len(bs, 1) == w * 32 * E
        want = {(d, kind, w) for d in ("fwd", "bwd")}
        _, got = _run_launched(call, _gain_launched, want)
    assert got == want, sorted(got)


# ------------------------------------------------------------------ 2. bit identity with the processors
def _procs(kind):
    D = _D()
    return (D.compressor, D.compressor_gain) if kind == "comp" else (D.expander, D.expander_gain)


@pytest.mark.parametrize("chs", CHANNELS)
@pytest.mark.parametrize("kind", KINDS)
def test_processor_is_delay_times_gain(cuda_device, kind, chs):
    """proc(x, la) == delay(x, la) * gain(x) bit for bit, for la in {0, 1, tile_len + 1, n - 1}; and the gradients of
    the composition agree with the processor's within the pin tolerance"""
    proc, gain = _procs(kind)
    bs = 4
    T = tile_len(bs, chs)
    n = 3 * T + 20
    x, params, _ = _inputs(kind, bs, chs, n, seed=7 * chs)
    xd = x.to(cuda_device)
    pd = [p.to(cuda_device) for p in params]
    G = gain(xd, SR, *pd)
    for la in (0, 1, T + 1, n - 1):
        y = proc(xd, SR, *pd, lookahead_samples=la)
        assert torch.equal(y, go.delay(xd, la) * G), (kind, chs, la)
    r = torch.randn(bs, chs, n, generator=torch.Generator().manual_seed(chs)).to(cuda_device)
    for la in (0, T + 1):
        grads = []
        for compose in (False, True):
            xx = xd.clone().requires_grad_(True)
            pp = [p.clone().requires_grad_(True) for p in pd]
            y = go.delay(xx, la) * gain(xx, SR, *pp) if compose else proc(xx, SR, *pp, lookahead_samples=la)
            (y * r).sum().backward()
            grads.append([xx.grad.cpu()] + [p.grad.cpu() for i, p in enumerate(pp) if i != 3])
        ref, got = grads
        assert (peak_err(got[0], ref[0]) < TOL).all(), (kind, chs, la)
        assert (param_grad_err(got[1:], ref[1:]) < TOL).all(), (kind, chs, la)


# ------------------------------------------------------------------ 3. edge cases
def test_silent_stretches_get_no_gradient(cuda_device):
    """where |side| < eps, dL/dx is exactly 0 in every channel; elsewhere the op is pinned as usual"""
    bs, chs, n = 5, 2, 9000
    x, params, own = _inputs("comp", bs, chs, n, seed=3)
    x[:, :, 2000:4000] = 0.0
    x[:, 1, 6000:7000] = -x[:, 0, 6000:7000]                  # the channels cancel: side == 0 exactly
    for db in (False, True):
        (_, dx, _), _ = pin(f"silent-{'db' if db else 'lin'}", "comp", x, params, own, cuda_device, db)
        assert torch.all(dx[:, :, 2000:4000] == 0) and torch.all(dx[:, :, 6000:7000] == 0)
        assert torch.all(dx[:, :, :2000].abs().amax(-1) > 0)


def test_expander_ratio_20_on_silence(cuda_device):
    """an expander at ratio 20 on silence: the dB curve is finite and pinned, the linear gain underflows to 0 there,
    and every gradient stays finite.  The curve reaches about -3000 dB, where one fp32 ulp is 2.4e-4 dB, so the dB
    bar is 1e-3 dB plus 1e-6 of the item's largest |dB| (about eight ulps)"""
    bs, chs, n = 5, 2, 12000
    x, params, own = _inputs("exp", bs, chs, n, seed=4)
    x[:, :, 4000:9000] = 0.0
    params[1] = torch.full((bs,), 20.0)
    peak = _oracle("exp", params, 1e-8, True)(x.double(), [p.double() for p in params], None).abs().amax((1, 2))
    (ydb, _, _), err = pin("exp-ratio20-db", "exp", x, params, own, cuda_device, True, db_tol=DB_TOL + 1e-6 * peak)
    assert ydb.min() < -1500
    D = _D()
    xx = x.to(cuda_device).requires_grad_(True)
    pp = [p.to(cuda_device).requires_grad_(True) for p in params]
    G = D.expander_gain(xx, SR, *pp)
    assert torch.all(G[ydb.to(cuda_device) < -1000] == 0) and bool((G[..., 8000:9000] == 0).all())
    (G * torch.randn_like(G)).sum().backward()
    assert torch.isfinite(xx.grad).all() and all(torch.isfinite(p.grad).all() for i, p in enumerate(pp) if i != 3)


def test_broadcast_dtypes_and_empty(cuda_device):
    D = _D()
    bs, chs, n = 3, 2, 5000
    x, params, _ = _inputs("comp", bs, chs, n, seed=5)
    xd = x.to(cuda_device)
    one = [p[:1].to(cuda_device) for p in params]
    full = [p[:1].expand(bs).to(cuda_device) for p in params]
    for fn in (D.compressor_gain, D.expander_gain):
        for db in (False, True):
            ref = fn(xd, SR, *full, db=db)
            assert torch.equal(fn(xd, SR, *one, db=db), ref)
            assert torch.equal(fn(xd, SR, *[float(p) for p in one], db=db), ref)
            for dt in (torch.bfloat16, torch.float64):
                got = fn(xd.to(dt), SR, *full, db=db)
                assert got.dtype == dt
                assert torch.equal(got, fn(xd.to(dt).float(), SR, *full, db=db).to(dt))
    for shape in ((0, 2, 100), (3, 2, 0)):
        xx = torch.zeros(shape, device=cuda_device, requires_grad=True)
        pp = [torch.zeros(shape[0], device=cuda_device, requires_grad=True) + 1 for _ in range(6)]
        G = D.compressor_gain(xx, SR, *pp)
        assert G.shape == (shape[0], 1, shape[2])
        G.sum().backward()
        assert xx.grad.shape == shape and bool((xx.grad == 0).all())


def test_no_checkpoint_without_gradients(cuda_device):
    """metering: without a gradient to compute the op allocates its output and nothing else; with one, the
    smoother checkpoint as well"""
    D = _D()
    x, params, _ = _inputs("comp", 4, 2, 48000, seed=6)
    xd = x.to(cuda_device)
    pd = [p.to(cuda_device) for p in params]
    D.compressor_gain(xd, SR, *pd)                                          # load the library, warm up
    count = lambda: torch.cuda.memory_stats(cuda_device)["allocation.all.allocated"]
    a = count()
    G = D.compressor_gain(xd, SR, *pd)
    assert count() - a == 1
    pg_ = [p.clone().requires_grad_(True) for p in pd]
    a = count()
    G = D.compressor_gain(xd, SR, *pg_)
    assert count() - a == 2 and G.requires_grad


def test_backward_is_deterministic(cuda_device):
    D = _D()
    x, params, _ = _inputs("exp", 6, 3, 20000, seed=8)
    out = []
    for _ in range(2):
        xx = x.to(cuda_device).requires_grad_(True)
        pp = [p.to(cuda_device).requires_grad_(True) for p in params]
        G = D.expander_gain(xx, SR, *pp, db=True)
        (G * torch.linspace(-1, 1, G.shape[-1], device=cuda_device)).sum().backward()
        out.append([xx.grad.clone()] + [p.grad.clone() for i, p in enumerate(pp) if i != 3])
    assert all(torch.equal(a, b) for a, b in zip(*out))


def test_cuda_graph_replay(cuda_device):
    D = _D()
    x, params, _ = _inputs("comp", 4, 2, 10000, seed=9)
    xd = x.to(cuda_device)
    pd = [p.to(cuda_device) for p in params]
    eager = [D.compressor_gain(xd, SR, *pd, db=db) for db in (False, True)]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for db in (False, True):
            D.compressor_gain(xd, SR, *pd, db=db)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs = [D.compressor_gain(xd, SR, *pd, db=db) for db in (False, True)]
    graph.replay()
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(outs, eager))


def test_processor_gain_curve(cuda_device):
    D = _D()
    bs, chs, n = 4, 2, 6000
    x = (torch.rand(bs, chs, n, generator=torch.Generator().manual_seed(10)) * 2 - 1).to(cuda_device)
    p01 = torch.rand(bs, 6, generator=torch.Generator().manual_seed(11)).to(cuda_device)
    for proc, fn in ((D.Compressor(SR), D.compressor_gain), (D.Expander(SR), D.expander_gain)):
        lo = torch.tensor([r[0] for r in proc.param_ranges.values()], device=cuda_device)
        hi = torch.tensor([r[1] for r in proc.param_ranges.values()], device=cuda_device)
        phys = p01 * (hi - lo) + lo
        for db in (False, True):
            got = proc.gain_curve(x, p01, db=db)
            ref = fn(x, SR, *phys.t(), db=db)
            torch.testing.assert_close(got, ref, rtol=1e-5, atol=1e-5 if db else 1e-7)
        y = proc.process_normalized(x, p01)
        torch.testing.assert_close(y, x * proc.gain_curve(x, p01), rtol=0, atol=0)
        p = p01.clone().requires_grad_(True)
        proc.gain_curve(x, p).sum().backward()
        assert p.grad is not None and torch.isfinite(p.grad).all()
        bad = p01.clone()
        bad[1, 2] = 1.5
        with pytest.raises(ValueError, match="Parameter attack_ms of is out of range"):
            proc.gain_curve(x, bad)
