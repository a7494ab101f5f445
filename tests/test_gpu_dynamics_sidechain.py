"""Pin the compressor / expander with an external side chain (key) to the fp64 oracle.

dynamics.cu instantiates dynamics_sc_fwd_kernel and dynamics_sc_bwd_kernel over curve {Compress, Expand} x warps per
item W {1, 2, 4, 8, 16} x look-ahead: 40 kernels.  A forced W that does not fit shared memory is halved by pick_warps,
so every case asserts the W it covers through dasp_dynamics_sidechain_tile_len.  n % 4 == 0 streams the tiles with TMA,
any other n with cooperative copies.  The arbiter is tests/dyn_sidechain_oracle.py (oracle._dynamics with the detector
on the key) on the enlarged frequency-sampling grid, with the metrics and tolerances of test_gpu_dynamics_pin.py and the
loss <y, r>.
"""
import re

import pytest
import torch

import dyn_sidechain_oracle as sco
from helpers import SR, param_grad_err, peak_err
from test_gpu_dynamics_pin import (E, EXP_RATIO_MAX, KINDS, PGRAD_TOL, TOL, WARPS, _params, forced_warps, fsm_tail,
                                   _lib)

pytestmark = pytest.mark.gpu


def _fns(kind):
    import dasp_pytorch_b200 as D
    return (D.sidechain_compressor, sco.compressor) if kind == "comp" else (D.sidechain_expander, sco.expander)


def sc_tile_len(bs, chs, kc):
    return int(_lib().dasp_dynamics_sidechain_tile_len(bs, chs, kc))


def _inputs(kind, bs, chs, kc, n, seed):
    g = torch.Generator().manual_seed(seed)
    level = 0.05 + 0.95 * torch.rand(bs, 1, 1, generator=g)
    x = (torch.rand(bs, chs, n, generator=g) * 2 - 1) * level
    key = (torch.rand(bs, kc, n, generator=g) * 2 - 1) * (0.05 + 0.95 * torch.rand(bs, 1, 1, generator=g))
    return x, key, _params(kind, bs, g), torch.randn(bs, chs, n, generator=g)


def _run(fn, x, key, params, r, device, dtype, grads=("x", "key", "p")):
    """y, dL/dx, dL/dkey, [dL/dparam] for L = <y, r>; only the leaves named in grads require a gradient"""
    xx = x.to(device=device, dtype=dtype).clone().requires_grad_("x" in grads)
    kk = key.to(device=device, dtype=dtype).clone().requires_grad_("key" in grads)
    pp = [p.to(device=device, dtype=dtype).clone().requires_grad_("p" in grads) for p in params]
    y = fn(xx, kk, pp)
    if y.requires_grad:
        (y * r.to(device=device, dtype=dtype)).sum().backward()
    cpu = lambda t: None if t is None else t.detach().cpu()
    return cpu(y), cpu(xx.grad), cpu(kk.grad), [cpu(p.grad) for p in pp]


def gpu_run(kind, x, key, params, r, device, eps=1e-8, la=0, grads=("x", "key", "p"), dtype=torch.float32):
    gpu, _ = _fns(kind)
    return _run(lambda xx, kk, pp: gpu(xx, SR, *pp, eps=eps, lookahead_samples=la, sidechain=kk), x, key, params, r,
                device, dtype, grads)


def oracle_run(kind, x, key, params, r, eps=1e-8, la=0):
    _, orc = _fns(kind)
    tail = fsm_tail(SR, float(params[2].max()))
    return _run(lambda xx, kk, pp: orc(xx, SR, *pp, eps=eps, lookahead_samples=la, fsm_tail=tail, sidechain=kk),
                x, key, params, r, "cpu", torch.float64)


def pin(case, kind, x, key, params, r, device, eps=1e-8, la=0, got=None):
    got = got or gpu_run(kind, x, key, params, r, device, eps, la)
    y, dx, dk, dp = got
    y64, dx64, dk64, dp64 = oracle_run(kind, x, key, params, r, eps, la)
    assert dp[3] is None and dp64[3] is None                      # release_ms: no gradient
    for t in [y, dx, dk] + [d for d in dp if d is not None]:
        assert torch.isfinite(t).all(), case
    assert torch.equal(dk, dk[:, :1].expand_as(dk))                # every key channel gets the same dL/dside
    errs = {"y": peak_err(y, y64), "dx": peak_err(dx, dx64), "dk": peak_err(dk, dk64), "dp": param_grad_err(dp, dp64)}
    print(f"PIN {case}: " + " ".join(f"{k} {v.max():.2e}" for k, v in errs.items()))
    for k in ("y", "dx", "dk"):
        assert (errs[k] < TOL).all(), (case, k, errs[k])
    assert (errs["dp"] < PGRAD_TOL).all(), (case, errs["dp"])
    return got


# ------------------------------------------------------------------ 1. instantiation matrix
CK = [(2, 1), (1, 2), (2, 2), (3, 1)]


def fits(w, chs, kc):
    """three backward stages of 2C + K tiles fit in 96 KB (200 KB at W = 16): pick_warps keeps a forced W"""
    return 3 * (2 * chs + kc) * w * 32 * E * 4 + 512 <= (200 if w == 16 else 96) * 1024


def _matrix():
    """per (kind, W): every (C, K) of CK whose stages fit at that W (at W = 8 and 16 only (1, 2) does, so (1, 1) is
    added there), each without and with a look-ahead between one and two tiles; TMA and cooperative copies alternate
    along the list"""
    cases = []
    for kind in KINDS:
        for w in WARPS:
            for j, (chs, kc) in enumerate([ck for ck in CK if fits(w, *ck)] + ([(1, 1)] if w >= 8 else [])):
                for la in (False, True):
                    pipe = ("tma", "coop")[(j + la) % 2]
                    cases.append(pytest.param(kind, w, chs, kc, la, pipe,
                                              id=f"{kind}-W{w}-C{chs}K{kc}-{'la1.5T' if la else 'la0'}-{pipe}"))
    return cases


@pytest.mark.parametrize("kind,w,chs,kc,la,pipe", _matrix())
def test_instantiation_matrix(cuda_device, kind, w, chs, kc, la, pipe):
    bs, T = 3, w * 32 * E
    n = 2 * T + (36 if pipe == "tma" else 37)
    la = T + T // 2 + 5 if la else 0
    x, key, params, r = _inputs(kind, bs, chs, kc, n, seed=100 * w + 10 * chs + kc + la)
    with forced_warps(w):
        assert sc_tile_len(bs, chs, kc) == T
        pin(f"{kind}-W{w}-C{chs}K{kc}-la{la}-n{n}", kind, x, key, params, r, cuda_device, la=la)


def test_every_instantiation_is_launched(cuda_device):
    from torch.profiler import ProfilerActivity, profile
    bs, chs, kc = 3, 1, 1
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for kind in KINDS:
            for w in WARPS:
                T = w * 32 * E
                x, key, params, r = _inputs(kind, bs, chs, kc, T + 5, seed=w)
                for la in (0, T + 1):
                    with forced_warps(w):
                        assert sc_tile_len(bs, chs, kc) == T
                        gpu_run(kind, x, key, params, r, cuda_device, la=la)
        torch.cuda.synchronize()
    names = {e.name for e in prof.events() if "dynamics_sc_" in e.name}
    pat = re.compile(r"dynamics_sc_(fwd|bwd)_kernel<(.+?), (\d+), (true|false)>")
    seen = set()
    for name in names:
        mt = pat.search(name)
        if mt:
            curve = "comp" if ("Compress" in mt[2] or mt[2].endswith("0")) else "exp"
            seen.add((mt[1], curve, int(mt[3]), mt[4] == "true"))
    want = {(d, k, w, la) for d in ("fwd", "bwd") for k in KINDS for w in WARPS for la in (False, True)}
    assert want <= seen, (sorted(want - seen), sorted(names))


# ------------------------------------------------------------------ 2. reduction to today's op
@pytest.mark.parametrize("la", [0, 29])
@pytest.mark.parametrize("kind", KINDS)
def test_sidechain_x_reduces_to_the_plain_op(cuda_device, monkeypatch, kind, la):
    """sidechain=x: y bit-identical to the generic channel loop of the plain op; x.grad (gain path + detector path
    through the key) matches the plain op's dL/dx"""
    import dasp_pytorch_b200 as D
    fn, sc = (D.compressor, D.sidechain_compressor) if kind == "comp" else (D.expander, D.sidechain_expander)
    x0, _, params, r = _inputs(kind, 4, 2, 1, 9001, seed=21)
    x0 = x0.to(cuda_device)
    p = [q.to(cuda_device) for q in params]
    rd = r.to(cuda_device)
    monkeypatch.setenv("DASP_DYN_GENERIC", "1")
    xa = x0.clone().requires_grad_(True)
    ya = fn(xa, SR, *p, lookahead_samples=la)
    (ya * rd).sum().backward()
    xb = x0.clone().requires_grad_(True)
    yb = sc(xb, SR, *p, lookahead_samples=la, sidechain=xb)
    (yb * rd).sum().backward()
    assert torch.equal(ya, yb)
    rel = (xb.grad - xa.grad).abs().max() / xa.grad.abs().max()
    print(f"REDUCE {kind} la{la}: y bit-identical, x.grad rel {float(rel):.2e}")
    assert rel <= 1e-6


# ------------------------------------------------------------------ 3. edges
@pytest.mark.parametrize("kind", KINDS)
def test_key_silent_in_stretches(cuda_device, kind):
    """exact digital zero in the key: the expander attenuates fully there, and dL/dkey is exactly 0 (|side| < eps)"""
    x, key, params, r = _inputs(kind, 3, 2, 2, 6000, seed=3)
    for a, b in ((0, 500), (2000, 3500), (5800, 6000)):
        key[:, :, a:b] = 0
    if kind == "exp":
        params[1] = torch.full((3,), EXP_RATIO_MAX)
        params[0] = torch.full((3,), -30.0)
    _, _, dk, _ = pin(f"{kind}-silent-key", kind, x, key, params, r, cuda_device)
    for a, b in ((0, 500), (2000, 3500), (5800, 6000)):
        assert float(dk[:, :, a:b].abs().max()) == 0.0


LA_EDGES = {"1": lambda T, n: 1, "T": lambda T, n: T, "n-1": lambda T, n: n - 1, "n": lambda T, n: n,
            "n+1": lambda T, n: n + 1}


@pytest.mark.parametrize("la_name", list(LA_EDGES))
@pytest.mark.parametrize("kind", KINDS)
def test_lookahead_edges(cuda_device, kind, la_name):
    bs, w = 3, 2
    T = w * 32 * E
    n = 3 * T + 13
    la = LA_EDGES[la_name](T, n)
    x, key, params, r = _inputs(kind, bs, 1, 2, n, seed=la)
    with forced_warps(w):
        assert sc_tile_len(bs, 1, 2) == T
        if la < n:
            pin(f"{kind}-la{la_name}={la}", kind, x, key, params, r, cuda_device, la=la)
            return
        y, dx, dk, dp = gpu_run(kind, x, key, params, r, cuda_device, la=la)
    # the audio path is delayed past its end: y and dL/dx are exactly 0 (dL/dx written in full, not left empty)
    assert float(y.abs().max()) == 0.0 and float(dx.abs().max()) == 0.0
    assert float(dk.abs().max()) == 0.0 and all(float(d.abs().max()) == 0.0 for d in dp if d is not None)


@pytest.mark.parametrize("grads", [("x",), ("key",), ("p",), ("x", "p")])
def test_partial_gradients(cuda_device, grads):
    """a fixed key writes no key gradient; whatever is requested matches the full run bit for bit"""
    x, key, params, r = _inputs("comp", 3, 2, 1, 5001, seed=8)
    full = gpu_run("comp", x, key, params, r, cuda_device, la=7)
    part = gpu_run("comp", x, key, params, r, cuda_device, la=7, grads=grads)
    assert torch.equal(full[0], part[0])
    assert (part[1] is not None) == ("x" in grads) and (part[2] is not None) == ("key" in grads)
    if "x" in grads:
        assert torch.equal(full[1], part[1])
    if "key" in grads:
        assert torch.equal(full[2], part[2])
    if "p" in grads:
        assert all(torch.equal(a, b) for a, b in zip(full[3], part[3]) if a is not None)


def test_widest_channel_combination(cuda_device):
    """2C + K = 76 runs on one warp with the full 200 KB of stages; 77 raises before any launch"""
    import dasp_pytorch_b200 as D
    assert sc_tile_len(3, 32, 12) == 32 * E and sc_tile_len(3, 32, 13) == 0
    x, key, params, r = _inputs("comp", 3, 32, 12, 3001, seed=76)
    pin("comp-C32K12", "comp", x, key, params, r, cuda_device)
    xx = x.to(cuda_device).requires_grad_(True)
    p = [q.to(cuda_device) for q in params]
    with pytest.raises(ValueError, match="exceeds 76"):
        D.sidechain_compressor(xx, SR, *p, sidechain=torch.zeros(3, 13, 3001, device=cuda_device))
    f = xx.detach()
    rc = _lib().dasp_dynamics_sidechain_fwd(0, f.data_ptr(), f.data_ptr(), 13, *[q.data_ptr() for q in p[:3] + p[4:]],
                                            f.data_ptr(), None, 3, 32, 3001, float(SR), 1e-8, 0, None)
    assert rc == -1


def test_bf16_inputs(cuda_device):
    """bf16 x and key compute in fp32; y and both gradients come back in bf16"""
    x, key, params, r = _inputs("comp", 3, 2, 1, 4000, seed=16)
    y, dx, dk, _ = gpu_run("comp", x, key, params, r, cuda_device, dtype=torch.bfloat16)
    assert y.dtype == dx.dtype == dk.dtype == torch.bfloat16
    yf = gpu_run("comp", x.bfloat16().float(), key.bfloat16().float(), [p.bfloat16().float() for p in params],
                 r.bfloat16().float(), cuda_device, grads=())[0]
    assert torch.equal(y, yf.bfloat16())
    assert torch.isfinite(dk.float()).all() and float(dk.float().abs().max()) > 0


@pytest.mark.parametrize("la", [0, 5])
@pytest.mark.parametrize("bs,n", [(3, 0), (0, 100)])
def test_empty_shapes(cuda_device, bs, n, la):
    import dasp_pytorch_b200 as D
    x = torch.zeros(bs, 2, n, device=cuda_device, requires_grad=True)
    key = torch.zeros(bs, 1, n, device=cuda_device, requires_grad=True)
    p = [torch.full((bs,), v, device=cuda_device, requires_grad=True) for v in (-20.0, 2.0, 10.0, 50.0, 6.0, 3.0)]
    y = D.sidechain_compressor(x, SR, *p, lookahead_samples=la, sidechain=key)
    assert y.shape == (bs, 2, n)
    y.sum().backward()
    assert x.grad.shape == (bs, 2, n) and key.grad.shape == (bs, 1, n)
    assert p[3].grad is None
    for q in p[:3] + p[4:]:
        assert q.grad.shape == (bs,) and float(q.grad.abs().sum()) == 0.0


# ------------------------------------------------------------------ 4. de-esser composition, ducking, modules
def test_deesser_composition(cuda_device):
    """compressor keyed by a presence-boosted EQ copy of x; gradients reach the EQ parameters and match the oracle
    composition"""
    import dasp_pytorch_b200 as D
    import oracle
    from helpers import eq_ranges, denorm
    bs, chs, n = 3, 2, 8192
    g = torch.Generator().manual_seed(11)
    x = (torch.rand(bs, chs, n, generator=g) * 2 - 1) * 0.5
    eqp = denorm(torch.rand(bs, 18, generator=g), eq_ranges())
    eqp[9] = torch.full((bs,), 12.0)                          # band2 +12 dB around 8-12 kHz: the sibilance band
    cp = _params("comp", bs, g)
    r = torch.randn(bs, chs, n, generator=g)
    tail = max(fsm_tail(SR, float(cp[2].max())), 1 << 16)

    def run(eq, comp, device, dtype, **kw):
        xx = x.to(device=device, dtype=dtype).clone().requires_grad_(True)
        ee = [p.to(device=device, dtype=dtype).clone().requires_grad_(True) for p in eqp]
        cc = [p.to(device=device, dtype=dtype).clone().requires_grad_(True) for p in cp]
        key = eq(xx, SR, *ee, **kw)
        y = comp(xx, SR, *cc, sidechain=key, **kw)
        (y * r.to(device=device, dtype=dtype)).sum().backward()
        return y.detach().cpu(), xx.grad.cpu(), torch.stack([e.grad.cpu() for e in ee], 1)

    y, dx, de = run(D.parametric_eq, D.sidechain_compressor, cuda_device, torch.float32)
    y64, dx64, de64 = run(oracle.parametric_eq, sco.compressor, "cpu", torch.float64, fsm_tail=tail)
    ey, edx = peak_err(y, y64), peak_err(dx, dx64)
    ede = ((de - de64).abs().amax(1) / de64.abs().amax(1))
    print(f"DEESSER y {ey.max():.2e} dx {edx.max():.2e} dEQ {ede.max():.2e}")
    assert (ey < TOL).all() and (edx < TOL).all() and (ede < 1e-3).all()


def test_ducking_window(cuda_device):
    """a key loud only in [a, b): the gain drops there and stays at the makeup gain before a; after b it recovers
    within the attack tail"""
    import dasp_pytorch_b200 as D
    bs, n, a, b = 2, 48000, 20000, 30000
    x = torch.rand(bs, 2, n, device=cuda_device) * 0.2 + 0.1           # positive: G = y / x
    key = torch.zeros(bs, 1, n, device=cuda_device)
    key[:, :, a:b] = 0.9
    p = [torch.full((bs,), v, device=cuda_device) for v in (-20.0, 8.0, 10.0, 50.0, 2.0, 0.0)]
    G = (D.sidechain_compressor(x, SR, *p, sidechain=key) / x)[:, 0]
    assert float((G[:, :a] - 1).abs().max()) < 1e-6
    assert float(G[:, a + 2000:b].max()) < 0.5                            # well into the window: ducked
    tail = int(SR * 10e-3 * 8)                                           # eight attack time constants
    assert float((G[:, b + tail:] - 1).abs().max()) < 1e-3


def test_process_normalized_with_key(cuda_device):
    """Compressor.process_normalized(x, p, sidechain=key) on the packed path equals sidechain_compressor() on the
    denormalised columns, and so does the by-name path with a caller's process_fn"""
    import dasp_pytorch_b200 as D
    from helpers import COMP_RANGES, denorm
    bs, n = 4, 5000
    x = torch.rand(bs, 2, n, device=cuda_device) - 0.5
    key = torch.rand(bs, 1, n, device=cuda_device) - 0.5
    p01 = torch.rand(bs, 6, device=cuda_device)
    proc = D.Compressor(SR)
    y = proc.process_normalized(x, p01, sidechain=key)
    ref = D.sidechain_compressor(x, SR, *[c.to(cuda_device) for c in denorm(p01.cpu(), COMP_RANGES)], sidechain=key)
    assert peak_err(y.cpu(), ref.cpu()).max() < 1e-5
    assert not torch.equal(y, proc.process_normalized(x, p01))
    proc.process_fn = lambda *a, **k: D.sidechain_compressor(*a, **k)    # not the kernel entry: the by-name path
    y2 = proc.process_normalized(x, p01, sidechain=key)
    assert peak_err(y2.cpu(), ref.cpu()).max() < 1e-5


# ------------------------------------------------------------------ 5. reproducibility and graph capture
def test_repeat_calls_and_graph_capture(cuda_device):
    import dasp_pytorch_b200 as D
    x0, k0, params, r = _inputs("exp", 4, 2, 1, 8192, seed=13)
    a = gpu_run("exp", x0, k0, params, r, cuda_device, la=33)
    b = gpu_run("exp", x0, k0, params, r, cuda_device, la=33)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and torch.equal(a[2], b[2])
    assert all(torch.equal(u, v) for u, v in zip(a[3], b[3]) if u is not None)

    x = x0.to(cuda_device).requires_grad_(True)
    key = k0.to(cuda_device).requires_grad_(True)
    p = [q.to(cuda_device).requires_grad_(True) for q in params]
    rd = r.to(cuda_device)
    leaves = [x, key] + p[:3] + p[4:]

    def step():
        y = D.sidechain_expander(x, SR, *p, lookahead_samples=33, sidechain=key)
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
    ref = eager()
    for t in leaves:
        t.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ys = step()
    graph.replay()
    torch.cuda.synchronize()
    got = [ys] + [t.grad for t in leaves]
    assert all(torch.equal(u, v) for u, v in zip(got, ref))
