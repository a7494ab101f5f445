"""parametric_eq_frequency_response on the GPU: the response pinned per bin to the fp64 oracle
(tests/eq_response_oracle.py) on rfft, log and edge grids at 44.1 and 48 kHz, every one of the 18 gradients pinned per
item with the owned-parameter adjoint test of tests/param_grad_pin.py, the response equal to the spectrum of the
filter parametric_eq runs, the packed / unpacked / Processor entry points, and the edge cases: broadcasting, empty
batches and grids, dtypes, frequencies from either device, deterministic backward, graph replay, no saved state."""
import pytest
import torch

import param_grad_pin as pg
from eq_response_oracle import log_grid, parametric_eq_response
from helpers import denorm, eq_ranges

pytestmark = pytest.mark.gpu
FWD_TOL = 5e-5
BS = 72                      # four owners of each of the 18 parameters
CORNERS = [None, "low", "extreme", "zero_db"]


def _grids(sr):
    return {"rfft4096": torch.fft.rfftfreq(4096, 1 / sr, dtype=torch.float64),
            "rfft131072": torch.fft.rfftfreq(131072, 1 / sr, dtype=torch.float64),
            "log512": log_grid(sr),
            "edges": torch.tensor([0.0, sr / 2], dtype=torch.float64)}


def _params(sr, corner, seed=5, bs=BS):
    _, params, own, alt = pg.eq_inputs(bs, 1, 1, seed, sr=sr, corner=corner)
    return params, own, alt


@pytest.mark.parametrize("sr", [44100, 48000])
@pytest.mark.parametrize("corner", CORNERS)
def test_response_pinned_to_oracle(cuda_device, sr, corner):
    import dasp_pytorch_b200 as D
    params, _, _ = _params(sr, corner)
    pp = [p.to(cuda_device) for p in params]
    worst = {}
    for name, f in _grids(sr).items():
        h = D.parametric_eq_frequency_response(sr, *pp, frequencies=f).cpu()
        ref = parametric_eq_response(sr, *[p.double() for p in params], frequencies=f)
        assert h.dtype == torch.complex64 and h.shape == ref.shape
        err = (h.to(torch.complex128) - ref).abs() / ref.abs()
        worst[name] = float(err.max())
        assert worst[name] <= FWD_TOL, (name, worst[name], divmod(int(err.argmax()), f.numel()))
    print(f"EQRESP sr {sr} corner {corner}: " + " ".join(f"{k} {v:.2e}" for k, v in worst.items()))


@pytest.mark.parametrize("sr", [44100, 48000])
@pytest.mark.parametrize("corner", CORNERS)
@pytest.mark.parametrize("grid", ["rfft4096", "log512"])
def test_gradients_pinned_to_oracle(cuda_device, sr, corner, grid):
    import dasp_pytorch_b200 as D
    params, own, alt = _params(sr, corner, seed=7)
    f = _grids(sr)[grid]
    fn = lambda xx, pp, s: torch.view_as_real(parametric_eq_response(sr, *pp, frequencies=f))
    y64 = fn(None, [p.double() for p in params], None)
    v = pg.owned_columns(fn, y64, params, own)
    v_alt = pg.owned_columns(fn, y64, alt, own) if alt is not None else None
    c, r, zero = pg.cotangent(v, y64, v_alt)
    pp = [p.to(cuda_device).clone().requires_grad_(True) for p in params]
    h = D.parametric_eq_frequency_response(sr, *pp, frequencies=f.to(cuda_device))
    (torch.view_as_real(h) * c.to(cuda_device)).sum().backward()
    pg.check(f"eq_response sr {sr} {corner} {grid}", pg.EQ_NAMES, own, pg.owned([p.grad.cpu() for p in pp], own),
             r, zero)


@pytest.mark.parametrize("sr", [44100, 48000])
def test_response_is_the_filter_parametric_eq_runs(cuda_device, sr):
    """rfft of the EQ's impulse response at 65536 samples is the op at rfftfreq(65536), for items whose impulse
    response has died out inside those samples (every draw of the ParametricEQ ranges away from the 20 Hz corner)"""
    import dasp_pytorch_b200 as D
    n = 65536
    params, _, _ = _params(sr, None, seed=9, bs=16)
    pp = [p.to(cuda_device) for p in params]
    x = torch.zeros(16, 1, n, device=cuda_device)
    x[:, :, 0] = 1.0
    spec = torch.fft.rfft(D.parametric_eq(x, sr, *pp)[:, 0].double()).cpu()
    f = torch.fft.rfftfreq(n, 1 / sr, dtype=torch.float64)
    h = D.parametric_eq_frequency_response(sr, *pp, frequencies=f).cpu().to(torch.complex128)
    # the items that qualify: the fp64 response's impulse response has no energy left in the second half of the window
    ref = parametric_eq_response(sr, *[p.double() for p in params], frequencies=f)
    ir = torch.fft.irfft(ref, n)
    keep = ir[:, n // 2:].abs().amax(1) <= 1e-9 * ir.abs().amax(1)
    assert int(keep.sum()) >= 12, keep
    err = (spec - h).abs().amax(1) / h.abs().amax(1)
    assert float(err[keep].max()) <= 1e-4, err


def test_packed_unpacked_and_processor_agree(cuda_device):
    import dasp_pytorch_b200 as D
    sr = 44100
    g = torch.Generator().manual_seed(12)
    p01 = torch.rand(8, 18, generator=g)
    p01[0, 1] = 0.0
    cols = denorm(p01, eq_ranges(sr))
    f = log_grid(sr).to(cuda_device)
    pp = [c.to(cuda_device) for c in cols]
    a = D.parametric_eq_frequency_response(sr, *pp, frequencies=f)
    b = D.parametric_eq_frequency_response_packed(sr, torch.stack(pp, 1), f)
    assert torch.equal(a, b)
    proc = D.ParametricEQ(sr)
    q = p01.to(cuda_device).requires_grad_(True)
    hp = proc.frequency_response(q, f)
    err = (hp - a).abs() / a.abs()
    assert hp.dtype == torch.complex64 and float(err.max()) <= FWD_TOL
    hp.abs().pow(2).sum().backward()
    assert q.grad is not None and q.grad.shape == q.shape and bool(torch.isfinite(q.grad).all())
    assert float(q.grad.abs().max()) > 0
    bad = p01.clone()
    bad[3, 7] = 1.5
    x = torch.zeros(8, 1, 64, device=cuda_device)
    with pytest.raises(ValueError) as e1:
        proc.process_normalized(x, bad.to(cuda_device))
    with pytest.raises(ValueError) as e2:
        proc.frequency_response(bad.to(cuda_device), f)
    assert str(e1.value) == str(e2.value) and "band1_cutoff_freq" in str(e2.value)


def test_broadcast_parameters(cuda_device):
    import dasp_pytorch_b200 as D
    sr, bs = 48000, 5
    params, _, _ = _params(sr, None, seed=3, bs=bs)
    full = [p.to(cuda_device) for p in params]
    mixed = [p if k % 2 else p[:1].reshape(1, 1) for k, p in enumerate(full)]
    expanded = [p if k % 2 else p[:1].expand(bs) for k, p in enumerate(full)]
    f = _grids(sr)["rfft4096"]
    pm = [p.clone().requires_grad_(True) for p in mixed]
    a = D.parametric_eq_frequency_response(sr, *pm, frequencies=f)
    b = D.parametric_eq_frequency_response(sr, *expanded, frequencies=f)
    assert a.shape == (bs, f.numel()) and torch.equal(a.detach(), b)
    a.abs().sum().backward()
    assert all(p.grad.shape == p.shape and bool(torch.isfinite(p.grad).all()) for p in pm)


def test_empty_batch_and_empty_grid(cuda_device):
    import dasp_pytorch_b200 as D
    f = torch.linspace(0, 22050, 7, dtype=torch.float64)
    p0 = [torch.zeros(0, device=cuda_device, requires_grad=True) for _ in range(18)]
    h = D.parametric_eq_frequency_response(44100, *p0, frequencies=f)
    assert h.shape == (0, 7) and h.dtype == torch.complex64
    h.abs().sum().backward()
    assert all(p.grad.shape == (0,) for p in p0)
    params, _, _ = _params(44100, None, bs=3)
    pp = [p.to(cuda_device).requires_grad_(True) for p in params]
    h = D.parametric_eq_frequency_response(44100, *pp, frequencies=torch.zeros(0))
    assert h.shape == (3, 0)
    h.abs().sum().backward()
    assert all(torch.equal(p.grad, torch.zeros_like(p)) for p in pp)


def test_dtypes_and_frequency_devices(cuda_device):
    import dasp_pytorch_b200 as D
    sr = 44100
    params, _, _ = _params(sr, "extreme", bs=4)
    f64 = log_grid(sr)
    ref = D.parametric_eq_frequency_response(sr, *[p.to(cuda_device) for p in params], frequencies=f64)
    for f in (f64.to(cuda_device), f64.float(), f64.float().to(cuda_device)):
        h = D.parametric_eq_frequency_response(sr, *[p.to(cuda_device) for p in params], frequencies=f)
        want = D.parametric_eq_frequency_response(sr, *[p.to(cuda_device) for p in params],
                                                  frequencies=f.double().cpu())
        assert torch.equal(h, want)
    assert torch.equal(D.parametric_eq_frequency_response(sr, *[p.to(cuda_device) for p in params],
                                                          frequencies=f64.to(cuda_device)), ref)
    bf = [p.to(cuda_device, torch.bfloat16).requires_grad_(True) for p in params]
    hb = D.parametric_eq_frequency_response(sr, *bf, frequencies=f64)
    assert hb.dtype == torch.complex64
    assert torch.equal(hb.detach(), D.parametric_eq_frequency_response(
        sr, *[p.detach().float() for p in bf], frequencies=f64))
    hb.abs().sum().backward()
    assert all(p.grad.dtype == torch.bfloat16 for p in bf)
    d = [p.to(cuda_device, torch.float64).requires_grad_(True) for p in params]
    hd = D.parametric_eq_frequency_response(sr, *d, frequencies=f64)
    assert hd.dtype == torch.complex128 and torch.equal(hd.detach(), ref.to(torch.complex128))
    hd.abs().sum().backward()
    assert all(p.grad.dtype == torch.float64 for p in d)
    hp = D.parametric_eq_frequency_response_packed(sr, torch.stack(d, 1).detach(), f64)
    assert hp.dtype == torch.complex128


def test_backward_is_deterministic_and_graph_replays(cuda_device):
    from dasp_pytorch_b200 import functional as F
    sr = 48000
    params, _, _ = _params(sr, "low", bs=6)
    p = torch.stack(params, 1).to(cuda_device).requires_grad_(True)
    f = _grids(sr)["rfft131072"].to(cuda_device)
    w = torch.randn(6, f.numel(), 2, device=cuda_device, generator=torch.Generator(cuda_device).manual_seed(0))

    def step():
        h = F.parametric_eq_frequency_response_packed(sr, p, f)
        (torch.view_as_real(h) * w).sum().backward()
        return h

    def eager():
        p.grad = None
        h = step()
        return h.detach().clone(), p.grad.clone()

    first, second = eager(), eager()
    assert torch.equal(first[1], second[1]) and torch.equal(first[0], second[0])
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            eager()
    torch.cuda.current_stream().wait_stream(side)
    p.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        hs = step()
    with torch.no_grad():
        p.grad.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(hs.detach(), first[0]) and torch.equal(p.grad, first[1])


def test_fixed_parameters_keep_nothing(cuda_device):
    import dasp_pytorch_b200 as D
    params, _, _ = _params(44100, None, bs=4)
    f = log_grid(44100)
    packs = []
    with torch.autograd.graph.saved_tensors_hooks(lambda t: packs.append(t) or t, lambda t: t):
        h = D.parametric_eq_frequency_response(44100, *[p.to(cuda_device) for p in params], frequencies=f)
        assert h.grad_fn is None and not packs
        pg_ = [p.to(cuda_device).requires_grad_(k == 4) for k, p in enumerate(params)]
        h2 = D.parametric_eq_frequency_response(44100, *pg_, frequencies=f)
    assert torch.equal(h, h2.detach()) and h2.grad_fn is not None
    # the op keeps the packed parameters and the fp64 frequencies, nothing per bin
    assert sorted((tuple(t.shape), str(t.dtype)) for t in packs) == [((4, 18), "torch.float32"),
                                                                     ((f.numel(),), "torch.float64")]
