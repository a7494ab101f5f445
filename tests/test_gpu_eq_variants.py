"""Pin every parametric EQ kernel instantiation to the fp64 oracle.

biquad.cu instantiates eq_fwd_kernel<C, W, S> and eq_bwd_kernel<C, W, S> for
  C: the coefficient table type -- float when both rows of every pair belong to one item (even channel counts), float2
     (one coefficient per row) otherwise, or at any channel count under dasp_debug_eq_pair_tables(1);
  W: warps per row pair -- forward 1, 2, 3, 4, 8, 16; backward 1, 2, 3, 4, 8 (a forced 16 runs the backward at 8);
  S: load stages per warp -- dasp_debug_eq_fwd_stages / dasp_debug_eq_bwd_stages.  The backward's (8, 2) does not fit
     in shared memory and dispatch_bwd runs (8, 1) in its place (asserted from the profiler trace below).
Each (W, S) runs at three table configurations: float tables at 2 channels, pair tables forced at 2 channels (a pair
inside one item) and pair tables at 3 channels (pairs straddling two items, an odd row count, so the last pair has one
row).  Setup of test_gpu_eq.py::test_eq_every_warps_per_pair_variant: about three tiles per warp at W = 16, a ragged
last tile, the loss <y, r> with a fixed random cotangent r, strict 1e-4 per item against the alias-free oracle
(fsm_tail).  Every pin prints its errors ("PIN <case>: ...").
"""
import contextlib
import functools
import gc
import re

import pytest
import torch

import oracle
from helpers import EQ_INSTANTIATIONS, SR, denorm, eq_kernel_instantiations, eq_ranges, param_grad_err, peak_err

pytestmark = pytest.mark.gpu
TOL = 1e-4
TILE = 480                                   # dasp_eq_tile_len()
BS, N = 3, TILE * 16 * 3 + 100
VARIANTS = [(w, s) for w in (1, 2, 3, 4, 8, 16) for s in (1, 2)]
TABLES = {"float-2ch": (2, 0), "pair-2ch": (2, 1), "pair-3ch": (3, 0)}     # name -> (channels, pair-table hook)


def _lib():
    from dasp_pytorch_b200 import _abi
    return _abi.lib()


@contextlib.contextmanager
def eq_variant(w, s, pair_tables=0):
    lib = _lib()
    lib.dasp_debug_force_warps(w)
    lib.dasp_debug_eq_fwd_stages(s)
    lib.dasp_debug_eq_bwd_stages(s)
    lib.dasp_debug_eq_pair_tables(pair_tables)
    try:
        yield
    finally:
        lib.dasp_debug_force_warps(0)
        lib.dasp_debug_eq_fwd_stages(0)
        lib.dasp_debug_eq_bwd_stages(0)
        lib.dasp_debug_eq_pair_tables(0)


@functools.lru_cache(maxsize=None)
def _inputs(chs, n=N):
    g = torch.Generator().manual_seed(40 + chs)
    x = torch.rand(BS, chs, n, generator=g) * 2 - 1
    params = denorm(torch.rand(BS, 18, generator=g), eq_ranges())
    r = torch.randn(BS, chs, n, generator=g)
    return x, params, r


def _run(fn, x, params, r, device, dtype):
    """y, dL/dx, [dL/dparam] for L = <y, r>"""
    xx = x.to(device=device, dtype=dtype).clone().requires_grad_(True)
    pp = [p.to(device=device, dtype=dtype).clone().requires_grad_(True) for p in params]
    y = fn(xx, pp)
    (y * r.to(device=device, dtype=dtype)).sum().backward()
    return y.detach().cpu(), xx.grad.detach().cpu(), [p.grad.detach().cpu() for p in pp]


def gpu_run(x, params, r, device):
    import dasp_pytorch_b200 as D
    return _run(lambda xx, pp: D.parametric_eq(xx, SR, *pp), x, params, r, device, torch.float32)


@functools.lru_cache(maxsize=None)
def _oracle(chs):
    x, params, r = _inputs(chs)
    return _run(lambda xx, pp: oracle.parametric_eq(xx, SR, *pp, fsm_tail=1 << 16), x, params, r, "cpu", torch.float64)


def pin(case, chs, got):
    y, dx, dp = got
    y64, dx64, dp64 = _oracle(chs)
    errs = {"y": peak_err(y, y64), "dx": peak_err(dx, dx64), "dp": param_grad_err(dp, dp64)}
    print(f"PIN {case}: y {errs['y'].max():.2e} dx {errs['dx'].max():.2e} dparams {errs['dp'].max():.2e}")
    for k, e in errs.items():
        assert (e < TOL).all(), (case, k, e)


@pytest.mark.parametrize("table", list(TABLES))
@pytest.mark.parametrize("w,s", VARIANTS, ids=[f"W{w}-S{s}" for w, s in VARIANTS])
def test_every_eq_instantiation(cuda_device, w, s, table):
    chs, pair = TABLES[table]
    x, params, r = _inputs(chs)
    with eq_variant(w, s, pair):
        got = gpu_run(x, params, r, cuda_device)
    pin(f"eq-{table}-W{w}-S{s}-n{N}", chs, got)
    if table == "pair-2ch":
        # both rows of a pair share their item: the pair tables hold the float tables' coefficients twice, and every
        # product is the same fp32 FMA on the same numbers
        with eq_variant(w, s, 0):
            ref = gpu_run(x, params, r, cuda_device)
        assert torch.equal(got[0], ref[0]) and torch.equal(got[1], ref[1])
        assert all(torch.equal(a, b) for a, b in zip(got[2], ref[2]))


_PROF_PAT = re.compile(r"eq_(fwd|bwd)_kernel<(float2|float), (?:\(int\))?(\d+), (?:\(int\))?(\d+)>")


def test_every_eq_instantiation_is_launched(cuda_device):
    """the kernels the profiler sees: every instantiation the library holds, forward and backward, and the backward's
    (8, 2) request served by (8, 1)"""
    from torch.profiler import ProfilerActivity, profile
    from dasp_pytorch_b200 import _abi
    compiled = eq_kernel_instantiations(_abi.LIB_PATH)
    if compiled is not None:
        assert compiled == EQ_INSTANTIATIONS
    seen = {}
    for table, (chs, pair) in TABLES.items():
        x, params, r = _inputs(chs, n=TILE * 16 * 2 + 4)
        for w, s in VARIANTS:
            c = "float" if table == "float-2ch" else "float2"
            want = {("fwd", c, w, s), ("bwd", c, min(w, 8), 1 if w >= 8 else s)}
            got = set()
            for attempt in range(3):
                # A torch.profiler.profile object is a reference cycle, so the cyclic collector tears down earlier
                # sessions' objects, and a pass inside this window has been seen to drop the window's kernel records
                # although the kernels ran.  The collector stays off while recording.  The profiler has also been
                # seen to drop a short call's records with the collector off, so a capture that misses a record is
                # repeated (the same call, at most three times); a record of any other variant stays in the union,
                # where the equality below fails on it.
                gc.disable()
                try:
                    with profile(activities=[ProfilerActivity.CUDA]) as prof:
                        with eq_variant(w, s, pair):
                            gpu_run(x, params, r, cuda_device)
                        torch.cuda.synchronize()
                finally:
                    gc.enable()
                for e in prof.events():
                    m = _PROF_PAT.search(e.name)
                    if m:
                        got.add((m[1], m[2], int(m[3]), int(m[4])))
                if want <= got:
                    break
                print(f"profiler records incomplete for {table} W{w} S{s} ({sorted(want - got)} missing), repeating")
            assert got == want, (table, w, s, sorted(got))
            for k in got:
                seen[k] = seen.get(k, 0) + 1
    print("EQ instantiations launched: " + ", ".join(f"{k[0]}<{k[1]},{k[2]},{k[3]}>" for k in sorted(seen)))
    assert set(seen) == EQ_INSTANTIATIONS, (sorted(EQ_INSTANTIATIONS - set(seen)), sorted(set(seen) - EQ_INSTANTIATIONS))
