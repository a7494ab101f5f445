"""The fp64 oracle on the GPU, for rows of minutes, long impulse responses and high sample rates.

The oracle functions are plain torch, so on CUDA fp64 tensors they run on cuFFT in double precision with no project
kernel involved.  At 2^24 points and with autograd that is seconds where the CPU takes many minutes.  This module moves
inputs there and results back, picks the frequency-sampling grid extension (``fsm_tail``) from the longest time
constant of the filters involved, and guards the device memory a test may take.
tests/test_long_oracle_host.py checks on the CPU that the tailed oracle equals the scipy fp64 recursions at the
lengths and rates used.
"""
import math

import numpy as np
import pytest
import torch

import oracle
from helpers import param_grad_err, peak_err

TOL = 1e-4
BUDGET = 40 << 30          # device bytes one test may take
DECAY = 1e-13              # the impulse response left past the grid, relative to its start


def need_memory(nbytes, device):
    """skip, naming the bytes, unless `nbytes` are free on `device` now; no case may plan for more than BUDGET"""
    free, _ = torch.cuda.mem_get_info(device)
    if nbytes > BUDGET:
        raise AssertionError(f"case needs {nbytes} B, above the {BUDGET} B budget")
    if free < nbytes:
        pytest.skip(f"needs {nbytes} B of device memory, {free} B free")


def peak():
    """device memory peak since the last call, as text for the PIN line ('' without CUDA)"""
    if not torch.cuda.is_initialized():
        return ""
    gb = torch.cuda.max_memory_allocated() / (1 << 30)
    torch.cuda.reset_peak_memory_stats()
    return f" (peak {gb:.1f} GB)"


def release():
    if torch.cuda.is_initialized():
        torch.cuda.synchronize()
        torch.cuda.empty_cache()


def _tail(radius):
    """samples until radius^t (times t, for a double pole) falls below DECAY, as a power of two (at least 2^16)"""
    r = float(radius)
    if r <= 0.0:
        return 1 << 16
    need = math.log(DECAY) / math.log(r)
    need *= 1.0 + math.log(max(need, 2.0)) / abs(math.log(DECAY))      # the t r^t envelope of a repeated pole
    return max(1 << 16, 1 << math.ceil(math.log2(need)))


def eq_pole_radius(sample_rate, params):
    """the largest pole magnitude of the 6 sections of every item (fp64, from the oracle's own design)"""
    sos = oracle.eq_sections(sample_rate, [torch.as_tensor(p).double().cpu() for p in params]).numpy()
    a1, a2 = sos[..., 4], sos[..., 5]
    disc = a1 * a1 - 4.0 * a2
    real = disc >= 0
    sq = np.sqrt(np.abs(disc))
    r_real = np.maximum(np.abs(-a1 + sq), np.abs(-a1 - sq)) / 2.0
    r_cplx = np.sqrt(np.abs(a2))
    return float(np.where(real, r_real, r_cplx).max())


def eq_tail(sample_rate, params):
    """fsm_tail of oracle.parametric_eq that makes the slowest section's impulse response die out inside the grid"""
    return _tail(eq_pole_radius(sample_rate, params))


def dyn_tail(sample_rate, attack_ms_max):
    """fsm_tail of the one-pole smoother at the longest attack (as test_gpu_dynamics_pin.fsm_tail)"""
    return _tail(math.exp(-math.log(9.0) / (sample_rate * attack_ms_max * 1e-3)))


def vjp(fn, x, params, c, device, group=None, dtype=torch.float64):
    """y, dL/dx, [dL/dparam] of L = <fn(x, params), c> in `dtype` on `device`, `group` items at a time (batch first;
    every parameter holds one element per item); results on the CPU"""
    bs = x.shape[0]
    group = group or bs
    ys, dxs, dps = [], [], []
    for a in range(0, bs, group):
        s = slice(a, min(bs, a + group))
        xx = x[s].to(device=device, dtype=dtype).requires_grad_(True)
        pp = [p[s].to(device=device, dtype=dtype).requires_grad_(True) for p in params]
        y = fn(xx, pp)
        (y * c[s].to(device=device, dtype=dtype)).sum().backward()
        ys.append(y.detach().cpu())
        dxs.append(xx.grad.cpu())
        dps.append([None if p.grad is None else p.grad.cpu() for p in pp])
        del xx, pp, y
        release()
    dp = [None if dps[0][j] is None else torch.cat([d[j] for d in dps]) for j in range(len(params))]
    return torch.cat(ys), torch.cat(dxs), dp


def pin(case, got, ref, tol=TOL, names=("y", "dx")):
    """hold (y, dL/dx, [dL/dparam]) to the fp64 result per item: peak_err for the tensors, param_grad_err for the
    parameters (an op without an input x passes None for dL/dx); prints the PIN line and returns the worst errors"""
    errs = {k: peak_err(a, b) for k, a, b in zip(names, got[:2], ref[:2]) if b is not None}
    if any(d is not None for d in ref[2]):
        errs["dp"] = param_grad_err(got[2], ref[2])
    for t in [a for a in got[:2] if a is not None] + [d for d in got[2] if d is not None]:
        assert bool(torch.isfinite(t).all()), case
    worst = {k: float(e.max()) for k, e in errs.items()}
    print(f"PIN {case}: " + " ".join(f"{k} {v:.2e}" for k, v in worst.items()) + peak())
    for k, e in errs.items():
        assert bool((e <= tol).all()), (case, k, e.tolist())
    return worst


def pin_tensors(case, named, tol=TOL):
    """hold each (name, got, fp64) to peak_err per item (batch first), print the PIN line, return the worst errors"""
    errs = {}
    for name, a, b in named:
        assert bool(torch.isfinite(a).all()), (case, name)
        errs[name] = peak_err(a, b)
    worst = {k: float(e.max()) for k, e in errs.items()}
    print(f"PIN {case}: " + " ".join(f"{k} {v:.2e}" for k, v in worst.items()) + peak())
    for k, e in errs.items():
        assert bool((e <= tol).all()), (case, k, e.tolist())
    return worst


def param_vjp(fn, params, c, device, dtype=torch.float64):
    """y, None, [dL/dparam] of L = <fn(params), c> for an op whose only inputs are its parameters (in `dtype`)"""
    pp = [p.to(device=device, dtype=dtype).requires_grad_(True) for p in params]
    y = fn(pp)
    (y * c.to(device=device, dtype=dtype)).sum().backward()
    out = y.detach().cpu(), None, [None if p.grad is None else p.grad.cpu() for p in pp]
    del pp, y
    release()
    return out


def gpu(fn, x, params, c, device):
    """y, dL/dx, [dL/dparam] of L = <fn(x, params), c> through the project's kernels (fp32), results on the CPU"""
    xx = x.to(device=device, dtype=torch.float32).requires_grad_(True)
    pp = [p.to(device=device, dtype=torch.float32).requires_grad_(True) for p in params]
    y = fn(xx, pp)
    (y * c.to(device)).sum().backward()
    out = y.detach().cpu(), xx.grad.cpu(), [None if p.grad is None else p.grad.cpu() for p in pp]
    del xx, pp, y
    release()
    return out
