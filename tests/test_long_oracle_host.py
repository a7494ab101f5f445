"""The arbiter of the long-form and high-rate pins (tests/long_oracle.py), checked on the CPU: at 2^20 samples and
192 kHz, the frequency-sampling oracle with the tail long_oracle picks equals the fp64 scipy recursion, for the EQ's
least well-damped corner (20 Hz low shelf, 80 Hz band 0, Q 0.1 and 6, +-20 dB) and for the 100 ms attack smoother."""
import pytest
import torch

import long_oracle
import oracle
from helpers import eq_ranges

N = 1 << 20
SR = 192000


def _eq_corner_params(bs):
    """item b: low shelf 20 Hz / band 0 80 Hz at Q 0.1 or 6 and +-20 dB, every other band mid-range"""
    lo = [a for a, _ in eq_ranges(SR)]
    hi = [b for _, b in eq_ranges(SR)]
    params = [torch.full((bs,), 0.5 * (a + b)) for a, b in zip(lo, hi)]
    for b in range(bs):
        q, g = (0.1, 6.0)[b % 2], (-20.0, 20.0)[(b // 2) % 2]
        params[0][b], params[1][b], params[2][b] = g, 20.0, q
        params[3][b], params[4][b], params[5][b] = -g, 80.0, q
    return [p.double() for p in params]


def test_eq_tail_matches_recursion_at_192k():
    params = _eq_corner_params(4)
    tail = long_oracle.eq_tail(SR, params)
    assert tail >= 1 << 16
    x = torch.rand(4, 1, N, generator=torch.Generator().manual_seed(0), dtype=torch.float64) * 2 - 1
    y = oracle.parametric_eq(x, SR, *params, fsm_tail=tail)
    yt = oracle.parametric_eq(x, SR, *params, method="recursion")
    err = ((y - yt).abs().amax(-1) / yt.abs().amax(-1)).max()
    print(f"eq 192 kHz n=2^20 tail={tail}: fsm vs recursion {float(err):.2e}")
    assert float(err) < 1e-9


@pytest.mark.parametrize("kind", ["comp", "exp"])
def test_smoother_tail_matches_recursion_at_192k(kind):
    g = torch.Generator().manual_seed(1)
    x = (torch.rand(2, 2, N, generator=g, dtype=torch.float64) * 2 - 1) * 0.5
    params = [torch.tensor([-30.0, -20.0]), torch.tensor([4.0, 3.0]), torch.tensor([100.0, 5.0]),
              torch.tensor([50.0, 50.0]), torch.tensor([6.0, 3.0]), torch.tensor([2.0, 0.0])]
    params = [p.double() for p in params]
    fn = oracle.compressor if kind == "comp" else oracle.expander
    tail = long_oracle.dyn_tail(SR, 100.0)
    y = fn(x, SR, *params, fsm_tail=tail)
    yt = fn(x, SR, *params, smoother="recursion")
    err = ((y - yt).abs().amax(-1) / yt.abs().amax(-1)).max()
    print(f"{kind} 192 kHz 100 ms n=2^20 tail={tail}: fsm vs recursion {float(err):.2e}")
    assert float(err) < 1e-9
