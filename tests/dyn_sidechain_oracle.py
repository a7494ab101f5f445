"""fp64 restatement of the compressor / expander with an external side chain (key), for the tests.

The reference has no side-chain input.  This is oracle._dynamics with one change: the detector reads
side = (x if sidechain is None else sidechain).sum(dim=1), while the gain is still applied to (the delayed) x.  It is
built from the oracle's own pieces (attack coefficient, static curves, frequency-sampling smoother), and
tests/test_dynamics_sidechain_host.py checks that with sidechain=x it equals oracle.compressor / oracle.expander,
values and gradients."""
import torch

from oracle import dasp_oracle as O


def _dynamics(x, sample_rate, threshold_db, ratio, attack_ms, knee_db, makeup_gain_db, eps, lookahead_samples, curve,
              smoother, fsm_tail=0, sidechain=None):
    bs, chs, n = x.shape
    side = (x if sidechain is None else sidechain).sum(dim=1, keepdim=True)
    t = threshold_db.reshape(bs, 1, 1)
    r = ratio.reshape(bs, 1, 1)
    w = knee_db.reshape(bs, 1, 1)
    m = makeup_gain_db.reshape(bs, 1, 1)
    alpha = O._attack_coefficient(attack_ms.reshape(bs, 1, 1), sample_rate)
    level_db = 20.0 * torch.log10(side.abs().clamp(min=eps))
    gc = curve(level_db, t, r, w)
    if smoother == "recursion":
        sm = O.one_pole_recursion_truth(gc, alpha).to(x.dtype)
    else:
        sm = O._one_pole_fsm(gc, alpha, fsm_tail)
    if lookahead_samples > 0:                               # the audio path only; the key is not delayed
        delayed = torch.zeros_like(x)
        if lookahead_samples < n:
            delayed[..., lookahead_samples:] = x[..., : n - lookahead_samples]
        x = delayed
    return x * torch.pow(10.0, (sm + m) / 20.0)


def compressor(x, sample_rate, threshold_db, ratio, attack_ms, release_ms, knee_db, makeup_gain_db, eps=1e-8,
               lookahead_samples=0, smoother="fsm", fsm_tail=0, sidechain=None):
    return _dynamics(x, sample_rate, threshold_db, ratio, attack_ms, knee_db, makeup_gain_db, eps, lookahead_samples,
                     O._compressor_curve, smoother, fsm_tail, sidechain)


def expander(x, sample_rate, threshold_db, ratio, attack_ms, release_ms, knee_db, makeup_gain_db, eps=1e-8,
             lookahead_samples=0, smoother="fsm", fsm_tail=0, sidechain=None):
    return _dynamics(x, sample_rate, threshold_db, ratio, attack_ms, knee_db, makeup_gain_db, eps, lookahead_samples,
                     O._expander_curve, smoother, fsm_tail, sidechain)
