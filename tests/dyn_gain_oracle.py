"""fp64 restatement of compressor_gain / expander_gain for the tests.

The gain G (bs, 1, n) that oracle._dynamics multiplies into the (delayed) audio, or its dB value s + M, built from the
oracle's own pieces (attack coefficient, static curves, frequency-sampling and recursion smoothers).
tests/test_dynamics_gain_host.py checks that delay(x, la) * compressor_gain(x) equals oracle.compressor (and the same
for the expander), values and gradients."""
import torch

from oracle import dasp_oracle as O


def _gain(x, sample_rate, threshold_db, ratio, attack_ms, knee_db, makeup_gain_db, eps, curve, smoother, fsm_tail, db):
    bs = x.shape[0]
    side = x.sum(dim=1, keepdim=True)
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
    out = sm + m
    return out if db else torch.pow(10.0, out / 20.0)


def compressor_gain(x, sample_rate, threshold_db, ratio, attack_ms, release_ms, knee_db, makeup_gain_db, eps=1e-8,
                    smoother="fsm", fsm_tail=0, db=False):
    return _gain(x, sample_rate, threshold_db, ratio, attack_ms, knee_db, makeup_gain_db, eps, O._compressor_curve,
                 smoother, fsm_tail, db)


def expander_gain(x, sample_rate, threshold_db, ratio, attack_ms, release_ms, knee_db, makeup_gain_db, eps=1e-8,
                  smoother="fsm", fsm_tail=0, db=False):
    return _gain(x, sample_rate, threshold_db, ratio, attack_ms, knee_db, makeup_gain_db, eps, O._expander_curve,
                 smoother, fsm_tail, db)


def delay(x, la):
    """x[..., t - la], 0 for t < la: the compressor's look-ahead on the audio path"""
    if la == 0:
        return x
    out = torch.zeros_like(x)
    if la < x.shape[-1]:
        out[..., la:] = x[..., : x.shape[-1] - la]
    return out
