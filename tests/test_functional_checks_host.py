"""CPU characterisation of every op's input checks: for each public op of ``functional`` and its packed twin, the
exception type and the exact message each malformed input raises before the first CUDA requirement, including the
"no CPU path" errors themselves.  Cases with two faults pin which check fires first."""
import pytest
import torch

import dasp_pytorch_b200 as D
from dasp_pytorch_b200 import functional as F
from dasp_pytorch_b200.functional import DaspError

SR = 48000
NO_CPU = "dasp_pytorch_b200 only runs on CUDA (H100) tensors and has no CPU path"
X_CPU = f"x is on cpu: {NO_CPU}"
X_SHAPE = "x must be a tensor of shape (batch, channels, samples)"


def z(*shape, **kw):
    return torch.zeros(*shape, **kw)


def meta(*shape):
    return torch.zeros(*shape, device="meta")


def params(counts, bad=None):
    """one tensor per element count; ``bad`` maps positions to replacement tensors"""
    ps = [z(c) for c in counts]
    for i, t in (bad or {}).items():
        ps[i] = t
    return ps


def eq(x, counts=(2,) * 18, bad=None):
    return F.parametric_eq(x, SR, *params(counts, bad))


def eq_response(counts=(2,) * 18, bad=None, sr=SR, freqs=None):
    return F.parametric_eq_frequency_response(sr, *params(counts, bad), z(5) if freqs is None else freqs)


def reverb(x, counts=(2,) * 25, bad=None, taps=31, noise=None):
    return F.noise_shaped_reverberation(x, SR, *params(counts, bad), num_samples=64, num_bandpass_taps=taps,
                                        noise=noise)


def nsir(counts=(2,) * 24, bad=None, sr=SR, L=64, taps=31, noise=None):
    return F.noise_shaped_impulse_response(sr, *params(counts, bad), num_samples=L, num_bandpass_taps=taps,
                                           noise=noise)


def dyn(fn, x, counts=(2,) * 6, bad=None, **kw):
    return fn(x, SR, *params(counts, bad), **kw)


# (id, call, exception type, exact message)
CASES = [
    # gain, distortion
    ("gain-rank", lambda: F.gain(z(2, 8), SR, z(2)), ValueError, X_SHAPE),
    ("gain-not-tensor", lambda: F.gain([[[0.0]]], SR, z(1)), ValueError, X_SHAPE),
    ("gain-cpu", lambda: F.gain(z(2, 1, 8), SR, z(2)), DaspError, X_CPU),
    ("gain-cpu-int-badparam", lambda: F.gain(z(2, 1, 8, dtype=torch.int32), SR, z(3)), DaspError, X_CPU),
    ("distortion-rank", lambda: F.distortion(z(8), SR, z(1)), ValueError, X_SHAPE),
    ("distortion-cpu-badparam", lambda: F.distortion(z(2, 2, 8), SR, z(3)), DaspError, X_CPU),
    # stereo mixing
    ("widener-rank", lambda: F.stereo_widener(z(2, 8), SR, z(2)), ValueError, "x must be a 3-dimensional tensor"),
    ("widener-cpu-3ch", lambda: F.stereo_widener(z(2, 3, 8), SR, z(2)), DaspError, X_CPU),
    ("panner-rank", lambda: F.stereo_panner(z(2, 2, 2, 8), SR, z(4)), ValueError, "x must be a 3-dimensional tensor"),
    ("panner-cpu-badparam", lambda: F.stereo_panner(z(2, 3, 8), SR, z(2)), DaspError, X_CPU),
    ("bus-rank", lambda: F.stereo_bus(z(2, 2, 8), SR, z(2)), ValueError, "x must be a 4-dimensional tensor"),
    ("bus-not-tensor", lambda: F.stereo_bus(None, SR, z(2)), ValueError, "x must be a 4-dimensional tensor"),
    ("bus-cpu-3ch", lambda: F.stereo_bus(z(2, 3, 2, 8), SR, z(4)), DaspError, X_CPU),
    # parametric EQ
    ("eq-rank", lambda: eq(z(2, 8)), ValueError, X_SHAPE),
    ("eq-cpu", lambda: eq(z(2, 1, 8)), DaspError, X_CPU),
    ("eq-cpu-badparam", lambda: eq(z(2, 1, 8), bad={4: z(3)}), DaspError, X_CPU),
    ("eq-packed-rank", lambda: F.parametric_eq_packed(z(2, 8), SR, z(2, 18)), ValueError, X_SHAPE),
    ("eq-packed-cpu-badshape", lambda: F.parametric_eq_packed(z(2, 1, 8), SR, z(2, 17)), DaspError, X_CPU),
    # compressor / expander
    ("comp-rank", lambda: dyn(F.compressor, z(2, 8)), ValueError, X_SHAPE),
    ("comp-cpu", lambda: dyn(F.compressor, z(2, 1, 8)), DaspError, X_CPU),
    ("comp-cpu-badparam", lambda: dyn(F.compressor, z(2, 1, 8), bad={0: z(3)}), DaspError, X_CPU),
    ("exp-cpu-badrelease", lambda: dyn(F.expander, z(2, 1, 8), bad={3: z(3)}), DaspError, X_CPU),
    ("dyn-packed-rank", lambda: F.dynamics_packed(0, z(2, 8), SR, z(2, 6)), ValueError, X_SHAPE),
    ("dyn-packed-cpu-badshape", lambda: F.dynamics_packed(1, z(2, 1, 8), SR, z(2, 5)), DaspError, X_CPU),
    # side chain
    ("sc-key-rank-x-rank", lambda: dyn(F.sidechain_compressor, z(2, 8), sidechain=z(2, 8)), ValueError,
     "sidechain must be a tensor of shape (batch, key_channels, samples)"),
    ("sc-x-rank", lambda: dyn(F.sidechain_compressor, z(2, 8), sidechain=z(2, 1, 8)), ValueError, X_SHAPE),
    ("sc-batch", lambda: dyn(F.sidechain_compressor, z(2, 1, 8), sidechain=z(3, 1, 8)), ValueError,
     "sidechain has shape (3, 1, 8): its batch and length must equal x's (2, 8)"),
    ("sc-length-and-keychs", lambda: dyn(F.sidechain_expander, z(2, 1, 8), sidechain=z(2, 33, 9)), ValueError,
     "sidechain has shape (2, 33, 9): its batch and length must equal x's (2, 8)"),
    ("sc-keychs-0", lambda: dyn(F.sidechain_compressor, z(2, 1, 8), sidechain=z(2, 0, 8)), ValueError,
     "sidechain: 1 to 32 key channels are supported, got 0"),
    ("sc-keychs-33-and-buffers", lambda: dyn(F.sidechain_compressor, z(2, 30, 8), sidechain=z(2, 33, 8)), ValueError,
     "sidechain: 1 to 32 key channels are supported, got 33"),
    ("sc-buffers", lambda: dyn(F.sidechain_expander, z(2, 30, 8), sidechain=z(2, 17, 8)), ValueError,
     "sidechain: 2 * 30 channels + 17 key channels exceeds 76"),
    ("sc-key-device", lambda: dyn(F.sidechain_compressor, z(2, 1, 8), sidechain=meta(2, 1, 8)), DaspError,
     "sidechain is on meta but x is on cpu"),
    ("sc-key-cpu-before-x", lambda: dyn(F.sidechain_compressor, z(2, 1, 8), sidechain=z(2, 1, 8)), DaspError,
     f"sidechain is on cpu: {NO_CPU}"),
    ("sc-none-is-plain", lambda: dyn(F.sidechain_expander, z(2, 1, 8), sidechain=None), DaspError, X_CPU),
    ("sc-packed-batch", lambda: F.dynamics_packed(0, z(2, 1, 8), SR, z(2, 5), sidechain=z(1, 1, 8)), ValueError,
     "sidechain has shape (1, 1, 8): its batch and length must equal x's (2, 8)"),
    ("sc-packed-key-cpu", lambda: F.dynamics_packed(1, z(2, 1, 8), SR, z(2, 5), sidechain=z(2, 2, 8)), DaspError,
     f"sidechain is on cpu: {NO_CPU}"),
    # the dynamics gain curve: parameters are checked against x before x's device
    ("gain-curve-rank", lambda: dyn(F.compressor_gain, z(2, 8), bad={0: z(3)}), ValueError, X_SHAPE),
    ("gain-curve-chs-0", lambda: dyn(F.compressor_gain, z(2, 0, 8)), ValueError,
     "x: 1 to 32 channels are supported, got 0"),
    ("gain-curve-chs-33-badparam", lambda: dyn(F.expander_gain, z(2, 33, 8), bad={0: z(3)}), ValueError,
     "x: 1 to 32 channels are supported, got 33"),
    ("gain-curve-threshold", lambda: dyn(F.compressor_gain, z(2, 1, 8), bad={0: z(3)}), RuntimeError,
     "threshold_db: expected 2 element(s) (one per batch item), got 3"),
    ("gain-curve-ratio-and-makeup", lambda: dyn(F.compressor_gain, z(2, 1, 8), bad={1: z(3), 5: z(4)}), RuntimeError,
     "ratio: expected 2 element(s) (one per batch item), got 3"),
    ("gain-curve-makeup-before-release", lambda: dyn(F.expander_gain, z(2, 1, 8), bad={3: z(3), 5: z(4)}),
     RuntimeError, "makeup_gain_db: expected 2 element(s) (one per batch item), got 4"),
    ("gain-curve-release", lambda: dyn(F.expander_gain, z(2, 1, 8), bad={3: z(3)}), RuntimeError,
     "release_ms: expected 2 element(s) (one per batch item), got 3"),
    ("gain-curve-param-device", lambda: dyn(F.compressor_gain, z(2, 1, 8), bad={2: meta(2)}), DaspError,
     "attack_ms is on meta but x is on cpu"),
    ("gain-curve-cpu", lambda: dyn(F.compressor_gain, z(2, 1, 8), counts=(1,) * 6), DaspError, X_CPU),
    ("gain-curve-cpu-numbers", lambda: F.expander_gain(z(2, 1, 8), SR, -20.0, 4.0, 10.0, 50.0, 6.0, 0.0, db=True),
     DaspError, X_CPU),
    ("gain-curve-packed-rank", lambda: F.dynamics_gain_packed(0, z(2, 8), SR, z(2, 5)), ValueError, X_SHAPE),
    ("gain-curve-packed-chs-33-badshape", lambda: F.dynamics_gain_packed(0, z(2, 33, 8), SR, z(2, 5)), ValueError,
     "x: 1 to 32 channels are supported, got 33"),
    ("gain-curve-packed-cols", lambda: F.dynamics_gain_packed(0, z(2, 1, 8), SR, z(2, 5)), ValueError,
     "params: expected a (2, 6) parameter tensor, got (2, 5)"),
    ("gain-curve-packed-batch", lambda: F.dynamics_gain_packed(1, z(2, 1, 8), SR, z(3, 6)), ValueError,
     "params: expected a (2, 6) parameter tensor, got (3, 6)"),
    ("gain-curve-packed-rank1", lambda: F.dynamics_gain_packed(1, z(2, 1, 8), SR, z(12)), ValueError,
     "params: expected a (2, 6) parameter tensor, got (12,)"),
    ("gain-curve-packed-list", lambda: F.dynamics_gain_packed(1, z(2, 1, 8), SR, [[0.0] * 6] * 2), ValueError,
     "params: expected a (2, 6) parameter tensor, got ()"),
    ("gain-curve-packed-device", lambda: F.dynamics_gain_packed(0, z(2, 1, 8), SR, meta(2, 6)), DaspError,
     "params is on meta but x is on cpu"),
    ("gain-curve-packed-cpu", lambda: F.dynamics_gain_packed(0, z(2, 1, 8), SR, z(2, 6, dtype=torch.int64)),
     DaspError, X_CPU),
    # the EQ's frequency response
    ("eqr-count", lambda: eq_response(counts=(3,) * 5 + (2,) + (3,) * 12), ValueError,
     "parametric_eq_frequency_response parameter 5: expected 3 element(s) (one per batch item) or 1, got 2"),
    ("eqr-count-and-sr", lambda: eq_response(counts=(2,) * 17 + (3,), sr=0), ValueError,
     "parametric_eq_frequency_response parameter 0: expected 3 element(s) (one per batch item) or 1, got 2"),
    ("eqr-sr-and-freqs", lambda: eq_response(sr=-1, freqs=z(2, 3)), ValueError, "sample_rate must be positive, got -1"),
    ("eqr-freqs-rank", lambda: eq_response(freqs=z(2, 3)), ValueError,
     "frequencies must be a 1-D tensor of frequencies in Hz, got (2, 3)"),
    ("eqr-freqs-list", lambda: eq_response(freqs=[100.0]), ValueError,
     "frequencies must be a 1-D tensor of frequencies in Hz, got list"),
    ("eqr-freqs-grad", lambda: eq_response(freqs=z(5, requires_grad=True)), ValueError,
     "frequencies must not require a gradient: the response is differentiated with respect to the 18 EQ parameters "
     "only"),
    ("eqr-devices", lambda: eq_response(bad={7: meta(2)}), DaspError,
     "parametric_eq_frequency_response: parameters on several devices ['cpu', 'meta']"),
    ("eqr-cpu", lambda: eq_response(counts=(1,) * 18), DaspError, f"parametric_eq_frequency_response: parameters are "
     f"on cpu: {NO_CPU}"),
    ("eqr-numbers", lambda: F.parametric_eq_frequency_response(SR, *([1.0] * 18), z(5)), DaspError,
     f"parametric_eq_frequency_response: parameters are on cpu: {NO_CPU}"),
    ("eqr-packed-shape-and-sr", lambda: F.parametric_eq_frequency_response_packed(0, z(2, 17), z(5)), ValueError,
     "params: expected a (bs, 18) parameter tensor, got (2, 17)"),
    ("eqr-packed-rank", lambda: F.parametric_eq_frequency_response_packed(SR, z(18), z(5)), ValueError,
     "params: expected a (bs, 18) parameter tensor, got (18,)"),
    ("eqr-packed-sr", lambda: F.parametric_eq_frequency_response_packed(0, z(2, 18), z(5)), ValueError,
     "sample_rate must be positive, got 0"),
    ("eqr-packed-freqs-grad", lambda: F.parametric_eq_frequency_response_packed(SR, meta(2, 18), z(
        5, requires_grad=True)), ValueError, "frequencies must not require a gradient: the response is differentiated "
     "with respect to the 18 EQ parameters only"),
    ("eqr-packed-cpu", lambda: F.parametric_eq_frequency_response_packed(SR, z(2, 18), z(5)), DaspError,
     f"parametric_eq_frequency_response: parameters are on cpu: {NO_CPU}"),
    ("eqr-packed-meta", lambda: F.parametric_eq_frequency_response_packed(SR, meta(2, 18), z(5)), DaspError,
     f"parametric_eq_frequency_response: parameters are on meta: {NO_CPU}"),
    # noise-shaped reverberation
    ("reverb-taps-and-rank", lambda: reverb(z(2, 8), taps=30), AssertionError, "num_bandpass_taps must be odd"),
    ("reverb-rank", lambda: reverb(z(2, 8)), ValueError, X_SHAPE),
    ("reverb-cpu-3ch", lambda: reverb(z(2, 3, 8)), DaspError, X_CPU),
    ("reverb-cpu-badparam-badnoise", lambda: reverb(z(2, 1, 8), bad={24: z(3)}, noise=z(1)), DaspError, X_CPU),
    ("reverb-packed-taps-and-cpu", lambda: F.noise_shaped_reverberation_packed(z(2, 1, 8), SR, z(2, 25),
                                                                               num_bandpass_taps=30),
     AssertionError, "num_bandpass_taps must be odd"),
    ("reverb-packed-rank", lambda: F.noise_shaped_reverberation_packed(z(2, 8), SR, z(2, 25)), ValueError, X_SHAPE),
    ("reverb-packed-cpu-badshape", lambda: F.noise_shaped_reverberation_packed(z(2, 1, 8), SR, z(2, 24)), DaspError,
     X_CPU),
    # the reverb's impulse response
    ("nsir-taps-even-and-L", lambda: nsir(taps=30, L=0), ValueError,
     "num_bandpass_taps must be a positive odd integer, got 30"),
    ("nsir-taps-0", lambda: nsir(taps=0), ValueError, "num_bandpass_taps must be a positive odd integer, got 0"),
    ("nsir-taps-frac", lambda: nsir(taps=31.5), ValueError,
     "num_bandpass_taps must be a positive odd integer, got 31.5"),
    ("nsir-L-and-sr", lambda: nsir(L=0, sr=32000), ValueError, "num_samples must be a positive integer, got 0"),
    ("nsir-sr-and-count", lambda: nsir(sr=32000, counts=(2,) * 23 + (3,)), ValueError,
     "sample_rate 32000 too low: the filter bank's 18 kHz high-pass needs sample_rate > 36000"),
    ("nsir-count-and-noise", lambda: nsir(counts=(3,) * 23 + (2,), noise=z(1)), ValueError,
     "noise_shaped_impulse_response parameter 23: expected 3 element(s) (one per batch item) or 1, got 2"),
    ("nsir-noise-and-cpu", lambda: nsir(noise=z(2, 12, 94)), ValueError,
     "noise must have shape (4, 12, 94), got (2, 12, 94)"),
    ("nsir-noise-broadcast-bs", lambda: nsir(counts=(1,) * 23 + (3,), noise=z(4, 12, 94)), ValueError,
     "noise must have shape (6, 12, 94), got (4, 12, 94)"),
    ("nsir-devices", lambda: nsir(bad={0: meta(2)}), DaspError,
     "noise_shaped_impulse_response: parameters on several devices ['cpu', 'meta']"),
    ("nsir-cpu", lambda: nsir(noise=z(4, 12, 94)), DaspError,
     f"noise_shaped_impulse_response: parameters are on cpu: {NO_CPU}"),
    ("nsir-numbers", lambda: F.noise_shaped_impulse_response(SR, *([0.5] * 24), num_samples=64, num_bandpass_taps=31),
     DaspError, f"noise_shaped_impulse_response: parameters are on cpu: {NO_CPU}"),
    ("nsir-packed-taps-and-shape", lambda: F.noise_shaped_impulse_response_packed(SR, z(2, 25), num_bandpass_taps=2),
     ValueError, "num_bandpass_taps must be a positive odd integer, got 2"),
    ("nsir-packed-shape-and-noise", lambda: F.noise_shaped_impulse_response_packed(SR, z(2, 25), 64, 31, noise=z(1)),
     ValueError, "params: expected a (bs, 24) parameter tensor, got (2, 25)"),
    ("nsir-packed-list", lambda: F.noise_shaped_impulse_response_packed(SR, [[0.0] * 24], 64, 31), ValueError,
     "params: expected a (bs, 24) parameter tensor, got ()"),
    ("nsir-packed-noise-and-cpu", lambda: F.noise_shaped_impulse_response_packed(SR, z(3, 24), 64, 31,
                                                                                 noise=z(4, 12, 94)),
     ValueError, "noise must have shape (6, 12, 94), got (4, 12, 94)"),
    ("nsir-packed-cpu", lambda: F.noise_shaped_impulse_response_packed(SR, z(2, 24), 64, 31), DaspError,
     f"noise_shaped_impulse_response: parameters are on cpu: {NO_CPU}"),
    # convolution reverberation
    ("conv-x-rank-ir-rank", lambda: F.convolution_reverberation(z(2, 8), SR, z(2, 8), z(2)), ValueError, X_SHAPE),
    ("conv-x-chs-ir-rank", lambda: F.convolution_reverberation(z(2, 3, 8), SR, z(2, 8), z(2)), ValueError,
     "x: only mono/stereo is supported, got 3 channels"),
    ("conv-ir-rank", lambda: F.convolution_reverberation(z(2, 2, 8), SR, z(2, 8), z(2)), ValueError,
     "impulse_response must be a tensor of shape (batch, channels, samples)"),
    ("conv-ir-chs-and-batch", lambda: F.convolution_reverberation(z(2, 2, 8), SR, z(3, 3, 4), z(2)), ValueError,
     "impulse_response: only mono/stereo/true-stereo (4) is supported, got 3 channels"),
    ("conv-ir-batch-and-taps", lambda: F.convolution_reverberation(z(2, 2, 8), SR, z(3, 2, 0), z(2)), ValueError,
     "impulse_response has batch 3, x has batch 2 (expected 2 or 1)"),
    ("conv-ir-shared-needs-batch", lambda: F.convolution_reverberation(z(0, 2, 8), SR, z(1, 2, 4), z(1)), ValueError,
     "impulse_response has batch 1, x has batch 0 (expected 0 or 1)"),
    ("conv-ir-taps-and-mix", lambda: F.convolution_reverberation(z(2, 2, 8), SR, z(1, 4, 0), z(3)), ValueError,
     "impulse_response needs at least one tap"),
    ("conv-mix-and-cpu", lambda: F.convolution_reverberation(z(2, 1, 8), SR, z(2, 1, 4), z(3)), ValueError,
     "mix: expected 2 element(s) (one per batch item) or 1, got 3"),
    ("conv-cpu", lambda: F.convolution_reverberation(z(2, 1, 8), SR, z(1, 2, 4), 0.5), DaspError, X_CPU),
    ("conv-x-meta-ir-cpu", lambda: F.convolution_reverberation(meta(2, 2, 8), SR, z(2, 2, 4), z(2)), DaspError,
     f"x is on meta: {NO_CPU}"),
    # convolution bus
    ("bus-x-rank-ir-rank", lambda: F.convolution_bus(z(2, 8), SR, z(2, 1, 8)), ValueError,
     "x must be a tensor of shape (batch, inputs, samples)"),
    ("bus-ir-rank", lambda: F.convolution_bus(z(2, 1, 8), SR, z(2, 1, 8)), ValueError,
     "impulse_response must be a tensor of shape (batch, inputs, outputs, taps)"),
    ("bus-inputs-0", lambda: F.convolution_bus(z(2, 0, 8), SR, z(2, 0, 1, 4)), ValueError,
     "convolution_bus: 1 to 32 input channels are supported, got 0"),
    ("bus-inputs-33-and-rows", lambda: F.convolution_bus(z(2, 33, 8), SR, z(2, 3, 1, 4)), ValueError,
     "convolution_bus: 1 to 32 input channels are supported, got 33"),
    ("bus-rows-and-outputs", lambda: F.convolution_bus(z(2, 2, 8), SR, z(2, 3, 3, 4)), ValueError,
     "impulse_response has 3 input rows, x has 2 channels"),
    ("bus-outputs-and-batch", lambda: F.convolution_bus(z(2, 2, 8), SR, z(3, 2, 3, 4)), ValueError,
     "impulse_response: a mono (1) or stereo (2) bus is supported, got 3 outputs"),
    ("bus-batch-and-taps", lambda: F.convolution_bus(z(2, 2, 8), SR, z(3, 2, 2, 0)), ValueError,
     "impulse_response has batch 3, x has batch 2 (expected 2 or 1)"),
    ("bus-taps-and-samples", lambda: F.convolution_bus(z(2, 2, 0), SR, z(1, 2, 2, 0)), ValueError,
     "impulse_response needs at least one tap"),
    ("bus-samples-and-cpu", lambda: F.convolution_bus(z(2, 2, 0), SR, z(2, 2, 2, 4)), ValueError,
     "x needs at least one sample"),
    ("bus-cpu", lambda: F.convolution_bus(z(2, 2, 7, dtype=torch.int16), SR, z(1, 2, 1, 4)), DaspError, X_CPU),
    ("bus-x-meta-ir-cpu", lambda: F.convolution_bus(meta(2, 2, 8), SR, z(2, 2, 2, 4)), DaspError,
     f"x is on meta: {NO_CPU}"),
]


@pytest.mark.parametrize("call,exc,msg", [pytest.param(c, e, m, id=i) for i, c, e, m in CASES])
def test_check_raises_exactly(call, exc, msg):
    with pytest.raises(exc) as info:
        call()
    assert type(info.value) is exc
    assert str(info.value) == msg


@pytest.mark.parametrize("proc,call,msg", [
    ("ParametricEQ", lambda p: p.frequency_response(z(2, 18), z(5)),
     "ParametricEQ.frequency_response: param_tensor must be a CUDA tensor; dasp_pytorch_b200 has no CPU path"),
    ("ParametricEQ", lambda p: p.frequency_response([[0.5] * 18], z(5)),
     "ParametricEQ.frequency_response: param_tensor must be a CUDA tensor; dasp_pytorch_b200 has no CPU path"),
    ("Compressor", lambda p: p.gain_curve(z(2, 1, 8), z(2, 6)),
     "Compressor.gain_curve: param_tensor must be a CUDA tensor; dasp_pytorch_b200 has no CPU path"),
    ("Expander", lambda p: p.gain_curve(z(2, 1, 8), meta(2, 6), db=True),
     "Expander.gain_curve: param_tensor must be a CUDA tensor; dasp_pytorch_b200 has no CPU path"),
])
def test_processor_cuda_guard(proc, call, msg):
    with pytest.raises(DaspError) as info:
        call(getattr(D, proc)(SR))
    assert str(info.value) == msg


@pytest.mark.parametrize("proc,fn", [("Compressor", "compressor"), ("Expander", "expander")])
def test_dynamics_processor_paths(proc, fn):
    """the processor's packed path mirrors its process_fn; on CPU parameters the by-name path runs and x's device
    check is the first to fail"""
    p = getattr(D, proc)(SR)
    assert p.process_fn is getattr(F, fn) and p._packed_path[1] is p.process_fn
    with pytest.raises(DaspError) as info:
        p.process_normalized(z(2, 1, 8), torch.full((2, 6), 0.5))
    assert str(info.value) == X_CPU
    with pytest.raises(DaspError) as info:
        p._packed_path[0](z(2, 1, 8), SR, z(2, 5), sidechain=z(2, 1, 8))
    assert str(info.value) == f"sidechain is on cpu: {NO_CPU}"
