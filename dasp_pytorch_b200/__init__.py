"""dasp_pytorch_b200: H100-native (sm_90a) kernels behind dasp_pytorch's functional audio processors.

Drop-in surface: the same names the reference package exports (``dasp_pytorch/__init__.py``) for the hot
path -- ``gain``, ``distortion``, ``parametric_eq``, ``compressor``, ``noise_shaped_reverberation`` and the
``Processor`` classes, ``stereo_bus``, ``stereo_panner``, ``stereo_widener`` -- plus ``expander`` (stubbed upstream)
``convolution_reverberation`` (the reverb's convolution with a caller-supplied impulse response) and
``sidechain_compressor`` / ``sidechain_expander`` (the detector on an external key signal) and
``noise_shaped_impulse_response`` (the reverb's impulse response on its own, with gradients to its band parameters) and
``parametric_eq_frequency_response`` (the EQ's complex transfer function at chosen frequencies, with gradients to its
18 parameters) and ``compressor_gain`` / ``expander_gain`` (the time-varying gain the compressor / expander multiplies
into the audio, linear or in dB, with gradients to the detector input and the parameters) and ``convolution_bus`` (any
number of input channels, each through its own impulse responses, summed into a mono or stereo bus) and
``time_varying_convolution_reverberation`` (a trajectory of impulse responses crossfaded along the output, for moving
sources and listeners) and ``time_varying_convolution_bus`` (several moving sources, each with its own trajectory of
impulse responses, crossfaded and summed into a mono or stereo bus; ``crossfade="input"`` crossfades on the source side,
so every emitted sample keeps the impulse response of its emission time) and ``multichannel_convolution`` (S sources
through an S x M matrix of impulse responses into up to 32 output channels: microphone arrays, ambisonics, multichannel
beds) and ``time_varying_multichannel_convolution`` (moving sources through a trajectory of such matrices, crossfaded on
the output or the source side: moving talkers at a microphone array, moving objects in ambisonic or 5.1 / 7.1 scenes).
"""
from dasp_pytorch_b200 import functional  # noqa: F401
from dasp_pytorch_b200.functional import (  # noqa: F401
    CONV_BUS_MAX_INPUTS,
    CONV_MC_MAX_OUTPUTS,
    CONV_PARTITION_SAMPLES,
    compressor,
    compressor_gain,
    convolution_bus,
    convolution_reverberation,
    distortion,
    expander,
    expander_gain,
    gain,
    multichannel_convolution,
    noise_shaped_impulse_response,
    noise_shaped_impulse_response_packed,
    noise_shaped_reverberation,
    parametric_eq,
    parametric_eq_frequency_response,
    parametric_eq_frequency_response_packed,
    sidechain_compressor,
    sidechain_expander,
    stereo_bus,
    stereo_panner,
    stereo_widener,
    time_varying_convolution_bus,
    time_varying_convolution_reverberation,
    time_varying_multichannel_convolution,
)
from dasp_pytorch_b200.modules import (  # noqa: F401
    Compressor,
    Distortion,
    Expander,
    Gain,
    NoiseShapedReverb,
    ParametricEQ,
    Processor,
)
