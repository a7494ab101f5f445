"""dasp_pytorch_b200: H100-native (sm_90a) kernels behind dasp_pytorch's functional audio processors.

Drop-in surface: the same names the reference package exports (``dasp_pytorch/__init__.py``) for the hot
path -- ``gain``, ``distortion``, ``parametric_eq``, ``compressor``, ``noise_shaped_reverberation`` and the
``Processor`` classes, ``stereo_bus``, ``stereo_panner``, ``stereo_widener`` -- plus ``expander`` (stubbed upstream)
``convolution_reverberation`` (the reverb's convolution with a caller-supplied impulse response) and
``sidechain_compressor`` / ``sidechain_expander`` (the detector on an external key signal).
"""
from dasp_pytorch_b200 import functional  # noqa: F401
from dasp_pytorch_b200.functional import (  # noqa: F401
    compressor,
    convolution_reverberation,
    distortion,
    expander,
    gain,
    noise_shaped_reverberation,
    parametric_eq,
    sidechain_compressor,
    sidechain_expander,
    stereo_bus,
    stereo_panner,
    stereo_widener,
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
