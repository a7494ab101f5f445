"""Normalised-parameter processors over the H100 kernels.

Same contract as the reference's ``dasp_pytorch/modules.py`` (@ c9ae0126): a ``Processor`` owns an ordered
``param_ranges`` dict, ``process_normalized(x, p)`` takes ``p`` in ``[0, 1]`` with shape
``(batch, num_params)`` (columns in ``param_ranges`` order), maps each column affinely onto its range and
calls ``process_fn(x, sample_rate, **params)`` with the parameter NAMES as keywords (reference
``modules.py:25-51``) -- which is why the keyword names of ``dasp_pytorch_b200.functional`` are part of the
drop-in contract.  ``process(x, *args)`` forwards positionally (``modules.py:53-54``).

Differences, all on the host side:
  * the range check of ``denormalize_param_dict`` (reference ``modules.py:83-84``) costs the reference two
    device->host synchronisations per parameter.  Here the packed path runs ONE kernel (``dasp_denormalize``)
    that maps the whole ``(batch, P)`` tensor and checks the range on the device: an offending value becomes
    NaN and raises a device flag.  Outside CUDA-graph capture the flag is read back once per call and the
    reference's ``ValueError`` (with the parameter name) is raised; under capture nothing is read back -- the
    flag stays on the device (``Processor.range_violation()``) and the NaN makes the offending item visible;
  * ``Distortion`` keeps the reference's positional order ``(min_gain_db, max_gain_db)`` and takes
    ``sample_rate`` as a trailing keyword; its parameter is keyed by the functional's real keyword ``drive_db``
    (the reference's key ``gain_db`` cannot be dispatched by name to ``distortion(x, sr, drive_db)`` --
    SURVEY.md fact 8); ``param_ranges["gain_db"]`` still resolves, as an alias.
"""
from __future__ import annotations

import functools
from typing import Dict

import torch

from dasp_pytorch_b200 import functional as _F
from dasp_pytorch_b200.functional import (
    compressor,
    distortion,
    expander,
    gain,
    noise_shaped_reverberation,
    parametric_eq,
    sidechain_compressor,
    sidechain_expander,
)


def denormalize(norm_val, max_val, min_val):
    return (norm_val * (max_val - min_val)) + min_val


def normalize(val, min_val, max_val):
    return (val - min_val) / (max_val - min_val)


class _DenormFn(torch.autograd.Function):
    """(bs, P) in [0, 1] -> physical units, one kernel (``dasp_denormalize``); gradient = g * span."""

    @staticmethod
    def forward(ctx, p01, lo, span, flag):
        from dasp_pytorch_b200 import _abi
        p = p01.to(torch.float32).contiguous()
        out = torch.empty_like(p)
        with torch.cuda.device(p.device):
            _abi.check(_abi.lib().dasp_denormalize(_abi.ptr(p), _abi.ptr(lo), _abi.ptr(span), _abi.ptr(out),
                                                   _abi.ptr(flag), p.shape[0], p.shape[1],
                                                   _abi.stream_ptr(p.device)), "dasp_denormalize")
        ctx.save_for_backward(span)
        ctx.in_dtype = p01.dtype
        return out

    @staticmethod
    def backward(ctx, g):
        (span,) = ctx.saved_tensors
        return (g * span).to(ctx.in_dtype), None, None, None


class _RangeDict(dict):
    """``param_ranges`` with read-only aliases (reference key names that differ from the functional keyword)."""

    def __init__(self, *a, aliases=None, **kw):
        super().__init__(*a, **kw)
        self._aliases = dict(aliases or {})

    def __missing__(self, key):
        if key in self._aliases:
            return self[self._aliases[key]]
        raise KeyError(key)


class Processor:
    """Base class: subclasses set ``sample_rate``, ``process_fn`` and ``param_ranges``."""

    sample_rate = None
    process_fn = None
    param_ranges: Dict[str, tuple] = {}
    # True (default): outside CUDA-graph capture an out-of-range parameter raises ValueError like the reference
    # (one device->host read per call).  False: never read back; use range_violation() when convenient.
    strict_range_check = True

    # Plain attribute like the reference (its subclasses assign ``self.num_params = len(self.param_ranges)``);
    # processors that never assign it get the length of their ranges.
    @property
    def num_params(self) -> int:
        return self.__dict__.get("_num_params", len(self.param_ranges))

    @num_params.setter
    def num_params(self, value) -> None:
        self.__dict__["_num_params"] = int(value)

    # subclasses with a packed kernel entry point set this to (callable(x, sr, packed), the process_fn it mirrors)
    _packed_path = None

    def process_normalized(self, x: torch.Tensor, param_tensor: torch.Tensor):
        """Run the processor with parameters normalised to (0, 1), shape ``(batch, num_params)``.

        Fast path (SURVEY.md 8f rank 1): when ``process_fn`` is still this package's kernel entry, the whole
        parameter handling is ONE range-check reduction and ONE affine kernel on the packed ``(batch, P)``
        tensor, which then goes to the kernels as is -- instead of the reference's per-parameter slicing,
        2 host syncs and ~3 tiny kernels per parameter (modules.py:56-91).  Same errors, same results.
        """
        return self._process_normalized(x, param_tensor)

    def _process_normalized(self, x: torch.Tensor, param_tensor: torch.Tensor, by_name=None, **fn_kw):
        """process_normalized; ``fn_kw`` (keyword arguments beyond the parameters) goes to either path's call, and
        ``by_name`` (default ``process_fn``) is the function the by-name path calls"""
        if self._packed_path is not None and self.process_fn is self._packed_path[1] and param_tensor.is_cuda:
            return self._packed_path[0](x, self.sample_rate, self._denormalize_packed(param_tensor), **fn_kw)
        param_dict = self.extract_param_dict(param_tensor)
        denorm = self.denormalize_param_dict(param_dict, _checked=self._range_check(param_tensor))
        return (by_name or self.process_fn)(x, self.sample_rate, **denorm, **fn_kw)

    def _denormalize_packed(self, param_tensor: torch.Tensor) -> torch.Tensor:
        """(batch, P) in [0, 1] on a CUDA device -> physical units: one ``dasp_denormalize`` kernel, and outside
        graph capture (with ``strict_range_check``) the reference's ``ValueError`` naming an out-of-range parameter"""
        if param_tensor.dim() != 2 or param_tensor.shape[1] != len(self.param_ranges):
            raise ValueError(
                f"Parameter tensor has {param_tensor.shape[1] if param_tensor.dim() == 2 else '?'} parameters, "
                f"but processor has {len(self.param_ranges)} parameters."
            )
        scale, offset = self._affine(param_tensor.device)
        flag = self._flag(param_tensor.device)
        phys = _DenormFn.apply(param_tensor, offset, scale, flag)
        if self.strict_range_check and not torch.cuda.is_current_stream_capturing():
            if int(flag.item()) != 0:
                flag.zero_()
                self.denormalize_param_dict(self.extract_param_dict(param_tensor))      # raises with the name
        return phys

    def _denormalize_cuda(self, param_tensor, caller: str) -> torch.Tensor:
        """``_denormalize_packed`` for the methods that have only the packed path: ``param_tensor`` must be on CUDA"""
        if not torch.is_tensor(param_tensor) or not param_tensor.is_cuda:
            raise _F.DaspError(f"{caller}: param_tensor must be a CUDA tensor; dasp_pytorch_b200 has no CPU path")
        return self._denormalize_packed(param_tensor)

    def _affine(self, device):
        key = (str(device), tuple(self.param_ranges.values()))
        cache = self.__dict__.setdefault("_affine_cache", {})
        if key not in cache:
            lo = torch.tensor([r[0] for r in self.param_ranges.values()], dtype=torch.float32)
            hi = torch.tensor([r[1] for r in self.param_ranges.values()], dtype=torch.float32)
            cache.clear()
            cache[key] = ((hi - lo).to(device), lo.to(device))
        return cache[key]

    def _flag(self, device) -> torch.Tensor:
        cache = self.__dict__.setdefault("_flag_cache", {})
        key = str(device)
        if key not in cache:
            cache[key] = torch.zeros(1, dtype=torch.int32, device=device)
        return cache[key]

    def range_violation(self, device=None) -> bool:
        """True if a packed ``process_normalized`` call on ``device`` saw a parameter outside [0, 1] since the
        last query (device->host read; meant for after a graph replay).  Resets the flag."""
        flags = list(self.__dict__.get("_flag_cache", {}).items())
        if device is not None:
            flags = [(k, f) for k, f in flags if k == str(device)]
        bad = False
        for _, f in flags:
            if int(f.item()) != 0:
                bad = True
                f.zero_()
        return bad

    def process(self, x: torch.Tensor, *args):
        return self.process_fn(x, *args)

    def extract_param_dict(self, param_tensor: torch.Tensor):
        if param_tensor.shape[1] != len(self.param_ranges):
            raise ValueError(
                f"Parameter tensor has {param_tensor.shape[1]} parameters, "
                f"but processor has {len(self.param_ranges)} parameters."
            )
        return {name: param_tensor[:, i] for i, name in enumerate(self.param_ranges.keys())}

    @staticmethod
    def _range_check(param_tensor: torch.Tensor) -> bool:
        # one reduction + one host read for the whole tensor instead of 2 per parameter
        lo, hi = torch.aminmax(param_tensor.detach())
        bad = bool((lo < 0) | (hi > 1))
        return not bad

    def denormalize_param_dict(self, param_dict: dict, _checked=None):
        """(0, 1) -> physical ranges; raises ``ValueError`` on out-of-range input like the reference."""
        if _checked is None:
            _checked = all(self._range_check(v.reshape(1, -1)) for v in param_dict.values())
        if not _checked:
            for name, v in param_dict.items():
                if v.min() < 0 or v.max() > 1:
                    raise ValueError(f"Parameter {name} of is out of range.")
        out = {}
        for name, v in param_dict.items():
            lo, hi = self.param_ranges[name]
            out[name] = denormalize(v, hi, lo)
        return out


class Gain(Processor):
    def __init__(self, sample_rate: int, min_gain_db: float = -24.0, max_gain_db: float = 24.0):
        self.sample_rate = sample_rate
        self.process_fn = gain
        self._packed_path = (lambda x, sr, p: gain(x, sr, p[:, 0]), gain)
        self.param_ranges = {"gain_db": (min_gain_db, max_gain_db)}
        self.num_params = len(self.param_ranges)


class Distortion(Processor):
    """Reference order ``Distortion(min_gain_db, max_gain_db)`` (``modules.py:110-121``); ``sample_rate`` is a
    trailing keyword (the reference class has none, which is why it cannot run ``process_normalized``)."""

    def __init__(self, min_gain_db: float = 0.0, max_gain_db: float = 24.0, sample_rate: int = 44100):
        self.sample_rate = sample_rate
        self.process_fn = distortion
        self._packed_path = (lambda x, sr, p: distortion(x, sr, p[:, 0]), distortion)
        self.param_ranges = _RangeDict({"drive_db": (min_gain_db, max_gain_db)}, aliases={"gain_db": "drive_db"})
        self.num_params = len(self.param_ranges)


class ParametricEQ(Processor):
    def __init__(self, sample_rate: int, min_gain_db: float = -20.0, max_gain_db: float = 20.0,
                 min_q_factor: float = 0.1, max_q_factor: float = 6.0):
        self.sample_rate = sample_rate
        self.process_fn = parametric_eq
        self._packed_path = (_F.parametric_eq_packed, parametric_eq)
        g, q = (min_gain_db, max_gain_db), (min_q_factor, max_q_factor)
        top = (sample_rate // 2) - 1000
        cut = {"low_shelf": (20, 2000), "band0": (80, 2000), "band1": (2000, 8000), "band2": (8000, 12000),
               "band3": (12000, top), "high_shelf": (4000, top)}
        self.param_ranges = {}
        for sec, fr in cut.items():
            self.param_ranges[f"{sec}_gain_db"] = g
            self.param_ranges[f"{sec}_cutoff_freq"] = fr
            self.param_ranges[f"{sec}_q_factor"] = q

    def frequency_response(self, param_tensor: torch.Tensor, frequencies: torch.Tensor) -> torch.Tensor:
        """The complex response ``(batch, F)`` of the EQ that ``process_normalized(x, param_tensor)`` applies, at
        ``frequencies`` in Hz (see ``functional.parametric_eq_frequency_response``).  ``param_tensor`` is
        ``(batch, 18)`` in [0, 1] on a CUDA device, mapped and range-checked exactly as ``process_normalized`` does;
        gradients flow back to it."""
        phys = self._denormalize_cuda(param_tensor, "ParametricEQ.frequency_response")
        return _F.parametric_eq_frequency_response_packed(self.sample_rate, phys, frequencies)


class _Dynamics(Processor):
    def __init__(self, kind: int, process_fn, sidechain_fn, sample_rate: int, min_threshold_db: float = -60.0,
                 max_threshold_db: float = 0.0, min_ratio: float = 1.0, max_ratio: float = 20.0,
                 min_attack_ms: float = 5.0, max_attack_ms: float = 100.0, min_release_ms: float = 5.0,
                 max_release_ms: float = 100.0, min_knee_db: float = 0.0, max_knee_db: float = 12.0,
                 min_makeup_gain_db: float = 0.0, max_makeup_gain_db: float = 12.0):
        self.sample_rate = sample_rate
        self.process_fn = process_fn
        # the side-chain counterpart of the package's process_fn (functional.sidechain_compressor / _expander)
        self._sidechain_fn = sidechain_fn
        self._kind = kind          # 0: compressor, 1: expander
        self._packed_path = (functools.partial(_F.dynamics_packed, self._kind), process_fn)
        self.param_ranges = {
            "threshold_db": (min_threshold_db, max_threshold_db),
            "ratio": (min_ratio, max_ratio),
            "attack_ms": (min_attack_ms, max_attack_ms),
            "release_ms": (min_release_ms, max_release_ms),
            "knee_db": (min_knee_db, max_knee_db),
            "makeup_gain_db": (min_makeup_gain_db, max_makeup_gain_db),
        }

    def process_normalized(self, x: torch.Tensor, param_tensor: torch.Tensor, sidechain=None):
        """``Processor.process_normalized`` with an optional key: ``sidechain`` (bs, K, n) drives the detector
        instead of x (see ``functional.sidechain_compressor``); ``None`` runs the plain processor.  With a key, the
        by-name path calls the side-chain function while ``process_fn`` is still this package's, otherwise
        ``process_fn(x, sample_rate, **params, sidechain=sidechain)``."""
        if sidechain is None:
            return self._process_normalized(x, param_tensor)
        by_name = self._sidechain_fn if self.process_fn is self._packed_path[1] else None
        return self._process_normalized(x, param_tensor, by_name, sidechain=sidechain)

    def gain_curve(self, x: torch.Tensor, param_tensor: torch.Tensor, *, db: bool = False) -> torch.Tensor:
        """The gain ``(batch, 1, n)`` that ``process_normalized(x, param_tensor)`` multiplies into the audio, with the
        detector on ``x`` (see ``functional.compressor_gain``); ``db=True`` returns it in dB.  ``param_tensor`` is
        ``(batch, 6)`` in [0, 1] on a CUDA device, mapped and range-checked exactly as ``process_normalized`` does;
        gradients flow back to it and to x."""
        phys = self._denormalize_cuda(param_tensor, f"{type(self).__name__}.gain_curve")
        return _F.dynamics_gain_packed(self._kind, x, self.sample_rate, phys, db=db)


class Compressor(_Dynamics):
    def __init__(self, sample_rate: int, **kw):
        super().__init__(0, compressor, sidechain_compressor, sample_rate, **kw)


class Expander(_Dynamics):
    """New: the reference advertises an expander but only stubs it (functional.py:402-403)."""

    def __init__(self, sample_rate: int, max_ratio: float = 4.0, **kw):
        super().__init__(1, expander, sidechain_expander, sample_rate, max_ratio=max_ratio, **kw)


class NoiseShapedReverb(Processor):
    def __init__(self, sample_rate, min_band_gain: float = 0.0, max_band_gain: float = 1.0,
                 min_band_decay: float = 0.0, max_band_decay: float = 1.0, min_mix: float = 0.0,
                 max_mix: float = 1.0):
        self.sample_rate = sample_rate
        self.process_fn = noise_shaped_reverberation
        self._packed_path = (_F.noise_shaped_reverberation_packed, noise_shaped_reverberation)
        self.param_ranges = {f"band{i}_gain": (min_band_gain, max_band_gain) for i in range(12)}
        self.param_ranges.update({f"band{i}_decay": (min_band_decay, max_band_decay) for i in range(12)})
        self.param_ranges["mix"] = (min_mix, max_mix)
