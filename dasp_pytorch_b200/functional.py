"""H100-native drop-in for ``dasp_pytorch.functional``'s audio-processor hot path.

Same function names, argument order, keyword names, defaults and
``(batch, channels, samples)`` tensor contract as the reference
(``dasp_pytorch/functional.py`` @ c9ae0126), so that
``Processor.process_normalized`` -> ``process_fn(x, sample_rate, **params)``
(reference ``modules.py:45-49``) and direct calls keep working unchanged.  Every
op is a ``torch.autograd.Function`` whose forward and backward call hand-written
sm_90a kernels through the C ABI in ``include/dasp_b200.h``; there is no PyTorch,
Triton or CPU fallback -- non-CUDA inputs raise ``DaspError``.

Arithmetic is fp32 (coefficient design in fp64 inside the kernels).  Inputs in
another floating dtype are computed in fp32 and returned in the input dtype.
"""
from __future__ import annotations

from typing import Optional

import torch

from dasp_pytorch_b200 import _abi
from dasp_pytorch_b200._abi import DaspError, check, ptr, stream_ptr

__all__ = [
    "gain",
    "distortion",
    "stereo_widener",
    "stereo_panner",
    "stereo_bus",
    "parametric_eq",
    "compressor",
    "expander",
    "sidechain_compressor",
    "sidechain_expander",
    "noise_shaped_reverberation",
    "convolution_reverberation",
]


# --------------------------------------------------------------------------------------
# helpers
# --------------------------------------------------------------------------------------


def _audio(x: torch.Tensor, name: str = "x"):
    """validate the (bs, chs, n) audio tensor -> (fp32 contiguous tensor, original dtype)"""
    if not torch.is_tensor(x) or x.dim() != 3:
        raise ValueError(f"{name} must be a tensor of shape (batch, channels, samples)")
    if not x.is_cuda:
        raise DaspError(
            f"{name} is on {x.device}: dasp_pytorch_b200 only runs on CUDA (H100) tensors and has no CPU path"
        )
    if not x.is_floating_point():
        raise DaspError(f"{name} must be a floating-point tensor, got {x.dtype}")
    return x.to(torch.float32).contiguous(), x.dtype


def _param(p, n_expected: int, like: torch.Tensor, name: str, allow_broadcast: bool = False) -> torch.Tensor:
    """flatten a parameter to fp32 ``(n_expected,)`` on x's device, keeping autograd history.

    The reference reshapes parameters with ``.view(bs, 1, 1)`` and friends, i.e. it accepts
    any shape holding the right number of elements (SURVEY.md 8b); integer tensors are
    promoted (examples/demo.py:44 passes int64 cut-offs).
    """
    if not torch.is_tensor(p):
        p = torch.as_tensor(p)
    if p.device != like.device:
        if p.numel() == 1 and not p.requires_grad:
            p = p.to(like.device)
        else:
            raise DaspError(f"{name} is on {p.device} but x is on {like.device}")
    p = p.reshape(-1).to(torch.float32)
    if p.numel() != n_expected:
        if allow_broadcast and p.numel() == 1:
            p = p.expand(n_expected)
        else:
            raise RuntimeError(
                f"{name}: expected {n_expected} element(s) (one per batch item), got {p.numel()}"
            )
    return p


def _ws(n_floats: int, device) -> torch.Tensor:
    return torch.empty(max(int(n_floats), 1), dtype=torch.float32, device=device)


# bench.py sets this to a list to collect (stage, start_event, end_event) around every C-ABI call
STAGE_TIMING = None


class _timed:
    """CUDA events on the launching stream around one C-ABI call (active only while benchmarking)."""

    def __init__(self, name, device):
        self.name, self.device = name, device

    def __enter__(self):
        if STAGE_TIMING is not None:
            self.a = torch.cuda.Event(enable_timing=True)
            self.b = torch.cuda.Event(enable_timing=True)
            self.a.record(torch.cuda.current_stream(self.device))
        return self

    def __exit__(self, *exc):
        if STAGE_TIMING is not None:
            self.b.record(torch.cuda.current_stream(self.device))
            STAGE_TIMING.append((self.name, self.a, self.b))
        return False


# --------------------------------------------------------------------------------------
# gain / distortion
# --------------------------------------------------------------------------------------


class _PointwiseFn(torch.autograd.Function):
    """y = f(x * 10^(p_db/20)) with one p_db per row; f = identity (gain) or tanh (distortion)."""

    @staticmethod
    def forward(ctx, x, p_db, kind: str, rows: int, n: int):
        lib = _abi.lib()
        y = torch.empty_like(x)
        with torch.cuda.device(x.device), _timed("dist_fwd", x.device):
            st = stream_ptr(x.device)
            if kind == "gain":
                check(lib.dasp_gain_fwd(ptr(x), ptr(p_db), ptr(y), rows, 1, n, st), "dasp_gain_fwd")
            else:
                check(lib.dasp_distortion_fwd(ptr(x), ptr(p_db), ptr(y), rows, n, st), "dasp_distortion_fwd")
        ctx.save_for_backward(x, p_db)
        ctx.kind, ctx.rows, ctx.n = kind, rows, n
        return y

    @staticmethod
    def backward(ctx, gy):
        lib = _abi.lib()
        x, p_db = ctx.saved_tensors
        rows, n = ctx.rows, ctx.n
        gy = gy.contiguous()
        gx = torch.empty_like(x)
        gp = torch.empty_like(p_db)
        nws = lib.dasp_pointwise_bwd_workspace_floats(rows, n)
        ws = _ws(nws, x.device)
        with torch.cuda.device(x.device), _timed("dist_bwd", x.device):
            st = stream_ptr(x.device)
            if ctx.kind == "gain":
                check(lib.dasp_gain_bwd(ptr(gy), ptr(x), ptr(p_db), ptr(gx), ptr(gp), ptr(ws), nws, rows, 1, n, st),
                      "dasp_gain_bwd")
            else:
                check(lib.dasp_distortion_bwd(ptr(gy), ptr(x), ptr(p_db), ptr(gx), ptr(gp), ptr(ws), nws, rows, n,
                                              st), "dasp_distortion_bwd")
        return gx, gp, None, None, None


def gain(x: torch.Tensor, sample_rate: int, gain_db: torch.Tensor):
    """Apply a per-item gain in dB (reference ``functional.py:10-29``).

    Args:
        x: audio ``(bs, chs, seq_len)``.
        sample_rate: unused (kept for the common processor signature).
        gain_db: ``bs`` elements, any shape.
    """
    xf, dt = _audio(x)
    bs, chs, n = xf.shape
    g = _param(gain_db, bs, xf, "gain_db")
    y = _PointwiseFn.apply(xf, g.contiguous(), "gain", bs, chs * n)
    return y.to(dt)


def distortion(x: torch.Tensor, sample_rate: int, drive_db: torch.Tensor):
    """tanh soft clipper with drive in dB (reference ``functional.py:65-78``).

    Like the reference's ``drive_db.view(bs, chs, -1)``, the drive needs one element per
    (item, channel) row -- i.e. ``bs`` elements for mono input, ``bs*chs`` for multichannel.
    """
    xf, dt = _audio(x)
    bs, chs, n = xf.shape
    d = _param(drive_db, bs * chs, xf, "drive_db")
    y = _PointwiseFn.apply(xf, d.contiguous(), "distortion", bs * chs, n)
    return y.to(dt)


# --------------------------------------------------------------------------------------
# stereo mixing processors
# --------------------------------------------------------------------------------------


class _StereoFn(torch.autograd.Function):
    """kind: 'widener' | 'panner' | 'bus' -- streaming mixes with one scalar parameter per row."""

    @staticmethod
    def forward(ctx, x, p, kind):
        lib = _abi.lib()
        dev = x.device
        with torch.cuda.device(dev):
            st = stream_ptr(dev)
            if kind == "widener":
                bs, _, n = x.shape
                y = torch.empty_like(x)
                check(lib.dasp_widener_fwd(ptr(x), ptr(p), ptr(y), bs, n, st), "dasp_widener_fwd")
            elif kind == "panner":
                bs, tracks, n = x.shape
                y = torch.empty(bs, 2, tracks, n, dtype=torch.float32, device=dev)
                check(lib.dasp_panner_fwd(ptr(x), ptr(p), ptr(y), bs, tracks, n, st), "dasp_panner_fwd")
            else:
                bs, _, tracks, n = x.shape
                y = torch.empty(bs, 2, n, dtype=torch.float32, device=dev)
                check(lib.dasp_bus_fwd(ptr(x), ptr(p), ptr(y), bs, tracks, n, st), "dasp_bus_fwd")
        ctx.save_for_backward(x, p)
        ctx.kind = kind
        return y

    @staticmethod
    def backward(ctx, gy):
        lib = _abi.lib()
        x, p = ctx.saved_tensors
        dev = x.device
        gy = gy.contiguous()
        gx = torch.empty_like(x)
        gp = torch.empty_like(p)
        with torch.cuda.device(dev):
            st = stream_ptr(dev)
            if ctx.kind == "widener":
                bs, _, n = x.shape
                nws = lib.dasp_stereo_bwd_workspace_floats(bs, n)
                ws = _ws(nws, dev)
                check(lib.dasp_widener_bwd(ptr(gy), ptr(x), ptr(p), ptr(gx), ptr(gp), ptr(ws), nws, bs, n, st),
                      "dasp_widener_bwd")
            elif ctx.kind == "panner":
                bs, tracks, n = x.shape
                nws = lib.dasp_stereo_bwd_workspace_floats(bs * tracks, n)
                ws = _ws(nws, dev)
                check(lib.dasp_panner_bwd(ptr(gy), ptr(x), ptr(p), ptr(gx), ptr(gp), ptr(ws), nws, bs, tracks, n, st),
                      "dasp_panner_bwd")
            else:
                bs, _, tracks, n = x.shape
                nws = lib.dasp_stereo_bwd_workspace_floats(bs * 2 * tracks, n)
                ws = _ws(nws, dev)
                check(lib.dasp_bus_bwd(ptr(gy), ptr(x), ptr(p), ptr(gx), ptr(gp), ptr(ws), nws, bs, tracks, n, st),
                      "dasp_bus_bwd")
        return gx, gp, None


def _audio_nd(x, ndim, name="x"):
    if not torch.is_tensor(x) or x.dim() != ndim:
        raise ValueError(f"{name} must be a {ndim}-dimensional tensor")
    if not x.is_cuda:
        raise DaspError(f"{name} is on {x.device}: dasp_pytorch_b200 only runs on CUDA (H100) tensors and has no CPU path")
    if not x.is_floating_point():
        raise DaspError(f"{name} must be a floating-point tensor, got {x.dtype}")
    return x.to(torch.float32).contiguous(), x.dtype


def stereo_widener(x: torch.Tensor, sample_rate: float, width: torch.Tensor):
    """Mid/side stereo widener (reference ``functional.py:580-604``).

    ``x`` is ``(bs, 2, seq_len)``, ``width`` holds ``bs`` elements (0 = mono sum, 0.5 = unchanged,
    1 = side only).  mid = (L+R)/sqrt2 scaled by 2(1-width), side = (L-R)/sqrt2 scaled by 2 width.
    """
    xf, dt = _audio_nd(x, 3)
    bs, chs, _ = xf.shape
    assert chs == 2, "Input tensor must have shape (bs, 2, seq_len)"
    w = _param(width, bs, xf, "width").contiguous()
    return _StereoFn.apply(xf, w, "widener").to(dt)


def stereo_panner(x: torch.Tensor, sample_rate: float, pan: torch.Tensor):
    """Pan mono tracks across the stereo field (reference ``functional.py:607-636``).

    ``x`` is ``(bs, num_tracks, seq_len)``, ``pan`` in ``[0, 1]`` holds ``bs*num_tracks`` elements; returns
    ``(bs, 2, num_tracks, seq_len)`` -- the layout the reference's code produces (its docstring says
    ``(bs, num_tracks, 2, seq_len)``, its ``unsqueeze(1).repeat(1, 2, 1, 1)`` does not).
    """
    xf, dt = _audio_nd(x, 3)
    bs, tracks, _ = xf.shape
    pn = _param(pan, bs * tracks, xf, "pan").contiguous()
    return _StereoFn.apply(xf, pn, "panner").to(dt)


def stereo_bus(x: torch.Tensor, sample_rate: int, send_db: torch.Tensor):
    """Sum stereo tracks to a stereo bus with per-track send levels in dB (reference ``functional.py:32-62``).

    ``x`` is ``(bs, 2, tracks, seq_len)``, ``send_db`` holds ``bs*tracks`` elements; returns ``(bs, 2, seq_len)``.
    """
    xf, dt = _audio_nd(x, 4)
    bs, chs, tracks, _ = xf.shape
    assert chs == 2, "Input tensor must have shape (bs, 2, tracks, seq_len)"
    sd = _param(send_db, bs * tracks, xf, "send_db").contiguous()
    return _StereoFn.apply(xf, sd, "bus").to(dt)


# --------------------------------------------------------------------------------------
# compressor / expander
# --------------------------------------------------------------------------------------


class _DynamicsFn(torch.autograd.Function):
    """Feed-forward dynamics processor: kind 0 = compressor, 1 = expander."""

    @staticmethod
    def forward(ctx, x, threshold, ratio, attack, knee, makeup, kind, sample_rate, eps, lookahead):
        lib = _abi.lib()
        bs, chs, n = x.shape
        y = torch.empty_like(x)
        need_bwd = any(ctx.needs_input_grad[:6])
        ckpt = None
        with torch.cuda.device(x.device):
            if need_bwd:
                tile = lib.dasp_dynamics_tile_len(bs, chs)     # depends on the device's SM count
                if tile <= 0:
                    raise DaspError(f"dynamics: unsupported channel count {chs}")
                ckpt = torch.empty(bs * max(1, -(-n // tile)), dtype=torch.float32, device=x.device)
            with _timed("comp_fwd", x.device):
                check(lib.dasp_dynamics_fwd(kind, ptr(x), ptr(threshold), ptr(ratio), ptr(attack), ptr(knee),
                                            ptr(makeup), ptr(y), ptr(ckpt), bs, chs, n, float(sample_rate),
                                            float(eps), int(lookahead), stream_ptr(x.device)), "dasp_dynamics_fwd")
        if need_bwd:
            ctx.save_for_backward(x, threshold, ratio, attack, knee, makeup, ckpt)
        ctx.cfg = (kind, float(sample_rate), float(eps), int(lookahead))
        return y

    @staticmethod
    def backward(ctx, gy):
        lib = _abi.lib()
        x, threshold, ratio, attack, knee, makeup, ckpt = ctx.saved_tensors
        kind, sample_rate, eps, lookahead = ctx.cfg
        bs, chs, n = x.shape
        gy = gy.contiguous()
        gx = torch.empty_like(x)
        gp = torch.empty(bs, 6, dtype=torch.float32, device=x.device)
        scratch = torch.empty(bs * n, dtype=torch.float32, device=x.device) if lookahead > 0 else None
        with torch.cuda.device(x.device), _timed("comp_bwd", x.device):
            check(lib.dasp_dynamics_bwd(kind, ptr(gy), ptr(x), ptr(threshold), ptr(ratio), ptr(attack), ptr(knee),
                                        ptr(makeup), ptr(ckpt), ptr(gx), ptr(gp), ptr(scratch), bs, chs, n,
                                        sample_rate, eps, lookahead, stream_ptr(x.device)), "dasp_dynamics_bwd")
        return gx, gp[:, 0], gp[:, 1], gp[:, 2], gp[:, 4], gp[:, 5], None, None, None, None


SIDECHAIN_MAX_CHANNELS = 32
# the backward streams x, dL/dy and the key through shared memory: 2 * channels + key channels tiles per stage
SIDECHAIN_MAX_BUFFERS = 76


class _DynamicsSidechainFn(torch.autograd.Function):
    """The dynamics processor with the detector on a key (bs, K, n): kind 0 = compressor, 1 = expander."""

    @staticmethod
    def forward(ctx, x, key, threshold, ratio, attack, knee, makeup, kind, sample_rate, eps, lookahead):
        lib = _abi.lib()
        bs, chs, n = x.shape
        kc = key.shape[1]
        y = torch.empty_like(x)
        need_bwd = any(ctx.needs_input_grad[:7])
        ckpt = None
        with torch.cuda.device(x.device):
            if need_bwd:
                tile = lib.dasp_dynamics_sidechain_tile_len(bs, chs, kc)
                if tile <= 0:
                    raise DaspError(f"dynamics: unsupported channel counts {chs} (x) and {kc} (sidechain)")
                ckpt = torch.empty(bs * max(1, -(-n // tile)), dtype=torch.float32, device=x.device)
            with _timed("comp_sc_fwd", x.device):
                check(lib.dasp_dynamics_sidechain_fwd(kind, ptr(x), ptr(key), kc, ptr(threshold), ptr(ratio),
                                                      ptr(attack), ptr(knee), ptr(makeup), ptr(y), ptr(ckpt), bs, chs,
                                                      n, float(sample_rate), float(eps), int(lookahead),
                                                      stream_ptr(x.device)), "dasp_dynamics_sidechain_fwd")
        if need_bwd:
            ctx.save_for_backward(x, key, threshold, ratio, attack, knee, makeup, ckpt)
        ctx.cfg = (kind, float(sample_rate), float(eps), int(lookahead))
        return y

    @staticmethod
    def backward(ctx, gy):
        lib = _abi.lib()
        x, key, threshold, ratio, attack, knee, makeup, ckpt = ctx.saved_tensors
        kind, sample_rate, eps, lookahead = ctx.cfg
        bs, chs, n = x.shape
        gy = gy.contiguous()
        gx = torch.empty_like(x)
        # a fixed key (e.g. a voice-over ducking music) writes no key gradient
        gkey = torch.empty_like(key) if ctx.needs_input_grad[1] else None
        gp = torch.empty(bs, 6, dtype=torch.float32, device=x.device)
        scratch = torch.empty(bs * n, dtype=torch.float32, device=x.device) if lookahead > 0 else None
        with torch.cuda.device(x.device), _timed("comp_sc_bwd", x.device):
            check(lib.dasp_dynamics_sidechain_bwd(kind, ptr(gy), ptr(x), ptr(key), key.shape[1], ptr(threshold),
                                                  ptr(ratio), ptr(attack), ptr(knee), ptr(makeup), ptr(ckpt), ptr(gx),
                                                  ptr(gkey), ptr(gp), ptr(scratch), bs, chs, n, sample_rate, eps,
                                                  lookahead, stream_ptr(x.device)), "dasp_dynamics_sidechain_bwd")
        return gx, gkey, gp[:, 0], gp[:, 1], gp[:, 2], gp[:, 4], gp[:, 5], None, None, None, None


def _sidechain(sidechain, x):
    """validate the key against x (before any conversion or launch) -> (fp32 contiguous key, its dtype)"""
    if not torch.is_tensor(sidechain) or sidechain.dim() != 3:
        raise ValueError("sidechain must be a tensor of shape (batch, key_channels, samples)")
    if not torch.is_tensor(x) or x.dim() != 3:
        raise ValueError("x must be a tensor of shape (batch, channels, samples)")
    bs, chs, n = x.shape
    kb, kc, kn = sidechain.shape
    if kb != bs or kn != n:
        raise ValueError(f"sidechain has shape {tuple(sidechain.shape)}: its batch and length must equal x's {(bs, n)}")
    if not 1 <= kc <= SIDECHAIN_MAX_CHANNELS:
        raise ValueError(f"sidechain: 1 to {SIDECHAIN_MAX_CHANNELS} key channels are supported, got {kc}")
    if 2 * chs + kc > SIDECHAIN_MAX_BUFFERS:
        raise ValueError(f"sidechain: 2 * {chs} channels + {kc} key channels exceeds {SIDECHAIN_MAX_BUFFERS}")
    if sidechain.device != x.device:
        raise DaspError(f"sidechain is on {sidechain.device} but x is on {x.device}")
    return _audio(sidechain, "sidechain")


def _dynamics(kind, x, sample_rate, threshold_db, ratio, attack_ms, release_ms, knee_db, makeup_gain_db, eps,
              lookahead_samples, sidechain=None):
    key = _sidechain(sidechain, x)[0] if sidechain is not None else None
    xf, dt = _audio(x)
    bs = xf.shape[0]
    ps = [
        _param(p, bs, xf, name, allow_broadcast=True).contiguous()
        for p, name in (
            (threshold_db, "threshold_db"),
            (ratio, "ratio"),
            (attack_ms, "attack_ms"),
            (knee_db, "knee_db"),
            (makeup_gain_db, "makeup_gain_db"),
        )
    ]
    # release_ms is validated for shape only: the reference accepts and ignores it
    # (functional.py:333,343-344), so it receives no gradient here either.
    _param(release_ms, bs, xf, "release_ms", allow_broadcast=True)
    if key is not None:
        y = _DynamicsSidechainFn.apply(xf, key, *ps, kind, sample_rate, eps, int(lookahead_samples))
    else:
        y = _DynamicsFn.apply(xf, *ps, kind, sample_rate, eps, int(lookahead_samples))
    return y.to(dt)


def dynamics_packed(kind: int, x: torch.Tensor, sample_rate: float, params: torch.Tensor, eps: float = 1e-8,
                    lookahead_samples: int = 0, *, sidechain: Optional[torch.Tensor] = None):
    """compressor (kind 0) / expander (kind 1) with the six parameters stacked as ``(bs, 6)`` in signature order
    (threshold, ratio, attack, release, knee, makeup).  One transpose instead of six column copies.  ``sidechain``:
    ``None`` for ``compressor`` / ``expander``, a key tensor for ``sidechain_compressor`` / ``sidechain_expander``."""
    key = _sidechain(sidechain, x)[0] if sidechain is not None else None
    xf, dt = _audio(x)
    pt = _packed(params, xf.shape[0], 6, xf, "params").t().contiguous()        # (6, bs): rows are contiguous
    if key is not None:
        y = _DynamicsSidechainFn.apply(xf, key, pt[0], pt[1], pt[2], pt[4], pt[5], kind, sample_rate, eps,
                                       int(lookahead_samples))
    else:
        y = _DynamicsFn.apply(xf, pt[0], pt[1], pt[2], pt[4], pt[5], kind, sample_rate, eps, int(lookahead_samples))
    return y.to(dt)


def compressor(
    x: torch.Tensor,
    sample_rate: float,
    threshold_db: torch.Tensor,
    ratio: torch.Tensor,
    attack_ms: torch.Tensor,
    release_ms: torch.Tensor,
    knee_db: torch.Tensor,
    makeup_gain_db: torch.Tensor,
    eps: float = 1e-8,
    lookahead_samples: int = 0,
):
    """Feed-forward dynamic range compressor (reference ``functional.py:275-399``).

    Side chain = sum of the channels, soft-knee static curve, one-pole *attack* smoothing of the
    gain-reduction curve (``release_ms`` is accepted and ignored exactly like the reference),
    makeup gain, optional look-ahead delay of the audio path.  The smoother is evaluated as
    the true zero-state recursion; the reference's frequency-sampling evaluation on
    ``n_fft = 2**ceil(log2(2n-1))`` points is identical up to the time-aliased tail of the smoother's
    impulse response, whose size is ``alpha**(n_fft - n)`` of the gain curve with
    ``alpha = exp(-ln 9 / (sample_rate * attack_ms / 1e3))``: < 1e-15 at the BASELINE length
    (n = 48000), 1.7e-2 at n = 8192 and 0.6 at n = 1024 for a 100 ms attack at 44.1 kHz
    (``tests/test_gpu_dynamics.py::test_compressor_gap_to_the_frequency_sampling_reference``
    tracks the gap).
    """
    return _dynamics(0, x, sample_rate, threshold_db, ratio, attack_ms, release_ms, knee_db, makeup_gain_db, eps,
                     lookahead_samples)


def expander(
    x: torch.Tensor,
    sample_rate: float,
    threshold_db: torch.Tensor,
    ratio: torch.Tensor,
    attack_ms: torch.Tensor,
    release_ms: torch.Tensor,
    knee_db: torch.Tensor,
    makeup_gain_db: torch.Tensor,
    eps: float = 1e-8,
    lookahead_samples: int = 0,
):
    """Downward expander with the compressor's signature.

    The reference only stubs this op (``functional.py:402-403`` raises
    ``NotImplementedError``), so there is no reference parity to claim: the static curve is the
    soft-knee downward expander of Giannoulis et al. (2012) -- gain ``(R-1)(x_dB-T)`` below the
    knee, quadratic knee of width ``knee_db``, unity above -- followed by the compressor's
    attack smoother and makeup gain.  Pinned to ``oracle.expander``.
    """
    return _dynamics(1, x, sample_rate, threshold_db, ratio, attack_ms, release_ms, knee_db, makeup_gain_db, eps,
                     lookahead_samples)


def sidechain_compressor(
    x: torch.Tensor,
    sample_rate: float,
    threshold_db: torch.Tensor,
    ratio: torch.Tensor,
    attack_ms: torch.Tensor,
    release_ms: torch.Tensor,
    knee_db: torch.Tensor,
    makeup_gain_db: torch.Tensor,
    eps: float = 1e-8,
    lookahead_samples: int = 0,
    *,
    sidechain: torch.Tensor,
):
    """``compressor`` whose detector listens to an external side chain, the *key* (no reference counterpart: the
    reference always detects on ``x.sum(dim=1)``).  ``compressor`` keeps the reference's signature; this function has
    the same parameters plus the keyword-only ``sidechain``.

    ``sidechain`` is a tensor ``(bs, K, n)`` with ``1 <= K <= 32`` and ``2 * channels + K <= 76``, with x's batch and
    length and any channel count of its own.  The detector reads ``side = sidechain.sum(dim=1)`` (accumulated in fp64,
    rounded once to fp32) instead of x; level, static curve, attack smoother and makeup are the compressor's, and the
    gain is applied to every channel of x: ``y[b, c, t] = x[b, c, t - lookahead_samples] * G[b, t]``.  The look-ahead
    delays the audio path only, not the key.  Uses: ducking (music keyed by a voice-over), a de-esser keyed by
    ``parametric_eq(x, ...)`` with a presence boost (gradients reach the EQ parameters).

    Gradients: x receives ``dL/dy * G`` (shifted by the look-ahead, no detector term); every key channel receives the
    same ``dL/dside``, which carries ``1/side`` and is 0 where ``|side| < eps``; the parameters as in ``compressor``
    (``release_ms`` gets none).  The key may be in any floating dtype (computed in fp32, its gradient returned in its
    dtype); a key that does not require a gradient gets none written.  ``sidechain=x`` gives the same ``y`` as
    ``compressor``; x's gradient is then the sum of both paths.
    """
    return _dynamics(0, x, sample_rate, threshold_db, ratio, attack_ms, release_ms, knee_db, makeup_gain_db, eps,
                     lookahead_samples, sidechain)


def sidechain_expander(
    x: torch.Tensor,
    sample_rate: float,
    threshold_db: torch.Tensor,
    ratio: torch.Tensor,
    attack_ms: torch.Tensor,
    release_ms: torch.Tensor,
    knee_db: torch.Tensor,
    makeup_gain_db: torch.Tensor,
    eps: float = 1e-8,
    lookahead_samples: int = 0,
    *,
    sidechain: torch.Tensor,
):
    """``expander`` whose detector listens to the key ``sidechain``, exactly as ``sidechain_compressor`` does for
    the compressor: gating one track from another."""
    return _dynamics(1, x, sample_rate, threshold_db, ratio, attack_ms, release_ms, knee_db, makeup_gain_db, eps,
                     lookahead_samples, sidechain)


# --------------------------------------------------------------------------------------
# parametric EQ
# --------------------------------------------------------------------------------------


class _ParametricEqFn(torch.autograd.Function):
    """x (bs, chs, n), params (bs, 18) -> y; six-section biquad cascade."""

    @staticmethod
    def forward(ctx, x, params, sample_rate):
        lib = _abi.lib()
        bs, chs, n = x.shape
        y = torch.empty_like(x)
        need_bwd = any(ctx.needs_input_grad[:2])
        ckpt = None
        with torch.cuda.device(x.device):
            if need_bwd:
                ckpt = torch.empty(max(1, lib.dasp_eq_ckpt_floats(bs, chs, n)), dtype=torch.float32, device=x.device)
            with _timed("eq_fwd", x.device):
                check(lib.dasp_eq_fwd(ptr(x), ptr(params), ptr(y), ptr(ckpt), bs, chs, n, float(sample_rate),
                                      stream_ptr(x.device)), "dasp_eq_fwd")
        if need_bwd:
            ctx.save_for_backward(x, params, ckpt)
        ctx.sample_rate = float(sample_rate)
        return y

    @staticmethod
    def backward(ctx, gy):
        lib = _abi.lib()
        x, params, ckpt = ctx.saved_tensors
        bs, chs, n = x.shape
        gy = gy.contiguous()
        gx = torch.empty_like(x)
        gp = torch.empty_like(params)
        nws = lib.dasp_eq_bwd_workspace_floats(bs, chs)
        ws = _ws(nws, x.device)
        with torch.cuda.device(x.device), _timed("eq_bwd", x.device):
            check(lib.dasp_eq_bwd(ptr(gy), ptr(x), ptr(params), ptr(ckpt), ptr(gx), ptr(gp), ptr(ws), nws, bs, chs, n,
                                  ctx.sample_rate, stream_ptr(x.device)), "dasp_eq_bwd")
        return gx, gp, None


def parametric_eq(
    x: torch.Tensor,
    sample_rate: float,
    low_shelf_gain_db: torch.Tensor,
    low_shelf_cutoff_freq: torch.Tensor,
    low_shelf_q_factor: torch.Tensor,
    band0_gain_db: torch.Tensor,
    band0_cutoff_freq: torch.Tensor,
    band0_q_factor: torch.Tensor,
    band1_gain_db: torch.Tensor,
    band1_cutoff_freq: torch.Tensor,
    band1_q_factor: torch.Tensor,
    band2_gain_db: torch.Tensor,
    band2_cutoff_freq: torch.Tensor,
    band2_q_factor: torch.Tensor,
    band3_gain_db: torch.Tensor,
    band3_cutoff_freq: torch.Tensor,
    band3_q_factor: torch.Tensor,
    high_shelf_gain_db: torch.Tensor,
    high_shelf_cutoff_freq: torch.Tensor,
    high_shelf_q_factor: torch.Tensor,
):
    """Six-band parametric equaliser: low shelf -> four peaking bands -> high shelf
    (reference ``functional.py:118-272``).

    Each parameter holds ``bs`` elements in any shape, or a single element that is broadcast
    over the batch (reference ``examples/virtual_analog.py:204-206``); integer cut-offs are
    accepted (``examples/demo.py:44``).  All channels of an item share the item's filter.

    The cascade is run as the true zero-state recursion (time-parallel scan, fp32 sigma-form
    sections designed in fp64); the reference evaluates the same filter by frequency sampling
    on ``n_fft = 2**ceil(log2(2n-1))`` points, which coincides with it whenever the impulse
    response fits in the ``n_fft - n`` samples of padding: wrap-around < e^-19 for every filter
    of the ``ParametricEQ`` ranges at n = 48000, but up to 3 % for a 20 Hz shelf at n = 4096
    (item 0 of ``tests/golden/parametric_eq.npz`` keeps such a case; DESIGN.md section 2).
    """
    xf, dt = _audio(x)
    bs = xf.shape[0]
    plist = (
        low_shelf_gain_db, low_shelf_cutoff_freq, low_shelf_q_factor,
        band0_gain_db, band0_cutoff_freq, band0_q_factor,
        band1_gain_db, band1_cutoff_freq, band1_q_factor,
        band2_gain_db, band2_cutoff_freq, band2_q_factor,
        band3_gain_db, band3_cutoff_freq, band3_q_factor,
        high_shelf_gain_db, high_shelf_cutoff_freq, high_shelf_q_factor,
    )
    packed = torch.stack([_param(p, bs, xf, f"parametric_eq parameter {i}", allow_broadcast=True)
                          for i, p in enumerate(plist)], dim=1).contiguous()
    y = _ParametricEqFn.apply(xf, packed, sample_rate)
    return y.to(dt)


def _packed(params, bs: int, ncol: int, like: torch.Tensor, name: str) -> torch.Tensor:
    if not torch.is_tensor(params) or params.dim() != 2 or tuple(params.shape) != (bs, ncol):
        raise ValueError(f"{name}: expected a ({bs}, {ncol}) parameter tensor, got {tuple(getattr(params, 'shape', ()))}")
    if params.device != like.device:
        raise DaspError(f"{name} is on {params.device} but x is on {like.device}")
    return params.to(torch.float32).contiguous()


def parametric_eq_packed(x: torch.Tensor, sample_rate: float, params: torch.Tensor):
    """``parametric_eq`` with its 18 parameters already stacked as ``(bs, 18)`` in signature order (physical
    units).  Used by ``modules.ParametricEQ.process_normalized`` so that the whole normalised-parameter path is
    one affine kernel + the EQ kernels (SURVEY.md 8f rank 1); gradients flow to ``params``."""
    xf, dt = _audio(x)
    return _ParametricEqFn.apply(xf, _packed(params, xf.shape[0], 18, xf, "params"), sample_rate).to(dt)


# --------------------------------------------------------------------------------------
# noise-shaped reverberation
# --------------------------------------------------------------------------------------

import os as _os

# Items per pass of the reverb pipeline (bounds the workspace).  Default: two items per SM of the device, so that the
# one-CTA-per-SM FFT kernels run in whole waves (ifft_shape_kernel: R CTAs per item -> exactly 2 R waves; the persistent
# block-transform kernels: the same number of blocks per CTA).  Measured on one H100 SXM (400 W), chain step at batch
# 1024: 66 items 23.4 ms, 132 items 22.5 ms, 264 items 22.1 ms.  With the forward's convolution of chunk k overlapping
# the IR synthesis of chunk k + 1 (smaller chunks would shorten the convolution left after the last synthesis), two
# runs each on an H100 80GB HBM3 at a 400 W limit: 132 items 20.26 / 20.52 ms (reverb_bwd 5.30 / 5.33 ms), 264 items
# 19.99 / 18.94 ms (reverb_bwd 5.11 / 5.12 ms).  Override for experiments with DASP_REVERB_CHUNK.
REVERB_CHUNK_ITEMS = int(_os.environ.get("DASP_REVERB_CHUNK", "0"))      # 0 = automatic


def reverb_chunk_items(device) -> int:
    """Items per pass of the reverb pipeline on ``device`` (see REVERB_CHUNK_ITEMS)."""
    if REVERB_CHUNK_ITEMS > 0:
        return REVERB_CHUNK_ITEMS
    return 2 * int(torch.cuda.get_device_properties(device).multi_processor_count)


def _noise_or_seed(noise, xf, bs, num_samples, num_bandpass_taps):
    """parity mode: validate the caller's noise tensor; default mode: draw the 64-bit Philox key ON THE DEVICE.

    The reference draws its noise with ``torch.randn`` (``functional.py:547-548``), which is reproducible under
    ``torch.manual_seed`` and, on CUDA, graph-safe (fresh values on every replay of a captured graph).  The key of
    the in-kernel generator is therefore one ``random_()`` word of torch's CUDA generator, left in device memory
    and read by the kernels when they run: no host round trip, same reproducibility, and a captured graph
    re-draws it on every replay (torch registers the generator's Philox offset with the graph)."""
    if noise is not None:
        expect = (bs * 2, 12, num_samples + num_bandpass_taps - 1)
        if tuple(noise.shape) != expect:
            raise ValueError(f"noise must have shape {expect}, got {tuple(noise.shape)}")
        return noise.to(device=xf.device, dtype=torch.float32).contiguous(), None
    return None, torch.empty(1, dtype=torch.int64, device=xf.device).random_()


class _ReverbFn(torch.autograd.Function):
    """x (bs, 1|2, n), params (bs, 25) -> y (bs, 2, n)."""

    @staticmethod
    def forward(ctx, x, params, noise, seed, sample_rate, num_samples, taps, chunk):
        lib = _abi.lib()
        bs, in_chs, n = x.shape
        dev = x.device
        y = torch.empty(bs, 2, n, dtype=torch.float32, device=dev)
        need_bwd = any(ctx.needs_input_grad[:2])
        geom = _abi.ReverbGeom()
        with torch.cuda.device(dev):
            check(lib.dasp_reverb_geometry(bs, n, num_samples, taps, chunk, geom), "dasp_reverb_geometry")
            ws = torch.empty(max(geom.fwd_workspace_bytes, 16), dtype=torch.uint8, device=dev)
            fsave = xspec = irspec = None
            if need_bwd:
                fsave = torch.empty(geom.f_floats, dtype=torch.float32, device=dev)
                xspec = torch.empty(geom.xspec_c64, dtype=torch.complex64, device=dev)
                irspec = torch.empty(geom.irspec_c64, dtype=torch.complex64, device=dev)
            with _timed("reverb_fwd", dev):
                check(lib.dasp_reverb_fwd(ptr(x), in_chs, ptr(params), ptr(noise), ptr(seed), ptr(y), ptr(fsave),
                                          ptr(xspec), ptr(irspec), ptr(ws), ws.numel(), bs, n, num_samples, taps, chunk,
                                          float(sample_rate), stream_ptr(dev)), "dasp_reverb_fwd")
        if need_bwd:
            # slot 2 (the wet signal, which the backward no longer needs) stays empty so that callers that inspect
            # grad_fn.saved_tensors keep the layout (x, params, -, f, X spectra, IR spectra)
            ctx.save_for_backward(x, params, None, fsave, xspec, irspec)
        ctx.cfg = (num_samples, taps, chunk, geom.bwd_workspace_bytes, 1 if noise is None else 0)
        return y

    @staticmethod
    def backward(ctx, gy):
        lib = _abi.lib()
        x, params, _, fsave, xspec, irspec = ctx.saved_tensors
        num_samples, taps, chunk, bwd_bytes, device_noise = ctx.cfg
        bs, in_chs, n = x.shape
        dev = x.device
        gy = gy.contiguous()
        gx = torch.empty_like(x)
        gp = torch.empty_like(params)
        ws = torch.empty(max(bwd_bytes, 16), dtype=torch.uint8, device=dev)
        with torch.cuda.device(dev), _timed("reverb_bwd", dev):
            check(lib.dasp_reverb_bwd(ptr(gy), ptr(x), in_chs, ptr(params), ptr(fsave), ptr(xspec), ptr(irspec),
                                      ptr(gx), ptr(gp), ptr(ws), ws.numel(), bs, n, num_samples, taps, chunk,
                                      device_noise, stream_ptr(dev)), "dasp_reverb_bwd")
        return gx, gp, None, None, None, None, None, None


def noise_shaped_reverberation(
    x: torch.Tensor,
    sample_rate: float,
    band0_gain: torch.Tensor,
    band1_gain: torch.Tensor,
    band2_gain: torch.Tensor,
    band3_gain: torch.Tensor,
    band4_gain: torch.Tensor,
    band5_gain: torch.Tensor,
    band6_gain: torch.Tensor,
    band7_gain: torch.Tensor,
    band8_gain: torch.Tensor,
    band9_gain: torch.Tensor,
    band10_gain: torch.Tensor,
    band11_gain: torch.Tensor,
    band0_decay: torch.Tensor,
    band1_decay: torch.Tensor,
    band2_decay: torch.Tensor,
    band3_decay: torch.Tensor,
    band4_decay: torch.Tensor,
    band5_decay: torch.Tensor,
    band6_decay: torch.Tensor,
    band7_decay: torch.Tensor,
    band8_decay: torch.Tensor,
    band9_decay: torch.Tensor,
    band10_decay: torch.Tensor,
    band11_decay: torch.Tensor,
    mix: torch.Tensor,
    num_samples: int = 65536,
    num_bandpass_taps: int = 1023,
    *,
    noise: Optional[torch.Tensor] = None,
):
    """Filtered-noise artificial reverberation (reference ``functional.py:406-577``).

    Twelve bands (12 Hz low-pass, ten octave band-passes, 18 kHz high-pass; ``signal.py:42-92``),
    each a white-noise signal filtered by a ``num_bandpass_taps`` FIR, shaped by
    ``exp(-(10*decay+1)*t)`` and its gain, averaged into a ``num_samples``-long stereo impulse
    response that is convolved with the input; ``mix`` blends wet and dry.  Mono input is
    duplicated and the output is always stereo, like the reference.

    Keyword-only extension ``noise``: the reference draws
    ``torch.randn(bs*2, 12, num_samples + num_bandpass_taps - 1)`` inside the call
    (``functional.py:547-548``).  Pass that tensor here to reproduce a seeded reference call
    exactly (parity tests); by default fresh N(0,1) noise is generated on the device with
    Philox4x32-10, keyed by one 64-bit word drawn from torch's CUDA generator and kept in device
    memory (``torch.manual_seed`` makes the call reproducible; a captured CUDA graph draws fresh
    noise on every replay, like the reference's ``torch.randn`` would).
    """
    assert num_bandpass_taps % 2 == 1, "num_bandpass_taps must be odd"
    xf, dt = _audio(x)
    bs, chs, n = xf.shape
    assert chs <= 2, "only mono/stereo signals are supported"
    plist = (
        band0_gain, band1_gain, band2_gain, band3_gain, band4_gain, band5_gain,
        band6_gain, band7_gain, band8_gain, band9_gain, band10_gain, band11_gain,
        band0_decay, band1_decay, band2_decay, band3_decay, band4_decay, band5_decay,
        band6_decay, band7_decay, band8_decay, band9_decay, band10_decay, band11_decay,
        mix,
    )
    packed = torch.stack([_param(p, bs, xf, f"noise_shaped_reverberation parameter {i}", allow_broadcast=True)
                          for i, p in enumerate(plist)], dim=1).contiguous()
    noise, seed = _noise_or_seed(noise, xf, bs, num_samples, num_bandpass_taps)
    y = _ReverbFn.apply(xf, packed, noise, seed, sample_rate, int(num_samples), int(num_bandpass_taps),
                        reverb_chunk_items(xf.device))
    return y.to(dt)


def noise_shaped_reverberation_packed(x: torch.Tensor, sample_rate: float, params: torch.Tensor, num_samples: int = 65536,
                                      num_bandpass_taps: int = 1023, *, noise: Optional[torch.Tensor] = None):
    """``noise_shaped_reverberation`` with its 25 parameters stacked as ``(bs, 25)`` (12 gains, 12 decays, mix)."""
    assert num_bandpass_taps % 2 == 1, "num_bandpass_taps must be odd"
    xf, dt = _audio(x)
    bs, chs, _ = xf.shape
    assert chs <= 2, "only mono/stereo signals are supported"
    packed = _packed(params, bs, 25, xf, "params")
    noise, seed = _noise_or_seed(noise, xf, bs, num_samples, num_bandpass_taps)
    y = _ReverbFn.apply(xf, packed, noise, seed, sample_rate, int(num_samples), int(num_bandpass_taps),
                        reverb_chunk_items(xf.device))
    return y.to(dt)


# --------------------------------------------------------------------------------------
# convolution reverberation (caller-supplied impulse response)
# --------------------------------------------------------------------------------------


class _ConvReverbFn(torch.autograd.Function):
    """x (bs, 1|2, n), ir (bs, 1|2|4, L), mix (bs,) -> y (bs, 2, n).  An ir of batch 1 with bs > 1 is one IR shared by
    the batch (the dasp_conv_shared_* entry points): its gradient is the sum over the items, shape (1, 1|2|4, L).  A
    4-channel (true-stereo) IR is sized by the *_ts_geometry queries and runs through the same entry points."""

    @staticmethod
    def forward(ctx, x, ir, mix, chunk):
        lib = _abi.lib()
        bs, in_chs, n = x.shape
        ir_bs, ir_chs, ir_len = ir.shape
        shared = ir_bs == 1 and bs > 1
        kind = "conv_shared" if shared else "conv"
        geom_fn = f"dasp_{kind}{'_ts' if ir_chs == 4 else ''}_geometry"
        dev = x.device
        y = torch.empty(bs, 2, n, dtype=torch.float32, device=dev)
        need_bwd = any(ctx.needs_input_grad[:3])
        geom = _abi.ConvGeom()
        with torch.cuda.device(dev):
            check(getattr(lib, geom_fn)(bs, n, ir_len, chunk, geom), geom_fn)
            ws = torch.empty(max(geom.fwd_workspace_bytes, 16), dtype=torch.uint8, device=dev)
            xspec = irspec = None
            if need_bwd:
                xspec = torch.empty(geom.xspec_c64, dtype=torch.complex64, device=dev)
                irspec = torch.empty(geom.irspec_c64, dtype=torch.complex64, device=dev)
            with _timed("conv_fwd", dev):
                check(getattr(lib, f"dasp_{kind}_fwd")(ptr(x), in_chs, ptr(ir), ir_chs, ir_len, ptr(mix), ptr(y),
                                                       ptr(xspec), ptr(irspec), ptr(ws), ws.numel(), bs, n, chunk,
                                                       stream_ptr(dev)),
                      f"dasp_{kind}_fwd")
        if need_bwd:
            ctx.save_for_backward(x, xspec, irspec, mix)
        ctx.cfg = (kind, ir_bs, ir_chs, ir_len, chunk, geom.bwd_workspace_bytes)
        return y

    @staticmethod
    def backward(ctx, gy):
        lib = _abi.lib()
        x, xspec, irspec, mix = ctx.saved_tensors
        kind, ir_bs, ir_chs, ir_len, chunk, bwd_bytes = ctx.cfg
        bs, in_chs, n = x.shape
        dev = x.device
        gy = gy.contiguous()
        gx = torch.empty_like(x)
        # a fixed IR (data augmentation with measured rooms) skips every dL/dIR kernel
        gir = torch.empty(ir_bs, ir_chs, ir_len, dtype=torch.float32, device=dev) if ctx.needs_input_grad[1] else None
        gmix = torch.empty_like(mix)
        ws = torch.empty(max(bwd_bytes, 16), dtype=torch.uint8, device=dev)
        with torch.cuda.device(dev), _timed("conv_bwd", dev):
            check(getattr(lib, f"dasp_{kind}_bwd")(ptr(gy), ptr(x), in_chs, ir_chs, ir_len, ptr(mix), ptr(xspec),
                                                   ptr(irspec), ptr(gx), ptr(gir), ptr(gmix), ptr(ws), ws.numel(), bs,
                                                   n, chunk, stream_ptr(dev)),
                  f"dasp_{kind}_bwd")
        return gx, gir, gmix, None


def convolution_reverberation(x: torch.Tensor, sample_rate: float, impulse_response: torch.Tensor, mix: torch.Tensor):
    """Convolution reverb with a caller-supplied impulse response: the apply stage of the reference's
    ``noise_shaped_reverberation`` (``functional.py:569-575``) with the IR given instead of synthesised::

        x_pad = pad(x, (L-1, 0)); wet = vmap(conv1d(groups=2))(x_pad, flip(IR)); y = (1-mix) x + mix wet

    Args:
        x: audio ``(bs, 1|2, n)``; mono is used for both channels.
        sample_rate: unused (kept for the common processor signature).
        impulse_response: ``(bs, 1|2|4, L)``, one IR per item, or ``(1, 1|2|4, L)``, one IR for the whole batch (a
            measured room applied to every item, or a single learnt FIR reverb); any ``L >= 1``; a mono IR is used for
            both channels.  Four channels are a true-stereo IR in input-major order: channel ``2 i + o`` is the path
            from input channel ``i`` to output channel ``o``, i.e. L->L, L->R, R->L, R->R, so that::

                wet_L = x_L * h0 + x_R * h2,   wet_R = x_L * h1 + x_R * h3,   y = (1 - mix) x + mix wet

            (``*`` the causal convolution cropped to ``n``; a mono ``x`` feeds both inputs, ``wet_L = x * (h0 + h2)``).
        mix: ``bs`` elements in any shape, or one element that is broadcast over the batch.

    Returns ``(bs, 2, n)`` in x's dtype (computed in fp32), like ``noise_shaped_reverberation``, so the two can replace
    each other in a chain.  Gradients flow to ``x``, ``impulse_response`` (a mono IR receives the sum of both channel
    gradients; taps at or beyond ``n`` reach no output and get exactly 0) and ``mix``.  The gradient of a ``(1, 1|2, L)``
    IR has that shape and is the sum over the items of each item's gradient, accumulated in fp64 in item order, so it
    does not depend on how the batch is chunked.  A shared IR is transformed once per call rather than once per item,
    and no per-item copy of it or of its gradient is ever made; ``ir.expand(bs, -1, -1)`` gives the same result at the
    per-item cost.  A true-stereo IR takes one window transform and one inverse transform per block, like a stereo one,
    where two stereo calls with ``(h0, h1)`` and ``(h2, h3)`` would take two of each; its gradient reaches all four
    channels.  When the IR does not require a gradient, the backward skips all dL/dIR work.  The convolution is the
    reverb's own: uniformly partitioned overlap-save on 4096-sample partitions with the in-shared-memory 8192-point FFT.
    """
    for t, name, chans, what in ((x, "x", (1, 2), "mono/stereo"),
                                 (impulse_response, "impulse_response", (1, 2, 4), "mono/stereo/true-stereo (4)")):
        if not torch.is_tensor(t) or t.dim() != 3:
            raise ValueError(f"{name} must be a tensor of shape (batch, channels, samples)")
        if t.shape[1] not in chans:
            raise ValueError(f"{name}: only {what} is supported, got {t.shape[1]} channels")
    bs = x.shape[0]
    if impulse_response.shape[0] != bs and not (impulse_response.shape[0] == 1 and bs > 1):
        raise ValueError(f"impulse_response has batch {impulse_response.shape[0]}, x has batch {bs} (expected {bs} or 1)")
    if impulse_response.shape[2] < 1:
        raise ValueError("impulse_response needs at least one tap")
    nmix = mix.numel() if torch.is_tensor(mix) else torch.as_tensor(mix).numel()
    if nmix not in (1, bs):
        raise ValueError(f"mix: expected {bs} element(s) (one per batch item) or 1, got {nmix}")
    xf, dt = _audio(x)
    irf, _ = _audio(impulse_response, "impulse_response")
    if irf.device != xf.device:
        raise DaspError(f"impulse_response is on {irf.device} but x is on {xf.device}")
    m = _param(mix, bs, xf, "mix", allow_broadcast=True).contiguous()
    y = _ConvReverbFn.apply(xf, irf, m, reverb_chunk_items(xf.device))
    return y.to(dt)
