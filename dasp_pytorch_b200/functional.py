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
    "compressor_gain",
    "expander_gain",
    "noise_shaped_reverberation",
    "convolution_reverberation",
    "convolution_bus",
    "multichannel_convolution",
    "time_varying_convolution_reverberation",
    "time_varying_convolution_bus",
    "time_varying_multichannel_convolution",
    "noise_shaped_impulse_response",
    "noise_shaped_impulse_response_packed",
    "parametric_eq_frequency_response",
    "parametric_eq_frequency_response_packed",
]


# --------------------------------------------------------------------------------------
# helpers
# --------------------------------------------------------------------------------------


def _audio(x: torch.Tensor, name: str = "x", rank: Optional[int] = None):
    """validate the (bs, chs, n) audio tensor, or one of rank ``rank`` -> (fp32 contiguous tensor, original dtype)"""
    if not torch.is_tensor(x) or x.dim() != (3 if rank is None else rank):
        raise ValueError(f"{name} must be a tensor of shape (batch, channels, samples)" if rank is None else
                         f"{name} must be a {rank}-dimensional tensor")
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


def _stack_params(plist, bs: int, like: torch.Tensor, what: str) -> torch.Tensor:
    """the parameters ``plist`` of op ``what``, each ``bs`` elements or one broadcast, as fp32 ``(bs, P)``"""
    return torch.stack([_param(p, bs, like, f"{what} parameter {i}", allow_broadcast=True)
                        for i, p in enumerate(plist)], dim=1).contiguous()


def _packed_shape(params, ncol: int, bs: Optional[int] = None):
    """packed parameters must be a ``(bs, ncol)`` tensor; without ``bs`` (the parameter-only ops) any batch"""
    if (not torch.is_tensor(params) or params.dim() != 2 or params.shape[1] != ncol
            or bs is not None and params.shape[0] != bs):
        raise ValueError(f"params: expected a ({'bs' if bs is None else bs}, {ncol}) parameter tensor, got "
                         f"{tuple(getattr(params, 'shape', ()))}")


def _packed(params, ncol: int, like: torch.Tensor) -> torch.Tensor:
    """the ``(bs, ncol)`` packed parameters of an op on x = ``like``, as fp32 contiguous"""
    _packed_shape(params, ncol, like.shape[0])
    if params.device != like.device:
        raise DaspError(f"params is on {params.device} but x is on {like.device}")
    return params.to(torch.float32).contiguous()


def _ws(n_floats: int, device) -> torch.Tensor:
    return torch.empty(max(int(n_floats), 1), dtype=torch.float32, device=device)


def _ws_bytes(n_bytes: int, device) -> torch.Tensor:
    return torch.empty(max(int(n_bytes), 16), dtype=torch.uint8, device=device)


def _params_device(tensors, what):
    """the one CUDA device of an op's parameter tensors (plain numbers have none)"""
    devs = {t.device for t in tensors if torch.is_tensor(t)}
    if len(devs) > 1:
        raise DaspError(f"{what}: parameters on several devices {sorted(map(str, devs))}")
    dev = next(iter(devs)) if devs else torch.device("cpu")
    if dev.type != "cuda":
        raise DaspError(f"{what}: parameters are on {dev}: dasp_pytorch_b200 only runs on CUDA "
                        "(H100) tensors and has no CPU path")
    return dev


def _promoted_dtype(tensors):
    dts = [t.dtype for t in tensors if torch.is_tensor(t) and t.is_floating_point()]
    out = dts[0] if dts else torch.float32
    for d in dts[1:]:
        out = torch.promote_types(out, d)
    return out


def _params_batch(plist, what: str) -> int:
    """the batch of a parameter-only op: the largest element count, which every parameter holds, or one element"""
    counts = [p.numel() if torch.is_tensor(p) else torch.as_tensor(p).numel() for p in plist]
    bs = max(counts)
    for i, c in enumerate(counts):
        if c not in (1, bs):
            raise ValueError(f"{what} parameter {i}: expected {bs} element(s) (one per batch item) or 1, got {c}")
    return bs


def _params_stacked(plist, bs: int, what: str):
    """a parameter-only op's parameters -> (fp32 ``(bs, P)`` on their one CUDA device, their promoted dtype)"""
    dev = _params_device(plist, what)
    return _stack_params(plist, bs, torch.empty(0, device=dev), what), _promoted_dtype(plist)


def _packed_params(params, what: str):
    """a parameter-only op's ``(bs, P)`` packed parameters -> (fp32 contiguous on their CUDA device, their dtype)"""
    dev = _params_device([params], what)
    dt = params.dtype if params.is_floating_point() else torch.float32
    return params.to(device=dev, dtype=torch.float32).contiguous(), dt


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


def stereo_widener(x: torch.Tensor, sample_rate: float, width: torch.Tensor):
    """Mid/side stereo widener (reference ``functional.py:580-604``).

    ``x`` is ``(bs, 2, seq_len)``, ``width`` holds ``bs`` elements (0 = mono sum, 0.5 = unchanged,
    1 = side only).  mid = (L+R)/sqrt2 scaled by 2(1-width), side = (L-R)/sqrt2 scaled by 2 width.
    """
    xf, dt = _audio(x, rank=3)
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
    xf, dt = _audio(x, rank=3)
    bs, tracks, _ = xf.shape
    pn = _param(pan, bs * tracks, xf, "pan").contiguous()
    return _StereoFn.apply(xf, pn, "panner").to(dt)


def stereo_bus(x: torch.Tensor, sample_rate: int, send_db: torch.Tensor):
    """Sum stereo tracks to a stereo bus with per-track send levels in dB (reference ``functional.py:32-62``).

    ``x`` is ``(bs, 2, tracks, seq_len)``, ``send_db`` holds ``bs*tracks`` elements; returns ``(bs, 2, seq_len)``.
    """
    xf, dt = _audio(x, rank=4)
    bs, chs, tracks, _ = xf.shape
    assert chs == 2, "Input tensor must have shape (bs, 2, tracks, seq_len)"
    sd = _param(send_db, bs * tracks, xf, "send_db").contiguous()
    return _StereoFn.apply(xf, sd, "bus").to(dt)


# --------------------------------------------------------------------------------------
# compressor / expander
# --------------------------------------------------------------------------------------


# the detector's channel limit (kMaxChs in dynamics.cu): x's channels for the gain ops, the key's for the side chain
DYNAMICS_MAX_CHANNELS = 32
SIDECHAIN_MAX_CHANNELS = DYNAMICS_MAX_CHANNELS
# the backward streams x, dL/dy and the key through shared memory: 2 * channels + key channels tiles per stage
SIDECHAIN_MAX_BUFFERS = 76


class _DynamicsFn(torch.autograd.Function):
    """Feed-forward dynamics processor: kind 0 = compressor, 1 = expander.  The detector listens to x, or to
    ``key`` (bs, K, n) when one is given."""

    @staticmethod
    def forward(ctx, x, key, threshold, ratio, attack, knee, makeup, kind, sample_rate, eps, lookahead):
        lib = _abi.lib()
        bs, chs, n = x.shape
        y = torch.empty_like(x)
        need_bwd = any(ctx.needs_input_grad[:7])
        ckpt = None
        with torch.cuda.device(x.device):
            if need_bwd:
                # depends on the device's SM count
                if key is None:
                    tile = lib.dasp_dynamics_tile_len(bs, chs)
                    what = f"channel count {chs}"
                else:
                    tile = lib.dasp_dynamics_sidechain_tile_len(bs, chs, key.shape[1])
                    what = f"channel counts {chs} (x) and {key.shape[1]} (sidechain)"
                if tile <= 0:
                    raise DaspError(f"dynamics: unsupported {what}")
                ckpt = torch.empty(bs * max(1, -(-n // tile)), dtype=torch.float32, device=x.device)
            args = (ptr(threshold), ptr(ratio), ptr(attack), ptr(knee), ptr(makeup), ptr(y), ptr(ckpt), bs, chs, n,
                    float(sample_rate), float(eps), int(lookahead), stream_ptr(x.device))
            if key is None:
                with _timed("comp_fwd", x.device):
                    check(lib.dasp_dynamics_fwd(kind, ptr(x), *args), "dasp_dynamics_fwd")
            else:
                with _timed("comp_sc_fwd", x.device):
                    check(lib.dasp_dynamics_sidechain_fwd(kind, ptr(x), ptr(key), key.shape[1], *args),
                          "dasp_dynamics_sidechain_fwd")
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
        with torch.cuda.device(x.device):
            params = (ptr(threshold), ptr(ratio), ptr(attack), ptr(knee), ptr(makeup), ptr(ckpt), ptr(gx))
            tail = (ptr(gp), ptr(scratch), bs, chs, n, sample_rate, eps, lookahead, stream_ptr(x.device))
            if key is None:
                with _timed("comp_bwd", x.device):
                    check(lib.dasp_dynamics_bwd(kind, ptr(gy), ptr(x), *params, *tail), "dasp_dynamics_bwd")
            else:
                with _timed("comp_sc_bwd", x.device):
                    check(lib.dasp_dynamics_sidechain_bwd(kind, ptr(gy), ptr(x), ptr(key), key.shape[1], *params,
                                                          ptr(gkey), *tail), "dasp_dynamics_sidechain_bwd")
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


def _dynamics_params(threshold_db, ratio, attack_ms, release_ms, knee_db, makeup_gain_db):
    """-> ``pack(x)``: the five ``(bs,)`` columns the dynamics kernels read, kept apart (a stack would add a launch)"""
    def pack(like):
        bs = like.shape[0]
        ps = [
            _param(p, bs, like, name, allow_broadcast=True).contiguous()
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
        _param(release_ms, bs, like, "release_ms", allow_broadcast=True)
        return ps
    return pack


def _dynamics_params_packed(params):
    """``(bs, 6)`` packed dynamics parameters -> ``pack(x)``: the same five columns, rows of one transpose"""
    def pack(like):
        pt = _packed(params, 6, like).t().contiguous()        # (6, bs): rows are contiguous
        return pt[0], pt[1], pt[2], pt[4], pt[5]
    return pack


def _dynamics(kind, x, sample_rate, pack, eps, lookahead_samples, sidechain=None):
    """the body of the compressor / expander ops and dynamics_packed; ``pack(xf)`` checks and packs the parameters"""
    key = _sidechain(sidechain, x)[0] if sidechain is not None else None
    xf, dt = _audio(x)
    y = _DynamicsFn.apply(xf, key, *pack(xf), kind, sample_rate, eps, int(lookahead_samples))
    return y.to(dt)


def dynamics_packed(kind: int, x: torch.Tensor, sample_rate: float, params: torch.Tensor, eps: float = 1e-8,
                    lookahead_samples: int = 0, *, sidechain: Optional[torch.Tensor] = None):
    """compressor (kind 0) / expander (kind 1) with the six parameters stacked as ``(bs, 6)`` in signature order
    (threshold, ratio, attack, release, knee, makeup).  One transpose instead of six column copies.  ``sidechain``:
    ``None`` for ``compressor`` / ``expander``, a key tensor for ``sidechain_compressor`` / ``sidechain_expander``."""
    return _dynamics(kind, x, sample_rate, _dynamics_params_packed(params), eps, lookahead_samples, sidechain)


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
    pack = _dynamics_params(threshold_db, ratio, attack_ms, release_ms, knee_db, makeup_gain_db)
    return _dynamics(0, x, sample_rate, pack, eps, lookahead_samples)


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
    pack = _dynamics_params(threshold_db, ratio, attack_ms, release_ms, knee_db, makeup_gain_db)
    return _dynamics(1, x, sample_rate, pack, eps, lookahead_samples)


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
    pack = _dynamics_params(threshold_db, ratio, attack_ms, release_ms, knee_db, makeup_gain_db)
    return _dynamics(0, x, sample_rate, pack, eps, lookahead_samples, sidechain)


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
    pack = _dynamics_params(threshold_db, ratio, attack_ms, release_ms, knee_db, makeup_gain_db)
    return _dynamics(1, x, sample_rate, pack, eps, lookahead_samples, sidechain)


# --------------------------------------------------------------------------------------
# the compressor's / expander's gain curve
# --------------------------------------------------------------------------------------


class _DynamicsGainFn(torch.autograd.Function):
    """Detector input x (bs, C, n) -> the gain (bs, 1, n): G, or s + M in dB when ``db``.  kind 0 = compressor,
    1 = expander.  The backward writes dL/dside once per item and hands it to every channel as an expanded view."""

    @staticmethod
    def forward(ctx, x, threshold, ratio, attack, knee, makeup, kind, sample_rate, eps, db):
        lib = _abi.lib()
        bs, chs, n = x.shape
        g = torch.empty(bs, 1, n, dtype=torch.float32, device=x.device)
        need_bwd = any(ctx.needs_input_grad[:6])
        ckpt = None
        with torch.cuda.device(x.device):
            if need_bwd:
                tile = lib.dasp_dynamics_tile_len(bs, chs)           # the compressor's tiles for (bs, chs)
                if tile <= 0:
                    raise DaspError(f"dynamics gain: unsupported channel count {chs}")
                ckpt = torch.empty(bs * max(1, -(-n // tile)), dtype=torch.float32, device=x.device)
            with _timed("dyn_gain_fwd", x.device):
                check(lib.dasp_dynamics_gain_fwd(kind, ptr(x), chs, ptr(threshold), ptr(ratio), ptr(attack), ptr(knee),
                                                 ptr(makeup), ptr(g), ptr(ckpt), bs, n, float(sample_rate), float(eps),
                                                 int(db), stream_ptr(x.device)), "dasp_dynamics_gain_fwd")
        if need_bwd:
            ctx.save_for_backward(x, threshold, ratio, attack, knee, makeup, ckpt)
        ctx.cfg = (kind, float(sample_rate), float(eps), int(db))
        return g

    @staticmethod
    def backward(ctx, gg):
        lib = _abi.lib()
        x, threshold, ratio, attack, knee, makeup, ckpt = ctx.saved_tensors
        kind, sample_rate, eps, db = ctx.cfg
        bs, chs, n = x.shape
        gg = gg.contiguous()
        gside = torch.empty(bs, 1, n, dtype=torch.float32, device=x.device)
        gp = torch.empty(bs, 6, dtype=torch.float32, device=x.device)
        with torch.cuda.device(x.device), _timed("dyn_gain_bwd", x.device):
            check(lib.dasp_dynamics_gain_bwd(kind, ptr(gg), ptr(x), ptr(threshold), ptr(ratio), ptr(attack), ptr(knee),
                                             ptr(makeup), ptr(ckpt), ptr(gside), ptr(gp), bs, chs, n, sample_rate, eps,
                                             db, stream_ptr(x.device)), "dasp_dynamics_gain_bwd")
        gx = gside.expand(bs, chs, n) if ctx.needs_input_grad[0] else None
        return gx, gp[:, 0], gp[:, 1], gp[:, 2], gp[:, 4], gp[:, 5], None, None, None, None


def _gain_input(x):
    """rank and channel count of the detector input, checked before anything touches a device"""
    if not torch.is_tensor(x) or x.dim() != 3:
        raise ValueError("x must be a tensor of shape (batch, channels, samples)")
    if not 1 <= x.shape[1] <= DYNAMICS_MAX_CHANNELS:
        raise ValueError(f"x: 1 to {DYNAMICS_MAX_CHANNELS} channels are supported, got {x.shape[1]}")


def _dynamics_gain(kind, x, sample_rate, pack, eps, db):
    """the body of compressor_gain, expander_gain and dynamics_gain_packed; ``pack(x)`` runs before x's device check"""
    _gain_input(x)
    ps = pack(x)
    xf, dt = _audio(x)
    return _DynamicsGainFn.apply(xf, *ps, kind, sample_rate, eps, bool(db)).to(dt)


def dynamics_gain_packed(kind: int, x: torch.Tensor, sample_rate: float, params: torch.Tensor, eps: float = 1e-8, *,
                         db: bool = False):
    """``compressor_gain`` (kind 0) / ``expander_gain`` (kind 1) with the six parameters stacked as ``(bs, 6)`` in
    signature order (threshold, ratio, attack, release, knee, makeup)."""
    return _dynamics_gain(kind, x, sample_rate, _dynamics_params_packed(params), eps, db)


def compressor_gain(
    x: torch.Tensor,
    sample_rate: float,
    threshold_db: torch.Tensor,
    ratio: torch.Tensor,
    attack_ms: torch.Tensor,
    release_ms: torch.Tensor,
    knee_db: torch.Tensor,
    makeup_gain_db: torch.Tensor,
    eps: float = 1e-8,
    *,
    db: bool = False,
):
    """The time-varying gain ``G`` that ``compressor`` multiplies into the audio, as an op of its own: ``(bs, 1, n)``,
    broadcasting against any ``(bs, C', n)``.

    ``x`` is the detector input ``(bs, C, n)``, ``1 <= C <= 32``: the audio itself, or a key of any channel count.  The
    detector is the compressor's: ``side = x.sum(dim=1)`` (accumulated in fp64, rounded once), ``level =
    20 log10(max(|side|, eps))``, the static curve, the zero-state one-pole attack smoother ``s`` and the makeup ``M``.
    The result is ``G = 10^((s + M) / 20)``, or ``s + M`` in dB with ``db=True`` (finite where the linear gain
    underflows, e.g. an expander at a high ratio on silence).  Computed in fp32, returned in x's dtype.  Parameters
    broadcast as in ``compressor``; ``release_ms`` is validated for shape and gets no gradient.  There is no look-ahead:
    it delays the audio path, never the gain, so for every C and look-ahead ``la``

        ``compressor(x, ..., lookahead_samples=la)[b, c, t] == x[b, c, t - la] * compressor_gain(x, ...)[b, 0, t]``

    bit for bit (0 for ``t < la``).  ``sidechain_compressor(x, sidechain=k)`` agrees with
    ``delay(x) * compressor_gain(k)`` to rounding, not bit for bit: its tiles depend on x's channels too.

    Gradients: every channel of x receives the same ``dL/dside``, which carries ``1/side`` and is 0 where
    ``|side| < eps`` (returned as an expanded view of one row per item); the five other parameters as in ``compressor``.
    Without a gradient to compute, no smoother checkpoint is kept.
    """
    pack = _dynamics_params(threshold_db, ratio, attack_ms, release_ms, knee_db, makeup_gain_db)
    return _dynamics_gain(0, x, sample_rate, pack, eps, db)


def expander_gain(
    x: torch.Tensor,
    sample_rate: float,
    threshold_db: torch.Tensor,
    ratio: torch.Tensor,
    attack_ms: torch.Tensor,
    release_ms: torch.Tensor,
    knee_db: torch.Tensor,
    makeup_gain_db: torch.Tensor,
    eps: float = 1e-8,
    *,
    db: bool = False,
):
    """The gain ``expander`` applies, exactly as ``compressor_gain`` is the compressor's: the expander's static curve,
    the same detector, smoother and makeup, the same bit-for-bit contract with ``expander``."""
    pack = _dynamics_params(threshold_db, ratio, attack_ms, release_ms, knee_db, makeup_gain_db)
    return _dynamics_gain(1, x, sample_rate, pack, eps, db)


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
    plist = (
        low_shelf_gain_db, low_shelf_cutoff_freq, low_shelf_q_factor,
        band0_gain_db, band0_cutoff_freq, band0_q_factor,
        band1_gain_db, band1_cutoff_freq, band1_q_factor,
        band2_gain_db, band2_cutoff_freq, band2_q_factor,
        band3_gain_db, band3_cutoff_freq, band3_q_factor,
        high_shelf_gain_db, high_shelf_cutoff_freq, high_shelf_q_factor,
    )
    return _parametric_eq(x, sample_rate, lambda xf: _stack_params(plist, xf.shape[0], xf, "parametric_eq"))


def _parametric_eq(x, sample_rate, pack):
    """the body of parametric_eq and parametric_eq_packed; ``pack(xf)`` checks and packs the parameters"""
    xf, dt = _audio(x)
    y = _ParametricEqFn.apply(xf, pack(xf), sample_rate)
    return y.to(dt)


def parametric_eq_packed(x: torch.Tensor, sample_rate: float, params: torch.Tensor):
    """``parametric_eq`` with its 18 parameters already stacked as ``(bs, 18)`` in signature order (physical
    units).  Used by ``modules.ParametricEQ.process_normalized`` so that the whole normalised-parameter path is
    one affine kernel + the EQ kernels (SURVEY.md 8f rank 1); gradients flow to ``params``."""
    return _parametric_eq(x, sample_rate, lambda xf: _packed(params, 18, xf))


# --------------------------------------------------------------------------------------
# the parametric EQ's frequency response
# --------------------------------------------------------------------------------------


class _EqResponseFn(torch.autograd.Function):
    """params (bs, 18), frequencies (F,) fp64 -> H (bs, F) complex64.  Only params and the frequencies are saved; the
    backward recomputes the sections from them."""

    @staticmethod
    def forward(ctx, params, freqs, sample_rate):
        lib = _abi.lib()
        bs, nf = params.shape[0], freqs.shape[0]
        dev = params.device
        h = torch.empty(bs, nf, 2, dtype=torch.float32, device=dev)
        nws = lib.dasp_eq_response_workspace_floats(bs, nf)
        with torch.cuda.device(dev):
            ws = _ws(nws, dev)
            with _timed("eq_response_fwd", dev):
                check(lib.dasp_eq_response_fwd(ptr(params), ptr(freqs), ptr(h), ptr(ws), nws, bs, nf,
                                               float(sample_rate), stream_ptr(dev)), "dasp_eq_response_fwd")
        if ctx.needs_input_grad[0]:
            ctx.save_for_backward(params, freqs)
        ctx.sample_rate = float(sample_rate)
        return torch.view_as_complex(h)

    @staticmethod
    def backward(ctx, gh):
        lib = _abi.lib()
        params, freqs = ctx.saved_tensors
        bs, nf = params.shape[0], freqs.shape[0]
        dev = params.device
        g = torch.view_as_real(gh.to(torch.complex64).resolve_conj().contiguous()) if gh.numel() else None
        gp = torch.empty_like(params)
        nws = lib.dasp_eq_response_workspace_floats(bs, nf)
        with torch.cuda.device(dev):
            ws = _ws(nws, dev)
            with _timed("eq_response_bwd", dev):
                check(lib.dasp_eq_response_bwd(ptr(g), ptr(params), ptr(freqs), ptr(gp), ptr(ws), nws, bs, nf,
                                               ctx.sample_rate, stream_ptr(dev)), "dasp_eq_response_bwd")
        return gp, None, None


def _eq_response_checks(sample_rate, frequencies):
    if not float(sample_rate) > 0.0:
        raise ValueError(f"sample_rate must be positive, got {sample_rate}")
    if not torch.is_tensor(frequencies) or frequencies.dim() != 1:
        raise ValueError("frequencies must be a 1-D tensor of frequencies in Hz, got "
                         f"{tuple(frequencies.shape) if torch.is_tensor(frequencies) else type(frequencies).__name__}")
    if frequencies.requires_grad:
        raise ValueError("frequencies must not require a gradient: the response is differentiated with respect to the "
                         "18 EQ parameters only")


def _eq_response_run(packed, dt, frequencies, sample_rate):
    dev = packed.device
    if frequencies.device.type != "cpu" and frequencies.device != dev:
        raise DaspError(f"frequencies are on {frequencies.device}; they must be on the CPU or on {dev}")
    freqs = frequencies.to(device=dev, dtype=torch.float64).contiguous()
    h = _EqResponseFn.apply(packed, freqs, sample_rate)
    return h.to(torch.complex128) if dt == torch.float64 else h


def parametric_eq_frequency_response(
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
    frequencies: torch.Tensor,
):
    """The complex frequency response of the filter ``parametric_eq`` runs, at chosen frequencies::

        H[b, f] = prod_k H_k(exp(j 2 pi frequencies[f] / sample_rate))

    over the six RBJ sections low shelf, band0..band3 (peaking), high shelf.  With
    ``frequencies = torch.fft.rfftfreq(n_fft, 1 / sample_rate)`` this is the reference's
    ``signal.fft_sosfreqz(sos, n_fft)``; at ``n_fft = 2**ceil(log2(2n - 1))`` it is the ``H`` the reference's
    ``parametric_eq`` multiplies into the spectrum of an ``n``-sample signal.  Losses on the curve (a target magnitude
    in dB on a log-frequency grid, a penalty on boosts) need no audio and no recursion.

    Args:
        sample_rate: positive.
        low_shelf_gain_db ... high_shelf_q_factor: the 18 parameters of ``parametric_eq``, in its order.  Each holds
            ``bs`` elements in any shape or one element that is broadcast; bs is the largest element count.  The
            parameters' device must be CUDA.
        frequencies: 1-D tensor of F >= 0 frequencies in Hz, on the CPU or on the parameters' device; converted to
            fp64, so an fp64 ``rfftfreq`` grid is taken exactly.  Any finite value (H is periodic in sample_rate).
            It receives no gradient and must not require one.

    Returns ``(bs, F)`` complex64, or complex128 when the parameters' promoted dtype is fp64.  The coefficients are
    designed in fp64 and H is evaluated in fp32 in the sigma form of ``parametric_eq``'s sections (DESIGN.md 4.3):
    within about 1e-5 of fp64 at every bin, where the reference's fp32 ``rfft`` of the coefficients is off by up to
    tens of percent near low shelves.  Gradients flow to all 18 parameters (torch's convention for complex outputs);
    only the packed parameters and the fp64 frequencies are kept for the backward.
    """
    plist = (
        low_shelf_gain_db, low_shelf_cutoff_freq, low_shelf_q_factor,
        band0_gain_db, band0_cutoff_freq, band0_q_factor,
        band1_gain_db, band1_cutoff_freq, band1_q_factor,
        band2_gain_db, band2_cutoff_freq, band2_q_factor,
        band3_gain_db, band3_cutoff_freq, band3_q_factor,
        high_shelf_gain_db, high_shelf_cutoff_freq, high_shelf_q_factor,
    )
    bs = _params_batch(plist, "parametric_eq_frequency_response")
    _eq_response_checks(sample_rate, frequencies)
    return _eq_response_run(*_params_stacked(plist, bs, "parametric_eq_frequency_response"), frequencies, sample_rate)


def parametric_eq_frequency_response_packed(sample_rate: float, params: torch.Tensor, frequencies: torch.Tensor):
    """``parametric_eq_frequency_response`` with its 18 parameters stacked as ``(bs, 18)`` in signature order
    (physical units), as ``parametric_eq_packed`` takes them.  Used by ``modules.ParametricEQ.frequency_response``."""
    _packed_shape(params, 18)
    _eq_response_checks(sample_rate, frequencies)
    return _eq_response_run(*_packed_params(params, "parametric_eq_frequency_response"), frequencies, sample_rate)


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


def _check_noise_shape(noise, bs, num_samples, num_bandpass_taps):
    if noise is not None:
        expect = (bs * 2, 12, num_samples + num_bandpass_taps - 1)
        if tuple(noise.shape) != expect:
            raise ValueError(f"noise must have shape {expect}, got {tuple(noise.shape)}")


def _noise_or_seed(noise, xf, bs, num_samples, num_bandpass_taps):
    """parity mode: validate the caller's noise tensor; default mode: draw the 64-bit Philox key ON THE DEVICE.

    The reference draws its noise with ``torch.randn`` (``functional.py:547-548``), which is reproducible under
    ``torch.manual_seed`` and, on CUDA, graph-safe (fresh values on every replay of a captured graph).  The key of
    the in-kernel generator is therefore one ``random_()`` word of torch's CUDA generator, left in device memory
    and read by the kernels when they run: no host round trip, same reproducibility, and a captured graph
    re-draws it on every replay (torch registers the generator's Philox offset with the graph)."""
    _check_noise_shape(noise, bs, num_samples, num_bandpass_taps)
    if noise is not None:
        return noise.to(device=xf.device, dtype=torch.float32).contiguous(), None
    return None, torch.empty(1, dtype=torch.int64, device=xf.device).random_()


def _geom_buffers(geom, geom_fn, args, dev, need_bwd, saved=("xspec_c64", "irspec_c64")):
    """the geometry query `geom_fn` (dasp_*_geometry) on `args` into `geom` (ReverbGeom or ConvGeom), the forward
    workspace and, when a backward follows, the buffers kept for it, one per size field in `saved` (``*_c64``:
    complex64, ``f_floats``: fp32); returns them and the backward's workspace bytes"""
    check(getattr(_abi.lib(), geom_fn)(*args, geom), geom_fn)
    ws = _ws_bytes(geom.fwd_workspace_bytes, dev)
    bufs = [torch.empty(getattr(geom, f), dtype=torch.complex64 if f.endswith("_c64") else torch.float32, device=dev)
            if need_bwd else None for f in saved]
    return ws, bufs, geom.bwd_workspace_bytes


class _ReverbFn(torch.autograd.Function):
    """x (bs, 1|2, n), params (bs, 25) -> y (bs, 2, n)."""

    @staticmethod
    def forward(ctx, x, params, noise, seed, sample_rate, num_samples, taps, chunk):
        lib = _abi.lib()
        bs, in_chs, n = x.shape
        dev = x.device
        y = torch.empty(bs, 2, n, dtype=torch.float32, device=dev)
        need_bwd = any(ctx.needs_input_grad[:2])
        with torch.cuda.device(dev):
            ws, (fsave, xspec, irspec), bwd_bytes = _geom_buffers(
                _abi.ReverbGeom(), "dasp_reverb_geometry", (bs, n, num_samples, taps, chunk), dev, need_bwd,
                ("f_floats", "xspec_c64", "irspec_c64"))
            with _timed("reverb_fwd", dev):
                check(lib.dasp_reverb_fwd(ptr(x), in_chs, ptr(params), ptr(noise), ptr(seed), ptr(y), ptr(fsave),
                                          ptr(xspec), ptr(irspec), ptr(ws), ws.numel(), bs, n, num_samples, taps, chunk,
                                          float(sample_rate), stream_ptr(dev)), "dasp_reverb_fwd")
        if need_bwd:
            # slot 2 (the wet signal, which the backward no longer needs) stays empty so that callers that inspect
            # grad_fn.saved_tensors keep the layout (x, params, -, f, X spectra, IR spectra)
            ctx.save_for_backward(x, params, None, fsave, xspec, irspec)
        ctx.cfg = (num_samples, taps, chunk, bwd_bytes, 1 if noise is None else 0)
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
        ws = _ws_bytes(bwd_bytes, dev)
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
    plist = (
        band0_gain, band1_gain, band2_gain, band3_gain, band4_gain, band5_gain,
        band6_gain, band7_gain, band8_gain, band9_gain, band10_gain, band11_gain,
        band0_decay, band1_decay, band2_decay, band3_decay, band4_decay, band5_decay,
        band6_decay, band7_decay, band8_decay, band9_decay, band10_decay, band11_decay,
        mix,
    )
    return _reverb(x, sample_rate, lambda xf: _stack_params(plist, xf.shape[0], xf, "noise_shaped_reverberation"),
                   num_samples, num_bandpass_taps, noise)


def _reverb(x, sample_rate, pack, num_samples, num_bandpass_taps, noise):
    """the body of noise_shaped_reverberation and its packed twin; ``pack(xf)`` checks and packs the parameters"""
    assert num_bandpass_taps % 2 == 1, "num_bandpass_taps must be odd"
    xf, dt = _audio(x)
    bs, chs, _ = xf.shape
    assert chs <= 2, "only mono/stereo signals are supported"
    packed = pack(xf)
    noise, seed = _noise_or_seed(noise, xf, bs, num_samples, num_bandpass_taps)
    y = _ReverbFn.apply(xf, packed, noise, seed, sample_rate, int(num_samples), int(num_bandpass_taps),
                        reverb_chunk_items(xf.device))
    return y.to(dt)


def noise_shaped_reverberation_packed(x: torch.Tensor, sample_rate: float, params: torch.Tensor, num_samples: int = 65536,
                                      num_bandpass_taps: int = 1023, *, noise: Optional[torch.Tensor] = None):
    """``noise_shaped_reverberation`` with its 25 parameters stacked as ``(bs, 25)`` (12 gains, 12 decays, mix)."""
    return _reverb(x, sample_rate, lambda xf: _packed(params, 25, xf), num_samples, num_bandpass_taps, noise)


# --------------------------------------------------------------------------------------
# the reverb's impulse response on its own
# --------------------------------------------------------------------------------------


class _NsirFn(torch.autograd.Function):
    """params (bs, 24) -> IR (bs, 2, num_samples)."""

    @staticmethod
    def forward(ctx, params, noise, seed, sample_rate, num_samples, taps, chunk):
        lib = _abi.lib()
        bs = params.shape[0]
        dev = params.device
        ir = torch.empty(bs, 2, num_samples, dtype=torch.float32, device=dev)
        need_bwd = ctx.needs_input_grad[0]
        with torch.cuda.device(dev):
            ws, (fsave,), bwd_bytes = _geom_buffers(_abi.ReverbGeom(), "dasp_nsir_geometry",
                                                    (bs, num_samples, taps, chunk), dev, need_bwd, ("f_floats",))
            with _timed("nsir_fwd", dev):
                check(lib.dasp_nsir_fwd(ptr(params), ptr(noise), ptr(seed), ptr(ir), ptr(fsave), ptr(ws), ws.numel(),
                                        bs, num_samples, taps, chunk, float(sample_rate), stream_ptr(dev)),
                      "dasp_nsir_fwd")
        if need_bwd:
            ctx.save_for_backward(params, fsave)
        ctx.cfg = (num_samples, taps, chunk, bwd_bytes, 1 if noise is None else 0)
        return ir

    @staticmethod
    def backward(ctx, gir):
        lib = _abi.lib()
        params, fsave = ctx.saved_tensors
        num_samples, taps, chunk, bwd_bytes, device_noise = ctx.cfg
        bs = params.shape[0]
        dev = params.device
        gir = gir.to(torch.float32).contiguous()
        gp = torch.empty_like(params)
        ws = _ws_bytes(bwd_bytes, dev)
        with torch.cuda.device(dev), _timed("nsir_bwd", dev):
            check(lib.dasp_nsir_bwd(ptr(gir), ptr(params), ptr(fsave), ptr(gp), ptr(ws), ws.numel(), bs, num_samples,
                                    taps, chunk, device_noise, stream_ptr(dev)), "dasp_nsir_bwd")
        return gp, None, None, None, None, None, None


def _nsir_checks(sample_rate, num_samples, num_bandpass_taps):
    if int(num_bandpass_taps) != num_bandpass_taps or num_bandpass_taps < 1 or num_bandpass_taps % 2 != 1:
        raise ValueError(f"num_bandpass_taps must be a positive odd integer, got {num_bandpass_taps}")
    if int(num_samples) != num_samples or num_samples < 1:
        raise ValueError(f"num_samples must be a positive integer, got {num_samples}")
    if not float(sample_rate) / 2.0 > 18000.0:
        raise ValueError(f"sample_rate {sample_rate} too low: the filter bank's 18 kHz high-pass needs sample_rate > 36000")


def _nsir_run(packed, dt, noise, sample_rate, num_samples, num_bandpass_taps):
    bs = packed.shape[0]
    noise, seed = _noise_or_seed(noise, packed, bs, num_samples, num_bandpass_taps)
    ir = _NsirFn.apply(packed, noise, seed, sample_rate, int(num_samples), int(num_bandpass_taps),
                       reverb_chunk_items(packed.device))
    return ir.to(dt)


def noise_shaped_impulse_response(
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
    num_samples: int = 65536,
    num_bandpass_taps: int = 1023,
    *,
    noise: Optional[torch.Tensor] = None,
):
    """The stereo impulse response ``noise_shaped_reverberation`` synthesises (reference ``functional.py:547-567``),
    returned instead of applied::

        IR[b, c, t] = (1/12) sum_k gain_k exp(-(10 decay_k + 1) t / (L - 1)) f[b, c, k, t],   t < L = num_samples

    with f the band-filtered noise of band k (the reverb's filter bank; ``t / (L - 1)`` is ``torch.linspace(0, 1, L)``,
    0 when ``L == 1``).  Every tap is synthesised: no audio length bounds the IR here.

    Args:
        sample_rate: must exceed 36 kHz (the filter bank's 18 kHz high-pass).
        band*_gain, band*_decay: the first 24 parameters of ``noise_shaped_reverberation`` (no ``mix``).  Each holds
            ``bs`` elements in any shape or one element that is broadcast; bs is the largest element count.  The
            parameters' device must be CUDA.
        num_samples, num_bandpass_taps: as in ``noise_shaped_reverberation`` (taps odd).
        noise: the ``(bs*2, 12, num_samples + num_bandpass_taps - 1)`` tensor the reference draws; by default the
            noise is drawn on the device exactly as ``noise_shaped_reverberation`` draws it (Philox keyed by one word of
            torch's CUDA generator: ``torch.manual_seed`` reproduces, a captured graph draws fresh noise per replay).

    Returns ``(bs, 2, num_samples)``, computed in fp32, in the parameters' promoted floating dtype (fp32 when none is
    floating).  Gradients flow to all 24 parameters.  With the same seed and ``n >= num_samples``,
    ``convolution_reverberation(x, sr, noise_shaped_impulse_response(...), mix)`` gives the bits of
    ``noise_shaped_reverberation(x, ..., mix)``.  When a parameter requires a gradient the forward keeps the
    band-filtered noise of every item for the backward (``f_floats`` of ``dasp_nsir_geometry``: 11 MB per item at
    ``L = 96000`` with 1023 taps, so about 11.3 GB for 1024 items); the backward does not regenerate it.
    """
    _nsir_checks(sample_rate, num_samples, num_bandpass_taps)
    plist = (
        band0_gain, band1_gain, band2_gain, band3_gain, band4_gain, band5_gain,
        band6_gain, band7_gain, band8_gain, band9_gain, band10_gain, band11_gain,
        band0_decay, band1_decay, band2_decay, band3_decay, band4_decay, band5_decay,
        band6_decay, band7_decay, band8_decay, band9_decay, band10_decay, band11_decay,
    )
    bs = _params_batch(plist, "noise_shaped_impulse_response")
    _check_noise_shape(noise, bs, num_samples, num_bandpass_taps)
    return _nsir_run(*_params_stacked(plist, bs, "noise_shaped_impulse_response"), noise, sample_rate, num_samples,
                     num_bandpass_taps)


def noise_shaped_impulse_response_packed(sample_rate: float, params: torch.Tensor, num_samples: int = 65536,
                                         num_bandpass_taps: int = 1023, *, noise: Optional[torch.Tensor] = None):
    """``noise_shaped_impulse_response`` with its 24 parameters stacked as ``(bs, 24)`` (12 gains, 12 decays)."""
    _nsir_checks(sample_rate, num_samples, num_bandpass_taps)
    _packed_shape(params, 24)
    _check_noise_shape(noise, params.shape[0], num_samples, num_bandpass_taps)
    return _nsir_run(*_packed_params(params, "noise_shaped_impulse_response"), noise, sample_rate, num_samples,
                     num_bandpass_taps)


# --------------------------------------------------------------------------------------
# convolution reverberation (caller-supplied impulse response)
# --------------------------------------------------------------------------------------


def _caller_ir_shape(impulse_response, bs: int):
    """a caller's IR, taps last, against x's batch: one IR per item, or one shared by a batch of more than one"""
    ir_bs = impulse_response.shape[0]
    if ir_bs != bs and not (ir_bs == 1 and bs > 1):
        raise ValueError(f"impulse_response has batch {ir_bs}, x has batch {bs} (expected {bs} or 1)")
    if impulse_response.shape[-1] < 1:
        raise ValueError("impulse_response needs at least one tap")


def _caller_ir(impulse_response, xf, rank=None):
    """a caller's IR (rank 3, or ``rank``) as fp32 contiguous on x's device"""
    irf, _ = _audio(impulse_response, "impulse_response", rank)
    if irf.device != xf.device:
        raise DaspError(f"impulse_response is on {irf.device} but x is on {xf.device}")
    return irf


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
        with torch.cuda.device(dev):
            ws, (xspec, irspec), bwd_bytes = _geom_buffers(_abi.ConvGeom(), geom_fn, (bs, n, ir_len, chunk), dev,
                                                           need_bwd)
            with _timed("conv_fwd", dev):
                check(getattr(lib, f"dasp_{kind}_fwd")(ptr(x), in_chs, ptr(ir), ir_chs, ir_len, ptr(mix), ptr(y),
                                                       ptr(xspec), ptr(irspec), ptr(ws), ws.numel(), bs, n, chunk,
                                                       stream_ptr(dev)),
                      f"dasp_{kind}_fwd")
        if need_bwd:
            ctx.save_for_backward(x, xspec, irspec, mix)
        ctx.cfg = (kind, ir_bs, ir_chs, ir_len, chunk, bwd_bytes)
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
        ws = _ws_bytes(bwd_bytes, dev)
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
    _caller_ir_shape(impulse_response, bs)
    nmix = mix.numel() if torch.is_tensor(mix) else torch.as_tensor(mix).numel()
    if nmix not in (1, bs):
        raise ValueError(f"mix: expected {bs} element(s) (one per batch item) or 1, got {nmix}")
    xf, dt = _audio(x)
    irf = _caller_ir(impulse_response, xf)
    m = _param(mix, bs, xf, "mix", allow_broadcast=True).contiguous()
    y = _ConvReverbFn.apply(xf, irf, m, reverb_chunk_items(xf.device))
    return y.to(dt)


# --------------------------------------------------------------------------------------
# convolution_bus
# --------------------------------------------------------------------------------------

CONV_BUS_MAX_INPUTS = 32      # DASP_CONV_BUS_MAX_INPUTS in include/dasp_b200.h
CONV_MC_MAX_OUTPUTS = 32      # DASP_CONV_MC_MAX_OUTPUTS in include/dasp_b200.h


class _ConvBusFn(torch.autograd.Function):
    """x (bs, S, n), ir (bs | 1, S, O, L) -> y (bs, O, n).  n % 4 == 0 and 16-byte aligned rows (_bus_inputs pads).
    entry "conv_bus" runs the bus (O <= 2), "conv_mc" multichannel_convolution (O <= CONV_MC_MAX_OUTPUTS).  An ir of
    batch 1 with bs > 1 runs the dasp_<entry>_shared_* entry points; its gradient is the sum over the items."""

    @staticmethod
    def forward(ctx, x, ir, chunk, entry="conv_bus"):
        lib = _abi.lib()
        bs, S, n = x.shape
        ir_bs, _, O, ir_len = ir.shape
        shared = ir_bs == 1 and bs > 1
        kind = f"{entry}_shared" if shared else entry
        dev = x.device
        y = torch.empty(bs, O, n, dtype=torch.float32, device=dev)
        need_bwd = any(ctx.needs_input_grad[:2])
        with torch.cuda.device(dev):
            ws, (xspec, irspec), bwd_bytes = _geom_buffers(_abi.ConvGeom(), f"dasp_{entry}_geometry",
                                                           (bs, n, ir_len, S, O, int(shared), chunk), dev, need_bwd)
            with _timed(f"{entry}_fwd", dev):
                check(getattr(lib, f"dasp_{kind}_fwd")(ptr(x), ptr(ir), ptr(y), ptr(xspec), ptr(irspec), ptr(ws),
                                                       ws.numel(), bs, n, ir_len, S, O, chunk, stream_ptr(dev)),
                      f"dasp_{kind}_fwd")
        if need_bwd:
            ctx.save_for_backward(xspec, irspec)
        ctx.cfg = (entry, kind, bs, S, O, n, ir.shape, chunk, bwd_bytes)
        return y

    @staticmethod
    def backward(ctx, gy):
        lib = _abi.lib()
        xspec, irspec = ctx.saved_tensors
        entry, kind, bs, S, O, n, ir_shape, chunk, bwd_bytes = ctx.cfg
        dev = gy.device
        gy = gy.contiguous()
        if gy.data_ptr() % 16:
            gy = gy.clone()
        gx = torch.empty(bs, S, n, dtype=torch.float32, device=dev)
        # a fixed IR (measured rooms, a fixed downmix) skips every dL/dIR kernel
        gir = torch.empty(ir_shape, dtype=torch.float32, device=dev) if ctx.needs_input_grad[1] else None
        ws = _ws_bytes(bwd_bytes, dev)
        with torch.cuda.device(dev), _timed(f"{entry}_bwd", dev):
            check(getattr(lib, f"dasp_{kind}_bwd")(ptr(gy), ptr(xspec), ptr(irspec), ptr(gx), ptr(gir), ptr(ws),
                                                   ws.numel(), bs, n, ir_shape[3], S, O, chunk, stream_ptr(dev)),
                  f"dasp_{kind}_bwd")
        return gx, gir, None, None


def _bus_inputs(x, impulse_response, name: str, max_outputs: int):
    """The checks and the padding of convolution_bus (max_outputs 2) and multichannel_convolution: x (bs, S, n) and
    the IR (bs | 1, S, O, L) as fp32, rows padded to n % 4 == 0 and 16-byte aligned, the taps that would reach only
    the padding dropped.  `name` heads the input-count message.  Returns (x, ir, n, x's dtype)."""
    if not torch.is_tensor(x) or x.dim() != 3:
        raise ValueError("x must be a tensor of shape (batch, inputs, samples)")
    if not torch.is_tensor(impulse_response) or impulse_response.dim() != 4:
        raise ValueError("impulse_response must be a tensor of shape (batch, inputs, outputs, taps)")
    bs, S, n = x.shape
    if not 1 <= S <= CONV_BUS_MAX_INPUTS:
        raise ValueError(f"{name}: 1 to {CONV_BUS_MAX_INPUTS} input channels are supported, got {S}")
    _, ir_s, O, L = impulse_response.shape
    if ir_s != S:
        raise ValueError(f"impulse_response has {ir_s} input rows, x has {S} channels")
    if max_outputs == 2 and O not in (1, 2):
        raise ValueError(f"impulse_response: a mono (1) or stereo (2) bus is supported, got {O} outputs")
    if not 1 <= O <= max_outputs:
        raise ValueError(f"impulse_response: 1 to {max_outputs} output channels are supported, got {O}")
    _caller_ir_shape(impulse_response, bs)
    if n < 1:
        raise ValueError("x needs at least one sample")
    xf, dt = _audio(x)
    irf = _caller_ir(impulse_response, xf, 4)
    n4 = (n + 3) // 4 * 4
    if n4 != n:
        xf = torch.nn.functional.pad(xf, (0, n4 - n))
        if L > n:                        # taps n .. n4 - 1 would reach the padding; their gradient is exactly 0
            irf = irf[..., :n].contiguous()
    elif xf.data_ptr() % 16:
        xf = xf.clone()
    return xf, irf, n, dt


def convolution_bus(x: torch.Tensor, sample_rate: float, impulse_response: torch.Tensor):
    """Any number of input channels, each convolved with its own impulse responses and summed into one mono or stereo
    bus::

        y[:, o] = sum_s (x[:, s] * h[:, s, o])[:n]

    (``*`` the causal convolution cropped to ``n``, exactly as ``convolution_reverberation`` defines its wet signal).
    Uses: reverberant multi-source mixtures (each speaker or noise source through the room impulse response of its
    own position), binaural or stereo downmixes of 5.1 / 7.1 audio through one set of BRIRs shared by the batch,
    multitrack mixing with a room per stem, and a learnable S-input FIR trained through its taps.

    Args:
        x: audio ``(bs, S, n)``, ``1 <= S <= CONV_BUS_MAX_INPUTS`` input channels (sources, stems, speaker feeds).
        sample_rate: unused (kept for the common processor signature).
        impulse_response: ``(bs, S, O, L)``, one IR set per item, or ``(1, S, O, L)``, one set shared by the batch;
            ``O`` is 1 (mono bus) or 2 (stereo bus), any ``L >= 1``.  Row ``(s, o)`` is the path from input ``s`` to
            output ``o``.

    Returns ``(bs, O, n)`` in x's dtype, computed in fp32.  There is no dry/wet mix: the inputs and the outputs differ
    in number, so no dry signal is defined; a caller who wants one adds it to the result.

    Identities (held to fp32 rounding):

    1. ``S = 2, O = 2``: ``convolution_reverberation(x, sr, h.reshape(bs, 4, L), mix=1)``, whose true-stereo row
       order ``2 i + o`` is this layout.
    2. ``S = 1, O = 2``: ``convolution_reverberation(x, sr, h[:, 0], mix=1)``.
    3. Any ``S``: the sum over ``s`` of ``convolution_bus(x[:, s:s+1], sr, h[:, s:s+1])``.

    Gradients flow to ``x`` (every input) and to every IR row; taps at or beyond ``n`` reach no output and get exactly
    0.  The gradient of a shared ``(1, S, O, L)`` IR has that shape and is the sum over the items, accumulated in fp64
    in item order, so it does not depend on ``REVERB_CHUNK_ITEMS``.  When the IR does not require a gradient, the
    backward skips all dL/dIR work.  The convolution is ``convolution_reverberation``'s (4096-sample partitions, the
    in-shared-memory 8192-point FFT) with the rows of every signal packed two per transform: one window transform per
    pair of inputs and block, and one inverse transform per block for the whole bus.  Rows whose length is not a
    multiple of 4 are zero-padded to one (the transforms bulk-copy 16-byte rows); a padding sample reaches no output
    sample below ``n``.
    """
    xf, irf, n, dt = _bus_inputs(x, impulse_response, "convolution_bus", 2)
    y = _ConvBusFn.apply(xf, irf, reverb_chunk_items(xf.device))
    return (y[..., :n] if xf.shape[-1] != n else y).to(dt)


def multichannel_convolution(x: torch.Tensor, sample_rate: float, impulse_response: torch.Tensor):
    """S input channels through an S x M matrix of impulse responses into M output channels::

        y[:, m] = sum_s (x[:, s] * h[:, s, m])[:n]

    (``*`` the causal convolution cropped to ``n``, as ``convolution_bus`` defines it; this is ``convolution_bus``
    with up to ``CONV_MC_MAX_OUTPUTS`` output rows).  Uses: microphone-array simulation for multichannel separation,
    enhancement, beamforming and direction-of-arrival training (S talkers or noise sources through the room impulse
    responses of an M-microphone array), ambisonic rendering (first order is 4 channels, third order 16, fourth order
    25) and multichannel reproduction such as 5.1 / 7.1 beds and upmixes through a room.

    Args:
        x: audio ``(bs, S, n)``, ``1 <= S <= CONV_BUS_MAX_INPUTS`` input channels (sources).
        sample_rate: unused (kept for the common processor signature).
        impulse_response: ``(bs, S, M, L)``, one matrix per item, or ``(1, S, M, L)``, one matrix shared by the batch;
            ``1 <= M <= CONV_MC_MAX_OUTPUTS``, any ``L >= 1``.  Row ``(s, m)`` is the path from input ``s`` to output
            ``m`` (microphone, ambisonic channel or speaker feed).

    Returns ``(bs, M, n)`` in x's dtype, computed in fp32.  There is no dry/wet mix, as in ``convolution_bus``.

    Identities (held to fp32 rounding):

    1. ``M <= 2``: ``convolution_bus(x, sr, h)``, bit for bit.
    2. Any ``M``: the concatenation over the output pairs ``q`` of ``convolution_bus(x, sr, h[:, :, 2q:2q+2])``.
    3. Any ``S``: the sum over ``s`` of ``multichannel_convolution(x[:, s:s+1], sr, h[:, s:s+1])``.

    Gradients flow to ``x`` (every input) and to every IR row; taps at or beyond ``n`` reach no output and get exactly
    0.  The gradient of a shared ``(1, S, M, L)`` matrix has that shape and is the sum over the items, accumulated in
    fp64 in item order, so it does not depend on ``REVERB_CHUNK_ITEMS``.  When the IR does not require a gradient, the
    backward skips all dL/dIR work.  The convolution is ``convolution_bus``'s: every input's windows are transformed
    (two inputs per transform) and kept for the backward once for all M outputs, the S M IR rows go two per partition
    transform, and the outputs, their gradients and dL/dx are transformed two rows per transform.  The ceil(M / 2)
    ``convolution_bus`` calls of identity 2 would transform and keep every window, and transform dL/dx, once per call.
    Rows whose length is not a multiple of 4 are zero-padded to one; a padding sample reaches no output sample below
    ``n``.
    """
    xf, irf, n, dt = _bus_inputs(x, impulse_response, "multichannel_convolution", CONV_MC_MAX_OUTPUTS)
    y = _ConvBusFn.apply(xf, irf, reverb_chunk_items(xf.device), "conv_mc")
    return (y[..., :n] if xf.shape[-1] != n else y).to(dt)


# --------------------------------------------------------------------------------------
# time_varying_convolution_reverberation
# --------------------------------------------------------------------------------------

CONV_PARTITION_SAMPLES = 4096      # conv_block of dasp_conv_geom: the partition length of every caller-IR convolution


def _anchor_hop(hop, K: int, n: int) -> int:
    """the anchor spacing of a trajectory of K impulse responses (sets) over n samples, as an int"""
    if isinstance(hop, bool) or not isinstance(hop, int) and not (torch.is_tensor(hop) and hop.numel() == 1
                                                                  and not hop.is_floating_point()):
        raise ValueError(f"hop must be an integer number of samples, got {hop!r}")
    hop = int(hop)
    if hop <= 0 or hop % CONV_PARTITION_SAMPLES:
        raise ValueError(f"hop must be a positive multiple of {CONV_PARTITION_SAMPLES} samples, got {hop}")
    if (K - 1) * hop >= n:
        raise ValueError(f"impulse response {K - 1} is anchored at (K - 1) * hop = {(K - 1) * hop}, at or after the "
                         f"end of x ({n} samples)")
    return hop


class _TvConvFn(torch.autograd.Function):
    """x (bs, 1|2, n), ir (bs | 1, K, 1|2, L), mix (bs,) -> y (bs, 2, n).  n % 4 == 0 and 16-byte aligned rows
    (time_varying_convolution_reverberation pads).  An ir of batch 1 with bs > 1 runs the dasp_tvconv_shared_* entry
    points; its gradient is the sum over the items."""

    @staticmethod
    def forward(ctx, x, ir, mix, hop, chunk):
        lib = _abi.lib()
        bs, in_chs, n = x.shape
        ir_bs, K, ir_chs, ir_len = ir.shape
        shared = ir_bs == 1 and bs > 1
        kind = "tvconv_shared" if shared else "tvconv"
        dev = x.device
        y = torch.empty(bs, 2, n, dtype=torch.float32, device=dev)
        need_bwd = any(ctx.needs_input_grad[:3])
        with torch.cuda.device(dev):
            ws, (xspec, irspec), bwd_bytes = _geom_buffers(
                _abi.ConvGeom(), "dasp_tvconv_geometry", (bs, n, ir_len, K, ir_chs, hop, int(shared), chunk), dev,
                need_bwd)
            with _timed("tvconv_fwd", dev):
                check(getattr(lib, f"dasp_{kind}_fwd")(ptr(x), in_chs, ptr(ir), ir_chs, ir_len, K, hop, ptr(mix),
                                                       ptr(y), ptr(xspec), ptr(irspec), ptr(ws), ws.numel(), bs, n,
                                                       chunk, stream_ptr(dev)),
                      f"dasp_{kind}_fwd")
        if need_bwd:
            ctx.save_for_backward(x, xspec, irspec, mix)
        ctx.cfg = (kind, ir.shape, hop, chunk, bwd_bytes)
        return y

    @staticmethod
    def backward(ctx, gy):
        lib = _abi.lib()
        x, xspec, irspec, mix = ctx.saved_tensors
        kind, ir_shape, hop, chunk, bwd_bytes = ctx.cfg
        bs, in_chs, n = x.shape
        dev = x.device
        gy = gy.contiguous()
        if gy.data_ptr() % 16:
            gy = gy.clone()
        gx = torch.empty_like(x)
        # a fixed trajectory (measured or simulated rooms) skips every dL/dIR kernel
        gir = torch.empty(ir_shape, dtype=torch.float32, device=dev) if ctx.needs_input_grad[1] else None
        gmix = torch.empty_like(mix)
        ws = _ws_bytes(bwd_bytes, dev)
        with torch.cuda.device(dev), _timed("tvconv_bwd", dev):
            check(getattr(lib, f"dasp_{kind}_bwd")(ptr(gy), ptr(x), in_chs, ir_shape[2], ir_shape[3], ir_shape[1], hop,
                                                   ptr(mix), ptr(xspec), ptr(irspec), ptr(gx), ptr(gir), ptr(gmix),
                                                   ptr(ws), ws.numel(), bs, n, chunk, stream_ptr(dev)),
                  f"dasp_{kind}_bwd")
        return gx, gir, gmix, None, None


def time_varying_convolution_reverberation(x: torch.Tensor, sample_rate: float, impulse_response: torch.Tensor,
                                           hop: int, mix: torch.Tensor):
    """Convolution reverb with a trajectory of K impulse responses, crossfaded along the output: a talker walking past
    a microphone, a head-tracked binaural rendering, a listener moving through a room, a door opening, an automated or
    learnt time-varying FIR.  IR ``k`` belongs to the anchor time ``t_k = k * hop``::

        wet(t) = sum_k w_k(t) (x * h_k)(t),    y = (1 - mix) x + mix wet

        k hop <= t < (k+1) hop, k < K - 1:   a = (t - k hop) / hop,   w_k = 1 - a,   w_{k+1} = a,   other w = 0
        t >= (K - 1) hop:                    w_{K-1} = 1

    (``*`` the causal convolution cropped to ``n``, exactly as ``convolution_reverberation`` defines its wet signal).
    At every anchor time, and after the last one, the output is the static convolution with that anchor's IR; between
    two anchors it is a linear crossfade of the outputs of the two neighbouring IRs.

    This is output-side (listener-side) interpolation because it is the interpolation that overlap-save supports
    without splitting the audio windows: every output block lies inside one anchor interval, so it needs the products
    of two IRs with the same window spectra a static convolution uses, and the crossfade is applied to the inverse
    transform's output.  Input-side weighting, ``sum_k (w_k x) * h_k``, would need zero-padded transforms per block
    and IR, because an overlap-save window straddles anchor boundaries.  A moving mono source (input-side weighting) is
    ``time_varying_convolution_bus`` with ``S = 1`` and ``crossfade="input"``.

    Args:
        x: audio ``(bs, 1|2, n)``; mono is used for both channels.
        sample_rate: unused (kept for the common processor signature).
        impulse_response: ``(bs, K, 1|2, L)``, one trajectory per item, or ``(1, K, 1|2, L)``, one trajectory shared by
            the batch; ``K >= 1``, any ``L >= 1``; a mono IR feeds both channels.
        hop: the anchor spacing in samples, a positive multiple of ``CONV_PARTITION_SAMPLES`` (4096), the partition
            length of the convolution, so that every output block and every gradient block lies inside one anchor
            interval; ``(K - 1) * hop < n``.
        mix: ``bs`` elements in any shape, or one element that is broadcast over the batch.

    Returns ``(bs, 2, n)`` in x's dtype, computed in fp32.  ``K = 1`` is ``convolution_reverberation(x, sr, h[:, 0],
    mix)``, and K equal IRs are that IR's static convolution, both to fp32 rounding.  Gradients flow to ``x``, to every
    IR of the trajectory (a mono IR receives the sum of both channel gradients; taps at or beyond ``min(L, n)`` get
    exactly 0) and to ``mix``.  The gradient of a shared ``(1, K, C, L)`` trajectory has that shape and is the sum over
    the items, accumulated in fp64 in item order, so it does not depend on ``REVERB_CHUNK_ITEMS``.  When the IRs do
    not require a gradient, the backward skips all dL/dIR work.

    Cost: the audio windows are transformed once, as for one static IR, and kept for the backward once; the K IRs'
    partitions are transformed once each; a block between two anchors takes two inverse transforms (the two IRs'
    products, one channel each), a block after the last anchor one.  K full-length ``convolution_reverberation`` calls
    would transform and keep the audio windows K times.  Rows whose length is not a multiple of 4 are zero-padded to
    one (the transforms bulk-copy 16-byte rows); a padding sample reaches no output sample below ``n``.
    """
    if not torch.is_tensor(x) or x.dim() != 3:
        raise ValueError("x must be a tensor of shape (batch, channels, samples)")
    if x.shape[1] not in (1, 2):
        raise ValueError(f"x: only mono/stereo is supported, got {x.shape[1]} channels")
    if not torch.is_tensor(impulse_response) or impulse_response.dim() != 4:
        raise ValueError("impulse_response must be a tensor of shape (batch, K, channels, taps)")
    _, K, ir_chs, L = impulse_response.shape
    if ir_chs not in (1, 2):
        raise ValueError(f"impulse_response: only mono/stereo is supported, got {ir_chs} channels")
    if K < 1:
        raise ValueError("impulse_response needs at least one impulse response (K >= 1)")
    bs, _, n = x.shape
    _caller_ir_shape(impulse_response, bs)
    if n < 1:
        raise ValueError("x needs at least one sample")
    hop = _anchor_hop(hop, K, n)
    nmix = mix.numel() if torch.is_tensor(mix) else torch.as_tensor(mix).numel()
    if nmix not in (1, bs):
        raise ValueError(f"mix: expected {bs} element(s) (one per batch item) or 1, got {nmix}")
    xf, dt = _audio(x)
    irf = _caller_ir(impulse_response, xf, 4)
    m = _param(mix, bs, xf, "mix", allow_broadcast=True).contiguous()
    n4 = (n + 3) // 4 * 4
    if n4 != n:
        xf = torch.nn.functional.pad(xf, (0, n4 - n))
        if L > n:                        # taps n .. n4 - 1 would reach the padding; their gradient is exactly 0
            irf = irf[..., :n].contiguous()
    elif xf.data_ptr() % 16:
        xf = xf.clone()
    y = _TvConvFn.apply(xf, irf, m, hop, reverb_chunk_items(xf.device))
    return (y[..., :n] if n4 != n else y).to(dt)


# --------------------------------------------------------------------------------------
# time_varying_convolution_bus
# --------------------------------------------------------------------------------------

class _TvBusFn(torch.autograd.Function):
    """x (bs, S, n), ir (bs | 1, K, S, O, L) -> y (bs, O, n).  n % 4 == 0 and 16-byte aligned rows
    (_tv_bus_inputs pads).  entry "tvbus" crossfades on the output side, "tvbus_in" on the source side (O <= 2);
    "tvmc" and "tvmc_in" are the same for time_varying_multichannel_convolution (O <= CONV_MC_MAX_OUTPUTS).  An ir of
    batch 1 with bs > 1 runs the dasp_<entry>_shared_* entry points; its gradient is the sum over the items."""

    @staticmethod
    def forward(ctx, x, ir, hop, chunk, entry="tvbus"):
        lib = _abi.lib()
        bs, S, n = x.shape
        ir_bs, K, _, O, ir_len = ir.shape
        shared = ir_bs == 1 and bs > 1
        kind = f"{entry}_shared" if shared else entry
        dev = x.device
        y = torch.empty(bs, O, n, dtype=torch.float32, device=dev)
        need_bwd = any(ctx.needs_input_grad[:2])
        with torch.cuda.device(dev):
            ws, (xspec, irspec), bwd_bytes = _geom_buffers(
                _abi.ConvGeom(), f"dasp_{entry}_geometry", (bs, n, ir_len, K, S, O, hop, int(shared), chunk), dev,
                need_bwd)
            with _timed(f"{entry}_fwd", dev):
                check(getattr(lib, f"dasp_{kind}_fwd")(ptr(x), ptr(ir), ptr(y), ptr(xspec), ptr(irspec), ptr(ws),
                                                       ws.numel(), bs, n, ir_len, K, S, O, hop, chunk,
                                                       stream_ptr(dev)),
                      f"dasp_{kind}_fwd")
        if need_bwd:
            ctx.save_for_backward(xspec, irspec)
        ctx.cfg = (entry, kind, bs, S, O, n, ir.shape, hop, chunk, bwd_bytes)
        return y

    @staticmethod
    def backward(ctx, gy):
        lib = _abi.lib()
        xspec, irspec = ctx.saved_tensors
        entry, kind, bs, S, O, n, ir_shape, hop, chunk, bwd_bytes = ctx.cfg
        dev = gy.device
        gy = gy.contiguous()
        if gy.data_ptr() % 16:
            gy = gy.clone()
        gx = torch.empty(bs, S, n, dtype=torch.float32, device=dev)
        # a fixed trajectory set (measured or simulated rooms) skips every dL/dIR kernel
        gir = torch.empty(ir_shape, dtype=torch.float32, device=dev) if ctx.needs_input_grad[1] else None
        ws = _ws_bytes(bwd_bytes, dev)
        with torch.cuda.device(dev), _timed(f"{entry}_bwd", dev):
            check(getattr(lib, f"dasp_{kind}_bwd")(ptr(gy), ptr(xspec), ptr(irspec), ptr(gx), ptr(gir), ptr(ws),
                                                   ws.numel(), bs, n, ir_shape[4], ir_shape[1], S, O, hop, chunk,
                                                   stream_ptr(dev)),
                  f"dasp_{kind}_bwd")
        return gx, gir, None, None, None


def _tv_bus_inputs(x, impulse_response, hop, crossfade, name: str, max_outputs: int):
    """The checks and the padding of time_varying_convolution_bus (max_outputs 2) and
    time_varying_multichannel_convolution: x (bs, S, n) and the trajectory (bs | 1, K, S, O, L) as fp32, rows padded to
    n % 4 == 0 and 16-byte aligned, the taps that would reach only the padding dropped.  `name` heads the input-count
    message.  Returns (x, ir, n, x's dtype, hop)."""
    if crossfade not in ("output", "input"):
        raise ValueError(f'crossfade must be "output" or "input", got {crossfade!r}')
    if not torch.is_tensor(x) or x.dim() != 3:
        raise ValueError("x must be a tensor of shape (batch, inputs, samples)")
    if not torch.is_tensor(impulse_response) or impulse_response.dim() != 5:
        raise ValueError("impulse_response must be a tensor of shape (batch, K, inputs, outputs, taps)")
    bs, S, n = x.shape
    if not 1 <= S <= CONV_BUS_MAX_INPUTS:
        raise ValueError(f"{name}: 1 to {CONV_BUS_MAX_INPUTS} input channels are supported, got {S}")
    _, K, ir_s, O, L = impulse_response.shape
    if ir_s != S:
        raise ValueError(f"impulse_response has {ir_s} input rows, x has {S} channels")
    if max_outputs == 2 and O not in (1, 2):
        raise ValueError(f"impulse_response: a mono (1) or stereo (2) bus is supported, got {O} outputs")
    if not 1 <= O <= max_outputs:
        raise ValueError(f"impulse_response: 1 to {max_outputs} output channels are supported, got {O}")
    if K < 1:
        raise ValueError("impulse_response needs at least one impulse-response set (K >= 1)")
    _caller_ir_shape(impulse_response, bs)
    if n < 1:
        raise ValueError("x needs at least one sample")
    hop = _anchor_hop(hop, K, n)
    xf, dt = _audio(x)
    irf = _caller_ir(impulse_response, xf, 5)
    n4 = (n + 3) // 4 * 4
    if n4 != n:
        xf = torch.nn.functional.pad(xf, (0, n4 - n))
        if L > n:                        # taps n .. n4 - 1 would reach the padding; their gradient is exactly 0
            irf = irf[..., :n].contiguous()
    elif xf.data_ptr() % 16:
        xf = xf.clone()
    return xf, irf, n, dt, hop


def time_varying_convolution_bus(x: torch.Tensor, sample_rate: float, impulse_response: torch.Tensor, hop: int, *,
                                 crossfade: str = "output"):
    """Several moving sources, each through its own trajectory of impulse responses, crossfaded and summed into one
    mono or stereo bus: ``convolution_bus`` whose IR set changes over time, as
    ``time_varying_convolution_reverberation``'s IR does.  Set ``k`` of the trajectory, ``h[:, k]``, is a complete
    ``convolution_bus`` IR set, the scene at the anchor time ``t_k = k * hop``.  ``crossfade`` chooses where the
    weights apply::

        "output":  y[:, o](t) = sum_k w_k(t) sum_s (x[:, s] * h[:, k, s, o])(t)
        "input":   y[:, o](t) = sum_k sum_s ((w_k x[:, s]) * h[:, k, s, o])(t)

        k hop <= t < (k+1) hop, k < K - 1:   a = (t - k hop) / hop,   w_k = 1 - a,   w_{k+1} = a,   other w = 0
        t >= (K - 1) hop:                    w_{K-1} = 1

    (``*`` the causal convolution cropped to ``n``, exactly as ``convolution_reverberation`` defines its wet signal;
    ``w_k`` are ``time_varying_convolution_reverberation``'s crossfade weights).  The output-side crossfade weights the
    time a sample is heard: it models a moving listener (or a static source heard through a changing room).  The
    input-side (source-side) crossfade weights the time a sample is emitted: a sample emitted at ``tau`` between anchors
    ``k`` and ``k + 1`` keeps ``(1 - a) h_k + a h_{k+1}`` over its whole reverb tail, also the part heard after later
    anchors, which is the model of a moving point source (propagation delay and Doppler aside).  The two agree when
    ``L = 1`` or all sets are equal; they differ most when ``L`` is long against ``hop``.  Uses: reverberant
    multi-talker mixtures with moving speakers for separation and enhancement training, binaural or stereo scenes with
    several moving objects, a stereo source moving through a room (``S = 2, O = 2`` is a time-varying true-stereo
    rendering), and a learnable time-varying S-input FIR.

    Args:
        x: audio ``(bs, S, n)``, ``1 <= S <= CONV_BUS_MAX_INPUTS`` sources.
        sample_rate: unused (kept for the common processor signature).
        impulse_response: ``(bs, K, S, O, L)``, one trajectory set per item, or ``(1, K, S, O, L)``, one set shared by
            the batch; ``K >= 1``, ``O`` is 1 (mono bus) or 2 (stereo bus), any ``L >= 1``.  Row ``(k, s, o)`` is the
            path from source ``s`` to output ``o`` at anchor ``k``.
        hop: the anchor spacing in samples, a positive multiple of ``CONV_PARTITION_SAMPLES`` (4096), so that every
            output block and every gradient block lies inside one anchor interval; ``(K - 1) * hop < n``.  All
            sources share the one anchor grid.
        crossfade: ``"output"`` (the default: a moving listener) or ``"input"`` (a moving source), keyword only.

    Returns ``(bs, O, n)`` in x's dtype, computed in fp32.  There is no dry/wet mix, as in ``convolution_bus``.

    Identities (held to fp32 rounding), for ``crossfade="output"``:

    1. ``K = 1``: ``convolution_bus(x, sr, h[:, 0])``; K equal sets: ``convolution_bus`` with that set.
    2. ``S = 1, O = 2``: ``time_varying_convolution_reverberation(x, sr, h[:, :, 0], hop, mix=1)``.
    3. Any ``S``: the sum over ``s`` of ``time_varying_convolution_bus(x[:, s:s+1], sr, h[:, :, s:s+1], hop)``.
    4. From the last anchor on (``t >= (K - 1) hop``): ``convolution_bus(x, sr, h[:, K - 1])``.

    and for ``crossfade="input"``:

    1. ``K = 1``: ``convolution_bus(x, sr, h[:, 0])``; K equal sets: ``convolution_bus`` with that set.
    2. Any ``S``: the sum over ``s`` of the single-source calls, as above.
    3. ``sum_k convolution_bus(w_k x, sr, h[:, k])``, the segment composition, with ``w_k`` broadcast over the sources.
    4. Emission time: a unit impulse at ``tau`` between anchors ``k`` and ``k + 1`` (weight ``a``) gives
       ``(1 - a) h[:, k] + a h[:, k + 1]`` starting at ``tau``, over its whole tail.

    Gradients flow to ``x`` (every source) and to every IR row; taps at or beyond ``min(L, n)`` reach no output and
    get exactly 0.  The gradient of a shared ``(1, K, S, O, L)`` set has that shape and is the sum over the items,
    accumulated in fp64 in item order, so it does not depend on ``REVERB_CHUNK_ITEMS``.  When the IRs do not require a
    gradient, the backward skips all dL/dIR work.  This holds for both crossfades.

    Cost of ``"output"``: the rows of every signal are packed two per transform, as in ``convolution_bus``: ceil(S / 2)
    window transforms per block, transformed and kept for the backward once for all K sets; the K S O IR rows' partitions in
    ceil(K S O / 2) transforms per partition; one product per IR set and block summed over the sources, and one inverse
    transform per output row and crossfaded block (a mono bus: per block).  S ``time_varying_convolution_reverberation``
    calls would transform and keep every window S times and take S sets of inverse transforms.  A source that does not
    move repeats its IR in every set: its partitions are transformed and kept K times, and a crossfaded block multiplies
    its windows by both copies, for the static convolution's result (a crossfade of two equal outputs).  Rows whose
    length is not a multiple of 4 are zero-padded to one (the transforms bulk-copy 16-byte rows); a padding sample
    reaches no output sample below ``n``.

    Cost of ``"input"``: a block between two anchors is weighted per source and transformed zero-padded, one transform
    per source carrying both weighted pieces (1 - a and a), so the window transforms and the spectra kept for the
    backward are S per crossfaded block instead of ceil(S / 2); after the last anchor two sources share a transform.
    The partitions are those of ``"output"``.  Each output block takes one product (both IR sets of every input block it
    reaches, summed over the sources, the overlap-add of the zero-padded blocks done on the spectra) and one inverse
    transform for both bus rows.  The backward transforms the gradient once per block for both rows, and takes one dL/dx
    inverse per source and crossfaded block (ceil(S / 2) per later block).  The segment composition above would
    transform every block of every source once per segment it falls in, and its segments' tails again.
    """
    xf, irf, n, dt, hop = _tv_bus_inputs(x, impulse_response, hop, crossfade, "time_varying_convolution_bus", 2)
    entry = "tvbus" if crossfade == "output" else "tvbus_in"
    y = _TvBusFn.apply(xf, irf, hop, reverb_chunk_items(xf.device), entry)
    return (y[..., :n] if xf.shape[-1] != n else y).to(dt)


def time_varying_multichannel_convolution(x: torch.Tensor, sample_rate: float, impulse_response: torch.Tensor,
                                          hop: int, *, crossfade: str = "output"):
    """Moving sources through a trajectory of S x M impulse-response matrices into M output channels:
    ``multichannel_convolution`` whose matrix changes over time, as ``time_varying_convolution_bus``'s IR sets do.
    Matrix ``k`` of the trajectory, ``h[:, k]``, is a complete ``multichannel_convolution`` matrix, the scene at the
    anchor time ``t_k = k * hop``.  ``crossfade`` chooses where the weights apply::

        "output":  y[:, m](t) = sum_k w_k(t) sum_s (x[:, s] * h[:, k, s, m])(t)
        "input":   y[:, m](t) = sum_k sum_s ((w_k x[:, s]) * h[:, k, s, m])(t)

    with ``time_varying_convolution_bus``'s crossfade weights ``w_k`` and ``*``.  This is that op with up to
    ``CONV_MC_MAX_OUTPUTS`` output rows.  ``"input"`` is the model of moving point sources: every emitted sample keeps
    the matrix of its emission time over its whole tail.  ``"output"`` models a moving array or listener.  Uses: moving
    talkers recorded by a 4- to 32-microphone array, to train direction-of-arrival tracking, multichannel separation and
    enhancement; ambisonic scenes with moving objects (4, 16 or 25 channels); 5.1 / 7.1 renders of moving sources.

    Args:
        x: audio ``(bs, S, n)``, ``1 <= S <= CONV_BUS_MAX_INPUTS`` sources.
        sample_rate: unused (kept for the common processor signature).
        impulse_response: ``(bs, K, S, M, L)``, one trajectory per item, or ``(1, K, S, M, L)``, one trajectory shared
            by the batch; ``K >= 1``, ``1 <= M <= CONV_MC_MAX_OUTPUTS``, any ``L >= 1``.  Row ``(k, s, m)`` is the
            path from source ``s`` to output ``m`` (microphone, ambisonic channel or speaker feed) at anchor ``k``.
        hop: the anchor spacing in samples, a positive multiple of ``CONV_PARTITION_SAMPLES`` (4096);
            ``(K - 1) * hop < n``.  All sources share the one anchor grid.
        crossfade: ``"output"`` (the default) or ``"input"``, keyword only.

    Returns ``(bs, M, n)`` in x's dtype, computed in fp32.  There is no dry/wet mix, as in ``convolution_bus``.

    Identities (held to fp32 rounding), for both crossfades:

    1. ``M <= 2``: ``time_varying_convolution_bus(x, sr, h, hop, crossfade=...)``, bit for bit.
    2. Any ``M``: the concatenation over the output pairs ``q`` of
       ``time_varying_convolution_bus(x, sr, h[:, :, :, 2q:2q+2], hop, crossfade=...)``.
    3. ``K = 1`` or K equal matrices: ``multichannel_convolution`` with that matrix.
    4. Any ``S``: the sum over ``s`` of the single-source calls ``x[:, s:s+1]``, ``h[:, :, s:s+1]``.
    5. ``"output"``: from the last anchor on (``t >= (K - 1) hop``), ``multichannel_convolution(x, sr, h[:, K - 1])``.
    6. ``"input"``: ``sum_k multichannel_convolution(w_k x, sr, h[:, k])``, and a unit impulse at ``tau`` between
       anchors ``k`` and ``k + 1`` (weight ``a``) gives ``(1 - a) h[:, k] + a h[:, k + 1]`` from ``tau`` on.

    Gradients flow to ``x`` (every source) and to every IR row; taps at or beyond ``min(L, n)`` reach no output and
    get exactly 0.  The gradient of a shared ``(1, K, S, M, L)`` trajectory has that shape and is the sum over the
    items, accumulated in fp64 in item order, so it does not depend on ``REVERB_CHUNK_ITEMS``.  When the IRs do not
    require a gradient, the backward skips all dL/dIR work.  Rows whose length is not a multiple of 4 are zero-padded
    to one; a padding sample reaches no output sample below ``n``.

    Cost, in 8192-point transforms per item, with ``I = ceil(n / 4096)`` blocks, ``nX = (K - 1) hop / 4096``
    crossfaded blocks, ``J = ceil(min(L, n) / 4096)`` partitions, ``P = ceil(S / 2)``, ``Q = ceil(M / 2)`` and
    ``NH = ceil(K S M / 2)``:

    ============================  ===========================  ===========================
    transforms                    ``"output"``                 ``"input"``
    ============================  ===========================  ===========================
    window (forward)              ``P I``                      ``S nX + P (I - nX)``
    partition (forward)           ``NH J``                     ``NH J``
    output inverse                ``M nX + Q (I - nX)``        ``Q I``
    gradient (backward)           ``M nX + Q (I - nX)``        ``Q I``
    dL/dx inverse                 ``P I``                      ``S nX + P (I - nX)``
    dL/dIR inverse                ``NH J``                     ``NH J``
    spectra kept for backward     ``P I + NH J``               ``S nX + P (I - nX) + NH J``
    ============================  ===========================  ===========================

    Identity 2's Q calls would take the window and dL/dx transforms, and keep the window spectra, Q times over, and
    autograd would sum their Q copies of dL/dx.  A crossfaded block takes one output inverse per output row
    (``"output"``: both IR sets of the row in one spectrum); ``"input"`` takes one per output pair and block.
    """
    xf, irf, n, dt, hop = _tv_bus_inputs(x, impulse_response, hop, crossfade, "time_varying_multichannel_convolution",
                                         CONV_MC_MAX_OUTPUTS)
    entry = "tvmc" if crossfade == "output" else "tvmc_in"
    y = _TvBusFn.apply(xf, irf, hop, reverb_chunk_items(xf.device), entry)
    return (y[..., :n] if xf.shape[-1] != n else y).to(dt)
