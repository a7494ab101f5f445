"""CPU checks of time_varying_multichannel_convolution: both time-varying bus oracles (tests/tv_bus_oracle.py,
tests/tv_bus_input_oracle.py) at M >= 3 outputs against their direct form and their output-pair composition; the
geometry queries of both crossfades without a GPU, up to S = M = 32 and at the benchmark's size; the entry points at
bs = 0 and on bad arguments; the Python checks; and time_varying_convolution_bus still rejecting three outputs."""
import pytest
import torch

import conv_bus_oracle
import tv_bus_input_oracle
import tv_bus_oracle
from helpers import SR

KB, NFFT = 4096, 8192
ORACLES = {"output": tv_bus_oracle, "input": tv_bus_input_oracle}
PREFIX = {"output": "dasp_tvmc", "input": "dasp_tvmc_in"}


@pytest.fixture(scope="module")
def lib():
    from dasp_pytorch_b200 import _abi, build
    build.build()
    return _abi.lib()


def _rand(gen, *shape):
    return torch.rand(*shape, generator=gen, dtype=torch.float64) * 2 - 1


def _rel(a, b):
    return float((a - b).abs().max() / b.abs().max())


def _align(v):
    return (v + 255) // 256 * 256


def _entries(crossfade):
    p = PREFIX[crossfade]
    return (f"{p}_fwd", f"{p}_shared_fwd", f"{p}_bwd", f"{p}_shared_bwd")


@pytest.mark.parametrize("crossfade", ["output", "input"])
@pytest.mark.parametrize("S,M,shared", [(1, 3, False), (3, 4, True), (2, 5, False), (4, 8, True), (2, 32, False)])
def test_tv_mc_oracles_direct_fft_and_output_pairs_agree(crossfade, S, M, shared):
    """the oracles state any M: their direct and FFT forms agree, and each is the concatenation of its output-pair
    calls"""
    oracle = ORACLES[crossfade]
    gen = torch.Generator().manual_seed(S * 40 + M)
    x, h = _rand(gen, 2, S, 3000), _rand(gen, 1 if shared else 2, 3, S, M, 700)
    y = oracle.time_varying_convolution_bus(x, SR, h, 1024)
    assert y.shape == (2, M, 3000)
    assert _rel(y, oracle.time_varying_convolution_bus(x, SR, h, 1024, method="direct")) < 1e-12
    pairs = torch.cat([oracle.time_varying_convolution_bus(x, SR, h[:, :, :, q:q + 2], 1024, method="direct")
                       for q in range(0, M, 2)], 1)
    assert _rel(y, pairs) < 1e-12


@pytest.mark.parametrize("crossfade", ["output", "input"])
def test_tv_mc_oracles_with_equal_sets_are_the_static_oracle(crossfade):
    gen = torch.Generator().manual_seed(7)
    x, h = _rand(gen, 2, 3, 2500), _rand(gen, 2, 1, 3, 6, 900)
    ref = conv_bus_oracle.convolution_bus(x, SR, h[:, 0])
    got = ORACLES[crossfade].time_varying_convolution_bus(x, SR, h.expand(2, 4, 3, 6, 900), 600)
    assert _rel(got, ref) < 1e-12


# (n, L, K, S, M, hop, leff, ir_partitions)
GEOMS = [(480000, 48000, 15, 4, 8, 8 * KB, 48000, 12), (480000, 48000, 15, 4, 4, 8 * KB, 48000, 12),
         (64000, 8000, 8, 2, 8, 2 * KB, 8000, 2), (60000, 9000, 5, 3, 5, 3 * KB, 9000, 3),
         (4097, 1, 2, 1, 3, KB, 1, 1), (20001, 30000, 3, 5, 7, KB, 20001, 5), (100, 50, 1, 32, 32, KB, 50, 1),
         (70000, 66000, 15, 2, 3, KB, 66000, 17), (200000, 5000, 4, 7, 16, 3 * KB, 5000, 2),
         (600000, 20000, 127, 32, 32, KB, 20000, 5), (20000, 9000, 3, 3, 1, KB, 9000, 3),
         (20000, 9000, 3, 5, 2, KB, 9000, 3)]


def _check_geometry(lib, crossfade, n, L, K, S, M, hop, leff, J, shared, bs=10, chunk=4):
    """the sizes follow from the design: P = ceil(S / 2), Q = ceil(M / 2), nX = (K - 1) hop / 4096 crossfaded blocks,
    NH = ceil(K S M / 2) partition sets.  Output side: P I window spectra, U = M nX + Q (I - nX) product and gradient
    slots per item.  Source side: XW = nX S + (I - nX) P window and dL/dx spectra, Q I product and gradient spectra per
    item.  A shared trajectory adds the fp64 sum of its dL/dIR spectra to the backward workspace."""
    from dasp_pytorch_b200 import _abi
    I, P, Q, NH, nX = -(-n // KB), (S + 1) // 2, (M + 1) // 2, (K * S * M + 1) // 2, (K - 1) * hop // KB
    if crossfade == "output":
        XW, U = P * I, M * nX + Q * (I - nX)
    else:
        XW, U = nX * S + (I - nX) * P, Q * I
    g = _abi.ConvGeom()
    assert getattr(lib, f"{PREFIX[crossfade]}_geometry")(bs, n, L, K, S, M, hop, shared, chunk, g) == 0
    c = g.chunk_items
    assert (g.leff, g.conv_block, g.x_blocks, g.ir_partitions) == (leff, KB, I, J)
    assert c == min(chunk, bs)
    assert g.xspec_c64 == bs * XW * NFFT
    assert g.irspec_c64 == (1 if shared else bs) * NH * J * NFFT
    blk = 8 * NFFT
    fwd = _align(c * U * blk) + _align(c * XW * blk) + _align((1 if shared else c) * NH * J * blk)
    bwd = (_align(c * U * blk) + _align(c * XW * blk) + _align(c * NH * J * blk)
           + (_align(16 * NH * J * NFFT) if shared else 0))
    assert g.fwd_workspace_bytes == fwd and g.bwd_workspace_bytes == bwd
    return g


@pytest.mark.parametrize("crossfade", ["output", "input"])
@pytest.mark.parametrize("shared", [0, 1])
@pytest.mark.parametrize("n,L,K,S,M,hop,leff,J", GEOMS)
def test_tv_mc_geometry_without_gpu(lib, crossfade, n, L, K, S, M, hop, leff, J, shared):
    _check_geometry(lib, crossfade, n, L, K, S, M, hop, leff, J, shared)


@pytest.mark.parametrize("crossfade", ["output", "input"])
@pytest.mark.parametrize("shared", [0, 1])
@pytest.mark.parametrize("S,M,K", [(3, 1, 1), (5, 2, 3), (16, 2, 4), (4, 1, 5)])
def test_tv_mc_geometry_is_the_tv_bus_geometry_up_to_two_outputs(lib, crossfade, S, M, K, shared):
    from dasp_pytorch_b200 import _abi
    a, b = _abi.ConvGeom(), _abi.ConvGeom()
    tv = "dasp_tvbus" if crossfade == "output" else "dasp_tvbus_in"
    assert getattr(lib, f"{PREFIX[crossfade]}_geometry")(6, 50000, 30000, K, S, M, KB, shared, 4, a) == 0
    assert getattr(lib, f"{tv}_geometry")(6, 50000, 30000, K, S, M, KB, shared, 4, b) == 0
    assert [getattr(a, f) for f, _ in a._fields_] == [getattr(b, f) for f, _ in b._fields_]


def test_tv_mc_geometry_at_the_benchmark_size(lib):
    """48 kHz, S 4, M 8, n 480 000, L 48 000, hop 32 768, K 15: I = 118, nX = 112, J = 12, 240 partition sets.  Kept
    for the backward per item: 236 window + 2880 partition spectra (output side), 460 + 2880 (source side); 920 and 472
    product slots"""
    g = _check_geometry(lib, "output", 480000, 48000, 15, 4, 8, 8 * KB, 48000, 12, 0, bs=2, chunk=2)
    assert (g.xspec_c64 + g.irspec_c64) // (2 * NFFT) == 3116
    g = _check_geometry(lib, "input", 480000, 48000, 15, 4, 8, 8 * KB, 48000, 12, 0, bs=2, chunk=2)
    assert (g.xspec_c64 + g.irspec_c64) // (2 * NFFT) == 3340


BAD_GEOMS = [  # (bs, n, L, K, S, M, hop, message)
    (2, 1000, 10, 1, 0, 4, KB, "tvmc: 1 to 32 inputs"), (2, 1000, 10, 1, 33, 4, KB, "tvmc: 1 to 32 inputs"),
    (2, 1000, 10, 1, 2, 0, KB, "tvmc: 1 to 32 outputs are supported, got 0"),
    (2, 1000, 10, 1, 2, 33, KB, "tvmc: 1 to 32 outputs are supported, got 33"),
    (2, 1000, 10, 0, 2, 4, KB, "K >= 1"), (2, 1000, 10, -1, 2, 4, KB, "K >= 1"),
    (2, 1000, 10, 1, 2, 4, 0, "multiple of 4096"), (2, 1000, 10, 1, 2, 4, 4000, "multiple of 4096"),
    (2, 1000, 10, 1, 2, 4, -KB, "multiple of 4096"),
    (2, 4096, 10, 2, 2, 4, KB, "end of x"), (2, 40000, 10, 11, 2, 5, KB, "end of x"),
    (2, 0, 10, 1, 2, 4, KB, "bad shape"), (2, 100, 0, 1, 2, 4, KB, "bad shape"), (-1, 100, 10, 1, 2, 4, KB, "bad shape"),
    (2, 1 << 40, 10, 1 << 40, 2, 4, KB, "end of x"),
    (2, 1 << 24, 10, 128, 32, 32, KB, "at most 65535 partition sets")]


@pytest.mark.parametrize("crossfade", ["output", "input"])
@pytest.mark.parametrize("bs,n,L,K,S,M,hop,msg", BAD_GEOMS)
def test_tv_mc_entry_points_reject_bad_arguments_before_any_launch(lib, crossfade, bs, n, L, K, S, M, hop, msg):
    """every entry point checks S, M, K, hop, lengths and the partition-set limit before it touches a pointer or the
    device (all pointers here are null, so any launch would fault)"""
    from dasp_pytorch_b200 import _abi
    assert getattr(lib, f"{PREFIX[crossfade]}_geometry")(bs, n, L, K, S, M, hop, 0, 4, _abi.ConvGeom()) < 0
    assert msg in lib.dasp_last_error().decode()
    for name in _entries(crossfade):
        assert getattr(lib, name)(None, None, None, None, None, None, 0, bs, n, L, K, S, M, hop, 4, None) < 0
        assert msg in lib.dasp_last_error().decode()


@pytest.mark.parametrize("crossfade", ["output", "input"])
def test_tv_mc_accepts_the_largest_trajectory_at_32_by_32(lib, crossfade):
    """S = M = 32: K = 127 is 65024 partition sets, K = 128 is 65536"""
    from dasp_pytorch_b200 import _abi
    geom = getattr(lib, f"{PREFIX[crossfade]}_geometry")
    assert geom(0, 127 * KB + 1, 10, 127, 32, 32, KB, 0, 4, _abi.ConvGeom()) == 0
    assert geom(0, 128 * KB + 1, 10, 128, 32, 32, KB, 0, 4, _abi.ConvGeom()) < 0


@pytest.mark.parametrize("crossfade", ["output", "input"])
def test_tv_mc_geometry_rejects_a_null_out(lib, crossfade):
    assert getattr(lib, f"{PREFIX[crossfade]}_geometry")(2, 8192, 100, 2, 3, 4, KB, 0, 4, None) < 0
    assert "null out" in lib.dasp_last_error().decode()


@pytest.mark.parametrize("crossfade", ["output", "input"])
def test_tv_mc_entry_points_reject_null_pointers_and_unaligned_rows(lib, crossfade):
    """with a valid geometry: null pointers, one of the two *_save buffers, n % 4 != 0 and unaligned x / gy rows are
    rejected before any launch (the fake addresses are never dereferenced)"""
    fake, odd = 1 << 20, (1 << 20) + 4
    p = PREFIX[crossfade]
    for f in (getattr(lib, f"{p}_fwd"), getattr(lib, f"{p}_shared_fwd")):
        fwd = lambda x, n=8192, xs=None, irs=None, ir=fake, y=fake: f(x, ir, y, xs, irs, fake, 1 << 40, 2, n, 100, 2,
                                                                       3, 5, KB, 2, None)
        assert fwd(None) < 0 and "null pointer" in lib.dasp_last_error().decode()
        assert fwd(fake, ir=None) < 0 and "null pointer" in lib.dasp_last_error().decode()
        assert fwd(fake, y=None) < 0 and "null pointer" in lib.dasp_last_error().decode()
        assert fwd(fake, xs=fake) < 0 and "both *_save" in lib.dasp_last_error().decode()
        assert fwd(fake, n=8190) < 0 and "n % 4 == 0" in lib.dasp_last_error().decode()
        assert fwd(odd) < 0 and "16-byte aligned" in lib.dasp_last_error().decode()
    for f in (getattr(lib, f"{p}_bwd"), getattr(lib, f"{p}_shared_bwd")):
        bwd = lambda gy, xs=fake, gx=fake, n=8192: f(gy, xs, fake, gx, None, fake, 1 << 40, 2, n, 100, 2, 3, 5, KB, 2,
                                                    None)
        assert bwd(None) < 0 and "null pointer" in lib.dasp_last_error().decode()
        assert bwd(fake, xs=None) < 0 and "null pointer" in lib.dasp_last_error().decode()
        assert bwd(fake, gx=None) < 0 and "null pointer" in lib.dasp_last_error().decode()
        assert bwd(fake, n=8190) < 0 and "n % 4 == 0" in lib.dasp_last_error().decode()
        assert bwd(odd) < 0 and "16-byte aligned" in lib.dasp_last_error().decode()


@pytest.mark.parametrize("crossfade", ["output", "input"])
def test_tv_mc_batch_zero_is_a_no_op(lib, crossfade):
    """bs = 0 returns before any pointer is read or any CUDA call is made"""
    from dasp_pytorch_b200 import _abi
    g = _abi.ConvGeom()
    assert getattr(lib, f"{PREFIX[crossfade]}_geometry")(0, 8192, 100, 2, 3, 6, KB, 0, 4, g) == 0
    assert g.xspec_c64 == 0 and g.irspec_c64 == 0
    for name in _entries(crossfade):
        assert getattr(lib, name)(None, None, None, None, None, None, 0, 0, 8192, 100, 2, 3, 6, KB, 4, None) == 0


def test_tv_bus_entry_points_still_reject_three_outputs(lib):
    from dasp_pytorch_b200 import _abi
    for p in ("dasp_tvbus", "dasp_tvbus_in"):
        assert getattr(lib, f"{p}_geometry")(0, 8192, 100, 2, 3, 3, KB, 0, 4, _abi.ConvGeom()) < 0
        assert "tvbus: a mono (1) or stereo (2) bus, got 3 outputs" in lib.dasp_last_error().decode()
        for name in (f"{p}_fwd", f"{p}_shared_fwd", f"{p}_bwd", f"{p}_shared_bwd"):
            assert getattr(lib, name)(None, None, None, None, None, None, 0, 2, 8192, 100, 2, 3, 3, KB, 4, None) < 0
            assert "tvbus: a mono (1) or stereo (2) bus, got 3 outputs" in lib.dasp_last_error().decode()


def _x(bs=2, S=3, n=9000):
    return torch.zeros(bs, S, n)


def _h(bs=2, K=2, S=3, M=6, L=10):
    return torch.zeros(bs, K, S, M, L)


def _call(x, ir, hop=KB, crossfade="output"):
    import dasp_pytorch_b200 as D
    return D.time_varying_multichannel_convolution(x, SR, ir, hop, crossfade=crossfade)


@pytest.mark.parametrize("crossfade", ["both", "Input", "", None, 1])
def test_tv_mc_rejects_a_bad_crossfade(crossfade):
    with pytest.raises(ValueError) as e:
        _call(_x(), _h(), crossfade=crossfade)
    assert str(e.value) == f'crossfade must be "output" or "input", got {crossfade!r}'


@pytest.mark.parametrize("crossfade", ["output", "input"])
@pytest.mark.parametrize("x,ir,hop,msg", [
    (torch.zeros(2, 9000), _h(), KB, "x must be a tensor of shape (batch, inputs, samples)"),
    (_x(), torch.zeros(2, 3, 6, 10), KB,
     "impulse_response must be a tensor of shape (batch, K, inputs, outputs, taps)"),
    (_x(S=0), _h(S=0), KB, "time_varying_multichannel_convolution: 1 to 32 input channels are supported, got 0"),
    (_x(S=33), _h(S=33), KB, "time_varying_multichannel_convolution: 1 to 32 input channels are supported, got 33"),
    (_x(), _h(S=4), KB, "impulse_response has 4 input rows, x has 3 channels"),
    (_x(), _h(M=0), KB, "impulse_response: 1 to 32 output channels are supported, got 0"),
    (_x(), _h(M=33), KB, "impulse_response: 1 to 32 output channels are supported, got 33"),
    (_x(), _h(K=0), KB, "impulse_response needs at least one impulse-response set (K >= 1)"),
    (_x(), _h(bs=3), KB, "impulse_response has batch 3, x has batch 2 (expected 2 or 1)"),
    (_x(n=0), _h(), KB, "x needs at least one sample"),
    (_x(), _h(), 4000, "hop must be a positive multiple of 4096 samples, got 4000"),
    (_x(n=8192), _h(K=3), KB, "impulse response 2 is anchored at (K - 1) * hop = 8192, at or after the end of x (8192 "
     "samples)")])
def test_tv_mc_value_errors(crossfade, x, ir, hop, msg):
    with pytest.raises(ValueError) as e:
        _call(x, ir, hop, crossfade)
    assert str(e.value) == msg


def test_tv_mc_rejects_an_ir_without_taps():
    with pytest.raises(ValueError, match="at least one tap"):
        _call(_x(), _h(L=0))


@pytest.mark.parametrize("crossfade", ["output", "input"])
def test_tv_bus_still_rejects_three_outputs(crossfade):
    import dasp_pytorch_b200 as D
    with pytest.raises(ValueError) as e:
        D.time_varying_convolution_bus(_x(), SR, _h(M=3), KB, crossfade=crossfade)
    assert str(e.value) == "impulse_response: a mono (1) or stereo (2) bus is supported, got 3 outputs"


def test_tv_mc_rejects_cpu_tensors_and_is_exported():
    import dasp_pytorch_b200 as D
    from dasp_pytorch_b200._abi import DaspError
    for crossfade in ("output", "input"):
        with pytest.raises(DaspError, match="no CPU path"):
            _call(_x(), _h(), crossfade=crossfade)
    assert "time_varying_multichannel_convolution" in D.functional.__all__
    assert D.time_varying_multichannel_convolution is D.functional.time_varying_multichannel_convolution


def test_tv_mc_crossfade_is_keyword_only():
    import dasp_pytorch_b200 as D
    with pytest.raises(TypeError):
        D.time_varying_multichannel_convolution(_x(), SR, _h(), KB, "input")
