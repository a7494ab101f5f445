"""CPU checks of time_varying_convolution_bus: its fp64 oracle (tests/tv_bus_oracle.py) against itself, against the
static bus oracle and against the single-source time-varying oracle; the geometry query without a GPU (including the
benchmark's size); the entry points at bs = 0 and on bad arguments; and the shapes and values the op rejects before
any launch."""
import pytest
import torch

import conv_bus_oracle
import tv_bus_oracle
import tv_conv_oracle
from helpers import SR

KB, NFFT = 4096, 8192


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


@pytest.mark.parametrize("S,O,shared", [(1, 2, False), (3, 1, True), (4, 2, True), (5, 1, False)])
def test_tv_bus_oracle_methods_agree(S, O, shared):
    gen = torch.Generator().manual_seed(S * 10 + O)
    x, h = _rand(gen, 2, S, 3000), _rand(gen, 1 if shared else 2, 3, S, O, 700)
    a = tv_bus_oracle.time_varying_convolution_bus(x, SR, h, 1024, method="fft")
    b = tv_bus_oracle.time_varying_convolution_bus(x, SR, h, 1024, method="direct")
    assert a.shape == (2, O, 3000) and _rel(a, b) < 1e-12


@pytest.mark.parametrize("method", ["fft", "direct"])
@pytest.mark.parametrize("S,O", [(3, 2), (2, 1)])
def test_tv_bus_oracle_at_one_anchor_is_the_bus_oracle(method, S, O):
    gen = torch.Generator().manual_seed(3 + S)
    x, h = _rand(gen, 3, S, 2500), _rand(gen, 3, 1, S, O, 900)
    got = tv_bus_oracle.time_varying_convolution_bus(x, SR, h, 4096, method=method)
    assert _rel(got, conv_bus_oracle.convolution_bus(x, SR, h[:, 0], method=method)) < 1e-12


def test_tv_bus_oracle_for_one_source_is_the_tv_oracle_at_mix_1():
    """S = 1: a stereo bus is the time-varying op with the stereo IR h[:, :, 0] at mix 1; a mono bus is channel 0 of
    the time-varying op with the mono IR"""
    gen = torch.Generator().manual_seed(5)
    x, h = _rand(gen, 2, 1, 5000), _rand(gen, 2, 4, 1, 2, 600)
    one = torch.ones(2, dtype=torch.float64)
    got = tv_bus_oracle.time_varying_convolution_bus(x, SR, h, 1000)
    assert _rel(got, tv_conv_oracle.time_varying_convolution_reverberation(x, SR, h[:, :, 0], 1000, one)) < 1e-12
    got = tv_bus_oracle.time_varying_convolution_bus(x, SR, h[..., :1, :], 1000)
    ref = tv_conv_oracle.time_varying_convolution_reverberation(x, SR, h[:, :, 0, :1], 1000, one)
    assert got.shape == (2, 1, 5000) and _rel(got, ref[:, :1]) < 1e-12


def test_tv_bus_oracle_is_the_sum_of_its_sources():
    gen = torch.Generator().manual_seed(6)
    S = 4
    x, h = _rand(gen, 2, S, 4000), _rand(gen, 2, 3, S, 2, 500)
    y = tv_bus_oracle.time_varying_convolution_bus(x, SR, h, 1500)
    parts = sum(tv_bus_oracle.time_varying_convolution_bus(x[:, s:s + 1], SR, h[:, :, s:s + 1], 1500, method="direct")
                for s in range(S))
    assert _rel(y, parts) < 1e-12


# (n, L, K, S, O, hop, leff, ir_partitions)
GEOMS = [(480000, 48000, 15, 4, 2, 8 * KB, 48000, 12), (60000, 9000, 5, 3, 1, 3 * KB, 9000, 3),
         (4097, 1, 2, 1, 2, KB, 1, 1), (20001, 30000, 3, 5, 1, KB, 20001, 5), (100, 50, 1, 32, 2, KB, 50, 1),
         (70000, 66000, 15, 2, 1, KB, 66000, 17)]


def _check_geometry(lib, n, L, K, S, O, hop, leff, J, shared, bs=10, chunk=4):
    """the sizes follow from the design: ceil(S / 2) window spectra per block (the bus's), ceil(K S O / 2) partition
    sets per trajectory set, and U product and gradient spectra per item: I + (K - 1) hop / 4096 for a stereo bus (two
    for every crossfaded block), I for a mono bus; a shared set adds the fp64 sum of its dL/dIR spectra to the backward
    workspace, and there is no dL/dmix region"""
    from dasp_pytorch_b200 import _abi
    I, P, NH = -(-n // KB), (S + 1) // 2, (K * S * O + 1) // 2
    U = I + (K - 1) * hop // KB if O == 2 else I
    g = _abi.ConvGeom()
    assert lib.dasp_tvbus_geometry(bs, n, L, K, S, O, hop, shared, chunk, g) == 0
    c = g.chunk_items
    assert (g.leff, g.conv_block, g.x_blocks, g.ir_partitions) == (leff, KB, I, J)
    assert c == min(chunk, bs)
    assert g.xspec_c64 == bs * P * I * NFFT
    assert g.irspec_c64 == (1 if shared else bs) * NH * J * NFFT
    blk = 8 * NFFT
    fwd = _align(c * U * blk) + _align(c * P * I * blk) + _align((1 if shared else c) * NH * J * blk)
    bwd = (_align(c * U * blk) + _align(c * P * I * blk) + _align(c * NH * J * blk)
           + (_align(16 * NH * J * NFFT) if shared else 0))
    assert g.fwd_workspace_bytes == fwd and g.bwd_workspace_bytes == bwd
    return g


@pytest.mark.parametrize("n,L,K,S,O,hop,leff,J", GEOMS)
@pytest.mark.parametrize("shared", [0, 1])
def test_tvbus_geometry_without_gpu(lib, n, L, K, S, O, hop, leff, J, shared):
    _check_geometry(lib, n, L, K, S, O, hop, leff, J, shared)


def test_tvbus_workspaces_grow_with_K_S_and_O(lib):
    from dasp_pytorch_b200 import _abi

    def sizes(K, S, O):
        g = _abi.ConvGeom()
        assert lib.dasp_tvbus_geometry(4, 100000, 20000, K, S, O, 2 * KB, 0, 4, g) == 0
        return g.xspec_c64, g.irspec_c64, g.fwd_workspace_bytes, g.bwd_workspace_bytes

    base = sizes(3, 3, 1)
    for more in (sizes(5, 3, 1), sizes(3, 5, 1), sizes(3, 3, 2)):
        assert all(b >= a for a, b in zip(base, more)) and more[1] > base[1]
        assert more[2] > base[2] and more[3] > base[3]
    assert sizes(3, 5, 1)[0] > base[0]                 # more window spectra per block


def test_tvbus_geometry_at_the_benchmark_size(lib):
    """64 x 4 x 480 000, L 48 000, hop 32 768, K 15, stereo bus, in one chunk: 2 x 118 window spectra and 720
    partition spectra (15 sets of 4 stereo IRs, 12 partitions each) of 64 KiB per item are kept for the backward"""
    for shared in (0, 1):
        g = _check_geometry(lib, 480000, 48000, 15, 4, 2, 8 * KB, 48000, 12, shared, bs=64, chunk=64)
        assert g.xspec_c64 * 8 == 64 * 236 * 64 * 1024
        assert g.irspec_c64 * 8 == (1 if shared else 64) * 720 * 64 * 1024


BAD_GEOMS = [  # (bs, n, L, K, S, O, hop, message)
    (2, 1000, 10, 1, 0, 2, KB, "1 to 32 inputs"), (2, 1000, 10, 1, 33, 2, KB, "1 to 32 inputs"),
    (2, 1000, 10, 1, 2, 0, KB, "mono (1) or stereo (2) bus"), (2, 1000, 10, 1, 2, 3, KB, "mono (1) or stereo (2)"),
    (2, 1000, 10, 0, 2, 2, KB, "K >= 1"), (2, 1000, 10, 1, 2, 2, 0, "multiple of 4096"),
    (2, 1000, 10, 1, 2, 2, 4000, "multiple of 4096"), (2, 1000, 10, 1, 2, 2, -KB, "multiple of 4096"),
    (2, 4096, 10, 2, 2, 2, KB, "end of x"), (2, 40000, 10, 11, 2, 1, KB, "end of x"),
    (2, 0, 10, 1, 2, 2, KB, "bad shape"), (2, 100, 0, 1, 2, 2, KB, "bad shape"), (-1, 100, 10, 1, 2, 2, KB, "bad shape"),
    (2, 1 << 40, 10, 1 << 40, 2, 2, KB, "end of x"), (2, 1 << 24, 10, 2048, 32, 2, KB, "at most 65535 partition sets")]


@pytest.mark.parametrize("bs,n,L,K,S,O,hop,msg", BAD_GEOMS)
def test_tvbus_entry_points_reject_bad_arguments_before_any_launch(lib, bs, n, L, K, S, O, hop, msg):
    """every entry point checks S, O, K, hop and lengths before it touches a pointer or the device (all pointers here
    are null, so any launch would fault)"""
    from dasp_pytorch_b200 import _abi
    assert lib.dasp_tvbus_geometry(bs, n, L, K, S, O, hop, 0, 4, _abi.ConvGeom()) < 0
    assert msg in lib.dasp_last_error().decode()
    for name in ("dasp_tvbus_fwd", "dasp_tvbus_shared_fwd", "dasp_tvbus_bwd", "dasp_tvbus_shared_bwd"):
        assert getattr(lib, name)(None, None, None, None, None, None, 0, bs, n, L, K, S, O, hop, 4, None) < 0
        assert msg in lib.dasp_last_error().decode()


def test_tvbus_entry_points_reject_null_pointers_and_unaligned_rows(lib):
    """with a valid geometry: null pointers, one of the two *_save buffers, n % 4 != 0 and unaligned x / gy rows are
    rejected before any launch (the fake addresses are never dereferenced)"""
    fake, odd = 1 << 20, (1 << 20) + 4
    for f in (lib.dasp_tvbus_fwd, lib.dasp_tvbus_shared_fwd):
        fwd = lambda x, n=8192, xs=None, irs=None, ir=fake, y=fake: f(x, ir, y, xs, irs, fake, 1 << 40, 2, n, 100, 2,
                                                                       3, 2, KB, 2, None)
        assert fwd(None) < 0 and "null pointer" in lib.dasp_last_error().decode()
        assert fwd(fake, ir=None) < 0 and "null pointer" in lib.dasp_last_error().decode()
        assert fwd(fake, y=None) < 0 and "null pointer" in lib.dasp_last_error().decode()
        assert fwd(fake, xs=fake) < 0 and "both *_save" in lib.dasp_last_error().decode()
        assert fwd(fake, n=8190) < 0 and "n % 4 == 0" in lib.dasp_last_error().decode()
        assert fwd(odd) < 0 and "16-byte aligned" in lib.dasp_last_error().decode()
    for f in (lib.dasp_tvbus_bwd, lib.dasp_tvbus_shared_bwd):
        bwd = lambda gy, xs=fake, gx=fake, n=8192: f(gy, xs, fake, gx, None, fake, 1 << 40, 2, n, 100, 2, 3, 2, KB, 2,
                                                    None)
        assert bwd(None) < 0 and "null pointer" in lib.dasp_last_error().decode()
        assert bwd(fake, xs=None) < 0 and "null pointer" in lib.dasp_last_error().decode()
        assert bwd(fake, gx=None) < 0 and "null pointer" in lib.dasp_last_error().decode()
        assert bwd(fake, n=8190) < 0 and "n % 4 == 0" in lib.dasp_last_error().decode()
        assert bwd(odd) < 0 and "16-byte aligned" in lib.dasp_last_error().decode()


def test_tvbus_batch_zero_is_a_no_op(lib):
    """bs = 0 returns before any pointer is read or any CUDA call is made"""
    from dasp_pytorch_b200 import _abi
    g = _abi.ConvGeom()
    assert lib.dasp_tvbus_geometry(0, 8192, 100, 2, 3, 2, KB, 0, 4, g) == 0 and g.xspec_c64 == 0
    for name in ("dasp_tvbus_fwd", "dasp_tvbus_shared_fwd", "dasp_tvbus_bwd", "dasp_tvbus_shared_bwd"):
        assert getattr(lib, name)(None, None, None, None, None, None, 0, 0, 8192, 100, 2, 3, 2, KB, 4, None) == 0


def _x(bs=2, S=3, n=9000):
    return torch.zeros(bs, S, n)


def _h(bs=2, K=2, S=3, O=2, L=10):
    return torch.zeros(bs, K, S, O, L)


BAD_CALLS = [  # (x, ir, hop, message)
    (torch.zeros(2, 9000), _h(), KB, "x must be a tensor of shape (batch, inputs, samples)"),
    (_x(), torch.zeros(2, 2, 3, 10), KB, "impulse_response must be a tensor of shape (batch, K, inputs, outputs, taps)"),
    (_x(S=0), _h(S=0), KB, "time_varying_convolution_bus: 1 to 32 input channels are supported, got 0"),
    (_x(S=33), _h(S=33), KB, "time_varying_convolution_bus: 1 to 32 input channels are supported, got 33"),
    (_x(), _h(S=4), KB, "impulse_response has 4 input rows, x has 3 channels"),
    (_x(), _h(O=3), KB, "impulse_response: a mono (1) or stereo (2) bus is supported, got 3 outputs"),
    (_x(), _h(K=0), KB, "impulse_response needs at least one impulse-response set (K >= 1)"),
    (_x(), _h(bs=3), KB, "impulse_response has batch 3, x has batch 2 (expected 2 or 1)"),
    (_x(bs=1), _h(bs=2), KB, "impulse_response has batch 2, x has batch 1 (expected 1 or 1)"),
    (_x(), _h(L=0), KB, "impulse_response needs at least one tap"),
    (_x(n=0), _h(K=1), KB, "x needs at least one sample"),
    (_x(), _h(), 4000, "hop must be a positive multiple of 4096 samples, got 4000"),
    (_x(), _h(), 0, "hop must be a positive multiple of 4096 samples, got 0"),
    (_x(), _h(), -KB, "hop must be a positive multiple of 4096 samples, got -4096"),
    (_x(), _h(), 4096.0, "hop must be an integer number of samples, got 4096.0"),
    (_x(), _h(), True, "hop must be an integer number of samples, got True"),
    (_x(n=8000), _h(K=3), KB, "impulse response 2 is anchored at (K - 1) * hop = 8192, at or after the end of x (8000 "
     "samples)"),
    (_x(n=8192), _h(K=3), KB, "impulse response 2 is anchored at (K - 1) * hop = 8192, at or after the end of x (8192 "
     "samples)"),
]


@pytest.mark.parametrize("x,ir,hop,msg", BAD_CALLS, ids=[c[3][:40] for c in BAD_CALLS])
def test_tv_bus_value_errors(x, ir, hop, msg):
    """every shape and value check raises ValueError with its message before anything reaches the device (these CPU
    tensors would otherwise be rejected as CPU tensors)"""
    import dasp_pytorch_b200 as D
    with pytest.raises(ValueError) as e:
        D.time_varying_convolution_bus(x, SR, ir, hop)
    assert str(e.value) == msg


def test_tv_bus_rejects_cpu_tensors():
    import dasp_pytorch_b200 as D
    from dasp_pytorch_b200._abi import DaspError
    with pytest.raises(DaspError, match="no CPU path"):
        D.time_varying_convolution_bus(_x(), SR, _h(), KB)


def test_tv_bus_is_exported():
    import dasp_pytorch_b200 as D
    assert "time_varying_convolution_bus" in D.functional.__all__
    assert D.time_varying_convolution_bus is D.functional.time_varying_convolution_bus
