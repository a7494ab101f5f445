"""CPU checks of time_varying_convolution_reverberation: its fp64 oracle (tests/tv_conv_oracle.py) against itself and
against the static oracle, the crossfade weights, the geometry query without a GPU (including the benchmark's size),
the entry points at bs = 0 and on bad arguments, and the shapes, values and devices the op rejects before any launch."""
import pytest
import torch

import conv_oracle
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


@pytest.mark.parametrize("in_chs,ir_chs,shared", [(2, 2, False), (1, 2, True), (2, 1, False), (1, 1, True)])
def test_tv_oracle_methods_agree(in_chs, ir_chs, shared):
    gen = torch.Generator().manual_seed(in_chs * 10 + ir_chs)
    x, h = _rand(gen, 2, in_chs, 3000), _rand(gen, 1 if shared else 2, 3, ir_chs, 700)
    mix = torch.rand(2, generator=gen, dtype=torch.float64)
    a = tv_conv_oracle.time_varying_convolution_reverberation(x, SR, h, 1024, mix, method="fft")
    b = tv_conv_oracle.time_varying_convolution_reverberation(x, SR, h, 1024, mix, method="direct")
    assert a.shape == (2, 2, 3000) and _rel(a, b) < 1e-12


@pytest.mark.parametrize("method", ["fft", "direct"])
def test_tv_oracle_at_one_anchor_is_the_static_oracle(method):
    gen = torch.Generator().manual_seed(3)
    x, h = _rand(gen, 3, 2, 2500), _rand(gen, 3, 1, 2, 900)
    mix = torch.rand(3, generator=gen, dtype=torch.float64)
    got = tv_conv_oracle.time_varying_convolution_reverberation(x, SR, h, 4096, mix, method=method)
    assert _rel(got, conv_oracle.convolution_reverberation(x, SR, h[:, 0], mix, method=method)) < 1e-12


def test_tv_oracle_with_equal_irs_is_the_static_oracle():
    gen = torch.Generator().manual_seed(4)
    x, h = _rand(gen, 2, 1, 5000), _rand(gen, 2, 1, 1, 600)
    mix = torch.rand(2, generator=gen, dtype=torch.float64)
    got = tv_conv_oracle.time_varying_convolution_reverberation(x, SR, h.expand(2, 5, 1, 600), 1000, mix)
    assert _rel(got, conv_oracle.convolution_reverberation(x, SR, h[:, 0], mix)) < 1e-12


@pytest.mark.parametrize("K,hop,n", [(1, 4096, 100), (2, 4096, 4097), (5, 3 * 4096, 60000), (15, 8 * 4096, 480000)])
def test_crossfade_weights_sum_to_one(K, hop, n):
    w = tv_conv_oracle.crossfade_weights(K, hop, n)
    assert torch.allclose(w.sum(0), torch.ones(n, dtype=torch.float64), rtol=0, atol=1e-15)
    assert bool((w >= 0).all())
    for k in range(K):                               # the anchor's own IR alone at its anchor time
        assert float(w[k, k * hop]) == 1.0
    assert bool((w[K - 1, (K - 1) * hop:] == 1).all())


# (n, L, K, ir_chs, hop, leff, ir_partitions)
GEOMS = [(480000, 48000, 15, 2, 8 * KB, 48000, 12), (60000, 9000, 5, 1, 3 * KB, 9000, 3), (4097, 1, 2, 2, KB, 1, 1),
         (20001, 30000, 3, 1, KB, 20001, 5), (100, 50, 1, 2, KB, 50, 1)]


def _check_geometry(lib, n, L, K, C, hop, leff, J, shared, bs=10, chunk=4):
    """the sizes follow from the design: one window spectrum per block (a static convolution's), ceil(K C / 2)
    partition sets per trajectory, and U = I + (K - 1) hop / 4096 product and gradient spectra per item (two for
    every crossfaded block); a shared trajectory adds the fp64 sum of its dL/dIR spectra to the backward workspace"""
    from dasp_pytorch_b200 import _abi
    I, sets = -(-n // KB), (K * C + 1) // 2
    U = I + (K - 1) * hop // KB
    g = _abi.ConvGeom()
    assert lib.dasp_tvconv_geometry(bs, n, L, K, C, hop, shared, chunk, g) == 0
    c = g.chunk_items
    assert (g.leff, g.conv_block, g.x_blocks, g.ir_partitions) == (leff, KB, I, J)
    assert c == min(chunk, bs)
    assert g.xspec_c64 == bs * I * NFFT
    assert g.irspec_c64 == (1 if shared else bs) * sets * J * NFFT
    blk = 8 * NFFT
    fwd = _align(c * U * blk) + _align(c * I * blk) + _align((1 if shared else c) * sets * J * blk)
    bwd = (_align(c * U * blk) + _align(c * I * blk) + _align(c * sets * J * blk) + _align(4 * c * I)
           + (_align(16 * sets * J * NFFT) if shared else 0))
    assert g.fwd_workspace_bytes == fwd and g.bwd_workspace_bytes == bwd
    return g


@pytest.mark.parametrize("n,L,K,C,hop,leff,J", GEOMS)
@pytest.mark.parametrize("shared", [0, 1])
def test_tvconv_geometry_without_gpu(lib, n, L, K, C, hop, leff, J, shared):
    _check_geometry(lib, n, L, K, C, hop, leff, J, shared)


def test_tvconv_geometry_at_the_benchmark_size(lib):
    """256 x 2 x 480 000, L 48 000, hop 32 768, K 15, in one chunk: 118 window spectra and 180 partition spectra
    (15 stereo IRs of 12 partitions) of 64 KiB per item are kept for the backward"""
    for shared in (0, 1):
        g = _check_geometry(lib, 480000, 48000, 15, 2, 8 * KB, 48000, 12, shared, bs=256, chunk=256)
        assert g.xspec_c64 * 8 == 256 * 118 * 64 * 1024
        assert g.irspec_c64 * 8 == (1 if shared else 256) * 180 * 64 * 1024
        assert g.fwd_workspace_bytes < 9 * 2 ** 30 and g.bwd_workspace_bytes < 9 * 2 ** 30


BAD_GEOMS = [  # (bs, n, L, K, C, hop, message)
    (2, 1000, 10, 0, 2, KB, "K >= 1"), (2, 1000, 10, 1, 3, KB, "mono or stereo"), (2, 1000, 10, 1, 4, KB, "mono or"),
    (2, 1000, 10, 1, 2, 0, "multiple of 4096"), (2, 1000, 10, 1, 2, 4000, "multiple of 4096"),
    (2, 1000, 10, 1, 2, -KB, "multiple of 4096"), (2, 4096, 10, 2, 2, KB, "end of x"),
    (2, 40000, 10, 11, 2, KB, "end of x"), (2, 0, 10, 1, 2, KB, "bad shape"), (2, 100, 0, 1, 2, KB, "bad shape"),
    (-1, 100, 10, 1, 2, KB, "bad shape"), (2, 1 << 40, 10, 1 << 40, 2, KB, "end of x")]


@pytest.mark.parametrize("bs,n,L,K,C,hop,msg", BAD_GEOMS)
def test_tvconv_entry_points_reject_bad_arguments_before_any_launch(lib, bs, n, L, K, C, hop, msg):
    """every entry point checks K, hop, channels and lengths before it touches a pointer or the device (all pointers
    here are null, so any launch would fault)"""
    from dasp_pytorch_b200 import _abi
    assert lib.dasp_tvconv_geometry(bs, n, L, K, C, hop, 0, 4, _abi.ConvGeom()) < 0
    assert msg in lib.dasp_last_error().decode()
    for name in ("dasp_tvconv_fwd", "dasp_tvconv_shared_fwd"):
        assert getattr(lib, name)(None, 2, None, C, L, K, hop, None, None, None, None, None, 0, bs, n, 4, None) < 0
        assert msg in lib.dasp_last_error().decode()
    for name in ("dasp_tvconv_bwd", "dasp_tvconv_shared_bwd"):
        assert getattr(lib, name)(None, None, 2, C, L, K, hop, None, None, None, None, None, None, None, 0, bs, n, 4,
                                  None) < 0
        assert msg in lib.dasp_last_error().decode()


def test_tvconv_entry_points_reject_bad_x_channels(lib):
    assert lib.dasp_tvconv_fwd(None, 3, None, 2, 10, 1, KB, None, None, None, None, None, 0, 2, 100, 4, None) < 0
    assert "mono/stereo signals" in lib.dasp_last_error().decode()
    assert lib.dasp_tvconv_bwd(None, None, 0, 2, 10, 1, KB, None, None, None, None, None, None, None, 0, 2, 100, 4,
                               None) < 0
    assert "mono/stereo signals" in lib.dasp_last_error().decode()


def test_tvconv_entry_points_reject_null_pointers_and_unaligned_rows(lib):
    """with a valid geometry: null pointers, one of the two *_save buffers, n % 4 != 0 and unaligned x / gy rows are
    rejected before any launch (the fake addresses are never dereferenced)"""
    fake, odd = 1 << 20, (1 << 20) + 4
    g = dict(bs=2, n=8192, L=100, K=2, C=2, hop=KB)
    fwd = lambda x, n=8192, xs=None, irs=None, mix=fake, y=fake: lib.dasp_tvconv_fwd(
        x, 2, fake, 2, 100, 2, KB, mix, y, xs, irs, fake, 1 << 40, 2, n, 2, None)
    assert fwd(None) < 0 and "null pointer" in lib.dasp_last_error().decode()
    assert fwd(fake, mix=None) < 0 and "null pointer" in lib.dasp_last_error().decode()
    assert fwd(fake, y=None) < 0 and "null pointer" in lib.dasp_last_error().decode()
    assert fwd(fake, xs=fake) < 0 and "both *_save" in lib.dasp_last_error().decode()
    assert fwd(fake, n=8190) < 0 and "n % 4 == 0" in lib.dasp_last_error().decode()
    assert fwd(odd) < 0 and "16-byte aligned" in lib.dasp_last_error().decode()
    bwd = lambda gy, gmix=fake, xs=fake, n=8192: lib.dasp_tvconv_bwd(
        gy, fake, 2, 2, 100, 2, KB, fake, xs, fake, fake, None, gmix, fake, 1 << 40, 2, n, 2, None)
    assert bwd(None) < 0 and "null pointer" in lib.dasp_last_error().decode()
    assert bwd(fake, gmix=None) < 0 and "null pointer" in lib.dasp_last_error().decode()
    assert bwd(fake, xs=None) < 0 and "null pointer" in lib.dasp_last_error().decode()
    assert bwd(fake, n=8190) < 0 and "n % 4 == 0" in lib.dasp_last_error().decode()
    assert bwd(odd) < 0 and "16-byte aligned" in lib.dasp_last_error().decode()


def test_tvconv_batch_zero_is_a_no_op(lib):
    """bs = 0 returns before any pointer is read or any CUDA call is made"""
    from dasp_pytorch_b200 import _abi
    g = _abi.ConvGeom()
    assert lib.dasp_tvconv_geometry(0, 8192, 100, 2, 2, KB, 0, 4, g) == 0 and g.xspec_c64 == 0
    for name in ("dasp_tvconv_fwd", "dasp_tvconv_shared_fwd"):
        assert getattr(lib, name)(None, 2, None, 2, 100, 2, KB, None, None, None, None, None, 0, 0, 8192, 4, None) == 0
    for name in ("dasp_tvconv_bwd", "dasp_tvconv_shared_bwd"):
        assert getattr(lib, name)(None, None, 2, 2, 100, 2, KB, None, None, None, None, None, None, None, 0, 0, 8192, 4,
                                  None) == 0


def _x(bs=2, c=2, n=9000):
    return torch.zeros(bs, c, n)


BAD_CALLS = [  # (x, ir, hop, mix, message)
    (torch.zeros(2, 9000), torch.zeros(2, 2, 2, 10), KB, 0.5, "x must be a tensor of shape (batch, channels, samples)"),
    (_x(c=3), torch.zeros(2, 2, 2, 10), KB, 0.5, "x: only mono/stereo is supported, got 3 channels"),
    (_x(), torch.zeros(2, 2, 10), KB, 0.5, "impulse_response must be a tensor of shape (batch, K, channels, taps)"),
    (_x(), torch.zeros(2, 2, 4, 10), KB, 0.5, "impulse_response: only mono/stereo is supported, got 4 channels"),
    (_x(), torch.zeros(2, 0, 2, 10), KB, 0.5, "impulse_response needs at least one impulse response (K >= 1)"),
    (_x(), torch.zeros(3, 2, 2, 10), KB, 0.5, "impulse_response has batch 3, x has batch 2 (expected 2 or 1)"),
    (_x(bs=1), torch.zeros(2, 2, 2, 10), KB, 0.5, "impulse_response has batch 2, x has batch 1 (expected 1 or 1)"),
    (_x(), torch.zeros(2, 2, 2, 0), KB, 0.5, "impulse_response needs at least one tap"),
    (_x(n=0), torch.zeros(2, 1, 2, 10), KB, 0.5, "x needs at least one sample"),
    (_x(), torch.zeros(2, 2, 2, 10), 4000, 0.5, "hop must be a positive multiple of 4096 samples, got 4000"),
    (_x(), torch.zeros(2, 2, 2, 10), 0, 0.5, "hop must be a positive multiple of 4096 samples, got 0"),
    (_x(), torch.zeros(2, 2, 2, 10), -KB, 0.5, "hop must be a positive multiple of 4096 samples, got -4096"),
    (_x(), torch.zeros(2, 2, 2, 10), 4096.0, 0.5, "hop must be an integer number of samples, got 4096.0"),
    (_x(), torch.zeros(2, 2, 2, 10), True, 0.5, "hop must be an integer number of samples, got True"),
    (_x(n=8000), torch.zeros(2, 3, 2, 10), KB, 0.5,
     "impulse response 2 is anchored at (K - 1) * hop = 8192, at or after the end of x (8000 samples)"),
    (_x(n=8192), torch.zeros(2, 3, 2, 10), KB, 0.5,
     "impulse response 2 is anchored at (K - 1) * hop = 8192, at or after the end of x (8192 samples)"),
    (_x(), torch.zeros(2, 2, 2, 10), KB, torch.zeros(3), "mix: expected 2 element(s) (one per batch item) or 1, got 3"),
]


@pytest.mark.parametrize("x,ir,hop,mix,msg", BAD_CALLS, ids=[c[4][:40] for c in BAD_CALLS])
def test_tv_op_value_errors(x, ir, hop, mix, msg):
    """every shape and value check raises ValueError with its message before anything reaches the device (these CPU
    tensors would otherwise be rejected as CPU tensors)"""
    import dasp_pytorch_b200 as D
    with pytest.raises(ValueError) as e:
        D.time_varying_convolution_reverberation(x, SR, ir, hop, mix)
    assert str(e.value) == msg


def test_tv_op_rejects_cpu_tensors():
    import dasp_pytorch_b200 as D
    from dasp_pytorch_b200._abi import DaspError
    with pytest.raises(DaspError, match="no CPU path"):
        D.time_varying_convolution_reverberation(_x(), SR, torch.zeros(2, 2, 2, 10), KB, 0.5)


def test_tv_partition_constant_is_the_conv_block(lib):
    import dasp_pytorch_b200 as D
    from dasp_pytorch_b200 import _abi
    g = _abi.ConvGeom()
    assert lib.dasp_tvconv_geometry(1, 100, 10, 1, 2, KB, 0, 1, g) == 0
    assert D.CONV_PARTITION_SAMPLES == g.conv_block == KB
