"""CPU checks of time_varying_convolution_bus with crossfade="input": its fp64 oracle (tests/tv_bus_input_oracle.py)
against itself, against the static bus oracle and on the emission-time identity, which the output-side oracle does not
satisfy; the geometry query without a GPU (including the benchmark's size); the entry points at bs = 0 and on bad
arguments; and the crossfade values the op rejects before any launch."""
import pytest
import torch

import conv_bus_oracle
import tv_bus_input_oracle
import tv_bus_oracle
from helpers import SR

KB, NFFT = 4096, 8192
ENTRIES = ("dasp_tvbus_in_fwd", "dasp_tvbus_in_shared_fwd", "dasp_tvbus_in_bwd", "dasp_tvbus_in_shared_bwd")


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
def test_tv_bus_input_oracle_methods_agree(S, O, shared):
    gen = torch.Generator().manual_seed(S * 10 + O)
    x, h = _rand(gen, 2, S, 3000), _rand(gen, 1 if shared else 2, 3, S, O, 700)
    a = tv_bus_input_oracle.time_varying_convolution_bus(x, SR, h, 1024, method="fft")
    b = tv_bus_input_oracle.time_varying_convolution_bus(x, SR, h, 1024, method="direct")
    assert a.shape == (2, O, 3000) and _rel(a, b) < 1e-12


@pytest.mark.parametrize("method", ["fft", "direct"])
@pytest.mark.parametrize("S,O", [(3, 2), (2, 1)])
def test_tv_bus_input_oracle_with_one_or_equal_sets_is_the_bus_oracle(method, S, O):
    gen = torch.Generator().manual_seed(3 + S)
    x, h = _rand(gen, 3, S, 2500), _rand(gen, 3, 1, S, O, 900)
    ref = conv_bus_oracle.convolution_bus(x, SR, h[:, 0], method=method)
    got = tv_bus_input_oracle.time_varying_convolution_bus(x, SR, h, 4096, method=method)
    assert _rel(got, ref) < 1e-12
    got = tv_bus_input_oracle.time_varying_convolution_bus(x, SR, h.expand(3, 4, S, O, 900), 600, method=method)
    assert _rel(got, ref) < 1e-12


def test_tv_bus_input_oracle_is_the_sum_of_its_sources():
    gen = torch.Generator().manual_seed(6)
    S = 4
    x, h = _rand(gen, 2, S, 4000), _rand(gen, 2, 3, S, 2, 500)
    y = tv_bus_input_oracle.time_varying_convolution_bus(x, SR, h, 1500)
    parts = sum(tv_bus_input_oracle.time_varying_convolution_bus(x[:, s:s + 1], SR, h[:, :, s:s + 1], 1500,
                                                                 method="direct") for s in range(S))
    assert _rel(y, parts) < 1e-12


def _impulse_case(oracle, L, hop=1000, K=4, n=6000, tau=1300):
    """a unit impulse on source 1 of 2 at tau (interval k = 1, weight a = 0.3): the output from tau on, and the
    emission-time response (1 - a) h_k + a h_k+1 over the same samples"""
    gen = torch.Generator().manual_seed(L)
    x = torch.zeros(1, 2, n, dtype=torch.float64)
    x[0, 1, tau] = 1
    h = _rand(gen, 1, K, 2, 2, L)
    k, a = tau // hop, (tau % hop) / hop
    y = oracle.time_varying_convolution_bus(x, SR, h, hop)
    m = min(L, n - tau)
    want = (1 - a) * h[0, k, 1, :, :m] + a * h[0, k + 1, 1, :, :m]
    return y[0, :, tau:tau + m], want, y[0, :, :tau]


@pytest.mark.parametrize("L", [300, 1000, 2500, 4700])
def test_tv_bus_input_oracle_keeps_the_emission_time_ir_over_the_whole_tail(L):
    """the tail of an impulse emitted between anchors 1 and 2 runs past anchors 2, 3 (L > hop) and keeps its IR"""
    got, want, before = _impulse_case(tv_bus_input_oracle, L)
    assert float(before.abs().max()) < 1e-12
    assert float((got - want).abs().max()) < 1e-12


def test_tv_bus_output_oracle_does_not_keep_the_emission_time_ir_when_L_exceeds_hop():
    """the output-side crossfade weights the tail by the time it is heard: it matches the emission-time response only
    at the emission sample, and past the next anchors it is made of other IR sets"""
    got, want, _ = _impulse_case(tv_bus_oracle, 2500)
    assert float((got[:, 0] - want[:, 0]).abs().max()) < 1e-12
    assert float((got[:, 1000:] - want[:, 1000:]).abs().max()) > 0.1


# (n, L, K, S, O, hop, leff, ir_partitions)
GEOMS = [(480000, 48000, 15, 4, 2, 8 * KB, 48000, 12), (60000, 9000, 5, 3, 1, 3 * KB, 9000, 3),
         (4097, 1, 2, 1, 2, KB, 1, 1), (20001, 30000, 3, 5, 1, KB, 20001, 5), (100, 50, 1, 32, 2, KB, 50, 1),
         (70000, 66000, 15, 2, 1, KB, 66000, 17), (200000, 5000, 4, 7, 2, 3 * KB, 5000, 2)]


def _check_geometry(lib, n, L, K, S, O, hop, leff, J, shared, bs=10, chunk=4):
    """the sizes follow from the design: XW = nX S + (I - nX) ceil(S / 2) window spectra per item (one per source in
    each of the nX = (K - 1) hop / 4096 crossfaded blocks, one per source pair after the last anchor), ceil(K S O / 2)
    partition sets per trajectory set, I product and gradient spectra per item, XW dL/dx spectra; a shared set adds the
    fp64 sum of its dL/dIR spectra to the backward workspace, and there is no dL/dmix region"""
    from dasp_pytorch_b200 import _abi
    I, P, NH, nX = -(-n // KB), (S + 1) // 2, (K * S * O + 1) // 2, (K - 1) * hop // KB
    XW = nX * S + (I - nX) * P
    g = _abi.ConvGeom()
    assert lib.dasp_tvbus_in_geometry(bs, n, L, K, S, O, hop, shared, chunk, g) == 0
    c = g.chunk_items
    assert (g.leff, g.conv_block, g.x_blocks, g.ir_partitions) == (leff, KB, I, J)
    assert c == min(chunk, bs)
    assert g.xspec_c64 == bs * XW * NFFT
    assert g.irspec_c64 == (1 if shared else bs) * NH * J * NFFT
    blk = 8 * NFFT
    fwd = _align(c * I * blk) + _align(c * XW * blk) + _align((1 if shared else c) * NH * J * blk)
    bwd = (_align(c * I * blk) + _align(c * XW * blk) + _align(c * NH * J * blk)
           + (_align(16 * NH * J * NFFT) if shared else 0))
    assert g.fwd_workspace_bytes == fwd and g.bwd_workspace_bytes == bwd
    return g


@pytest.mark.parametrize("n,L,K,S,O,hop,leff,J", GEOMS)
@pytest.mark.parametrize("shared", [0, 1])
def test_tvbus_in_geometry_without_gpu(lib, n, L, K, S, O, hop, leff, J, shared):
    _check_geometry(lib, n, L, K, S, O, hop, leff, J, shared)


def test_tvbus_in_geometry_leaves_the_output_side_sizes_alone(lib):
    """K = 1 (no crossfaded block) keeps ceil(S / 2) windows per block, as the output-side op; the output-side op's
    numbers do not depend on the new entry points"""
    from dasp_pytorch_b200 import _abi
    a, b = _abi.ConvGeom(), _abi.ConvGeom()
    assert lib.dasp_tvbus_in_geometry(6, 50000, 7000, 1, 5, 1, KB, 0, 4, a) == 0
    assert lib.dasp_tvbus_geometry(6, 50000, 7000, 1, 5, 1, KB, 0, 4, b) == 0
    assert (a.xspec_c64, a.irspec_c64, a.fwd_workspace_bytes, a.bwd_workspace_bytes) == \
        (b.xspec_c64, b.irspec_c64, b.fwd_workspace_bytes, b.bwd_workspace_bytes)


def test_tvbus_in_geometry_at_the_benchmark_size(lib):
    """64 x 4 x 480 000, L 48 000, hop 32 768, K 15, stereo bus, in one chunk: 460 window spectra (112 crossfaded
    blocks of 4 sources, 6 later blocks of 2 source pairs) and 720 partition spectra of 64 KiB per item are kept for the
    backward, 1180 in all"""
    for shared in (0, 1):
        g = _check_geometry(lib, 480000, 48000, 15, 4, 2, 8 * KB, 48000, 12, shared, bs=64, chunk=64)
        assert g.xspec_c64 * 8 == 64 * 460 * 64 * 1024
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
def test_tvbus_in_entry_points_reject_bad_arguments_before_any_launch(lib, bs, n, L, K, S, O, hop, msg):
    """every entry point checks S, O, K, hop and lengths before it touches a pointer or the device (all pointers here
    are null, so any launch would fault)"""
    from dasp_pytorch_b200 import _abi
    assert lib.dasp_tvbus_in_geometry(bs, n, L, K, S, O, hop, 0, 4, _abi.ConvGeom()) < 0
    assert msg in lib.dasp_last_error().decode()
    for name in ENTRIES:
        assert getattr(lib, name)(None, None, None, None, None, None, 0, bs, n, L, K, S, O, hop, 4, None) < 0
        assert msg in lib.dasp_last_error().decode()


def test_tvbus_in_entry_points_reject_null_pointers_and_unaligned_rows(lib):
    """with a valid geometry: null pointers, one of the two *_save buffers, n % 4 != 0 and unaligned x / gy rows are
    rejected before any launch (the fake addresses are never dereferenced)"""
    fake, odd = 1 << 20, (1 << 20) + 4
    for f in (lib.dasp_tvbus_in_fwd, lib.dasp_tvbus_in_shared_fwd):
        fwd = lambda x, n=8192, xs=None, irs=None, ir=fake, y=fake: f(x, ir, y, xs, irs, fake, 1 << 40, 2, n, 100, 2,
                                                                       3, 2, KB, 2, None)
        assert fwd(None) < 0 and "null pointer" in lib.dasp_last_error().decode()
        assert fwd(fake, ir=None) < 0 and "null pointer" in lib.dasp_last_error().decode()
        assert fwd(fake, y=None) < 0 and "null pointer" in lib.dasp_last_error().decode()
        assert fwd(fake, xs=fake) < 0 and "both *_save" in lib.dasp_last_error().decode()
        assert fwd(fake, n=8190) < 0 and "n % 4 == 0" in lib.dasp_last_error().decode()
        assert fwd(odd) < 0 and "16-byte aligned" in lib.dasp_last_error().decode()
    for f in (lib.dasp_tvbus_in_bwd, lib.dasp_tvbus_in_shared_bwd):
        bwd = lambda gy, xs=fake, gx=fake, n=8192: f(gy, xs, fake, gx, None, fake, 1 << 40, 2, n, 100, 2, 3, 2, KB, 2,
                                                    None)
        assert bwd(None) < 0 and "null pointer" in lib.dasp_last_error().decode()
        assert bwd(fake, xs=None) < 0 and "null pointer" in lib.dasp_last_error().decode()
        assert bwd(fake, gx=None) < 0 and "null pointer" in lib.dasp_last_error().decode()
        assert bwd(fake, n=8190) < 0 and "n % 4 == 0" in lib.dasp_last_error().decode()
        assert bwd(odd) < 0 and "16-byte aligned" in lib.dasp_last_error().decode()


def test_tvbus_in_batch_zero_is_a_no_op(lib):
    """bs = 0 returns before any pointer is read or any CUDA call is made"""
    from dasp_pytorch_b200 import _abi
    g = _abi.ConvGeom()
    assert lib.dasp_tvbus_in_geometry(0, 8192, 100, 2, 3, 2, KB, 0, 4, g) == 0 and g.xspec_c64 == 0
    for name in ENTRIES:
        assert getattr(lib, name)(None, None, None, None, None, None, 0, 0, 8192, 100, 2, 3, 2, KB, 4, None) == 0


def _x(bs=2, S=3, n=9000):
    return torch.zeros(bs, S, n)


def _h(bs=2, K=2, S=3, O=2, L=10):
    return torch.zeros(bs, K, S, O, L)


@pytest.mark.parametrize("crossfade", ["both", "Input", "", None, 1])
def test_tv_bus_rejects_a_bad_crossfade(crossfade):
    import dasp_pytorch_b200 as D
    with pytest.raises(ValueError) as e:
        D.time_varying_convolution_bus(_x(), SR, _h(), KB, crossfade=crossfade)
    assert str(e.value) == f'crossfade must be "output" or "input", got {crossfade!r}'


@pytest.mark.parametrize("x,ir,hop,msg", [
    (torch.zeros(2, 9000), _h(), KB, "x must be a tensor of shape (batch, inputs, samples)"),
    (_x(S=33), _h(S=33), KB, "time_varying_convolution_bus: 1 to 32 input channels are supported, got 33"),
    (_x(), _h(O=3), KB, "impulse_response: a mono (1) or stereo (2) bus is supported, got 3 outputs"),
    (_x(), _h(bs=3), KB, "impulse_response has batch 3, x has batch 2 (expected 2 or 1)"),
    (_x(), _h(), 4000, "hop must be a positive multiple of 4096 samples, got 4000"),
    (_x(n=8192), _h(K=3), KB, "impulse response 2 is anchored at (K - 1) * hop = 8192, at or after the end of x (8192 "
     "samples)")])
def test_tv_bus_input_value_errors(x, ir, hop, msg):
    """the source-side crossfade runs the same checks with the same messages"""
    import dasp_pytorch_b200 as D
    with pytest.raises(ValueError) as e:
        D.time_varying_convolution_bus(x, SR, ir, hop, crossfade="input")
    assert str(e.value) == msg


def test_tv_bus_input_rejects_cpu_tensors():
    import dasp_pytorch_b200 as D
    from dasp_pytorch_b200._abi import DaspError
    with pytest.raises(DaspError, match="no CPU path"):
        D.time_varying_convolution_bus(_x(), SR, _h(), KB, crossfade="input")


def test_tv_bus_crossfade_is_keyword_only():
    import dasp_pytorch_b200 as D
    with pytest.raises(TypeError):
        D.time_varying_convolution_bus(_x(), SR, _h(), KB, "input")
