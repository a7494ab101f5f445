"""The pipelined reverb forward transforms the whole batch's audio windows in one launch on the caller's stream while
chunk 0's IR synthesis runs on a side stream, and each chunk's convolution then transforms only its IR partitions.
Every unit still writes fixed addresses keyed by the absolute item index, so at batch sizes that hit the chunk plan's
edges the pipelined forward agrees bit for bit with the serial one (no saved buffers) and with a single chunk, and so
do the gradients; and at the benchmark's batch a captured step replays the eager one."""
import pytest
import torch

import reverb_pin as rp
from test_gpu_reverb_overlap import _fwd_bwd, _reverb_step

pytestmark = pytest.mark.gpu


# (batch, chunk items): one item; fewer items than one wave of synthesis clusters in one chunk; a last chunk of one
# item; exactly two full chunks
@pytest.mark.parametrize("bs,chunk", [(1, 1), (5, 5), (5, 2), (4, 2), (3, 1)])
def test_windows_first_matches_serial_and_one_chunk(cuda_device, bs, chunk):
    dev = cuda_device
    n, L = rp.default_case(6)
    gen = torch.Generator().manual_seed(900 + 10 * bs + chunk)
    x = (torch.rand(bs, 2, n, generator=gen) * 2 - 1).to(dev)
    params = torch.rand(bs, 25, generator=gen).to(dev)

    used, y1, _, xs1, hs1, gx1, gp1, _ = _fwd_bwd(dev, x, params, L, bs)         # one chunk
    assert used == 2
    used, y, _, xs, hs, gx, gp, g = _fwd_bwd(dev, x, params, L, chunk)
    assert used == 2 and g.chunk_items == chunk
    assert torch.isfinite(xs).all() and torch.isfinite(hs).all()
    assert torch.equal(xs, xs1) and torch.equal(hs, hs1)
    assert torch.equal(y, y1)
    assert torch.equal(gx, gx1) and torch.equal(gp, gp1)
    _, y_serial, *_ = _fwd_bwd(dev, x, params, L, chunk, save=False)
    assert torch.equal(y_serial, y1)


def test_benchmark_batch_captured_matches_eager_and_serial(cuda_device):
    """bench.py's reverb geometry (1024 x 2 x 48000, IR 96000, chunks of two items per SM): a captured forward +
    backward replays the eager one after the same manual_seed, and its output is the serial forward's."""
    import dasp_pytorch_b200 as D
    from helpers import SR
    dev = cuda_device
    bs, n, L, taps = 1024, 48000, 96000, 1023
    gen = torch.Generator().manual_seed(1024)
    x = (torch.rand(bs, 2, n, generator=gen) * 2 - 1).to(dev)
    p = [q.to(dev) for q in torch.rand(25, bs, generator=gen)]

    def step():
        xx = x.detach().requires_grad_(True)
        pp = [q.detach().requires_grad_(True) for q in p]
        y = D.noise_shaped_reverberation(xx, SR, *pp, num_samples=L, num_bandpass_taps=taps)
        grads = torch.autograd.grad(y.square().sum(), [xx, *pp])
        return y.detach(), grads[0], torch.stack(grads[1:], 1)

    torch.manual_seed(5)
    eager = step()
    torch.manual_seed(5)
    with torch.no_grad():                          # no backward: the serial forward
        y_serial = D.noise_shaped_reverberation(x, SR, *p, num_samples=L, num_bandpass_taps=taps)
    assert torch.equal(y_serial, eager[0])

    side = torch.cuda.Stream(dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        step()
    torch.cuda.current_stream(dev).wait_stream(side)
    torch.cuda.synchronize(dev)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = step()
    torch.manual_seed(5)
    graph.replay()
    torch.cuda.synchronize(dev)
    for a, b in zip(out, eager):
        assert torch.isfinite(a).all()
        assert torch.equal(a, b)
