"""Multi-GPU property (SURVEY.md 8e / section 4): items are independent, so a batch sharded over two devices
gives BIT-IDENTICAL per-item results (outputs and gradients) to the unsharded batch on one device.  Skipped on
single-GPU machines; run on a machine with at least two GPUs."""
import pytest
import torch

import oracle
from dasp_pytorch_b200.dist import shard_bounds
from helpers import COMP_RANGES, SR, denorm, eq_ranges

pytestmark = pytest.mark.gpu


def _need2():
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs 2 CUDA devices")


def _run(dev, x, eq, comp, rev, drive, noise, L, taps):
    import dasp_pytorch_b200 as D
    c = lambda t: t.to(dev)
    xx = c(x).requires_grad_(True)
    pe = [c(q).requires_grad_(True) for q in eq]
    y = D.parametric_eq(xx, SR, *pe)
    y = D.compressor(y, SR, *[c(q) for q in comp])
    y = D.noise_shaped_reverberation(y, SR, *[c(q) for q in rev], num_samples=L, num_bandpass_taps=taps, noise=c(noise))
    y = D.distortion(y, SR, c(drive))
    (y * y).sum().backward()
    return y.detach().cpu(), xx.grad.cpu(), torch.stack([q.grad.cpu() for q in pe], 1)


def test_two_device_shards_are_bit_identical():
    _need2()
    torch.manual_seed(0)
    bs, n, L, taps = 6, 9000, 5000, 255
    x = torch.rand(bs, 2, n) * 2 - 1
    eq = denorm(torch.rand(bs, 18), eq_ranges())
    comp = denorm(torch.rand(bs, 6).clamp(min=0.05), COMP_RANGES)
    rev = [torch.rand(bs) for _ in range(25)]
    drive = torch.rand(bs * 2) * 12
    noise = oracle.reverb_noise(bs, L, taps, 3)
    full = _run("cuda:0", x, eq, comp, rev, drive, noise, L, taps)
    parts = []
    for r in range(2):
        lo, hi = shard_bounds(bs, 2, r)
        parts.append(_run(f"cuda:{r}", x[lo:hi], [q[lo:hi] for q in eq], [q[lo:hi] for q in comp],
                          [q[lo:hi] for q in rev], drive[2 * lo:2 * hi], noise[2 * lo:2 * hi], L, taps))
    for i in range(3):
        assert torch.equal(torch.cat([p[i] for p in parts]), full[i]), i


def _nccl_worker(rank, world, port, tmpdir):
    import os
    import torch.distributed as dist
    import dasp_pytorch_b200 as D
    from dasp_pytorch_b200 import dist as ddist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    try:
        bs, n = 7, 6000                                   # uneven shards: 4 + 3
        g = torch.Generator().manual_seed(5)
        x = torch.rand(bs, 2, n, generator=g) * 2 - 1
        p01 = torch.rand(bs, 18, generator=g)
        eq = torch.stack(denorm(p01, eq_ranges()), 1)     # (bs, 18)
        xs = ddist.scatter_batch(x.to(dev) if rank == 0 else None, bs, (2, n), torch.float32, dev)
        ps = ddist.scatter_batch(eq.to(dev) if rank == 0 else None, bs, (18,), torch.float32, dev)
        y = D.parametric_eq(xs, SR, *ps.unbind(1))
        y = D.compressor(y, SR, *[torch.full((xs.shape[0],), v, device=dev) for v in (-20.0, 4.0, 10.0, 50.0, 6.0, 3.0)])
        full = ddist.gather_batch(y, bs)
        if rank == 0:
            ref = D.parametric_eq(x.to(dev), SR, *eq.to(dev).unbind(1))
            ref = D.compressor(ref, SR, *[torch.full((bs,), v, device=dev) for v in (-20.0, 4.0, 10.0, 50.0, 6.0, 3.0)])
            torch.save({"ok": bool(torch.equal(full, ref)), "max": float((full - ref).abs().max())},
                       os.path.join(tmpdir, "result.pt"))
        else:
            assert full is None
    finally:
        dist.destroy_process_group()


def test_nccl_scatter_process_gather_matches_single_device(tmp_path):
    """the edge path of SURVEY 8e over REAL NCCL (two ranks, one GPU each): rank 0 scatters x and the packed parameters
    with one grouped send/recv (uneven shards 4 + 3, no padding), every rank runs eq -> compressor on its shard, rank 0
    gathers; the result must be bit-identical to the unsharded run on one device."""
    _need2()
    import torch.multiprocessing as mp
    mp.spawn(_nccl_worker, args=(2, 29533, str(tmp_path)), nprocs=2, join=True)
    res = torch.load(str(tmp_path / "result.pt"))
    assert res["ok"], res
