"""Host (gloo, CPU tensors): the deterministic bucket reduction's gather.  parallel.gather_ranks gives every rank the same
[world, n] stack with rank r's bucket in row r, so the fixed-order sum over rows (teco_sum_ranks_f32 on the device, restated
here) gives every rank the same bits; NCCL's sum promises neither."""
import os
import tempfile

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp


def _worker(rank, world, init, out_dir):
    dist.init_process_group("gloo", init_method=init, rank=rank, world_size=world)
    try:
        from tecogan_b200.parallel import gather_ranks
        rng = np.random.default_rng(100 + rank)
        bucket = torch.from_numpy(rng.standard_normal(1001).astype(np.float32))
        g = gather_ranks(bucket)
        np.save(os.path.join(out_dir, "g%d.npy" % rank), g.numpy())
        np.save(os.path.join(out_dir, "b%d.npy" % rank), bucket.numpy())
    finally:
        dist.destroy_process_group()


def test_gather_ranks_rows_in_rank_order_on_every_rank():
    world = 3
    with tempfile.TemporaryDirectory() as d:
        init = "file://" + os.path.join(d, "init")
        mp.spawn(_worker, args=(world, init, d), nprocs=world, join=True)
        gs = [np.load(os.path.join(d, "g%d.npy" % r)) for r in range(world)]
        bs = [np.load(os.path.join(d, "b%d.npy" % r)) for r in range(world)]
    for g in gs:
        assert g.shape == (world, 1001)
        assert np.array_equal(g.view(np.int32), gs[0].view(np.int32))
        for r in range(world):
            assert np.array_equal(g[r].view(np.int32), bs[r].view(np.int32))
    s = gs[0][0].copy()
    for r in range(1, world):              # the declared order: ((b0 + b1) + b2) in float32
        s = (s + gs[0][r]).astype(np.float32)
    assert s.dtype == np.float32 and np.isfinite(s).all()
