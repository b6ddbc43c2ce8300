"""world_size-2 gloo test (CPU) of the BatchNorm buffer exchange of data-parallel Conformer training: every rank takes the
first rank's running statistics, as the reference's DistributedDataParallel broadcasts its buffers."""
import os

import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from opentransformer_b200 import dp
from tests.test_dp_gloo import _free_port


def _worker(rank, world, port, q):
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    mean = torch.full((4,), float(rank + 1))
    count = torch.tensor(10 * (rank + 1), dtype=torch.int64)
    dp.broadcast_from_first_([mean, count])
    q.put((rank, mean.tolist(), int(count)))
    dist.destroy_process_group()


def test_buffers_follow_the_first_rank():
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = _free_port()
    ps = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in ps:
        p.start()
    res = sorted(q.get(timeout=120) for _ in range(2))
    for p in ps:
        p.join(timeout=60)
    assert res == [(0, [1.0] * 4, 10), (1, [1.0] * 4, 10)]


def test_no_process_group_is_a_no_op():
    t = torch.ones(3)
    dp.broadcast_from_first_([t])
    assert torch.equal(t, torch.ones(3))
