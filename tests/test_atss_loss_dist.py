"""CPU: ``LIGAATSSHead.loss`` all-reduces both of its normalisers (num_total_pos and the sum of the
centerness targets) to their mean over ranks in one call, and the restatement's normalisers are
the reference's reduce_mean of each, over two gloo ranks."""
import socket

import torch

from depth_from_motion_b200 import modules
from tests import atss_loss_oracle as O


def _worker(rank, port, out):
    import torch.distributed as dist
    dist.init_process_group('gloo', init_method=f'tcp://127.0.0.1:{port}', rank=rank,
                            world_size=2)
    norm = torch.tensor([3.0 + 4.0 * rank, 1.5 + 2.0 * rank])
    v = modules._dist_reduce_mean(norm)
    out[rank] = (v.tolist(), norm.tolist(), O.dist_reduce_mean(torch.tensor(2.0 * rank)).item())
    dist.destroy_process_group()


def test_both_normalisers_are_the_mean_over_two_ranks():
    import torch.multiprocessing as mp
    with socket.socket() as s:
        s.bind(('127.0.0.1', 0))
        port = s.getsockname()[1]
    out = mp.Manager().dict()
    mp.spawn(_worker, args=(port, out), nprocs=2, join=True)
    assert out[0][0] == out[1][0] == [5.0, 2.5]
    # the forward's own counts are left as they were
    assert out[0][1] == [3.0, 1.5] and out[1][1] == [7.0, 3.5]
    assert out[0][2] == out[1][2] == 1.0
