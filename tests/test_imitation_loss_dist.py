"""CPU: the imitation loss's one packed all-reduce (per pair: count / world, count, per-channel
|teacher| sums) gives the reference's normaliser (dist_reduce_mean of the positive count) and its
NormalizeLayer update (all-reduced row count and |x| sums, three collectives) bit for bit over two
gloo ranks, one of which has no positive."""
import socket

import torch

from tests import imitation_loss_oracle as O


def _case(rank):
    g = torch.Generator().manual_seed(40 + rank)
    B, ny, nx, nz = 1, 6, 7, 3
    ts = [torch.relu(torch.randn((B, 8, ny, nx), generator=g)),
          torch.relu(torch.randn((B, 4, nz, ny, nx), generator=g))]
    inbox = torch.rand((B, ny, nx), generator=g) < (0.5 if rank == 0 else 0.0)
    return ts, inbox


def _worker(rank, port, out):
    import torch.distributed as dist
    dist.init_process_group('gloo', init_method=f'tcp://127.0.0.1:{port}', rank=rank,
                            world_size=2)
    ts, inbox = _case(rank)
    scales = [torch.full((1, 8), 0.9), torch.full((1, 4), 1.1)]
    # the reference: dist_reduce_mean(positives.sum().float()), then NormalizeLayer.update
    ref_mean, ref_scale = [], []
    for t, s in zip(ts, scales):
        pos = O.positives(inbox, t)
        n = pos.sum().float().clone()
        dist.all_reduce(n.div_(float(dist.get_world_size())), op=dist.ReduceOp.SUM)
        ref_mean.append(n.item())
        rows = O._rows(t)[pos]
        bsize = torch.tensor(rows.shape[0], dtype=torch.long)
        dist.all_reduce(bsize, op=dist.ReduceOp.SUM)
        new = s.clone()
        if bsize > 10:
            sum_x = torch.sum(rows.abs(), dim=0, keepdim=True)
            dist.all_reduce(sum_x, op=dist.ReduceOp.SUM)
            new *= 0.99
            new += sum_x / torch.clamp(bsize, min=1) * (1 - 0.99)
        ref_scale.append(new)
    # the packed buffer, all-reduced once
    counts = [O.positives(inbox, t).sum() for t in ts]
    sums = [torch.sum(O._rows(t)[O.positives(inbox, t)].abs(), dim=0) for t in ts]
    buf = O.pack(counts, sums, dist.get_world_size())
    dist.all_reduce(buf)
    got = O.unpack(buf, [8, 4])
    out[rank] = dict(
        counts=[int(c) for c in counts],
        mean_equal=[float(m) == r for (m, _, _), r in zip(got, ref_mean)],
        scale_equal=[torch.equal(O.update_scale(s, n, a), r)
                     for s, (_, n, a), r in zip(scales, got, ref_scale)],
        updated=[not torch.equal(r, s) for r, s in zip(ref_scale, scales)])
    dist.destroy_process_group()


def test_packed_all_reduce_gives_the_reference_normaliser_and_update():
    import torch.multiprocessing as mp
    with socket.socket() as s:
        s.bind(('127.0.0.1', 0))
        port = s.getsockname()[1]
    out = mp.Manager().dict()
    mp.spawn(_worker, args=(port, out), nprocs=2, join=True)
    assert out[1]['counts'] == [0, 0] and min(out[0]['counts']) > 10
    for r in (0, 1):
        assert out[r]['mean_equal'] == [True, True]
        assert out[r]['scale_equal'] == [True, True]
        assert out[r]['updated'] == [True, True]
