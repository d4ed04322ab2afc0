"""world_size-2 test of the CUDA trainer itself (``ops.MlpTrainer(process_group=...)``): two processes share cuda:0
and exchange over gloo (NCCL refuses two ranks on one device), each holding a RAGGED shard of the rows; three steps must
reproduce the single-process trainer on the concatenated rows — confidence statistics, loss terms, parameters (2e-5).
The N>1 NCCL path (library-owned communicator) is exercised by bench.py on a multi-GPU node."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, shards, p0, ret):
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.cuda.set_device(0)
    from wild_visual_navigation_b200 import ops

    feat, n_rows, y, yv = (t.cuda() for t in shards[rank])
    tr = ops.MlpTrainer(p0.cuda().clone(), feat.shape[-1], 256, 32, max_rows=feat.shape[0] * feat.shape[1],
                        process_group=dist.group.WORLD)
    metrics = []
    for _ in range(3):
        tr.step_padded(feat, n_rows, y, yv)
        metrics.append(tr.metrics.cpu().clone())
    torch.cuda.synchronize()
    ret[rank] = {"params": tr.params.cpu(), "metrics": metrics, "step": int(tr.step_counter)}
    dist.destroy_process_group()


def test_two_rank_cuda_trainer_equals_single_process():
    from wild_visual_navigation_b200 import ops

    torch.manual_seed(0)
    D, S = 384, 16
    # rank 0: 3 frames with 16 / 5 / 11 live rows, rank 1: 2 frames with 9 / 16 live rows (ragged on purpose)
    n0, n1 = torch.tensor([16, 5, 11], dtype=torch.int32), torch.tensor([9, 16], dtype=torch.int32)
    f0, f1 = torch.randn(3, S, D), torch.randn(2, S, D)

    def labels(n, seed):
        g = torch.Generator().manual_seed(seed)
        yv = torch.rand(n, generator=g) < 0.35
        yv[0] = True
        return torch.where(yv, torch.rand(n, generator=g).clamp(min=0.001), torch.zeros(n)), yv

    y0, yv0 = labels(int(n0.sum()), 1)
    y1, yv1 = labels(int(n1.sum()), 2)
    p0 = torch.randn(ops.lib().wvn_mlp_param_count(D, 256, 32)) * 0.05
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_worker, args=(2, _free_port(), [(f0, n0, y0, yv0), (f1, n1, y1, yv1)], p0, ret), nprocs=2, join=True)

    def rows(f, n):
        return torch.cat([f[g, : int(n[g])] for g in range(f.shape[0])])

    x = torch.cat([rows(f0, n0), rows(f1, n1)]).cuda()
    y, yv = torch.cat([y0, y1]).cuda(), torch.cat([yv0, yv1]).cuda()
    single = ops.MlpTrainer(p0.cuda().clone(), D, 256, 32, max_rows=x.shape[0])
    for s in range(3):
        single.step(x, y, yv)
        m = single.metrics.cpu()
        for r in (0, 1):
            got = ret[r]["metrics"][s]
            assert (got - m).abs().max() <= 2e-5 * max(1.0, m.abs().max().item()), (s, r, got, m)
    for r in (0, 1):
        d = (ret[r]["params"] - single.params.cpu()).norm() / single.params.cpu().norm()
        print(f"rank {r}: param rel diff vs single process {d:.2e}")
        assert d <= 2e-5 and ret[r]["step"] == 3
    assert torch.equal(ret[0]["params"], ret[1]["params"])  # replicas stay bit-identical (same reduced gradient)
