"""N > 1 host logic on CPU: world_size-2 gloo processes exercise the gradient all-reduce and the batch sharding
that bench.py / training use on NCCL."""
import importlib
import os
import sys

import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    par = importlib.import_module("3dunetcnn_b200").parallel
    r, w, _ = par.init_process_group_from_env("gloo")
    assert (r, w) == (rank, world)
    torch.manual_seed(rank)
    params = [torch.nn.Parameter(torch.randn(5, 3)), torch.nn.Parameter(torch.randn(7)), torch.nn.Parameter(torch.randn(2, 2))]
    params[2].requires_grad_(False)
    sync = par.GradAllReduce(params)
    sync.broadcast_parameters(0)
    for p in params[:2]:
        p.grad = torch.full_like(p, float(rank + 1))
    sync()
    # flat-gradient mode: the gradients are views of one persistent bucket which is all-reduced in place (no copies)
    class Bucketed:
        def __init__(self, ps):
            self.bucket = torch.zeros(sum(p.numel() for p in ps))
            off = 0
            for p in ps:
                p.grad = self.bucket[off:off + p.numel()].view_as(p)
                off += p.numel()

        def flat_gradient_bucket(self):
            return self.bucket
    qs = [torch.nn.Parameter(torch.zeros(4, 2)), torch.nn.Parameter(torch.zeros(3))]
    model = Bucketed(qs)
    model.bucket.fill_(float(10 * (rank + 1)))
    ptrs = [q_.grad.data_ptr() for q_ in qs]
    sync2 = par.GradAllReduce(qs, model=model)
    sync2()
    assert [q_.grad.data_ptr() for q_ in qs] == ptrs and sync2.flat is None      # reduced in place, no staging buffer
    out = {"p0": params[0].detach().clone(), "g0": params[0].grad.clone(), "g1": params[1].grad.clone(),
           "shard": list(par.shard_batch(7, rank, world)), "bucket": model.bucket.clone()}
    q.put((rank, out))
    dist.barrier()
    dist.destroy_process_group()


def test_grad_allreduce_in_place_and_sharding_world2():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + os.getpid() % 2000
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=120) for _ in range(2))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert torch.equal(res[0]["p0"], res[1]["p0"])                       # broadcast from rank 0
    for r in (0, 1):
        assert torch.allclose(res[r]["g0"], torch.full((5, 3), 1.5))      # mean of 1 and 2
        assert torch.allclose(res[r]["g1"], torch.full((7,), 1.5))
    assert res[0]["shard"] == [0, 1, 2, 3] and res[1]["shard"] == [4, 5, 6]
    for r in (0, 1):
        assert torch.allclose(res[r]["bucket"], torch.full((11,), 15.0))  # mean of 10 and 20, in the bucket itself


def test_single_process_is_a_noop():
    par = importlib.import_module("3dunetcnn_b200").parallel
    p = torch.nn.Parameter(torch.ones(3))
    p.grad = torch.ones(3) * 2
    par.GradAllReduce([p])()
    assert torch.equal(p.grad, torch.ones(3) * 2)
    assert list(par.shard_batch(5, 0, 1)) == [0, 1, 2, 3, 4]
