"""Run under torchrun with >= 2 ranks (one GPU each): the graphed training step of train.GraphedTrainStep with the NCCL all-reduce
of the flat gradient bucket must leave every rank with the same parameters, bit for bit.  Prints one line on rank 0 and exits
non-zero on a mismatch."""
import importlib
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
pkg = importlib.import_module("3dunetcnn_b200")
rank, world, local = pkg.parallel.init_process_group_from_env("nccl")
assert world >= 2, "run with torchrun --nproc-per-node >= 2"
dev = torch.device("cuda", local)
KW = dict(n_features=4, n_outputs=3, base_width=16)
SHAPE, TSHAPE = (2, 4, 64, 64, 64), (2, 3, 64, 64, 64)

torch.manual_seed(0)
model = pkg.UNet3D(precision="bf16", deterministic=True, dropout=0.0, **KW).to(dev)
crit = pkg.DiceLoss(sigmoid=True)
opt = torch.optim.Adam(model.parameters(), lr=1e-3, fused=True)
sync = pkg.parallel.GradAllReduce(model.parameters(), model=model)
sync.broadcast_parameters(0)
step = pkg.train.GraphedTrainStep(model, crit, opt, SHAPE, TSHAPE, grad_sync=sync)
losses = []
for i in range(4):
    g = torch.Generator().manual_seed(1000 * rank + i)          # every rank its own shard
    x = torch.randn(SHAPE, generator=g).to(dev)
    t = (torch.rand(TSHAPE, generator=g) > 0.7).to(torch.uint8).to(dev)
    losses.append(float(step(x, t).item()))
torch.cuda.synchronize()
flat = torch.cat([p.detach().reshape(-1) for p in model.ordered_parameters()])
gathered = [torch.empty_like(flat) for _ in range(world)]
dist.all_gather(gathered, flat)
same = all(torch.equal(gathered[0], g_) for g_ in gathered[1:])
if rank == 0:
    print("ddp_check world=%d: ranks agree bit for bit %s; losses %s" % (world, same, ["%.5f" % v for v in losses]), flush=True)
dist.barrier()
dist.destroy_process_group()
sys.exit(0 if same else 1)
