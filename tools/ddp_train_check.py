"""Data-parallel training check over NCCL (launch: python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1
--master-port 29533 tools/ddp_train_check.py).  Each rank runs forward + backward on its half of a global batch; the engine
all-reduces the flat gradient buffer once (mean).  Rank 0 then recomputes the gradients of the FULL batch alone and compares:
the data-parallel gradient must equal the single-process one (GroupNorm is per-sample, the loss is a mean over equal shards).
"""
import json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.distributed as dist
from audio_diffusion_b200.parallel import broadcast_parameters
from audio_diffusion_b200.unet import UNet2DModel

rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ.get("LOCAL_RANK", 0))
torch.cuda.set_device(local)
dev = torch.device("cuda", local)
dist.init_process_group("nccl", device_id=dev)
CFG = dict(in_channels=1, out_channels=1, layers_per_block=2, block_out_channels=(128, 256),
           down_block_types=("DownBlock2D", "AttnDownBlock2D"), up_block_types=("AttnUpBlock2D", "UpBlock2D"))
model = UNet2DModel(sample_size=(32, 32), seed=rank, **CFG).to(dev).train()     # different init per rank on purpose
broadcast_parameters(model.parameters(), src=0)                                  # the one weight broadcast
g = torch.Generator().manual_seed(0)
x = torch.randn(2 * world, 1, 32, 32, generator=g)
tgt = torch.randn(2 * world, 1, 32, 32, generator=g)
t = torch.randint(0, 1000, (2 * world,), generator=g)
sl = slice(2 * rank, 2 * rank + 2)
pred = model(x[sl].to(dev), t[sl].to(dev))["sample"]
torch.nn.functional.mse_loss(pred, tgt[sl].to(dev)).backward()                   # all-reduce happens inside backward
torch.cuda.synchronize()
flat_dp = model._grad_flat.clone()

gathered = [torch.empty_like(flat_dp) for _ in range(world)]
dist.all_gather(gathered, flat_dp)
same = all(torch.equal(gathered[0], gg) for gg in gathered)
dist.barrier()
dist.destroy_process_group()
if rank == 0:
    for p in model.parameters():
        p.grad = None
    pred = model(x.to(dev), t.to(dev))["sample"]                                 # full batch, no process group any more
    torch.nn.functional.mse_loss(pred, tgt.to(dev)).backward()
    ref = model._grad_flat
    rel = ((flat_dp - ref).norm() / ref.norm()).item()
    print(json.dumps({"world": world, "ranks_identical": bool(same), "rel_l2_vs_single_process": rel,
                      "grad_floats": ref.numel()}))
    assert same and rel < 5e-3, (same, rel)
