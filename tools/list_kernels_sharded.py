"""torchrun --nproc-per-node G tools/list_kernels_sharded.py <out.txt>: every CUDA kernel rank 0 launches during ONE
particle-sharded forward at the bench configuration (1024 particles per rank), from torch.profiler (CUPTI) -- shows that
no collective-library (nccl*) kernel is on the data path: results and feature maps travel by peer stores + flag barriers."""
import collections
import os
import sys

import torch
import torch.distributed as dist
from torch.profiler import ProfilerActivity, profile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pips_b200 import synthetic

rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dev = torch.device("cuda", local)
dist.init_process_group("nccl", device_id=dev)
B, S, H, W, NPER, ITERS = 4, 8, 384, 512, 1024, 6
rgbs = synthetic.smooth_video(B, S, H, W, seed=1234).to(torch.bfloat16).to(dev)
xys = synthetic.random_queries(B, NPER * world, H, W, seed=4321).to(dev)
model = synthetic.seeded_model(stride=8, seed=0).to(dev).eval()
model.shard_particles()
with torch.no_grad():
    for _ in range(3):
        model(xys, rgbs, iters=ITERS)
    torch.cuda.synchronize()
    dist.barrier()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        model(xys, rgbs, iters=ITERS)
        torch.cuda.synchronize()
if rank == 0:
    tot, cnt = collections.Counter(), collections.Counter()
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and e.name and not e.name.startswith("Memcpy") and not e.name.startswith("Memset"):
            name = e.name.replace("(anonymous namespace)::", "").split("(")[0][:90]
            tot[name] += e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
            cnt[name] += 1
    T = sum(tot.values())
    nccl = [k for k in tot if "nccl" in k.lower()]
    lines = [f"# one particle-sharded Pips.forward on {world} H100s (rank 0; cfg 2 sizes, 1024 particles per rank, frame-sharded encoder), torch.profiler / CUPTI",
             f"# {sum(cnt.values())} kernel launches, {T / 1e3:.2f} ms of kernel time; collective-library kernels on the data path: {nccl if nccl else 'none'}"]
    for k, v in tot.most_common():
        lines.append(f"{v / 1e3:9.3f} ms  x{cnt[k]:4d}  {k}")
    text = "\n".join(lines) + "\n"
    open(sys.argv[1] if len(sys.argv) > 1 else "gpurun_out/sharded_kernels.txt", "w").write(text)
    print(text[:3000])
model.close_peer_slabs()
dist.barrier()
dist.destroy_process_group()
