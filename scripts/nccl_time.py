#!/usr/bin/env python3
"""Device time of the library's all-reduce at the sizes the sharded solve uses. Run under torchrun."""
import os
import sys
sys.path.insert(0, ".")
import torch
import torch.distributed as dist
rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device("cuda", local))
from mrcal_b200 import _capi, distributed
distributed.init_comm(rank, world, local)
f = _capi.lib.mrcal_b200_debug_time_allreduce
for count in (8, 4821, 231 * 4096 + 8, 1035 * 4096 + 8):
    ms = f(count, 50)
    if rank == 0:
        print(f"world {world}: all-reduce of {count} doubles ({count * 8 / 1e6:.2f} MB): {ms * 1e3:.1f} us  NCCL_ALGO={os.environ.get('NCCL_ALGO')} NCCL_PROTO={os.environ.get('NCCL_PROTO')}", flush=True)
dist.barrier()
dist.destroy_process_group()
