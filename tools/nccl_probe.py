"""all-reduce (AVG, fp32) time by payload on this machine.
    python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 tools/nccl_probe.py"""
import os, torch, torch.distributed as dist
lr = int(os.environ["LOCAL_RANK"]); torch.cuda.set_device(lr)
dist.init_process_group("nccl", device_id=torch.device("cuda", lr))
for mb in (0.08, 2.6, 4.0, 21.0, 94.0):
    t = torch.randn(int(mb * 1024 * 1024 / 4), device="cuda")
    for _ in range(5): dist.all_reduce(t, op=dist.ReduceOp.AVG)
    torch.cuda.synchronize(); dist.barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(20): dist.all_reduce(t, op=dist.ReduceOp.AVG)
    e1.record(); torch.cuda.synchronize()
    us = e0.elapsed_time(e1) / 20 * 1e3
    if dist.get_rank() == 0:
        print("all_reduce %6.2f MB: %8.1f us  algbw %6.1f GB/s (world %d)" % (mb, us, mb * 1.048576e6 / us / 1e3, dist.get_world_size()), flush=True)
dist.barrier(); torch.cuda.synchronize(); os._exit(0)
