import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "distributed-join_b200"))
import torch, torch.distributed as dist
import djb200 as dj
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(rank); dev = torch.device("cuda", rank)
dist.init_process_group("nccl", device_id=dev)
comm = dj.Comm.from_torch_distributed()
n = int(os.environ.get("DJ_TRACE_ROWS", 400_000_000)) // world
g = dj.gen_params(n, n, 0.3, 2 * n, True)
(lk, lp), (rk, rp) = dj.generate_tables_distributed(g, rank, world, dev)
cap = int(n * 0.35) + 1_000_000
outs = [torch.empty(cap, dtype=torch.int64, device=dev) for _ in range(4)]
ws = dj.workspace(dj.lib().dj_distributed_inner_join_workspace_bytes(n, n, world, 1), dev)
import time
for i in range(6):
    os.environ["DJ_TRACE"] = "1" if i == 5 else "0"
    t0 = time.time()
    res = dj.distributed_inner_join(comm, lk, lp, rk, rp, capacity=cap, ws=ws, outs=outs)
    if rank == 0:
        print(f"[trace rank 0] call {i}: {1e3 * (time.time() - t0):.3f} ms wall (no barrier between calls)", flush=True)
comm.destroy(); dist.destroy_process_group()
