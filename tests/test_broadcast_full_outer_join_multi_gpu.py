"""The broadcast full outer join across processes and GPUs (CUDA IPC peer exchange and NCCL), which the
in-process rank group of tests/broadcast_full_outer_group_worker.py cannot reach.  Skipped below 2 GPUs.

The pytest case launches this file under torchrun at the visible GPU count.  Every rank draws every rank's
left and right slices from one seed (right slices of sizes off the 32-row grid), runs the join on both
local-join paths, and compares its rows and opts.bytes_sent with test_broadcast_full_outer_join.restated.
A second launch runs the same under DJ_EXCHANGE=nccl.
"""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def main():
    for p in (os.path.join(ROOT, "oracle"), os.path.join(ROOT, "distributed-join_b200"), os.path.join(ROOT, "tests")):
        sys.path.insert(0, p)
    import numpy as np
    import torch
    import torch.distributed as dist

    import djb200 as dj
    import test_broadcast_full_outer_join as TF

    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", rank)))
    dev = torch.device("cuda", torch.cuda.current_device())
    dist.init_process_group("nccl", device_id=dev)
    comm = dj.Comm.from_torch_distributed()
    failures = 0
    for total_right in (100_000, dj.BROADCAST_TABLE_MAX_ROWS + 1):
        lefts, rights = [], []
        for r in range(world):
            rng = np.random.default_rng([1, r, total_right])
            rk = rng.integers(0, total_right, total_right // world + 7 * r + 5, dtype=np.int64)
            rights.append((rk, TF._ids(rk.size, (r + 1) << 40)))
            lk = rng.integers(0, total_right // 2, 500_000 + 1000 * r, dtype=np.int64)
            lefts.append((lk, TF._ids(lk.size, r << 32)))
        t = [TF._t(a) for a in (*lefts[rank], *rights[rank])]
        sizes = [x[0].size for x in rights]
        at = [sum(sizes[:p]) for p in range(world)]
        words = [((at[p] + sizes[p] + 31) >> 5) - (at[p] >> 5) for p in range(world)]
        ok = True
        try:
            res = dj.distributed_broadcast_full_outer_join(comm, *t)
            TF.assert_full(res.cols, res.n_out, TF.restated(lefts, rights, rank), f"rank {rank}")
            want = (world - 1) * sizes[rank] * 16 + 4 * sum(words[p] for p in range(world) if p != rank)
            ok = res.options.bytes_sent == want
        except AssertionError as e:
            print(f"rank {rank}: {e}", flush=True)
            ok = False
        print(f"rank {rank} R={total_right} exchange={os.environ.get('DJ_EXCHANGE', 'default')}: "
              f"{'OK' if ok else 'MISMATCH'}", flush=True)
        failures += 0 if ok else 1
    comm.destroy()
    f = torch.tensor([failures], device=dev)
    dist.all_reduce(f)
    dist.destroy_process_group()
    if int(f.item()):
        sys.exit(1)
    if rank == 0:
        print("broadcast full outer join multi-gpu: all cases passed", flush=True)


@pytest.mark.gpu
@pytest.mark.parametrize("exchange", ["default", "nccl"])
def test_broadcast_full_outer_join_across_gpus(dj, exchange):
    import torch

    ngpu = torch.cuda.device_count()
    if ngpu < 2:
        pytest.skip("needs at least 2 GPUs")
    env = {k: v for k, v in os.environ.items() if k != "DJ_EXCHANGE"}
    env["PYTHONDONTWRITEBYTECODE"] = "1"
    if exchange == "nccl":
        env["DJ_EXCHANGE"] = "nccl"
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + \
        ["-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={ngpu}", "--master-addr", "127.0.0.1",
         "--master-port", "29537" if exchange == "nccl" else "29536", __file__]
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0 and "all cases passed" in r.stdout, r.stdout[-4000:] + r.stderr[-3000:]


if __name__ == "__main__":
    main()
