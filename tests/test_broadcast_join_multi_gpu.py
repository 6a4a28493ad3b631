"""The broadcast join across processes and GPUs (CUDA IPC peer exchange and NCCL), which the in-process rank
group of tests/broadcast_group_worker.py cannot reach.  Skipped below 2 GPUs.

The pytest case launches this file under torchrun at the visible GPU count.  Every rank draws every rank's
right slice from one seed and its own left slice from its rank, runs each kind on both local-join paths,
and compares its rows with the CPU oracle's join of its own left slice and the concatenated right slices.
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
    import test_broadcast_join as TB

    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", rank)))
    dev = torch.device("cuda", torch.cuda.current_device())
    dist.init_process_group("nccl", device_id=dev)
    comm = dj.Comm.from_torch_distributed()
    failures = 0
    for total_right in (100_000, dj.BROADCAST_TABLE_MAX_ROWS + 1):
        rights = []
        for r in range(world):
            rng = np.random.default_rng([1, r, total_right])
            rk = rng.integers(0, total_right // 2, total_right // world + r, dtype=np.int64)
            rights.append((rk, TB._ids(rk.size, (r + 1) << 40)))
        rng = np.random.default_rng([2, rank])
        lk = rng.integers(0, total_right, 500_000 + 1000 * rank, dtype=np.int64)
        lp = TB._ids(lk.size, rank << 32)
        grk = np.concatenate([x[0] for x in rights])
        grp = np.concatenate([x[1] for x in rights])
        t = [TB._t(a) for a in (lk, lp, *rights[rank])]
        for kind in TB.KINDS:
            ok = True
            try:
                res = dj.distributed_broadcast_join(comm, TB.kind_code(dj, kind), *t)
                TB.assert_join(dj, kind, res.cols, res.n_out, TB.oracle_join(kind, lk, lp, grk, grp))
                row_bytes = 8 if kind in ("semi", "anti") else 16
                ok = res.options.bytes_sent == (world - 1) * rights[rank][0].size * row_bytes
            except AssertionError as e:
                print(f"rank {rank}: {e}", flush=True)
                ok = False
            print(f"rank {rank} case {kind} R={total_right} exchange={os.environ.get('DJ_EXCHANGE', 'default')}: "
                  f"{'OK' if ok else 'MISMATCH'}", flush=True)
            failures += 0 if ok else 1
    comm.destroy()
    f = torch.tensor([failures], device=dev)
    dist.all_reduce(f)
    dist.destroy_process_group()
    if int(f.item()):
        sys.exit(1)
    if rank == 0:
        print("broadcast join multi-gpu: all cases passed", flush=True)


@pytest.mark.gpu
@pytest.mark.parametrize("exchange", ["default", "nccl"])
def test_broadcast_join_across_gpus(dj, exchange):
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
         "--master-port", "29535" if exchange == "nccl" else "29534", __file__]
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0 and "all cases passed" in r.stdout, r.stdout[-4000:] + r.stderr[-3000:]


if __name__ == "__main__":
    main()
