"""The distributed left / full outer join across processes and GPUs (CUDA IPC peer exchange and NCCL),
which the in-process rank group of tests/outer_group_worker.py cannot reach.  Skipped below 2 GPUs.

The pytest case launches this file under torchrun at the visible GPU count.  Each rank generates its
slice with the shared counter-based generator (probe table as left, unique build table as right),
joins at odf 1 and 2, and checks that every row's placing key belongs to it; per class of rows
(sides 3 / 1 / 2) the ranks' counts and summed multiset checksums must equal the CPU oracle's global
outer join.  A second launch runs the same under DJ_EXCHANGE=nccl.
"""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
M64 = (1 << 64) - 1


def _signed(x):
    return x - (1 << 64) if x >= (1 << 63) else x


def main():
    for p in (os.path.join(ROOT, "oracle"), os.path.join(ROOT, "distributed-join_b200"), os.path.join(ROOT, "tests")):
        sys.path.insert(0, p)
    import numpy as np
    import torch
    import torch.distributed as dist

    import djb200 as dj
    import oracle as O
    import outer_oracle as OO

    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", rank)))
    dev = torch.device("cuda", torch.cuda.current_device())
    dist.init_process_group("nccl", device_id=dev)
    comm = dj.Comm.from_torch_distributed()
    failures = 0
    nb, np_ = 1_000_000, 2_000_000
    g_d = dj.gen_params(nb, np_, 0.3, 2 * np_, True)
    g_o = O.gen_params(nb, np_, 0.3, 2 * np_, True)
    (bk, bp), (pk, pp) = dj.generate_tables_distributed(g_d, rank, world, dev)
    ref = None
    if rank == 0:
        tabs = [O.generate_tables_distributed(g_o, r, world) for r in range(world)]
        gl = [np.concatenate([t[1][i] for t in tabs]) for i in range(2)]
        gr = [np.concatenate([t[0][i] for t in tabs]) for i in range(2)]
        ref = {full: OO.outer_join(*gl, *gr, full) for full in (False, True)}
    for kind, full in ((dj.JOIN_LEFT_OUTER, False), (dj.JOIN_FULL_OUTER, True)):
        for odf in (1, 2):
            res = dj.distributed_outer_join(comm, kind, pk, pp, bk, bp, odf=odf)
            cols = [c.contiguous() for c in res.cols]
            stats = []
            if res.n_out:
                place = torch.where(cols[4] == OO.SIDE_RIGHT, cols[2], cols[0]).contiguous()
                ids = dj.partition_ids(place, dj.SEED_NVLINK, world * odf)
                assert bool((ids % world == rank).all()), "a row landed on the wrong rank"
            for s in (OO.BOTH, OO.SIDE_LEFT, OO.SIDE_RIGHT):
                m = cols[4] == s
                n = int(m.sum())
                ck = dj.multiset_checksum4(*[c[m].contiguous() for c in cols[:4]]) if n else (0, 0)
                stats += [n, _signed(ck[0]), _signed(ck[1])]
            t = torch.tensor(stats, dtype=torch.int64, device=dev)
            allt = [torch.zeros_like(t) for _ in range(world)]
            dist.all_gather(allt, t)
            if rank == 0:
                ok = True
                for i, s in enumerate((OO.BOTH, OO.SIDE_LEFT, OO.SIDE_RIGHT)):
                    n = sum(int(x[3 * i]) for x in allt)
                    ck = (sum(int(x[3 * i + 1]) & M64 for x in allt) & M64, sum(int(x[3 * i + 2]) & M64 for x in allt) & M64)
                    want = ref[full][4] == s
                    ok &= n == int(want.sum()) and (n == 0 or ck == O.multiset_checksum4(*[c[want] for c in ref[full][:4]]))
                print(f"case {'full' if full else 'left'} outer odf={odf} exchange={os.environ.get('DJ_EXCHANGE', 'default')}: "
                      f"{'OK' if ok else 'MISMATCH'}", flush=True)
                failures += 0 if ok else 1
    comm.destroy()
    f = torch.tensor([failures], device=dev)
    dist.broadcast(f, 0)
    dist.destroy_process_group()
    if int(f.item()):
        sys.exit(1)
    if rank == 0:
        print("outer join multi-gpu: all cases passed", flush=True)


@pytest.mark.gpu
@pytest.mark.parametrize("exchange", ["default", "nccl"])
def test_outer_join_across_gpus(dj, exchange):
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
         "--master-port", "29533" if exchange == "nccl" else "29532", __file__]
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0 and "all cases passed" in r.stdout, r.stdout[-4000:] + r.stderr[-3000:]


if __name__ == "__main__":
    main()
