"""GPU: the multi-rank distributed join (N = 2, 3, 4) on one GPU, every rank against the CPU oracle.

An in-process rank group (dj_comm_create_local_group) runs the whole N > 1 path -- hello round and
agreed radix plan, the fused destination-major partition, the receive layout and its segment tables,
the copy-engine and fused exchanges, the batch loop, the collective overflow verdict, workspace
regrow and the peer-mapping cache -- with one host thread per rank.  tests/local_group_worker.py
holds the cases; each (exchange flavour, N) runs in a fresh process, because the library reads the
flavour once per process and the group needs CUDA_DEVICE_MAX_CONNECTIONS set before CUDA starts.

Not covered here (test_multi_gpu.py under torchrun on >= 2 GPUs): CUDA IPC mappings across
processes, NVLink and cross-device memory ordering, the NCCL exchange fallback, and the C++ ports.
"""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = os.path.join(ROOT, "tests", "local_group_worker.py")

FLAVOURS = {"default": {}, "exchange-fused": {"DJ_EXCHANGE": "fused"}, "no-fuse": {"DJ_NO_FUSE": "1"}}


@pytest.mark.parametrize("world", [2, 3, 4])
@pytest.mark.parametrize("flavour", list(FLAVOURS))
def test_local_group(dj, flavour, world):
    env = {k: v for k, v in os.environ.items() if k not in ("DJ_EXCHANGE", "DJ_NO_FUSE")}
    # world * (world + 2) streams, each on its own hardware queue (dj_b200.h)
    env.update(PYTHONDONTWRITEBYTECODE="1", CUDA_DEVICE_MAX_CONNECTIONS="32", **FLAVOURS[flavour])
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [WORKER, str(world)]
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=1200)
    failed = [line for line in r.stdout.splitlines() if line.startswith("FAIL")]
    assert r.returncode == 0 and not failed, "\n".join(failed) + "\n" + r.stdout[-3000:] + r.stderr[-3000:]
    assert f"cases passed (W={world}" in r.stdout
