"""The multi-rank broadcast join on ONE GPU: W ranks of an in-process group, one host thread per rank.

    CUDA_DEVICE_MAX_CONNECTIONS=32 python tests/broadcast_group_worker.py W [case ...]

tests/test_broadcast_join.py runs it in a fresh process per W, as tests/test_outer_join.py runs
outer_group_worker.py, whose group plumbing (local_group_worker.py) this worker shares.  Rank r's result
must equal the oracle's join of rank r's OWN left slice with the concatenation of every rank's right
slice, for every kind, on both local-join paths (the hash table up to DJ_BROADCAST_TABLE_MAX_ROWS gathered
right rows, the radix-partitioned join beyond).
"""
import ctypes as C
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "oracle"), os.path.join(ROOT, "distributed-join_b200"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

import djb200 as dj  # noqa: E402
import local_group_worker as LG  # noqa: E402  (reads W from argv like this worker)
import oracle as O  # noqa: E402
import test_broadcast_join as TB  # noqa: E402
from local_group_worker import RankError, W, run_ranks, split, upload, with_payloads  # noqa: E402

KINDS = TB.KINDS
MAX_ROWS = dj.BROADCAST_TABLE_MAX_ROWS


# ------------------------------------------------------------------------------------------ checks
def expected(tables, kind):
    """Per rank: the oracle's join of its own left slice with every rank's right rows."""
    rk = np.concatenate([t[2] for t in tables])
    rp = np.concatenate([t[3] for t in tables])
    return [TB.oracle_join(kind, t[0], t[1], rk, rp) for t in tables]


def check(tables, kind, results, what=""):
    """results[r]: a JoinResult or (n, cols)."""
    for r, (res, ref) in enumerate(zip(results, expected(tables, kind))):
        n, cols = (res.n_out, res.cols) if isinstance(res, dj.JoinResult) else res
        TB.assert_join(dj, kind, cols, n, ref, f", rank {r}{what}")


def out_columns(kind, cap):
    cols = [torch.empty(cap, dtype=torch.int64, device="cuda") for _ in range(TB.NCOLS[kind] if kind != "left" else 4)]
    return cols + ([torch.empty(cap, dtype=torch.uint8, device="cuda")] if kind == "left" else [])


def raw_join(comm, kind, t, cap, ws, outs):
    """One call of the C entry without the binding's retry loop."""
    cnt, opts = C.c_int64(0), dj.JoinOptions(1, 0)
    L = dj.lib()
    pairs = kind in ("inner", "left")
    ptr = [o.data_ptr() for o in outs] + [None] * (5 - len(outs))
    rc = L.dj_broadcast_join_i64(comm.handle, TB.kind_code(dj, kind), t[0].data_ptr(), t[1].data_ptr(), t[0].numel(),
                                 t[2].data_ptr(), t[3].data_ptr() if pairs else None, t[2].numel(), *ptr, cap,
                                 C.byref(cnt), C.byref(opts), ws.data_ptr(), ws.numel(), dj._stream())
    return rc, cnt.value, opts, (L.dj_last_error().decode() if rc else "")


def ws_bytes(tables, r):
    return dj.lib().dj_broadcast_join_workspace_bytes(len(tables[r][0]), sum(len(t[2]) for t in tables))


def join_ranks(dev, kind):
    """The binding on every rank (both retry loops), allocations before the barrier."""
    def fn(r, comm, sync):
        t = dev[r]
        sync()
        return dj.distributed_broadcast_join(comm, TB.kind_code(dj, kind), *t)
    return run_ranks(fn)


def run_and_check(tables):
    dev = upload(tables)
    for kind in KINDS:
        check(tables, kind, join_ranks(dev, kind), f", {kind}")


def _keys(rng, n, key_range):
    return rng.integers(0, key_range, n, dtype=np.int64)


# ------------------------------------------------------------------------------------------- cases
def case_random(nr_total):
    """Uneven slices with duplicates on both sides; opts.bytes_sent is (W-1) * nright * row bytes."""
    rng = np.random.default_rng([W, nr_total])
    lk, rk = _keys(rng, 400_000 * W, nr_total), _keys(rng, nr_total, nr_total // 2)
    tables = with_payloads(split(lk, rng), split(rk, rng))
    dev = upload(tables)
    for kind in KINDS:
        row_bytes = 8 if kind in ("semi", "anti") else 16

        def fn(r, comm, sync):
            t = dev[r]
            ws = dj.workspace(ws_bytes(tables, r))
            sync()
            return dj.distributed_broadcast_join(comm, TB.kind_code(dj, kind), *t, ws=ws)

        res = run_ranks(fn)
        check(tables, kind, res, f", {kind}")
        for r, x in enumerate(res):
            want = (W - 1) * len(tables[r][2]) * row_bytes
            assert x.options.bytes_sent == want, f"{kind} rank {r}: bytes_sent {x.options.bytes_sent}, expected {want}"


def case_uneven():
    """Rank 0 holds no left rows, the last rank no right rows."""
    rng = np.random.default_rng([W, 2])
    lk, rk = _keys(rng, 300_000, 100_000), _keys(rng, 60_000, 50_000)
    ls, rs = split(lk, rng), split(rk, rng)
    ls[1], ls[0] = np.concatenate([ls[0], ls[1]]), ls[0][:0]
    rs[0], rs[-1] = np.concatenate([rs[0], rs[-1]]), rs[-1][:0]
    run_and_check(with_payloads(ls, rs))


def case_right_table_empty():
    """No right rows anywhere: nothing for inner and semi, every own left row for anti and left outer."""
    rng = np.random.default_rng([W, 3])
    tables = with_payloads(split(_keys(rng, 200_000, 1 << 40), rng), [np.empty(0, np.int64)] * W)
    run_and_check(tables)


def case_left_table_empty():
    """No left rows anywhere: every rank returns 0 rows, but still exchanges and agrees on the verdict."""
    rng = np.random.default_rng([W, 4])
    tables = with_payloads([np.empty(0, np.int64)] * W, split(_keys(rng, 50_000, 1 << 40), rng))
    run_and_check(tables)


def case_hot_key():
    """A right key with 20k copies dealt over every rank, matched by 500 left rows on one rank."""
    rng = np.random.default_rng([W, 5])
    hot = np.int64(0x1234_5678_9ABC)
    rk = rng.permutation(np.concatenate([np.full(20_000, hot), _keys(rng, 30_000, 1 << 40)]))
    ls = split(_keys(rng, 100_000, 1 << 40), rng)
    ls[W - 1] = rng.permutation(np.concatenate([ls[W - 1], np.full(500, hot)]))
    tables = with_payloads(ls, np.array_split(rk, W))
    dev = upload(tables)
    for kind in ("inner", "left"):
        check(tables, kind, join_ranks(dev, kind), f", {kind}")


def case_overflow():
    """Only the rank with the largest result exceeds the capacity (rank 0 holds 20k left rows of a key with
    two right rows): every rank returns DJ_ERR_OVERFLOW with its exact count, and the binding's collective
    retry reproduces the oracle."""
    rng = np.random.default_rng([W, 6])
    hot = np.int64(987_654_321_987)
    ls = split(_keys(rng, 50_000 * W, 400_000), rng)
    ls[0] = np.concatenate([ls[0], np.full(20_000, hot)])
    rk = np.concatenate([[hot, hot], _keys(rng, 40_000, 400_000)])
    tables = with_payloads(ls, split(rk, rng))
    dev = upload(tables)
    for kind in KINDS:
        counts = [e[0].size for e in expected(tables, kind)]
        cap = max(counts) - 1
        assert sum(c > cap for c in counts) == 1, counts

        def fn(r, comm, sync):
            t = dev[r]
            ws = dj.workspace(ws_bytes(tables, r))
            outs = out_columns(kind, cap)
            sync()
            over = raw_join(comm, kind, t, cap, ws, outs)
            sync()
            retried = dj.distributed_broadcast_join(comm, TB.kind_code(dj, kind), *t, capacity=cap, ws=ws)
            return over, retried

        res = run_ranks(fn)
        for r, (over, _) in enumerate(res):
            assert over[0] == dj.ERR_OVERFLOW, f"{kind} rank {r}: rc {over[0]} at capacity {cap}"
            assert over[1] == counts[r], f"{kind} rank {r}: count {over[1]} under overflow, oracle {counts[r]}"
        check(tables, kind, [x[1] for x in res], f", {kind} retried")


def case_workspace_short_on_one_rank():
    """Rank W-1's workspace is one byte short: DJ_ERR_WORKSPACE on every rank, workspace_needed is each
    rank's own need, and a retry at that size succeeds."""
    rng = np.random.default_rng([W, 7])
    tables = with_payloads(split(_keys(rng, 200_000, 100_000), rng), split(_keys(rng, 30_000, 100_000), rng))
    dev = upload(tables)
    for kind in ("inner", "semi"):
        cap = 400_000

        def fn(r, comm, sync):
            t = dev[r]
            q = ws_bytes(tables, r)
            ws = dj.workspace(q - 1 if r == W - 1 else q)
            outs = out_columns(kind, cap)
            sync()
            first = raw_join(comm, kind, t, cap, ws, outs)
            comm.release_workspace()
            ws = dj.workspace(first[2].workspace_needed)
            sync()
            again = raw_join(comm, kind, t, cap, ws, outs)
            return first, again, q, [o[:again[1]].clone() for o in outs]

        res = run_ranks(fn)
        for r, (first, again, q, _) in enumerate(res):
            assert first[0] == dj.ERR_WORKSPACE, f"{kind} rank {r}: rc {first[0]} ({first[3]})"
            assert first[2].workspace_needed == q, f"{kind} rank {r}: needs {first[2].workspace_needed}, query {q}"
            assert again[0] == 0, f"{kind} rank {r}: {again[3]}"
        check(tables, kind, [(x[1][1], x[3]) for x in res], f", {kind} after the regrow")


def case_kind_mismatch():
    """Rank 0 asks for a broadcast semi join while the others ask for a broadcast inner join, then rank 0
    is inside a broadcast join while the others are inside distributed_inner_join: DJ_ERR_ARG on every
    rank, no hang; the group then runs a broadcast inner join normally."""
    rng = np.random.default_rng([W, 8])
    tables = with_payloads(split(_keys(rng, 60_000, 100_000), rng), split(_keys(rng, 40_000, 100_000), rng))
    dev = upload(tables)
    cap = 200_000

    def fn(r, comm, sync):
        t = dev[r]
        size = max(ws_bytes(tables, r), dj.lib().dj_distributed_inner_join_workspace_bytes(60_000, 40_000, W, 1))
        ws = dj.workspace(size)
        outs = out_columns("inner", cap)
        sync()
        kinds = raw_join(comm, "semi" if r == 0 else "inner", t, cap, ws, outs)
        sync()
        if r == 0:
            entries = raw_join(comm, "inner", t, cap, ws, outs)
        else:
            cnt, opts = C.c_int64(0), dj.JoinOptions(1, 0)
            L = dj.lib()
            rc = L.dj_distributed_inner_join_i64(comm.handle, *[x.data_ptr() for x in t[:2]], t[0].numel(),
                                                 *[x.data_ptr() for x in t[2:]], t[2].numel(),
                                                 *[o.data_ptr() for o in outs], cap, C.byref(cnt), C.byref(opts),
                                                 ws.data_ptr(), ws.numel(), dj._stream())
            entries = (rc, cnt.value, opts, L.dj_last_error().decode() if rc else "")
        sync()
        good = raw_join(comm, "inner", t, cap, ws, outs)
        return kinds, entries, good, [o[:good[1]].clone() for o in outs]

    res = run_ranks(fn)
    for r, (kinds, entries, good, _) in enumerate(res):
        assert kinds[0] == dj.ERR_ARG and "kind" in kinds[3], f"rank {r}: rc {kinds[0]} ({kinds[3]})"
        assert entries[0] == dj.ERR_ARG and "kind" in entries[3], f"rank {r}: rc {entries[0]} ({entries[3]})"
        assert good[0] == 0, f"rank {r}: {good[3]}"
    check(tables, "inner", [(x[2][1], x[3]) for x in res], ", after the mismatches")


def case_alternating_entries():
    """Several consecutive calls in one group on the same workspaces, alternating broadcast joins (both
    paths) and repartitioned joins: every result against the oracle."""
    rng = np.random.default_rng([W, 9])
    small = with_payloads(split(_keys(rng, 300_000, 200_000), rng), split(_keys(rng, 50_000, 100_000), rng))
    big = with_payloads(split(_keys(rng, 300_000, 2 * MAX_ROWS), rng), split(_keys(rng, MAX_ROWS + 7, MAX_ROWS), rng))
    dsmall, dbig = upload(small), upload(big)
    gl = [np.concatenate([t[i] for t in small]) for i in range(4)]
    _, ref_inner = O.inner_join(*gl)
    ref_n = ref_inner[0].size

    def fn(r, comm, sync):
        L = dj.lib()
        size = max(ws_bytes(small, r), ws_bytes(big, r),
                   L.dj_distributed_inner_join_workspace_bytes(len(small[r][0]), len(small[r][2]), W, 1) * 2,
                   L.dj_distributed_outer_join_workspace_bytes(len(small[r][0]), len(small[r][2]), W, 1) * 2)
        ws = dj.workspace(size)
        sync()
        out = []
        for step in range(3):
            for kind in KINDS:
                out.append(("b-small", kind, dj.distributed_broadcast_join(comm, TB.kind_code(dj, kind), *dsmall[r], ws=ws)))
            out.append(("inner", None, dj.distributed_inner_join(comm, *dsmall[r], ws=ws)))
            out.append(("b-big", "semi", dj.distributed_broadcast_join(comm, dj.JOIN_LEFT_SEMI, *dbig[r], ws=ws)))
            out.append(("outer", None, dj.distributed_left_outer_join(comm, *dsmall[r], ws=ws)))
            out.append(("b-big", "left", dj.distributed_broadcast_join(comm, dj.JOIN_LEFT_OUTER, *dbig[r], ws=ws)))
        return out

    res = run_ranks(fn)
    exp = {(name, kind): expected(small if name == "b-small" else big, kind)
           for name, kind, _ in res[0] if name.startswith("b-")}
    for r in range(W):
        for name, kind, x in res[r]:
            if name.startswith("b-"):
                TB.assert_join(dj, kind, x.cols, x.n_out, exp[(name, kind)][r], f", rank {r} {name}")
    assert sum(x.n_out for r in range(W) for name, _, x in res[r] if name == "inner") == 3 * ref_n


CASES = {
    "random-hash-table": lambda: case_random(200_000),
    "random-radix": lambda: case_random(MAX_ROWS + 1),
    "uneven-slices": case_uneven,
    "right-table-empty": case_right_table_empty,
    "left-table-empty": case_left_table_empty,
    "hot-key": case_hot_key,
    "overflow-one-rank": case_overflow,
    "workspace-short-on-one-rank": case_workspace_short_on_one_rank,
    "kind-mismatch": case_kind_mismatch,
    "alternating-entries": case_alternating_entries,
}


def main():
    names = sys.argv[2:] or list(CASES)
    torch.cuda.init()
    O.build()
    LG.COMMS = dj.Comm.local_group(W)  # before torch's stream pool: see local_group_worker.py
    LG.STREAMS = [torch.cuda.Stream() for _ in range(W)]
    failed = []
    for name in names:
        t0 = time.time()
        print(f"run  {name}", flush=True)
        try:
            CASES[name]()
            print(f"ok   {name} ({time.time() - t0:.1f} s)", flush=True)
        except RankError as e:
            print(f"FAIL {name}: {e}", flush=True)
            print("a rank thread failed: the remaining cases are skipped", flush=True)
            os._exit(1)
        except Exception as e:  # noqa: BLE001 -- reported per case
            print(f"FAIL {name}: {type(e).__name__}: {e}", flush=True)
            failed.append(name)
    torch.cuda.synchronize()
    for c in LG.COMMS:
        c.destroy()
    print(f"{len(names) - len(failed)} of {len(names)} cases passed (W={W})", flush=True)
    sys.exit(1 if failed else 0)


if __name__ == "__main__":
    main()
