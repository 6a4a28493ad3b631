"""The multi-rank broadcast full outer join on ONE GPU: W ranks of an in-process group, one host thread per rank.

    CUDA_DEVICE_MAX_CONNECTIONS=32 python tests/broadcast_full_outer_group_worker.py W [case ...]

tests/test_broadcast_full_outer_join.py runs it in a fresh process per W on the group plumbing of
local_group_worker.py.  Rank r's result must equal test_broadcast_full_outer_join.restated: the left outer join
of its own left slice with every rank's right slice, then the rows of its own right slice whose key no rank's
left rows hold.  Right slices have sizes and offsets that are not multiples of 32, so every rank's match bits
for a peer's slice start inside a word.
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
import test_broadcast_full_outer_join as TF  # noqa: E402
from local_group_worker import RankError, W, run_ranks, upload, with_payloads  # noqa: E402

MAX_ROWS = dj.BROADCAST_TABLE_MAX_ROWS


# ------------------------------------------------------------------------------------------ checks
def expected(tables):
    lefts = [(t[0], t[1]) for t in tables]
    rights = [(t[2], t[3]) for t in tables]
    return [TF.restated(lefts, rights, r) for r in range(W)]


def check(tables, results, what=""):
    """results[r]: a JoinResult or (n, cols)."""
    for r, (res, ref) in enumerate(zip(results, expected(tables))):
        n, cols = (res.n_out, res.cols) if isinstance(res, dj.JoinResult) else res
        TF.assert_full(cols, n, ref, f"rank {r}{what}")


def bits_words(before, n):
    """32-bit words of the gathered match bitmap that cover rows [before, before + n)."""
    return ((before + n + 31) >> 5) - (before >> 5) if n else 0


def bytes_sent(tables, r):
    """comm.cu's formula: the right slice to every peer, and every peer's words of this rank's bitmap."""
    sizes = [t[2].size for t in tables]
    at = np.concatenate([[0], np.cumsum(sizes)])
    return (W - 1) * sizes[r] * 16 + 4 * sum(bits_words(int(at[p]), sizes[p]) for p in range(W) if p != r)


def out_columns(cap):
    return [torch.empty(cap, dtype=torch.int64, device="cuda") for _ in range(4)] + \
        [torch.empty(cap, dtype=torch.uint8, device="cuda")]


def raw_join(comm, t, cap, ws, outs):
    """One call of the C entry without the binding's retry loop."""
    cnt, opts = C.c_int64(0), dj.JoinOptions(1, 0)
    L = dj.lib()
    rc = L.dj_broadcast_full_outer_join_i64(comm.handle, *[x.data_ptr() for x in t[:2]], t[0].numel(),
                                            *[x.data_ptr() for x in t[2:]], t[2].numel(),
                                            *[o.data_ptr() for o in outs], cap, C.byref(cnt), C.byref(opts),
                                            ws.data_ptr(), ws.numel(), dj._stream())
    return rc, cnt.value, opts, (L.dj_last_error().decode() if rc else "")


def ws_bytes(tables, r):
    return dj.lib().dj_broadcast_full_outer_join_workspace_bytes(len(tables[r][0]), len(tables[r][2]),
                                                                 sum(len(t[2]) for t in tables), W)


def join_ranks(dev, tables, ws=None):
    """The binding on every rank (both retry loops), allocations before the barrier."""
    def fn(r, comm, sync):
        w = ws[r] if ws else dj.workspace(ws_bytes(tables, r))
        sync()
        return dj.distributed_broadcast_full_outer_join(comm, *dev[r], ws=w)
    return run_ranks(fn)


def odd_slices(a, rng, empty=None):
    """`a` dealt into W slices whose sizes and offsets are not multiples of 32; slice `empty` (if given) holds
    no rows, its neighbour takes them."""
    n = a.size
    while True:
        sizes = np.diff(np.concatenate([[0], np.sort(rng.integers(1, n, W - 1)), [n]]))
        if empty is not None:
            sizes[(empty + 1) % W] += sizes[empty]
            sizes[empty] = 0
        offs = np.cumsum(sizes) - sizes
        if all(s % 32 for s in sizes if s) and all(o % 32 for o, s in zip(offs[1:], sizes[1:]) if s):
            return np.split(a, np.cumsum(sizes)[:-1])


# ------------------------------------------------------------------------------------------- cases
def case_uneven(nr_total, empty_right):
    """Right slices of sizes and offsets off the 32-row grid (with `empty_right`, the last rank holds none);
    rank 0 holds no left rows; about half the right keys match; opts.bytes_sent exact."""
    rng = np.random.default_rng([W, nr_total, empty_right])
    lk = rng.integers(0, nr_total, 300_000 * W, dtype=np.int64)
    rk = rng.integers(0, 2 * nr_total, nr_total, dtype=np.int64)
    ls = [lk[:0]] + np.array_split(lk, W - 1)
    rs = odd_slices(rk, rng, empty=W - 1 if empty_right else None)
    tables = with_payloads(ls, rs)
    assert tables[0][0].size == 0 and (tables[-1][2].size == 0) == empty_right
    res = join_ranks(upload(tables), tables)
    check(tables, res)
    for r, x in enumerate(res):
        want = bytes_sent(tables, r)
        assert x.options.bytes_sent == want, f"rank {r}: bytes_sent {x.options.bytes_sent}, expected {want}"


def case_cross_rank():
    """Right keys matched only by ANOTHER rank's left rows (their owners must not emit them), and unmatched
    keys with copies in several ranks' slices (each owner emits its own copies once)."""
    rng = np.random.default_rng([W, 2])
    base = rng.permutation(np.arange(1 << 20, (1 << 20) + 8000, dtype=np.int64))
    other = [base[r * 1000:(r + 1) * 1000] for r in range(W)]  # right keys of rank r, left keys of rank r+1
    shared_lone = base[W * 1000:W * 1000 + 50]
    rs, ls = [], []
    for r in range(W):
        rs.append(rng.permutation(np.concatenate([other[r], shared_lone, rng.integers(0, 1 << 40, 333 + 7 * r)])))
        ls.append(rng.permutation(np.concatenate([other[(r - 1) % W], rng.integers(1 << 41, 1 << 42, 5000)])))
    tables = with_payloads(ls, rs)
    exp = expected(tables)
    for r in range(W):  # the restatement: none of the cross-matched keys emitted, every shared lone copy once
        emitted = exp[r][2][exp[r][4] == dj.SIDE_RIGHT]
        assert not np.isin(other[r], emitted).any() and np.isin(shared_lone, emitted).all()
    check(tables, join_ranks(upload(tables), tables))


def case_overflow():
    """Only rank 0 exceeds the capacity: every rank returns DJ_ERR_OVERFLOW with its exact count, and the
    binding's collective retry reproduces the restatement."""
    rng = np.random.default_rng([W, 6])
    hot = np.int64(987_654_321_987)
    ls = [rng.integers(0, 400_000, 50_000, dtype=np.int64) for _ in range(W)]
    ls[0] = np.concatenate([ls[0], np.full(20_000, hot)])
    rk = np.concatenate([[hot, hot], rng.integers(0, 800_000, 40_000, dtype=np.int64)])
    tables = with_payloads(ls, odd_slices(rk, rng))
    dev = upload(tables)
    counts = [e[0].size for e in expected(tables)]
    cap = max(counts) - 1
    assert sum(c > cap for c in counts) == 1, counts

    def fn(r, comm, sync):
        t = dev[r]
        ws = dj.workspace(ws_bytes(tables, r))
        outs = out_columns(cap)
        sync()
        over = raw_join(comm, t, cap, ws, outs)
        sync()
        retried = dj.distributed_broadcast_full_outer_join(comm, *t, capacity=cap, ws=ws)
        return over, retried

    res = run_ranks(fn)
    for r, (over, _) in enumerate(res):
        assert over[0] == dj.ERR_OVERFLOW, f"rank {r}: rc {over[0]} at capacity {cap}"
        assert over[1] == counts[r], f"rank {r}: count {over[1]} under overflow, restated {counts[r]}"
    check(tables, [x[1] for x in res], ", retried")


def case_workspace_short_on_one_rank():
    """Rank W-1's workspace is one byte short: DJ_ERR_WORKSPACE on every rank, workspace_needed is each
    rank's own need, and a retry at that size succeeds."""
    rng = np.random.default_rng([W, 7])
    rk = rng.integers(0, 100_000, 30_001, dtype=np.int64)
    ls = [rng.integers(0, 100_000, 40_000 + r, dtype=np.int64) for r in range(W)]
    tables = with_payloads(ls, odd_slices(rk, rng))
    dev = upload(tables)
    cap = 400_000

    def fn(r, comm, sync):
        t = dev[r]
        q = ws_bytes(tables, r)
        ws = dj.workspace(q - 1 if r == W - 1 else q)
        outs = out_columns(cap)
        sync()
        first = raw_join(comm, t, cap, ws, outs)
        comm.release_workspace()
        ws = dj.workspace(first[2].workspace_needed)
        sync()
        again = raw_join(comm, t, cap, ws, outs)
        return first, again, q, [o[:again[1]].clone() for o in outs]

    res = run_ranks(fn)
    for r, (first, again, q, _) in enumerate(res):
        assert first[0] == dj.ERR_WORKSPACE, f"rank {r}: rc {first[0]} ({first[3]})"
        assert first[2].workspace_needed == q, f"rank {r}: needs {first[2].workspace_needed}, query {q}"
        assert again[0] == 0, f"rank {r}: {again[3]}"
    check(tables, [(x[1][1], x[3]) for x in res], ", after the regrow")


def case_kind_mismatch():
    """Rank 0 is inside the broadcast full outer join while the others are inside dj_broadcast_join_i64's left
    outer join: DJ_ERR_ARG on every rank, no hang; then the group runs the full outer join normally."""
    rng = np.random.default_rng([W, 8])
    rk = rng.integers(0, 100_000, 40_000, dtype=np.int64)
    ls = [rng.integers(0, 100_000, 15_000, dtype=np.int64) for _ in range(W)]
    tables = with_payloads(ls, odd_slices(rk, rng))
    dev = upload(tables)
    cap = 200_000

    def fn(r, comm, sync):
        t = dev[r]
        size = max(ws_bytes(tables, r), dj.lib().dj_broadcast_join_workspace_bytes(t[0].numel(), rk.size))
        ws = dj.workspace(size)
        outs = out_columns(cap)
        sync()
        if r == 0:
            mixed = raw_join(comm, t, cap, ws, outs)
        else:
            cnt, opts = C.c_int64(0), dj.JoinOptions(1, 0)
            L = dj.lib()
            rc = L.dj_broadcast_join_i64(comm.handle, dj.JOIN_LEFT_OUTER, *[x.data_ptr() for x in t[:2]], t[0].numel(),
                                         *[x.data_ptr() for x in t[2:]], t[2].numel(), *[o.data_ptr() for o in outs],
                                         cap, C.byref(cnt), C.byref(opts), ws.data_ptr(), ws.numel(), dj._stream())
            mixed = (rc, cnt.value, opts, L.dj_last_error().decode() if rc else "")
        sync()
        good = raw_join(comm, t, cap, ws, outs)
        return mixed, good, [o[:good[1]].clone() for o in outs]

    res = run_ranks(fn)
    for r, (mixed, good, _) in enumerate(res):
        assert mixed[0] == dj.ERR_ARG and "kind" in mixed[3], f"rank {r}: rc {mixed[0]} ({mixed[3]})"
        assert good[0] == 0, f"rank {r}: {good[3]}"
    check(tables, [(x[1][1], x[2]) for x in res], ", after the mismatch")


def case_back_to_back():
    """Three calls in a row on the same workspaces with different tables (hash table, radix, hash table): the
    inboxes, the flags and the gathered columns are reused call after call."""
    rng = np.random.default_rng([W, 9])
    sets = []
    for i, nr in enumerate((60_001, MAX_ROWS + 77, 9_999)):
        rk = rng.integers(0, 2 * nr, nr, dtype=np.int64)
        ls = [rng.integers(i * 1000, nr + i * 1000, 100_000 + 13 * r, dtype=np.int64) for r in range(W)]
        sets.append(with_payloads(ls, odd_slices(rk, rng)))
    devs = [upload(t) for t in sets]

    def fn(r, comm, sync):
        ws = dj.workspace(max(ws_bytes(t, r) for t in sets))
        sync()
        return [dj.distributed_broadcast_full_outer_join(comm, *d[r], ws=ws) for d in devs]

    res = run_ranks(fn)
    for i, tables in enumerate(sets):
        check(tables, [x[i] for x in res], f", call {i}")


CASES = {
    "uneven-hash-table": lambda: case_uneven(200_001, False),
    "uneven-radix": lambda: case_uneven(MAX_ROWS + 1, False),
    "empty-right-slice-hash-table": lambda: case_uneven(100_003, True),
    "empty-right-slice-radix": lambda: case_uneven(MAX_ROWS + 5, True),
    "cross-rank-matches": case_cross_rank,
    "overflow-one-rank": case_overflow,
    "workspace-short-on-one-rank": case_workspace_short_on_one_rank,
    "kind-mismatch": case_kind_mismatch,
    "back-to-back": case_back_to_back,
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
