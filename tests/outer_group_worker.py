"""The multi-rank left outer / full outer join on ONE GPU: W ranks of an in-process group, one host
thread per rank, every rank's result against the CPU oracle for both kinds.

    CUDA_DEVICE_MAX_CONNECTIONS=32 python tests/outer_group_worker.py W [case ...]

tests/test_outer_join.py runs it in a fresh process per (exchange flavour, W), as
tests/test_left_filter_join.py runs left_filter_group_worker.py, whose group plumbing this worker
shares.  Rank r's output must equal the oracle's outer join of all ranks' tables restricted to the rows
whose key r owns (partition id % W == r; the right key for a right-only row).  A case that passes the
restated overflows to run_and_check also checks the radix repair counts.
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
import outer_oracle as OO  # noqa: E402
import test_radix_repair as RR  # noqa: E402
from local_group_worker import RankError, W, owner, run_ranks, split, upload, with_payloads  # noqa: E402

KINDS = (("left", dj.JOIN_LEFT_OUTER), ("full", dj.JOIN_FULL_OUTER))


# ------------------------------------------------------------------------------------------ checks
def expected(tables, odf, full):
    """Per rank: the oracle's rows of the global outer join whose placing key rank r owns."""
    gl = [np.concatenate([t[i] for t in tables]) for i in range(4)]
    ref = OO.outer_join(*gl, full)
    own = owner(OO.row_keys(ref), odf)
    return [tuple(c[own == r] for c in ref) for r in range(W)]


def check_rank(r, ref, n, cols, what=""):
    tag = f"rank {r}{what}"
    assert n == ref[0].size, f"{tag}: {n} rows, oracle {ref[0].size}"
    got = [c.cpu().numpy() if hasattr(c, "cpu") else c for c in cols]
    got = got[:4] + [got[4].astype(np.int64)]
    for i, (a, b) in enumerate(zip(O.sort_rows(*got), O.sort_rows(*ref))):
        assert (a == b).all(), f"{tag}: column {i} differs from the oracle"


def check(tables, odf, full, results, what=""):
    """results[r]: a JoinResult or (n, cols)."""
    exp = expected(tables, odf, full)
    for r, res in enumerate(results):
        n, cols = (res.n_out, res.cols) if isinstance(res, dj.JoinResult) else res
        check_rank(r, exp[r], n, cols, what)
    return exp


def out_columns(cap):
    return [torch.empty(cap, dtype=torch.int64, device="cuda") for _ in range(4)] + \
        [torch.empty(cap, dtype=torch.uint8, device="cuda")]


def raw_join(comm, kind, t, odf, cap, ws, outs):
    """One call of the C entry without the binding's retry loop."""
    cnt, opts = C.c_int64(0), dj.JoinOptions(odf, 0)
    L = dj.lib()
    rc = L.dj_distributed_outer_join_i64(comm.handle, kind, *[x.data_ptr() for x in t[:2]], t[0].numel(),
                                         *[x.data_ptr() for x in t[2:]], t[2].numel(), *[o.data_ptr() for o in outs],
                                         cap, C.byref(cnt), C.byref(opts), ws.data_ptr(), ws.numel(), dj._stream())
    return rc, cnt.value, opts, (L.dj_last_error().decode() if rc else "")


def ws_bytes(t, odf):
    return dj.lib().dj_distributed_outer_join_workspace_bytes(t[0].numel(), t[2].numel(), W, odf)


def ws_bytes_global(tables):
    """Room for any rank's receive pieces, however unevenly the slices are dealt."""
    return dj.lib().dj_distributed_outer_join_workspace_bytes(sum(len(t[0]) for t in tables),
                                                              sum(len(t[2]) for t in tables), W, 1)


def first_capacity(t):
    return max(t[0].numel() + t[2].numel(), 1)


def join_ranks(dev, kind, odf=1):
    """The binding on every rank (both retry loops), allocations before the barrier."""
    def fn(r, comm, sync):
        t = dev[r]
        ws = dj.workspace(ws_bytes(t, odf))
        cap = first_capacity(t)
        outs = out_columns(cap)
        sync()
        return dj.distributed_outer_join(comm, kind, *t, odf=odf, capacity=cap, ws=ws, outs=outs)
    return run_ranks(fn)


def overflows(tables, odf):
    """The receivers' children over capacity under the outer join's plan (the filter plan), restated."""
    return RR.receiver_overflows([t[0] for t in tables], [t[2] for t in tables], W, odf, LG.NO_FUSE, True)


def run_and_check(tables, odf=1, over=None):
    """Both kinds against the oracle; the two kinds agree on every row but the right-only ones.  With
    `over` (overflows(tables, odf)), each kind's radix repair counts too."""
    dev = upload(tables)
    got = {}
    for name, kind in KINDS:
        res = join_ranks(dev, kind, odf)
        exp = check(tables, odf, name == "full", res, f", {name}")
        if over is not None:
            calls = 2 if any(e[0].size > max(len(t[0]) + len(t[2]), 1) for e, t in zip(exp, tables)) else 1
            got_r, want = LG.radix_repairs(), RR.expected_repairs(over, calls)
            assert got_r == want, f"radix repairs, {name}: {got_r}, expected {want} from {over}"
        got[name] = res
    for r in range(W):
        right_only = int((got["full"][r].cols[4] == OO.SIDE_RIGHT).sum())
        assert got["left"][r].n_out + right_only == got["full"][r].n_out, f"rank {r}: left + right-only = full"
    return got


# ------------------------------------------------------------------------------------------- cases
def case_generator(odf):
    """The benchmark's generator: the probe table as left, the unique build table as right.  Also
    checks the per-rank oracle restatement against the owner restriction."""
    g = dj.gen_params(500_000, 1_000_000, 0.3, 2_000_000, True)
    tables = []
    for r in range(W):
        (bk, bp), (pk, pp) = dj.generate_tables_distributed(g, r, W)
        tables.append(tuple(x.cpu().numpy() for x in (pk, pp, bk, bp)))
    got = run_and_check(tables, odf)
    for name, full in (("left", False), ("full", True)):
        sim = OO.simulate_distributed_outer_join([t[:2] for t in tables], [t[2:] for t in tables], odf, full)
        for r in range(W):
            check_rank(r, sim[r], got[name][r].n_out, got[name][r].cols, f", {name} vs simulation")


def _random(rng, nl, nr, key_range):
    return rng.integers(0, key_range, nl, dtype=np.int64), rng.integers(0, key_range, nr, dtype=np.int64)


def case_left_slice_empty():
    """The last rank holds no left rows (it still receives its share)."""
    rng = np.random.default_rng([W, 31])
    lk, rk = _random(rng, 300_000, 200_000, 400_000)
    ls, rs = split(lk, rng), split(rk, rng)
    ls[0], ls[-1] = np.concatenate([ls[0], ls[-1]]), ls[-1][:0]
    run_and_check(with_payloads(ls, rs), 2)


def case_right_slice_empty():
    """The last rank holds no right rows (it still receives its share)."""
    rng = np.random.default_rng([W, 32])
    lk, rk = _random(rng, 300_000, 200_000, 400_000)
    ls, rs = split(lk, rng), split(rk, rng)
    rs[0], rs[-1] = np.concatenate([rs[0], rs[-1]]), rs[-1][:0]
    run_and_check(with_payloads(ls, rs), 2)


def case_right_table_empty():
    """No right rows anywhere: every batch is empty on the right, and both kinds append every received
    left row (pieces with gaps between their sources) with a null right side."""
    rng = np.random.default_rng([W, 33])
    lk = rng.integers(0, 1 << 40, 250_000, dtype=np.int64)
    tables = with_payloads(split(lk, rng), [np.empty(0, np.int64)] * W)
    got = run_and_check(tables, 2)
    for name, _ in KINDS:
        assert sum(x.n_out for x in got[name]) == lk.size


def case_left_table_empty():
    """No left rows anywhere: every batch is empty on the left; a full outer join appends every
    received right row with a null left side, a left outer join returns nothing."""
    rng = np.random.default_rng([W, 34])
    rk = rng.integers(0, 1 << 40, 250_000, dtype=np.int64)
    tables = with_payloads([np.empty(0, np.int64)] * W, split(rk, rng))
    got = run_and_check(tables, 2)
    assert sum(x.n_out for x in got["full"]) == rk.size and sum(x.n_out for x in got["left"]) == 0


def case_hot_key():
    """A key with 3000 right copies and 50 left copies dealt over every source lands on one rank
    (150,000 pairs in a bucket of several build jobs)."""
    rng = np.random.default_rng([W, 35])
    hot = np.int64(0x1234_5678_9ABC)
    lk = rng.permutation(np.concatenate([np.full(50, hot), rng.integers(0, 1 << 40, 60_000 * W, dtype=np.int64)]))
    rk = rng.permutation(np.concatenate([np.full(3000, hot), rng.integers(0, 1 << 40, 40_000 * W, dtype=np.int64)]))
    run_and_check(with_payloads(np.array_split(lk, W), np.array_split(rk, W)))


def case_repair_level2_receiver():
    """A two-level plan from the right side's size; one level-2 child of the left rows rank W-1
    receives passes the capacity computed from its level-1 bucket's exact size, with rows from every
    source (left_filter_group_worker.py's case, with right payloads)."""
    rng = np.random.default_rng([W, 44])
    totr, totl = LG.two_level_tot(), 100_000 * W
    b1, b2, sub = RR.dist_radix_plan(totl, totr, W, 1, LG.NO_FUSE, True)
    assert b2 > 0 and sub == (0 if LG.NO_FUSE else b1), (b1, b2, sub)
    j, c = 5, 40
    crowd = LG.crowd_keys(int(2.5 * RR._margin(totl / W / (1 << (b1 + b2)))) + W, W - 1, b1 + b2, (j << b2) | c, rng)
    rf = rng.integers(-(1 << 62), 1 << 62, totr - crowd.size // 4, dtype=np.int64)
    rk = rng.permutation(np.concatenate([rf, crowd[:crowd.size // 4]]))
    lf = np.concatenate([rng.choice(rf, totl // 3), rng.integers(-(1 << 62), 1 << 62, totl - totl // 3, dtype=np.int64)])
    ls = [rng.permutation(np.concatenate([a, b])) for a, b in zip(np.array_split(lf, W), np.array_split(crowd, W))]
    tables = with_payloads(ls, split(rk, rng))
    over = overflows(tables, 1)
    assert over == [(W - 1, 0, 0, 1, j, c)], over
    run_and_check(tables, over=over)


def case_overflow():
    """Only the rank owning a hot left key exceeds the capacity: every rank returns DJ_ERR_OVERFLOW
    with its own exact count, a capacity equal to the largest count fits, and the binding's
    collective retry reproduces the oracle."""
    rng = np.random.default_rng([W, 36])
    hot = np.int64(987_654_321_987)
    lk = rng.permutation(np.concatenate([np.full(20_000, hot), rng.integers(0, 400_000, 100_000, dtype=np.int64)]))
    rk = rng.permutation(np.concatenate([[hot], rng.integers(0, 400_000, 80_000, dtype=np.int64)]))
    tables = with_payloads(split(lk, rng), split(rk, rng))
    dev = upload(tables)
    for name, kind in KINDS:
        exp = expected(tables, 1, name == "full")
        counts = [e[0].size for e in exp]
        top = max(counts)
        cap = top - 1
        over_ranks = [r for r in range(W) if counts[r] > cap]
        assert len(over_ranks) == 1, counts
        size = ws_bytes_global(tables)

        def fn(r, comm, sync):
            t = dev[r]
            ws = dj.workspace(size)
            outs, outs2 = out_columns(top), out_columns(cap)
            sync()
            over = raw_join(comm, kind, t, 1, cap, ws, outs)
            sync()
            exact = raw_join(comm, kind, t, 1, top, ws, outs)
            exact_cols = [o[:exact[1]].clone() for o in outs]
            sync()
            retried = dj.distributed_outer_join(comm, kind, *t, capacity=cap, ws=ws, outs=outs2)
            return over, exact, exact_cols, retried

        res = run_ranks(fn)
        for r, (over, exact, _, _) in enumerate(res):
            assert over[0] == dj.ERR_OVERFLOW, f"{name} rank {r}: rc {over[0]} at capacity {cap}"
            assert over[1] == counts[r], f"{name} rank {r}: count {over[1]} under overflow, oracle {counts[r]}"
            assert exact[0] == 0, f"{name} rank {r}: {exact[3]}"
        check(tables, 1, name == "full", [(x[1][1], x[2]) for x in res], f", {name} exact")
        check(tables, 1, name == "full", [x[3] for x in res], f", {name} retried")


def case_workspace_regrow():
    """Rank 0 holds both tables: every rank returns DJ_ERR_WORKSPACE, and a retry on a workspace of
    exactly the reported size succeeds."""
    rng = np.random.default_rng(37)
    lk = [rng.integers(0, 600_000, 300_000, dtype=np.int64)] + [np.empty(0, np.int64)] * (W - 1)
    rk = [rng.integers(0, 600_000, 400_000, dtype=np.int64)] + [np.empty(0, np.int64)] * (W - 1)
    tables = with_payloads(lk, rk)
    dev = upload(tables)
    for name, kind in KINDS:
        caps = [max(e[0].size, 1) for e in expected(tables, 1, name == "full")]

        def fn(r, comm, sync):
            t = dev[r]
            ws = dj.workspace(ws_bytes(t, 1))
            outs = out_columns(caps[r])
            sync()
            first = raw_join(comm, kind, t, 1, caps[r], ws, outs)
            comm.release_workspace()
            ws = dj.workspace(max(ws.numel(), first[2].workspace_needed))
            sync()
            again = raw_join(comm, kind, t, 1, caps[r], ws, outs)
            cols = [o[:again[1]].clone() for o in outs]
            return first, again, cols

        res = run_ranks(fn)
        assert all(x[0][0] == dj.ERR_WORKSPACE for x in res), [x[0][0] for x in res]
        for r, x in enumerate(res):
            assert x[1][0] == 0, f"{name} rank {r}: retry on the reported size failed: {x[1][3]}"
        check(tables, 1, name == "full", [(x[1][1], x[2]) for x in res], f", {name} reported size")


def case_kind_mismatch():
    """Rank 0 asks for a left outer join, the others for an inner join: DJ_ERR_ARG on every rank, no
    hang; the group then runs a full outer join normally."""
    rng = np.random.default_rng([W, 38])
    lk, rk = _random(rng, 50_000, 40_000, 100_000)
    tables = with_payloads(split(lk, rng), split(rk, rng))
    dev = upload(tables)
    cap = lk.size + rk.size

    def fn(r, comm, sync):
        t = dev[r]
        ws = dj.workspace(ws_bytes_global(tables))
        outs = out_columns(cap)
        sync()
        if r == 0:
            bad = raw_join(comm, dj.JOIN_LEFT_OUTER, t, 1, cap, ws, outs)
        else:
            cnt, opts = C.c_int64(0), dj.JoinOptions(1, 0)
            L = dj.lib()
            rc = L.dj_distributed_inner_join_i64(comm.handle, *[x.data_ptr() for x in t[:2]], t[0].numel(),
                                                 *[x.data_ptr() for x in t[2:]], t[2].numel(),
                                                 *[o.data_ptr() for o in outs[:4]], cap, C.byref(cnt), C.byref(opts),
                                                 ws.data_ptr(), ws.numel(), dj._stream())
            bad = (rc, cnt.value, opts, L.dj_last_error().decode() if rc else "")
        sync()
        good = raw_join(comm, dj.JOIN_FULL_OUTER, t, 1, cap, ws, outs)
        return bad, good, [o[:good[1]].clone() for o in outs]

    res = run_ranks(fn)
    for r, (bad, good, _) in enumerate(res):
        assert bad[0] == dj.ERR_ARG and "kind" in bad[3], f"rank {r}: rc {bad[0]} ({bad[3]})"
        assert good[0] == 0, f"rank {r}: {good[3]}"
    check(tables, 1, True, [(x[1][1], x[2]) for x in res], ", after the mismatch")


CASES = {
    "generator-odf1": lambda: case_generator(1),
    "generator-odf2": lambda: case_generator(2),
    "left-slice-empty": case_left_slice_empty,
    "right-slice-empty": case_right_slice_empty,
    "right-table-empty": case_right_table_empty,
    "left-table-empty": case_left_table_empty,
    "hot-key": case_hot_key,
    "repair-level2-receiver": case_repair_level2_receiver,
    "overflow-one-rank": case_overflow,
    "workspace-regrow": case_workspace_regrow,
    "kind-mismatch": case_kind_mismatch,
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
            LG.radix_repairs()  # reset: every case counts its own repairs
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
    print(f"{len(names) - len(failed)} of {len(names)} cases passed (W={W}, "
          f"flavour {'fused' if LG.FUSED else 'no-fuse' if LG.NO_FUSE else 'default'})", flush=True)
    sys.exit(1 if failed else 0)


if __name__ == "__main__":
    main()
