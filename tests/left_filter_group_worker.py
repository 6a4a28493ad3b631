"""The multi-rank left semi / left anti join on ONE GPU: W ranks of an in-process group, one host
thread per rank, every rank's result against the CPU oracle for both kinds.

    CUDA_DEVICE_MAX_CONNECTIONS=32 python tests/left_filter_group_worker.py W [case ...]

tests/test_left_filter_join.py runs it in a fresh process per (exchange flavour, W), as
tests/test_local_group.py runs local_group_worker.py, whose group plumbing (rank threads, streams,
table helpers) this worker reuses.  Rank r's output must equal the oracle's semi (anti) join of all
ranks' tables restricted to the left keys r owns (partition id % W == r).  A case that passes the
restated overflows to run_and_check also checks the radix repair counts, as local_group_worker.py
does.
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
import filter_oracle as FO  # noqa: E402
import local_group_worker as LG  # noqa: E402  (reads W from argv like this worker)
import oracle as O  # noqa: E402
import test_radix_repair as RR  # noqa: E402
from local_group_worker import RankError, W, owner, run_ranks, split, upload  # noqa: E402

KINDS = (("semi", dj.JOIN_LEFT_SEMI), ("anti", dj.JOIN_LEFT_ANTI))


# ------------------------------------------------------------------------------------------ tables
def with_payloads(lkeys, rkeys):
    """Per-rank (lk, lp, rk): left payloads mix64((rank << 36) + row), unique over all ranks."""
    return [(np.ascontiguousarray(lk, np.int64), LG.K.mix64((r << 36) + np.arange(len(lk), dtype=np.int64)),
             np.ascontiguousarray(rk, np.int64)) for r, (lk, rk) in enumerate(zip(lkeys, rkeys))]


def expected(tables, odf, anti):
    """Per rank: the oracle's rows of the global semi (anti) join whose key rank r owns."""
    lk = np.concatenate([t[0] for t in tables])
    lp = np.concatenate([t[1] for t in tables])
    rk = np.concatenate([t[2] for t in tables])
    ref = FO.left_semi_join(lk, lp, rk, anti)
    own = owner(ref[0], odf)
    return [(ref[0][own == r], ref[1][own == r]) for r in range(W)]


def check_rank(r, ref, n, cols, what=""):
    tag = f"rank {r}{what}"
    assert n == ref[0].size, f"{tag}: {n} rows, oracle {ref[0].size}"
    got = [c.cpu().numpy() if hasattr(c, "cpu") else c for c in cols]
    for i, (a, b) in enumerate(zip(O.sort_rows(*got), O.sort_rows(*ref))):
        assert (a == b).all(), f"{tag}: column {i} differs from the oracle"


def check(tables, odf, anti, results, what=""):
    """results[r]: a JoinResult or (n, cols)."""
    exp = expected(tables, odf, anti)
    for r, res in enumerate(results):
        n, cols = (res.n_out, res.cols) if isinstance(res, dj.JoinResult) else res
        check_rank(r, exp[r], n, cols, what)
    return exp


def raw_join(comm, kind, t, odf, cap, ws, outs):
    """One call of the C entry without the binding's retry loop."""
    cnt, opts = C.c_int64(0), dj.JoinOptions(odf, 0)
    L = dj.lib()
    rc = L.dj_distributed_left_filter_join_i64(comm.handle, kind, t[0].data_ptr(), t[1].data_ptr(), t[0].numel(),
                                               t[2].data_ptr(), t[2].numel(), outs[0].data_ptr(), outs[1].data_ptr(),
                                               cap, C.byref(cnt), C.byref(opts), ws.data_ptr(), ws.numel(), dj._stream())
    return rc, cnt.value, opts, (L.dj_last_error().decode() if rc else "")


def ws_bytes(t, odf):
    return dj.lib().dj_distributed_left_filter_join_workspace_bytes(t[0].numel(), t[2].numel(), W, odf)


def ws_bytes_global(tables):
    """Room for any rank's receive pieces, however unevenly the slices are dealt."""
    return dj.lib().dj_distributed_left_filter_join_workspace_bytes(sum(len(t[0]) for t in tables),
                                                                    sum(len(t[2]) for t in tables), W, 1)


def join_ranks(dev, kind, odf=1):
    """The binding on every rank (both retry loops), allocations before the barrier."""
    def fn(r, comm, sync):
        lk, lp, rk = dev[r]
        ws = dj.workspace(ws_bytes(dev[r], odf))
        cap = max(lk.numel(), 1)
        outs = [torch.empty(cap, dtype=torch.int64, device="cuda") for _ in range(2)]
        sync()
        return dj.distributed_left_filter_join(comm, kind, lk, lp, rk, odf=odf, capacity=cap, ws=ws, outs=outs)
    return run_ranks(fn)


def assert_repairs(tables, exp, over, what):
    """dj_testing_radix_repairs after one binding call per rank, against the restatement's children
    over capacity `over` (receiver_overflows)."""
    calls = 2 if any(e[0].size > max(t[0].size, 1) for e, t in zip(exp, tables)) else 1
    got, want = LG.radix_repairs(), RR.expected_repairs(over, calls)
    assert got == want, f"radix repairs{what}: {got}, expected {want} from {over}"


def overflows(tables, odf):
    """The receivers' children over capacity under the filter join's plan, restated."""
    return RR.receiver_overflows([t[0] for t in tables], [t[2] for t in tables], W, odf, LG.NO_FUSE, True)


def run_and_check(tables, odf=1, over=None):
    """Both kinds; per rank, semi and anti together are the left rows it owns.  With `over`
    (overflows(tables, odf)), each kind's radix repair counts too."""
    dev = upload(tables)
    got = {}
    for name, kind in KINDS:
        res = join_ranks(dev, kind, odf)
        exp = check(tables, odf, name == "anti", res, f", {name}")
        if over is not None:
            assert_repairs(tables, exp, over, f", {name}")
        got[name] = res
    own = owner(np.concatenate([t[0] for t in tables]), odf)
    for r in range(W):
        assert got["semi"][r].n_out + got["anti"][r].n_out == (own == r).sum(), f"rank {r}: semi + anti"
    return got


# ------------------------------------------------------------------------------------------- cases
def case_generator(odf):
    """The benchmark's generator: the probe table as left, the unique build table's keys as right.
    Also checks the per-rank oracle restatement against the owner restriction."""
    g = dj.gen_params(500_000, 1_000_000, 0.3, 2_000_000, True)
    tables = []
    for r in range(W):
        (bk, _), (pk, pp) = dj.generate_tables_distributed(g, r, W)
        tables.append((pk.cpu().numpy(), pp.cpu().numpy(), bk.cpu().numpy()))
    got = run_and_check(tables, odf)
    for name, anti in (("semi", False), ("anti", True)):
        sim = FO.simulate_distributed_left_semi_join([t[:2] for t in tables], [t[2] for t in tables], odf, anti)
        for r in range(W):
            check_rank(r, sim[r], got[name][r].n_out, got[name][r].cols, f", {name} vs simulation")


def case_right_slice_empty():
    """The last rank holds no right rows (it still receives its share)."""
    rng = np.random.default_rng([W, 21])
    lk = rng.integers(0, 400_000, 300_000, dtype=np.int64)
    rk = rng.integers(0, 400_000, 200_000, dtype=np.int64)
    ls, rs = split(lk, rng), split(rk, rng)
    rs[0], rs[-1] = np.concatenate([rs[0], rs[-1]]), rs[-1][:0]
    run_and_check(with_payloads(ls, rs), 2)


def case_right_table_empty():
    """No right rows anywhere: semi keeps nothing, anti every left row (received pieces with gaps)."""
    rng = np.random.default_rng([W, 22])
    lk = rng.integers(0, 1 << 40, 250_000, dtype=np.int64)
    tables = with_payloads(split(lk, rng), [np.empty(0, np.int64)] * W)
    got = run_and_check(tables, 2)
    assert sum(x.n_out for x in got["anti"]) == lk.size and sum(x.n_out for x in got["semi"]) == 0


def case_hot_key():
    """A key with 3000 right copies and 5000 left copies dealt over every source lands on one rank."""
    rng = np.random.default_rng([W, 23])
    hot = np.int64(0x1234_5678_9ABC)
    lk = rng.permutation(np.concatenate([np.full(5000, hot), rng.integers(0, 1 << 40, 60_000 * W, dtype=np.int64)]))
    rk = rng.permutation(np.concatenate([np.full(3000, hot), rng.integers(0, 1 << 40, 40_000 * W, dtype=np.int64)]))
    run_and_check(with_payloads(np.array_split(lk, W), np.array_split(rk, W)))


def case_repair_level2_receiver():
    """A two-level plan from the right side's size; one level-2 child of the left rows rank W-1
    receives passes the capacity computed from its level-1 bucket's exact size, with rows from every
    source.  Level 1 fused, the repair re-scatters a parent of W segments; under DJ_NO_FUSE=1 the
    receiver's level 1 stays clean.  (0, 1) for each kind; the filter bits of the repaired left
    side are indexed by its repaired layout."""
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
    rng = np.random.default_rng([W, 24])
    hot = np.int64(987_654_321_987)
    lk = rng.permutation(np.concatenate([np.full(20_000, hot), rng.integers(0, 400_000, 100_000, dtype=np.int64)]))
    rk = rng.permutation(np.concatenate([[hot], rng.integers(0, 400_000, 80_000, dtype=np.int64)]))
    tables = with_payloads(split(lk, rng), split(rk, rng))
    dev = upload(tables)
    for name, kind in KINDS:
        exp = expected(tables, 1, name == "anti")
        counts = [e[0].size for e in exp]
        top = max(counts)
        cap = top - 1
        over_ranks = [r for r in range(W) if counts[r] > cap]
        assert len(over_ranks) == 1, counts
        size = ws_bytes_global(tables)

        def fn(r, comm, sync):
            t = dev[r]
            ws = dj.workspace(size)
            outs = [torch.empty(top, dtype=torch.int64, device="cuda") for _ in range(2)]
            outs2 = [torch.empty(cap, dtype=torch.int64, device="cuda") for _ in range(2)]
            sync()
            over = raw_join(comm, kind, t, 1, cap, ws, outs)
            sync()
            exact = raw_join(comm, kind, t, 1, top, ws, outs)
            exact_cols = [o[:exact[1]].clone() for o in outs]
            sync()
            retried = dj.distributed_left_filter_join(comm, kind, *t, capacity=cap, ws=ws, outs=outs2)
            return over, exact, exact_cols, retried

        res = run_ranks(fn)
        for r, (over, exact, _, _) in enumerate(res):
            assert over[0] == dj.ERR_OVERFLOW, f"{name} rank {r}: rc {over[0]} at capacity {cap}"
            assert over[1] == counts[r], f"{name} rank {r}: count {over[1]} under overflow, oracle {counts[r]}"
            assert exact[0] == 0, f"{name} rank {r}: {exact[3]}"
        check(tables, 1, name == "anti", [(x[1][1], x[2]) for x in res], f", {name} exact")
        check(tables, 1, name == "anti", [x[3] for x in res], f", {name} retried")


def case_workspace_regrow():
    """Rank 0 holds both tables: every rank returns DJ_ERR_WORKSPACE, and a retry on a workspace of
    exactly the reported size succeeds."""
    rng = np.random.default_rng(25)
    lk = [rng.integers(0, 600_000, 300_000, dtype=np.int64)] + [np.empty(0, np.int64)] * (W - 1)
    rk = [rng.integers(0, 600_000, 400_000, dtype=np.int64)] + [np.empty(0, np.int64)] * (W - 1)
    tables = with_payloads(lk, rk)
    dev = upload(tables)
    for name, kind in KINDS:
        caps = [max(e[0].size, 1) for e in expected(tables, 1, name == "anti")]

        def fn(r, comm, sync):
            t = dev[r]
            ws = dj.workspace(ws_bytes(t, 1))
            outs = [torch.empty(caps[r], dtype=torch.int64, device="cuda") for _ in range(2)]
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
        check(tables, 1, name == "anti", [(x[1][1], x[2]) for x in res], f", {name} reported size")


def case_kind_mismatch():
    """Rank 0 asks for a semi join, the others for an anti join: DJ_ERR_ARG on every rank, no hang;
    the group then joins normally."""
    rng = np.random.default_rng([W, 26])
    lk = rng.integers(0, 100_000, 50_000, dtype=np.int64)
    rk = rng.integers(0, 100_000, 40_000, dtype=np.int64)
    tables = with_payloads(split(lk, rng), split(rk, rng))
    dev = upload(tables)

    def fn(r, comm, sync):
        t = dev[r]
        ws = dj.workspace(ws_bytes_global(tables))
        outs = [torch.empty(lk.size, dtype=torch.int64, device="cuda") for _ in range(2)]
        sync()
        kind = dj.JOIN_LEFT_SEMI if r == 0 else dj.JOIN_LEFT_ANTI
        bad = raw_join(comm, kind, t, 1, lk.size, ws, outs)
        sync()
        good = raw_join(comm, dj.JOIN_LEFT_SEMI, t, 1, lk.size, ws, outs)
        return bad, good, [o[:good[1]].clone() for o in outs]

    res = run_ranks(fn)
    for r, (bad, good, _) in enumerate(res):
        assert bad[0] == dj.ERR_ARG and "kind" in bad[3], f"rank {r}: rc {bad[0]} ({bad[3]})"
        assert good[0] == 0, f"rank {r}: {good[3]}"
    check(tables, 1, False, [(x[1][1], x[2]) for x in res], ", after the mismatch")


CASES = {
    "generator-odf1": lambda: case_generator(1),
    "generator-odf2": lambda: case_generator(2),
    "right-slice-empty": case_right_slice_empty,
    "right-table-empty": case_right_table_empty,
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
