"""The host-buffer entries of the semi, anti, left outer and full outer joins at N > 1, on ONE GPU: W
ranks of an in-process group, one host thread per rank.

    CUDA_DEVICE_MAX_CONNECTIONS=32 python tests/host_kinds_group_worker.py W [case ...]

tests/test_host_join_kinds.py runs it in a fresh process per W, as tests/test_outer_join.py runs
outer_group_worker.py, whose group plumbing this worker shares.  At N > 1 the entries stage their
columns in front of the device entry's workspace: the generator case holds every kind against the
simulated distributed oracle, and the skewed case makes every rank fail with DJ_ERR_WORKSPACE once
and succeed on a workspace of exactly the size the error reported (staged columns included).
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
import outer_oracle as OO  # noqa: E402
from local_group_worker import RankError, W, owner, run_ranks  # noqa: E402

KINDS = {"semi": dj.JOIN_LEFT_SEMI, "anti": dj.JOIN_LEFT_ANTI, "left": dj.JOIN_LEFT_OUTER, "full": dj.JOIN_FULL_OUTER}


def is_filter(name):
    return name in ("semi", "anti")


def simulated(name, tables, odf=1):
    """Per rank, the columns the distributed join of kind `name` leaves there (sides last, int64)."""
    lefts, rights = [t[:2] for t in tables], [t[2:] for t in tables]
    if is_filter(name):
        return FO.simulate_distributed_left_semi_join(lefts, [r[0] for r in rights], odf, name == "anti")
    return OO.simulate_distributed_outer_join(lefts, rights, odf, name == "full")


def owned(name, tables):
    """The same by restriction: the global join's rows whose placing key rank r owns."""
    gl = [np.concatenate([t[i] for t in tables]) for i in range(4)]
    if is_filter(name):
        ref = FO.left_semi_join(gl[0], gl[1], gl[2], name == "anti")
        own = owner(ref[0], 1)
    else:
        ref = OO.outer_join(*gl, name == "full")
        own = owner(OO.row_keys(ref), 1)
    return [tuple(c[own == r] for c in ref) for r in range(W)]


def _sorted(cols):
    cols = [np.asarray(c, dtype=np.int64) for c in cols]
    order = np.lexsort(cols[::-1]) if cols[0].size else np.empty(0, np.int64)
    return [c[order] for c in cols]


def check_rank(r, ref, n, h_outs, what):
    assert n == ref[0].size, f"rank {r}, {what}: {n} rows, oracle {ref[0].size}"
    got = [o.numpy()[:n] for o in h_outs]
    for i, (a, b) in enumerate(zip(_sorted(got), _sorted(ref))):
        assert (a == b).all(), f"rank {r}, {what}: column {i} differs from the oracle"


def pin(tables):
    return [tuple(torch.from_numpy(np.ascontiguousarray(a)).pin_memory() for a in t) for t in tables]


def host_columns(name, cap):
    cols = [torch.empty(cap, dtype=torch.int64).pin_memory() for _ in range(2 if is_filter(name) else 4)]
    return cols if is_filter(name) else cols + [torch.empty(cap, dtype=torch.uint8).pin_memory()]


def ws_query(name, t, cap):
    L = dj.lib()
    fn = L.dj_distributed_left_filter_join_host_workspace_bytes if is_filter(name) else \
        L.dj_distributed_outer_join_host_workspace_bytes
    return fn(t[0].numel(), t[2].numel(), cap, W, 1)


def raw_host_join(comm, name, t, cap, ws, outs):
    """One call of the C entry without the binding's retry loop."""
    cnt, opts = C.c_int64(0), dj.JoinOptions(1, 0)
    L = dj.lib()
    if is_filter(name):
        rc = L.dj_distributed_left_filter_join_i64_host(comm.handle, KINDS[name], t[0].data_ptr(), t[1].data_ptr(),
                                                        t[0].numel(), t[2].data_ptr(), t[2].numel(),
                                                        outs[0].data_ptr(), outs[1].data_ptr(), cap, C.byref(cnt),
                                                        C.byref(opts), ws.data_ptr(), ws.numel(), dj._stream())
    else:
        rc = L.dj_distributed_outer_join_i64_host(comm.handle, KINDS[name], *[x.data_ptr() for x in t[:2]],
                                                  t[0].numel(), *[x.data_ptr() for x in t[2:]], t[2].numel(),
                                                  *[o.data_ptr() for o in outs], cap, C.byref(cnt), C.byref(opts),
                                                  ws.data_ptr(), ws.numel(), dj._stream())
    return rc, cnt.value, opts, (L.dj_last_error().decode() if rc else "")


def binding(comm, name, t, outs, ws):
    if is_filter(name):
        return dj.distributed_left_filter_join_host(comm, KINDS[name], t[0], t[1], t[2], outs, ws=ws)
    return dj.distributed_outer_join_host(comm, KINDS[name], *t, outs, ws=ws)


# ------------------------------------------------------------------------------------------- cases
def case_generator():
    """The benchmark's generator (the probe table as left, the unique build table as right) through
    the binding, every kind against the simulated oracle and against the owner restriction."""
    g = dj.gen_params(400_000, 800_000, 0.3, 1_600_000, True)
    tables = []
    for r in range(W):
        (bk, bp), (pk, pp) = dj.generate_tables_distributed(g, r, W)
        tables.append(tuple(x.cpu().numpy() for x in (pk, pp, bk, bp)))
    pinned = pin(tables)
    for name in KINDS:
        sim, exp = simulated(name, tables), owned(name, tables)
        h_outs = [host_columns(name, max(e[0].size, 1)) for e in exp]

        def fn(r, comm, sync):
            ws = dj.workspace(ws_query(name, pinned[r], h_outs[r][0].numel()))
            sync()
            return binding(comm, name, pinned[r], h_outs[r], ws)[0]

        for r, n in enumerate(run_ranks(fn)):
            check_rank(r, sim[r], n, h_outs[r], f"{name} vs simulation")
            check_rank(r, exp[r], n, h_outs[r], f"{name} vs owner restriction")


def case_workspace_regrow():
    """Rank 0 holds both tables: the balanced estimate behind the staged columns is too small on the
    receivers, every rank returns DJ_ERR_WORKSPACE, and a retry on a workspace of exactly the reported
    size succeeds; then the binding's own grow-and-retry loop from the queried size."""
    rng = np.random.default_rng(7)
    lk = [rng.integers(0, 600_000, 300_000, dtype=np.int64)] + [np.empty(0, np.int64)] * (W - 1)
    rk = [rng.integers(0, 600_000, 400_000, dtype=np.int64)] + [np.empty(0, np.int64)] * (W - 1)
    tables = LG.with_payloads(lk, rk)
    pinned = pin(tables)
    for name in KINDS:
        exp = owned(name, tables)
        caps = [max(e[0].size, 1) for e in exp]
        h_outs = [(host_columns(name, c), host_columns(name, c)) for c in caps]

        def fn(r, comm, sync):
            t, (outs, outs2) = pinned[r], h_outs[r]
            size = ws_query(name, t, caps[r])
            ws = dj.workspace(size)
            sync()
            first = raw_host_join(comm, name, t, caps[r], ws, outs)
            comm.release_workspace()
            ws = dj.workspace(max(ws.numel(), first[2].workspace_needed))
            sync()
            again = raw_host_join(comm, name, t, caps[r], ws, outs)
            if again[0]:  # the verdict is collective: every rank stops here
                return first, again, None
            ws = dj.workspace(size)
            sync()
            return first, again, binding(comm, name, t, outs2, ws)[0]

        res = run_ranks(fn)
        assert all(x[0][0] == dj.ERR_WORKSPACE for x in res), (name, [x[0][0] for x in res])
        assert any(x[0][2].workspace_needed > ws_query(name, pinned[r], caps[r]) for r, x in enumerate(res)), name
        for r, (first, again, n2) in enumerate(res):
            assert again[0] == 0, f"{name} rank {r}: retry on the reported size failed: {again[3]}"
            check_rank(r, exp[r], again[1], h_outs[r][0], f"{name}, reported size")
            check_rank(r, exp[r], n2, h_outs[r][1], f"{name}, binding")


def case_overflow():
    """A capacity one below the largest rank's count: DJ_ERR_OVERFLOW on every rank with its own exact
    count, min(count, capacity) rows copied down, and the binding raises on every rank."""
    rng = np.random.default_rng([W, 9])
    lk = rng.integers(0, 200_000, 150_000, dtype=np.int64)
    rk = rng.integers(0, 200_000, 100_000, dtype=np.int64)
    tables = LG.with_payloads(LG.split(lk, rng), LG.split(rk, rng))
    pinned = pin(tables)
    lk_all, rk_all = torch.from_numpy(lk), torch.from_numpy(rk)
    for name in ("anti", "full"):
        exp = owned(name, tables)
        counts = [e[0].size for e in exp]
        cap = max(counts) - 1
        h_outs = [host_columns(name, cap) for _ in range(W)]

        def fn(r, comm, sync):
            ws = dj.workspace(ws_query(name, (lk_all, None, rk_all), cap))  # room for any rank's share
            sync()
            raw = raw_host_join(comm, name, pinned[r], cap, ws, h_outs[r])
            kept = [o.numpy()[:min(raw[1], cap)].copy() for o in h_outs[r]]
            sync()
            try:
                binding(comm, name, pinned[r], h_outs[r], ws)
                raised = False
            except dj.DjError:
                raised = True
            return raw, kept, raised

        for r, (raw, kept, raised) in enumerate(run_ranks(fn)):
            assert raw[0] == dj.ERR_OVERFLOW and raw[1] == counts[r], f"{name} rank {r}: rc {raw[0]}, count {raw[1]}"
            assert raised, f"{name} rank {r}: the binding did not raise"
            ref = _sorted(exp[r])
            if counts[r] <= cap:  # this rank's rows all fit: they are all there
                for a, b in zip(_sorted(kept), ref):
                    assert (a == b).all(), f"{name} rank {r}: rows under a peer's overflow"


CASES = {"generator": case_generator, "workspace-regrow": case_workspace_regrow, "overflow": case_overflow}


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
