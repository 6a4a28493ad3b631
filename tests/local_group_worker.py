"""The multi-rank distributed join on ONE GPU: W ranks of an in-process group
(dj_comm_create_local_group), one host thread per rank, every rank's result against the CPU oracle.

    CUDA_DEVICE_MAX_CONNECTIONS=32 python tests/local_group_worker.py W [case ...]

tests/test_local_group.py runs it in a fresh process per (exchange flavour, W); the flavour comes from
the environment (DJ_EXCHANGE=fused, DJ_NO_FUSE=1), where the library reads it.  Prints one line per
case and exits non-zero when a case failed.

Rank r's output must equal the oracle's join of all ranks' tables restricted to the keys r owns
(partition id % W == r), and opts.bytes_sent must be 16 bytes per row r sends to another rank.

Streams: every rank queues work on W + 2 streams (its caller stream, the communicator's two, W - 1
push streams).  A stream parked on a peer's flag blocks its hardware queue, so no two of these
streams may share one.  The driver hands queues out round-robin in stream-creation order, so the
group is created once, before torch creates its stream pool, and the rank streams are the first
W streams taken from that pool; the group lives for the whole process.
"""
import ctypes as C
import os
import sys
import threading
import time
import traceback

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "oracle"), os.path.join(ROOT, "distributed-join_b200"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

import djb200 as dj  # noqa: E402
import keys as K  # noqa: E402
import oracle as O  # noqa: E402
from test_kernel_edges import SORTED_COMPARE_MAX, TARGET, dist_plan  # noqa: E402

W = int(sys.argv[1])
FUSED = os.environ.get("DJ_EXCHANGE", "")[:1] in ("f", "F")
NO_FUSE = os.environ.get("DJ_NO_FUSE", "") == "1"
SEED = dj.SEED_NVLINK
RANK_TIMEOUT_S = 180  # beyond the group's own 120 s bound on a collective
COUNTS = [0, 1, 31, 32, 33, 4097]  # rows one source sends into one segment: padding edges of 32-row runs

COMMS = None
STREAMS = None


class RankError(RuntimeError):
    """A rank thread raised: the group's call sequence may be out of step, so later cases are skipped."""


def run_ranks(fn):
    """fn(rank, comm, sync) on one thread per rank, each under its own stream.  `sync()` is a host
    barrier the ranks pass between allocating and each collective call.  Returns the per-rank
    results after synchronising the device; a rank's exception is re-raised here."""
    bar = threading.Barrier(W, timeout=RANK_TIMEOUT_S)
    res, err = [None] * W, [None] * W

    def body(r):
        try:
            with torch.cuda.stream(STREAMS[r]):
                res[r] = fn(r, COMMS[r], bar.wait)
        except BaseException as e:  # noqa: BLE001 -- re-raised in the main thread
            err[r] = "".join(traceback.format_exception(e))
            bar.abort()

    ths = [threading.Thread(target=body, args=(r,), daemon=True) for r in range(W)]
    for t in ths:
        t.start()
    for t in ths:
        t.join(RANK_TIMEOUT_S)
    if any(t.is_alive() for t in ths):
        raise RankError(f"rank threads still running after {RANK_TIMEOUT_S} s")
    for r, e in enumerate(err):
        if e is not None:
            raise RankError(f"rank {r}: {e}")
    torch.cuda.synchronize()
    return res


# ------------------------------------------------------------------------------------------ tables
def with_payloads(lkeys, rkeys):
    """Per-rank (lk, lp, rk, rp) with payloads unique over all ranks and both sides."""
    out = []
    for r, (lk, rk) in enumerate(zip(lkeys, rkeys)):
        lk, rk = np.ascontiguousarray(lk, np.int64), np.ascontiguousarray(rk, np.int64)
        out.append((lk, (r << 36) + np.arange(lk.size, dtype=np.int64), rk,
                    (1 << 48) + (r << 36) + np.arange(rk.size, dtype=np.int64)))
    return out


def split(a, rng):
    """`a` dealt into W slices of uneven sizes."""
    cuts = np.sort(rng.integers(0, a.size + 1, W - 1))
    return np.split(a, cuts)


def upload(tables):
    dev = [tuple(torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in t) for t in tables]
    torch.cuda.synchronize()
    return dev


def owner(keys, odf):
    return O.partition_ids(keys, SEED, W * odf) % W if len(keys) else np.empty(0, np.int32)


def expected(tables, odf):
    """Per rank: the oracle's rows of the global join whose key rank r owns."""
    gl = [np.concatenate([t[i] for t in tables]) for i in range(4)]
    _, ref = O.inner_join(*gl)
    own = owner(ref[0], odf)
    return [tuple(c[own == r] for c in ref) for r in range(W)]


def sent_bytes(tables, r, odf):
    lk, _, rk, _ = tables[r]
    return 16 * sum(int((owner(k, odf) != r).sum()) for k in (lk, rk))


def check_rank(r, ref, n, cols, what=""):
    tag = f"rank {r}{what}"
    assert n == ref[0].size, f"{tag}: {n} rows, oracle {ref[0].size}"
    if n == 0:
        return
    if n <= SORTED_COMPARE_MAX:
        got = [c.cpu().numpy() for c in cols]
        for i, (a, b) in enumerate(zip(O.sort_rows(*got), O.sort_rows(*ref))):
            assert (a == b).all(), f"{tag}: column {i} differs from the oracle"
    else:
        ck = dj.multiset_checksum4(*cols) if cols[0].is_cuda else O.multiset_checksum4(*[c.numpy() for c in cols])
        assert ck == O.multiset_checksum4(*ref), f"{tag}: checksum differs"


def check(tables, odf, results, exp=None, what=""):
    """results[r]: a JoinResult, or (n, cols, bytes_sent or None)."""
    exp = exp or expected(tables, odf)
    for r, res in enumerate(results):
        n, cols, sent = (res.n_out, res.cols, res.options.bytes_sent) if isinstance(res, dj.JoinResult) else res
        check_rank(r, exp[r], n, cols, what)
        if sent is not None:
            assert sent == sent_bytes(tables, r, odf), f"rank {r}{what}: bytes_sent {sent}, " \
                f"expected {sent_bytes(tables, r, odf)}"


def join_ranks(dev, odf=1, capacity=None, **kw):
    """dj.distributed_inner_join on every rank, allocations before the barrier."""
    def fn(r, comm, sync):
        lk, lp, rk, rp = dev[r]
        ws = dj.workspace(dj.lib().dj_distributed_inner_join_workspace_bytes(lk.numel(), rk.numel(), W, odf))
        cap = capacity or max(lk.numel(), rk.numel(), 1)
        outs = [torch.empty(cap, dtype=torch.int64, device="cuda") for _ in range(4)]
        sync()
        return dj.distributed_inner_join(comm, lk, lp, rk, rp, odf=odf, capacity=cap, ws=ws, outs=outs, **kw)
    return run_ranks(fn)


def run_and_check(tables, odf=1, **kw):
    check(tables, odf, join_ranks(upload(tables), odf, **kw))


def raw_join(comm, t, odf, cap, ws, outs, host=False):
    """One call of the C entry (device or host tables) without the binding's retry loop."""
    cnt, opts = C.c_int64(0), dj.JoinOptions(odf, 0)
    L = dj.lib()
    f = L.dj_distributed_inner_join_i64_host if host else L.dj_distributed_inner_join_i64
    rc = f(comm.handle, t[0].data_ptr(), t[1].data_ptr(), t[0].numel(), t[2].data_ptr(), t[3].data_ptr(),
           t[2].numel(), *[o.data_ptr() for o in outs], cap, C.byref(cnt), C.byref(opts), ws.data_ptr(), ws.numel(),
           dj._stream())
    return rc, cnt.value, opts, (L.dj_last_error().decode() if rc else "")


def keys_pool(n, rng):
    return np.unique(rng.integers(-(1 << 62), 1 << 62, n, dtype=np.int64))


# ------------------------------------------------------------------------------------------- cases
def case_generator(nb, np_, sel, unique, odf):
    g = dj.gen_params(nb, np_, sel, 2 * max(nb, np_), unique)
    tables = []
    for r in range(W):
        (lk, lp), (rk, rp) = dj.generate_tables_distributed(g, r, W)
        tables.append(tuple(x.cpu().numpy() for x in (lk, lp, rk, rp)))
    run_and_check(tables, odf)


def case_plan_edge(two_level):
    """Total sizes on both sides of the single-/two-level edge of the agreed plan (odf 1)."""
    est = (TARGET + 1) * 1024 - (0 if two_level else 1)  # estimated build rows per rank and batch
    tot = (est - 1) * W
    b1, b2, sub = dist_plan(tot, tot + 5000, W, 1, NO_FUSE)
    assert (b2 > 0) == two_level and (sub > 0) == (two_level and not NO_FUSE), (b1, b2, sub)
    rng = np.random.default_rng([W, two_level])
    lk = rng.integers(0, 2 * tot, tot, dtype=np.int64)
    rk = rng.integers(0, 4 * tot, tot + 5000, dtype=np.int64)
    run_and_check(with_payloads(split(lk, rng), split(rk, rng)))


def case_plan_clamped():
    """bits1 > fit: 34 partitions (odf 17 at W = 2) leave room for 4 fused bits, fewer than the 5
    level-1 bits of a 5+6 plan, which becomes 4+7; 26.8M rows per rank and table.  Size-independent checks: the total is the generator's hit count, every
    row joins equal keys, every key lands on its owner."""
    odf, n = 17, 26_800_000
    b1, b2, sub = dist_plan(W * n, W * n, W, odf, NO_FUSE)
    assert (b1, b2, sub) == ((5, 6, 0) if NO_FUSE else (4, 7, 4)), (b1, b2, sub)
    g = dj.gen_params(n, n, 0.3, 2 * n, True)
    g_o = O.gen_params(n, n, 0.3, 2 * n, True)
    hits = sum(O.generate_rows(g_o, 1, s, 0, (n // W) * W, materialize=False)[2] for s in range(W))
    dev = []
    for r in range(W):
        (lk, lp), (rk, rp) = dj.generate_tables_distributed(g, r, W)
        dev.append((lk, lp, rk, rp))
    torch.cuda.synchronize()
    res = join_ranks(dev, odf, capacity=n // 2)
    assert sum(x.n_out for x in res) == hits, ([x.n_out for x in res], hits)
    for r, x in enumerate(res):
        assert bool((x.cols[0] == x.cols[2]).all()), f"rank {r}: unequal keys joined"
        assert bool((dj.partition_ids(x.cols[0], SEED, W * odf) % W == r).all()), f"rank {r}: key of another rank"


def case_padding(odf):
    """No filler: source s sends exactly COUNTS[...] rows into every (destination, batch) bucket, so
    the receive pieces' 32-row-aligned runs meet every padding edge."""
    rng = np.random.default_rng([W, odf, 3])
    nparts = W * odf
    pool = keys_pool(nparts * 3 * W * 4097 * 2, rng)
    pid = O.partition_ids(pool, SEED, nparts)
    lkeys, rkeys = [[] for _ in range(W)], [[] for _ in range(W)]
    for q in range(nparts):
        kq = pool[pid == q]
        cl = [COUNTS[(s + q) % 6] for s in range(W)]
        cr = [COUNTS[(s + 2 * q + 1) % 6] for s in range(W)]
        assert kq.size >= sum(cl) + sum(cr)
        at = 0
        for s in range(W):
            lkeys[s].append(kq[at:at + cl[s]])
            at += cl[s]
        at = sum(cl) // 2  # right rows overlap the second half of the left keys, then run past them
        for s in range(W):
            rkeys[s].append(kq[at:at + cr[s]])
            at += cr[s]
    tables = with_payloads([rng.permutation(np.concatenate(x)) for x in lkeys],
                           [rng.permutation(np.concatenate(x)) for x in rkeys])
    run_and_check(tables, odf)


def case_segments():
    """A two-level plan with the first level fused into the senders' partition: two
    (destination, sub-bucket) segments hold nothing but rows placed there, COUNTS[...] from every
    source, while filler keeps the plan two-level."""
    tot = (TARGET + 1) * 1024 * W * 11 // 10  # the right filler loses its rows in the two segments
    _, _, sub = dist_plan(tot, tot, W, 1, NO_FUSE)
    bits = 5  # the fused plan's sub_bits here (W <= 4); the unfused flavour keys on the same bits
    assert sub == (0 if NO_FUSE else bits), sub
    rng = np.random.default_rng([W, 5])
    segs = [(0, 3, lambda s: COUNTS[s % 6], lambda s: COUNTS[(s + 3) % 6]),
            (W - 1, 17, lambda s: COUNTS[(s + 2) % 6], lambda s: COUNTS[(s + 4) % 6])]
    def in_seg(k, d, j):
        return (owner(k, 1) == d) & ((K.local_hash(k) >> np.uint32(32 - bits)) == j)

    pool = keys_pool(3 * tot, rng)
    placed = np.zeros(pool.size, bool)
    lkeys, rkeys = [[] for _ in range(W)], [[] for _ in range(W)]
    for d, j, cl, cr in segs:
        mask = in_seg(pool, d, j)
        placed |= mask
        kseg = pool[mask]
        at = 0
        for s in range(W):
            lkeys[s].append(kseg[at:at + cl(s)])
            at += cl(s)
        at //= 2
        for s in range(W):
            rkeys[s].append(kseg[at:at + cr(s)])
            at += cr(s)
    filler = pool[~placed][:tot]
    assert filler.size == tot
    lf = split(filler, rng)
    rf = split(np.concatenate([rng.choice(filler, tot // 2), rng.integers(0, 1 << 62, tot - tot // 2, dtype=np.int64)]),
               rng)
    rf = [x[~(in_seg(x, 0, 3) | in_seg(x, W - 1, 17))] for x in rf]
    tables = with_payloads([rng.permutation(np.concatenate(lkeys[s] + [lf[s]])) for s in range(W)],
                           [rng.permutation(np.concatenate(rkeys[s] + [rf[s]])) for s in range(W)])
    totl, totr = sum(t[0].size for t in tables), sum(t[2].size for t in tables)
    assert dist_plan(totl, totr, W, 1, NO_FUSE)[2] == sub, (totl, totr)
    for d, j, cl, cr in segs:  # every segment holds exactly the placed rows
        for s in range(W):
            for k, c in ((tables[s][0], cl(s)), (tables[s][2], cr(s))):
                assert in_seg(k, d, j).sum() == c
    run_and_check(tables)


def case_empty(kind):
    rng = np.random.default_rng([W, len(kind)])
    odf = 2
    n = 100_000
    lk = rng.integers(0, 3 * n, n, dtype=np.int64)
    rk = rng.integers(0, 3 * n, n, dtype=np.int64)
    lpid, rpid = O.partition_ids(lk, SEED, W * odf), O.partition_ids(rk, SEED, W * odf)
    if kind == "one-side":  # batch 0 of rank 0 and batch 1 of rank 1: no left rows
        lk = lk[(lpid != 0) & (lpid != W + 1)]
    elif kind == "everywhere":  # batch 1 of every rank: no rows on either side
        lk, rk = lk[lpid < W], rk[rpid < W]
    ls, rs = split(lk, rng), split(rk, rng)
    if kind == "rank-slice":  # the last rank holds nothing
        ls[0], ls[-1] = np.concatenate([ls[0], ls[-1]]), ls[-1][:0]
        rs[0], rs[-1] = np.concatenate([rs[0], rs[-1]]), rs[-1][:0]
    elif kind == "right-table":
        rs = [x[:0] for x in rs]
    run_and_check(with_payloads(ls, rs), odf)


def case_hot_key():
    """One key with 3000 left x 2000 right rows dealt over every source: 6M rows on its owner, beyond
    the first attempt's capacity, so the collective overflow retry runs too."""
    rng = np.random.default_rng([W, 7])
    hot = np.int64(0x1234_5678_9ABC)
    lk = np.concatenate([np.full(3000, hot), rng.integers(0, 1 << 40, 50_000 * W, dtype=np.int64)])
    rk = np.concatenate([np.full(2000, hot), rng.integers(0, 1 << 40, 40_000 * W, dtype=np.int64)])
    lk, rk = rng.permutation(lk), rng.permutation(rk)
    run_and_check(with_payloads(np.array_split(lk, W), np.array_split(rk, W)))


def case_slot_twins():
    """Different keys with the same slot hash in the same receive-side bucket, all on rank 0."""
    rng = np.random.default_rng([W, 11])
    nl, nr = 60_000, 50_000
    b1, b2, _ = dist_plan(nl, nr, W, 1, NO_FUSE)
    bits = b1 + b2
    base = keys_pool(40_000, rng)
    base = rng.permutation(base[owner(base, 1) == 0])
    tw = K.slot_twins(base, bits, rng)
    keep = owner(tw, 1) == 0
    base, tw = base[keep][:4000], tw[keep][:4000]
    assert base.size >= 1000
    h = base.size // 2
    lk = np.concatenate([base, tw, rng.integers(1 << 62, (1 << 63) - 1, nl - 2 * base.size, dtype=np.int64)])
    rk = np.concatenate([base[:h], tw[h:], np.repeat(base[:50], 3),
                         rng.integers(1 << 61, 1 << 62, nr - base.size - 150, dtype=np.int64)])
    assert lk.size == nl and rk.size == nr
    run_and_check(with_payloads(split(rng.permutation(lk), rng), split(rng.permutation(rk), rng)))


def skewed_tables():
    """Rank 0 holds both tables; the others hold nothing but receive their share."""
    rng = np.random.default_rng(7)
    lk = [rng.permutation(300_000).astype(np.int64)] + [np.empty(0, np.int64)] * (W - 1)
    rk = [rng.integers(0, 300_000, 400_000, dtype=np.int64)] + [np.empty(0, np.int64)] * (W - 1)
    return with_payloads(lk, rk)


def case_workspace_regrow():
    """DJ_ERR_WORKSPACE on every rank; a retry on exactly the reported size; a second call on it
    (cached peer mappings); then six calls rotating over three workspaces (the two-entry mapping
    cache evicts)."""
    tables = skewed_tables()
    dev = upload(tables)
    exp = expected(tables, 1)
    caps = [max(e[0].size, 1) for e in exp]

    def fn(r, comm, sync):
        t = dev[r]
        L = dj.lib()
        ws = dj.workspace(L.dj_distributed_inner_join_workspace_bytes(t[0].numel(), t[2].numel(), W, 1))
        outs = [torch.empty(caps[r], dtype=torch.int64, device="cuda") for _ in range(4)]
        sync()
        first = raw_join(comm, t, 1, caps[r], ws, outs)
        comm.release_workspace()
        ws = dj.workspace(max(ws.numel(), first[2].workspace_needed))
        sync()
        rot = [dj.workspace(ws.numel()) for _ in range(3)]
        calls = []
        for w in [ws, ws] + rot + rot:
            sync()
            rc, n, opts, err = raw_join(comm, t, 1, caps[r], w, outs)
            calls.append((rc, err, n, [o[:n].clone() for o in outs], opts.bytes_sent))
        return first[0], first[2].workspace_needed, ws.numel(), calls

    res = run_ranks(fn)
    assert all(x[0] == dj.ERR_WORKSPACE for x in res), [x[0] for x in res]
    assert any(x[1] > 0 for x in res)
    for i in range(len(res[0][3])):
        assert all(x[3][i][0] == 0 for x in res), f"call {i}: " + "; ".join(x[3][i][1] for x in res)
        check(tables, 1, [x[3][i][2:] for x in res], exp, f", call {i}")


def case_overflow():
    """Capacity one below the largest rank's count: every rank returns DJ_ERR_OVERFLOW with its own
    exact count, and the binding's collective retry reproduces the oracle.  Capacity equal to it:
    no rank overflows."""
    rng = np.random.default_rng([W, 13])
    hot = np.int64(987_654_321_987)
    lk = rng.permutation(np.concatenate([np.full(60, hot), rng.integers(0, 400_000, 200_000, dtype=np.int64)]))
    rk = rng.permutation(np.concatenate([np.full(50, hot), rng.integers(0, 400_000, 150_000, dtype=np.int64)]))
    tables = with_payloads(split(lk, rng), split(rk, rng))
    exp = expected(tables, 1)
    counts = [e[0].size for e in exp]
    top = max(counts)
    assert sorted(counts)[-2] < top, counts
    dev = upload(tables)
    # room for any rank's receive pieces: the slices are uneven
    ws_bytes = dj.lib().dj_distributed_inner_join_workspace_bytes(lk.size, rk.size, W, 1)

    def fn(r, comm, sync):
        t = dev[r]
        ws = dj.workspace(ws_bytes)
        outs = [torch.empty(top, dtype=torch.int64, device="cuda") for _ in range(4)]
        outs2 = [torch.empty(top - 1, dtype=torch.int64, device="cuda") for _ in range(4)]
        sync()
        over = raw_join(comm, t, 1, top - 1, ws, outs)
        sync()
        exact = raw_join(comm, t, 1, top, ws, outs)
        exact_cols = [o[:exact[1]].clone() for o in outs]
        sync()
        retried = dj.distributed_inner_join(comm, *t, capacity=top - 1, ws=ws, outs=outs2)
        return over, exact, exact_cols, retried

    res = run_ranks(fn)
    for r, (over, exact, exact_cols, retried) in enumerate(res):
        assert over[0] == dj.ERR_OVERFLOW, f"rank {r}: rc {over[0]} at capacity {top - 1}"
        assert over[1] == counts[r], f"rank {r}: count {over[1]} under overflow, oracle {counts[r]}"
        assert exact[0] == 0, f"rank {r}: {exact[3]}"
    check(tables, 1, [(x[1][1], x[2], None) for x in res], exp, ", exact")
    check(tables, 1, [x[3] for x in res], exp, ", retried")


def case_repeated():
    """Calls with changing sizes and odf on one group: inbox banks, sequence numbers and the verdict
    slots are reused call after call."""
    rng = np.random.default_rng([W, 17])
    shapes = [(200_000, 300_000, 1), (5_000, 1_000, 2), (0, 40_000, 1), (1_000_000, 800_000, 4), (3, 2, 1),
              (200_000, 300_000, 2)]
    all_tables = []
    for nl, nr, odf in shapes:
        lk = rng.integers(0, max(nl, 1) * 2, nl, dtype=np.int64)
        rk = rng.integers(0, max(nl, 1) * 2, nr, dtype=np.int64)
        all_tables.append((with_payloads(split(lk, rng), split(rk, rng)), odf))
    devs = [upload(t) for t, _ in all_tables]

    def fn(r, comm, sync):
        out = []
        for dev, (_, odf) in zip(devs, all_tables):
            lk, lp, rk, rp = dev[r]
            ws = dj.workspace(dj.lib().dj_distributed_inner_join_workspace_bytes(lk.numel(), rk.numel(), W, odf))
            cap = max(lk.numel(), rk.numel(), 1)
            outs = [torch.empty(cap, dtype=torch.int64, device="cuda") for _ in range(4)]
            sync()
            out.append(dj.distributed_inner_join(comm, lk, lp, rk, rp, odf=odf, capacity=cap, ws=ws, outs=outs))
        return out

    res = run_ranks(fn)
    for i, (tables, odf) in enumerate(all_tables):
        check(tables, odf, [x[i] for x in res], what=f", call {i}")


def case_odf(odf):
    rng = np.random.default_rng([W, odf])
    lk = rng.integers(0, 600_000, 300_000, dtype=np.int64)
    rk = rng.integers(0, 600_000, 250_000, dtype=np.int64)
    tables = with_payloads(split(lk, rng), split(rk, rng))
    if odf <= 31:  # 2 * odf <= 62 data flag slots: the last odf the peer exchange carries
        run_and_check(tables, odf)
        return
    dev = upload(tables)

    def fn(r, comm, sync):
        t = dev[r]
        ws = dj.workspace(dj.lib().dj_distributed_inner_join_workspace_bytes(t[0].numel(), t[2].numel(), W, odf))
        outs = [torch.empty(max(t[0].numel(), 1), dtype=torch.int64, device="cuda") for _ in range(4)]
        sync()
        return raw_join(comm, t, odf, outs[0].numel(), ws, outs)

    for r, (rc, _, _, err) in enumerate(run_ranks(fn)):
        assert rc == 2 and "NCCL" in err, f"rank {r}: rc {rc} ({err})"


def case_host_entry(kind):
    """dj_distributed_inner_join_i64_host at N > 1.  Skewed: every rank fails with DJ_ERR_WORKSPACE,
    and a retry on a workspace of exactly the reported size must fit (the report counts the staged
    columns), then the binding's own retry loop."""
    if kind == "generator":
        g = dj.gen_params(500_000, 500_000, 0.5, 1_000_000, True)
        tables = []
        for r in range(W):
            (lk, lp), (rk, rp) = dj.generate_tables_distributed(g, r, W)
            tables.append(tuple(x.cpu().numpy() for x in (lk, lp, rk, rp)))
    else:
        tables = skewed_tables()
    exp = expected(tables, 1)
    pinned = [tuple(torch.from_numpy(np.ascontiguousarray(a)).pin_memory() for a in t) for t in tables]
    caps = [max(e[0].size, 1) for e in exp]
    h_outs = [[torch.empty(c, dtype=torch.int64).pin_memory() for _ in range(2 * 4)] for c in caps]

    def fn(r, comm, sync):
        t, outs = pinned[r], h_outs[r]
        out = {}
        L = dj.lib()
        ws_bytes = L.dj_distributed_inner_join_host_workspace_bytes(t[0].numel(), t[2].numel(), caps[r], W, 1)
        if kind == "skewed":
            ws = dj.workspace(ws_bytes)
            sync()
            first = raw_join(comm, t, 1, caps[r], ws, outs[:4], host=True)
            comm.release_workspace()
            ws = dj.workspace(max(ws.numel(), first[2].workspace_needed))
            sync()
            again = raw_join(comm, t, 1, caps[r], ws, outs[:4], host=True)
            out["raw"] = (first[0], again[0], again[3], again[1])
            if again[0]:  # the verdict is collective: every rank stops here
                return out, outs
        ws = dj.workspace(ws_bytes)
        sync()
        n, _ = dj.distributed_inner_join_host(comm, *t, outs[4:], ws=ws)
        out["binding"] = n
        return out, outs

    res = run_ranks(fn)
    if kind == "skewed":
        assert all(o["raw"][0] == dj.ERR_WORKSPACE for o, _ in res), [o["raw"][0] for o, _ in res]
        for r, (o, outs) in enumerate(res):
            assert o["raw"][1] == 0, f"rank {r}: retry on the reported workspace size failed: {o['raw'][2]}"
            check_rank(r, exp[r], o["raw"][3], [x[:o["raw"][3]] for x in outs[:4]], ", reported size")
    for r, (o, outs) in enumerate(res):
        check_rank(r, exp[r], o["binding"], [x[:o["binding"]] for x in outs[4:]], ", binding")


def case_timing():
    rng = np.random.default_rng([W, 19])
    lk = rng.integers(0, 2_000_000, 1_000_000, dtype=np.int64)
    rk = rng.integers(0, 2_000_000, 1_200_000, dtype=np.int64)
    tables = with_payloads(split(lk, rng), split(rk, rng))
    res = join_ranks(upload(tables), 2, report_timing=True, measure_exchange=True)
    for r, x in enumerate(res):
        o = x.options
        vals = [o.t_partition_ms, o.t_comm_ms, o.t_join_ms, o.t_exchange_ms[0], o.t_exchange_ms[1],
                o.t_exchange_total_ms]
        assert all(v >= 0 for v in vals), f"rank {r}: {vals}"
    check(tables, 2, res)


def case_nccl_only_entries():
    """Entry points that need NCCL fail with an error on a local group, and group creation refuses
    DJ_EXCHANGE=nccl and a stream count beyond CUDA_DEVICE_MAX_CONNECTIONS (before creating anything)."""
    L = dj.lib()
    c = COMMS[0].handle
    buf = torch.zeros(64, dtype=torch.int64, device="cuda")
    vp = C.c_void_p
    for name, rc in [
        ("send", L.dj_comm_send(c, buf.data_ptr(), 8, 1, None)),
        ("recv", L.dj_comm_recv(c, buf.data_ptr(), 8, 1, None)),
        ("group_start", L.dj_comm_group_start(c)),
        ("group_end", L.dj_comm_group_end(c)),
        ("all_to_all", L.dj_all_to_all(c, W, (C.c_int * W)(*range(W)), 0, (vp * 1)(buf.data_ptr()),
                                       (vp * 1)(buf.data_ptr()), (C.c_int64 * (W + 1))(), (C.c_int64 * (W + 1))(),
                                       (C.c_int * 1)(8), 1, 0, None)),
    ]:
        assert rc == 2 and b"NCCL" in L.dj_last_error(), f"{name}: rc {rc} ({L.dj_last_error()})"
    handles = (vp * 3)()
    saved = {k: os.environ.get(k) for k in ("DJ_EXCHANGE", "CUDA_DEVICE_MAX_CONNECTIONS")}
    try:
        os.environ["DJ_EXCHANGE"] = "nccl"
        assert L.dj_comm_create_local_group(2, handles) == 2 and b"NCCL" in L.dj_last_error()
        del os.environ["DJ_EXCHANGE"]
        os.environ["CUDA_DEVICE_MAX_CONNECTIONS"] = "8"  # read at the call; the device keeps its 32 queues
        assert L.dj_comm_create_local_group(3, handles) == 2 and b"CUDA_DEVICE_MAX_CONNECTIONS" in L.dj_last_error()
    finally:
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    assert not any(handles)


CASES = {
    "generator-unique-odf1": lambda: case_generator(1_000_000, 1_000_000, 0.3, True, 1),
    "generator-unique-odf4": lambda: case_generator(1_000_000, 1_000_000, 0.3, True, 4),
    "generator-duplicates-odf2": lambda: case_generator(500_000, 2_000_000, 0.9, False, 2),
    "generator-tiny": lambda: case_generator(4_000, 4_000, 1.0, True, 1),
    "plan-single-level": lambda: case_plan_edge(False),
    "plan-two-level": lambda: case_plan_edge(True),
    "padding-odf1": lambda: case_padding(1),
    "padding-odf2": lambda: case_padding(2),
    "segments": case_segments,
    "empty-batch-one-side": lambda: case_empty("one-side"),
    "empty-batch-everywhere": lambda: case_empty("everywhere"),
    "empty-rank-slice": lambda: case_empty("rank-slice"),
    "empty-right-table": lambda: case_empty("right-table"),
    "hot-key": case_hot_key,
    "slot-twins": case_slot_twins,
    "workspace-regrow": case_workspace_regrow,
    "overflow": case_overflow,
    "repeated-calls": case_repeated,
    "odf31": lambda: case_odf(31),
    "odf32-error": lambda: case_odf(32),
    "host-generator": lambda: case_host_entry("generator"),
    "host-skewed": lambda: case_host_entry("skewed"),
    "timing": case_timing,
    "nccl-only-entries": case_nccl_only_entries,
}
if W == 2:
    CASES["plan-clamped"] = case_plan_clamped


def main():
    global COMMS, STREAMS
    names = sys.argv[2:] or list(CASES)
    torch.cuda.init()
    O.build()
    COMMS = dj.Comm.local_group(W)  # before torch's stream pool: see the module docstring
    STREAMS = [torch.cuda.Stream() for _ in range(W)]
    failed = []
    for name in names:
        t0 = time.time()
        print(f"run  {name}", flush=True)
        try:
            CASES[name]()
            print(f"ok   {name} ({time.time() - t0:.1f} s)", flush=True)
        except RankError as e:
            # the group may be out of step and its streams parked on flags nobody raises: no
            # synchronisation, no further cases; exiting tears the context down
            print(f"FAIL {name}: {e}", flush=True)
            print("a rank thread failed: the remaining cases are skipped", flush=True)
            os._exit(1)
        except Exception as e:  # noqa: BLE001 -- reported per case
            print(f"FAIL {name}: {type(e).__name__}: {e}", flush=True)
            failed.append(name)
    torch.cuda.synchronize()
    for c in COMMS:
        c.destroy()
    print(f"{len(names) - len(failed)} of {len(names)} cases passed (W={W}, "
          f"flavour {'fused' if FUSED else 'no-fuse' if NO_FUSE else 'default'})", flush=True)
    sys.exit(1 if failed else 0)


if __name__ == "__main__":
    main()
