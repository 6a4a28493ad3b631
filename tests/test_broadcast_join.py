"""Broadcast joins (dj_broadcast_join_i64): every rank joins its own left rows against the all-gathered
right table.  Single-rank cases compare every kind row for row with the CPU oracles (oracle.np_inner_join,
filter_oracle.py, outer_oracle.py):

  workspace query   CPU: needs no GPU, grows with the gathered right rows and (on the radix path) with
                    the left rows;
  both paths        random tables with duplicates on both sides at DJ_BROADCAST_TABLE_MAX_ROWS right
                    rows (hash table) and one more (radix-partitioned fallback);
  hot right key     20k right copies of one key matched by 500 left rows, next to left and right keys
                    whose table slots follow the hot key's slot;
  edge words        INT64_MIN (the table's "free slot" key), INT64_MAX, 0, -1 and the 32-bit half
                    boundaries as keys and payloads, duplicated on both sides;
  empty tables      the left, the right and both, for every kind;
  capacity          n-1 / n / n+1 output rows, exact counts, untouched guard tails on every column;
  workspace         exactly the queried size (with a sentinel tail), one byte less, and the retry at
                    the size the call reports;
  kinds             the full outer join and an unknown kind are rejected;
  rank groups       N = 2, 3, 4 on one GPU (tests/broadcast_group_worker.py).
"""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import filter_oracle as FO
import keys as K
import outer_oracle as OO
from test_kernel_edges import SENTINEL, SORTED_COMPARE_MAX, _edge_table, _edge_words, _ids, _n, _t

O = FO.O
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = os.path.join(ROOT, "tests", "broadcast_group_worker.py")
KINDS = ["inner", "semi", "anti", "left"]
NCOLS = {"inner": 4, "semi": 2, "anti": 2, "left": 5}
EMPTY_KEY = np.iinfo(np.int64).min  # the key broadcast.cu's table claim treats as a free slot (kEmptyKey)
SIDES_SENTINEL = 0xA5
GUARD = 1024


def _max_rows():
    """DJ_BROADCAST_TABLE_MAX_ROWS as the header states it."""
    with open(os.path.join(ROOT, "include", "dj_b200.h")) as f:
        m = re.search(r"DJ_BROADCAST_TABLE_MAX_ROWS\s*=\s*([^}]*)}", f.read())
    return int(eval(m.group(1), {}))  # an integer expression such as 1 << 20


MAX_ROWS = _max_rows()


def table_slots(nr):
    """broadcast.cu table_slots: the smallest power of two >= 2 * nr, at least 64."""
    s = 64
    while s < 2 * nr:
        s *= 2
    return s


def kind_code(dj, kind):
    return {"inner": 0, "semi": dj.JOIN_LEFT_SEMI, "anti": dj.JOIN_LEFT_ANTI, "left": dj.JOIN_LEFT_OUTER}[kind]


def oracle_join(kind, lk, lp, rk, rp):
    """The oracle's result of `kind` as int64 columns (left outer: sides as a fifth column)."""
    if kind == "inner":
        return O.np_inner_join(lk, lp, rk, rp)
    if kind in ("semi", "anti"):
        return FO.left_semi_join(lk, lp, rk, anti=kind == "anti")
    return OO.outer_join(lk, lp, rk, rp, full=False)


def assert_join(dj, kind, cols, n, ref, what=""):
    """n and the columns equal the oracle's rows `ref`: row for row, or above SORTED_COMPARE_MAX rows by
    count and multiset checksum (per class of sides for a left outer join)."""
    tag = f"{kind}{what}"
    assert len(cols) == NCOLS[kind], f"{tag}: {len(cols)} columns"
    assert n == ref[0].size, f"{tag}: {n} rows, oracle {ref[0].size}"
    got = [c if isinstance(c, np.ndarray) else _n(c) for c in cols]
    if kind == "left":
        got = got[:4] + [got[4].astype(np.int64)]
    if n <= SORTED_COMPARE_MAX:
        for i, (a, b) in enumerate(zip(O.sort_rows(*got), O.sort_rows(*ref))):
            assert (a == b).all(), f"{tag}: column {i} differs from the oracle"
        return
    classes = [(got, ref)] if kind != "left" else \
        [([c[got[4] == s] for c in got[:4]], [c[ref[4] == s] for c in ref[:4]]) for s in (OO.BOTH, OO.SIDE_LEFT)]
    for g, r in classes:
        g4, r4 = (g * 2, r * 2) if len(g) == 2 else (g, r)
        assert g4[0].size == r4[0].size and O.multiset_checksum4(*g4) == O.multiset_checksum4(*r4), f"{tag}: checksum"


def run(dj, kind, lk, lp, rk, rp, **kw):
    """The binding with comm None, checked against the oracle."""
    res = dj.distributed_broadcast_join(None, kind_code(dj, kind), _t(lk), _t(lp), _t(rk), _t(rp), **kw)
    ref = oracle_join(kind, lk, lp, rk, rp)
    assert_join(dj, kind, res.cols, res.n_out, ref)
    return res, ref


def raw(dj, kind, lk, lp, rk, rp, cap, ws=None, guard=GUARD, kind_value=None):
    """One call of the C entry (comm NULL) without the binding's retry loop; every output column carries
    a sentinel guard tail past the capacity.  Semi / anti calls pass NULL for the right payload and the
    unused output columns."""
    import torch

    L = dj.lib()
    k = kind_code(dj, kind) if kind_value is None else kind_value
    pairs = kind in ("inner", "left")
    tl, tp, tr, trp = _t(lk), _t(lp), _t(rk), _t(rp)
    if ws is None:
        ws = dj.workspace(L.dj_broadcast_join_workspace_bytes(len(lk), len(rk)))
    outs = [torch.full((cap + guard,), SENTINEL, dtype=torch.int64, device="cuda") for _ in range(4)]
    outs.append(torch.full((cap + guard,), SIDES_SENTINEL, dtype=torch.uint8, device="cuda"))
    ptr = [o.data_ptr() for o in outs]
    if not pairs:
        ptr[2:] = [None] * 3
    elif kind == "inner":
        ptr[4] = None
    cnt, opts = C.c_int64(-1), dj.JoinOptions(1, 0)
    rc = L.dj_broadcast_join_i64(None, k, tl.data_ptr(), tp.data_ptr(), len(lk), tr.data_ptr(),
                                 trp.data_ptr() if pairs else None, len(rk), *ptr, cap, C.byref(cnt), C.byref(opts),
                                 ws.data_ptr(), ws.numel(), dj._stream())
    torch.cuda.synchronize()
    return rc, cnt.value, [_n(o) for o in outs], opts, (L.dj_last_error().decode() if rc else "")


def random_tables(rng, nl, nr, right_range, left_range):
    """Duplicates on both sides: right keys from a range smaller than the right table, left keys from a
    range that half covers the right keys."""
    lk = rng.integers(0, left_range, nl, dtype=np.int64)
    rk = rng.integers(0, right_range, nr, dtype=np.int64)
    return lk, _ids(nl), rk, _ids(nr, 1 << 40)


# ------------------------------------------------------------------------------------------- CPU
def test_workspace_query_needs_no_gpu_and_grows():
    """The query is plain host arithmetic: it runs here without a device.  It grows with the gathered
    right rows on both paths, and with the left rows where the radix-partitioned path runs (the hash
    table path probes the left columns in place)."""
    sys.path.insert(0, os.path.join(ROOT, "distributed-join_b200"))
    import djb200

    assert djb200.BROADCAST_TABLE_MAX_ROWS == MAX_ROWS
    q = djb200.lib().dj_broadcast_join_workspace_bytes
    for R in (0, 1000, MAX_ROWS // 2, MAX_ROWS + 1):
        assert q(1000, R + 1000) > q(1000, R), R
    for R in (0, MAX_ROWS):  # the hash table path: the left columns are probed where they are
        assert q(10 ** 8, R) == q(1000, R)
    for R in (MAX_ROWS + 1, 4 * MAX_ROWS):
        assert q(10 ** 7, R) > q(1000, R)
    # the gathered columns alone are 16 bytes per right row
    assert q(0, 4 * MAX_ROWS) >= 16 * 4 * MAX_ROWS


def test_hot_key_neighbours_share_its_cluster():
    """CPU: the hot-key case's neighbour keys do land in the slots right after the hot key's slot."""
    hot, near, nslots = _hot_tables(np.random.default_rng(3))[4:]
    slot = K.local_hash(np.array([hot])).astype(np.int64)[0] % nslots
    got = K.local_hash(near).astype(np.int64) % nslots
    assert ((got - slot) % nslots).min() >= 1 and ((got - slot) % nslots).max() <= 8


# ------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("path", ["hash-table", "radix"])
def test_both_paths_against_the_oracle(dj, oracle, kind, path):
    """R = DJ_BROADCAST_TABLE_MAX_ROWS runs the hash table, one row more the radix fallback."""
    rng = np.random.default_rng([1, KINDS.index(kind), len(path)])
    nr = MAX_ROWS if path == "hash-table" else MAX_ROWS + 1
    lk, lp, rk, rp = random_tables(rng, 1_500_000, nr, nr // 2, nr)
    run(dj, kind, lk, lp, rk, rp)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_small_random_tables(dj, oracle, kind):
    rng = np.random.default_rng([2, KINDS.index(kind)])
    lk, lp, rk, rp = random_tables(rng, 300_000, 5000, 4000, 8000)
    run(dj, kind, lk, lp, rk, rp)


def _hot_tables(rng):
    """(lk, lp, rk, rp, hot key, neighbour keys, table slots): 20k right rows of one key, 500 left rows of
    it, and keys whose slots are the 8 after the hot key's -- half of them right keys too, so the hot
    key's slot sits inside a cluster that the neighbours' probes and inserts walk."""
    hot = np.int64(0x0123_4567_89AB_CDEF)
    nr_other = 30_000
    nslots = table_slots(20_000 + nr_other + 64)
    slot = int(K.local_hash(np.array([hot]))[0]) % nslots
    cand = rng.integers(-(1 << 62), 1 << 62, 4_000_000, dtype=np.int64)
    d = (K.local_hash(cand).astype(np.int64) % nslots - slot) % nslots
    near = np.unique(cand[(d >= 1) & (d <= 8)])[:64]
    rk = np.concatenate([np.full(20_000, hot), near[::2], rng.integers(0, 1 << 40, nr_other, dtype=np.int64)])
    lk = np.concatenate([np.full(500, hot), np.repeat(near, 3), rng.integers(0, 1 << 40, 50_000, dtype=np.int64)])
    rk = rng.permutation(rk)[: 20_000 + nr_other + 64]
    lk = rng.permutation(lk)
    return lk, _ids(lk.size), rk, _ids(rk.size, 1 << 40), hot, near, table_slots(rk.size)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_hot_right_key(dj, oracle, kind):
    """Every pair of the hot key (10M for inner and left outer, in 500 warp-written runs) and every
    neighbour's rows."""
    lk, lp, rk, rp, hot, near, _ = _hot_tables(np.random.default_rng(3))
    assert int((rk == hot).sum()) == 20_000 and int((lk == hot).sum()) == 500
    assert np.isin(near, rk).any() and not np.isin(near, rk).all()
    run(dj, kind, lk, lp, rk, rp, capacity=20_000 * 500 + lk.size)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_edge_words(dj, oracle, kind):
    """Edge words (INT64_MIN, the free-slot key, among them) as keys and payloads, 1-3 times per side."""
    ew = _edge_words()
    assert {EMPTY_KEY, np.iinfo(np.int64).max, 0, -1} <= set(ew.tolist())
    rk, rp, lk, lp = _edge_table(np.random.default_rng([4, KINDS.index(kind)]), 2000, 6000)
    # the free-slot key duplicated on both sides, whatever the table drew
    rk = np.concatenate([rk, [EMPTY_KEY, EMPTY_KEY]])
    rp = np.concatenate([rp, [0, EMPTY_KEY]])
    lk = np.concatenate([lk, [EMPTY_KEY, EMPTY_KEY]])
    lp = np.concatenate([lp, [EMPTY_KEY, 0]])
    run(dj, kind, lk, lp, rk, rp)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("empty", ["left", "right", "both"])
def test_empty_tables(dj, oracle, kind, empty):
    rng = np.random.default_rng(5)
    lk, lp, rk, rp = random_tables(rng, 0 if empty != "right" else 20_000, 0 if empty != "left" else 3000, 5000, 5000)
    res, _ = run(dj, kind, lk, lp, rk, rp)
    if empty == "right" and kind in ("anti", "left"):
        assert res.n_out == lk.size


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("cap_delta", ["n-1", "n", "n+1"])
def test_capacity_edges(dj, oracle, kind, cap_delta):
    """The count is exact past the capacity, and no column is written past min(count, capacity)."""
    rng = np.random.default_rng([6, KINDS.index(kind)])
    lk, lp, rk, rp = random_tables(rng, 100_000, 60_000, 40_000, 80_000)
    # a few long runs too, so that warp-written rows meet the capacity as well
    rk[:200] = 7
    lk[:50] = 7
    ref = oracle_join(kind, lk, lp, rk, rp)
    n = ref[0].size
    cap = {"n-1": n - 1, "n": n, "n+1": n + 1}[cap_delta]
    rc, cnt, outs, _, err = raw(dj, kind, lk, lp, rk, rp, cap)
    assert cnt == n
    assert rc == (0 if cap >= n else dj.ERR_OVERFLOW), err
    written = min(cap, n)
    for c in range(NCOLS[kind]):
        fill = SIDES_SENTINEL if c == 4 else SENTINEL
        assert (outs[c][written:] == fill).all(), f"column {c} written past the rows or the capacity"
    for c in range(NCOLS[kind], 5):
        assert (outs[c] == (SIDES_SENTINEL if c == 4 else SENTINEL)).all(), f"unused column {c} written"
    if cap >= n:
        got = [o[:n] for o in outs[:NCOLS[kind]]]
        assert_join(dj, kind, got, n, ref)


WS_GUARD_BYTES, WS_GUARD_BYTE = 4096, 0xA5


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("nr", [3000, MAX_ROWS + 1])
def test_workspace_of_the_queried_size(dj, oracle, kind, nr):
    """Exactly the queried size succeeds without writing past it; one byte less returns DJ_ERR_WORKSPACE
    with the size it needs, and a retry at that size succeeds."""
    import torch

    rng = np.random.default_rng([7, KINDS.index(kind)])
    lk, lp, rk, rp = random_tables(rng, 200_000, nr, nr, 2 * nr)
    q = dj.lib().dj_broadcast_join_workspace_bytes(lk.size, rk.size)
    buf = torch.empty(q + WS_GUARD_BYTES, dtype=torch.uint8, device="cuda")
    buf[q:].fill_(WS_GUARD_BYTE)
    ref = oracle_join(kind, lk, lp, rk, rp)
    cap = max(ref[0].size, 1)
    rc, cnt, outs, _, err = raw(dj, kind, lk, lp, rk, rp, cap, ws=buf[:q], guard=0)
    assert rc == 0, err
    assert bool((buf[q:] == WS_GUARD_BYTE).all()), "the join wrote past the queried workspace"
    assert_join(dj, kind, [o[:cnt] for o in outs[:NCOLS[kind]]], cnt, ref)
    rc, _, _, opts, err = raw(dj, kind, lk, lp, rk, rp, cap, ws=buf[:q - 1], guard=0)
    assert rc == dj.ERR_WORKSPACE, err
    assert opts.workspace_needed == q
    rc, cnt, outs, _, err = raw(dj, kind, lk, lp, rk, rp, cap, ws=buf[:opts.workspace_needed], guard=0)
    assert rc == 0, err
    assert_join(dj, kind, [o[:cnt] for o in outs[:NCOLS[kind]]], cnt, ref, " (retry)")


@pytest.mark.gpu
@pytest.mark.parametrize("bad", ["full-outer", "unknown"])
def test_rejected_kinds(dj, bad):
    rng = np.random.default_rng(8)
    lk, lp, rk, rp = random_tables(rng, 1000, 1000, 1000, 1000)
    value = dj.JOIN_FULL_OUTER if bad == "full-outer" else 7
    rc, cnt, outs, _, err = raw(dj, "left", lk, lp, rk, rp, 4000, kind_value=value)
    assert rc == dj.ERR_ARG, err
    assert all((o == (SIDES_SENTINEL if i == 4 else SENTINEL)).all() for i, o in enumerate(outs))


# ------------------------------------------------------------------------------------ rank groups
@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3, 4])
def test_rank_group(dj, world):
    env = {k: v for k, v in os.environ.items() if k not in ("DJ_EXCHANGE", "DJ_NO_FUSE")}
    env.update(PYTHONDONTWRITEBYTECODE="1", CUDA_DEVICE_MAX_CONNECTIONS="32")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [WORKER, str(world)]
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=1800)
    failed = [line for line in r.stdout.splitlines() if line.startswith("FAIL")]
    assert r.returncode == 0 and not failed, "\n".join(failed) + "\n" + r.stdout[-3000:] + r.stderr[-3000:]
