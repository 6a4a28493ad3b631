"""Broadcast full outer join (dj_broadcast_full_outer_join_i64): rank r returns the left outer join of its own
left rows with the all-gathered right table, plus the rows of its own right slice that no rank's left rows
matched.  Single-rank cases compare row for row with outer_oracle.outer_join(..., full=True):

  workspace query   CPU: needs no GPU, grows with this rank's right rows, the gathered right rows and
                    the rank count, and is at least the broadcast join's on both local-join paths;
  restatement       CPU: the per-rank result restated (own left outer ++ own right rows whose key is in
                    no rank's left keys); its union over the ranks is the global full outer join;
  both paths        DJ_BROADCAST_TABLE_MAX_ROWS right rows (hash table) and one more (radix-partitioned),
                    duplicates on both sides, about half the right keys unmatched, distinct right payloads
                    (a pair carrying the gathered row index instead of the payload shows);
  all / none        every right row matched (no sides-2 rows) and no right row matched;
  hot keys          20k right copies of a matched key and 20k of an unmatched one, next to keys whose
                    table slots follow the matched hot key's slot;
  edge words        INT64_MIN (the side slot's key) on the right, matched and unmatched;
  empty tables      the left, the right and both;
  capacity          n-1 / n / n+1 with the boundary inside the left outer rows and inside the emitted
                    right rows: exact counts, untouched guard tails on all five columns;
  workspace         exactly the queried size (sentinel tail), one byte less, and the retry;
  back to back      two calls with different tables in one workspace;
  variants          the radix-path cases again under DJ_JOIN_SHAPE=B and DJ_RADIX_EXACT=1;
  rank groups       N = 2, 3, 4 on one GPU (tests/broadcast_full_outer_group_worker.py).
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import outer_oracle as OO
from test_broadcast_join import (GUARD, MAX_ROWS, SENTINEL, SIDES_SENTINEL, _hot_tables, _ids, _t,
                                 random_tables)
from test_kernel_edges import SORTED_COMPARE_MAX, _edge_table, _n

import oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = os.path.join(ROOT, "tests", "broadcast_full_outer_group_worker.py")
EMPTY_KEY = np.iinfo(np.int64).min
CLASSES = (OO.BOTH, OO.SIDE_LEFT, OO.SIDE_RIGHT)


def _lib():
    sys.path.insert(0, os.path.join(ROOT, "distributed-join_b200"))
    import djb200

    return djb200.lib()


def restated(lefts, rights, r):
    """Rank r's rows restated: the left outer join of its own left rows with every rank's right rows, then
    its own right rows whose key is in no rank's left keys, as (0, 0, key, payload, SIDE_RIGHT)."""
    grk = np.concatenate([x[0] for x in rights])
    grp = np.concatenate([x[1] for x in rights])
    lo = OO.outer_join(*lefts[r], grk, grp, full=False)
    all_left = np.concatenate([x[0] for x in lefts])
    rk, rp = rights[r]
    lone = ~np.isin(rk, all_left)
    z = np.zeros(int(lone.sum()), np.int64)
    em = (z, z, rk[lone], rp[lone], np.full(z.size, OO.SIDE_RIGHT, np.int64))
    return tuple(np.concatenate([a, b]) for a, b in zip(lo, em))


def assert_full(cols, n, ref, what=""):
    """n and the five columns equal the oracle's rows: row for row, or above SORTED_COMPARE_MAX rows by count
    and multiset checksum per class of sides."""
    assert len(cols) == 5, f"{what}: {len(cols)} columns"
    assert n == ref[0].size, f"{what}: {n} rows, oracle {ref[0].size}"
    got = [c if isinstance(c, np.ndarray) else _n(c) for c in cols]
    got = got[:4] + [got[4].astype(np.int64)]
    if n <= SORTED_COMPARE_MAX:
        for i, (a, b) in enumerate(zip(O.sort_rows(*got), O.sort_rows(*ref))):
            assert (a == b).all(), f"{what}: column {i} differs from the oracle"
        return
    for s in CLASSES:
        g, r = [c[got[4] == s] for c in got[:4]], [c[ref[4] == s] for c in ref[:4]]
        assert g[0].size == r[0].size, f"{what}: sides {s}: {g[0].size} rows, oracle {r[0].size}"
        assert O.multiset_checksum4(*g) == O.multiset_checksum4(*r), f"{what}: sides {s}: checksum"


def run(dj, lk, lp, rk, rp, **kw):
    """The binding with comm None, checked against the oracle."""
    res = dj.distributed_broadcast_full_outer_join(None, _t(lk), _t(lp), _t(rk), _t(rp), **kw)
    ref = OO.outer_join(lk, lp, rk, rp, full=True)
    assert_full(res.cols, res.n_out, ref)
    return res, ref


def raw(dj, lk, lp, rk, rp, cap, ws=None, guard=GUARD):
    """One call of the C entry (comm NULL) without the binding's retry loop; every output column carries a
    sentinel guard tail past the capacity."""
    import torch

    L = dj.lib()
    tl, tp, tr, trp = _t(lk), _t(lp), _t(rk), _t(rp)
    if ws is None:
        ws = dj.workspace(L.dj_broadcast_full_outer_join_workspace_bytes(len(lk), len(rk), len(rk), 1))
    outs = [torch.full((cap + guard,), SENTINEL, dtype=torch.int64, device="cuda") for _ in range(4)]
    outs.append(torch.full((cap + guard,), SIDES_SENTINEL, dtype=torch.uint8, device="cuda"))
    cnt, opts = C.c_int64(-1), dj.JoinOptions(1, 0)
    rc = L.dj_broadcast_full_outer_join_i64(None, tl.data_ptr(), tp.data_ptr(), len(lk), tr.data_ptr(),
                                            trp.data_ptr(), len(rk), *[o.data_ptr() for o in outs], cap,
                                            C.byref(cnt), C.byref(opts), ws.data_ptr(), ws.numel(), dj._stream())
    torch.cuda.synchronize()
    return rc, cnt.value, [_n(o) for o in outs], opts, (L.dj_last_error().decode() if rc else "")


def half_matched(rng, nl, nr):
    """Right keys from [0, 2 nr), left keys from [0, nr): duplicates on both sides, and the right keys at
    or above nr (about half) match nothing.  Right payloads are distinct."""
    return random_tables(rng, nl, nr, 2 * nr, nr)


# ------------------------------------------------------------------------------------------- CPU
def test_workspace_query_needs_no_gpu_and_grows():
    L = _lib()
    q = L.dj_broadcast_full_outer_join_workspace_bytes
    b = L.dj_broadcast_join_workspace_bytes
    for R in (0, 1000, MAX_ROWS // 2, MAX_ROWS, MAX_ROWS + 1, 4 * MAX_ROWS):
        for nl in (0, 1000, 10 ** 7):
            for world in (1, 2, 4):
                nr = R // world
                got = q(nl, nr, R, world)
                assert got >= b(nl, R), (nl, nr, R, world)
                assert q(nl, nr + 10_000, R, world) > got, (nl, nr, R, world)  # own slice: the inbox rows
                if (R <= MAX_ROWS) == (R + 10_000 <= MAX_ROWS):  # the same local-join path
                    assert q(nl, nr, R + 10_000, world) > got, (nl, nr, R, world)  # gathered rows
                wide = q(nl, nr + 10_000, R + 10_000, world)
                assert q(nl, nr + 10_000, R + 10_000, world + 1) > wide, (nl, nr, R, world)  # one more inbox row
    # the inbox holds world rows of (nright + 31) / 32 + 1 words
    assert q(1000, 32 * 10_000, 32 * 10_000, 64) - q(1000, 32 * 10_000, 32 * 10_000, 1) >= 63 * 4 * 10_001 - 256


def test_restatement_unions_to_the_global_full_outer_join():
    """Per class of sides, the union over the ranks of the restated rows is the global full outer join: the
    pairs and lone left rows split by left slice, each lone right row appears once, on its owner."""
    rng = np.random.default_rng(11)
    for world in (1, 2, 3, 4):
        lk, rk = rng.integers(0, 3000, 5000, dtype=np.int64), rng.integers(0, 6000, 2500, dtype=np.int64)
        rk[:40] = rk[0]  # a key several ranks hold copies of
        lc = np.sort(rng.integers(0, lk.size + 1, world - 1))
        rc = np.sort(rng.integers(0, rk.size + 1, world - 1))
        lefts = [(k, _ids(k.size, i << 32)) for i, k in enumerate(np.split(lk, lc))]
        rights = [(k, _ids(k.size, (i + 1) << 40)) for i, k in enumerate(np.split(rk, rc))]
        per = [restated(lefts, rights, r) for r in range(world)]
        got = tuple(np.concatenate([p[c] for p in per]) for c in range(5))
        ref = OO.outer_join(lk, np.concatenate([x[1] for x in lefts]), rk, np.concatenate([x[1] for x in rights]),
                            full=True)
        for s in CLASSES:
            g = O.sort_rows(*[c[got[4] == s] for c in got[:4]])
            r = O.sort_rows(*[c[ref[4] == s] for c in ref[:4]])
            assert all((a == b).all() for a, b in zip(g, r)), (world, s)
        assert (ref[4] == OO.SIDE_RIGHT).any() and (ref[4] == OO.BOTH).any()


# ------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("path", ["hash-table", "radix"])
def test_both_paths_against_the_oracle(dj, oracle, path):
    rng = np.random.default_rng([21, len(path)])
    nr = MAX_ROWS if path == "hash-table" else MAX_ROWS + 1
    lk, lp, rk, rp = half_matched(rng, 1_500_000, nr)
    _, ref = run(dj, lk, lp, rk, rp)
    lone_r = int((ref[4] == OO.SIDE_RIGHT).sum())
    assert 0.35 * nr < lone_r < 0.65 * nr, lone_r


@pytest.mark.gpu
@pytest.mark.parametrize("matched", ["all", "none"])
@pytest.mark.parametrize("path", ["hash-table", "radix"])
def test_every_or_no_right_row_matched(dj, oracle, matched, path):
    rng = np.random.default_rng([22, len(matched), len(path)])
    nr = 50_000 if path == "hash-table" else MAX_ROWS + 1
    rk = rng.integers(0, nr // 2, nr, dtype=np.int64)
    if matched == "all":
        lk = rng.permutation(np.concatenate([np.unique(rk), rng.integers(nr, 4 * nr, 100_000, dtype=np.int64)]))
    else:
        lk = rng.integers(nr, 4 * nr, 300_000, dtype=np.int64)
    res, ref = run(dj, lk, _ids(lk.size), rk, _ids(nr, 1 << 40))
    lone_r = int((_n(res.sides) == dj.SIDE_RIGHT).sum())
    assert lone_r == (0 if matched == "all" else nr)


@pytest.mark.gpu
def test_hot_keys(dj, oracle):
    """20k right copies of a key 500 left rows match (10M pairs, none emitted), 20k copies of a key no left row
    holds (all emitted), and keys whose slots follow the matched hot key's slot."""
    rng = np.random.default_rng(23)
    lk, lp, rk, rp, hot, near, _ = _hot_tables(rng)
    cold = np.int64(0x7EDC_BA98_7654_3210)
    assert not (lk == cold).any() and not (rk == cold).any()
    rk = rng.permutation(np.concatenate([rk, np.full(20_000, cold)]))
    rp = _ids(rk.size, 1 << 40)
    res, ref = run(dj, lk, lp, rk, rp, capacity=20_000 * 500 + lk.size + rk.size)
    sides, rkey = _n(res.sides), _n(res.cols[2])
    assert int(((sides == dj.SIDE_RIGHT) & (rkey == cold)).sum()) == 20_000
    assert not ((sides == dj.SIDE_RIGHT) & (rkey == hot)).any()


@pytest.mark.gpu
@pytest.mark.parametrize("min_key", ["matched", "unmatched"])
def test_edge_words(dj, oracle, min_key):
    """Edge words as keys and payloads; INT64_MIN (the key of the table's side slot) twice on the right, and on
    the left only when it is to be matched."""
    rk, rp, lk, lp = _edge_table(np.random.default_rng([24, len(min_key)]), 2000, 6000)
    rk = np.concatenate([rk, [EMPTY_KEY, EMPTY_KEY]])
    rp = np.concatenate([rp, [0, EMPTY_KEY]])
    keep = lk != EMPTY_KEY
    lk, lp = lk[keep], lp[keep]
    if min_key == "matched":
        lk = np.concatenate([lk, [EMPTY_KEY]])
        lp = np.concatenate([lp, [5]])
    res, _ = run(dj, lk, lp, rk, rp)
    sides, rkey = _n(res.sides), _n(res.cols[2])
    emitted_min = int(((sides == dj.SIDE_RIGHT) & (rkey == EMPTY_KEY)).sum())
    assert emitted_min == (0 if min_key == "matched" else int((rk == EMPTY_KEY).sum()))


@pytest.mark.gpu
@pytest.mark.parametrize("empty,path", [("left", "hash-table"), ("right", "hash-table"), ("both", "hash-table"),
                                        ("left", "radix")])  # no right rows: the hash-table path
def test_empty_tables(dj, oracle, empty, path):
    rng = np.random.default_rng(25)
    nr = 0 if empty != "left" else 3000 if path == "hash-table" else MAX_ROWS + 1
    nl = 0 if empty != "right" else 20_000
    lk, rk = rng.integers(0, 6000, nl, dtype=np.int64), rng.integers(0, 6000, nr, dtype=np.int64)
    lp, rp = _ids(nl), _ids(nr, 1 << 40)
    res, _ = run(dj, lk, lp, rk, rp)
    assert res.n_out == lk.size + rk.size


@pytest.mark.gpu
@pytest.mark.parametrize("boundary", ["left-outer-rows", "emitted-rows"])
@pytest.mark.parametrize("cap_delta", ["n-1", "n", "n+1"])
@pytest.mark.parametrize("path", ["hash-table", "radix"])
def test_capacity_edges(dj, oracle, boundary, cap_delta, path):
    """The count is exact past the capacity, and no column is written past min(count, capacity).  The emitted
    right rows follow the left outer rows, so without unmatched right rows the boundary lies inside the left
    outer rows."""
    rng = np.random.default_rng([26, len(boundary), len(path)])
    nr = 60_000 if path == "hash-table" else MAX_ROWS + 1
    rk = rng.integers(0, nr, nr, dtype=np.int64)
    lk = rng.integers(0, 2 * nr, 100_000, dtype=np.int64)
    if boundary == "left-outer-rows":
        lk = np.concatenate([lk, np.unique(rk)])
    rk[:200] = 7  # a long run too, so that warp-written rows meet the capacity as well
    lk[:50] = 7
    lp, rp = _ids(lk.size), _ids(nr, 1 << 40)
    ref = OO.outer_join(lk, lp, rk, rp, full=True)
    n = ref[0].size
    assert ((ref[4] == OO.SIDE_RIGHT).sum() == 0) == (boundary == "left-outer-rows")
    cap = {"n-1": n - 1, "n": n, "n+1": n + 1}[cap_delta]
    rc, cnt, outs, _, err = raw(dj, lk, lp, rk, rp, cap)
    assert cnt == n
    assert rc == (0 if cap >= n else dj.ERR_OVERFLOW), err
    written = min(cap, n)
    for c in range(5):
        fill = SIDES_SENTINEL if c == 4 else SENTINEL
        assert (outs[c][written:] == fill).all(), f"column {c} written past the rows or the capacity"
    if cap >= n:
        assert_full([o[:n] for o in outs], n, ref)


WS_GUARD_BYTES, WS_GUARD_BYTE = 4096, 0xA5


@pytest.mark.gpu
@pytest.mark.parametrize("nr", [3000, MAX_ROWS + 1], ids=["hash-table", "radix"])
def test_workspace_of_the_queried_size(dj, oracle, nr):
    import torch

    rng = np.random.default_rng([27, nr])
    lk, lp, rk, rp = half_matched(rng, 200_000, nr)
    q = dj.lib().dj_broadcast_full_outer_join_workspace_bytes(lk.size, rk.size, rk.size, 1)
    buf = torch.empty(q + WS_GUARD_BYTES, dtype=torch.uint8, device="cuda")
    buf[q:].fill_(WS_GUARD_BYTE)
    ref = OO.outer_join(lk, lp, rk, rp, full=True)
    cap = ref[0].size
    rc, cnt, outs, _, err = raw(dj, lk, lp, rk, rp, cap, ws=buf[:q], guard=0)
    assert rc == 0, err
    assert bool((buf[q:] == WS_GUARD_BYTE).all()), "the join wrote past the queried workspace"
    assert_full([o[:cnt] for o in outs], cnt, ref)
    rc, _, _, opts, err = raw(dj, lk, lp, rk, rp, cap, ws=buf[:q - 1], guard=0)
    assert rc == dj.ERR_WORKSPACE, err
    assert opts.workspace_needed == q
    rc, cnt, outs, _, err = raw(dj, lk, lp, rk, rp, cap, ws=buf[:opts.workspace_needed], guard=0)
    assert rc == 0, err
    assert_full([o[:cnt] for o in outs], cnt, ref, " (retry)")


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["hash-table", "radix"])
def test_back_to_back_calls_in_one_workspace(dj, oracle, path):
    """Two calls with different tables in one workspace: nothing of the first call's marks or bits remains."""
    nr = 40_000 if path == "hash-table" else MAX_ROWS + 1
    tables = [half_matched(np.random.default_rng([28, i]), 300_000, nr) for i in range(2)]
    tables[1] = (tables[1][0] + nr // 2,) + tables[1][1:]  # other keys matched
    q = max(dj.lib().dj_broadcast_full_outer_join_workspace_bytes(t[0].size, nr, nr, 1) for t in tables)
    ws = dj.workspace(q)
    for i, t in enumerate(tables):
        res = dj.distributed_broadcast_full_outer_join(None, *[_t(a) for a in t], ws=ws)
        assert_full(res.cols, res.n_out, OO.outer_join(*t, full=True), f" (call {i})")


# ------------------------------------------------------------------------------------ variants
VARIANTS = {"shapeB": {"DJ_JOIN_SHAPE": "B"}, "radix-exact": {"DJ_RADIX_EXACT": "1"}}


@pytest.mark.gpu
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_radix_path_variants(dj, variant):
    """The radix-path cases of this module in a fresh process under the variant (the library reads each
    variable once per process)."""
    env = dict(os.environ, PYTHONDONTWRITEBYTECODE="1", **VARIANTS[variant])
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + \
        ["-m", "pytest", "-q", "-x", "-p", "no:cacheprovider", "-m", "gpu", "-k",
         "radix and not variants and not rank_group", __file__]
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0 and " passed" in r.stdout, r.stdout[-4000:] + r.stderr[-2000:]


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
