"""Left outer / full outer joins (dj_distributed_outer_join_i64), every case against the CPU oracle
(tests/outer_oracle.py), row for row after sorting with `sides` as a fifth column, for both kinds.
Above SORTED_COMPARE_MAX rows, per-class counts and per-class multiset checksums are compared.

  oracle            CPU: the N-rank simulation is the global result restricted to the owned keys,
                    and the three classes of rows are the inner join and the two anti joins;
  random tables     duplicates on both sides;
  empty sides       both, left only, right only, through comm NULL;
  edge words        0, +-1, INT64_MIN/MAX and the words around the 32-bit half boundaries as keys and
                    payloads, plus real (0, 0) rows that must not pass for an absent side;
  multi-job bucket  a right bucket spanning several build jobs -- a 3000-copy hot key, or more
                    distinct keys than one build chunk -- with rows of that bucket unmatched on each
                    side: a probe row's verdict is carried across the jobs, and each job emits its
                    own unmatched build rows;
  empty buckets     half the buckets empty on the right side, and half (a different half) on the left;
  lopsided sides    20M left rows against 1K right rows, and (full outer) 1K against 20M: nearly every
                    bucket then has build rows and no probe rows;
  capacity          0 / n-1 / n / n+1 output rows, exact counts, untouched guard tails on all five
                    columns;
  workspace         a workspace of exactly the queried size, with a sentinel tail behind it;
  repairs           crowded radix children at level 1 and level 2 of each side;
  variants          this module again under DJ_JOIN_SHAPE=B and DJ_RADIX_EXACT=1;
  rank groups       N = 2, 3, 4 on one GPU (tests/outer_group_worker.py).
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import filter_oracle as FO
import keys as K
import outer_oracle as OO
import test_radix_repair as RR
from test_kernel_edges import BC, PC, SENTINEL, SORTED_COMPARE_MAX, _edge_table, _ids, _n, _t
from test_left_filter_join import FILTER_MIN_BITS, _multi_job_tables, filter_bits

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = os.path.join(ROOT, "tests", "outer_group_worker.py")
KINDS = ["left", "full"]
SIDES_SENTINEL = 0xA5  # guard-tail fill of the sides column
GUARD = 1024


def _kind(dj, kind):
    return dj.JOIN_LEFT_OUTER if kind == "left" else dj.JOIN_FULL_OUTER


def _host(cols):
    return [c if isinstance(c, np.ndarray) else _n(c) for c in cols]


def assert_outer(dj, kind, cols, n, lk, lp, rk, rp):
    """n and the 5 columns cols equal the oracle's outer join of (lk, lp) with (rk, rp)."""
    ref = OO.outer_join(lk, lp, rk, rp, full=kind == "full")
    assert n == ref[0].size, f"{kind}: {n} rows, oracle {ref[0].size}"
    if n <= SORTED_COMPARE_MAX:
        got = _host(cols)
        got = got[:4] + [got[4].astype(np.int64)]
        for i, (a, b) in enumerate(zip(FO.O.sort_rows(*got), FO.O.sort_rows(*ref))):
            assert (a == b).all(), f"{kind}: column {i} differs from the oracle"
    else:
        for s in (OO.BOTH, OO.SIDE_LEFT, OO.SIDE_RIGHT):
            want = ref[4] == s
            if isinstance(cols[0], np.ndarray):
                m = cols[4] == s
                got_n, got_ck = int(m.sum()), FO.O.multiset_checksum4(*[c[m] for c in cols[:4]])
            else:
                m = cols[4] == s
                got_n, got_ck = int(m.sum()), dj.multiset_checksum4(*[c[m] for c in cols[:4]])
            assert got_n == int(want.sum()), f"{kind}: {got_n} rows of sides {s}, oracle {int(want.sum())}"
            assert got_ck == FO.O.multiset_checksum4(*[c[want] for c in ref[:4]]), f"{kind}: sides {s} checksum"
    return ref


def _run(dj, kind, lk, lp, rk, rp, **kw):
    res = dj.distributed_outer_join(None, _kind(dj, kind), _t(lk), _t(lp), _t(rk), _t(rp), **kw)
    assert res.sides is not None and len(res.cols) == 5
    return assert_outer(dj, kind, res.cols, res.n_out, lk, lp, rk, rp)


def _raw(dj, kind, lk, lp, rk, rp, cap, ws=None, guard=GUARD):
    """One call of the C entry (comm NULL) without the binding's retry loop; the outputs carry
    sentinel guard tails past the capacity."""
    import torch

    L = dj.lib()
    tl, tp, tr, trp = _t(lk), _t(lp), _t(rk), _t(rp)
    if ws is None:
        ws = dj.workspace(L.dj_distributed_outer_join_workspace_bytes(len(lk), len(rk), 1, 1))
    outs = [torch.full((cap + guard,), SENTINEL, dtype=torch.int64, device="cuda") for _ in range(4)]
    outs.append(torch.full((cap + guard,), SIDES_SENTINEL, dtype=torch.uint8, device="cuda"))
    cnt, opts = C.c_int64(-1), dj.JoinOptions(1, 0)
    rc = L.dj_distributed_outer_join_i64(None, _kind(dj, kind), tl.data_ptr(), tp.data_ptr(), len(lk), tr.data_ptr(),
                                         trp.data_ptr(), len(rk), *[o.data_ptr() for o in outs], cap, C.byref(cnt),
                                         C.byref(opts), ws.data_ptr(), ws.numel(), dj._stream())
    torch.cuda.synchronize()
    return rc, cnt.value, [_n(o) for o in outs], (L.dj_last_error().decode() if rc else "")


def _random_tables(rng, nl, nr, key_range):
    lk = rng.integers(0, key_range, nl, dtype=np.int64)
    rk = rng.integers(0, key_range, nr, dtype=np.int64)
    return lk, _ids(nl), rk, _ids(nr, 1 << 40)


# ------------------------------------------------------------------------------------------ oracle
def test_oracle_simulation_and_classes(oracle):
    """CPU: the per-rank restatement equals the global outer join restricted to the keys each rank
    owns (partition id % W); the sides-3 rows are the C oracle's inner join, the sides-1 rows the anti
    join of left against right, and the sides-2 rows the anti join of right against left."""
    rng = np.random.default_rng(5)
    W, odf = 3, 2
    lefts = [(rng.integers(0, 5000, n, dtype=np.int64), _ids(n, 1000 * r)) for r, n in enumerate((3000, 0, 2500))]
    rights = [(rng.integers(0, 5000, n, dtype=np.int64), _ids(n, 1 << 40 | 1000 * r))
              for r, n in enumerate((1000, 2000, 0))]
    gl = [np.concatenate([t[i] for t in lefts]) for i in range(2)]
    gr = [np.concatenate([t[i] for t in rights]) for i in range(2)]
    for full in (False, True):
        sim = OO.simulate_distributed_outer_join(lefts, rights, odf, full)
        ref = OO.outer_join(*gl, *gr, full)
        own = oracle.partition_ids(OO.row_keys(ref), oracle.SEED_NVLINK, W * odf) % W
        for r in range(W):
            for a, b in zip(oracle.sort_rows(*sim[r]), oracle.sort_rows(*[c[own == r] for c in ref])):
                assert (a == b).all()
        assert sum(s[0].size for s in sim) == ref[0].size
        classes = {s: [c[ref[4] == s] for c in ref[:4]] for s in (OO.BOTH, OO.SIDE_LEFT, OO.SIDE_RIGHT)}
        _, inner = oracle.inner_join(*gl, *gr)
        for a, b in zip(oracle.sort_rows(*classes[OO.BOTH]), oracle.sort_rows(*inner)):
            assert (a == b).all()
        anti_l = FO.left_semi_join(*gl, gr[0], anti=True)
        for a, b in zip(oracle.sort_rows(*classes[OO.SIDE_LEFT][:2]), oracle.sort_rows(*anti_l)):
            assert (a == b).all()
        assert not classes[OO.SIDE_LEFT][2].any() and not classes[OO.SIDE_LEFT][3].any()
        anti_r = FO.left_semi_join(*gr, gl[0], anti=True) if full else (np.empty(0, np.int64),) * 2
        for a, b in zip(oracle.sort_rows(*classes[OO.SIDE_RIGHT][2:]), oracle.sort_rows(*anti_r)):
            assert (a == b).all()
        assert not classes[OO.SIDE_RIGHT][0].any() and not classes[OO.SIDE_RIGHT][1].any()
        assert classes[OO.SIDE_LEFT][0].size > 0 and (classes[OO.SIDE_RIGHT][0].size > 0) == full


# -------------------------------------------------------------------------------------- GPU cases
@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_random_tables_with_duplicates(dj, oracle, kind):
    rng = np.random.default_rng(1)
    lk, lp, rk, rp = _random_tables(rng, 300_000, 200_000, 400_000)
    assert np.unique(rk).size < rk.size and np.unique(lk).size < lk.size
    ref = _run(dj, kind, lk, lp, rk, rp)
    assert (ref[4] == OO.BOTH).any() and (ref[4] == OO.SIDE_LEFT).any()
    assert (ref[4] == OO.SIDE_RIGHT).any() == (kind == "full")


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("empty", ["both", "left", "right"])
def test_empty_sides(dj, oracle, kind, empty):
    rng = np.random.default_rng(2)
    lk, lp, rk, rp = _random_tables(rng, 0 if empty in ("both", "left") else 50_000,
                                    0 if empty in ("both", "right") else 40_000, 100_000)
    ref = _run(dj, kind, lk, lp, rk, rp)
    want = {"both": 0, "right": lk.size, "left": rk.size if kind == "full" else 0}[empty]
    assert ref[0].size == want


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_edge_words(dj, oracle, kind):
    """Edge words as keys and payloads, and real rows (0, 0): two left and one right (a matched pair
    that is all zeros but sides 3), one left (0x55, 0) and one right (0x77, 0) without a match."""
    rng = np.random.default_rng(0xE1)
    bk, bp, pk, pp = _edge_table(rng, 2000, 6000)
    keep_r, keep_l = ~np.isin(bk, [0, 0x55, 0x77]), ~np.isin(pk, [0, 0x55, 0x77])
    lk = np.concatenate([pk[keep_l], [0, 0, 0x55]])
    lp = np.concatenate([pp[keep_l], [0, 0, 0]])
    rk = np.concatenate([bk[keep_r], [0, 0x77]])
    rp = np.concatenate([bp[keep_r], [0, 0]])
    perm_l, perm_r = rng.permutation(lk.size), rng.permutation(rk.size)
    ref = _run(dj, kind, lk[perm_l], lp[perm_l], rk[perm_r], rp[perm_r])
    zero_rows = (ref[0] == 0) & (ref[1] == 0) & (ref[2] == 0) & (ref[3] == 0)
    assert (zero_rows & (ref[4] == OO.BOTH)).sum() == 2
    assert ((ref[0] == 0x55) & (ref[4] == OO.SIDE_LEFT)).sum() == 1
    assert ((ref[2] == 0x77) & (ref[4] == OO.SIDE_RIGHT)).sum() == (kind == "full")


def _multi_job_outer_tables(what, rng):
    """The semi / anti multi-job tables with right payloads; for `wide-bucket`, the left rows of
    every other right key of the crowded bucket are dropped, so that bucket keeps build rows without a
    match in several jobs (the hot-key bucket has some from the spread right keys)."""
    lk, lp, rk = _multi_job_tables(what, rng)
    bits = filter_bits(rk.size)
    rb = K.bucket_of(rk, bits)
    bucket = int(np.bincount(rb).argmax())
    if what == "wide-bucket":
        drop = np.unique(rk[rb == bucket])[::2]
        keep = ~np.isin(lk, drop)
        lk, lp = lk[keep], lp[keep]
    in_l = np.isin(rk[rb == bucket], lk)
    assert in_l.any() and not in_l.all(), "the bucket has matched and unmatched build rows"
    lb = K.bucket_of(lk, bits) == bucket
    assert lb.sum() > PC and (rb == bucket).sum() > BC
    miss = ~np.isin(lk[lb], rk)
    assert miss.any() and not miss.all(), "the bucket has matched and unmatched probe rows"
    return lk, lp, rk, _ids(rk.size, 1 << 50)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("what", ["hot-key", "wide-bucket"])
def test_bucket_spanning_build_jobs(dj, oracle, kind, what):
    rng = np.random.default_rng([3, len(what)])
    lk, lp, rk, rp = _multi_job_outer_tables(what, rng)
    _run(dj, kind, lk, lp, rk, rp)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_half_the_buckets_empty(dj, oracle, kind):
    """Right rows only in even buckets, left rows only in buckets 0 and 1 mod 4: every combination of
    empty and non-empty sides occurs, each in a quarter of the buckets."""
    rng = np.random.default_rng(4)
    bits = FILTER_MIN_BITS
    rk = rng.integers(0, 1 << 40, 200_000, dtype=np.int64)
    rk = rk[K.bucket_of(rk, bits) % 2 == 0][:60_000]
    assert filter_bits(rk.size) == bits
    lk = np.concatenate([rng.choice(rk, 100_000), rng.integers(0, 1 << 40, 400_000, dtype=np.int64)])
    lk = rng.permutation(lk[K.bucket_of(lk, bits) % 4 < 2])
    lb, rb = K.bucket_of(lk, bits), K.bucket_of(rk, bits)
    assert np.unique(lb).size == (1 << bits) // 2 and np.unique(rb).size == (1 << bits) // 2
    ref = _run(dj, kind, lk, _ids(lk.size), rk, _ids(rk.size, 1 << 40))
    assert (ref[4] == OO.SIDE_LEFT).sum() >= (lb % 4 == 1).sum()
    if kind == "full":
        assert (ref[4] == OO.SIDE_RIGHT).sum() >= (rb % 4 == 2).sum()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_tiny_right_side_huge_left_side(dj, oracle, kind):
    rng = np.random.default_rng(6)
    rk = rng.integers(0, 1 << 40, 1000, dtype=np.int64)
    lk = rng.permutation(np.concatenate([rng.choice(rk[:700], 2_000_000),
                                         rng.integers(0, 1 << 40, 18_000_000, dtype=np.int64)]))
    _run(dj, kind, lk, _ids(lk.size), rk, _ids(rk.size, 1 << 40))


@pytest.mark.gpu
def test_full_outer_tiny_left_side_huge_right_side(dj, oracle):
    """1K left rows against 20M right rows: nearly every bucket has build rows and no probe rows, and
    a full outer join must still emit them all."""
    rng = np.random.default_rng(7)
    rk = rng.integers(0, 1 << 40, 20_000_000, dtype=np.int64)
    lk = np.concatenate([rng.choice(rk, 700), rng.integers(0, 1 << 40, 300, dtype=np.int64)])
    ref = _run(dj, "full", lk, _ids(lk.size), rk, _ids(rk.size, 1 << 40))
    assert (ref[4] == OO.SIDE_RIGHT).sum() > 19_000_000


def _sub_multiset5(sub, ref):
    """True when the rows of `sub` (5 int64 columns) form a sub-multiset of the rows of `ref`."""
    a, b = np.stack(ref, 1), np.stack(sub, 1)
    rows = np.ascontiguousarray(np.concatenate([a, b])).view(np.dtype((np.void, 40))).ravel()
    _, inv = np.unique(rows, return_inverse=True)
    inv = inv.ravel()
    m = int(inv.max()) + 1 if inv.size else 0
    return bool((np.bincount(inv[len(a):], minlength=m) <= np.bincount(inv[:len(a)], minlength=m)).all())


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("cap_delta", ["0", "n-1", "n", "n+1"])
def test_capacity_edges(dj, oracle, kind, cap_delta):
    rng = np.random.default_rng(8)
    lk, lp, rk, rp = _random_tables(rng, 100_000, 60_000, 200_000)
    ref = OO.outer_join(lk, lp, rk, rp, full=kind == "full")
    n = ref[0].size
    cap = {"0": 0, "n-1": n - 1, "n": n, "n+1": n + 1}[cap_delta]
    rc, cnt, outs, err = _raw(dj, kind, lk, lp, rk, rp, cap)
    assert cnt == n
    assert rc == (0 if cap >= n else dj.ERR_OVERFLOW), err
    written = min(cap, n)
    for o in outs[:4]:
        assert (o[written:] == SENTINEL).all(), "write past the rows of the result or the capacity"
    assert (outs[4][written:] == SIDES_SENTINEL).all(), "sides written past the rows or the capacity"
    got = [o[:written] for o in outs[:4]] + [outs[4][:written].astype(np.int64)]
    assert _sub_multiset5(got, ref), "rows written are not rows of the result"
    if cap >= n:
        for a, b in zip(FO.O.sort_rows(*got), FO.O.sort_rows(*ref)):
            assert (a == b).all()


WS_SHAPES = {
    "empty": (0, 0), "left-only": (5000, 0), "right-only": (0, 5000), "random": (300_000, 200_000),
    "hot-key": None, "wide-bucket": None, "tiny-right": (20_000_000, 1000),
}
WS_GUARD_BYTES, WS_GUARD_BYTE = 4096, 0xA5


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("shape", list(WS_SHAPES))
def test_workspace_of_the_queried_size(dj, oracle, kind, shape):
    import torch

    rng = np.random.default_rng([9, len(shape)])
    if WS_SHAPES[shape] is None:
        lk, lp, rk, rp = _multi_job_outer_tables(shape, rng)
    else:
        nl, nr = WS_SHAPES[shape]
        lk, lp, rk, rp = _random_tables(rng, nl, nr, 4 * max(nl, nr, 1))
    ref_n = OO.outer_join(lk, lp, rk, rp, full=kind == "full")[0].size
    q = dj.lib().dj_distributed_outer_join_workspace_bytes(lk.size, rk.size, 1, 1)
    buf = torch.empty(q + WS_GUARD_BYTES, dtype=torch.uint8, device="cuda")
    buf[q:].fill_(WS_GUARD_BYTE)
    rc, cnt, outs, err = _raw(dj, kind, lk, lp, rk, rp, max(ref_n, 1), ws=buf[:q], guard=0)
    assert rc == 0, err
    assert bool((buf[q:] == WS_GUARD_BYTE).all()), "the join wrote past the queried workspace"
    assert_outer(dj, kind, [o[:cnt] for o in outs], cnt, lk, lp, rk, rp)


# ---------------------------------------------------------------------------------- radix repairs
NL_REPAIR = 1_000_000
REPAIR_CASES = {  # crowd -> crowded children (side, level, parent, child) given (H1, C2)
    "right-level1": lambda h, c: [("right", 0, 0, h)],
    "right-level2": lambda h, c: [("right", 1, h, c)],
    "left-level1": lambda h, c: [("left", 0, 0, h)],
    "left-level2": lambda h, c: [("left", 1, h, c)],
}


def _repair_tables(crowd, rng):
    """(left keys, right keys, plan, crowded level-1 bucket, crowded child) of a two-level filter plan
    (an outer join's plan) with one side crowded at one level.  The other side hits some of the
    crowded keys, so the crowded bucket holds matched and unmatched rows."""
    b1, b2 = RR.filter_plan(RR.NB)
    assert b2 > 0
    H1, C2 = 6, 9
    side, level = crowd.split("-")
    n = RR.NB if side == "right" else NL_REPAIR
    m1 = n / (1 << b1)
    e1 = int(3 * RR._margin(m1)) if level == "level1" else 0
    e2 = int(3 * RR._margin(m1 / (1 << b2))) if level == "level2" else 0
    crowded, parts = RR._crowded_side(n, b1, b2, H1, C2, e1, e2, rng)
    if side == "right":
        return RR._probe(parts, NL_REPAIR, rng), crowded, (b1, b2), H1, C2
    crowd_keys = parts[1] if e1 else parts[2]
    shared = crowd_keys[: crowd_keys.size // 4]  # some crowded left keys are right keys too
    rk = rng.permutation(np.concatenate([RR._spread(RR.NB - shared.size, rng), shared]))
    lk = rng.permutation(np.concatenate([crowd_keys, parts[0][: NL_REPAIR // 2],
                                         rng.choice(rk, NL_REPAIR - NL_REPAIR // 2 - crowd_keys.size)]))
    return lk, rk, (b1, b2), H1, C2


def test_repair_tables_crowd_what_they_claim():
    """CPU: each repair case's tables pass exactly the capacities the case names."""
    for crowd in REPAIR_CASES:
        lk, rk, (b1, b2), H1, C2 = _repair_tables(crowd, np.random.default_rng([24, len(crowd)]))
        over = RR.tagged(("right",), RR.side_overflows(rk, b1, b2)) + \
            RR.tagged(("left",), RR.side_overflows(lk, b1, b2))
        assert over == REPAIR_CASES[crowd](H1, C2), (crowd, over)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("crowd", list(REPAIR_CASES))
def test_outer_join_repairs(dj, oracle, crowd, kind):
    """One side crowded at one radix level, in a workspace of exactly the queried size with a
    sentinel tail: the repaired buckets' rows (and the left rows' probe bits, indexed by the repaired
    layout) give the oracle's result, and dj_testing_radix_repairs counts the crowded parents."""
    rng = np.random.default_rng([24, len(crowd)])
    lk, rk, (b1, b2), H1, C2 = _repair_tables(crowd, rng)
    over = RR.tagged(("right",), RR.side_overflows(rk, b1, b2)) + RR.tagged(("left",), RR.side_overflows(lk, b1, b2))
    assert over == REPAIR_CASES[crowd](H1, C2), over
    lp, rp = _ids(lk.size), _ids(rk.size, 1 << 40)
    q = dj.lib().dj_distributed_outer_join_workspace_bytes(lk.size, rk.size, 1, 1)
    buf, ws = RR._guarded_workspace(q)
    RR._repairs(dj)
    res = dj.distributed_outer_join(None, _kind(dj, kind), _t(lk), _t(lp), _t(rk), _t(rp), ws=ws)
    assert RR._repairs(dj) == RR.expected_repairs(over)
    RR._assert_guard(buf, q)
    assert_outer(dj, kind, res.cols, res.n_out, lk, lp, rk, rp)


# ---------------------------------------------------------------------------------- variant sweep
VARIANTS = {"shapeB": {"DJ_JOIN_SHAPE": "B"}, "radix-exact": {"DJ_RADIX_EXACT": "1"}}


@pytest.mark.gpu
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_variant_sweep(dj, variant):
    """This module again in a fresh process (the library reads each variant once per process)."""
    env = dict(os.environ, PYTHONDONTWRITEBYTECODE="1", **VARIANTS[variant])
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + \
        ["-m", "pytest", "-q", "-x", "-p", "no:cacheprovider", "-m", "gpu", "-k",
         "not variant_sweep and not rank_group", __file__]
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=3000)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-2000:]
    assert " passed" in r.stdout and " failed" not in r.stdout


# ------------------------------------------------------------------------------------ rank groups
FLAVOURS = {"default": {}, "exchange-fused": {"DJ_EXCHANGE": "fused"}, "no-fuse": {"DJ_NO_FUSE": "1"}}


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3, 4])
@pytest.mark.parametrize("flavour", list(FLAVOURS))
def test_rank_group(dj, flavour, world):
    env = {k: v for k, v in os.environ.items() if k not in ("DJ_EXCHANGE", "DJ_NO_FUSE")}
    env.update(PYTHONDONTWRITEBYTECODE="1", CUDA_DEVICE_MAX_CONNECTIONS="32", **FLAVOURS[flavour])
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [WORKER, str(world)]
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=1200)
    failed = [line for line in r.stdout.splitlines() if line.startswith("FAIL")]
    assert r.returncode == 0 and not failed, "\n".join(failed) + "\n" + r.stdout[-3000:] + r.stderr[-3000:]
    assert f"cases passed (W={world}" in r.stdout
