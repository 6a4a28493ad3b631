"""GPU: the join and partition kernels at the places where they branch on structure, each case
against the CPU oracle (oracle.inner_join / oracle.hash_partition).

  radix plan     one level up to 10 bits, then bits1 = bits/2, bits2 = bits - bits1 (join.cu
                 make_radix_plan): the single-/two-level edge and odd splits (bits1 != bits2);
  skew           one bucket of many DISTINCT keys spanning several build chunks while its probe
                 side re-streams, buckets empty on one side only;
  output tiles   a build job producing tile-1 .. 2*tile+1 matches, and one that spills many tiles;
  slot twins     different keys with the same slot and 20-bit fingerprint in the same bucket, so
                 only the full key comparison separates them;
  capacity       truncated outputs, exact counts, no write past the capacity;
  unaligned      input columns that are offset views (skip_of == 1 in the TMA staging windows);
  streamed host  dj_distributed_inner_join_i64_host with several probe chunks, and its overflow.

The keys are built by inverting the join's hashes (tests/keys.py, pinned by tests/test_keys.py).
Kernel variants chosen by environment variables are covered by re-running this module in a fresh
process (test_variant_sweep), since the library caches each choice for the life of the process.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import keys as K

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# Compile-time CTA shapes of the join kernel (join.cu:48-49, CfgA / CfgB): rows per build chunk,
# rows per probe chunk (one per consumer thread), rows per output tile, planned build rows per bucket.
SHAPES = {
    "A": dict(build_chunk=1792, probe_chunk=992, out_tile=576, target=1536),
    "B": dict(build_chunk=1024, probe_chunk=480, out_tile=256, target=768),
}
SHAPE = SHAPES["B" if os.environ.get("DJ_JOIN_SHAPE", "")[:1] in ("B", "b") else "A"]
BC, PC, OT, TARGET = SHAPE["build_chunk"], SHAPE["probe_chunk"], SHAPE["out_tile"], SHAPE["target"]

SORTED_COMPARE_MAX = 2_000_000  # larger joins: cardinality + multiset checksum
SENTINEL = -0x5A5A5A5A5A5A5A5B  # guard-tail fill


def plan_split(nbuild):
    """(bits1, bits2) of the join's radix plan: join.cu make_radix_plan + api.cu plan_for."""
    bits = 0
    while bits < 20 and (nbuild >> bits) > TARGET:
        bits += 1
    if bits <= 10:
        return max(bits, 1), 0
    return bits // 2, bits - bits // 2


def plan_bits(nbuild):
    return sum(plan_split(nbuild))


MAX_FANOUT = 1024  # dj_internal.h kMaxFanout


def dist_plan(tot_left, tot_right, world, odf, no_fuse=False):
    """(bits1, bits2, sub_bits) of the multi-rank join (comm.cu, after the hello): the plan for the
    estimated build rows per rank and batch; a two-level plan moves up to `fit` level-1 bits into the
    sender's partition (sub_bits) when the rest still fits one level of at most 10 bits."""
    nparts = world * odf
    bits1, bits2 = plan_split(min(tot_left, tot_right) // nparts + 1)
    fit = 0  # largest sub_bits with nparts << sub_bits <= MAX_FANOUT
    while (nparts << (fit + 1)) <= MAX_FANOUT:
        fit += 1
    if bits2 > 0 and fit > 0 and not no_fuse:
        b1 = min(bits1, fit)
        if bits1 + bits2 - b1 <= 10:
            return b1, bits1 + bits2 - b1, b1
    return bits1, bits2, 0


def host_chunks(nprobe):
    """(chunk rows, chunk count) of the streamed host entry (comm.cu streamed_shape)."""
    n = int(os.environ.get("DJ_HOST_CHUNKS", "0") or 0)
    n = n if n > 0 else 16
    chunk = -(-nprobe // n)
    if chunk < (1 << 20):
        chunk = min(nprobe, 1 << 20)
    chunk = max((chunk + 1) // 2 * 2, 2)
    return chunk, max(-(-nprobe // chunk), 1)


def _t(a):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.int64)).cuda()


def _n(t):
    return t.cpu().numpy()


def _ids(n, base=0):
    return np.arange(base, base + n, dtype=np.int64)


def _sub_multiset(sub, ref):
    """True when the rows of `sub` (4 columns) form a sub-multiset of the rows of `ref`."""
    a, b = np.stack(ref, 1), np.stack(sub, 1)
    rows = np.ascontiguousarray(np.concatenate([a, b])).view(np.dtype((np.void, 32))).ravel()
    _, inv = np.unique(rows, return_inverse=True)
    inv = inv.ravel()
    m = int(inv.max()) + 1 if inv.size else 0
    return bool((np.bincount(inv[len(a):], minlength=m) <= np.bincount(inv[:len(a)], minlength=m)).all())


def _assert_rows(dj, oracle, cols, n, ref_n, ref):
    assert n == ref_n
    on_host = isinstance(cols[0], np.ndarray)
    if n <= SORTED_COMPARE_MAX:
        got = [c if on_host else _n(c) for c in cols]
        for a, b in zip(oracle.sort_rows(*got), oracle.sort_rows(*ref)):
            assert (a == b).all()
    else:
        ck = oracle.multiset_checksum4(*cols) if on_host else dj.multiset_checksum4(*cols)
        assert ck == oracle.multiset_checksum4(*ref)


def _swap_sides(cols):
    return cols[2], cols[3], cols[0], cols[1]


# ------------------------------------------------------------------------------------ radix plan
RADIX_CASES = [
    (TARGET, (1, 0)),  # largest single bucket (the plan still makes one level of 2 buckets)
    (TARGET + 1, (1, 0)),
    ((TARGET + 1) * 1024 - 1, (10, 0)),  # largest single-level plan
    ((TARGET + 1) * 1024, (5, 6)),  # smallest two-level plan: odd split, F1 = 32 parents, F2 = 64 children
    ((TARGET + 1) * 4096, (6, 7)),  # odd split with more bits (~6.3M rows with shape A)
]


@pytest.mark.parametrize("nbuild,split", RADIX_CASES, ids=[f"nb{n}-{s[0]}+{s[1]}" for n, s in RADIX_CASES])
def test_radix_plan_edges(dj, oracle, nbuild, split):
    """inner_join and distributed_inner_join(None, ...) with both side orders, at plan edges."""
    assert plan_split(nbuild) == split
    rng = np.random.default_rng(nbuild)
    nprobe = 2 * nbuild + 3  # >= 9/8 of the build side: the single-rank path builds on the smaller side
    bk = rng.integers(0, 2 * nbuild, nbuild, dtype=np.int64)  # duplicates on the build side
    pk = rng.integers(0, 4 * nbuild, nprobe, dtype=np.int64)
    bp, pp = _ids(nbuild), _ids(nprobe, 1 << 40)
    ref_n, ref = oracle.inner_join(bk, bp, pk, pp)
    tb, tbp, tpk, tpp = _t(bk), _t(bp), _t(pk), _t(pp)

    cols, n = dj.inner_join(tb, tbp, tpk, tpp)
    _assert_rows(dj, oracle, cols, n, ref_n, ref)
    del cols
    res = dj.distributed_inner_join(None, tb, tbp, tpk, tpp)  # left is the build side
    _assert_rows(dj, oracle, res.cols, res.n_out, ref_n, ref)
    del res
    res = dj.distributed_inner_join(None, tpk, tpp, tb, tbp)  # right is clearly smaller: built on the right
    _assert_rows(dj, oracle, _swap_sides(res.cols), res.n_out, ref_n, ref)


# ------------------------------------------------------------------------------ distinct-key skew
SKEW_NB = 20_000  # 4-bit plan with shape A (16 buckets), 5-bit with shape B


def _spread(bits, n, skip, rng):
    """n distinct keys spread over every bucket of a `bits`-bit plan except those in `skip`."""
    buckets = [b for b in range(1 << bits) if b not in skip]
    per = np.full(len(buckets), n // len(buckets))
    per[: n % len(buckets)] += 1
    return np.concatenate([K.keys_in_bucket(bits, b, int(c), rng) for b, c in zip(buckets, per)])


@pytest.mark.parametrize("dp", [-1, 0, 1])
@pytest.mark.parametrize("db", [-1, 0, 1])
@pytest.mark.parametrize("k", [1, 2, 5])
def test_skewed_bucket_of_distinct_keys(dj, oracle, k, db, dp):
    """One bucket holds k*build_chunk+db distinct build keys (k build jobs, re-streaming its
    2*probe_chunk+dp probe rows each time); one bucket is empty on the build side only and one on
    the probe side only."""
    bits = plan_bits(SKEW_NB)
    rng = np.random.default_rng(100 * k + 10 * db + dp)
    hot, build_empty, probe_empty = 3, 5, 7
    nhot = k * BC + db
    hot_keys = K.keys_in_bucket(bits, hot, nhot, rng)
    bk = np.concatenate([hot_keys, _spread(bits, SKEW_NB - nhot, {hot, build_empty}, rng)])
    perm = rng.permutation(bk.size)
    bk = bk[perm]
    # probe: the hot bucket gets 2 chunks +dp rows (matches with repeats, plus misses in the same
    # bucket); every other bucket but `probe_empty` gets 64 rows, half of them matches
    nph = 2 * PC + dp
    hot_probe = np.concatenate([rng.choice(hot_keys, nph // 2), K.keys_in_bucket(bits, hot, nph - nph // 2, rng)])
    other = []
    for b in range(1 << bits):
        if b in (hot, probe_empty):
            continue
        mine = bk[K.bucket_of(bk, bits) == b]
        hits = rng.choice(mine, 32) if mine.size else np.empty(0, np.int64)
        other.append(np.concatenate([hits, K.keys_in_bucket(bits, b, 64 - hits.size, rng)]))
    pk = rng.permutation(np.concatenate([hot_probe] + other))
    cb = np.bincount(K.bucket_of(bk, bits), minlength=1 << bits)
    cp = np.bincount(K.bucket_of(pk, bits), minlength=1 << bits)
    assert bk.size == SKEW_NB and plan_bits(bk.size) == bits
    assert cb[hot] == nhot and cb[build_empty] == 0 and cp[build_empty] > 0
    assert cp[hot] == nph and cp[probe_empty] == 0 and cb[probe_empty] > 0
    bp, pp = _ids(bk.size), _ids(pk.size, 1 << 40)
    ref_n, ref = oracle.inner_join(bk, bp, pk, pp)
    cols, n = dj.inner_join(_t(bk), _t(bp), _t(pk), _t(pp))
    _assert_rows(dj, oracle, cols, n, ref_n, ref)


def test_skewed_level2_bucket_in_two_level_plan(dj, oracle):
    """Two-level plan (odd split): a single level-2 bucket of one level-1 bucket holds more than
    three build chunks of distinct keys."""
    nb = (TARGET + 1) * 1024
    bits = plan_bits(nb)
    assert plan_split(nb) == (5, 6)
    rng = np.random.default_rng(77)
    hot = (17 << 6) | 41  # level-1 bucket 17, level-2 bucket 41
    hot_keys = K.keys_in_bucket(bits, hot, 3 * BC + 100, rng)
    bk = rng.permutation(np.concatenate([hot_keys, rng.integers(0, 4 * nb, nb - hot_keys.size, dtype=np.int64)]))
    pk = rng.permutation(np.concatenate([rng.choice(hot_keys, PC + 5), K.keys_in_bucket(bits, hot, PC, rng),
                                         rng.integers(0, 8 * nb, 500_000, dtype=np.int64)]))
    assert (K.bucket_of(bk, bits) == hot).sum() > 3 * BC
    bp, pp = _ids(nb), _ids(pk.size, 1 << 40)
    ref_n, ref = oracle.inner_join(bk, bp, pk, pp)
    cols, n = dj.inner_join(_t(bk), _t(bp), _t(pk), _t(pp))
    _assert_rows(dj, oracle, cols, n, ref_n, ref)


# ----------------------------------------------------------------------------- output tiles/spill
TILE_CASES = [OT - 1, OT, OT + 1, 2 * OT + 1, 40 * OT]


@pytest.mark.parametrize("matches", TILE_CASES, ids=["tile-1", "tile", "tile+1", "2tile+1", "40tiles"])
def test_output_tile_boundaries(dj, oracle, matches):
    """One build job (bucket 0 of a 1-bit plan, one build chunk) producing `matches` rows: the tile
    takes the first out_tile, the rest spill straight to the output.  The last case overflows the
    tile forty times over, so nearly all of its matches take the spill path.  Bucket 1 holds a
    second, small job so that the tile rotation runs too."""
    rng = np.random.default_rng(matches)
    nb0 = min(BC, TARGET) - 24
    b0 = K.keys_in_bucket(1, 0, nb0, rng)
    b1 = K.keys_in_bucket(1, 1, 20, rng)
    bk = np.concatenate([b0, b1])
    assert plan_split(bk.size) == (1, 0)
    hits0 = b0[np.arange(matches) % nb0]  # each build key once before any repeats
    pk = rng.permutation(np.concatenate([hits0, K.keys_in_bucket(1, 0, 700, rng), b1[:10],
                                         K.keys_in_bucket(1, 1, 50, rng)]))
    bp, pp = _ids(bk.size), _ids(pk.size, 1 << 40)
    ref_n, ref = oracle.inner_join(bk, bp, pk, pp)
    assert ref_n == matches + 10
    cols, n = dj.inner_join(_t(bk), _t(bp), _t(pk), _t(pp))
    _assert_rows(dj, oracle, cols, n, ref_n, ref)


# ------------------------------------------------------------------------------- slot-hash twins
TWIN_PLANS = {
    "1bucket": TARGET - 200,  # every key in bucket 0 of the (forced) 1-bit plan
    "10bit": TARGET * 1024 - 1000,
}


def _twin_tables(kind, plan, rng):
    nb = TWIN_PLANS[plan]
    bits = plan_bits(nb)
    ntw = 300 if plan == "1bucket" else 5000
    if plan == "1bucket":
        base = K.keys_in_bucket(1, 0, nb, rng)
    else:
        base = np.unique(rng.integers(-(1 << 62), 1 << 62, nb + 100, dtype=np.int64))[:nb]
        base = rng.permutation(base)
    sub = base[:ntw]
    tw = K.slot_twins(sub, bits, rng)
    miss = rng.integers(1 << 62, (1 << 63) - 1, 2000, dtype=np.int64)
    if kind == "probe_twins":
        # build: keys; probe: each key's twin right next to the key itself (expected: the true matches only)
        bk = base
        pk = np.empty(2 * ntw, np.int64)
        pk[0::2], pk[1::2] = tw, sub
        pk = np.concatenate([pk, miss])
    elif kind == "build_twins":
        # key and twin both in the build table (same cluster, same fingerprint); probe with either
        bk = rng.permutation(np.concatenate([base[: nb - ntw], tw]))
        pk = rng.permutation(np.concatenate([sub[: ntw // 2], tw[ntw // 2:], miss]))
    else:  # "dup_twins": key x3 and twin x2 in the build table, key x2 and twin x1 probing
        reps = ntw // 3
        bk = rng.permutation(np.concatenate([base[: nb - 4 * reps], np.repeat(sub[:reps], 2),
                                             np.repeat(tw[:reps], 2)]))
        pk = rng.permutation(np.concatenate([np.repeat(sub[:reps], 2), tw[:reps], miss]))
    assert plan_bits(bk.size) == bits
    return bk, pk


TWIN_KINDS = ["probe_twins", "build_twins", "dup_twins"]


@pytest.mark.parametrize("plan", list(TWIN_PLANS))
@pytest.mark.parametrize("kind", TWIN_KINDS)
def test_slot_hash_twins(dj, oracle, kind, plan):
    """Different keys with the same 32-bit slot hash (slot and fingerprint) in the same bucket:
    a probe must confirm the key itself, never the fingerprint alone."""
    rng = np.random.default_rng([TWIN_KINDS.index(kind), list(TWIN_PLANS).index(plan)])
    bk, pk = _twin_tables(kind, plan, rng)
    bp, pp = _ids(bk.size), _ids(pk.size, 1 << 40)
    ref_n, ref = oracle.inner_join(bk, bp, pk, pp)
    if kind == "probe_twins":
        assert ref_n == (300 if plan == "1bucket" else 5000)
    cols, n = dj.inner_join(_t(bk), _t(bp), _t(pk), _t(pp))
    _assert_rows(dj, oracle, cols, n, ref_n, ref)


# -------------------------------------------------------------------------------------- capacity
GUARD = 1024


@pytest.mark.parametrize("cap_delta", ["1", "n-1", "n", "n+1"])
def test_capacity_edges(dj, oracle, cap_delta):
    """Output capacity 1, n-1, n, n+1 on a join whose biggest job spills past its tile: the count is
    exact, the retry reproduces the oracle, a truncated first attempt holds a sub-multiset of the
    oracle's rows, and nothing is written past the capacity (guard tail keeps its sentinel)."""
    import torch

    rng = np.random.default_rng(5)
    nb = 3000
    bk = rng.permutation(np.unique(rng.integers(0, 1 << 40, nb + 50, dtype=np.int64))[:nb])
    pk = rng.permutation(np.concatenate([bk, bk[: nb // 2], rng.integers(1 << 41, 1 << 42, 2000, dtype=np.int64)]))
    bp, pp = _ids(nb), _ids(pk.size, 1 << 40)
    ref_n, ref = oracle.inner_join(bk, bp, pk, pp)
    assert ref_n == nb + nb // 2
    cap = {"1": 1, "n-1": ref_n - 1, "n": ref_n, "n+1": ref_n + 1}[cap_delta]
    outs = [torch.full((cap + GUARD,), SENTINEL, dtype=torch.int64, device="cuda") for _ in range(4)]
    cols, n = dj.inner_join(_t(bk), _t(bp), _t(pk), _t(pp), capacity=cap, outs=outs)
    _assert_rows(dj, oracle, cols, n, ref_n, ref)
    first = [_n(o) for o in outs]
    kept = min(cap, ref_n)
    assert _sub_multiset([c[:kept] for c in first], ref)
    for c in first:
        assert (c[kept:] == SENTINEL).all()


# ------------------------------------------------------------------------------ unaligned columns
UNALIGNED_N = [1, 2, 4095, 4096, 4097, 8193]
# which inputs are offset views; hash_partition reads bits 1, 2, 4 as key, payload 0, payload 1
UNALIGNED_MASKS = {"build_key": 1, "build_pay": 2, "probe_key": 4, "probe_pay": 8, "all": 15}
POISON_PAY = -777


def _column(vals, offset, poison):
    """`vals` on the GPU, either as a fresh column or as the view buf[1:n+1] of a buffer whose
    neighbouring words buf[0] and buf[n+1] hold `poison` (skip_of == 1 for the view's first row)."""
    if not offset:
        return _t(vals)
    buf = np.full(vals.size + 2, poison, dtype=np.int64)
    buf[1:-1] = vals
    view = _t(buf)[1:vals.size + 1]
    assert view.data_ptr() % 16 == 8
    return view


@pytest.mark.parametrize("mask", list(UNALIGNED_MASKS))
@pytest.mark.parametrize("n", UNALIGNED_N)
def test_unaligned_input_columns(dj, oracle, n, mask):
    """Offset column views through inner_join, distributed_inner_join(None, ...) and hash_partition
    (one payload column: the TMA kernel; two: the plain scatter).  The words around each view
    hold keys that would match, so a read outside the view shows up as extra or wrong rows."""
    m = UNALIGNED_MASKS[mask]
    rng = np.random.default_rng(n * 31 + m)
    bk = rng.permutation(np.unique(rng.integers(0, 1 << 40, n + 20, dtype=np.int64))[:n])
    nhit = (n + 1) // 2
    miss = rng.integers(1 << 41, 1 << 42, n - nhit, dtype=np.int64)
    pk = rng.permutation(np.concatenate([bk[:nhit], miss]))
    bp, pp = _ids(n, 1 << 20), _ids(n, 1 << 40)
    poison_b = miss[0] if miss.size else np.int64(1 << 43)  # a probe key absent from the build side
    poison_p = bk[-1]  # a build key
    cols_in = [_column(bk, m & 1, poison_b), _column(bp, m & 2, POISON_PAY), _column(pk, m & 4, poison_p),
               _column(pp, m & 8, POISON_PAY)]
    ref_n, ref = oracle.inner_join(bk, bp, pk, pp)

    cols, cnt = dj.inner_join(*cols_in)
    _assert_rows(dj, oracle, cols, cnt, ref_n, ref)
    res = dj.distributed_inner_join(None, *cols_in)
    _assert_rows(dj, oracle, res.cols, res.n_out, ref_n, ref)

    # hash_partition: key = bk, payload 0 = row id, payload 1 = a function of it
    pay1 = bp * 3 + 1
    keys_t = _column(bk, m & 1, poison_b)
    p0 = _column(bp, m & 2, POISON_PAY)
    p1 = _column(pay1, m & 4, POISON_PAY)
    ok, op, ooff = oracle.hash_partition(bk, bp, 8, oracle.SEED_NVLINK)
    for pays in ([p0], [p0, p1]):
        ko, pos, off = dj.hash_partition(keys_t, pays, 8, dj.SEED_NVLINK)
        ko, pos, off = _n(ko), [_n(p) for p in pos], _n(off)
        assert (off == ooff).all()
        for p in range(8):
            assert (np.sort(pos[0][off[p]:off[p + 1]]) == np.sort(op[ooff[p]:ooff[p + 1]])).all()
        assert (ko == bk[pos[0] - (1 << 20)]).all()
        if len(pays) == 2:
            assert (pos[1] == pos[0] * 3 + 1).all()


# --------------------------------------------------------------------------- streamed host entry
STREAM_NB = 200_000


def _host_tables(nprobe, swap, seed):
    """Build side 200K rows with duplicate keys, probe side `nprobe` rows; with `swap` the probe is
    the LEFT table (clearly larger, so the call builds on the right)."""
    rng = np.random.default_rng(seed)
    bk = rng.integers(0, 150_000, STREAM_NB, dtype=np.int64)
    pk = rng.integers(0, 400_000, nprobe, dtype=np.int64)
    bp, pp = _ids(STREAM_NB), _ids(nprobe, 1 << 40)
    return (pk, pp, bk, bp) if swap else (bk, bp, pk, pp)


def _pinned(a):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.int64)).pin_memory()


@pytest.mark.parametrize("swap", [False, True], ids=["build-left", "build-right"])
@pytest.mark.parametrize("nprobe", [(1 << 20) + 1, 3_000_001])
def test_streamed_host_join(dj, oracle, nprobe, swap):
    """Host tables in, host rows out, the probe side uploaded and joined in >= 2 chunks (the last one
    of a single row for 2^20+1 rows); the guard tail of the host output stays untouched."""
    import torch

    assert host_chunks(nprobe)[1] >= 2
    lk, lp, rk, rp = _host_tables(nprobe, swap, nprobe + swap)
    ref_n, ref = oracle.inner_join(lk, lp, rk, rp)
    h_out = [torch.full((ref_n + GUARD,), SENTINEL, dtype=torch.int64).pin_memory() for _ in range(4)]
    n, _ = dj.distributed_inner_join_host(None, *map(_pinned, (lk, lp, rk, rp)), h_out)
    out = [o.numpy() for o in h_out]
    _assert_rows(dj, oracle, [o[:n] for o in out], n, ref_n, ref)
    for o in out:
        assert (o[n:] == SENTINEL).all()


def test_streamed_host_join_repeated(dj, oracle):
    """The same 3-chunk streamed join ten times, every result against the oracle.  A join kernel that
    released a probe stage before its rows had landed in registers miscounted a few percent of such
    calls (the stage's refill raced the copies to the host running next to it); one call rarely shows it."""
    import torch

    lk, lp, rk, rp = _host_tables(3_000_001, False, 3_000_001)
    ref_n, ref = oracle.inner_join(lk, lp, rk, rp)
    ck = oracle.multiset_checksum4(*ref)
    h_in = list(map(_pinned, (lk, lp, rk, rp)))
    h_out = [torch.empty(ref_n + GUARD, dtype=torch.int64).pin_memory() for _ in range(4)]
    for _ in range(10):
        n, _ = dj.distributed_inner_join_host(None, *h_in, h_out)
        assert n == ref_n
        assert oracle.multiset_checksum4(*[o[:n].numpy() for o in h_out]) == ck


@pytest.mark.parametrize("swap", [False, True], ids=["build-left", "build-right"])
def test_streamed_host_join_overflow(dj, oracle, swap):
    """An undersized host output through the C ABI: DJ_ERR_OVERFLOW with the exact count, and the
    first `capacity` host rows (cut inside the second chunk) are a sub-multiset of the oracle's."""
    import torch

    nprobe = 3_000_001
    lk, lp, rk, rp = _host_tables(nprobe, swap, 99 + swap)
    ref_n, ref = oracle.inner_join(lk, lp, rk, rp)
    cap = ref_n * 2 // 3
    chunk = host_chunks(nprobe)[0]
    bk, pk = (rk, lk) if swap else (lk, rk)
    first_chunk_n, _ = oracle.inner_join(bk, bk, pk[:chunk], pk[:chunk], count_only=True)
    assert first_chunk_n < cap < ref_n  # the cut lies inside a later chunk's matches
    h_in = list(map(_pinned, (lk, lp, rk, rp)))
    h_out = [torch.full((cap + GUARD,), SENTINEL, dtype=torch.int64).pin_memory() for _ in range(4)]
    L = dj.lib()
    ws = dj.workspace(L.dj_distributed_inner_join_host_workspace_bytes(len(lk), len(rk), cap, 1, 1))
    cnt = C.c_int64(0)
    opts = dj.JoinOptions(1, 0)
    rc = L.dj_distributed_inner_join_i64_host(None, h_in[0].data_ptr(), h_in[1].data_ptr(), len(lk),
                                              h_in[2].data_ptr(), h_in[3].data_ptr(), len(rk),
                                              *[o.data_ptr() for o in h_out], cap, C.byref(cnt), C.byref(opts),
                                              ws.data_ptr(), ws.numel(), dj._stream())
    torch.cuda.synchronize()
    assert rc == dj.ERR_OVERFLOW, L.dj_last_error()
    assert cnt.value == ref_n
    out = [o.numpy() for o in h_out]
    assert _sub_multiset([o[:cap] for o in out], ref)
    for o in out:
        assert (o[cap:] == SENTINEL).all()


# ---------------------------------------------------------------------------------- variant sweep
# Each variant re-runs (part of) this module in a fresh process.  Subsets:
#   DJ_JOIN_SHAPE=B     every case: the shape table above switches to CfgB's chunk/tile/target sizes
#   DJ_SCATTER_LEAN=0   every case: the join's internal partitioner is scatter_rows_kernel<..., false>
#   DJ_SCATTER=legacy   the cases that call hash_partition with one payload column (scatter_kernel
#                       instead of the TMA kernel): unaligned columns + the hash_partition parity rows
#   DJ_HOST_CHUNKS=2    the streamed host cases (3,000,001 rows then run as 1,500,002 + 1,499,999)
VARIANTS = {
    "shapeB": ({"DJ_JOIN_SHAPE": "B"}, [__file__], None),
    "scatter-lean0": ({"DJ_SCATTER_LEAN": "0"}, [__file__], None),
    "scatter-legacy": ({"DJ_SCATTER": "legacy"},
                       [__file__, os.path.join(ROOT, "tests", "test_gpu_parity.py") + "::test_hash_partition_matches_oracle"],
                       "unaligned or hash_partition"),
    "host-chunks2": ({"DJ_HOST_CHUNKS": "2"}, [__file__], "streamed"),
}


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_variant_sweep(dj, variant):
    env_add, targets, expr = VARIANTS[variant]
    env = dict(os.environ, PYTHONDONTWRITEBYTECODE="1", **env_add)
    k = "not variant_sweep" + (f" and ({expr})" if expr else "")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + \
        ["-m", "pytest", "-q", "-x", "-p", "no:cacheprovider", "-m", "gpu", "-k", k] + targets
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=3000)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-2000:]
    assert " passed" in r.stdout and " failed" not in r.stdout
