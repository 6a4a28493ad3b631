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
  streamed host  dj_distributed_inner_join_i64_host with several probe chunks, and its overflow;
  edge words     0, +-1, INT64_MIN/MAX and the words around the 32-bit half boundaries as keys and
                 payloads, through every join entry, hash_partition and partition_ids;
  single bucket  partition tiles whose rows all go to one bucket (one key, one partition, two
                 partitions alternating), joins with every row in the first or last radix bucket;
  large counts   join counts past 2^31 out of one build job and past 2^32 over many buckets, exact
                 through every entry, with valid, distinct rows below a small capacity;
  checksum       dj_multiset_checksum4 itself, past its grid-stride cap and accumulating.

Every payload is a full-width word (K.mix64 of a row id), so a 32-bit half that is sign-extended
while a row is packed into or unpacked from its int4 form changes the result.
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
    """Payloads of rows base .. base+n-1: full-width words (mix64), decoded with K.unmix64."""
    return K.mix64(np.arange(base, base + n, dtype=np.int64))


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

    # hash_partition: key = bk, payload 0 = mixed row id, payload 1 = a function of it
    pay1 = K.mix64(bp)
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
        assert (ko == bk[K.unmix64(pos[0]) - (1 << 20)]).all()
        if len(pays) == 2:
            assert (pos[1] == K.mix64(pos[0])).all()


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


def _device_join_raw(dj, lk, lp, rk, rp, cap):
    """One dj_distributed_inner_join_i64(NULL, ...) call into guarded device columns.
    Returns (rc, count, the four columns with their guard tails on the host)."""
    import torch

    L = dj.lib()
    t = [_t(a) for a in (lk, lp, rk, rp)]
    outs = [torch.full((cap + GUARD,), SENTINEL, dtype=torch.int64, device="cuda") for _ in range(4)]
    ws = dj.workspace(L.dj_distributed_inner_join_workspace_bytes(len(lk), len(rk), 1, 1))
    cnt, opts = C.c_int64(0), dj.JoinOptions(1, 0)
    rc = L.dj_distributed_inner_join_i64(None, t[0].data_ptr(), t[1].data_ptr(), len(lk), t[2].data_ptr(),
                                         t[3].data_ptr(), len(rk), *[o.data_ptr() for o in outs], cap,
                                         C.byref(cnt), C.byref(opts), ws.data_ptr(), ws.numel(), dj._stream())
    torch.cuda.synchronize()
    return rc, cnt.value, [_n(o) for o in outs]


def _host_join_raw(dj, lk, lp, rk, rp, cap):
    """One streamed dj_distributed_inner_join_i64_host(NULL, ...) call into guarded pinned columns."""
    import torch

    L = dj.lib()
    h_in = list(map(_pinned, (lk, lp, rk, rp)))
    h_out = [torch.full((cap + GUARD,), SENTINEL, dtype=torch.int64).pin_memory() for _ in range(4)]
    ws = dj.workspace(L.dj_distributed_inner_join_host_workspace_bytes(len(lk), len(rk), cap, 1, 1))
    cnt, opts = C.c_int64(0), dj.JoinOptions(1, 0)
    rc = L.dj_distributed_inner_join_i64_host(None, h_in[0].data_ptr(), h_in[1].data_ptr(), len(lk),
                                              h_in[2].data_ptr(), h_in[3].data_ptr(), len(rk),
                                              *[o.data_ptr() for o in h_out], cap, C.byref(cnt), C.byref(opts),
                                              ws.data_ptr(), ws.numel(), dj._stream())
    torch.cuda.synchronize()
    return rc, cnt.value, [o.numpy().copy() for o in h_out]


# ------------------------------------------------------------------------------------ edge words
_M64 = (1 << 64) - 1
EDGE_WORDS = [0, 1, -1, -(1 << 63), (1 << 63) - 1, 0x7FFFFFFF, 0x80000000, 0xFFFFFFFF, 0x7FFFFFFF_80000000,
              0x80000000_00000000, 0x80000000_80000000, 0xFFFFFFFF_00000000]


def _edge_words():
    """Every EDGE_WORDS entry +-3 (64-bit wrap), as distinct int64 words."""
    ws = {((w + d) & _M64) for w in EDGE_WORDS for d in range(-3, 4)}
    return np.array(sorted(ws), dtype=np.uint64).view(np.int64)


def _edge_table(rng, n_pad_build, n_pad_probe):
    """Build and probe tables keyed by the edge words, each word 1-3 times per side (a few on one
    side only), padded with random full-width misses.  The payloads are the edge words again
    (shuffled), then mixed row ids."""
    ew = _edge_words()
    i64 = np.iinfo(np.int64)

    def misses(n):
        m = rng.integers(i64.min, i64.max, n + 64, dtype=np.int64, endpoint=True)
        return m[~np.isin(m, ew)][:n]

    def side(drop, n_pad, base):
        keep = ew[rng.permutation(ew.size)[drop:]]
        k = np.concatenate([np.repeat(keep, rng.integers(1, 4, keep.size)), misses(n_pad)])
        k = rng.permutation(k)
        p = np.concatenate([rng.permutation(ew), _ids(k.size, base)])[:k.size]
        return k, p

    bk, bp = side(3, n_pad_build, 0)
    pk, pp = side(3, n_pad_probe, 1 << 40)
    return bk, bp, pk, pp


def test_extreme_words_join(dj, oracle):
    """Edge words as keys and payloads through inner_join and distributed_inner_join(None, ...) in
    both side orders, row for row against the oracle."""
    rng = np.random.default_rng(0xE0)
    bk, bp, pk, pp = _edge_table(rng, 2000, 6000)
    ref_n, ref = oracle.inner_join(bk, bp, pk, pp)
    assert ref_n > _edge_words().size
    tb, tbp, tpk, tpp = _t(bk), _t(bp), _t(pk), _t(pp)
    cols, n = dj.inner_join(tb, tbp, tpk, tpp)
    _assert_rows(dj, oracle, cols, n, ref_n, ref)
    res = dj.distributed_inner_join(None, tb, tbp, tpk, tpp)
    _assert_rows(dj, oracle, res.cols, res.n_out, ref_n, ref)
    res = dj.distributed_inner_join(None, tpk, tpp, tb, tbp)
    _assert_rows(dj, oracle, _swap_sides(res.cols), res.n_out, ref_n, ref)


@pytest.mark.parametrize("swap", [False, True], ids=["build-left", "build-right"])
def test_streamed_host_join_extreme_words(dj, oracle, swap):
    """The edge-word table through the streamed host entry, its probe side padded past 2^20 rows so
    that the edge rows are spread over at least two probe chunks."""
    rng = np.random.default_rng(0xE1 + swap)
    bk, bp, pk, pp = _edge_table(rng, 2000, (1 << 20) + 4000)
    assert host_chunks(pk.size)[1] >= 2
    lk, lp, rk, rp = (pk, pp, bk, bp) if swap else (bk, bp, pk, pp)
    ref_n, ref = oracle.inner_join(lk, lp, rk, rp)
    rc, n, out = _host_join_raw(dj, lk, lp, rk, rp, ref_n)
    assert rc == 0, dj.lib().dj_last_error()
    _assert_rows(dj, oracle, [o[:n] for o in out], n, ref_n, ref)
    for o in out:
        assert (o[n:] == SENTINEL).all()


def _assert_partitions(oracle, keys, pays, nparts, hid, ko, pos, off):
    """hash_partition's result against the oracle: offsets bit-identical, every partition equal to
    the oracle's as a multiset of whole rows (key and every payload column)."""
    _, oidx, ooff = oracle.hash_partition(keys, np.arange(keys.size, dtype=np.int64), nparts, oracle.SEED_NVLINK, hid)
    assert (off == ooff).all()
    part = np.repeat(np.arange(nparts), np.diff(off))
    got = [ko] + list(pos)
    ref = [keys[oidx]] + [p[oidx] for p in pays]
    og, orf = np.lexsort(got[::-1] + [part]), np.lexsort(ref[::-1] + [part])
    for a, b in zip(got, ref):
        assert (a[og] == b[orf]).all()


@pytest.mark.parametrize("nparts", [8, 100])
def test_hash_partition_extreme_words(dj, oracle, nparts):
    """Edge words as keys and payloads through hash_partition with 1, 2 and 3 payload columns:
    F = 8 ranks warp-aggregated, F = 100 per row."""
    rng = np.random.default_rng(nparts)
    keys, p0, _, _ = _edge_table(rng, 5000, 0)
    pays = [p0, rng.permutation(p0), K.mix64(p0)]
    for npay in (1, 2, 3):
        ko, pos, off = dj.hash_partition(_t(keys), [_t(p) for p in pays[:npay]], nparts, dj.SEED_NVLINK)
        _assert_partitions(oracle, keys, pays[:npay], nparts, dj.HASH_MURMUR3, _n(ko), [_n(p) for p in pos], _n(off))


def test_partition_ids_extreme_words(dj, oracle):
    """partition_ids of the edge words under both hashes (the identity hash keeps the low word only)."""
    w = _edge_words()
    for hid in (dj.HASH_MURMUR3, dj.HASH_IDENTITY):
        for nparts in (8, 100, 1024):
            got = _n(dj.partition_ids(_t(w), dj.SEED_NVLINK, nparts, hid))
            want = oracle.partition_ids(w, oracle.SEED_NVLINK, nparts, hid)
            assert (got == want).all() and (want == oracle.np_partition_ids(w, oracle.SEED_NVLINK, nparts, hid)).all()


# ----------------------------------------------------------------------------- single-bucket tiles
SB_FANOUTS = [2, 32, 33, 1024]
SB_N = [4096, 4097, 32769]  # one full 4096-row tile, one row past it, past the 32768-row histogram tile
SB_DISTS = ["same-key", "last-partition", "last-partition-identity", "alternating"]


def _keys_by_partition(oracle, nparts, hid, want, n, rng):
    """{pid: n distinct random full-width keys whose partition id is pid} for every pid in `want`."""
    i64 = np.iinfo(np.int64)
    found = {p: np.empty(0, np.int64) for p in want}
    while min(v.size for v in found.values()) < n:
        cand = rng.integers(i64.min, i64.max, 1 << 22, dtype=np.int64, endpoint=True)
        pid = oracle.partition_ids(cand, oracle.SEED_NVLINK, nparts, hid)
        for p in want:
            found[p] = np.unique(np.concatenate([found[p], cand[pid == p]]))
    return {p: rng.permutation(v)[:n] for p, v in found.items()}


@pytest.mark.parametrize("nparts", SB_FANOUTS)
@pytest.mark.parametrize("dist", SB_DISTS)
def test_hash_partition_single_bucket_tiles(dj, oracle, dist, nparts):
    """Tiles whose rows all go to one partition (or to two, alternating), with 1-3 payload columns:
    one run per tile in the copy-out, tile ranks up to 4095, and __match_any_sync over warps of one
    or two groups.  Offsets bit-identical, partitions equal as multisets of whole rows."""
    rng = np.random.default_rng([SB_DISTS.index(dist), nparts])
    hid = dj.HASH_IDENTITY if dist.endswith("identity") else dj.HASH_MURMUR3
    nmax = max(SB_N)
    if dist == "same-key":
        pool = np.full(nmax, K.mix64(np.array([nparts]))[0])
    elif dist == "alternating":
        by = _keys_by_partition(oracle, nparts, hid, [0, nparts - 1], nmax, rng)
        pool = np.empty(nmax, np.int64)
        pool[0::2], pool[1::2] = by[0][: (nmax + 1) // 2], by[nparts - 1][: nmax // 2]
    else:
        pool = _keys_by_partition(oracle, nparts, hid, [nparts - 1], nmax, rng)[nparts - 1]
    for n in SB_N:
        keys = pool[:n]
        pays = [_ids(n, c << 40) for c in range(3)]
        pid = oracle.partition_ids(keys, oracle.SEED_NVLINK, nparts, hid)
        if dist == "alternating":
            assert (pid[0::2] == 0).all() and (pid[1::2] == nparts - 1).all()
        else:
            assert (pid == pid[0]).all() and (dist == "same-key" or pid[0] == nparts - 1)
        for npay in (1, 2, 3):
            ko, pos, off = dj.hash_partition(_t(keys), [_t(p) for p in pays[:npay]], nparts, dj.SEED_NVLINK, hid)
            _assert_partitions(oracle, keys, pays[:npay], nparts, hid, _n(ko), [_n(p) for p in pos], _n(off))


SINGLE_BUCKET_PLANS = {
    "1bit": (TARGET, (1, 0)),
    "10bit": ((TARGET + 1) * 1024 - 1, (10, 0)),  # largest single-level plan
    "5+6": ((TARGET + 1) * 1024, (5, 6)),  # smallest two-level plan; last = level-1 31, level-2 63
}


@pytest.mark.parametrize("where", ["first", "last"])
@pytest.mark.parametrize("plan", list(SINGLE_BUCKET_PLANS))
def test_join_single_radix_bucket(dj, oracle, plan, where):
    """Every build and probe row in one radix bucket, the first or the last: distinct build keys
    (one bucket of up to ~900 build jobs), probe rows half hits and half misses of that bucket."""
    nb, split = SINGLE_BUCKET_PLANS[plan]
    assert plan_split(nb) == split
    bits = sum(split)
    bucket = 0 if where == "first" else (1 << bits) - 1
    rng = np.random.default_rng([bits, bucket])
    nhit = min(nb, 2000)
    ks = K.keys_in_bucket(bits, bucket, nb + nhit, rng)  # distinct: the last nhit miss every build key
    bk = ks[:nb]
    pk = rng.permutation(np.concatenate([rng.choice(bk, nhit, replace=False), ks[nb:]]))
    assert (K.bucket_of(bk, bits) == bucket).all() and (K.bucket_of(pk, bits) == bucket).all()
    bp, pp = _ids(nb), _ids(pk.size, 1 << 40)
    ref_n, ref = oracle.inner_join(bk, bp, pk, pp)
    assert ref_n == nhit
    cols, n = dj.inner_join(_t(bk), _t(bp), _t(pk), _t(pp))
    _assert_rows(dj, oracle, cols, n, ref_n, ref)


def test_join_single_key_two_build_jobs(dj, oracle):
    """One key on both sides, build_chunk + 5 build rows (two build jobs of one bucket) x 1000 probe
    rows, plus misses: every pair once, row for row."""
    rng = np.random.default_rng(2)
    key = np.int64(-0x7FFFFFFF_7FFFFFFF)  # 0x80000000_80000001
    bk = rng.permutation(np.concatenate([np.full(BC + 5, key), rng.integers(0, 1 << 62, 50, dtype=np.int64)]))
    pk = rng.permutation(np.concatenate([np.full(1000, key), rng.integers(0, 1 << 62, 300, dtype=np.int64)]))
    assert plan_split(bk.size) == (1, 0)
    bp, pp = _ids(bk.size), _ids(pk.size, 1 << 40)
    ref_n, ref = oracle.inner_join(bk, bp, pk, pp)
    assert ref_n >= (BC + 5) * 1000
    cols, n = dj.inner_join(_t(bk), _t(bp), _t(pk), _t(pp))
    _assert_rows(dj, oracle, cols, n, ref_n, ref)


# ------------------------------------------------------------------------ counts past 2^31 / 2^32
COUNT_CAP = 2_000_000  # output rows actually written: a few million, never the count


def analytic_count(a, b):
    """Matches of an inner join of key columns a and b: the sum over keys of count in a x count in
    b, in Python integers."""
    ua, ca = np.unique(a, return_counts=True)
    ub, cb = np.unique(b, return_counts=True)
    _, ia, ib = np.intersect1d(ua, ub, assume_unique=True, return_indices=True)
    return sum(int(x) * int(y) for x, y in zip(ca[ia], cb[ib]))


def _assert_hot_rows(cols, hot, lk, lbase, rk, rbase):
    """Output rows of a hot-key join: equal keys, each a hot key; each payload decodes (unmix64 minus
    its side's base) to a row of that side holding the key; no (left row, right row) pair twice."""
    k0, p0, k2, p2 = cols
    assert (k0 == k2).all() and np.isin(k0, hot).all()
    rl, rr = K.unmix64(p0) - lbase, K.unmix64(p2) - rbase
    assert ((rl >= 0) & (rl < lk.size)).all() and ((rr >= 0) & (rr < rk.size)).all()
    assert (lk[rl] == k0).all() and (rk[rr] == k2).all()
    assert np.unique(rl * rk.size + rr).size == k0.size


def one_job_tables(nprobe):
    """build_chunk rows of one key against `nprobe` rows of it: all matches in one build job."""
    key = np.int64(-0x7FFFFFFF_7FFFFFFF)
    assert plan_split(BC) == (1, 0)
    return np.full(BC, key), _ids(BC), np.full(nprobe, key), _ids(nprobe, 1 << 40)


ONE_JOB_NPROBE = -(-(1 << 31) // BC) + 3 * PC + 1


def test_join_count_past_2_31_in_one_build_job(dj, oracle):
    """build_chunk x (2^31 / build_chunk + 3 probe chunks + 1) matches, all out of one build job,
    through dj_inner_join_i64 at a capacity of 2M rows: the count is exact, the rows written are
    valid and distinct, nothing lands past the capacity."""
    import torch

    bk, bp, pk, pp = one_job_tables(ONE_JOB_NPROBE)
    want = analytic_count(bk, pk)
    assert want == BC * ONE_JOB_NPROBE > 1 << 31
    L = dj.lib()
    t = [_t(a) for a in (bk, bp, pk, pp)]
    outs = [torch.full((COUNT_CAP + GUARD,), SENTINEL, dtype=torch.int64, device="cuda") for _ in range(4)]
    cnt = torch.zeros(1, dtype=torch.int64, device="cuda")
    ws = dj.workspace(L.dj_inner_join_workspace_bytes(bk.size, pk.size))
    rc = L.dj_inner_join_i64(*[x.data_ptr() for x in t[:2]], bk.size, *[x.data_ptr() for x in t[2:]], pk.size,
                             *[o.data_ptr() for o in outs], COUNT_CAP, cnt.data_ptr(), ws.data_ptr(), ws.numel(),
                             dj._stream())
    assert rc == 0, L.dj_last_error()
    assert int(cnt.item()) == want
    out = [_n(o) for o in outs]
    _assert_hot_rows([o[:COUNT_CAP] for o in out], bk[:1], bk, 0, pk, 1 << 40)
    for o in out:
        assert (o[COUNT_CAP:] == SENTINEL).all()


MANY_BUCKETS_HOT = 32


def many_bucket_tables(total_probe, rng):
    """MANY_BUCKETS_HOT hot keys, one per radix bucket of the build side's plan, build_chunk build
    rows each; `total_probe` probe rows shared evenly among them."""
    k = MANY_BUCKETS_HOT
    bits = plan_bits(k * BC)
    hot = np.concatenate([K.keys_in_bucket(bits, b * (1 << bits) // k, 1, rng) for b in range(k)])
    assert np.unique(K.bucket_of(hot, bits)).size == k
    bk = rng.permutation(np.repeat(hot, BC))
    pk = rng.permutation(np.repeat(hot, -(-total_probe // k)))
    return hot, bk, _ids(bk.size), pk, _ids(pk.size, 1 << 40)


MANY_BUCKETS_NPROBE = -(-(1 << 32) // BC) + MANY_BUCKETS_HOT * PC


def _count_past_2_32(dj, run, swap):
    rng = np.random.default_rng(32 + swap)
    hot, bk, bp, pk, pp = many_bucket_tables(MANY_BUCKETS_NPROBE, rng)
    assert pk.size > 1 << 20
    want = analytic_count(bk, pk)
    assert want > 1 << 32
    lk, lp, rk, rp = (pk, pp, bk, bp) if swap else (bk, bp, pk, pp)
    rc, n, out = run(dj, lk, lp, rk, rp, COUNT_CAP)
    assert rc == dj.ERR_OVERFLOW, dj.lib().dj_last_error()
    assert n == want
    lbase, rbase = (1 << 40, 0) if swap else (0, 1 << 40)
    _assert_hot_rows([o[:COUNT_CAP] for o in out], hot, lk, lbase, rk, rbase)
    for o in out:
        assert (o[COUNT_CAP:] == SENTINEL).all()


@pytest.mark.parametrize("swap", [False, True], ids=["build-left", "build-right"])
def test_join_count_past_2_32_over_buckets(dj, swap):
    """More than 2^32 matches over 32 buckets through dj_distributed_inner_join_i64(NULL, ...):
    DJ_ERR_OVERFLOW with the exact count, valid distinct rows below the capacity."""
    _count_past_2_32(dj, _device_join_raw, swap)


@pytest.mark.parametrize("swap", [False, True], ids=["build-left", "build-right"])
def test_streamed_host_join_count_past_2_32(dj, swap):
    """The same tables through the streamed host entry: the count is summed over >= 2 probe chunks."""
    assert host_chunks(MANY_BUCKETS_NPROBE)[1] >= 2
    _count_past_2_32(dj, _host_join_raw, swap)


# -------------------------------------------------------------------------------------- checksum
def test_multiset_checksum4_matches_oracle(dj, oracle):
    """dj_multiset_checksum4 on random full-width columns: empty, tiny, and one past the grid cap
    (sm_count * 16 blocks of 256 threads) so the grid-stride loop runs; two calls accumulating into
    one result equal the oracle over the concatenated rows."""
    import torch

    cap = torch.cuda.get_device_properties(0).multi_processor_count * 16 * 256
    rng = np.random.default_rng(4)
    i64 = np.iinfo(np.int64)
    for n in (0, 1, 33, cap + 1001):
        cols = [rng.integers(i64.min, i64.max, n, dtype=np.int64, endpoint=True) for _ in range(4)]
        assert dj.multiset_checksum4(*map(_t, cols)) == oracle.multiset_checksum4(*cols)
    t = [_t(c) for c in cols]
    out = torch.zeros(2, dtype=torch.int64, device="cuda")
    L = dj.lib()
    for lo, hi in ((0, 777), (777, n)):
        assert L.dj_multiset_checksum4(*[c[lo:hi].data_ptr() for c in t], hi - lo, out.data_ptr(), dj._stream()) == 0
    a, b = out.tolist()
    assert (a & _M64, b & _M64) == oracle.multiset_checksum4(*cols)
    # the same rows in another order and split: a multiset checksum
    perm = rng.permutation(n)
    assert dj.multiset_checksum4(*[_t(c[perm]) for c in cols]) == oracle.multiset_checksum4(*cols)


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
