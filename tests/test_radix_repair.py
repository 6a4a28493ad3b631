"""The repair path of the join's bounded radix passes (partition.cu run_bounded_pass) at every site
that runs one, against a Python restatement of the capacity rule.

A bounded pass gives each of a parent's F children a capacity from the parent's row count,
child_capacity(n, F) = floor(m + 8*sqrt(m)) + 32 with m = n / F.  A run that would pass it is dropped
and the parent is flagged; the repair re-scatters the flagged parents with exact offsets.  A repair
does not change results, so every case here also asserts dj_testing_radix_repairs: which level
repaired how many parents.  The expected counts are not literals: side_overflows restates the
capacity rule on the exact keys of the constructed tables, every case first asserts that exactly the
children it crowded pass their capacity, and the expected tuple follows from that list.

  CPU       the capacity rule and bounded_pass_rows, the bound the workspace reserves for a pass's
            output, at adversarial parent sizes; the binomial tail behind every "no repair" case;
  inner     a crowded child of a single-level plan, a crowded level-1 bucket, a crowded level-2
            child, both in one side: each in a workspace of exactly the queried size with a
            sentinel tail behind it;
  streamed  the host entry's resident build side and a crowded probe chunk in the middle;
  filter    left semi / anti with a two-level plan: the right side crowded at level 1, the left at
            level 2, and one key holding most of the right side (hundreds of build jobs in one
            repaired bucket);
  spread    generator tables with duplicates, 16 streamed chunks and a 1K-key semi join: nothing
            repairs;
  variants  this module and test_optimistic_radix.py again under DJ_JOIN_SHAPE=B,
            DJ_SCATTER_LEAN=0 and DJ_RADIX_EXACT=1 (exact histograms: nothing may repair).

The rank-group receivers (the only site where a parent gathers rows from several segments) are
covered by tests/local_group_worker.py and tests/left_filter_group_worker.py, which use the
restatement below through receiver_overflows.
"""
import math
import os
import subprocess
import sys

import numpy as np
import pytest

import keys as K
from test_kernel_edges import MAX_FANOUT, SHAPES, TARGET, dist_plan, host_chunks, plan_split
from test_left_filter_join import FILTER_MIN_BITS, _assert_filter

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXACT = os.environ.get("DJ_RADIX_EXACT") == "1"  # exact histograms: no bounded pass runs
KINDS = ["semi", "anti"]

# ------------------------------------------------------------------------------ the capacity rule
CAP_Z, CAP_MARGIN = 8.0, 32  # partition.cu kCapZ, kCapMargin


def child_capacity(n, F):
    """partition.cu child_capacity: the same double arithmetic (n / F, sqrt, a truncating cast)."""
    mean = np.asarray(n, dtype=np.float64) / F
    return (mean + CAP_Z * np.sqrt(mean)).astype(np.int64) + CAP_MARGIN


def bounded_pass_rows(nrows, P, F):
    """partition.cu bounded_pass_rows: the rows a pass of P parents x F children may lay out."""
    nb = float(P) * F
    return int(nrows) + math.ceil(CAP_Z * math.sqrt(nb * float(nrows))) + int(nb) * (CAP_MARGIN + 1)


def _margin(m):
    """Rows a child of mean m may gain before it passes its capacity (roughly)."""
    return CAP_Z * math.sqrt(m) + CAP_MARGIN


def radix_plan(nbuild, target=TARGET):
    """(bits1, bits2) of the local join's plan: join.cu make_radix_plan + api.cu plan_for."""
    bits = 0
    while bits < 20 and (nbuild >> bits) > target:
        bits += 1
    return (max(bits, 1), 0) if bits <= 10 else (bits // 2, bits - bits // 2)


def filter_plan(nright, target=TARGET):
    """api.cu filter_plan: at least FILTER_MIN_BITS bits, in one level."""
    b1, b2 = radix_plan(nright, target)
    return (b1, b2) if b1 + b2 >= FILTER_MIN_BITS else (FILTER_MIN_BITS, 0)


def dist_radix_plan(tot_left, tot_right, world, odf, no_fuse=False, filter_join=False):
    """(bits1, bits2, sub_bits) the ranks agree on (comm.cu, after the hello): the plan of the
    estimated build rows per rank and batch (the right table for semi / anti), with up to `fit`
    level-1 bits moved into the senders' partition when the rest fits one level of <= 10 bits."""
    nparts = world * odf
    est = (tot_right if filter_join else min(tot_left, tot_right)) // nparts + 1
    b1, b2 = filter_plan(est) if filter_join else radix_plan(est)
    fit = 0
    while (nparts << (fit + 1)) <= MAX_FANOUT:
        fit += 1
    if b2 > 0 and fit > 0 and not no_fuse:
        f = min(b1, fit)
        if b1 + b2 - f <= 10:
            return f, b1 + b2 - f, f
    return b1, b2, 0


def side_overflows(keys, bits1, bits2, level1_done=False):
    """The children of one prepared side that pass their capacity, as (level, parent, child).
    Level 0 has one parent, the whole side (skipped when the senders' partition already ran it:
    level1_done); level 1's parents are level 0's buckets at their exact sizes."""
    keys = np.ascontiguousarray(keys, dtype=np.int64)
    F1, F2 = 1 << bits1, 1 << bits2
    c1 = np.bincount(K.bucket_of(keys, bits1), minlength=F1)
    out = []
    if not level1_done:
        out += [(0, 0, int(c)) for c in np.flatnonzero(c1 > child_capacity(keys.size, F1))]
    if bits2:
        c2 = np.bincount(K.bucket_of(keys, bits1 + bits2), minlength=F1 * F2).reshape(F1, F2)
        over = c2 > child_capacity(c1, F2)[:, None]
        out += [(1, int(p), int(c)) for p, c in zip(*np.nonzero(over))]
    return out


def tagged(tag, over):
    return [tuple(tag) + o for o in over]


def repairs_of(over):
    """(level-1 parents, level-2 parents) a list of tagged overflows repairs: a pass repairs every
    flagged parent once.  Tags name the pass's side (and rank, batch, chunk)."""
    l1 = {o[:-3] for o in over if o[-3] == 0}
    l2 = {o[:-3] + (o[-2],) for o in over if o[-3] == 1}
    return len(l1), len(l2)


def expected_repairs(over, calls=1):
    """What dj_testing_radix_repairs must report after `calls` identical calls."""
    if EXACT:
        return 0, 0
    r1, r2 = repairs_of(over)
    return r1 * calls, r2 * calls


def receiver_overflows(lkeys, rkeys, world, odf, no_fuse=False, filter_join=False):
    """The children over capacity on the receiving ranks of a rank group, as (rank, batch, side,
    level, parent, child), side 0 = left.  lkeys / rkeys: every source rank's keys.  Batch b's
    bucket b*W + r of the murmur3 rank partition goes to rank r; a batch with an empty side is not
    joined.  With a fused level 1 the senders' sub-buckets are the level-2 pass's parents."""
    import oracle as O

    nparts = world * odf
    b1, b2, sub = dist_radix_plan(sum(len(k) for k in lkeys), sum(len(k) for k in rkeys), world, odf, no_fuse,
                                  filter_join)
    pids = [[O.partition_ids(k, O.SEED_NVLINK, nparts) if len(k) else np.empty(0, np.int32) for k in ks]
            for ks in (lkeys, rkeys)]
    out = []
    for q in range(nparts):
        recv = [np.concatenate([k[p == q] for k, p in zip(ks, ps)]) for ks, ps in zip((lkeys, rkeys), pids)]
        if recv[0].size == 0 or recv[1].size == 0:
            continue
        for side, keys in enumerate(recv):
            out += tagged((q % world, q // world, side), side_overflows(keys, b1, b2, level1_done=sub > 0))
    return out


# ------------------------------------------------------------------------------------ CPU checks
PASS_SHAPES = [(1, 2), (1, 32), (1, 1024), (2, 64), (32, 64), (64, 64), (512, 512), (512, 1024)]
TOTALS = [0, 1, 977, 1_000_000, 123_456_789, 400_000_000]


def _parent_vectors(P, n, rng):
    yield "one", np.array([n] + [0] * (P - 1))
    yield "equal", np.full(P, n // P) + (np.arange(P) < n % P)
    yield "zeros", np.zeros(P, np.int64)
    yield "ones", np.ones(P, np.int64)
    w = 0.5 ** np.arange(P)
    geo = np.floor(n * w / w.sum()).astype(np.int64)
    geo[0] += n - geo.sum()
    yield "geometric", geo
    yield "random", rng.multinomial(n, rng.dirichlet(np.ones(P)))


@pytest.mark.parametrize("P,F", PASS_SHAPES, ids=[f"P{p}xF{f}" for p, f in PASS_SHAPES])
def test_capacities_fit_the_reserved_rows(P, F):
    """Σ_p F * child_capacity(n_p, F) <= bounded_pass_rows(Σ n_p, P, F): the laid-out regions of
    any parent sizes stay inside the output array side_ws_bytes reserves."""
    rng = np.random.default_rng([P, F])
    for n in TOTALS:
        for name, sizes in _parent_vectors(P, n, rng):
            sizes = sizes.astype(np.int64)
            laid = int((F * child_capacity(sizes, F)).sum())
            bound = bounded_pass_rows(int(sizes.sum()), P, F)
            assert laid <= bound, (name, n, laid, bound)


def test_region_holds_its_parent():
    """F * child_capacity(n, F) >= n: a repaired parent's exact layout fits its region."""
    rng = np.random.default_rng(11)
    ns = np.concatenate([np.arange(0, 200_000), rng.integers(0, 400_000_001, 200_000),
                         [2**31 - 1, 2**31, 2**32 + 1, 400_000_000]]).astype(np.int64)
    for bits in range(1, 11):
        F = 1 << bits
        assert (F * child_capacity(ns, F) >= ns).all(), F


def test_plan_restatements_agree():
    """radix_plan / dist_radix_plan restate the same plans as test_kernel_edges's helpers."""
    for n in list(range(0, 5000, 7)) + [TARGET << b for b in range(21)] + [(TARGET << b) + 1 for b in range(21)]:
        assert radix_plan(n) == plan_split(n), n
    for world in (2, 3, 4, 8):
        for odf in (1, 2, 4, 17):
            for tot in (0, 4000, 10**6, 3 * 10**6, 7 * 10**6, 10**8, 10**9):
                for no_fuse in (False, True):
                    assert dist_radix_plan(tot, tot + 5000, world, odf, no_fuse) == \
                        dist_plan(tot, tot + 5000, world, odf, no_fuse)


def _side_tail(n, bits1, bits2):
    """Probability that any child of one side passes its capacity when its n keys fall into the
    buckets independently and uniformly (distinct keys under a mixing hash): the exact binomial
    tail summed over all buckets.  Level 2 at both a mean level-1 bucket and the largest one a
    clean level 1 allows."""
    from scipy.stats import binom

    if n == 0:
        return 0.0
    F1, F2 = 1 << bits1, 1 << bits2
    t = F1 * binom.sf(int(child_capacity(n, F1)), n, 1.0 / F1)
    if bits2:
        t += F1 * F2 * max(binom.sf(int(child_capacity(p, F2)), p, 1.0 / F2)
                           for p in (n // F1, int(child_capacity(n, F1))))
    return float(t)


def _zero_repair_shapes(target):
    """(name, plan, side sizes) of every table this suite asserts zero repairs on, plus the
    benchmark's: single-rank sides and, for rank groups, the rows one receiver gets per batch."""
    yield "bench-400m", radix_plan(400_000_000, target), [400_000_000, 400_000_000]
    yield "gen-20m-dups", radix_plan(20_000_000, target), [20_000_000, 20_000_000]
    yield "streamed-16", radix_plan(2_000_000, target), [2_000_000] + [1_250_000] * 16
    yield "semi-1k", filter_plan(1000, target), [20_000_000, 1000]
    yield "clean-2m", radix_plan(2_000_000, target), [2_000_000, 2_500_000]
    for w in (2, 3, 4):
        for nb, np_, odf in ((1_000_000, 1_000_000, 1), (1_000_000, 1_000_000, 4), (500_000, 2_000_000, 2),
                             (4_000, 4_000, 1)):
            est = min(nb, np_) // (w * odf) + 1
            yield f"group-gen-w{w}-odf{odf}", radix_plan(est, target), [nb // (w * odf), np_ // (w * odf)]
        tot = (target + 1) * 1024 * w * 11 // 10
        yield f"group-two-level-w{w}", radix_plan(tot // w + 1, target), [tot // w, tot // w]


@pytest.mark.parametrize("shape", list(SHAPES))
def test_binomial_tail_of_zero_repair_shapes(shape):
    """Every "no repair" assertion of the suite, and the benchmark's 400M x 400M join, rests on a
    summed binomial tail below 1e-9 (the seeds are fixed anyway, so each such case is
    deterministic)."""
    target = SHAPES[shape]["target"]
    for name, (b1, b2), sides in _zero_repair_shapes(target):
        tail = sum(_side_tail(n, b1, b2) for n in sides)
        assert tail < 1e-9, (name, b1, b2, tail)


# ------------------------------------------------------------------------------------- GPU helpers
NB = 2_000_000  # a two-level plan under either join shape
GUARD_BYTES = 4096
GUARD_BYTE = 0xA5


def _repairs(dj):
    """Repairs per level since the last read (a device counter; the read synchronises and resets)."""
    import ctypes as C

    out = (C.c_int64 * 2)()
    assert dj.lib().dj_testing_radix_repairs(out) == 0
    return out[0], out[1]


def _t(a):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.int64)).cuda()


def _ids(n, base=0):
    return K.mix64(np.arange(base, base + n, dtype=np.int64))


def _spread(n, rng):
    return rng.integers(-(1 << 62), 1 << 62, n, dtype=np.int64)


def _crowded_side(n, bits1, bits2, parent, child, extra1, extra2, rng):
    """n keys: `extra1` spread over level-1 bucket `parent`, `extra2` in its level-2 child `child`,
    the rest spread by the hash.  Returns (keys, [spread part, level-1 crowd, child crowd])."""
    parts = [_spread(n - extra1 - extra2, rng),
             K.keys_in_bucket(bits1, parent, extra1, rng) if extra1 else np.empty(0, np.int64),
             K.keys_in_bucket(bits1 + bits2, (parent << bits2) | child, extra2, rng) if extra2
             else np.empty(0, np.int64)]
    return rng.permutation(np.concatenate(parts)), parts


def _probe(parts, n, rng, crowd_hits=100):
    """n probe keys: half hits (spread build keys, and up to `crowd_hits` of each crowd), half misses."""
    crowd = [rng.choice(p, min(crowd_hits, p.size), replace=False) for p in parts[1:] if p.size]
    nc = sum(c.size for c in crowd)
    hits = np.concatenate([rng.choice(parts[0], n // 2 - nc)] + crowd)
    return rng.permutation(np.concatenate([hits, _spread(n - hits.size, rng)]))


def _guarded_workspace(nbytes):
    """A workspace of exactly `nbytes` with a sentinel tail behind it: (whole buffer, workspace view)."""
    import torch

    buf = torch.empty(nbytes + GUARD_BYTES, dtype=torch.uint8, device="cuda")
    buf[nbytes:].fill_(GUARD_BYTE)
    return buf, buf[:nbytes]


def _assert_guard(buf, nbytes):
    import torch

    torch.cuda.synchronize()
    assert bool((buf[nbytes:] == GUARD_BYTE).all()), "a pass wrote past the queried workspace"


def _assert_rows(oracle, n, cols, ref_n, ref):
    assert n == ref_n
    got = [c.cpu().numpy() if hasattr(c, "cpu") else c for c in cols]
    if n <= 2_000_000:
        for a, b in zip(oracle.sort_rows(*got), oracle.sort_rows(*ref)):
            assert (a == b).all()
    else:
        assert oracle.multiset_checksum4(*got) == oracle.multiset_checksum4(*ref)


# --------------------------------------------------------------------------- single-rank inner join
INNER_CASES = {  # crowd -> (build rows, crowd level 1, crowd level 2)
    "single-level": (200_000, True, False),
    "level1": (NB, True, False),
    "level2": (NB, False, True),
    "both": (NB, True, True),
}


@pytest.mark.gpu
@pytest.mark.parametrize("crowd", list(INNER_CASES))
def test_inner_join_repair_in_exact_workspace(dj, oracle, crowd):
    """One crowded build side through dj_inner_join_i64, in a workspace of exactly the queried size
    followed by a sentinel tail: a repair must stay inside its parent's region.  `both` crowds a
    level-1 bucket and, inside it, a child beyond the capacity computed from that bucket's exact
    size, so one side repairs at both levels in one call."""
    nb, c1, c2 = INNER_CASES[crowd]
    b1, b2 = radix_plan(nb)
    assert (b2 == 0) == (crowd == "single-level")
    H1, C2 = (1 << b1) - 3, 5
    rng = np.random.default_rng([21, len(crowd)])
    m1 = nb / (1 << b1)
    e1 = int(3 * _margin(m1)) if c1 else 0
    e2 = int(3 * _margin((m1 + e1) / (1 << b2))) if c2 else 0
    bk, parts = _crowded_side(nb, b1, b2, H1, C2, e1, e2, rng)
    pk = _probe(parts, nb, rng)
    over = tagged(("build",), side_overflows(bk, b1, b2)) + tagged(("probe",), side_overflows(pk, b1, b2))
    assert over == [("build", 0, 0, H1)] * c1 + [("build", 1, H1, C2)] * c2, over
    bp, pp = _ids(bk.size), _ids(pk.size, 1 << 40)
    ref_n, ref = oracle.inner_join(bk, bp, pk, pp)
    q = dj.lib().dj_inner_join_workspace_bytes(bk.size, pk.size)
    buf, ws = _guarded_workspace(q)
    _repairs(dj)
    cols, n = dj.inner_join(_t(bk), _t(bp), _t(pk), _t(pp), capacity=max(ref_n, 1), ws=ws)
    assert _repairs(dj) == expected_repairs(over)
    _assert_guard(buf, q)
    _assert_rows(oracle, n, cols, ref_n, ref)


# ------------------------------------------------------------------------------ streamed host entry
NP_STREAM = 3 * (1 << 20) + (1 << 19)


@pytest.mark.gpu
@pytest.mark.parametrize("build", ["spread", "level1"])
def test_streamed_repairs(dj, oracle, build):
    """dj_distributed_inner_join_i64_host: the build side is prepared once with its plan and every
    probe chunk with the same plan.  The middle chunk has a level-2 child past the capacity of its
    own level-1 bucket; with `level1` the resident build side is crowded at level 1 as well."""
    import torch

    chunk, nchunks = host_chunks(NP_STREAM)
    assert nchunks >= 3
    mid = nchunks // 2
    b1, b2 = radix_plan(NB)
    assert b2 > 0
    H1, C2 = 11, (1 << b2) - 2
    rng = np.random.default_rng([22, len(build)])
    e1 = int(3 * _margin(NB / (1 << b1))) if build == "level1" else 0
    bk, parts = _crowded_side(NB, b1, b2, H1, 0, e1, 0, rng)
    chunks, over = [], tagged(("build",), side_overflows(bk, b1, b2))
    for c in range(nchunks):
        n = min(chunk, NP_STREAM - c * chunk)
        e2 = int(3 * _margin(n / (1 << (b1 + b2)))) if c == mid else 0
        ck = _probe([parts[0]], n - e2, rng)
        if e2:
            ck = rng.permutation(np.concatenate([ck, K.keys_in_bucket(b1 + b2, (H1 << b2) | C2, e2, rng)]))
        chunks.append(ck)
        over += tagged(("chunk", c), side_overflows(ck, b1, b2))
    assert over == [("build", 0, 0, H1)] * (build == "level1") + [("chunk", mid, 1, H1, C2)], over
    pk = np.concatenate(chunks)
    bp, pp = _ids(bk.size), _ids(pk.size, 1 << 40)
    ref_n, ref = oracle.inner_join(bk, bp, pk, pp)
    h_in = [torch.from_numpy(a).pin_memory() for a in (bk, bp, pk, pp)]
    h_out = [torch.empty(ref_n + 16, dtype=torch.int64).pin_memory() for _ in range(4)]
    _repairs(dj)
    n, _ = dj.distributed_inner_join_host(None, *h_in, h_out)
    assert _repairs(dj) == expected_repairs(over)
    _assert_rows(oracle, n, [o[:n].numpy() for o in h_out], ref_n, ref)


# ------------------------------------------------------------------------------ left semi / anti
NL_FILTER = 1_000_000
HOT_COPIES = 1_500_000


def _filter_tables(crowd, rng):
    """(left keys, right keys, plan, crowded level-1 bucket, crowded child) of a two-level filter plan."""
    b1, b2 = filter_plan(NB)
    assert b2 > 0
    H1, C2 = 6, 9
    if crowd == "right-level1":
        e1 = int(3 * _margin(NB / (1 << b1)))
        rk, parts = _crowded_side(NB, b1, b2, H1, C2, e1, 0, rng)
        lk = _probe(parts, NL_FILTER, rng)
    elif crowd == "left-level2":
        e2 = int(3 * _margin(NL_FILTER / (1 << (b1 + b2))))
        lk, lparts = _crowded_side(NL_FILTER, b1, b2, H1, C2, 0, e2, rng)
        shared = lparts[2][: e2 // 4]  # some crowded left keys are right keys too
        rk = rng.permutation(np.concatenate([_spread(NB - shared.size, rng), shared]))
        lk = rng.permutation(np.concatenate([lparts[2], lparts[0][: NL_FILTER // 2],
                                             rng.choice(rk, NL_FILTER - NL_FILTER // 2 - e2)]))
    else:  # hot-key: one key holds most of the right side
        hot = K.keys_in_bucket(b1 + b2, (H1 << b2) | C2, 1, rng)
        spread = _spread(NB - HOT_COPIES, rng)
        rk = rng.permutation(np.concatenate([np.repeat(hot, HOT_COPIES), spread]))
        misses = K.keys_in_bucket(b1 + b2, (H1 << b2) | C2, 60, rng)
        misses = misses[~np.isin(misses, rk)]
        lk = np.concatenate([np.repeat(hot, 20), misses, rng.choice(spread, NL_FILTER // 3)])
        lk = rng.permutation(np.concatenate([lk, _spread(NL_FILTER - lk.size, rng)]))
    return lk, rk, (b1, b2), H1, C2


FILTER_EXPECT = {  # crowd -> crowded children (side, level, parent, child) given (H1, C2)
    "right-level1": lambda h, c: [("right", 0, 0, h)],
    "left-level2": lambda h, c: [("left", 1, h, c)],
    "hot-key": lambda h, c: [("right", 0, 0, h), ("right", 1, h, c)],
}


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("crowd", list(FILTER_EXPECT))
def test_filter_join_repairs(dj, oracle, crowd, kind):
    """Semi / anti with a two-level plan (the right side's, more than 1024 target-sized buckets), in
    a workspace of exactly the queried size.  `hot-key`: 1.5M of the 2M right rows share one key, so
    the right side repairs at both levels and the repaired bucket is hundreds of build jobs long;
    the left rows' filter bits are carried over all of them, indexed by positions in the repaired
    layout."""
    rng = np.random.default_rng([23, len(crowd)])
    lk, rk, (b1, b2), H1, C2 = _filter_tables(crowd, rng)
    over = tagged(("right",), side_overflows(rk, b1, b2)) + tagged(("left",), side_overflows(lk, b1, b2))
    assert over == FILTER_EXPECT[crowd](H1, C2), over
    lp = _ids(lk.size)
    q = dj.lib().dj_distributed_left_filter_join_workspace_bytes(lk.size, rk.size, 1, 1)
    buf, ws = _guarded_workspace(q)
    _repairs(dj)
    res = dj.distributed_left_filter_join(None, dj.JOIN_LEFT_SEMI if kind == "semi" else dj.JOIN_LEFT_ANTI,
                                          _t(lk), _t(lp), _t(rk), ws=ws)
    assert _repairs(dj) == expected_repairs(over)
    _assert_guard(buf, q)
    ref = _assert_filter(dj, kind, res.cols, res.n_out, lk, lp, rk)
    assert 0 < ref[0].size < lk.size


# ------------------------------------------------------------------------------ spread data: none
@pytest.mark.gpu
def test_generated_20m_with_duplicates_repairs_nothing(dj, oracle):
    """The benchmark's generator at 20M x 20M with duplicate build keys and selectivity 0.9."""
    n = 20_000_000
    g = dj.gen_params(n, n, 0.9, 2 * n, False)
    bk, bp = dj.generate_rows(g, 0, 0, 0, n)
    pk, pp = dj.generate_rows(g, 1, 0, 0, n)
    go = oracle.gen_params(n, n, 0.9, 2 * n, False)
    obk, obp, _ = oracle.generate_rows(go, 0, 0, 0, n)
    opk, opp, _ = oracle.generate_rows(go, 1, 0, 0, n)
    assert np.unique(obk).size < n  # duplicates
    b1, b2 = radix_plan(n)
    over = tagged(("build",), side_overflows(obk, b1, b2)) + tagged(("probe",), side_overflows(opk, b1, b2))
    assert over == []
    _repairs(dj)
    res = dj.distributed_inner_join(None, bk, bp, pk, pp)
    assert _repairs(dj) == (0, 0)
    ref_n, ref = oracle.inner_join(obk, obp, opk, opp)
    assert res.n_out == ref_n
    assert dj.multiset_checksum4(*res.cols) == oracle.multiset_checksum4(*ref)


@pytest.mark.gpu
def test_streamed_16_chunks_repair_nothing(dj, oracle):
    """A 20M-row probe side streamed in 16 chunks against a resident 2M-row build side."""
    import torch

    np_ = 20_000_000
    chunk, nchunks = host_chunks(np_)
    rng = np.random.default_rng(24)
    bk = _spread(NB, rng)
    pk = rng.permutation(np.concatenate([rng.choice(bk, np_ // 10), _spread(np_ - np_ // 10, rng)]))
    b1, b2 = radix_plan(NB)
    over = tagged(("build",), side_overflows(bk, b1, b2))
    for c in range(nchunks):
        over += tagged(("chunk", c), side_overflows(pk[c * chunk:(c + 1) * chunk], b1, b2))
    assert over == []
    bp, pp = _ids(bk.size), _ids(pk.size, 1 << 40)
    ref_n, ref = oracle.inner_join(bk, bp, pk, pp)
    h_in = [torch.from_numpy(a).pin_memory() for a in (bk, bp, pk, pp)]
    h_out = [torch.empty(ref_n + 16, dtype=torch.int64).pin_memory() for _ in range(4)]
    _repairs(dj)
    n, _ = dj.distributed_inner_join_host(None, *h_in, h_out)
    assert _repairs(dj) == (0, 0)
    _assert_rows(oracle, n, [o[:n].numpy() for o in h_out], ref_n, ref)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_semi_20m_against_1k_keys_repairs_nothing(dj, oracle, kind):
    """20M left rows against 1K right keys: the right side has less than one row per bucket."""
    rng = np.random.default_rng(25)
    rk = _spread(1000, rng)
    lk = rng.permutation(np.concatenate([rng.choice(rk, 200_000), _spread(19_800_000, rng)]))
    b1, b2 = filter_plan(rk.size)
    over = tagged(("right",), side_overflows(rk, b1, b2)) + tagged(("left",), side_overflows(lk, b1, b2))
    assert over == []
    lp = _ids(lk.size)
    _repairs(dj)
    res = dj.distributed_left_filter_join(None, dj.JOIN_LEFT_SEMI if kind == "semi" else dj.JOIN_LEFT_ANTI,
                                          _t(lk), _t(lp), _t(rk))
    assert _repairs(dj) == (0, 0)
    _assert_filter(dj, kind, res.cols, res.n_out, lk, lp, rk)


# ---------------------------------------------------------------------------------- variant sweep
# This module and test_optimistic_radix.py again in a fresh process (the library reads each
# variable once per process): shape B's plans (one more radix bit at these sizes), the non-lean
# scatter (its own drop-and-flag copy-out), and exact histograms (expected repairs become (0, 0)).
SWEEPS = {"shapeB": {"DJ_JOIN_SHAPE": "B"}, "scatter-lean0": {"DJ_SCATTER_LEAN": "0"},
          "radix-exact": {"DJ_RADIX_EXACT": "1"}}


@pytest.mark.gpu
@pytest.mark.parametrize("variant", list(SWEEPS))
def test_variant_sweep(dj, variant):
    env = dict(os.environ, PYTHONDONTWRITEBYTECODE="1", **SWEEPS[variant])
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + \
        ["-m", "pytest", "-q", "-x", "-p", "no:cacheprovider", "-m", "gpu", "-k",
         "not variant_sweep and not kernel_edges_with_exact_histograms", __file__,
         os.path.join(ROOT, "tests", "test_optimistic_radix.py")]
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=3000)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-2000:]
    assert " passed" in r.stdout and " failed" not in r.stdout
