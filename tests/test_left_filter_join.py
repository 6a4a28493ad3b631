"""Left semi / left anti joins (dj_distributed_left_filter_join_i64), every case against the CPU
oracle (tests/filter_oracle.py), row for row after sorting, for both kinds.

  random tables     duplicates on both sides;
  empty sides       both, left only, right only (anti keeps every left row), through comm NULL;
  edge words        0, +-1, INT64_MIN/MAX and the words around the 32-bit half boundaries as keys;
  multi-job bucket  a right bucket spanning several build jobs -- a 3000-copy hot key, or more
                    distinct keys than one build chunk in one bucket: the probe side is re-streamed
                    per job, so a row's verdict must be carried across the jobs;
  empty buckets     half the buckets empty on the right side: an anti join keeps their left rows;
  tiny right side   20M left rows against 1K right keys, spread over at least one bucket per SM;
  capacity          0 / n-1 / n output rows, exact counts, an untouched guard tail;
  workspace         a workspace of exactly the queried size;
  invariants        semi + anti = the left table, and with unique right keys the semi join equals
                    the inner join's probe-side columns;
  variants          this module again under DJ_JOIN_SHAPE=B and DJ_RADIX_EXACT=1;
  rank groups       N = 2, 3, 4 on one GPU (tests/left_filter_group_worker.py).

Payloads are mix64(base + row) and adversarial keys come from tests/keys.py.
"""
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

import filter_oracle as FO
import keys as K
from test_kernel_edges import BC, GUARD, PC, SENTINEL, SORTED_COMPARE_MAX, _edge_table, _ids, _n, _t, plan_bits

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = os.path.join(ROOT, "tests", "left_filter_group_worker.py")
KINDS = ["semi", "anti"]
FILTER_MIN_BITS = 10  # dj_internal.h kFilterMinBits


def filter_bits(nright):
    """Radix bits of a semi / anti join's plan (api.cu filter_plan)."""
    return max(plan_bits(nright), FILTER_MIN_BITS)


def _kind(dj, kind):
    return dj.JOIN_LEFT_SEMI if kind == "semi" else dj.JOIN_LEFT_ANTI


def _assert_filter(dj, kind, cols, n, lk, lp, rk):
    """n and the rows cols[0..1] equal the oracle's semi / anti join of (lk, lp) against rk."""
    ref = FO.left_semi_join(lk, lp, rk, anti=kind == "anti")
    assert n == ref[0].size, f"{kind}: {n} rows, oracle {ref[0].size}"
    if n <= SORTED_COMPARE_MAX:
        got = [c if isinstance(c, np.ndarray) else _n(c) for c in cols]
        for a, b in zip(FO.O.sort_rows(*got), FO.O.sort_rows(*ref)):
            assert (a == b).all(), f"{kind}: rows differ from the oracle"
    else:
        ck = FO.O.multiset_checksum4 if isinstance(cols[0], np.ndarray) else dj.multiset_checksum4
        assert ck(cols[0], cols[1], cols[0], cols[1]) == \
            FO.O.multiset_checksum4(ref[0], ref[1], ref[0], ref[1]), f"{kind}: checksum differs"
    return ref


def _run(dj, kind, lk, lp, rk, **kw):
    res = dj.distributed_left_filter_join(None, _kind(dj, kind), _t(lk), _t(lp), _t(rk), **kw)
    return _assert_filter(dj, kind, res.cols, res.n_out, lk, lp, rk)


def _raw(dj, kind, lk, lp, rk, cap, ws_bytes=None, guard=GUARD):
    """One call of the C entry (comm NULL) without the binding's retry loop; the outputs carry a
    sentinel guard tail past the capacity."""
    import torch

    L = dj.lib()
    tl, tp, tr = _t(lk), _t(lp), _t(rk)
    if ws_bytes is None:
        ws_bytes = L.dj_distributed_left_filter_join_workspace_bytes(len(lk), len(rk), 1, 1)
    ws = dj.workspace(ws_bytes)
    outs = [torch.full((cap + guard,), SENTINEL, dtype=torch.int64, device="cuda") for _ in range(2)]
    cnt, opts = C.c_int64(-1), dj.JoinOptions(1, 0)
    rc = L.dj_distributed_left_filter_join_i64(None, _kind(dj, kind), tl.data_ptr(), tp.data_ptr(), len(lk),
                                               tr.data_ptr(), len(rk), outs[0].data_ptr(), outs[1].data_ptr(), cap,
                                               C.byref(cnt), C.byref(opts), ws.data_ptr(), ws.numel(), dj._stream())
    torch.cuda.synchronize()
    return rc, cnt.value, [_n(o) for o in outs], (L.dj_last_error().decode() if rc else "")


def _random_tables(rng, nl, nr, key_range):
    lk = rng.integers(0, key_range, nl, dtype=np.int64)
    rk = rng.integers(0, key_range, nr, dtype=np.int64)
    return lk, _ids(nl), rk


# ------------------------------------------------------------------------------------------ oracle
def test_oracle_simulation_matches_owner_restriction(oracle):
    """CPU: the per-rank restatement equals the global semi / anti join restricted to the keys each
    rank owns (partition id % W)."""
    rng = np.random.default_rng(5)
    W, odf = 3, 2
    lefts = [(rng.integers(0, 5000, n, dtype=np.int64), _ids(n, 1000 * r)) for r, n in enumerate((3000, 0, 2500))]
    rights = [rng.integers(0, 5000, n, dtype=np.int64) for n in (1000, 2000, 0)]
    gl = [np.concatenate([t[i] for t in lefts]) for i in range(2)]
    for anti in (False, True):
        sim = FO.simulate_distributed_left_semi_join(lefts, rights, odf, anti)
        ref = FO.left_semi_join(*gl, np.concatenate(rights), anti)
        own = oracle.partition_ids(ref[0], oracle.SEED_NVLINK, W * odf) % W
        for r in range(W):
            for a, b in zip(oracle.sort_rows(*sim[r]), oracle.sort_rows(ref[0][own == r], ref[1][own == r])):
                assert (a == b).all()
        assert sum(s[0].size for s in sim) == ref[0].size


# -------------------------------------------------------------------------------------- GPU cases
@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_random_tables_with_duplicates(dj, oracle, kind):
    rng = np.random.default_rng(1)
    lk, lp, rk = _random_tables(rng, 300_000, 200_000, 400_000)
    assert np.unique(rk).size < rk.size and np.unique(lk).size < lk.size
    ref = _run(dj, kind, lk, lp, rk)
    assert 0 < ref[0].size < lk.size


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("empty", ["both", "left", "right"])
def test_empty_sides(dj, oracle, kind, empty):
    rng = np.random.default_rng(2)
    lk, lp, rk = _random_tables(rng, 0 if empty in ("both", "left") else 50_000,
                                0 if empty in ("both", "right") else 40_000, 100_000)
    ref = _run(dj, kind, lk, lp, rk)
    assert ref[0].size == (lk.size if (kind == "anti" and empty == "right") else 0)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_edge_words(dj, oracle, kind):
    rng = np.random.default_rng(0xE1)
    bk, _, pk, pp = _edge_table(rng, 2000, 6000)
    ref = _run(dj, kind, pk, pp, bk)
    assert ref[0].size > 0


def _multi_job_tables(what, rng):
    """Right keys with one radix bucket spanning several build jobs, and left rows probing it: keys
    of every job of that bucket, several copies each, and misses in the same bucket."""
    nr_fill = 60_000
    if what == "hot-key":
        hot = np.int64(0x0123_4567_89AB_CDEF)
        in_bucket = np.array([hot])
        rk = np.concatenate([np.full(3000, hot), rng.integers(1, 1 << 62, nr_fill, dtype=np.int64)])
        bits = filter_bits(rk.size)
        bucket = int(K.bucket_of(in_bucket, bits)[0])
    else:
        bits = filter_bits(nr_fill + 2 * BC + 200)
        bucket = 5
        pool = K.keys_in_bucket(bits, bucket, 2 * BC + 200 + 4000, rng)
        in_bucket, misses_pool = pool[:2 * BC + 200], pool[2 * BC + 200:]
        rk = np.concatenate([in_bucket, rng.integers(1, 1 << 62, nr_fill, dtype=np.int64)])
    assert bits == filter_bits(rk.size)
    rk = rng.permutation(rk)
    if what == "hot-key":
        misses = K.keys_in_bucket(bits, bucket, 4000, rng)
        misses = misses[~np.isin(misses, rk)]
    else:
        misses = misses_pool[~np.isin(misses_pool, rk)]
    hits = np.repeat(in_bucket, 3) if in_bucket.size > 1 else np.full(40, in_bucket[0])
    lk = np.concatenate([hits, misses, rng.integers(1, 1 << 62, 3 * PC + 50_000, dtype=np.int64)])
    lk = rng.permutation(lk)
    # the bucket really spans several build jobs and its probe side several probe chunks
    assert (K.bucket_of(rk, bits) == bucket).sum() > BC
    assert (K.bucket_of(lk, bits) == bucket).sum() > PC
    return lk, _ids(lk.size, 1 << 40), rk


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("what", ["hot-key", "wide-bucket"])
def test_bucket_spanning_build_jobs(dj, oracle, kind, what):
    rng = np.random.default_rng([3, len(what)])
    lk, lp, rk = _multi_job_tables(what, rng)
    ref = _run(dj, kind, lk, lp, rk)
    assert ref[0].size > 0


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_half_the_buckets_empty_on_the_right(dj, oracle, kind):
    rng = np.random.default_rng(4)
    bits = FILTER_MIN_BITS
    rk = rng.integers(0, 1 << 40, 200_000, dtype=np.int64)
    rk = rk[K.bucket_of(rk, bits) % 2 == 0][:60_000]
    assert filter_bits(rk.size) == bits
    lk = np.concatenate([rng.choice(rk, 100_000), rng.integers(0, 1 << 40, 200_000, dtype=np.int64)])
    lk = rng.permutation(lk)
    lb = K.bucket_of(lk, bits)
    assert np.unique(lb[lb % 2 == 1]).size == (1 << bits) // 2  # every empty right bucket has left rows
    ref = _run(dj, kind, lk, _ids(lk.size), rk)
    if kind == "anti":
        assert ref[0].size >= (lb % 2 == 1).sum()


def _join_grids(trace_path):
    with open(trace_path) as f:
        events = json.load(f)["traceEvents"]
    return [e["args"]["grid"] for e in events
            if e.get("cat") == "kernel" and "bucket_join_kernel" in e.get("name", "")]


@pytest.mark.gpu
def test_tiny_right_side_huge_left_side(dj, oracle):
    """20M left rows against 1K right keys, both kinds: correct, and the join kernel runs at least one
    CTA per SM (its grid is capped at the plan's bucket count, so the plan has at least that many
    buckets).  The grids come from one profiler session for both kinds: a later session in the same
    process may record no kernels."""
    import torch

    rng = np.random.default_rng(6)
    rk = rng.integers(0, 1 << 40, 1000, dtype=np.int64)
    lk = np.concatenate([rng.choice(rk, 2_000_000), rng.integers(0, 1 << 40, 18_000_000, dtype=np.int64)])
    lk = rng.permutation(lk)
    lp = _ids(lk.size)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert (1 << filter_bits(rk.size)) >= sms
    tl, tp, tr = _t(lk), _t(lp), _t(rk)
    for kind in KINDS:  # warm-up: module load, workspace
        dj.distributed_left_filter_join(None, _kind(dj, kind), tl, tp, tr)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        res = {kind: dj.distributed_left_filter_join(None, _kind(dj, kind), tl, tp, tr) for kind in KINDS}
        torch.cuda.synchronize()
    for kind in KINDS:
        _assert_filter(dj, kind, res[kind].cols, res[kind].n_out, lk, lp, rk)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        grids = _join_grids(path)
    assert len(grids) == len(KINDS), grids
    assert all(g[0] >= sms for g in grids), (grids, sms)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("cap_delta", ["0", "n-1", "n"])
def test_capacity_edges(dj, oracle, kind, cap_delta):
    rng = np.random.default_rng(7)
    lk, lp, rk = _random_tables(rng, 100_000, 60_000, 200_000)
    ref = FO.left_semi_join(lk, lp, rk, anti=kind == "anti")
    n = ref[0].size
    cap = {"0": 0, "n-1": n - 1, "n": n}[cap_delta]
    rc, cnt, outs, err = _raw(dj, kind, lk, lp, rk, cap)
    assert cnt == n
    assert rc == (0 if cap == n else dj.ERR_OVERFLOW), err
    for o in outs:
        assert (o[cap:] == SENTINEL).all(), "write past the capacity"
    got = FO.O.sort_rows(outs[0][:cap], outs[1][:cap])
    # the rows written are distinct rows of the result (left payloads are unique)
    assert np.unique(got[1]).size == cap and np.isin(got[1], ref[1]).all()
    ref_by_pay = dict(zip(ref[1].tolist(), ref[0].tolist()))
    assert all(ref_by_pay[p] == k for k, p in zip(got[0].tolist(), got[1].tolist()))


WS_SHAPES = {
    "empty": (0, 0), "left-only": (5000, 0), "right-only": (0, 5000), "random": (300_000, 200_000),
    "hot-key": None, "wide-bucket": None, "tiny-right": (20_000_000, 1000),
}


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("shape", list(WS_SHAPES))
def test_workspace_of_the_queried_size(dj, oracle, kind, shape):
    rng = np.random.default_rng([8, len(shape)])
    if WS_SHAPES[shape] is None:
        lk, lp, rk = _multi_job_tables(shape, rng)
    else:
        nl, nr = WS_SHAPES[shape]
        lk, lp, rk = _random_tables(rng, nl, nr, 4 * max(nl, nr, 1))
    ref = FO.left_semi_join(lk, lp, rk, anti=kind == "anti")
    ws_bytes = dj.lib().dj_distributed_left_filter_join_workspace_bytes(lk.size, rk.size, 1, 1)
    rc, cnt, outs, err = _raw(dj, kind, lk, lp, rk, max(ref[0].size, 1), ws_bytes, guard=0)
    assert rc == 0, err
    _assert_filter(dj, kind, [o[:cnt] for o in outs], cnt, lk, lp, rk)


@pytest.mark.gpu
def test_semi_plus_anti_is_the_left_table_and_semi_matches_inner(dj, oracle):
    rng = np.random.default_rng(9)
    lk, lp, rk = _random_tables(rng, 400_000, 150_000, 500_000)
    tl, tp, tr = _t(lk), _t(lp), _t(rk)
    semi = dj.distributed_left_semi_join(None, tl, tp, tr)
    anti = dj.distributed_left_anti_join(None, tl, tp, tr)
    assert semi.n_out + anti.n_out == lk.size
    both = FO.O.sort_rows(np.concatenate([_n(semi.cols[0]), _n(anti.cols[0])]),
                          np.concatenate([_n(semi.cols[1]), _n(anti.cols[1])]))
    for a, b in zip(both, FO.O.sort_rows(lk, lp)):
        assert (a == b).all()
    # unique right keys: the inner join (right table as its left side) keeps each probe row at most once
    uk = np.unique(rk)
    tu = _t(uk)
    semi_u = dj.distributed_left_semi_join(None, tl, tp, tu)
    inner = dj.distributed_inner_join(None, tu, _t(_ids(uk.size, 1 << 40)), tl, tp)
    assert semi_u.n_out == inner.n_out
    for a, b in zip(FO.O.sort_rows(*[_n(c) for c in semi_u.cols]),
                    FO.O.sort_rows(_n(inner.cols[2]), _n(inner.cols[3]))):
        assert (a == b).all()


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
