"""GPU: the join kernel's consumer groups (join.cu bucket_join_kernel).  A CTA of shape A runs two
groups, and group g takes the valid buckets of even (g = 0) or odd (g = 1) ordinal in the CTA's
range.  Each case is compared with the CPU oracle:

  odd walks         CTA ranges with an odd number of valid buckets, and runs of buckets that are empty
                    on one side, so that the two groups' walks diverge; every join kind;
  multi-job pairs   buckets 0 and 1 (the same CTA, one per group) each spanning several build jobs,
                    with matched and unmatched rows on both sides of every job: semi, anti, left
                    outer, full outer and the streamed full outer (its chunks record matches per row
                    of the right table);
  hot tiles         a hot key in every bucket, so that both groups of every CTA fill their output
                    tiles at once and spill past them.
"""
import os
import subprocess
import sys

import numpy as np
import pytest

import keys as K
import test_host_join_kinds as HK
import test_left_filter_join as LF
import test_outer_join as OJ
import test_radix_repair as RR
from test_kernel_edges import BC, PC, _assert_rows, _ids, _t

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHAPE_B = os.environ.get("DJ_JOIN_SHAPE", "")[:1] in ("B", "b")
KINDS = ["inner", "semi", "anti", "left", "full"]
OUT_TILE = 512 if SHAPE_B else 1024  # rows of a group's output tile (join.cu CfgA / CfgB)


def _bits(kind, nbuild):
    return sum(RR.radix_plan(nbuild) if kind == "inner" else RR.filter_plan(nbuild))


def _cta_ranges(nbuckets):
    """[lo, hi) bucket range of every CTA of the join's grid (join.cu launch_join)."""
    import torch

    grid = min(torch.cuda.get_device_properties(0).multi_processor_count * (2 if SHAPE_B else 1), nbuckets)
    return [(nbuckets * c // grid, nbuckets * (c + 1) // grid) for c in range(grid)]


def _valid(kind, has_build, has_probe):
    """Buckets the kernel walks (join.cu next_valid_bucket)."""
    if kind in ("anti", "left"):
        return has_probe
    if kind == "full":
        return has_build | has_probe
    return has_build & has_probe


def _keys_in(buckets, bits, n, rng):
    """n random keys whose radix buckets are in `buckets`."""
    allowed = np.zeros(1 << bits, bool)
    allowed[buckets] = True
    out = np.empty(0, np.int64)
    while out.size < n:
        k = rng.integers(0, 1 << 62, 4 * n, dtype=np.int64)
        out = np.concatenate([out, k[allowed[K.bucket_of(k, bits)]]])
    return out[:n]


def _check(dj, oracle, kind, lk, lp, rk, rp):
    """The join of kind `kind` of left (lk, lp) with right (rk, rp) against the oracle; the right table
    is the build side of every kind.  Returns the number of result rows."""
    if kind == "inner":
        cols, n = dj.inner_join(_t(rk), _t(rp), _t(lk), _t(lp))
        ref_n, ref = oracle.inner_join(rk, rp, lk, lp)
        _assert_rows(dj, oracle, cols, n, ref_n, ref)
        return n
    if kind in ("semi", "anti"):
        return LF._run(dj, kind, lk, lp, rk)[0].size
    return OJ._run(dj, kind, lk, lp, rk, rp)[0].size


# ------------------------------------------------------------------------------------ odd walks
@pytest.mark.parametrize("kind", KINDS)
def test_odd_walks_and_one_sided_neighbours(dj, oracle, kind):
    """Every bucket is one of: rows on both sides, build rows only, probe rows only, no rows.  Which
    buckets a kind walks differs, and many CTA ranges hold an odd number of them."""
    rng = np.random.default_rng([11, KINDS.index(kind)])
    nbuild = 450_000 if kind == "inner" else 200_000
    bits = _bits(kind, nbuild)
    nb = 1 << bits
    cls = rng.choice(4, nb, p=[0.35, 0.2, 0.2, 0.25])  # 0 both, 1 build only, 2 probe only, 3 none
    has_build, has_probe = (cls == 0) | (cls == 1), (cls == 0) | (cls == 2)
    rk = _keys_in(np.flatnonzero(has_build), bits, nbuild, rng)
    assert _bits(kind, rk.size) == bits
    lk = np.concatenate([rng.choice(rk[has_probe[K.bucket_of(rk, bits)]], 150_000),
                         _keys_in(np.flatnonzero(has_probe), bits, 150_000, rng)])
    lk = rng.permutation(lk)
    # the tables have the bucket classes drawn above
    assert (np.bincount(K.bucket_of(rk, bits), minlength=nb) > 0).tolist() == has_build.tolist()
    assert (np.bincount(K.bucket_of(lk, bits), minlength=nb) > 0).tolist() == has_probe.tolist()
    valid = _valid(kind, has_build, has_probe)
    per_cta = [int(valid[lo:hi].sum()) for lo, hi in _cta_ranges(nb)]
    assert sum(c % 2 for c in per_cta) >= 10, per_cta
    one_sided = (cls == 1) | (cls == 2)
    assert (one_sided[:-1] & one_sided[1:]).sum() >= 10
    assert _check(dj, oracle, kind, lk, _ids(lk.size), rk, _ids(rk.size, 1 << 40)) > 0


# ------------------------------------------------------------------------------ multi-job pairs
def _multi_job_pair(rng, nl):
    """Right rows with buckets 0 and 1 of the filter plan spanning several build jobs each -- bucket 0
    with more distinct keys than two build chunks, bucket 1 with a 3000-copy hot key and a few distinct
    keys -- and left rows: matches of every job of both buckets, and rows of both buckets that match
    nothing."""
    spread = rng.integers(0, 1 << 62, 60_000, dtype=np.int64)
    bits = sum(RR.filter_plan(spread.size + 2 * BC + 3300))
    wide = K.keys_in_bucket(bits, 0, 2 * BC + 200, rng)
    b1 = K.keys_in_bucket(bits, 1, 300, rng)
    hot = b1[:1]
    rk = rng.permutation(np.concatenate([wide, np.repeat(hot, 3000), b1[1:], spread]))
    assert sum(RR.filter_plan(rk.size)) == bits
    rb = K.bucket_of(rk, bits)
    assert (rb == 0).sum() > 2 * BC and (rb == 1).sum() > BC
    strangers = np.concatenate([K.keys_in_bucket(bits, b, 1200, rng) for b in (0, 1)])
    strangers = strangers[~np.isin(strangers, rk)]
    matched = np.concatenate([wide[::3], np.repeat(hot, 40), b1[1::2]])
    filler = rng.integers(0, 1 << 62, nl - matched.size - strangers.size, dtype=np.int64)
    lk = rng.permutation(np.concatenate([matched, strangers, filler]))
    lb = K.bucket_of(lk, bits)
    assert (lb == 0).sum() > PC and (lb == 1).sum() > PC
    assert (_cta_ranges(1 << bits)[0][1]) >= 2  # buckets 0 and 1 are in the same CTA
    return lk, _ids(lk.size), rk, _ids(rk.size, 1 << 40)


@pytest.mark.parametrize("kind", ["semi", "anti", "left", "full"])
def test_multi_job_bucket_in_each_group(dj, oracle, kind):
    lk, lp, rk, rp = _multi_job_pair(np.random.default_rng([12, len(kind)]), 200_000)
    assert _check(dj, oracle, kind, lk, lp, rk, rp) > 0


def test_multi_job_bucket_in_each_group_streamed_full_outer(dj):
    """The host entry's full outer join streams the left table in chunks, each joined by the kernel
    that records matched right rows in a bit per row."""
    nl = (1 << 20) + 50_000
    assert HK.host_chunks(nl)[1] >= 2
    lk, lp, rk, rp = _multi_job_pair(np.random.default_rng(13), nl)
    ref = HK.run_exact(dj, "full", lk, lp, rk, rp)
    assert (ref[4] == OJ.OO.SIDE_RIGHT).any() and (ref[4] == OJ.OO.SIDE_LEFT).any()


# ------------------------------------------------------------------------------------ hot tiles
@pytest.mark.parametrize("kind", ["inner", "semi", "left", "full"])
def test_hot_keys_fill_tiles_in_both_groups(dj, oracle, kind):
    """Every bucket has a key with 2 right and 1100 left copies: a job of any bucket yields more rows
    than one output tile (the semi join: more matching probe rows than one tile), in both groups of
    every CTA at once."""
    rng = np.random.default_rng([14, len(kind)])
    nbuild = 260_000 if kind == "inner" else 60_000
    bits = _bits(kind, nbuild)
    hot = np.concatenate([K.keys_in_bucket(bits, b, 1, rng) for b in range(1 << bits)])
    spread = rng.integers(0, 1 << 62, nbuild - 2 * hot.size, dtype=np.int64)
    rk = rng.permutation(np.concatenate([np.repeat(hot, 2), spread]))
    assert _bits(kind, rk.size) == bits
    lk = rng.permutation(np.concatenate([np.repeat(hot, 1100), rng.choice(spread, 50_000)]))
    assert 1100 > OUT_TILE
    n = _check(dj, oracle, kind, lk, _ids(lk.size), rk, _ids(rk.size, 1 << 40))
    assert n >= hot.size * 1100


# ---------------------------------------------------------------------------------- variant sweep
@pytest.mark.parametrize("variant", ["shapeB"])
def test_variant_sweep(dj, variant):
    """This module again in a fresh process under DJ_JOIN_SHAPE=B (one group per CTA, two CTAs per SM)."""
    env = dict(os.environ, PYTHONDONTWRITEBYTECODE="1", DJ_JOIN_SHAPE="B")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + \
        ["-m", "pytest", "-q", "-x", "-p", "no:cacheprovider", "-m", "gpu", "-k", "not variant_sweep", __file__]
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=3000)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-2000:]
    assert " passed" in r.stdout and " failed" not in r.stdout
