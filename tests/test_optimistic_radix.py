"""The join's bounded radix passes (partition.cu run_bounded_pass): every child bucket gets a capacity
from its parent's row count instead of an exact histogram, and a parent whose child outgrew its
capacity is repaired (re-scattered with exact offsets).  Keys built by inverting the radix hash
(tests/keys.py) force each kind of overflow; every result is compared row for row with the oracle,
and dj_testing_radix_repairs says which level repaired how many parents.

The plan of a 2M-row build side is two levels: 5 + 6 bits under shape A (1536-row buckets, 32
level-1 parents of ~62K rows, each split into 64 children of ~1K rows), 6 + 6 under shape B.  The
plans come from the restatement in test_radix_repair.py, so the module runs under either shape;
under DJ_RADIX_EXACT=1 (exact histograms) every case expects no repair and the same rows.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import keys as K
from test_radix_repair import expected_repairs, radix_plan, side_overflows, tagged

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NB = 2_000_000
BITS1, BITS2 = radix_plan(NB)  # level 1 = the top BITS1 bits of the local hash, level 2 = the next BITS2
BITS = BITS1 + BITS2
HOT1 = 19  # the level-1 bucket the adversarial tables crowd


def _want(bk, pk, literal):
    """The repairs of one join of bk with pk: derived from the capacity restatement, which must
    agree with the count the case was built for."""
    over = tagged(("build",), side_overflows(bk, BITS1, BITS2)) + tagged(("probe",), side_overflows(pk, BITS1, BITS2))
    assert expected_repairs(over) == ((0, 0) if os.environ.get("DJ_RADIX_EXACT") == "1" else literal), over
    return expected_repairs(over)


def _repairs(dj):
    out = (C.c_int64 * 2)()
    assert dj.lib().dj_testing_radix_repairs(out) == 0
    return out[0], out[1]


def _t(a):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.int64)).cuda()


def _ids(n, base=0):
    return K.mix64(np.arange(base, base + n, dtype=np.int64))


def _crowded(n, rng, share=0.7):
    """n distinct keys, `share` of them in level-1 bucket HOT1, the rest spread by the hash."""
    hot = K.keys_in_bucket(BITS1, HOT1, int(n * share), rng)
    rest = rng.integers(-(1 << 62), 1 << 62, n - hot.size, dtype=np.int64)
    return rng.permutation(np.concatenate([hot, rest]))


def _probe_for(bk, n, rng, crowd, bits=BITS1, hot=HOT1):
    """n probe keys, half of them drawn from the build keys.  crowd: the misses crowd level-1 bucket
    HOT1.  Otherwise the misses are spread and radix bucket `hot` of a `bits`-bit plan gets its fair
    share of the hits, however crowded it is on the build side."""
    nh = n // 2
    if crowd:
        return rng.permutation(np.concatenate([rng.choice(bk, nh), _crowded(n - nh, rng, share=0.9)]))
    in_hot = K.bucket_of(bk, bits) == hot
    hh = nh >> bits
    hits = np.concatenate([rng.choice(bk[in_hot], hh), rng.choice(bk[~in_hot], nh - hh)])
    return rng.permutation(np.concatenate([hits, rng.integers(-(1 << 62), 1 << 62, n - nh)]))


def _check(dj, oracle, cols, n, bk, bp, pk, pp):
    ref_n, ref = oracle.inner_join(bk, bp, pk, pp)
    assert n == ref_n
    got = [c.cpu().numpy() for c in cols]
    if n <= 2_000_000:
        for a, b in zip(oracle.sort_rows(*got), oracle.sort_rows(*ref)):
            assert (a == b).all()
    else:
        assert oracle.multiset_checksum4(*got) == oracle.multiset_checksum4(*ref)


def _join(dj, bk, pk, ws=None):
    bp, pp = _ids(bk.size), _ids(pk.size, 1 << 40)
    cols, n = dj.inner_join(_t(bk), _t(bp), _t(pk), _t(pp), capacity=pk.size, ws=ws)
    return cols, n, bp, pp


@pytest.mark.gpu
@pytest.mark.parametrize("side", ["build", "probe", "both"])
def test_level1_overflow(dj, oracle, side):
    """Most rows of one side in one level-1 bucket: that side's level 1 re-scatters its whole table,
    its level 2 then splits the crowded parent from its exact count."""
    rng = np.random.default_rng({"build": 1, "probe": 2, "both": 3}[side])
    bk = _crowded(NB, rng) if side != "probe" else rng.integers(-(1 << 62), 1 << 62, NB)
    bk = np.unique(bk)
    assert (K.bucket_of(bk, BITS1) == HOT1).mean() > (0.6 if side != "probe" else 0.0)
    pk = _probe_for(bk, NB + NB // 4, rng, crowd=side != "build")
    want = _want(bk, pk, ({"build": 1, "probe": 1, "both": 2}[side], 0))
    _repairs(dj)
    cols, n, bp, pp = _join(dj, bk, pk)
    assert _repairs(dj) == want
    _check(dj, oracle, cols, n, bk, bp, pk, pp)


def _one_child_overfull(rng, extra=700, hot=(7 << BITS2) | 45):
    """92 % of a full bucket's distinct keys in every level-2 bucket of the plan and `extra` more in
    bucket `hot`: its parent stays inside its level-1 capacity, the child outgrows its level-2
    capacity."""
    per = int(0.92 * (NB >> BITS))
    counts = np.full(1 << BITS, per)
    counts[hot] += extra
    return rng.permutation(np.concatenate([K.keys_in_bucket(BITS, b, int(c), rng) for b, c in enumerate(counts)]))


@pytest.mark.gpu
def test_level2_overflow_in_one_parent(dj, oracle):
    rng = np.random.default_rng(4)
    hot = (7 << BITS2) | 45
    bk = _one_child_overfull(rng, hot=hot)
    assert radix_plan(bk.size) == (BITS1, BITS2)  # the same plan as NB rows
    pk = _probe_for(bk, bk.size, rng, False, BITS, hot)
    want = _want(bk, pk, (0, 1))
    _repairs(dj)
    cols, n, bp, pp = _join(dj, bk, pk)
    assert _repairs(dj) == want
    _check(dj, oracle, cols, n, bk, bp, pk, pp)


@pytest.mark.gpu
def test_overflow_then_clean_call_on_one_workspace(dj, oracle):
    """Flags, cursors and capacities are rebuilt by every call: a clean join right after an
    overflowing one, in the same workspace, repairs nothing and is exact."""
    rng = np.random.default_rng(5)
    ws = dj.workspace(dj.lib().dj_inner_join_workspace_bytes(NB, NB + NB // 4))
    bk = np.unique(_crowded(NB, rng))
    pk = _probe_for(bk, NB + NB // 4, rng, crowd=True)
    want = _want(bk, pk, (2, 0))
    _repairs(dj)
    cols, n, bp, pp = _join(dj, bk, pk, ws)
    assert _repairs(dj) == want
    _check(dj, oracle, cols, n, bk, bp, pk, pp)
    bk = np.unique(rng.integers(-(1 << 62), 1 << 62, NB))
    pk = _probe_for(bk, NB + NB // 4, rng, crowd=False)
    assert _want(bk, pk, (0, 0)) == (0, 0)
    ws.fill_(-1)  # nothing from the earlier call may be needed
    cols, n, bp, pp = _join(dj, bk, pk, ws)
    assert _repairs(dj) == (0, 0)
    _check(dj, oracle, cols, n, bk, bp, pk, pp)


@pytest.mark.gpu
def test_streamed_host_entry_with_overflowing_probe_chunk(dj, oracle):
    """dj_distributed_inner_join_i64_host streams the probe table in 1M-row chunks against the
    resident build buckets; only the second chunk is crowded, so exactly one level-1 pass repairs."""
    import torch

    rng = np.random.default_rng(6)
    lk = np.unique(rng.integers(-(1 << 62), 1 << 62, NB))
    chunk = 1 << 20  # streamed_shape: 16 chunks, at least 1M rows each
    rk = np.concatenate([_probe_for(lk, chunk, rng, False), _probe_for(lk, chunk, rng, True),
                         _probe_for(lk, chunk // 2, rng, False)])
    over = tagged(("build",), side_overflows(lk, BITS1, BITS2))
    for c, at in enumerate(range(0, rk.size, chunk)):
        over += tagged(("chunk", c), side_overflows(rk[at:at + chunk], BITS1, BITS2))
    want = expected_repairs(over)
    assert over == [("chunk", 1, 0, 0, HOT1)], over
    lp, rp = _ids(lk.size), _ids(rk.size, 1 << 40)
    ref_n, ref = oracle.inner_join(lk, lp, rk, rp)
    h_in = [torch.from_numpy(a).pin_memory() for a in (lk, lp, rk, rp)]
    h_out = [torch.empty(ref_n + 16, dtype=torch.int64).pin_memory() for _ in range(4)]
    _repairs(dj)
    n, _ = dj.distributed_inner_join_host(None, *h_in, h_out)
    assert _repairs(dj) == want
    assert n == ref_n
    for a, b in zip(oracle.sort_rows(*[o[:n].numpy() for o in h_out]), oracle.sort_rows(*ref)):
        assert (a == b).all()


@pytest.mark.gpu
def test_generated_20m_join_repairs_nothing(dj, oracle):
    """The benchmark's generator at 20M x 20M (a two-level plan): no bucket reaches its capacity."""
    n = 20_000_000
    g = dj.gen_params(n, n, 0.3, 2 * n, True)
    bk, bp = dj.generate_rows(g, 0, 0, 0, n)
    pk, pp = dj.generate_rows(g, 1, 0, 0, n)
    _repairs(dj)
    res = dj.distributed_inner_join(None, bk, bp, pk, pp)
    assert _repairs(dj) == (0, 0)
    go = oracle.gen_params(n, n, 0.3, 2 * n, True)
    obk, obp, _ = oracle.generate_rows(go, 0, 0, 0, n)
    opk, opp, hits = oracle.generate_rows(go, 1, 0, 0, n)
    ref_n, ref = oracle.inner_join(obk, obp, opk, opp)
    assert res.n_out == ref_n == hits
    assert dj.multiset_checksum4(*res.cols) == oracle.multiset_checksum4(*ref)


@pytest.mark.gpu
def test_kernel_edges_with_exact_histograms(dj):
    """tests/test_kernel_edges.py again, in a fresh process with DJ_RADIX_EXACT=1 (exact histogram
    passes, buckets without gaps)."""
    env = dict(os.environ, PYTHONDONTWRITEBYTECODE="1", DJ_RADIX_EXACT="1")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + \
        ["-m", "pytest", "-q", "-x", "-p", "no:cacheprovider", "-m", "gpu", "-k", "not variant_sweep",
         os.path.join(ROOT, "tests", "test_kernel_edges.py")]
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=3000)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-2000:]
    assert " passed" in r.stdout and " failed" not in r.stdout


def test_400m_join_fits_one_80gb_card():
    """Capacity padding included, the benchmark's 400M x 400M join fits one 80 GB H100: the
    device-resident call (inputs, outputs, workspace) and the host-buffer leg (its workspace next to
    the resident inputs)."""
    import djb200

    L = djb200.lib()
    n = 400_000_000
    cap = int(n * 0.35) + 1_000_000
    inputs, outputs = 4 * 8 * n, 4 * 8 * cap
    resident = inputs + outputs + L.dj_distributed_inner_join_workspace_bytes(n, n, 1, 1)
    host_leg = inputs + L.dj_distributed_inner_join_host_workspace_bytes(n, n, cap, 1, 1)
    assert max(resident, host_leg) < 76 * 10**9  # 80 GB less the CUDA context and allocator slack
