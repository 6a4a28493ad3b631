"""The host-buffer entries of the semi, anti, left outer and full outer joins
(dj_distributed_left_filter_join_i64_host, dj_distributed_outer_join_i64_host) against
tests/filter_oracle.py and tests/outer_oracle.py.

  chunks         left tables past 2^20 rows run >= 2 chunks (2^20 + 1 rows: a last chunk of one row);
  cross-chunk    the full outer case a per-chunk verdict gets wrong: right keys matched only by the
                 first chunk, only by the last, by every chunk, by none;
  multi-job      a hot right key of 3000 copies and a bucket of more distinct right keys than one
                 build chunk, matched and unmatched left rows in different chunks;
  empty sides, edge words, capacities 0 / n-1 / n / n+1 with guard tails on every host column,
  a workspace of exactly the queried size (sentinel tail) and one byte less, two calls back to back
  on one workspace, equality with the device entry, variants in fresh processes, rank groups.

Every workspace is pre-filled with a non-zero pattern: in the default mode the gaps between the
buckets of a prepared side hold whatever the workspace held, and a walk over them must not depend on
luck.  The CPU test checks this module's restatement of the workspace arithmetic and the chunk shape
against the library's query functions.
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

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = os.path.join(ROOT, "tests", "host_kinds_group_worker.py")
KINDS = {"semi": 1, "anti": 2, "left": 3, "full": 4}  # dj_b200.h DJ_JOIN_*
GUARD = 4096
SENTINEL = -0x5A5A5A5A5A5A5A5B
SIDES_SENTINEL = 0xEE
WS_FILL = 0xA5
BC = 1024 if os.environ.get("DJ_JOIN_SHAPE", "")[:1] in ("B", "b") else 1792  # join.cu build chunk
RADIX_EXACT = os.environ.get("DJ_RADIX_EXACT", "") == "1"


# ------------------------------------------------------------------------- restated arithmetic
def host_chunks(nleft):
    """(chunk rows, chunk count) of the streamed entries (comm.cu streamed_shape): the left table is chunked."""
    n = int(os.environ.get("DJ_HOST_CHUNKS", "0") or 0)
    n = n if n > 0 else 16
    chunk = -(-nleft // n)
    if chunk < (1 << 20):
        chunk = min(nleft, 1 << 20)
    chunk = max((chunk + 1) // 2 * 2, 2)
    return chunk, max(-(-nleft // chunk), 1)


def _align(x, a=256):
    return (x + a - 1) // a * a


def bits_bytes(span_rows, nright):
    """api.cu filter_bits_bytes: one bit per row of a side of `span_rows` rows prepared with the filter plan."""
    b1, b2 = RR.filter_plan(nright if nright > 0 else 1)
    rows = (RR.bounded_pass_rows(span_rows, 1 << b1, 1 << b2) if b2 else RR.bounded_pass_rows(span_rows, 1, 1 << b1)) + 8
    return _align((rows + 31) // 32 * 4) + 256


def streamed_ws_bytes(L, kind, nleft, nright, cap):
    """comm.cu streamed_ws_bytes for kind != 0.  The two prepared sides and one chunk's probe-row bits
    are what the device entry of a (chunk x nright) join needs, less its two 8 KiB margins."""
    filt, outer = kind in (1, 2), kind in (3, 4)
    chunk, nchunks = host_chunks(nleft)
    total = 256 + (1 if filt else 2) * _align(nright * 8) + (4 if nchunks > 1 else 2) * _align(chunk * 8)
    total += (2 if filt else 4) * _align(cap * 8) + (_align(cap) if outer else 0)
    total += L.dj_distributed_left_filter_join_workspace_bytes(chunk, nright, 1, 1) - 2 * 8192
    if kind == 4:
        total += bits_bytes(nright, nright)
    return total + (64 << 10)


def staged_ws_bytes(L, kind, nleft, nright, cap, world, odf):
    """The N > 1 queries: the device entry's workspace behind the staged input and output columns."""
    filt = kind in (1, 2)
    dev = (L.dj_distributed_left_filter_join_workspace_bytes if filt else L.dj_distributed_outer_join_workspace_bytes)
    prefix = 2 * _align(nleft * 8) + (1 if filt else 2) * _align(nright * 8) + (2 if filt else 4) * _align(cap * 8)
    return dev(nleft, nright, world, odf) + prefix + (0 if filt else _align(cap))


def query(L, kind, nleft, nright, cap, world=1, odf=1):
    fn = L.dj_distributed_left_filter_join_host_workspace_bytes if kind in (1, 2) else \
        L.dj_distributed_outer_join_host_workspace_bytes
    return fn(nleft, nright, cap, world, odf)


def test_workspace_arithmetic_restated():
    """No GPU: the restatements above against the library's queries, every kind, a grid of sizes."""
    import djb200

    L = djb200.lib()
    assert host_chunks((1 << 20) + 1)[1] == 2 and host_chunks(1 << 20) == (1 << 20, 1)
    for nl in (1, 1000, (1 << 20) + 1, 3_000_001, 40_000_000):
        for nr in (1, 777, 200_000, 5_000_000):
            for cap in (0, 1, nl, nl + nr):
                for name, kind in KINDS.items():
                    # the outer query is sized for the full outer join, the filter query serves both kinds
                    sized_as = 4 if kind in (3, 4) else 1
                    assert query(L, kind, nl, nr, cap) == streamed_ws_bytes(L, sized_as, nl, nr, cap), (name, nl, nr, cap)
                    for world, odf in ((2, 1), (3, 2)):
                        assert query(L, kind, nl, nr, cap, world, odf) == \
                            staged_ws_bytes(L, kind, nl, nr, cap, world, odf), (name, nl, nr, cap, world)


# ------------------------------------------------------------------------------------- helpers
# The variant re-runs and the rank groups are fresh processes (the library reads each variable once
# per process; a group wants its own stream pool).  Most of such a process's time is start-up, so they
# are all started when the module starts, run next to the cases below, and each is awaited by the
# test that reports it.
VARIANTS = {
    "host-chunks2": ({"DJ_HOST_CHUNKS": "2"}, "streamed_chunks or across_chunks or capacity_edges"),
    "shapeB": ({"DJ_JOIN_SHAPE": "B"}, "multi_job or across_chunks or back_to_back or workspace_exact"),
    "radix-exact": ({"DJ_RADIX_EXACT": "1"}, "multi_job or across_chunks or back_to_back or workspace_exact"),
}
WORLDS = [2, 3]
CHILDREN = {}  # test name -> (process, its output file)


def _child_commands():
    py = [sys.executable] + (["-s"] if sys.flags.no_user_site else [])
    base = dict(os.environ, PYTHONDONTWRITEBYTECODE="1")
    cmds = {}
    for variant, (env_add, expr) in VARIANTS.items():
        cmds[f"test_variant_sweep[{variant}]"] = (
            py + ["-m", "pytest", "-q", "-x", "-p", "no:cacheprovider", "-k",
                  f"({expr} or restated) and not variant_sweep and not rank_group", __file__], dict(base, **env_add))
    genv = {k: v for k, v in base.items() if k not in ("DJ_EXCHANGE", "DJ_NO_FUSE")}
    for world in WORLDS:
        cmds[f"test_rank_group[{world}]"] = (py + [WORKER, str(world)], dict(genv, CUDA_DEVICE_MAX_CONNECTIONS="32"))
    return cmds


@pytest.fixture(scope="module", autouse=True)
def _children_and_cached_memory(request):
    import tempfile

    import torch

    selected = {item.name for item in request.session.items}
    if torch.cuda.is_available():
        for name, (cmd, env) in _child_commands().items():
            if name in selected:
                out = tempfile.TemporaryFile(mode="w+")
                CHILDREN[name] = (subprocess.Popen(cmd, cwd=ROOT, env=env, stdout=out, stderr=subprocess.STDOUT), out)
    yield
    for proc, out in CHILDREN.values():  # a test that did not get to await its process
        if proc.poll() is None:
            proc.kill()
            proc.wait()
        out.close()
    CHILDREN.clear()
    # this module allocates workspaces and pinned columns of many sizes, which torch keeps cached: hand
    # them back, so that the modules (and their child processes) that run later find the memory free
    if torch.cuda.is_available():
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        if hasattr(torch._C, "_host_emptyCache"):
            torch._C._host_emptyCache()


def _await_child(name):
    proc, out = CHILDREN[name]
    try:
        rc = proc.wait(timeout=1500)
    except subprocess.TimeoutExpired:
        proc.kill()
        proc.wait()
        rc = None
    out.seek(0)
    return rc, out.read()


def _ids(n, base=0):
    return K.mix64(np.arange(base, base + n, dtype=np.int64))


def _pin(a, dtype=np.int64):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a, dtype=dtype)).pin_memory()


def reference(name, lk, lp, rk, rp):
    """The oracle's columns: 2 for semi / anti, 5 (sides last) for the outer joins."""
    if name in ("semi", "anti"):
        return FO.left_semi_join(lk, lp, rk, anti=name == "anti")
    return OO.outer_join(lk, lp, rk, rp, full=name == "full")


def _sorted(cols):
    cols = [np.asarray(c, dtype=np.int64) for c in cols]
    order = np.lexsort(cols[::-1]) if cols[0].size else np.empty(0, np.int64)
    return [c[order] for c in cols]


def assert_rows(got, ref, what=""):
    assert got[0].size == ref[0].size, f"{what}: {got[0].size} rows, oracle {ref[0].size}"
    for i, (a, b) in enumerate(zip(_sorted(got), _sorted(ref))):
        assert (a == b).all(), f"{what}: column {i} differs from the oracle"


def _sub_multiset(sub, ref):
    a = np.stack([np.asarray(c, np.int64) for c in ref], 1)
    b = np.stack([np.asarray(c, np.int64) for c in sub], 1)
    rows = np.ascontiguousarray(np.concatenate([a, b])).view(np.dtype((np.void, 8 * a.shape[1]))).ravel()
    _, inv = np.unique(rows, return_inverse=True)
    inv = inv.ravel()
    m = int(inv.max()) + 1 if inv.size else 0
    return bool((np.bincount(inv[len(a):], minlength=m) <= np.bincount(inv[:len(a)], minlength=m)).all())


class Workspace:
    """A device workspace of exactly `nbytes` usable bytes, everything pre-filled with a non-zero
    pattern, followed by a sentinel tail."""

    def __init__(self, nbytes):
        import torch

        self.nbytes = int(nbytes)
        self.buf = torch.full((self.nbytes + GUARD,), WS_FILL, dtype=torch.uint8, device="cuda")

    def refill(self):
        self.buf.fill_(WS_FILL)

    def tail_intact(self):
        return bool((self.buf[self.nbytes:] == WS_FILL).all().item())


def host_call(dj, name, lk, lp, rk, rp, cap, ws=None, ws_bytes=None, kind=None):
    """One call of the C entry of kind `name` (passing `kind` instead, when given) into guarded pinned
    columns.  Returns (rc, count, columns with their guard tails as numpy arrays (sides last, as
    int64), options, workspace)."""
    import torch

    L, filt = dj.lib(), name in ("semi", "anti")
    kind = KINDS[name] if kind is None else kind
    h_in = [_pin(a) for a in ((lk, lp, rk) if filt else (lk, lp, rk, rp))]
    h_out = [torch.full((cap + GUARD,), SENTINEL, dtype=torch.int64).pin_memory() for _ in range(2 if filt else 4)]
    sides = None if filt else torch.full((cap + GUARD,), SIDES_SENTINEL, dtype=torch.uint8).pin_memory()
    if ws is None:
        ws = Workspace(query(L, KINDS[name], len(lk), len(rk), cap) if ws_bytes is None else ws_bytes)
    cnt, opts = C.c_int64(0), dj.JoinOptions(1, 0)
    if filt:
        rc = L.dj_distributed_left_filter_join_i64_host(None, kind, h_in[0].data_ptr(), h_in[1].data_ptr(), len(lk),
                                                        h_in[2].data_ptr(), len(rk), h_out[0].data_ptr(),
                                                        h_out[1].data_ptr(), cap, C.byref(cnt), C.byref(opts),
                                                        ws.buf.data_ptr(), ws.nbytes, dj._stream())
    else:
        rc = L.dj_distributed_outer_join_i64_host(None, kind, h_in[0].data_ptr(), h_in[1].data_ptr(), len(lk),
                                                  h_in[2].data_ptr(), h_in[3].data_ptr(), len(rk),
                                                  *[o.data_ptr() for o in h_out], sides.data_ptr(), cap, C.byref(cnt),
                                                  C.byref(opts), ws.buf.data_ptr(), ws.nbytes, dj._stream())
    torch.cuda.synchronize()
    cols = [o.numpy().copy() for o in h_out] + ([] if filt else [sides.numpy().astype(np.int64)])
    return rc, cnt.value, cols, opts, ws


def assert_guards(cols, n, name):
    for i, c in enumerate(cols):
        tail = SIDES_SENTINEL if (name in ("left", "full") and i == 4) else SENTINEL
        assert (c[n:] == tail).all(), f"column {i} written past row {n}"


def run_exact(dj, name, lk, lp, rk, rp, ws=None):
    """The call at a capacity equal to the oracle's count, against the oracle; returns the oracle's columns."""
    ref = reference(name, lk, lp, rk, rp)
    n_ref = ref[0].size
    rc, n, cols, _, ws = host_call(dj, name, lk, lp, rk, rp, n_ref, ws)
    assert rc == 0, dj.lib().dj_last_error()
    assert n == n_ref
    assert_rows([c[:n] for c in cols], ref, name)
    assert_guards(cols, n, name)
    assert ws.tail_intact()
    return ref


def random_tables(nl, seed, nr=200_000):
    rng = np.random.default_rng(seed)
    lk = rng.integers(0, 400_000, nl, dtype=np.int64)
    rk = rng.integers(0, 300_000, nr, dtype=np.int64)  # duplicates on both sides, unmatched rows on both
    return lk, _ids(nl), rk, _ids(nr, 1 << 40)


# --------------------------------------------------------------------------------------- chunks
@pytest.mark.gpu
@pytest.mark.parametrize("nl", [(1 << 20) + 1, 1_300_001])
@pytest.mark.parametrize("name", list(KINDS))
def test_streamed_chunks(dj, name, nl):
    """Random tables with duplicate keys on both sides, the left table joined in >= 2 chunks."""
    assert host_chunks(nl)[1] >= 2
    if nl == (1 << 20) + 1:
        assert nl - host_chunks(nl)[0] * (host_chunks(nl)[1] - 1) == 1  # a last chunk of one row
    run_exact(dj, name, *random_tables(nl, nl))


@pytest.mark.gpu
def test_full_outer_across_chunks(dj):
    """Right keys matched only by rows of the first chunk, only of the last, in every chunk, in none:
    right-only rows appear exactly once each, and only for the last class."""
    nl = 2 * (1 << 20) + 1000
    chunk, nchunks = host_chunks(nl)
    assert nchunks >= 2
    rng = np.random.default_rng(11)
    ncls = 200
    cls = (rng.permutation(4 * ncls).astype(np.int64) + 1).reshape(4, ncls)  # first / last / every / none
    none_rows = np.concatenate([cls[3], cls[3][:50]])  # class `none` has duplicate rows too
    rk = rng.permutation(np.concatenate([cls[:3].ravel(), none_rows]))
    lk = -1 - rng.integers(0, 1 << 40, nl, dtype=np.int64)  # filler: left rows without a match
    for c in range(nchunks):
        lo, hi = c * chunk, min((c + 1) * chunk, nl)
        assert hi - lo >= 2 * ncls
        at = lo + rng.choice(hi - lo, 2 * ncls, replace=False)
        lk[at[:ncls]] = cls[2]  # every key of class `every` in each chunk
        if c == 0:
            lk[at[ncls:]] = cls[0]
        if c == nchunks - 1:
            lk[at[ncls:]] = cls[1]
    assert not np.isin(lk[chunk:], cls[0]).any() and not np.isin(lk[:(nchunks - 1) * chunk], cls[1]).any()
    ref = run_exact(dj, "full", lk, _ids(nl), rk, _ids(rk.size, 1 << 40))
    right_only = ref[4] == OO.SIDE_RIGHT
    assert (np.sort(ref[2][right_only]) == np.sort(none_rows)).all()


def _multi_job_tables(what, rng, nl):
    """Right table with a bucket of several build jobs; left rows that match it and rows that fall into
    the same bucket without a match, both kinds in the first and in the last chunk."""
    chunk, nchunks = host_chunks(nl)
    nr = 60_000
    bits = sum(RR.filter_plan(nr + 3000))
    spread = rng.integers(0, 1 << 40, nr, dtype=np.int64)
    if what == "hot-key":
        hot = np.int64(0x1234_5678_9ABC)
        rk = np.concatenate([np.full(3000, hot), spread])
        bucket = int(K.bucket_of(np.array([hot]), bits)[0])
        matched = np.full(40, hot)
    else:
        bucket = 77
        wide = K.keys_in_bucket(bits, bucket, BC + BC // 2, rng)  # more distinct keys than one build chunk
        rk = np.concatenate([wide, spread])
        matched = wide[::3]  # a third of the bucket's right keys match, the others are right-only
    assert sum(RR.filter_plan(rk.size)) == bits and (K.bucket_of(rk, bits) == bucket).sum() > BC
    strangers = K.keys_in_bucket(bits, bucket, 600, rng)
    strangers = strangers[~np.isin(strangers, rk)]  # probe rows of the bucket that match nothing
    lk = np.concatenate([rng.choice(spread, nl // 3), -1 - rng.integers(0, 1 << 40, nl - nl // 3, dtype=np.int64)])
    lk = rng.permutation(lk)
    for lo in (0, (nchunks - 1) * chunk):  # first and last chunk
        hi = min(lo + chunk, nl)
        at = lo + rng.choice(hi - lo, matched.size + strangers.size, replace=False)
        lk[at[:matched.size]] = matched
        lk[at[matched.size:]] = strangers
    return lk, _ids(nl), rng.permutation(rk), None


@pytest.mark.gpu
@pytest.mark.parametrize("what", ["hot-key", "wide-bucket"])
@pytest.mark.parametrize("name", list(KINDS))
def test_multi_job_buckets(dj, name, what):
    nl = (1 << 20) + 50_000
    assert host_chunks(nl)[1] >= 2
    lk, lp, rk, _ = _multi_job_tables(what, np.random.default_rng(len(what)), nl)
    run_exact(dj, name, lk, lp, rk, _ids(rk.size, 1 << 40))


# ---------------------------------------------------------------------------------- empty sides
@pytest.mark.gpu
@pytest.mark.parametrize("empty", ["left", "right", "both"])
@pytest.mark.parametrize("name", list(KINDS))
def test_empty_sides(dj, name, empty):
    lk, lp, rk, rp = random_tables(5000, 5, 3000)
    if empty in ("left", "both"):
        lk, lp = lk[:0], lp[:0]
    if empty in ("right", "both"):
        rk, rp = rk[:0], rp[:0]
    ref = run_exact(dj, name, lk, lp, rk, rp)
    want = {"left": {"full": 3000}, "right": {"anti": 5000, "left": 5000, "full": 5000}}.get(empty, {}).get(name, 0)
    assert ref[0].size == want
    if want:  # and under an overflow: the first rows, nothing past them
        rc, n, cols, _, _ = host_call(dj, name, lk, lp, rk, rp, want - 1)
        assert rc == dj.ERR_OVERFLOW and n == want
        assert _sub_multiset([c[:want - 1] for c in cols], ref)
        assert_guards(cols, want - 1, name)


# ----------------------------------------------------------------------------------- edge words
_M64 = (1 << 64) - 1
EDGE_WORDS = [0, 1, -1, -(1 << 63), (1 << 63) - 1, 0x7FFFFFFF, 0x80000000, 0xFFFFFFFF, 0x7FFFFFFF_80000000,
              0x80000000_00000000, 0x80000000_80000000, 0xFFFFFFFF_00000000]


def _edge_side(rng, ew, drop, n_pad):
    i64 = np.iinfo(np.int64)
    pad = rng.integers(i64.min, i64.max, n_pad + 64, dtype=np.int64, endpoint=True)
    pad = pad[~np.isin(pad, ew)][:n_pad]
    keep = ew[rng.permutation(ew.size)[drop:]]
    k = rng.permutation(np.concatenate([np.repeat(keep, rng.integers(1, 4, keep.size)), pad]))
    p = np.concatenate([rng.permutation(ew), _ids(k.size)])[:k.size]
    return k, rng.permutation(p)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(KINDS))
def test_edge_words(dj, name):
    """0, +-1, INT64_MIN/MAX and the words around the 32-bit half boundaries as keys and payloads, the
    left rows spread over >= 2 chunks; a few words on one side only."""
    ew = np.array(sorted({((w + d) & _M64) for w in EDGE_WORDS for d in range(-3, 4)}), dtype=np.uint64).view(np.int64)
    rng = np.random.default_rng(0xE2)
    lk, lp = _edge_side(rng, ew, 3, (1 << 20) + 4000)
    rk, rp = _edge_side(rng, ew, 3, 2000)
    assert host_chunks(lk.size)[1] >= 2
    run_exact(dj, name, lk, lp, rk, rp)


# ------------------------------------------------------------------------------------- capacity
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(KINDS))
def test_capacity_edges(dj, name):
    """Capacity 0, n-1, n, n+1 and (full outer) a cut inside the right-only tail: exact counts, the
    first `capacity` rows valid, every host column including `sides` untouched past them."""
    nl = (1 << 20) + 7000
    lk, lp, rk, rp = random_tables(nl, 21)
    ref = reference(name, lk, lp, rk, rp)
    n_ref = ref[0].size
    caps = [0, n_ref - 1, n_ref, n_ref + 1]
    if name == "full":
        tail = int((ref[4] == OO.SIDE_RIGHT).sum())
        assert tail > 100
        caps.append(n_ref - tail // 2)
    for cap in caps:
        rc, n, cols, _, ws = host_call(dj, name, lk, lp, rk, rp, cap)
        assert n == n_ref, (cap, n, n_ref)
        assert rc == (dj.ERR_OVERFLOW if cap < n_ref else 0), (cap, rc, dj.lib().dj_last_error())
        kept = min(cap, n_ref)
        if cap >= n_ref:
            assert_rows([c[:kept] for c in cols], ref, f"{name} cap {cap}")
        else:
            assert _sub_multiset([c[:kept] for c in cols], ref), f"{name} cap {cap}"
        assert_guards(cols, kept, name)
        assert ws.tail_intact()


# ------------------------------------------------------------------------------------ workspace
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(KINDS))
def test_workspace_exact_and_one_byte_less(dj, name):
    """A workspace of exactly the queried size works and its sentinel tail stays intact (run_exact);
    one byte less is DJ_ERR_WORKSPACE with workspace_needed equal to the query of the kind's entry."""
    nl = (1 << 20) + 3
    lk, lp, rk, rp = random_tables(nl, 31, 50_000)
    ref = run_exact(dj, name, lk, lp, rk, rp)
    cap = ref[0].size
    q = query(dj.lib(), KINDS[name], nl, rk.size, cap)
    # the outer query is sized for a full outer join; a left outer join needs less
    need = streamed_ws_bytes(dj.lib(), {"semi": 1, "anti": 1, "left": 3, "full": 4}[name], nl, rk.size, cap)
    assert need <= q and (name == "left" or need == q)
    rc, n, cols, opts, ws = host_call(dj, name, lk, lp, rk, rp, cap, ws_bytes=need - 1)
    assert rc == dj.ERR_WORKSPACE and opts.workspace_needed == need
    assert n == 0 and ws.tail_intact()
    assert_guards(cols, 0, name)
    rc, n, cols, _, ws = host_call(dj, name, lk, lp, rk, rp, cap, ws_bytes=need)
    assert rc == 0 and n == cap and ws.tail_intact()
    assert_rows([c[:n] for c in cols], ref, name)


@pytest.mark.gpu
def test_back_to_back_calls_share_a_workspace(dj):
    """A full outer join, then a semi join of other tables on the same stream and workspace, then the
    full outer join again: nothing leaks through the bit arrays."""
    a = random_tables((1 << 20) + 9, 41)
    b = random_tables((1 << 20) + 5000, 42, 150_000)
    L = dj.lib()
    ref_a, ref_b = reference("full", *a), reference("semi", *b)
    size = max(query(L, 4, len(a[0]), len(a[2]), ref_a[0].size), query(L, 1, len(b[0]), len(b[2]), ref_b[0].size))
    ws = Workspace(size)
    for name, t, ref in (("full", a, ref_a), ("semi", b, ref_b), ("full", a, ref_a)):
        rc, n, cols, _, _ = host_call(dj, name, *t, ref[0].size, ws)
        assert rc == 0, L.dj_last_error()
        assert_rows([c[:n] for c in cols], ref, name)
        assert ws.tail_intact()


# -------------------------------------------------------------------------- the device entries
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(KINDS))
def test_equals_device_entry(dj, name):
    """The binding's host call and the device entry of the same kind on the same tables, as multisets."""
    import torch

    nl = (1 << 20) + 12_345
    lk, lp, rk, rp = random_tables(nl, 51)
    t = [torch.from_numpy(a).cuda() for a in (lk, lp, rk, rp)]
    kind = KINDS[name]
    if kind in (1, 2):
        dev = dj.distributed_left_filter_join(None, kind, t[0], t[1], t[2])
        h_outs = [torch.empty(dev.n_out, dtype=torch.int64).pin_memory() for _ in range(2)]
        n, _ = dj.distributed_left_filter_join_host(None, kind, _pin(lk), _pin(lp), _pin(rk), h_outs)
    else:
        dev = dj.distributed_outer_join(None, kind, *t)
        h_outs = [torch.empty(dev.n_out, dtype=torch.int64).pin_memory() for _ in range(4)] + \
            [torch.empty(dev.n_out, dtype=torch.uint8).pin_memory()]
        n, _ = dj.distributed_outer_join_host(None, kind, _pin(lk), _pin(lp), _pin(rk), _pin(rp), h_outs)
    assert n == dev.n_out
    assert_rows([o.numpy()[:n] for o in h_outs], [c.cpu().numpy() for c in dev.cols], name)
    # the host outputs belong to the caller: an overflow raises
    with pytest.raises(dj.DjError):
        short = [o[:n - 1] for o in h_outs]
        if kind in (1, 2):
            dj.distributed_left_filter_join_host(None, kind, _pin(lk), _pin(lp), _pin(rk), short)
        else:
            dj.distributed_outer_join_host(None, kind, _pin(lk), _pin(lp), _pin(rk), _pin(rp), short)


@pytest.mark.gpu
def test_unknown_kind(dj):
    lk, lp, rk, rp = random_tables(1000, 61, 1000)
    for name, bad in (("semi", 3), ("anti", 0), ("left", 1), ("full", 5)):
        rc, _, cols, _, _ = host_call(dj, name, lk, lp, rk, rp, 10, ws_bytes=1 << 20, kind=bad)
        assert rc == dj.ERR_ARG and "kind" in dj.lib().dj_last_error().decode()
        assert_guards(cols, 0, name)


# ------------------------------------------------------------------ variant re-runs, rank groups
@pytest.mark.gpu
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_variant_sweep(dj, variant):
    """The cases a variant can change, again in a fresh process: the chunk shape for every case that
    runs the chunk loop once per kind; the CTA shape and the exact radix passes for the cases whose
    buckets matter (multi-job buckets, the cross-chunk bits, the walk over the build side)."""
    rc, text = _await_child(f"test_variant_sweep[{variant}]")
    assert rc == 0, text[-6000:]
    assert " passed" in text and " failed" not in text


@pytest.mark.gpu
@pytest.mark.parametrize("world", WORLDS)
def test_rank_group(dj, world):
    rc, text = _await_child(f"test_rank_group[{world}]")
    failed = [line for line in text.splitlines() if line.startswith("FAIL")]
    assert rc == 0 and not failed, "\n".join(failed) + "\n" + text[-6000:]
    assert f"cases passed (W={world}" in text
