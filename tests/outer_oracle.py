"""CPU oracle of the left / full outer joins (test infrastructure): numpy restatements next to
oracle.py's inner join and filter_oracle.py's semi / anti joins.

outer_join                       (lk, lp, rk, rp, sides) of the left or full outer join of two tables;
simulate_distributed_outer_join  what each rank of the distributed outer join returns: batch b's
                                 bucket b*G + i of the murmur3 rank partition goes to rank i, which
                                 joins the left and right rows of that bucket.

The matched pairs come from oracle.np_inner_join (sort + searchsorted) and the rows without a match
from np.isin, so that a test can hold each class of rows against the C oracle's inner join and the
semi / anti oracle, which compute them differently.
"""
import numpy as np

import oracle as O

SIDE_LEFT, SIDE_RIGHT = 1, 2  # dj_b200.h DJ_SIDE_*
BOTH = SIDE_LEFT | SIDE_RIGHT


def _i64(a):
    return np.ascontiguousarray(a, dtype=np.int64)


def outer_join(lk, lp, rk, rp, full=False):
    """(lk, lp, rk, rp, sides) as int64 columns: every matching pair with sides 3, every left row
    without a match with sides 1 and, for a full outer join, every right row without a match with
    sides 2.  Absent columns are 0."""
    lk, lp, rk, rp = map(_i64, (lk, lp, rk, rp))
    pairs = O.np_inner_join(lk, lp, rk, rp)
    lone_l = ~np.isin(lk, rk) if rk.size else np.ones(lk.size, bool)
    cols = [[pairs[0], lk[lone_l]], [pairs[1], lp[lone_l]], [pairs[2], np.zeros(lone_l.sum(), np.int64)],
            [pairs[3], np.zeros(lone_l.sum(), np.int64)]]
    sides = [np.full(pairs[0].size, BOTH, np.int64), np.full(lone_l.sum(), SIDE_LEFT, np.int64)]
    if full:
        lone_r = ~np.isin(rk, lk) if lk.size else np.ones(rk.size, bool)
        n = int(lone_r.sum())
        for c, v in zip(cols, (np.zeros(n, np.int64), np.zeros(n, np.int64), rk[lone_r], rp[lone_r])):
            c.append(v)
        sides.append(np.full(n, SIDE_RIGHT, np.int64))
    return tuple(np.concatenate(c) for c in cols) + (np.concatenate(sides),)


def row_keys(res):
    """The key that places each output row on a rank: the left key, or the right key of a right-only row."""
    return np.where(res[4] == SIDE_RIGHT, res[2], res[0])


def simulate_distributed_outer_join(lefts, rights, odf=1, full=False, seed=O.SEED_NVLINK):
    """lefts / rights: per-rank (keys, payloads).  Returns per rank the 5 columns the distributed
    outer join leaves there."""
    G = len(lefts)
    if G == 1:
        return [outer_join(*lefts[0], *rights[0], full)]
    nparts = G * odf
    parts_l = [O.hash_partition(k, p, nparts, seed) for k, p in lefts]
    parts_r = [O.hash_partition(k, p, nparts, seed) for k, p in rights]
    results = []
    for dst in range(G):
        outs = []
        for b in range(odf):
            q = b * G + dst

            def gather(parts):
                return (np.concatenate([k[off[q]:off[q + 1]] for k, _, off in parts]),
                        np.concatenate([p[off[q]:off[q + 1]] for _, p, off in parts]))

            outs.append(outer_join(*gather(parts_l), *gather(parts_r), full))
        results.append(tuple(np.concatenate([o[c] for o in outs]) for c in range(5)))
    return results
