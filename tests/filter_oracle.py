"""CPU oracle of the left semi / left anti joins (test infrastructure): numpy restatements next to
oracle.py's inner join and its N-rank simulation.

left_semi_join                        every left row whose key is (semi) or is not (anti) in rk, once;
simulate_distributed_left_semi_join   what each rank of the distributed join keeps: batch b's bucket
                                      b*G + i of the murmur3 rank partition goes to rank i, which
                                      filters the left rows of that bucket against its right keys.
"""
import numpy as np

import oracle as O


def left_semi_join(lk, lp, rk, anti=False):
    """(keys, payloads) of the left rows whose key appears in rk (anti: does not), in left order."""
    lk, lp, rk = (np.ascontiguousarray(a, dtype=np.int64) for a in (lk, lp, rk))
    keep = np.isin(lk, rk, invert=anti)
    return lk[keep], lp[keep]


def simulate_distributed_left_semi_join(lefts, right_keys, odf=1, anti=False, seed=O.SEED_NVLINK):
    """lefts: per-rank (keys, payloads); right_keys: per-rank key arrays.  Returns per rank the
    (keys, payloads) the distributed semi (anti) join leaves there."""
    G = len(lefts)
    if G == 1:
        return [left_semi_join(*lefts[0], right_keys[0], anti)]
    nparts = G * odf
    parts_l = [O.hash_partition(k, p, nparts, seed) for k, p in lefts]
    parts_r = [O.hash_partition(k, k, nparts, seed) for k in right_keys]
    results = []
    for dst in range(G):
        ks, ps = [], []
        for b in range(odf):
            q = b * G + dst
            lk = np.concatenate([k[off[q]:off[q + 1]] for k, _, off in parts_l])
            lp = np.concatenate([p[off[q]:off[q + 1]] for _, p, off in parts_l])
            rk = np.concatenate([k[off[q]:off[q + 1]] for k, _, off in parts_r])
            k, p = left_semi_join(lk, lp, rk, anti)
            ks.append(k)
            ps.append(p)
        results.append((np.concatenate(ks), np.concatenate(ps)))
    return results
