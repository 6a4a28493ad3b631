"""Time the broadcast full outer join against the repartitioned full outer join and the broadcast left outer
join on one GPU (N = 1), in one process.

    python scripts/bench_broadcast_full_outer_join.py [--rows 400000000] [--rounds 3] [--calls 3]

Tables as in scripts/bench_broadcast_join.py: the left table is the benchmark generator's probe table (--rows
rows, selectivity 0.3) with its keys folded into [0, 2R), the right table the keys 0 .. R-1 in shuffled order
with mixed payloads, so that about half the left rows match, each exactly once, and nearly every right key
is matched.  R is 2^16, 2^20 and 2^22 (above DJ_BROADCAST_TABLE_MAX_ROWS: the radix path).

For every R the three entries alternate --rounds times: dj_broadcast_full_outer_join_i64, the repartitioned
dj_distributed_outer_join_i64(DJ_JOIN_FULL_OUTER) (at N = 1 the radix-partitioned local join) and
dj_broadcast_join_i64(DJ_JOIN_LEFT_OUTER).  Each round warms an entry up with one call and times --calls
calls with CUDA events.  Both full outer results are held against each other: row count and
dj_multiset_checksum4 per class of sides.  The card's name, power limit and max SM clock are read in the
same run.  Prints one JSON line per R and one summary line.
"""
import argparse
import gc
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "distributed-join_b200"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_broadcast_join import SELECTIVITY, gpu_identity  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=400_000_000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--calls", type=int, default=3)
    args = ap.parse_args()

    import ctypes as C

    import torch

    import djb200 as dj

    assert torch.cuda.is_available(), "the benchmark needs a GPU"
    torch.cuda.set_device(0)
    L = dj.lib()
    ident = gpu_identity()
    n = args.rows
    g = dj.gen_params(n, n, SELECTIVITY, 2 * n, True)
    orig_k, lp = dj.generate_rows(g, 1, 0, 0, n)
    lk = torch.empty_like(orig_k)
    stream = dj._stream()

    def per_class(outs, cnt):
        cols = [c[:cnt] for c in outs]
        res = {}
        for s in (dj.SIDE_LEFT | dj.SIDE_RIGHT, dj.SIDE_LEFT, dj.SIDE_RIGHT):
            m = cols[4] == s
            sel = [c[m] for c in cols[:4]]
            res[s] = (int(sel[0].numel()), dj.multiset_checksum4(*sel) if sel[0].numel() else (0, 0))
            del sel, m
        return cnt, res

    results = []
    for R in (1 << 16, 1 << 20, 1 << 22):
        torch.remainder(orig_k, 2 * R, out=lk)
        rk = torch.randperm(R, device="cuda", dtype=torch.int64)
        rp = rk * 1_000_003 + 17
        cap = n + R
        outs = [torch.empty(cap, dtype=torch.uint8 if c == 4 else torch.int64, device="cuda") for c in range(5)]
        ptr = [o.data_ptr() for o in outs]
        ws = dj.workspace(max(L.dj_broadcast_full_outer_join_workspace_bytes(n, R, R, 1),
                              L.dj_distributed_outer_join_workspace_bytes(n, R, 1, 1),
                              L.dj_broadcast_join_workspace_bytes(n, R)))
        torch.cuda.synchronize()

        def call(entry):
            cnt, opts = C.c_int64(0), dj.JoinOptions(1, 0)
            common = (lk.data_ptr(), lp.data_ptr(), n, rk.data_ptr(), rp.data_ptr(), R, *ptr, cap, C.byref(cnt),
                      C.byref(opts), ws.data_ptr(), ws.numel(), stream)
            if entry == "broadcast_full_outer":
                rc = L.dj_broadcast_full_outer_join_i64(None, *common)
            elif entry == "repartitioned_full_outer":
                rc = L.dj_distributed_outer_join_i64(None, dj.JOIN_FULL_OUTER, *common)
            else:
                rc = L.dj_broadcast_join_i64(None, dj.JOIN_LEFT_OUTER, *common)
            if rc:
                raise RuntimeError(f"{entry} R={R}: rc {rc}: {L.dj_last_error().decode()}")
            return cnt.value

        times = {"broadcast_full_outer": [], "repartitioned_full_outer": [], "broadcast_left_outer": []}
        check = {}
        for _ in range(args.rounds):
            for entry in times:
                cnt = call(entry)  # warm-up, and the parity check
                torch.cuda.synchronize()
                if entry != "broadcast_left_outer":
                    s = per_class(outs, cnt)
                    assert check.setdefault(entry, s) == s, f"{entry} R={R}: results differ between calls"
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for _ in range(args.calls):
                    call(entry)
                b.record()
                b.synchronize()
                times[entry].append(a.elapsed_time(b) / args.calls)
        same = check["broadcast_full_outer"] == check["repartitioned_full_outer"]
        row = {"R": R, "left_rows": n, "out_rows": check["broadcast_full_outer"][0],
               "lone_right_rows": check["broadcast_full_outer"][1][dj.SIDE_RIGHT][0], "results_equal": same}
        for entry, t in times.items():
            row[entry + "_ms"] = round(statistics.median(t), 3)
            row[entry + "_ms_all"] = [round(x, 3) for x in t]
        print(json.dumps(row), flush=True)
        results.append(row)
        del outs, ws
        gc.collect()
        torch.cuda.empty_cache()
    print(json.dumps({"gpu": ident, "all_results_equal": all(r["results_equal"] for r in results),
                      "rounds": args.rounds, "calls": args.calls}), flush=True)
    if not all(r["results_equal"] for r in results):
        sys.exit(1)


if __name__ == "__main__":
    main()
