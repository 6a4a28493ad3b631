"""Time the broadcast join against the repartitioned joins on one GPU (N = 1), in one process.

    python scripts/bench_broadcast_join.py [--rows 400000000] [--rounds 3] [--calls 5]

Left table: the benchmark generator's probe table (--rows rows, selectivity 0.3), its keys folded into
[0, 2R) (key mod 2R), so that it is a fact table whose foreign keys take 2R values.  Right table: the
keys 0 .. R-1 in shuffled order with mixed payloads, a dimension table that about half the left rows
match, each exactly once.  R is 2^16, 2^20, DJ_BROADCAST_TABLE_MAX_ROWS and 4x that, each timed once
(2^20 and the threshold coincide today).

For every R and kind (inner, left semi, left outer) the broadcast entry (dj_broadcast_join_i64) and the
repartitioned entry of the same kind (at N = 1 the radix-partitioned local join) are alternated --rounds
times; each round warms both up with one call and times --calls calls with CUDA events.  A separate pass
per configuration reads the per-category kernel times (dj_profile_*).  Every result is checked against
the other entry's: row count and dj_multiset_checksum4 (semi: of (key, payload, key, payload); left
outer: also the number of rows without a match).  The card's name, power limit and max SM clock are read
in the same run.  Prints one JSON line per (R, kind) and one summary line.
"""
import argparse
import gc
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "distributed-join_b200"))

SELECTIVITY = 0.3


def gpu_identity():
    import torch

    ident = {"name": torch.cuda.get_device_name(0), "power_limit_w": None, "sm_max_mhz": None}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                              "-i", "0"], capture_output=True, text=True, timeout=30).stdout
        pl, clk = out.split(",")[:2]
        ident["power_limit_w"], ident["sm_max_mhz"] = float(pl), float(clk)
    except Exception:
        pass
    return ident


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=400_000_000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--calls", type=int, default=5)
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

    def checksum(cols):
        return dj.multiset_checksum4(*cols) if cols[0].numel() else (0, 0)

    def summary(kind, cols, cnt):
        cols = [c[:cnt] for c in cols]
        if kind == dj.JOIN_LEFT_SEMI:
            return cnt, checksum([cols[0], cols[1], cols[0], cols[1]])
        if kind == dj.JOIN_LEFT_OUTER:
            return cnt, checksum(cols[:4]), int((cols[4] == dj.SIDE_LEFT).sum())
        return cnt, checksum(cols)

    results = []
    for R in sorted({1 << 16, 1 << 20, dj.BROADCAST_TABLE_MAX_ROWS, 4 * dj.BROADCAST_TABLE_MAX_ROWS}):
        torch.remainder(orig_k, 2 * R, out=lk)
        rk = torch.randperm(R, device="cuda", dtype=torch.int64)
        rp = rk * 1_000_003 + 17
        torch.cuda.synchronize()
        matched = None
        for kname, kind in (("inner", 0), ("semi", dj.JOIN_LEFT_SEMI), ("left_outer", dj.JOIN_LEFT_OUTER)):
            ncols = 2 if kind == dj.JOIN_LEFT_SEMI else 5 if kind == dj.JOIN_LEFT_OUTER else 4
            cap = n if kind else n // 2 + n // 20
            outs = [torch.empty(cap, dtype=torch.uint8 if c == 4 else torch.int64, device="cuda") for c in range(ncols)]
            ptr = [o.data_ptr() for o in outs] + [None] * (5 - ncols)
            ws_b = dj.workspace(L.dj_broadcast_join_workspace_bytes(n, R))
            if kind == 0:
                ws_r = dj.workspace(L.dj_distributed_inner_join_workspace_bytes(n, R, 1, 1))
            elif kind == dj.JOIN_LEFT_SEMI:
                ws_r = dj.workspace(L.dj_distributed_left_filter_join_workspace_bytes(n, R, 1, 1))
            else:
                ws_r = dj.workspace(L.dj_distributed_outer_join_workspace_bytes(n, R, 1, 1))

            def call(entry):
                cnt, opts = C.c_int64(0), dj.JoinOptions(1, 0)
                if entry == "broadcast":
                    rc = L.dj_broadcast_join_i64(None, kind, lk.data_ptr(), lp.data_ptr(), n, rk.data_ptr(),
                                                 rp.data_ptr(), R, *ptr, cap, C.byref(cnt), C.byref(opts),
                                                 ws_b.data_ptr(), ws_b.numel(), stream)
                elif kind == 0:
                    rc = L.dj_distributed_inner_join_i64(None, lk.data_ptr(), lp.data_ptr(), n, rk.data_ptr(),
                                                         rp.data_ptr(), R, *ptr[:4], cap, C.byref(cnt), C.byref(opts),
                                                         ws_r.data_ptr(), ws_r.numel(), stream)
                elif kind == dj.JOIN_LEFT_SEMI:
                    rc = L.dj_distributed_left_filter_join_i64(None, kind, lk.data_ptr(), lp.data_ptr(), n,
                                                               rk.data_ptr(), R, *ptr[:2], cap, C.byref(cnt),
                                                               C.byref(opts), ws_r.data_ptr(), ws_r.numel(), stream)
                else:
                    rc = L.dj_distributed_outer_join_i64(None, kind, lk.data_ptr(), lp.data_ptr(), n, rk.data_ptr(),
                                                         rp.data_ptr(), R, *ptr, cap, C.byref(cnt), C.byref(opts),
                                                         ws_r.data_ptr(), ws_r.numel(), stream)
                if rc:
                    raise RuntimeError(f"{entry} {kname} R={R}: rc {rc}: {L.dj_last_error().decode()}")
                return cnt.value

            times = {"broadcast": [], "repartitioned": []}
            check = {}
            for _ in range(args.rounds):
                for entry in times:
                    cnt = call(entry)  # warm-up, and the parity check
                    torch.cuda.synchronize()
                    s = summary(kind, outs, cnt)
                    assert check.setdefault(entry, s) == s, f"{entry} {kname} R={R}: results differ between calls"
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record()
                    for _ in range(args.calls):
                        call(entry)
                    b.record()
                    b.synchronize()
                    times[entry].append(a.elapsed_time(b) / args.calls)
            same = check["broadcast"] == check["repartitioned"]
            prof = {}
            for entry in times:
                dj.profile_enable(True)
                dj.profile_read()
                call(entry)
                torch.cuda.synchronize()
                prof[entry] = {k: round(v[0], 3) for k, v in dj.profile_read().items()}
                dj.profile_enable(False)
            if kind == dj.JOIN_LEFT_SEMI:
                matched = check["broadcast"][0]
            row = {"R": R, "kind": kname, "left_rows": n, "out_rows": check["broadcast"][0],
                   "results_equal": same,
                   "broadcast_ms": round(statistics.median(times["broadcast"]), 3),
                   "repartitioned_ms": round(statistics.median(times["repartitioned"]), 3),
                   "broadcast_ms_all": [round(t, 3) for t in times["broadcast"]],
                   "repartitioned_ms_all": [round(t, 3) for t in times["repartitioned"]],
                   "profile_ms": prof}
            if matched is not None:
                row["matched_left_share"] = round(matched / n, 4)
            print(json.dumps(row), flush=True)
            results.append(row)
            del outs, ws_b, ws_r
            gc.collect()
            torch.cuda.empty_cache()
    print(json.dumps({"gpu": ident, "all_results_equal": all(r["results_equal"] for r in results),
                      "rounds": args.rounds, "calls": args.calls}), flush=True)
    if not all(r["results_equal"] for r in results):
        sys.exit(1)


if __name__ == "__main__":
    main()
