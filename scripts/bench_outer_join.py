"""Time the left outer / full outer joins next to the inner join on one GPU, in one process.

    python scripts/bench_outer_join.py [--rows 400000000] [--small-right 1000000] [--rounds 3] [--calls 5]

Workloads (the benchmark's generator, selectivity 0.3, unique build keys):
  inner      the benchmark's join: the unique build table as left, the probe table as right;
  left/full  the probe table as left, the build table as right (rows x rows);
  left-1M    the probe table as left against the first 1M rows of the build table.
The configurations are alternated --rounds times; each round warms a configuration up with one call
and times --calls calls with CUDA events.  A separate pass per configuration reads the per-category
kernel times (dj_profile_*).

Parity at full size, against existing entries (each class of output rows one at a time, to stay
within one 80 GB card next to the inputs, the workspace and the full outer join's output):
  sides 3  the inner join's rows with the sides swapped: same count, and dj_multiset_checksum4 of
           (lk, lp, rk, rp) equals the inner join's checksum of (rk, rp, lk, lp);
  sides 1  the anti join of left against the right keys: count and checksum4(lk, lp, lk, lp);
  sides 2  (full) the anti join of the build table against the probe keys: count and
           checksum4(rk, rp, rk, rp) against the anti join's checksum4(k, p, k, p).
Prints one JSON line per configuration and one summary line; the card's name and power limit are
read in the same run.
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

    ident = {"name": torch.cuda.get_device_name(0), "power_limit_w": None}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout
        ident["power_limit_w"] = float(out.split()[0])
    except Exception:
        pass
    return ident


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=400_000_000)
    ap.add_argument("--small-right", type=int, default=1_000_000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--calls", type=int, default=5)
    args = ap.parse_args()

    import torch

    import djb200 as dj

    assert torch.cuda.is_available(), "this measurement needs a GPU"
    torch.cuda.set_device(0)
    n, ns = args.rows, args.small_right
    L = dj.lib()
    g = dj.gen_params(n, n, SELECTIVITY, 2 * n, True)
    (bk, bp), (pk, pp) = dj.generate_tables_distributed(g, 0, 1)
    sbk, sbp = bk[:ns], bp[:ns]

    def ck(a, b, c, d):
        return dj.multiset_checksum4(a, b, c, d)

    # one workspace serves every configuration (the calls run one after the other)
    ws = dj.workspace(max(L.dj_distributed_inner_join_workspace_bytes(n, n, 1, 1),
                          L.dj_distributed_outer_join_workspace_bytes(n, n, 1, 1),
                          L.dj_distributed_outer_join_workspace_bytes(n, ns, 1, 1)))
    inner_cap = int(n * (SELECTIVITY + 0.05)) + 1_000_000

    # ---- reference counts and checksums from the existing entries (their outputs freed at once)
    ref = {}
    r = dj.distributed_inner_join(None, bk, bp, pk, pp, capacity=inner_cap, ws=ws)
    ref["both"] = (r.n_out, ck(r.cols[2], r.cols[3], r.cols[0], r.cols[1]))
    del r
    r = dj.distributed_left_anti_join(None, pk, pp, bk, capacity=n, ws=ws)
    ref["left"] = (r.n_out, ck(r.cols[0], r.cols[1], r.cols[0], r.cols[1]))
    del r
    r = dj.distributed_left_anti_join(None, bk, bp, pk, capacity=n, ws=ws)
    ref["right"] = (r.n_out, ck(r.cols[0], r.cols[1], r.cols[0], r.cols[1]))
    del r
    gc.collect()
    torch.cuda.empty_cache()

    # one output buffer, sized for the full outer join, serves every configuration
    full_cap = ref["both"][0] + ref["left"][0] + ref["right"][0]
    flat = torch.empty(4 * full_cap, dtype=torch.int64, device="cuda")
    sides = torch.empty(full_cap, dtype=torch.uint8, device="cuda")

    def outs(cap):
        return [flat[i * cap:(i + 1) * cap] for i in range(4)] + [sides[:cap]]

    left_cap = ref["both"][0] + ref["left"][0]
    configs = {
        "inner": lambda: dj.distributed_inner_join(None, bk, bp, pk, pp, capacity=inner_cap, ws=ws,
                                                   outs=outs(inner_cap)[:4]),
        "left-outer": lambda: dj.distributed_left_outer_join(None, pk, pp, bk, bp, capacity=left_cap, ws=ws,
                                                             outs=outs(left_cap)),
        "full-outer": lambda: dj.distributed_full_outer_join(None, pk, pp, bk, bp, capacity=full_cap, ws=ws,
                                                             outs=outs(full_cap)),
        "left-outer-1M": lambda: dj.distributed_left_outer_join(None, pk, pp, sbk, sbp, capacity=n, ws=ws,
                                                                outs=outs(n)),
    }
    rows = {"inner": 2 * n, "left-outer": 2 * n, "full-outer": 2 * n, "left-outer-1M": n + ns}
    torch.cuda.synchronize()

    # ---- timing: configurations alternated, CUDA events around --calls calls
    times = {k: [] for k in configs}
    n_out = {}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(args.rounds):
        for name, fn in configs.items():
            n_out[name] = fn().n_out
            torch.cuda.synchronize()
            e0.record()
            for _ in range(args.calls):
                fn()
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1) / args.calls)

    # ---- per-category kernel time, one separate pass per configuration
    prof = {}
    for name, fn in configs.items():
        dj.profile_enable(True)
        dj.profile_read()
        for _ in range(args.calls):
            fn()
        torch.cuda.synchronize()
        p = dj.profile_read()
        dj.profile_enable(False)
        prof[name] = {c: round(ms / args.calls, 3) for c, (ms, _) in p.items()}

    # ---- parity, one class of rows at a time (the workspace is no longer needed)
    parity = {}
    for name in ("left-outer", "full-outer"):
        res = configs[name]()
        torch.cuda.synchronize()
        if name == "full-outer":
            del ws
            gc.collect()
            torch.cuda.empty_cache()
        c, sd = [x for x in res.cols[:4]], res.cols[4]
        got = {}
        for cls, s, pick in (("both", 3, (0, 1, 2, 3)), ("left", 1, (0, 1, 0, 1)), ("right", 2, (2, 3, 2, 3))):
            idx = torch.nonzero(sd == s).squeeze(1)
            cols = {i: c[i].index_select(0, idx) for i in set(pick)}
            got[cls] = (int(idx.numel()), ck(*[cols[i] for i in pick]) if idx.numel() else (0, 0))
            del idx, cols
            torch.cuda.empty_cache()
        want = dict(ref, right=ref["right"] if name == "full-outer" else (0, (0, 0)))
        parity[name] = {cls: {"count": got[cls][0], "ref_count": want[cls][0], "ok": got[cls] == want[cls]}
                        for cls in got}
        parity[name]["ok"] = res.n_out == sum(got[k][0] for k in got) and all(v["ok"] for v in parity[name].values()
                                                                               if isinstance(v, dict))
        del res, c, sd

    ident = gpu_identity()
    for name in configs:
        ms = statistics.median(times[name])
        print(json.dumps({"config": name, "ms_per_call": round(ms, 3),
                          "ms_rounds": [round(t, 3) for t in times[name]], "n_out": n_out[name],
                          "rows_per_s": rows[name] / (ms * 1e-3), "kernel_ms": prof[name], "gpu": ident}))
    print(json.dumps({"parity": parity, "rows": n, "small_right": ns, "gpu": ident,
                      "all_ok": all(v["ok"] for v in parity.values())}))


if __name__ == "__main__":
    main()
