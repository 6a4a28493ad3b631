"""Time the left semi / left anti joins next to the inner join on one GPU, in one process.

    python scripts/bench_left_filter_join.py [--rows 400000000] [--small-right 1000000] [--rounds 3] [--calls 5]

Workloads (the benchmark's generator, selectivity 0.3, unique build keys):
  inner     the benchmark's join: the unique build table as left, the probe table as right;
  semi/anti the probe table as left, the build table's keys as right (rows x rows);
  semi-1M   the probe table as left against the first 1M rows' keys of the build table;
  inner-1M  the inner join of those 1M build rows with the probe table, for comparison.
The configurations are alternated --rounds times; each round warms a configuration up with one call
and times --calls calls with CUDA events.  A separate pass per configuration reads the per-category
kernel times (dj_profile_*).  Parity: with unique build keys the semi join keeps exactly the probe
rows the inner join returns, so its count and dj_multiset_checksum4(k, p, k, p) must equal the inner
join's on its right-side (probe) columns, and anti count = rows - semi count.  Prints one JSON line
per configuration and one summary line; the card's name and power limit are read in the same run.
"""
import argparse
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

    # one workspace and one output buffer serve every configuration (the calls run one after the other)
    ws_bytes = max(L.dj_distributed_inner_join_workspace_bytes(n, n, 1, 1),
                   L.dj_distributed_left_filter_join_workspace_bytes(n, n, 1, 1),
                   L.dj_distributed_inner_join_workspace_bytes(ns, n, 1, 1),
                   L.dj_distributed_left_filter_join_workspace_bytes(n, ns, 1, 1))
    ws = dj.workspace(ws_bytes)
    inner_cap = int(n * (SELECTIVITY + 0.05)) + 1_000_000
    flat = torch.empty(max(2 * n, 4 * inner_cap), dtype=torch.int64, device="cuda")
    inner_outs = [flat[i * inner_cap:(i + 1) * inner_cap] for i in range(4)]
    filter_outs = [flat[:n], flat[n:2 * n]]
    torch.cuda.synchronize()

    configs = {
        "inner": lambda: dj.distributed_inner_join(None, bk, bp, pk, pp, capacity=inner_cap, ws=ws, outs=inner_outs),
        "semi": lambda: dj.distributed_left_semi_join(None, pk, pp, bk, capacity=n, ws=ws, outs=filter_outs),
        "anti": lambda: dj.distributed_left_anti_join(None, pk, pp, bk, capacity=n, ws=ws, outs=filter_outs),
        "inner-1M": lambda: dj.distributed_inner_join(None, sbk, sbp, pk, pp, capacity=inner_cap, ws=ws,
                                                      outs=inner_outs),
        "semi-1M": lambda: dj.distributed_left_semi_join(None, pk, pp, sbk, capacity=n, ws=ws, outs=filter_outs),
    }
    rows = {"inner": 2 * n, "semi": 2 * n, "anti": 2 * n, "inner-1M": n + ns, "semi-1M": n + ns}

    # ---- parity at full size
    def checksum(res, a, b):
        return dj.multiset_checksum4(res.cols[a], res.cols[b], res.cols[a], res.cols[b])

    parity = {}
    for inner_name, semi_name in (("inner", "semi"), ("inner-1M", "semi-1M")):
        r = configs[inner_name]()
        n_inner, ck_inner = r.n_out, checksum(r, 2, 3)
        r = configs[semi_name]()
        n_semi, ck_semi = r.n_out, checksum(r, 0, 1)
        parity[semi_name] = {"count": n_semi, "inner_count": n_inner, "ok": n_semi == n_inner and ck_semi == ck_inner}
    r = configs["anti"]()
    parity["anti"] = {"count": r.n_out, "ok": r.n_out == n - parity["semi"]["count"]}

    # ---- timing: configurations alternated, CUDA events around --calls calls
    times = {k: [] for k in configs}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(args.rounds):
        for name, fn in configs.items():
            fn()
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

    ident = gpu_identity()
    for name in configs:
        ms = statistics.median(times[name])
        print(json.dumps({"config": name, "ms_per_call": round(ms, 3),
                          "ms_rounds": [round(t, 3) for t in times[name]],
                          "rows_per_s": rows[name] / (ms * 1e-3), "kernel_ms": prof[name], "gpu": ident}))
    print(json.dumps({"parity": parity, "rows": n, "small_right": ns, "gpu": ident,
                      "all_ok": all(v["ok"] for v in parity.values())}))


if __name__ == "__main__":
    main()
