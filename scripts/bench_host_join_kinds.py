"""Time the host-buffer entries of the semi, anti, left outer and full outer joins on one GPU, each
against its staged equivalent, with the inner host entry as the yardstick of the same session.

    python scripts/bench_host_join_kinds.py [--rows 200000000] [--rounds 3] [--calls 3]

Tables: the benchmark's generator, selectivity 0.3, unique build keys; the probe table is the left
table, the build table the right one (rows x rows), all host buffers pinned.
  streamed   dj_distributed_*_i64_host: the right table up once, the left table in chunks, rows down
             while the next chunk comes up;
  staged     what a caller had to do before: both tables up, the device entry, the result down, on
             one stream.
The two are alternated --rounds times per kind; a round is one warm-up call and --calls timed calls
that end in a synchronise (host clock).  Bytes up and down are computed from the shapes.  A separate
pass reads the per-category kernel times (dj_profile_*) of the streamed call, and one profiled full
outer call gives the device time of emit_unmatched_build_kernel.  Parity: count and
dj_multiset_checksum4 per class of rows, streamed host entry against the device entry, at the timed
size.  Prints one JSON line per configuration; the card's name and power limit are read in the same run.
"""
import argparse
import gc
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "distributed-join_b200"))

SELECTIVITY = 0.3
KINDS = {"semi": 1, "anti": 2, "left-outer": 3, "full-outer": 4}


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


def host_bytes_available():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=200_000_000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--calls", type=int, default=3)
    args = ap.parse_args()

    import torch

    import djb200 as dj

    assert torch.cuda.is_available(), "this measurement needs a GPU"
    torch.cuda.set_device(0)
    n = args.rows
    L = dj.lib()
    n_both = int(n * (SELECTIVITY + 0.02)) + 1_000_000  # upper bounds on the classes of rows
    cap = {"inner": n_both, "semi": n_both, "anti": n, "left-outer": n, "full-outer": 2 * n}
    pinned_need = 4 * n * 8 + cap["full-outer"] * 33
    avail = host_bytes_available()
    if avail is not None and pinned_need > 0.8 * avail:
        sys.exit(f"{n} x {n} rows need {pinned_need / 1e9:.1f} GB of pinned host memory (inputs and the full outer "
                 f"join's output); {avail / 1e9:.1f} GB are available: use a smaller --rows")

    g = dj.gen_params(n, n, SELECTIVITY, 2 * n, True)
    (bk, bp), (pk, pp) = dj.generate_tables_distributed(g, 0, 1)
    dev_in = {"lk": pk, "lp": pp, "rk": bk, "rp": bp}
    h = {k: torch.empty(n, dtype=torch.int64).pin_memory() for k in dev_in}
    for k, t in dev_in.items():
        h[k].copy_(t)
    h_flat = torch.empty(4 * cap["full-outer"], dtype=torch.int64).pin_memory()
    h_sides = torch.empty(cap["full-outer"], dtype=torch.uint8).pin_memory()

    def h_outs(name):
        c = cap[name]
        cols = [h_flat[i * c:(i + 1) * c] for i in range(2 if name in ("semi", "anti") else 4)]
        return cols + [h_sides[:c]] if name.endswith("outer") else cols

    def ck(cols, pick):
        return dj.multiset_checksum4(*[cols[i] for i in pick])

    def classes(name, cols, n_out):
        """{class: (count, checksum)} of device columns trimmed to n_out."""
        if name in ("semi", "anti"):
            return {"rows": (n_out, ck(cols, (0, 1, 0, 1)) if n_out else (0, 0))}
        got = {}
        for cls, s, pick in (("both", 3, (0, 1, 2, 3)), ("left", 1, (0, 1, 0, 1)), ("right", 2, (2, 3, 2, 3))):
            idx = torch.nonzero(cols[4] == s).squeeze(1)
            sel = {i: cols[i].index_select(0, idx) for i in set(pick)}
            got[cls] = (int(idx.numel()), ck(sel, pick) if idx.numel() else (0, 0))
        return got

    # ---- the device entries' results: the parity reference (outputs freed at once)
    ref = {}
    for name, kind in KINDS.items():
        if kind in (1, 2):
            r = dj.distributed_left_filter_join(None, kind, pk, pp, bk, capacity=cap[name])
        else:
            r = dj.distributed_outer_join(None, kind, pk, pp, bk, bp, capacity=cap[name])
        ref[name] = classes(name, r.cols, r.n_out)
        del r
        gc.collect()
        torch.cuda.empty_cache()
    del dev_in, bk, bp, pk, pp
    gc.collect()
    torch.cuda.empty_cache()

    # ---- one workspace serves every configuration; the staged calls carve their columns from it too
    def host_query(name):
        if name == "inner":
            return L.dj_distributed_inner_join_host_workspace_bytes(n, n, cap[name], 1, 1)
        fn = L.dj_distributed_left_filter_join_host_workspace_bytes if KINDS[name] in (1, 2) else \
            L.dj_distributed_outer_join_host_workspace_bytes
        return fn(n, n, cap[name], 1, 1)

    ws = dj.workspace(max(host_query(k) for k in cap))
    d_in = {k: torch.empty(n, dtype=torch.int64, device="cuda") for k in h}
    d_flat = torch.empty(4 * cap["full-outer"], dtype=torch.int64, device="cuda")
    d_sides = torch.empty(cap["full-outer"], dtype=torch.uint8, device="cuda")
    dev_ws = dj.workspace(max(L.dj_distributed_outer_join_workspace_bytes(n, n, 1, 1),
                              L.dj_distributed_left_filter_join_workspace_bytes(n, n, 1, 1)))

    def streamed(name):
        if name == "inner":  # the unique build table as left, as the benchmark calls it
            return dj.distributed_inner_join_host(None, h["rk"], h["rp"], h["lk"], h["lp"], h_outs(name), ws=ws)[0]
        if KINDS[name] in (1, 2):
            return dj.distributed_left_filter_join_host(None, KINDS[name], h["lk"], h["lp"], h["rk"], h_outs(name),
                                                        ws=ws)[0]
        return dj.distributed_outer_join_host(None, KINDS[name], h["lk"], h["lp"], h["rk"], h["rp"], h_outs(name),
                                              ws=ws)[0]

    def staged(name):
        kind, c = KINDS[name], cap[name]
        filt = kind in (1, 2)
        for k in (("lk", "lp", "rk") if filt else ("lk", "lp", "rk", "rp")):
            d_in[k].copy_(h[k], non_blocking=True)
        outs = [d_flat[i * c:(i + 1) * c] for i in range(2 if filt else 4)] + ([] if filt else [d_sides[:c]])
        if filt:
            r = dj.distributed_left_filter_join(None, kind, d_in["lk"], d_in["lp"], d_in["rk"], capacity=c, ws=dev_ws,
                                                outs=outs)
        else:
            r = dj.distributed_outer_join(None, kind, d_in["lk"], d_in["lp"], d_in["rk"], d_in["rp"], capacity=c,
                                          ws=dev_ws, outs=outs)
        for o, d in zip(h_outs(name), outs):
            o[:r.n_out].copy_(d[:r.n_out], non_blocking=True)
        torch.cuda.synchronize()
        return r.n_out

    def timed(fn, name):
        fn(name)  # warm-up
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(args.calls):
            fn(name)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3 / args.calls

    times = {("inner", "streamed"): []}
    n_out = {}
    for name in KINDS:
        times[(name, "streamed")], times[(name, "staged")] = [], []
    for _ in range(args.rounds):
        times[("inner", "streamed")].append(timed(streamed, "inner"))
        for name in KINDS:
            times[(name, "streamed")].append(timed(streamed, name))
            times[(name, "staged")].append(timed(staged, name))
    for name in cap:
        n_out[name] = streamed(name)

    # ---- per-category kernel time of the streamed calls, and the emit kernel's own time
    prof = {}
    for name in cap:
        dj.profile_enable(True)
        dj.profile_read()
        streamed(name)
        torch.cuda.synchronize()
        prof[name] = {c: round(ms, 3) for c, (ms, _) in dj.profile_read().items()}
        dj.profile_enable(False)
    emit_ms = None
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as tp:
        streamed("full-outer")
        torch.cuda.synchronize()
    for ev in tp.events():
        if "emit_unmatched_build_kernel" in ev.name:
            emit_ms = (emit_ms or 0.0) + (getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)) / 1e3
    n_right_only = ref["full-outer"]["right"][0]
    emit = {"ms": emit_ms, "bytes": 16 * n + n // 8 + 33 * n_right_only}  # rows and bits read, rows written
    if emit_ms:
        emit["gb_per_s"] = emit["bytes"] / (emit_ms * 1e-3) / 1e9

    # ---- parity at the timed size: the streamed host rows, uploaded, against the device entry's
    del dev_ws, d_in
    gc.collect()
    torch.cuda.empty_cache()
    parity = {}
    for name in KINDS:
        m = streamed(name)
        c = cap[name]
        ncols = 2 if name in ("semi", "anti") else 4
        cols = [d_flat[i * c:i * c + m].copy_(h_flat[i * c:i * c + m]) for i in range(ncols)]
        if ncols == 4:
            cols.append(d_sides[:m].copy_(h_sides[:m]))
        got = classes(name, cols, m)
        parity[name] = {k: {"count": got[k][0], "ref_count": ref[name][k][0], "ok": got[k] == ref[name][k]} for k in got}
        parity[name]["ok"] = m == sum(v[0] for v in got.values()) and all(v["ok"] for v in parity[name].values())

    ident = gpu_identity()
    for (name, how), ts in times.items():
        ms = statistics.median(ts)
        filt = name in ("semi", "anti")
        up = (3 if filt else 4) * n * 8
        down = n_out[name] * (16 if filt else 33 if name.endswith("outer") else 32)
        line = {"config": name, "path": how, "ms_per_call": round(ms, 2), "ms_rounds": [round(t, 2) for t in ts],
                "n_out": n_out[name], "bytes_up": up, "bytes_down": down,
                "link_gb_per_s": max(up, down) / (ms * 1e-3) / 1e9, "gpu": ident}
        if how == "streamed":
            line["kernel_ms"] = prof[name]
        print(json.dumps(line))
    print(json.dumps({"emit_unmatched_build_kernel": emit, "parity": parity, "rows": n, "gpu": ident,
                      "all_ok": all(v["ok"] for v in parity.values())}))


if __name__ == "__main__":
    main()
