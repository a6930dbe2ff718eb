"""profile_step.py — where the time of bench.py's timed region goes, kernel by kernel (torch.profiler, CUDA activities).

  python -m krakenuniq_b200.profile_step --out DIR [--steps 10] [--warmup 3]

Builds the configs[1] workload exactly as bench.py's replicas arm does (same generator, seeds, read pool, Classifier
with 3 slots, hll_mode 0, per-batch work units) and replays its order: warm-up steps, finish(), then the timed region of
K steps + finish() — here under the profiler.  Writes to DIR:

  kernels.txt     torch.profiler's per-kernel table (device time)
  summary.json    per-kernel ms per step, the busy / idle split of the region from the trace, the card, its power limit
                  and the random-sector gather peak
  trace.json      the Chrome trace of the region

A second, unprofiled round (K more steps, then finish()) gives the steps and the harvest by CUDA events, and counts the
32-byte record sectors the harvest has to write back (sectors holding a flagged record): the harvest's bytes / s.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

import bench  # noqa: E402  (workload generation and constants are bench.py's own)


def card_info(index=0):
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                            "-i", str(index)], capture_output=True, text=True, timeout=30)
        name, power, clock = [x.strip() for x in r.stdout.strip().split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:  # noqa: BLE001
        return {"error": str(e)[:200]}


def trace_breakdown(trace_path, n_steps):
    """kernel / memset / memcpy intervals of the trace: time per name, and how much of the region's span they cover"""
    ev = json.load(open(trace_path))
    ev = ev["traceEvents"] if isinstance(ev, dict) else ev
    dev = [e for e in ev if e.get("ph") == "X" and e.get("cat") in ("kernel", "gpu_memset", "gpu_memcpy")]
    if not dev:
        return {"error": "no device events in the trace"}
    per = defaultdict(lambda: [0.0, 0])
    iv = []
    for e in dev:
        per[(e["cat"], e["name"])][0] += e["dur"]
        per[(e["cat"], e["name"])][1] += 1
        iv.append((e["ts"], e["ts"] + e["dur"]))
    iv.sort()
    busy, cur_s, cur_e = 0.0, iv[0][0], iv[0][1]
    for s, e in iv[1:]:
        if s > cur_e:
            busy += cur_e - cur_s
            cur_s, cur_e = s, e
        else:
            cur_e = max(cur_e, e)
    busy += cur_e - cur_s
    span = iv[-1][1] - iv[0][0]
    rows = sorted(({"kind": k[0], "name": k[1][:120], "calls": c, "total_ms": t / 1e3, "ms_per_step": t / 1e3 / n_steps}
                   for k, (t, c) in per.items()), key=lambda r: -r["total_ms"])
    return {"span_ms": span / 1e3, "busy_ms": busy / 1e3, "idle_ms": (span - busy) / 1e3, "by_name": rows}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for kernels.txt, summary.json and trace.json")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--no-gather-peak", action="store_true")
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    from krakenuniq_b200 import binding

    if not torch.cuda.is_available():
        raise SystemExit("profile_step.py needs a GPU")
    os.makedirs(args.out, exist_ok=True)
    dev = "cuda:0"
    torch.cuda.set_device(0)
    # bench.py's defaults for everything that shapes the workload
    bargs = argparse.Namespace(db_records=0, db_passes=0, genomes=2000, reads=10_000_000, batch_reads=1_000_000,
                               hll_mode=0, warmup=args.warmup, steps=args.steps)
    B, L = bargs.batch_reads, bench.READ_LEN
    steps_rep = (args.warmup + args.steps) + 5 + (max(args.warmup, 3) + args.steps)
    w = bench.build_workload(bargs, "replicas", 0, 1, dev, None, steps_rep)
    db, pool = w.db, w.pool_bases
    n_batches = w.n_pool // B
    clf = binding.Classifier(device=0, n_slots=3, max_reads=B, max_bases=B * L + 4096, hll_mode=0,
                             sparse_set_slots=1 << 31)
    clf.attach_db_device(db.records.data_ptr(), db.key_ct, db.offsets.data_ptr(), bench.K, bench.NT, 2)
    clf.set_taxonomy(*db.parent_map())
    d_offsets = torch.arange(B + 2, dtype=torch.int64, device=dev) * L
    per_unit = -(-500000 // L)
    units_per_batch = -(-B // per_unit)
    unit_local = (torch.arange(B, dtype=torch.int64, device=dev) // per_unit).to(torch.int32)
    unit_bufs = {}

    def d_units(i):
        t = unit_local + i * units_per_batch
        unit_bufs[i % 8] = t
        return t.data_ptr()

    def step_fn(i):
        clf.classify_device(0, pool.data_ptr() + (i % n_batches) * B * L, d_offsets.data_ptr(), B, B * L, d_units(i))

    stream = torch.cuda.ExternalStream(clf.slot_stream(0), device=dev)
    step = 0
    for _ in range(args.warmup):
        step_fn(step); step += 1
    clf.sync(0)
    clf.finish()
    torch.cuda.synchronize()

    # ---- profiled region: bench.py's timed region (K steps + the end-of-run harvest) ------------------------------
    launches0 = clf.launch_count()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            step_fn(step); step += 1
        clf.finish()
        clf.sync(0)
        torch.cuda.synchronize()
    launches = clf.launch_count() - launches0
    harvest_profiled = clf.sparse_tier_info()["last_harvest_ms"]
    trace = os.path.join(args.out, "trace.json")
    prof.export_chrome_trace(trace)
    with open(os.path.join(args.out, "kernels.txt"), "w") as f:
        f.write(prof.key_averages().table(sort_by="self_device_time_total", row_limit=60, max_name_column_width=90))

    # ---- second round, unprofiled: steps and harvest by CUDA events; sectors the harvest writes back --------------
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    with torch.cuda.stream(stream):
        ev[0].record(stream)
    for _ in range(args.steps):
        step_fn(step); step += 1
    with torch.cuda.stream(stream):
        ev[1].record(stream)
    clf.sync(0)
    torch.cuda.synchronize()
    hi = db.records.view(torch.int32).view(-1, 3)[:, 1]
    flagged = torch.nonzero(hi < 0).squeeze(1)                 # SEEN_BIT is the sign bit of the record's high key word
    n_flagged = int(flagged.numel())
    dirty_sectors = int(torch.unique_consecutive((flagged * 12 + 4) // 32).numel()) if n_flagged else 0
    del hi, flagged
    torch.cuda.synchronize()
    with torch.cuda.stream(stream):
        ev[2].record(stream)
    clf.finish()
    with torch.cuda.stream(stream):
        ev[3].record(stream)
    clf.sync(0)
    torch.cuda.synchronize()
    steps_ms, finish_ms = ev[0].elapsed_time(ev[1]), ev[2].elapsed_time(ev[3])
    harvest_ms = clf.sparse_tier_info()["last_harvest_ms"]
    rec_bytes = db.key_ct * 12
    peaks = {}
    try:
        peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
    except Exception:  # noqa: BLE001
        pass
    hbm_peak = float(peaks["hbm_gbs"]) if "hbm_gbs" in peaks else bench.HBM_DATASHEET_GBS
    moved = rec_bytes + 32 * dirty_sectors

    gather = None
    if not args.no_gather_peak:
        try:
            gs, gb, _ = binding.random_gather_peak(0, 16 << 30, 1 << 29, 32)
            gather = {"gsectors_per_s": gs, "gb_per_s": gb}
        except Exception as e:  # noqa: BLE001
            gather = {"error": str(e)[:200]}

    summary = {
        "card": card_info(0),
        "workload": w.workload,
        "steps": args.steps,
        "profiled_region": {"launches": launches, "harvest_ms": harvest_profiled,
                            "trace": trace_breakdown(trace, args.steps)},
        "unprofiled_round": {"steps_ms": steps_ms, "ms_per_step": steps_ms / args.steps,
                             "steps_mreads_s": B * args.steps / steps_ms / 1e3, "finish_ms": finish_ms,
                             "harvest_ms": harvest_ms, "records": db.key_ct, "flagged_records": n_flagged,
                             "dirty_sectors": dirty_sectors,
                             "harvest_bytes": moved,
                             "harvest_gb_per_s": moved / (harvest_ms / 1e3) / 1e9 if harvest_ms else None,
                             "hbm_peak_gb_per_s": hbm_peak,
                             "hbm_peak_source": "MEASURED_PEAKS.json hbm_gbs" if "hbm_gbs" in peaks
                             else "H100 SXM data sheet (3350 GB/s)",
                             "how": "bytes = every record read once + one 32-byte write-back per sector holding a "
                                    "flagged record; harvest_ms = device time of kuq_finish's harvest"},
        "random_gather_peak": gather,
    }
    json.dump(summary, open(os.path.join(args.out, "summary.json"), "w"), indent=1)
    t = summary["profiled_region"]["trace"]
    print(json.dumps({"card": summary["card"], "span_ms": t.get("span_ms"), "idle_ms": t.get("idle_ms"),
                      "harvest_ms": harvest_profiled, "unprofiled": summary["unprofiled_round"],
                      "gather": gather}))
    for r in t.get("by_name", [])[:25]:
        print(f"{r['ms_per_step']:9.4f} ms/step {r['calls']:6d} calls  {r['kind']:10s} {r['name']}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
