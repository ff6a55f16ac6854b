"""Timeline of the encode stage on the bench job: where the stage's time goes that belongs to no kernel on the job's main stream.

Stages the job the way bench.py does (synth.stage_bench_inputs, BENCH_JOB, profile=1, device-resident inputs), warms it up, then traces
`--steps` runs with torch.profiler (CUDA activities) in a run of their own.  For each step it prints the library's kernels on the job's
two streams in time order, the idle gap in front of each main-stream kernel, and attributes the encode stage's idle time:

- sync1:  end of the merge (merge_sizes_fix_kernel) -> first encode kernel: the host reads the survivor count and sizes the encoder
- stitch: end of encode_tables_kernel -> encode_tilestate_kernel: the stitch walk (side stream) running past the tables kernel
- sync2:  last kernel of the block cut -> encode_blocklist_kernel: block / file counts read back, output layout, small uploads
- sync3:  last main-stream encode kernel -> end of scatter_tails_kernel: per-file records read back, tails built, scatter, and any
          wait for the side stream's index kernels (reported apart as `side_trail`)

Helper launches (small gathers / copies, the tail scatter, memsets) count as idle time: they are part of the host round trips.  Tracing slows the host a
little, so the gaps here are upper bounds of the untraced ones; `bench.py` gives the untraced step time.  Prints the card name and power
limit first.  `python tools/stage_timeline.py [--workload cfg2] [--json out.json]` on the GPU to be measured."""
import argparse
import json
import os
import re
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HELPERS = ("gather_small_kernel", "copy_small_kernel", "scatter_tails_kernel", "[memset]", "[memcpy]")
BUCKETS = ("sync1", "stitch", "sync2", "sync3", "other")


def card():
    try:
        q = "name,power.limit,clocks.sm,clocks.max.sm"
        return subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except Exception as e:  # the timeline itself does not need it
        return f"unknown ({e})"


def short(name):
    """`void b200c::(anonymous namespace)::encode_tables_kernel<unsigned int>(...)` -> `encode_tables_kernel`"""
    s = name.split("(")[0] if not name.startswith("(") else name
    s = re.sub(r"<.*>$", "", s.strip())
    return s.split("::")[-1].split(" ")[-1]


def load_trace(path):
    evs = json.load(open(path))
    evs = evs.get("traceEvents", evs)
    out = []
    for e in evs:
        cat = e.get("cat", "")
        if cat not in ("kernel", "gpu_memset", "gpu_memcpy") or "dur" not in e:
            continue
        a = e.get("args", {})
        nm = short(e["name"]) if cat == "kernel" else ("[memset]" if cat == "gpu_memset" else "[memcpy]")
        out.append({"name": nm, "ts": float(e["ts"]), "end": float(e["ts"]) + float(e["dur"]), "stream": a.get("stream")})
    out.sort(key=lambda x: x["ts"])
    return out


def busy(evs, t0, t1, work_only):
    """union of the intervals of `evs` clipped to [t0, t1] (work_only: without the helper launches)"""
    iv = sorted((max(e["ts"], t0), min(e["end"], t1)) for e in evs
                if e["end"] > t0 and e["ts"] < t1 and not (work_only and e["name"] in HELPERS))
    tot, cur_a, cur_b = 0.0, None, None
    for a, b in iv:
        if cur_b is None or a > cur_b:
            if cur_b is not None:
                tot += cur_b - cur_a
            cur_a, cur_b = a, b
        else:
            cur_b = max(cur_b, b)
    if cur_b is not None:
        tot += cur_b - cur_a
    return tot


def analyse(evs, verbose=True):
    main_s = next(e["stream"] for e in evs if e["name"] == "encode_tables_kernel")
    side_s = next((e["stream"] for e in evs if e["name"] == "encode_stitch_kernel"), None)
    main = [e for e in evs if e["stream"] == main_s]
    side = [e for e in evs if e["stream"] == side_s] if side_s is not None else []
    anchors = [i for i, e in enumerate(main) if e["name"] == "merge_sizes_fix_kernel"]
    steps = []
    for a in anchors:
        end_i = next((i for i in range(a + 1, len(main)) if main[i]["name"] == "scatter_tails_kernel"), None)
        if end_i is None:
            continue
        seg = main[a:end_i + 1]
        t0, t_end = seg[0]["end"], seg[-1]["end"]
        sd = [e for e in side if e["ts"] >= t0 and e["ts"] < t_end]

        def first(name):
            return next((e for e in seg if e["name"] == name), None)

        def idle(ta, tb):  # main-stream time in [ta, tb] without a work kernel
            return max(0.0, (tb - ta) - busy(seg, ta, tb, True)) if tb > ta else 0.0

        work = [e for e in seg[1:] if e["name"] not in HELPERS]
        tables, tilestate, blocklist = first("encode_tables_kernel"), first("encode_tilestate_kernel"), first("encode_blocklist_kernel")
        first_enc = work[0]
        last_cut = max((e for e in work if e["end"] <= blocklist["ts"]), key=lambda e: e["end"])
        last_work = max(work, key=lambda e: e["end"])
        b = {
            "sync1": idle(t0, first_enc["ts"]),
            "stitch": idle(tables["end"], tilestate["ts"]),
            "sync2": idle(last_cut["end"], blocklist["ts"]),
        }
        side_end = max((e["end"] for e in sd), default=0.0)
        side_trail = max(0.0, min(side_end, t_end) - last_work["end"])
        b["sync3"] = idle(last_work["end"], t_end)
        total_idle = idle(t0, t_end)
        b["other"] = total_idle - sum(b.values())
        step = {"encode_span_us": t_end - t0, "main_work_us": busy(seg[1:], t0, t_end, True), "idle_us": total_idle,
                "side_trail_us": side_trail, "stitch_end_minus_tables_end_us": None, "gaps_us": b}
        st = [e for e in sd if e["name"] == "encode_stitch_kernel"]
        if st:
            step["stitch_end_minus_tables_end_us"] = max(e["end"] for e in st) - tables["end"]
        if verbose:
            print(f"-- step {len(steps)}: encode span {step['encode_span_us']:.1f} us, main-stream work {step['main_work_us']:.1f} us, "
                  f"idle {total_idle:.1f} us")
            rows = sorted([(e, "main") for e in seg] + [(e, "side") for e in sd], key=lambda x: x[0]["ts"])
            prev_end = None
            for e, s in rows:
                gap = ""
                if s == "main":
                    if prev_end is not None:
                        gap = f"{max(0.0, e['ts'] - prev_end):9.1f}"
                    prev_end = max(prev_end or 0.0, e["end"])
                print(f"   {s:4s} {e['ts'] - t0:10.1f} {e['end'] - e['ts']:9.1f} {gap:>9s}  {e['name']}")
            print("   gaps (us): " + ", ".join(f"{k} {v:.1f}" for k, v in b.items()) + f"; side_trail {side_trail:.1f}")
        steps.append(step)
    return steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="cfg2")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--json", help="also write the per-step numbers here")
    ap.add_argument("--quiet", action="store_true", help="no per-kernel listing")
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    import toplingdb_b200 as T
    from toplingdb_b200 import synth
    from toplingdb_b200.synth_workloads import BENCH_JOB, WORKLOADS
    print("card:", card())
    w = WORKLOADS[args.workload]
    images, _ = synth.stage_bench_inputs(args.workload, rank=0, scale=1.0, device_index=0)
    job = T.CompactionJob(output_mem="device", profile=1, device=0, bottommost_level=w["bottommost"], **BENCH_JOB)
    for i, img in enumerate(images):
        job.add_input(img, level=0, file_number=100 + i)
    for _ in range(args.warmup):
        job.run()
    torch.cuda.synchronize()
    stage = []
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            job.run()
            s = job.stats()
            stage.append({"encode_us": s.encode_us, "total_us": s.total_us, "launches": s.kernel_launches,
                          "kernels": dict(job.kernel_times())})
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, "trace.json")
        prof.export_chrome_trace(path)
        evs = load_trace(path)
    steps = analyse(evs, verbose=not args.quiet)
    for s, g in zip(steps, stage):
        main_groups = sum(us for k, us in g["kernels"].items() if k.startswith("encode.") and not k.startswith("~"))
        s["stage_us_encode"] = g["encode_us"]
        s["stage_minus_main_groups_us"] = g["encode_us"] - main_groups
        s["kernel_launches"] = g["launches"]
    summ = {k: statistics.median(s["gaps_us"][k] for s in steps) for k in BUCKETS}
    res = {"card": card(), "workload": args.workload, "steps": steps, "median_gaps_us": summ,
           "median_idle_us": statistics.median(s["idle_us"] for s in steps),
           "median_side_trail_us": statistics.median(s["side_trail_us"] for s in steps),
           "median_stage_minus_main_groups_us": statistics.median(s["stage_minus_main_groups_us"] for s in steps)}
    print(json.dumps({k: v for k, v in res.items() if k != "steps"}))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
