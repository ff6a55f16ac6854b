#!/usr/bin/env python
"""Turns an ncu launch list (`ncu --metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum --csv`) of a bench run
into (1) the launches of the LAST job (one row per launch), (2) a per-kernel summary with shares and DRAM bytes, (3) profiles/ncu_traffic.json
(DRAM bytes per bench kernel group, stamped with the digest of the CUDA sources so that bench.py only reports it for the same build).

usage: tools/ncu_launch_summary.py <ncu.csv> <tag>      -> profiles/<tag>_ncu_launches_last_step.csv, profiles/<tag>_ncu_launch_summary.json"""
import csv
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
GROUP = {  # kernel -> bench.py kernel group
    "index_decode_kernel": "decode.index", "block_decode_fused_kernel": "decode.blocks", "merge_partition_grouped_kernel": "merge.partition",
    "merge_partition_kernel": "merge.partition", "merge_tiles_kernel": "merge.tiles", "merge_sizes_fix_kernel": "merge.sizes_fix",
    "encode_tables_kernel": "encode.tables", "encode_stitch_kernel": "~encode.stitch", "encode_tilestate_kernel": "encode.tilestate",
    "encode_blocklist_kernel": "encode.blocklist", "encode_emit_kernel": "encode.emit", "encode_filestats_kernel": "~encode.filestats+index",
    "encode_index_size_kernel": "~encode.filestats+index",
    "encode_index_write_kernel": "~encode.filestats+index", "file_block_contrib_kernel": "~encode.filestats+index",
    "file_block_trailer_kernel": "~encode.filestats+index", "scan_tile_sums": "~encode.filestats+index", "scan_of_sums": "~encode.filestats+index",
    "scan_downsweep": "~encode.filestats+index", "run_bounds_kernel": "merge.partition",
}


def main():
    path, tag = sys.argv[1], sys.argv[2]
    rows = []
    hdr = None
    for r in csv.reader(open(path, errors="replace")):
        if hdr is None:
            if r and r[0] == "ID":
                hdr = r
            continue
        if len(r) != len(hdr):
            continue
        rows.append(dict(zip(hdr, r)))
    # long format: one row per (launch, metric)
    launches = {}
    for r in rows:
        k = int(r["ID"])
        name = r["Kernel Name"].split("(")[0].split("<")[0].replace("void ", "").replace("b200c::", "")
        e = launches.setdefault(k, {"kernel": name, "grid": r.get("Grid Size", ""), "block": r.get("Block Size", "")})
        v = float(r["Metric Value"].replace(",", ""))
        unit = r.get("Metric Unit", "")
        m = r["Metric Name"]
        if m == "gpu__time_duration.sum":
            e["time_us"] = v / 1e3 if unit in ("ns", "nsecond") else (v * 1e3 if unit in ("ms", "msecond") else v)
        elif m == "dram__bytes_read.sum":
            e["dram_read_bytes"] = v * {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}.get(unit, 1)
        elif m == "dram__bytes_write.sum":
            e["dram_write_bytes"] = v * {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}.get(unit, 1)
    ids = sorted(launches)
    # the last job = from the last index_decode_kernel launch on
    last = max((i for i in ids if launches[i]["kernel"] == "index_decode_kernel"), default=ids[0])
    job = [launches[i] for i in ids if i >= last]
    os.makedirs(os.path.join(ROOT, "profiles"), exist_ok=True)
    with open(os.path.join(ROOT, "profiles", f"{tag}_ncu_launches_last_step.csv"), "w") as f:
        f.write("kernel,grid,block,time_us,dram_read_bytes,dram_write_bytes\n")
        for e in job:
            f.write('%s,"%s","%s",%.2f,%d,%d\n' % (e["kernel"], e["grid"], e["block"], e.get("time_us", 0), e.get("dram_read_bytes", 0), e.get("dram_write_bytes", 0)))
    total = sum(e.get("time_us", 0) for e in job)
    summ, traffic = {}, {}
    for e in job:
        s = summ.setdefault(e["kernel"], {"launches": 0, "us": 0.0, "dram_read_bytes": 0, "dram_write_bytes": 0})
        s["launches"] += 1
        s["us"] += e.get("time_us", 0)
        s["dram_read_bytes"] += int(e.get("dram_read_bytes", 0))
        s["dram_write_bytes"] += int(e.get("dram_write_bytes", 0))
        g = GROUP.get(e["kernel"])
        if g:
            traffic[g] = traffic.get(g, 0) + int(e.get("dram_read_bytes", 0)) + int(e.get("dram_write_bytes", 0))
    for s in summ.values():
        s["us"] = round(s["us"], 1)
        s["share"] = round(s["us"] / total, 4) if total else 0
    out = {"source": f"ncu launch list {os.path.basename(path)} (cfg2 full size, last job of the run; cold-cache serialised launches: compare shares)",
           "sum_us": round(total, 1), "dram_bytes_total": sum(s["dram_read_bytes"] + s["dram_write_bytes"] for s in summ.values()),
           "kernels": dict(sorted(summ.items(), key=lambda kv: -kv[1]["us"]))}
    json.dump(out, open(os.path.join(ROOT, "profiles", f"{tag}_ncu_launch_summary.json"), "w"), indent=1)
    from bench import source_sha16
    traffic["_source"] = f"profiles/{tag}_ncu_launch_summary.json (dram__bytes_read.sum + dram__bytes_write.sum per launch, cfg2 full size)"
    traffic["lib_source_sha16"] = source_sha16()
    json.dump(traffic, open(os.path.join(ROOT, "profiles", "ncu_traffic.json"), "w"), indent=1)
    print(json.dumps({"sum_us": out["sum_us"], "dram_GB": out["dram_bytes_total"] / 1e9}, indent=1))


if __name__ == "__main__":
    main()
