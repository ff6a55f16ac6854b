"""Measures what the optional parts of the compaction path cost on the bench workload (BASELINE.json configs[1], cfg2: 8 x 256 MiB runs,
16 B keys / 32 B values): the same job with a Bloom filter policy, with paranoid_file_checks, with grandparent files, clipped to a
quarter of the key space, and with a fixed-prefix SST partitioner, each timed on the device with the per-kernel events of `profile=1`.
cfg2's keys share their first byte, split into ~580 groups on their first 3 bytes and are unique in their first 8: the partitioner arms
are a job the walk descends into nowhere (len 1), one with ~580 partition cuts (len 3), and one the device refuses (len 8: an event at
every entry), timed from the run call to the refusal.  Prints one JSON object:
`python tools/feature_cost.py > feature_cost.json` on the GPU to be measured."""
import json
import os
import statistics
import struct
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import torch
    import toplingdb_b200 as T
    from toplingdb_b200 import synth
    scale = float(os.environ.get("FEATURE_COST_SCALE", "1.0"))
    k, vlen = 8, 32
    n_total = int((256 << 20) * scale) // 56 * k
    images, kv_bytes = synth.stage_runs(n_total, k, vlen, key_base=0, seed=2, device_index=0)
    common = dict(device=0, output_level=1, bottommost_level=False, max_output_file_size=64 << 20, file_creation_times=[1700000000],
                  first_file_number=1, db_id="bench", db_session_id="BENCH", db_host_id="b200", output_mem="device", profile=1)

    def key(idx):  # synth.make_run_columns: high word = (key_base + index) * KEY_MULT
        return struct.pack(">QQ", idx * synth.KEY_MULT, 0)

    gps = []
    ngp = 64
    for i in range(ngp):  # 64 grandparent files of 48 MiB tiling the key space, small gaps between them
        a, b = n_total * i // ngp, n_total * (i + 1) // ngp - 1000
        gps.append((key(a), key(b), 48 << 20))
    variants = {
        "baseline": {},
        "bloom_10_bits": dict(bloom_millibits_per_key=10000),
        "paranoid_file_checks": dict(paranoid_file_checks=1),
        "grandparents_64": dict(grandparents=gps, max_output_file_size=128 << 20, target_output_file_size=64 << 20,
                                level_compaction_dynamic_file_size=1),
        "range_second_quarter": dict(range_start=key(n_total // 4), range_end=key(n_total // 2)),
        "partitioner_len1": dict(sst_partitioner_prefix_len=1),
        "partitioner_len3": dict(sst_partitioner_prefix_len=3),
    }
    out = {"workload": "cfg2", "scale": scale, "input_kv_bytes": kv_bytes, "variants": {}}
    for name, extra in variants.items():
        job = T.CompactionJob(**dict(common, **extra))
        for i, img in enumerate(images):
            job.add_input(img, level=0, file_number=100 + i)
        for _ in range(2):
            job.run()
        tot, kt = [], {}
        for _ in range(3):
            job.run()
            tot.append(job.stats().total_us)
            for kn, us in job.kernel_times():
                kt.setdefault(kn, []).append(us)
        st = job.stats()
        out["variants"][name] = {
            "total_us": round(statistics.mean(tot), 1), "output_files": job.output_count(), "num_input_records": st.num_input_records,
            "num_output_records": st.num_output_records, "kernel_launches": st.kernel_launches,
            "kernels_us": {kn: round(statistics.mean(v), 1) for kn, v in sorted(kt.items(), key=lambda x: -statistics.mean(x[1]))}}
        job.close()
        torch.cuda.synchronize()
    import time
    job = T.CompactionJob(**dict(common, sst_partitioner_prefix_len=8))
    for i, img in enumerate(images):
        job.add_input(img, level=0, file_number=100 + i)
    refusal = []
    for _ in range(3):
        t0 = time.perf_counter()
        try:
            job.run()
            code = 0
        except T.B200cError as e:
            code = e.code
        refusal.append((time.perf_counter() - t0) * 1e6)
    out["variants"]["partitioner_len8_refused"] = {"status": code, "wall_us_to_refusal": round(statistics.mean(refusal), 1)}
    job.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
