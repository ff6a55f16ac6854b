"""Runs the product (libb200c.so through toplingdb_b200.CompactionJob) on a helpers.Params job."""
import struct

import toplingdb_b200 as T


def job_from_params(p, output_mem="host", **extra):
    kw = dict(output_level=p.output_level, bottommost_level=p.bottommost_level, max_output_file_size=p.max_output_file_size,
              block_size=p.block_size, block_size_deviation=p.block_size_deviation,
              block_restart_interval=p.block_restart_interval, index_block_restart_interval=p.index_block_restart_interval,
              format_version=p.format_version, checksum=p.checksum, snapshots=list(p.snapshots),
              column_family_id=p.column_family_id, column_family_name=p.column_family_name, db_id=p.db_id,
              db_session_id=p.db_session_id, db_host_id=p.db_host_id, creation_time=p.creation_time,
              oldest_key_time=p.oldest_key_time, file_creation_times=list(p.file_creation_times),
              first_file_number=p.first_file_number, output_mem=output_mem, compaction_filter=p.compaction_filter,
              ttl=p.ttl, ttl_now=p.now, grandparents=list(p.grandparents),
              level_compaction_dynamic_file_size=int(p.level_compaction_dynamic_file_size),
              max_compaction_bytes=p.max_compaction_bytes, target_output_file_size=p.target_output_file_size,
              range_start=p.range_start, range_end=p.range_end, bloom_millibits_per_key=p.bloom_millibits_per_key)
    kw.update(extra)
    return T.CompactionJob(**kw)


def run_product(p, inputs, device_inputs=False, levels=None, **extra):
    """levels: the level of every input (files of one level > 0, listed one after the other, form one sorted run); default: all L0"""
    job = job_from_params(p, **extra)
    keep = []
    for i, data in enumerate(inputs):
        lvl = 0 if levels is None else levels[i]
        if device_inputs:
            import torch
            t = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
            keep.append(t)
            job.add_input(t, level=lvl, file_number=i)
        else:
            job.add_input(data, level=lvl, file_number=i)
    job.run()
    files = job.outputs()
    metas = [job.output_meta(i) for i in range(job.output_count())]
    st = job.stats()
    job.close()
    return files, metas, st


def _describe(ikey, value):
    tr = struct.unpack("<Q", ikey[-8:])[0]
    return f"user key {ikey[:-8].hex() or '(empty)'} seq {tr >> 8} type {tr & 0xff} value {len(value)} B"


def assert_merged_matches(job, want, label=""):
    """job: after run(until=2); want: [(internal key, value)] of the oracle's compaction iterator over the merged inputs.  Compares the
    merge stage's output entry by entry and names the first one that differs (the input tile cannot be told from an output position;
    the key is what leads to it)."""
    recs = parse_key_recs(job.debug(T.native.DBG_MERGED_KEYS))
    vals = job.debug(T.native.DBG_MERGED_VALUES)
    off = 0
    for i, ((uk, tr, vlen), (ik, v)) in enumerate(zip(recs, want)):
        got_ik, got_v = uk + struct.pack("<Q", tr), vals[off:off + vlen]
        assert got_ik == ik and got_v == v, \
            f"{label}: merged entry {i} of {len(recs)} (oracle: {len(want)}) differs: device {_describe(got_ik, got_v)}, oracle {_describe(ik, v)}"
        off += vlen
    n = min(len(recs), len(want))
    assert len(recs) == len(want), f"{label}: device wrote {len(recs)} merged entries, oracle {len(want)}; the first {n} agree" + \
        ("" if n == 0 else f", the last of them {_describe(*want[n - 1])}")


def assert_decoded_matches(job, run, entries, label="", where=None):
    """job: after run(until=1); entries: [(internal key, value)] that run `run` must hold, in order; where: for every entry a dict
    (block, offset, phase, path) -- the block index in the file, the entry's offset in the block, the block's file offset mod 16 and
    the path the decoder is expected to take (decode_cases.located_entries).  Names the first entry that differs."""
    recs = parse_key_recs(job.debug(T.native.DBG_DECODED_KEYS, run))
    vals = job.debug(T.native.DBG_DECODED_VALUES, run)
    off = 0

    def at(i):
        if where is None or i >= len(where):
            return ""
        w = where[i]
        return f" (block {w['block']}, offset {w['offset']} in the block, phase {w['phase']}, expected path {w['path']})"
    for i, ((uk, tr, vlen), (ik, v)) in enumerate(zip(recs, entries)):
        got_ik, got_v = uk + struct.pack("<Q", tr), vals[off:off + vlen]
        assert got_ik == ik and got_v == v, \
            f"{label}: run {run} entry {i}{at(i)} differs: device {_describe(got_ik, got_v)}, table {_describe(ik, v)}"
        off += vlen
    n = min(len(recs), len(entries))
    assert len(recs) == len(entries), f"{label}: run {run} decoded {len(recs)} entries, the table holds {len(entries)}; the first {n} agree" + \
        ("" if n == len(entries) else f"; the next one is{at(n)}")


def parse_key_recs(b):
    """32-byte debug records -> list of (user_key bytes, trailer, vlen)"""
    out = []
    for i in range(0, len(b), 32):
        hi, lo, tr, ulen, vlen = struct.unpack_from("<QQQII", b, i)
        uk = struct.pack(">QQ", hi, lo)[:ulen]
        out.append((uk, tr, vlen))
    return out
