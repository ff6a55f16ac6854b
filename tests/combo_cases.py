"""Jobs that switch the device path's optional parts on together, as a DB does: one job per row of a pairwise covering array over the
factors below, so that every pair of levels of every two factors meets in at least one job.

Every job is built from one seeded key set: user keys of 0-16 bytes with zero-padding ties (`ab`, `ab\\0`, `ab\\0\\0`), two-byte prefixes
from a small alphabet (so a 2-byte partitioner cuts a few times and a 16-byte one at every user key), a hot key whose versions span
data blocks of one run (the index of that run keeps sequence numbers), SingleDelete / Put pairs, deletions, empty values and values
that carry a DBWithTTL write time.  The inputs are either built by the oracle (format_version 3, 4 and 5 mixed in one job) or written
by the compiled reference with kZlibCompression (`helpers.run_reference(input_compression="zlib")`, as decode_cases.inflate_case does;
the same ops in the same order, so the sequence numbers are the planned ones).

The checker is `partition_cases.oracle_compact` (helpers.oracle_compact for jobs without a partitioner; key ranges and grandparents
included).  Only the product's own options (`paranoid_file_checks`, input residency, `output_mem`) are not seen by the checker: they
must not change the output."""
import copy
import functools
import itertools
import os
import random
import re
import struct

import helpers as H
import partition_cases as PC
import sstfmt

VALUE, DELETION, SINGLE_DELETION = 1, 0, 7


def _constant(name):
    src = open(os.path.join(H.ROOT, "toplingdb_b200", "csrc", "kernels.h")).read()
    return int(re.search(r"constexpr\s+\w+\s+%s\s*=\s*(\d+)\s*;" % name, src).group(1))


MERGE_TILE = _constant("kMergeTile")
STITCH_GROUP = _constant("kEncTile") * _constant("kEncGroupTiles")  # entries of one stitch group of the block-cut planner

FACTORS = {
    "inputs": ("oracle", "zlib"),  # oracle-built, format_version 3 / 4 / 5 mixed | reference-written kZlibCompression
    "runs": ("l0", "l0+level"),  # L0 files only | L0 files plus one level of three files
    "single_delete": (0, 1),
    "snapshots": (0, 3, 17),
    "bottommost": (0, 1),
    "filter": ("none", "remove_empty_value", "ttl"),
    "grandparents": ("none", "dynamic", "static"),  # level_compaction_dynamic_file_size on / off
    "prefix_len": (0, 2, 16),
    "range": ("none", "start", "end", "both"),
    "bloom": (0, 10),
    "format": ((5, "xxh3"), (4, "crc32c"), (3, "none")),  # output format_version, checksum
    "paranoid": (0, 1),
    "output_level": (0, 1),
    "residency": ("host", "device", "deferred"),  # deferred: host images uploaded range by range, the job run as a sub-job
    "output_mem": ("host", "device"),
}
NAMES = tuple(FACTORS)

# pairs no job may hold, each with its reason.  Output level 0 with a partitioner or grandparents is allowed on purpose: the outputs
# must still match, the partitioner and the cuts being ignored there (compaction_outputs.cc:793-795).
EXCLUDED = [
    (("bloom", 10), ("format", (4, "crc32c")), "a Bloom filter block needs format_version 5 (FastLocalBloom): b200c_job_create refuses it"),
    (("bloom", 10), ("format", (3, "none")), "a Bloom filter block needs format_version 5 (FastLocalBloom): b200c_job_create refuses it"),
    (("residency", "deferred"), ("range", "none"), "host-deferred inputs are uploaded range by range for a sub-job: it needs a key range"),
]
SEED = 20261018
CANDIDATES = 40


def _allowed(row):
    return not any(row.get(a[0]) == a[1] and row.get(b[0]) == b[1] for a, b, _ in EXCLUDED)


def all_pairs():
    """every pair of levels of two factors that a job may hold"""
    out = set()
    for (i, f), (j, g) in itertools.combinations(enumerate(NAMES), 2):
        for a in FACTORS[f]:
            for b in FACTORS[g]:
                if _allowed({f: a, g: b}):
                    out.add(((f, a), (g, b)))
    return out


def row_pairs(row):
    return {((f, row[f]), (g, row[g])) for f, g in itertools.combinations(NAMES, 2)}


@functools.lru_cache(maxsize=None)
def covering_array():
    """greedy pairwise covering array (AETG-style, deterministic under SEED): each new row is the best of CANDIDATES rows, every
    candidate filling the factors in a random order with the level that covers the most still uncovered pairs"""
    rnd = random.Random(SEED)
    todo = all_pairs()
    rows = []
    while todo:
        best, gain = None, -1
        for _ in range(CANDIDATES):
            order = list(NAMES)
            rnd.shuffle(order)
            row = {}
            for f in order:
                scored = []
                for lv in FACTORS[f]:
                    row[f] = lv
                    if not _allowed(row):
                        continue
                    n = sum(1 for g in row if g != f and (((f, lv), (g, row[g])) in todo or ((g, row[g]), (f, lv)) in todo))
                    scored.append((n, rnd.random(), lv))
                del row[f]
                row[f] = max(scored)[2]
            g = len(row_pairs(row) & todo)
            if g > gain:
                best, gain = dict(row), g
        rows.append(best)
        todo -= row_pairs(best)
    return tuple(tuple(sorted(r.items(), key=lambda kv: NAMES.index(kv[0]))) for r in rows)


def rows():
    return [dict(r) for r in covering_array()]


# ------------------------------------------------------------------------------------------------ the data
NRUNS_L0 = 6
LEVEL_FILES = 3
HOT_VERSIONS = 20  # one run holds 20 versions of 500 bytes: they span data blocks (and stay below the SingleDelete path's 32-entry move)
T0, TTL = 1_700_000_000, 1000


def _user_keys(rnd, n):
    """n distinct user keys of 0-16 bytes; every eighth short enough one also with one and two zero bytes appended"""
    ks = {b"", b"a", b"a\0", b"b", b"bx", b"bx\0", b"c\0", b"c\0\0"}
    while len(ks) < n:
        k = bytes([rnd.choice(b"abc"), rnd.choice(b"\0xy")]) + rnd.randbytes(rnd.randint(0, 14))
        ks.add(k)
        if len(k) <= 14 and rnd.random() < 0.125:
            ks |= {k + b"\0", k + b"\0\0"}
    return sorted(ks)[:n]


_WORDS = [b"compaction", b"level", b"block", b"table", b"snapshot", b"filter", b"index", b"range", b"tile", b"merge"]


def _value(rnd, ts, n=None):
    """texty bytes (zlib compresses them) or, one in ten, random ones; the last four bytes are a DBWithTTL write time"""
    if n is None:
        if rnd.random() < 0.06:
            return b""
        n = rnd.randint(4, 120)
    body = bytes(rnd.randbytes(n)) if rnd.random() < 0.1 else b" ".join(rnd.choice(_WORDS) for _ in range(n // 6 + 1))[:n]
    return body + struct.pack("<I", ts)


@functools.lru_cache(maxsize=None)
def plan(seed, nkeys, per_run):
    """runs oldest first: [[(user key, seq, type, value)]], the hot key, the last seq, the user keys and the seq intervals [put, sd) of
    the "tight" SingleDeletes.  Seqs follow the write order, which the reference's DB assigns the same way (every op of the script
    takes the next one): a run writes its tight SingleDeletes first, then its keys in order, then the Puts of next run's tight
    SingleDeletes, so that a snapshot set can leave those pairs unseparated."""
    rnd = random.Random(seed)
    keys = _user_keys(rnd, nkeys)
    hot = keys[2 * len(keys) // 3 + 7]
    sd_keys = sorted(rnd.sample([k for k in keys if k != hot], nkeys // 20))
    tight = set(sd_keys[::3])
    sd_put_run = {k: rnd.randrange(1, NRUNS_L0) for k in sd_keys}  # the run of the Put a SingleDelete of the next run deletes
    plain = [k for k in keys if k not in tight and k != hot and k not in sd_put_run]
    runs, seq, put_seq, intervals = [], 1, {}, []
    for r in range(NRUNS_L0 + 1):  # run 0 is the level (three files)
        ts = T0 + 300 * r  # write time: the older runs are stale at the compaction's clock
        chosen = set(rnd.sample(plain, min(len(plain), per_run * (2 if r == 0 else 1))))
        sd_here = {k for k in sd_keys if sd_put_run[k] + 1 == r}
        put_here = {k for k in sd_keys if sd_put_run[k] == r}
        order = sorted(sd_here & tight) + sorted(chosen | (sd_here - tight) | (put_here - tight) | ({hot} if r == 3 else set())) + \
            sorted(put_here & tight)
        ents = []
        for k in order:
            n = HOT_VERSIONS if k == hot else 1
            for _ in range(n):
                if k == hot:
                    ents.append((k, seq, VALUE, _value(rnd, ts, 500)))
                elif k in sd_here:
                    ents.append((k, seq, SINGLE_DELETION, b""))
                    if k in tight:
                        intervals.append((put_seq[k], seq))
                elif k in put_here:
                    ents.append((k, seq, VALUE, _value(rnd, ts)))
                    put_seq[k] = seq
                else:
                    t = DELETION if rnd.random() < 0.08 else VALUE
                    ents.append((k, seq, t, _value(rnd, ts) if t == VALUE else b""))
                seq += 1
        runs.append(ents)
    return runs, hot, seq - 1, keys, tuple(intervals)


def _internal_sorted(ents):
    return sorted(ents, key=lambda e: (e[0], -e[1]))


def _files(runs, with_sd, level_files):
    """[(level, [(user key, seq, type, value)])] newest first; the level run cut into `level_files` files by key"""
    sd = {e[0] for ents in runs for e in ents if e[2] == SINGLE_DELETION}
    if not with_sd:  # without: the SingleDeletes and their Puts left out, the other entries numbered on in write order
        kept = sorted((e for ents in runs for e in ents if e[0] not in sd), key=lambda e: e[1])
        renum = {e[1]: i + 1 for i, e in enumerate(kept)}
        runs = [[(k, renum[s], t, v) for k, s, t, v in ents if k not in sd] for ents in runs]
    out = []
    for r, ents in enumerate(runs):
        ents = _internal_sorted(ents)
        if r == 0:  # the level: cut by key into files (it holds one version of a key, so no key spans two of them)
            per = (len(ents) + level_files - 1) // level_files
            out += [(1, ents[i:i + per]) for i in range(0, len(ents), per)]
        else:
            out.append((0, ents))
    return [f for f in out if f[0] == 0][::-1] + [f for f in out if f[0] == 1]


def _ops_run(ops, ents):
    """one run's ops in seq order, then the flush; the hot key's older versions are kept through the flush by snapshots"""
    by_seq = sorted(ents, key=lambda e: e[1])
    for i, (k, s, t, v) in enumerate(by_seq):
        if t == VALUE:
            ops.put(k, v)
        elif t == DELETION:
            ops.delete(k)
        else:
            ops.single_delete(k)
        if i + 1 < len(by_seq) and by_seq[i + 1][0] == k:
            ops.snapshot()
    ops.flush()


def _ops(files):
    """the ops script that makes the reference flush exactly these files, oldest first"""
    ops = H.Ops()
    for _, ents in sorted(files, key=lambda f: min(e[1] for e in f[1])):
        _ops_run(ops, ents)
    return ops


def _entries(ents):
    return [(H.ikey(k, s, t), v) for k, s, t, v in ents]


FORMATS = ((3, "crc32c"), (4, "xxh3"), (5, "none"), (5, "xxh3"), (4, "crc32c"), (3, "xxh3"))


@functools.lru_cache(maxsize=None)
def inputs_for(seed, nkeys, per_run, kind, with_sd, index_compression):
    """(inputs newest first, levels, hot key, last seq, keys)"""
    runs, hot, last, keys, _ = plan(seed, nkeys, per_run)
    files = _files(runs, with_sd, LEVEL_FILES)
    levels = [lv for lv, _ in files]
    if kind == "oracle":
        inputs = []
        for i, (_, ents) in enumerate(files):
            fv, ck = FORMATS[i % len(FORMATS)]
            inputs.append(H.oracle_build_sst(H.Params(format_version=fv, checksum=ck), H.kvstream(_entries(ents))))
    else:
        fv, ck = (5, "xxh3") if index_compression else (4, "crc32c")
        ref = H.run_reference(_ops(files), input_compression="zlib", index_compression=index_compression, format_version=fv,
                              checksum=ck, block_size=4096, target_file_size=1 << 30)
        by_first_seq = {min(int.from_bytes(ik[-8:], "little") >> 8 for ik, _ in sstfmt.parse_sst(d)["entries"]): d for d in ref["inputs"]}
        inputs = [by_first_seq[min(e[1] for e in ents)] for _, ents in files]  # every flush wrote one planned file
        for data, (_, ents) in zip(inputs, files):  # the reference wrote the planned entries, sequence numbers included
            assert sstfmt.parse_sst(data)["entries"] == _entries(ents)
        assert len(inputs) == len(files)
    return tuple(inputs), tuple(levels), hot, last, tuple(keys)


# ------------------------------------------------------------------------------------------------ the jobs
def _grandparents(keys):
    """files one level below the output: every 150 user keys a file over the first half of them, some sharing a boundary key, a few
    bounds shorter than the keys (a one-byte prefix)"""
    gps, i = [], 3
    while i + 150 < len(keys):
        a, b = keys[i], keys[i + 75]
        if i // 150 % 5 == 2 and len(b) > 1:
            b = b[:1] if b[:1] > a else b
        gps.append((a, b, 40 << 10))
        i += 150 if i // 150 % 4 else 75  # every fourth file starts at the previous one's largest key
    return [g for j, g in enumerate(gps) if j == 0 or g[0] >= gps[j - 1][1]]


def _range(kind, keys, hot):
    """bounds: `b` / `bx`, shorter than the keys around them, and the hot key, a user key with several versions"""
    short = b"b"
    if kind == "start":
        return hot, None
    if kind == "end":
        return None, short + b"x"
    if kind == "both":
        return short, hot
    return None, None


def job_size(big=False):
    """(number of user keys, entries per L0 run): enough for two merge tiles inside any range; a big job's output inside its range
    spans more than one stitch group"""
    if big:
        return 60000, 30000
    return 3000, 2000


# two jobs over more than one stitch group, shaped for the stitch walk: output level 1, a 2-byte partitioner and grandparents (dynamic
# file size on / off), so partition, grandparent and size cuts meet across group boundaries; the first starts at its range's first key.
# Snapshots and a non-bottommost level keep most versions, so the output holds about as many entries as the input range.
BIG = {
    "big_range_grandparents_p2": dict(inputs="oracle", runs="l0+level", single_delete=1, snapshots=17, bottommost=0, filter="ttl",
                                      grandparents="dynamic", prefix_len=2, range="both", bloom=10, format=(5, "xxh3"), paranoid=1,
                                      output_level=1, residency="host", output_mem="device"),
    "big_static_grandparents_p2": dict(inputs="oracle", runs="l0", single_delete=0, snapshots=3, bottommost=0,
                                       filter="remove_empty_value", grandparents="static", prefix_len=2, range="none", bloom=0,
                                       format=(4, "crc32c"), paranoid=0, output_level=1, residency="device", output_mem="host"),
}


def names():
    return [f"combo_{i:02d}" for i in range(len(rows()))] + sorted(BIG)


REFUSAL = "sd_range_zlib_write_conflict"
REFUSAL_TWIN = "sd_range_zlib"


def row_of(name):
    if name in (REFUSAL, REFUSAL_TWIN):
        return dict(inputs="zlib", runs="l0+level", single_delete=1, snapshots=3, bottommost=0, filter="none", grandparents="none",
                    prefix_len=0, range="both", bloom=10, format=(5, "xxh3"), paranoid=0, output_level=1, residency="host",
                    output_mem="host")
    if name in BIG:
        return BIG[name]
    return rows()[int(name.split("_")[1])]


def needs_reference(name):
    return row_of(name)["inputs"] == "zlib"


def build_row(row, index, big=False, **override):
    """dict(params, inputs, levels, residency, extras, row) of a factor row; `override` sets Params fields after the row"""
    nkeys, per_run = job_size(big)
    seed = 7 if big else 3
    ic = index % 2 if row["inputs"] == "zlib" else 0
    inputs, levels, hot, last, keys = inputs_for(seed, nkeys, per_run, row["inputs"], bool(row["single_delete"]), ic)
    intervals = plan(seed, nkeys, per_run)[4]
    taken = {s for a, b in intervals for s in range(a, b)}
    free = [s for s in range(1, last) if s not in taken]  # no snapshot separates a tight SingleDelete
    if row["runs"] == "l0":
        levels = tuple(0 for _ in levels)
    rnd = random.Random(SEED + index)
    fv, ck = row["format"]
    p = H.Params(output_level=row["output_level"], bottommost_level=bool(row["bottommost"]), max_output_file_size=32 << 10,
                 target_output_file_size=24 << 10, block_size=4096, format_version=fv, checksum=ck,
                 snapshots=sorted(rnd.sample(free, row["snapshots"])), file_creation_times=[T0 + 7, T0 + 8],
                 compaction_filter=row["filter"], ttl=TTL if row["filter"] == "ttl" else 0, now=T0 + 300 * 4 + TTL,
                 bloom_millibits_per_key=1000 * row["bloom"])
    if row["grandparents"] != "none":
        p.grandparents = _grandparents(list(keys))
        p.level_compaction_dynamic_file_size = row["grandparents"] == "dynamic"
        p.max_compaction_bytes = 100 << 10
    p.range_start, p.range_end = _range(row["range"], keys, hot)
    p.sst_partitioner_prefix_len = row["prefix_len"]
    for k, v in override.items():
        setattr(p, k, v)
    extras = dict(paranoid_file_checks=row["paranoid"], output_mem=row["output_mem"], sst_partitioner_prefix_len=row["prefix_len"])
    return dict(params=p, inputs=list(inputs), levels=list(levels), residency=row["residency"], extras=extras, row=row, hot=hot,
                index_compression=ic)


@functools.lru_cache(maxsize=None)
def build(name):
    """dict(params, inputs, levels, residency, extras, row)"""
    if name in (REFUSAL, REFUSAL_TWIN):
        c = build_row(row_of(name), 1)
        if name == REFUSAL:
            c["params"].earliest_write_conflict_snapshot = c["params"].snapshots[-1] + 1
            c["extras"]["earliest_write_conflict_snapshot"] = c["params"].earliest_write_conflict_snapshot
        return c
    if name in BIG:
        return build_row(BIG[name], 100 + sorted(BIG).index(name), big=True)
    i = int(name.split("_")[1])
    return build_row(rows()[i], i)


def check(p, inputs):
    """the checker: files, metas, stats"""
    return PC.oracle_compact(p, inputs)


@functools.lru_cache(maxsize=None)
def expected(name):
    """the case with the checker's job over it: files, metas, stats"""
    c = build(name)
    files, metas, stats = check(c["params"], c["inputs"])
    return dict(c, files=files, metas=metas, stats=stats)


def variant(name, **override):
    """the checker's job over the case with some Params fields changed (the census: the job without one factor)"""
    c = build(name)
    p = copy.copy(c["params"])
    for k, v in override.items():
        setattr(p, k, v)
    return check(p, c["inputs"])


# ------------------------------------------------------------------------------------------------ scripts for the live reference
# what the reference driver expresses: ops scripts with snapshots and SingleDeletes, input_compression / index_compression, bloom_bits,
# filter / ttl, paranoid, mode=range (grandparents from a set-up compaction), format_version / checksum (kCRC32c, kXXH3), the
# partitioner and max_subcompactions.  Not expressible: kNoChecksum outputs, output level 0 with grandparents, a key range without
# sub-compactions, grandparents over zlib inputs (DB::CompactRange writes the job's outputs with the inputs' compression, the device
# writes uncompressed ones), host / device residency and output_mem (product options).
REF_COMBOS = {
    "zlib_bloom_paranoid_p2": dict(plen=2, input_compression="zlib", index_compression=1, bloom_bits=10, paranoid=1, format_version=5,
                                   checksum="xxh3"),
    "zlib_filter_p16_fv4": dict(plen=16, input_compression="zlib", filter="remove_empty_value", format_version=4, checksum="crc32c"),
    "ttl_zlib_p2_fv3": dict(plen=2, input_compression="zlib", ttl=TTL, format_version=3, checksum="crc32c"),
    "grandparents_bloom_paranoid_p2": dict(plen=2, grandparents=1, bloom_bits=10, paranoid=1),
    "grandparents_static_p0_fv4": dict(plen=0, grandparents=1, dynamic_file_size=0, format_version=4, checksum="crc32c"),
    "subcompactions_bloom_paranoid_p2": dict(plen=2, bloom_bits=10, max_subcompactions=4, paranoid=1),
    "grandparents_subcompactions_bloom_paranoid_p2": dict(plen=2, grandparents=1, bloom_bits=10, max_subcompactions=4, paranoid=1),
    "subcompactions_filter_p16": dict(plen=16, filter="remove_empty_value", max_subcompactions=3, format_version=4, checksum="crc32c"),
}


def ref_combo(name):
    """(ops, opts) of a combination: the planned runs of combo_cases (SingleDeletes, the hot key kept by snapshots, deletions, empty
    values); with grandparents the level run is compacted to L2 first and the job is DB::CompactRange L0 -> L1; with ttl the runs are
    written at clock readings 300 s apart"""
    kw = dict(REF_COMBOS[name])
    plen = kw.pop("plen")
    gp = kw.pop("grandparents", 0)
    ttl = kw.get("ttl", 0)
    runs = plan(3, 3000, 2000)[0] if kw.get("max_subcompactions", 1) > 1 else plan(3, 1500, 1000)[0]
    files = _files(runs, True, 1)
    ops = H.Ops()
    for r, (_, ents) in enumerate(reversed(files)):
        if ttl:
            ops.set_time(T0 + 300 * r)
        _ops_run(ops, ents)
        if gp and r == 0:
            ops.compact_all_to(2)
    if ttl:
        ops.set_time(T0 + 300 * 4 + TTL)
    opts = dict(kw, target_file_size=24 << 10)
    if gp:
        opts.update(mode="range", setup_file_size=12 << 10)
    return ops, opts, plen
