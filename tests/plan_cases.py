"""Jobs for the encoder's block-cut planner (encode_tables_kernel, encode_stitch_kernel, encode_tilestate_kernel and
encode_blocklist_kernel in csrc/encode.cu).

The planner tabulates, per tile of kEncTile entries, where a data block that starts at each entry ends; the stitch kernel walks
those tables group by group (kEncGroupTiles tiles), descends to tile and block level only where a file may end, and the block list
replays the walk per tile.  The jobs below put the output side on the planner's branches:
- restart intervals that the window's per-class scan does not take (3 and 64), with block_size_deviation 0 (no BlockAlmostFull
  rule) and 10;
- max_output_file_size values that end a file on the first / last entry of a tile, on the first entry of a group, and inside a
  group after a file that spans whole groups;
- files of one block plus the size rule's single-entry block, and a last file of one entry;
- a smallest entry that puts the block-chain candidate count hc at kEncHalo and one past it (refused with ERR_NOT_SUPPORTED);
- a value of 1 MiB, which selects the 64-bit window;
- grandparent boundaries inside groups that the walk would otherwise skip whole.

`build(name) -> (params, inputs)`: inputs are SST images, newest run first.  The file-end cases place the end exactly: the job is
first cut by the oracle as one file, and max_output_file_size is set to the offset of the data block that starts at the wanted
entry, so that entry is the first the size rule sees past the limit.  tests/test_plan_cases_cpu.py proves from the oracle's output
layout that each case reaches the branch it is named for."""
import functools
import os
import random
import re
import struct

import helpers as H
import sstfmt

_CSRC = os.path.join(H.ROOT, "toplingdb_b200", "csrc")


def _constant(path, name):
    m = re.search(r"constexpr\s+\w+\s+%s\s*=\s*(\d+)\s*;" % name, open(os.path.join(_CSRC, path)).read())
    assert m, f"{name} not found in {path}"
    return int(m.group(1))


TILE = _constant("kernels.h", "kEncTile")
HALO = _constant("kernels.h", "kEncHalo")
GROUP = TILE * _constant("kernels.h", "kEncGroupTiles")  # entries per stitch group
WINDOW = TILE + HALO
BIG = 64 << 20


def _varint_len(v):
    n = 1
    while v >= 128:
        v >>= 7
        n += 1
    return n


def entry_size(shared, ks, vs):
    """encoded size of an entry in a data block (block_builder.cc:97-126)"""
    return _varint_len(shared) + _varint_len(ks - shared) + _varint_len(vs) + ks - shared + vs


def _runs(n, vlen, seed, big_value=0):
    """n distinct 8-byte user keys (consecutive ones share 6 or 7 bytes) with vlen-byte values, dealt into two runs; with
    big_value, the middle entry holds a value of that many bytes"""
    rnd = random.Random(seed)
    runs = [[], []]
    for i in range(n):
        v = rnd.randbytes(big_value if big_value and i == n // 2 else vlen)
        runs[i & 1].append((H.ikey(struct.pack(">Q", 7 * i + 3), i + 1), v))
    return [runs[1], runs[0]]


def _mixed_runs(n, seed):
    """distinct user keys of 4 to 16 bytes over a two-letter alphabet and values of 0 to 96 bytes: restart entries and shared
    prefixes of every size"""
    rnd = random.Random(seed)
    keys = set()
    while len(keys) < n:
        keys.add(bytes(rnd.choice(b"ab") for _ in range(rnd.randint(4, 16))))
    runs = [[], []]
    for i, kb in enumerate(sorted(keys)):
        runs[i & 1].append((H.ikey(kb, i + 1), rnd.randbytes(rnd.choice((0, 5, 17, 96)))))
    return [runs[1], runs[0]]


@functools.lru_cache(maxsize=None)
def _inputs(data):
    kind, args = data
    runs = _runs(*args) if kind == "uniform" else _mixed_runs(*args)
    return tuple(H.oracle_build_sst(H.Params(), H.kvstream(r)) for r in runs)


# With restart interval 1 every entry is a restart entry of 1 + 1 + 1 + 16 + 9 bytes plus its 4-byte restart slot, so with
# block_size_deviation 0 every data block holds exactly k = ceil((block_size - 4) / 32) entries: 16 at 500 bytes, 3 at 100.
K16 = ("uniform", (170002, 9, 1))       # 2.6 groups; n - 2 is a multiple of 16
K3 = ("uniform", (20000, 9, 2))
K3_SMALL = ("uniform", (6000, 9, 5))   # one file per 4 entries stays below the encoder's kMaxOutFiles
MIXED = ("mixed", (30000, 3))
WIDE = ("uniform", (3000, 24, 4, 1 << 20))
UNIFORM_BLOCKS = dict(block_restart_interval=1, block_size_deviation=0)

CASES = {
    # restart intervals outside the per-class scan: Hillis-Steele scan, / R in div_r (3) and a power of two above 32 (64)
    "restart3_dev0": dict(data=MIXED, params=dict(block_restart_interval=3, block_size_deviation=0, max_output_file_size=200 << 10)),
    "restart64_dev0": dict(data=MIXED, params=dict(block_restart_interval=64, block_size_deviation=0, block_size=16384,
                                                   max_output_file_size=300 << 10)),
    "restart3_dev10": dict(data=MIXED, params=dict(block_restart_interval=3, block_size_deviation=10, max_output_file_size=200 << 10)),
    # the first file ends on entry `end` (its single-entry block)
    "end_tile_first": dict(data=K16, params=dict(block_size=500, **UNIFORM_BLOCKS), end=3 * TILE),
    "end_tile_last": dict(data=K3, params=dict(block_size=100, **UNIFORM_BLOCKS), end=4 * TILE - 1),
    "end_group_first": dict(data=K16, params=dict(block_size=500, **UNIFORM_BLOCKS), end=GROUP),
    # the first file spans groups 0 and 1 whole and ends inside group 2
    "end_inside_group": dict(data=K16, params=dict(block_size=500, **UNIFORM_BLOCKS), end=2 * GROUP + 6 * TILE + 16 * 40),
    "last_file_one_entry": dict(data=K16, params=dict(block_size=500, **UNIFORM_BLOCKS), end=K16[1][0] - 2),
    "one_block_files": dict(data=K3_SMALL, params=dict(block_size=100, max_output_file_size=1, **UNIFORM_BLOCKS)),
    # hc = (block_size - 1) / smallest entry + 3 at kEncHalo and one past it
    "hc_at_halo": dict(data=K3, params=dict(**UNIFORM_BLOCKS), hc=HALO),
    "hc_over_halo": dict(data=K3, params=dict(**UNIFORM_BLOCKS), hc=HALO + 1),
    "wide_window": dict(data=WIDE, params=dict(block_size=4096)),
    # one file; boundaries of three grandparents inside groups 0, 1 and 2.  max_compaction_bytes makes the second one cut a file
    "gp_in_skipped_groups": dict(data=K16, params=dict(block_size=500, max_compaction_bytes=3000 << 10, **UNIFORM_BLOCKS),
                                 gp=((20000, 20010), (90000, 90030), (140000, 140005))),
}


def user_key(data, e):
    """user key of merged entry e of a uniform data set"""
    assert data[0] == "uniform"
    return struct.pack(">Q", 7 * e + 3)


def layout(files):
    """oracle output files -> (entries [(internal key, value)], files [[(first entry, entries, offset, payload bytes)]])"""
    entries, out = [], []
    for data in files:
        blocks = []
        for _, h in sstfmt.parse_sst(data)["index"]:
            payload, _, _ = sstfmt.read_block(data, h)
            ents = sstfmt.block_entries(payload)
            blocks.append((len(entries), len(ents), h[0], h[1]))
            entries += [(k, v) for k, v, _ in ents]
        out.append(blocks)
    return entries, out


def min_s1(entries):
    """smallest entry size as the encoder computes it (shared prefix with the previous internal key of the whole stream)"""
    best, prev = None, b""
    for k, v in entries:
        sh = 0
        while sh < min(len(k), len(prev)) and k[sh] == prev[sh]:
            sh += 1
        s1 = entry_size(sh, len(k), len(v))
        best = s1 if best is None else min(best, s1)
        prev = k
    return best


@functools.lru_cache(maxsize=None)
def build(name):
    c = CASES[name]
    inputs = list(_inputs(c["data"]))
    p = H.Params(**c["params"])
    if "end" in c or "hc" in c:
        p.max_output_file_size = BIG
        entries, files = layout(H.oracle_compact(p, inputs)[0])
        if "end" in c:
            starts = {b[0]: b[2] for b in files[0]}
            assert c["end"] in starts, f"{name}: no data block starts at entry {c['end']}"
            p.max_output_file_size = starts[c["end"]]
        else:
            p.block_size = (c["hc"] - 3) * min_s1(entries) + 1
            p.max_output_file_size = 1 << 20
    if "gp" in c:
        p.grandparents = [(user_key(c["data"], a), user_key(c["data"], b), 1 << 20) for a, b in c["gp"]]
    return p, inputs
