"""Jobs for what the encoder writes behind the data blocks of every output file: the index block (index_entry and
shortest_separator in encode_index_size_kernel, then encode_index_write_kernel in csrc/encode.cu), the full Bloom filter block (bloom_count_kernel,
bloom_layout_kernel, bloom_slices_kernel) and the checksums of both (file_block_contrib_kernel, file_block_trailer_kernel over
xxh3_64_warp_t's precomputed-block path in csrc/common.cuh).

- `sep_*`: designed key pairs at block boundaries for every branch of FindShortestSeparator (util/comparator.cc:42-91): a difference
  in front of the next key's last byte, at its last byte with room to increment, at its last byte behind runs of 0-14 0xff bytes
  (incremented, or left unchanged when the tail is all 0xff), prefixes `k` / `k\\0` / `k\\0\\0`, the empty key, differences at bytes 0,
  7, 8 and 15 of 16-byte keys; and one user key whose versions are kept by snapshots, so that one file of the job keeps sequence
  numbers in its index and its neighbours do not.  format_version 3 / 4 / 5 x xxh3 / crc32c.
- `handles_v3`, `handles_v5`: block offsets and sizes whose varints are 1-5 and 1-4 bytes wide; three values of 2^27 - 1 bytes put
  later blocks at offsets past 2^28.  SLOW: these jobs hold about 400 MB of values each.
- `index_len_*`: one-file jobs whose index block (without trailer) is exactly 240 ... 9217 bytes: the lengths at which the split XXH3
  of file_block_contrib_kernel / file_block_trailer_kernel changes shape; `index_len_multi_*` holds several of them in one job.
- `filter_*`: filters of exactly one slice (kBloomSliceBytes of filter bits), one slice + 64 bytes, two slices and 8 slices; files
  of different slice counts in one job; filter blocks at all 16 phases of `data_size % 16`; filter lengths 64 m + 5; millibits at
  every threshold of bloom_num_probes and one past it; user keys of every length 0-16; hot keys whose kept versions repeat a hash;
  size cuts inside one key's versions.
- `files_max`, `files_max_filter`, `files_over`: exactly kMaxOutFiles output files, and one more (refused).

`build(name) -> (params, inputs)`: inputs are SST images, newest run first.  Sizes that must come out exact (index lengths, file
counts) are found at build time against the oracle's output layout.  tests/test_index_filter_cases_cpu.py proves from that layout
that each case reaches its edge."""
import functools
import os
import random
import re
import struct

import helpers as H
import plan_cases
import sstfmt


def _slice_bytes():
    """kBloomSliceBytes (csrc/encode.cu), written there as a product"""
    src = open(os.path.join(plan_cases._CSRC, "encode.cu")).read()
    m = re.search(r"constexpr\s+uint32_t\s+kBloomSliceBytes\s*=\s*(\d+)\s*\*\s*(\d+)\s*;", src)
    assert m, "kBloomSliceBytes not found in encode.cu"
    return int(m.group(1)) * int(m.group(2))


SLICE = _slice_bytes()
MAX_FILES = plan_cases._constant("kernels.h", "kMaxOutFiles")
BIG = 64 << 20
UNIFORM_BLOCKS = dict(block_restart_interval=1, block_size_deviation=0)
# block_size 64 (the smallest the library takes) and values of 48 bytes or more: every data block holds exactly one entry, so every
# pair of consecutive keys is a block boundary
ONE_ENTRY_BLOCKS = dict(block_size=64, **UNIFORM_BLOCKS)


def bloom_bits_bytes(n, millibits):
    """FastLocalBloomBitsBuilder::CalculateSpace without the metadata (filter_policy.cc:409-424)"""
    return ((n * millibits + 7999) // 8000 + 63) & ~63


def num_probes(millibits):
    """FastLocalBloomImpl::ChooseNumProbes (util/bloom_impl.h:156-198)"""
    for i, lim in enumerate((2080, 3580, 5100, 6640, 8300, 10070, 11720, 14001, 16050, 18300, 22001, 25501)):
        if millibits <= lim:
            return i + 1
    return 24 if millibits > 50000 else (millibits - 1) // 2000 - 1


PROBE_LIMITS = (2080, 3580, 5100, 6640, 8300, 10070, 11720, 14001, 16050, 18300, 22001, 25501, 50000)


def _deal(entries):
    """sorted (internal key, value) entries dealt into two input runs (newest first)"""
    runs = [[], []]
    for i, e in enumerate(entries):
        runs[i & 1].append(e)
    return tuple(H.oracle_build_sst(H.Params(), H.kvstream(r)) for r in reversed(runs) if r)


def _hkey(i):
    return struct.pack(">Q", (i * 0x9E3779B97F4A7C15 + 0x1234567) & ((1 << 64) - 1))


def _distinct(n, vlen, seed, seq0=1):
    """n distinct 8-byte hashed user keys in order, values of vlen bytes (or a random length when vlen is a range)"""
    rnd = random.Random(seed)
    keys = sorted(_hkey(i + seed * 10_000_019) for i in range(n))
    out = []
    for i, k in enumerate(keys):
        vl = rnd.randint(*vlen) if isinstance(vlen, tuple) else vlen
        out.append((H.ikey(k, seq0 + i), rnd.randbytes(vl)))
    return out


# ---------------------------------------------------------------------------------------------------------------- separators
def separator_user_keys():
    """(user keys in order, the hot key whose versions are kept).  Each shape sits in its own range of first-byte values, and the
    shapes come twice, so that a file cut (which ends a file at a pair instead of separating it) cannot take a shape out of the job."""
    g = [2]
    keys = [b"", b"\x00\x05"]  # the empty key is a file's first key; its separator to the next one is itself

    def take(k=1):
        b = g[0]
        g[0] += k
        return b
    hot = None
    for copy in range(2):
        G = take()
        keys += [bytes([G]) + b"aaaa", bytes([G]) + b"abzz"]                       # d < nul - 1
        G = take()
        keys += [bytes([G]) + b"abaxyz", bytes([G]) + b"abc"]                      # d == nul - 1, s[d] + 1 < l[d]
        for r in range(0, 15):                                                     # s[d] + 1 == l[d], 0xff run of r, then a byte to increment
            G = take(2)
            keys += [bytes([G]) + b"\xff" * r + b"q", bytes([G + 1])]
            if copy == 0 and r == 7:
                G = take()
                hot = bytes([G]) + b"hot"  # versions kept by snapshots; shortened separators on both sides
                keys += [bytes([G]) + b"hoszz", hot, bytes([G]) + b"houzz", bytes([G]) + b"hpa"]
        for r in range(1, 16):                                                     # the same with an all-0xff tail: unchanged
            G = take(2)
            keys += [bytes([G]) + b"\xff" * r, bytes([G + 1])]
        G = take()
        keys += [bytes([G]) + b"k", bytes([G]) + b"k\x00", bytes([G]) + b"k\x00\x00"]  # prefixes
        G = take(3)
        keys += [bytes([G]) + b"m" * 15, bytes([G + 2]) + b"m" * 15]               # 16-byte keys differing at byte 0
        G = take()
        keys += [bytes([G]) + b"m" * 6 + b"a" + b"z" * 8, bytes([G]) + b"m" * 6 + b"c" + b"z" * 8]  # at byte 7
        G = take()
        keys += [bytes([G]) + b"m" * 7 + b"a" + b"z" * 7, bytes([G]) + b"m" * 7 + b"c" + b"z" * 7]  # at byte 8
        G = take()
        keys += [bytes([G]) + b"m" * 14 + b"a", bytes([G]) + b"m" * 14 + b"c"]     # at byte 15, incremented
        G = take()
        keys += [bytes([G]) + b"m" * 14 + b"a", bytes([G]) + b"m" * 14 + b"b"]     # at byte 15, nothing behind it
        G = take()
        keys += [bytes([G]) + b"m" * 6 + b"a\xffq", bytes([G]) + b"m" * 6 + b"b"]  # walk from byte 7 across the word boundary
        G = take()
        keys += [bytes([G]) + b"m" * 6 + b"axyz", bytes([G]) + b"m" * 6 + b"c"]    # at byte 7, the next key's last
    assert keys == sorted(keys) and len(set(keys)) == len(keys) and max(map(len, keys)) <= 16 and g[0] <= 256
    return keys, hot


HOT_VERSIONS = 24


@functools.lru_cache(maxsize=None)
def _separator_data():
    """(entries, snapshots): every key once, the hot key HOT_VERSIONS times, each version in its own snapshot stripe"""
    keys, hot = separator_user_keys()
    rnd = random.Random(31)
    ents, seq, snaps = [], 1, []
    for k in keys:
        if k == hot:
            vs = []
            for _ in range(HOT_VERSIONS):
                vs.append(seq)
                seq += 1
            snaps += vs[:-1]
            ents += [(H.ikey(k, s), rnd.randbytes(48)) for s in reversed(vs)]
        else:
            ents.append((H.ikey(k, seq), rnd.randbytes(48)))
            seq += 1
    return ents, snaps


# ---------------------------------------------------------------------------------------------------------------- handles
# values whose blocks (one entry each) cross the varint widths of offsets and sizes: 2^7, 2^14, 2^21 and, behind the values of
# 2^27 - 1 bytes, offsets of 2^28 and more
HANDLE_VALUES = (48, 48, 150, 300, 20_000, 40_000, 3_000_000, (1 << 27) - 1, (1 << 27) - 1, (1 << 27) - 1, 48, 60)


@functools.lru_cache(maxsize=None)
def _handle_inputs():
    rnd = random.Random(41)
    ents = [(H.ikey(struct.pack(">Q", 0x1000 + 17 * i), i + 1), rnd.randbytes(v)) for i, v in enumerate(HANDLE_VALUES)]
    return _deal(ents)


# ---------------------------------------------------------------------------------------------------------------- index lengths
INDEX_LENGTHS = (240, 241, 1024, 1025, 1088, 8192, 8193, 9216, 9217)
PAD = 140_000     # value of a region's second-to-last entry: it takes the file past CUT, so the region's last entry ends the file
CUT = 131_072     # max_output_file_size of the index-length jobs


def _region(r, n, extra):
    """n one-entry blocks under first byte r; the last key is extra bytes longer (its index key grows by as many bytes)"""
    rnd = random.Random(r * 1000 + n)
    out = []
    for i in range(n):
        uk = bytes([r]) + struct.pack(">H", 3 * i + 1) + (b"\x01" * extra if i == n - 1 else b"")
        out.append((H.ikey(uk, 100_000 * r + i + 1), rnd.randbytes(PAD if i == n - 2 else 48)))
    return out


def _index_params(checksum):
    return H.Params(max_output_file_size=CUT, checksum=checksum, **ONE_ENTRY_BLOCKS)


def index_block_len(data):
    return sstfmt.parse_footer(data)["index"][1]


@functools.lru_cache(maxsize=None)
def _region_index_len(r, n, extra):
    files, _, _ = H.oracle_compact(_index_params("xxh3"), list(_deal(_region(r, n, extra))))
    assert len(files) == 1
    return index_block_len(files[0])


@functools.lru_cache(maxsize=None)
def region_for_length(r, length):
    """(n, extra) of the region under first byte r whose file has an index block of exactly `length` bytes"""
    lo, hi = 3, CUT // 100  # (a region of n one-entry blocks stays below CUT until its pad)
    assert _region_index_len(r, hi, 0) > length
    while hi - lo > 1:  # largest n whose index block is not longer than `length`
        mid = (lo + hi) // 2
        if _region_index_len(r, mid, 0) <= length:
            lo = mid
        else:
            hi = mid
    extra = length - _region_index_len(r, lo, 0)
    assert 0 <= extra <= 13, (length, lo, extra)
    assert _region_index_len(r, lo, extra) == length
    return lo, extra


MULTI_LENGTHS = (241, 1025, 8193, 9217)


# ---------------------------------------------------------------------------------------------------------------- filters
def _filter_keys_for_bits(bits, millibits):
    """smallest number of distinct keys whose filter has exactly `bits` bytes of bits"""
    n = bits * 8000 // millibits
    while bloom_bits_bytes(n, millibits) > bits:
        n -= 1
    while bloom_bits_bytes(n, millibits) < bits:
        n += 1
    assert bloom_bits_bytes(n, millibits) == bits
    return n


def _hot_entries(n_distinct, n_hot, versions, vlen, hot_vlen, seed):
    """n_distinct keys once and n_hot keys `versions` times; snapshots put every version of every hot key into its own stripe"""
    rnd = random.Random(seed)
    base = _distinct(n_distinct, vlen, seed)
    hot_keys = sorted({_hkey(10**9 + seed * 1000 + h) for h in range(n_hot)})
    seq0 = n_distinct + 1
    ents = list(base)
    for h, k in enumerate(hot_keys):
        ents += [(H.ikey(k, seq0 + v * n_hot + h), rnd.randbytes(hot_vlen)) for v in range(versions)]
    snaps = [seq0 + v * n_hot + n_hot - 1 for v in range(versions - 1)]
    ents.sort(key=lambda e: (e[0][:-8], -struct.unpack("<Q", e[0][-8:])[0]))
    return ents, snaps


@functools.lru_cache(maxsize=None)
def _filter_data(kind, args):
    if kind == "distinct":
        return _distinct(*args), ()
    if kind == "two_regions":  # large values (small filters per file) in front of empty values (large filters per file)
        a = _distinct(args[0], 200, 71)
        b = _distinct(args[1], 0, 72, seq0=args[0] + 1)
        b = [(H.ikey(b"\xff" + k[:7], i + args[0] + 1), v) for i, (k, v) in enumerate(b)]
        a = [(H.ikey(b"\x00" + k[:7], i + 1), v) for i, (k, v) in enumerate(a)]
        return a + b, ()
    if kind == "key_lengths":  # distinct user keys of every length 0..16
        rnd = random.Random(81)
        keys = set()
        for ln in range(17):
            of_len = set()
            while len(of_len) < min(256 ** ln, 3800):
                of_len.add(rnd.randbytes(ln))
            keys |= of_len
        return [(H.ikey(k, i + 1), rnd.randbytes(3)) for i, k in enumerate(sorted(keys))], ()
    if kind == "hot":
        ents, snaps = _hot_entries(*args)
        return ents, tuple(snaps)
    raise KeyError(kind)


@functools.lru_cache(maxsize=None)
def _filter_inputs(kind, args):
    return _deal(_filter_data(kind, args)[0])


def _fcase(kind, args, millibits, **params):
    return dict(kind="filter", data=(kind, args), params=dict(bloom_millibits_per_key=millibits, **params))


# ---------------------------------------------------------------------------------------------------------------- file count
def _uniform(n):
    rnd = random.Random(5)
    return [(H.ikey(struct.pack(">Q", 7 * i + 3), i + 1), rnd.randbytes(9)) for i in range(n)]


FILE_PARAMS = dict(block_size=100, max_output_file_size=1, **UNIFORM_BLOCKS)  # one 3-entry block + one single-entry block per file


@functools.lru_cache(maxsize=None)
def _file_count(n):
    return len(H.oracle_compact(H.Params(**FILE_PARAMS), list(_deal(_uniform(n))))[0])


@functools.lru_cache(maxsize=None)
def entries_for_files(nfiles):
    n = 4 * nfiles
    while _file_count(n) > nfiles:
        n -= 1
    while _file_count(n) < nfiles:
        n += 1
    return n


# ---------------------------------------------------------------------------------------------------------------- the cases
CASES = {}
for fv in (3, 4, 5):
    for ck in ("xxh3", "crc32c"):
        CASES[f"sep_v{fv}_{ck}"] = dict(kind="sep", params=dict(format_version=fv, checksum=ck, **ONE_ENTRY_BLOCKS))
for fv in (3, 5):
    CASES[f"handles_v{fv}"] = dict(kind="handles", params=dict(format_version=fv, max_output_file_size=1 << 30, **ONE_ENTRY_BLOCKS))
for ck in ("xxh3", "crc32c"):
    for ln in INDEX_LENGTHS:
        CASES[f"index_len_{ln}_{ck}"] = dict(kind="index_len", lengths=(ln,), checksum=ck)
    CASES[f"index_len_multi_{ck}"] = dict(kind="index_len", lengths=MULTI_LENGTHS, checksum=ck)
CASES.update({
    "filter_slice1": _fcase("distinct", (_filter_keys_for_bits(SLICE, 50000), 1, 1), 50000),
    "filter_slice1_64": _fcase("distinct", (_filter_keys_for_bits(SLICE + 64, 50000), 1, 2), 50000),
    "filter_slice2": _fcase("distinct", (_filter_keys_for_bits(2 * SLICE, 50000), 1, 3), 50000),
    "filter_slice8": _fcase("distinct", (1_100_000, 1, 4), 10000),   # 1.1 M keys at 10 bits: 7.6 slices
    "filter_slices_per_file": _fcase("two_regions", (30000, 400000), 50000, max_output_file_size=4 << 20),
    "filter_phases": _fcase("distinct", (48000, (0, 64), 5), 10000, max_output_file_size=24 << 10),
    "filter_key_lengths": _fcase("key_lengths", (), 50000),
    "filter_hot_keys": _fcase("hot", (40000, 50, 30, 1, 8, 6), 50000),
    "filter_cut_in_versions": _fcase("hot", (2000, 5, 30, 32, 600, 7), 10000, max_output_file_size=6 << 10),
})
for m in (3, 4, 15, 16, 127, 128, 129):
    CASES[f"filter_len_64x{m}"] = _fcase("distinct", (_filter_keys_for_bits(64 * m, 10000), 4, 100 + m), 10000)
for lim in PROBE_LIMITS:
    for mb in (lim, lim + 1):
        CASES[f"filter_probes_{mb}"] = _fcase("distinct", (3000, 4, 8), mb)
CASES.update({
    "files_max": dict(kind="files", nfiles=MAX_FILES, params=dict(FILE_PARAMS)),
    "files_max_filter": dict(kind="files", nfiles=MAX_FILES, params=dict(FILE_PARAMS, bloom_millibits_per_key=10000)),
    "files_over": dict(kind="files", nfiles=MAX_FILES + 1, params=dict(FILE_PARAMS)),
})
SLOW = ("handles_v3", "handles_v5")  # about 400 MB of values each


@functools.lru_cache(maxsize=None)
def build(name):
    c = CASES[name]
    kind = c["kind"]
    if kind == "sep":
        ents, snaps = _separator_data()
        p = H.Params(bottommost_level=False, snapshots=list(snaps), **c["params"])
        p.max_output_file_size = BIG
        files, _, _ = H.oracle_compact(p, list(_deal(ents)))
        # about five files: the hot key's versions (and with them the index keys with sequence numbers) in one or two of them
        p.max_output_file_size = index_offset(files[0]) // 5
        return p, list(_deal(ents))
    if kind == "handles":
        return H.Params(**c["params"]), list(_handle_inputs())
    if kind == "index_len":
        ents = []
        for r, ln in enumerate(c["lengths"], 1):
            ents += _region(r, *region_for_length(r, ln))
        return _index_params(c["checksum"]), list(_deal(ents))
    if kind == "filter":
        _, snaps = _filter_data(*c["data"])
        p = H.Params(bottommost_level=not snaps, snapshots=list(snaps), **c["params"])
        return p, list(_filter_inputs(*c["data"]))
    if kind == "files":
        return H.Params(**c["params"]), list(_deal(_uniform(entries_for_files(c["nfiles"]))))
    raise KeyError(kind)


# ---------------------------------------------------------------------------------------------------------------- output layout
def index_offset(data):
    """where the index block starts: behind the data blocks and the filter block"""
    return sstfmt.parse_footer(data)["index"][0]


def table_layout(data):
    """footer, metaindex, index [(key, (offset, size))] and properties of an output file, without decoding its data blocks"""
    ft = sstfmt.parse_footer(data)
    mblock, _, _ = sstfmt.read_block(data, ft["metaindex"])
    meta = {}
    for k, v, _ in sstfmt.block_entries(mblock):
        o, q = sstfmt.varint(v, 0)
        s, q = sstfmt.varint(v, q)
        meta[k.decode()] = (o, s)
    props = {}
    if "rocksdb.properties" in meta:
        pblock, _, _ = sstfmt.read_block(data, meta["rocksdb.properties"])
        props = {k.decode(): v for k, v, _ in sstfmt.block_entries(pblock)}
    iblock, _, _ = sstfmt.read_block(data, ft["index"])
    index = []
    if ft["format_version"] < 4:  # values are block handles behind a value-length varint
        for k, v, _ in sstfmt.block_entries(iblock):
            o, q = sstfmt.varint(v, 0)
            s, q = sstfmt.varint(v, q)
            index.append((k, (o, s)))
    else:  # no value length; index restart interval 1: every entry is a restart and holds its whole handle
        for k, q, shared in sstfmt.block_entries(iblock, value_delta=True):
            assert shared == 0
            o, q = sstfmt.varint(iblock, q)
            s, q = sstfmt.varint(iblock, q)
            index.append((k, (o, s)))
    return dict(footer=ft, metaindex=meta, properties=props, index=index)


FILTER_META = "fullfilter.rocksdb.BuiltinBloomFilter"


def filter_block(data, lay=None):
    """(offset, bits bytes, probes) of the file's filter block, or None"""
    lay = lay or table_layout(data)
    if FILTER_META not in lay["metaindex"]:
        return None
    off, size = lay["metaindex"][FILTER_META]
    md = data[off + size - 5:off + size]
    assert md[0] == 0xff and md[1] == 0, md.hex()
    return off, size - 5, md[2]


def shortest_separator(s, l):
    """BytewiseComparator::FindShortestSeparator (util/comparator.cc:42-91) -> (separator, branch)"""
    minl = min(len(s), len(l))
    d = 0
    while d < minl and s[d] == l[d]:
        d += 1
    if d >= minl:
        return s, "empty" if not s else "prefix"
    assert s[d] < l[d]
    if d < len(l) - 1:
        return s[:d] + bytes([s[d] + 1]), f"before_last@{d}"
    if s[d] + 1 < l[d]:
        return s[:d] + bytes([s[d] + 1]), f"last_byte@{d}"
    for i in range(d + 1, len(s)):
        if s[i] < 0xff:
            return s[:i] + bytes([s[i] + 1]), f"ff_run{i - d - 1}"
    return s, f"ff_tail{len(s) - d - 1}"
