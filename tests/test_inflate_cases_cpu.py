"""The inflate cases (inflate_cases.py) without a GPU: proof that every case reaches the edge it is named for, that the test's own
DEFLATE walker agrees with zlib on every block, and that the oracle reproduces the reference on every accepted job.

 (a) per case, a census of every compressed block from the walker: size-prefix width, deflate block types, stored lengths, code words
     longer than the device's first-level tables (kInfLBits / kInfDBits, read out of csrc/inflate_rules.h), distance symbols, length
     symbol 285, windowed or direct (kInflateWindow, read out of csrc/decode.cu).  Every count a case exists for must be >= 1; the
     counts are printed and are in every assertion message;
 (b) many_blocks: the pairs of blocks one inflate warp takes back to back, from the kernel's grid rule at 132 and 114 SMs;
 (c) the refusals patch what they claim to patch, and the checksums of the patched blocks are right.
Needs oracle/_ref (the compiled reference); skipped without it."""
import collections
import zlib

import pytest

import helpers as H
import inflate_cases as I
import sstfmt


def _need_ref():
    if not I.have_ref():
        pytest.skip("oracle/_ref/ref_compact_zlib not built (needs /root/reference)")


def _all_positive(counts, label):
    print(label, dict(counts))
    assert counts and min(counts.values()) >= 1, f"{label}: {dict(counts)}"


def _census(name):
    """aggregate census of a case's compressed data blocks"""
    c = collections.Counter()
    for _, b in I.blocks(I.case(name)["ref"]["inputs"]):
        if b["ctype"] != 2:
            c["stored raw"] += 1
            continue
        cen = b["census"]
        c["compressed"] += 1
        c[("prefix bytes", b["prefix"])] += 1
        c["windowed" if b["windowed"] else "direct"] += 1
        for t in cen["types"]:
            c[("deflate block", ("stored", "fixed", "dynamic")[t])] += 1
        for n in cen["stored"]:
            if n in (0, 65535):
                c[("stored length", n)] += 1
        c["literal/length codes > kInfLBits"] += cen["long_l"]
        c["distance codes > kInfDBits"] += cen["long_d"]
        c["length symbol 285"] += cen["sym285"]
        c["matches"] += sum(cen["dsyms"].values())
        for ds in (28, 29):
            c[("distance symbol", ds)] += cen["dsyms"][ds]
        c[("max distance", "> 16384" if cen["maxdist"] > 16384 else "> 512" if cen["maxdist"] > 512 else "<= 512")] += 1
        if b["u"] in (I.INFLATE_WINDOW - 1, I.INFLATE_WINDOW, I.INFLATE_WINDOW + 1):
            c[("inflated size", b["u"], "windowed" if b["windowed"] else "direct")] += 1
    return c


# what each case exists for: the census keys that must be >= 1 (and, after "==0", the ones that must be 0)
_EDGES = {
    "wbits15": [("distance symbol", 28), ("distance symbol", 29), ("prefix bytes", 3), "direct", ("max distance", "> 16384")],
    "wbits9": ["windowed", "matches"],
    "stored_level0": [("stored length", 65535), ("deflate block", "stored"), ("prefix bytes", 3)],
    "half_random": [("deflate block", "stored"), ("deflate block", "dynamic"), "direct"],
    "big_value": [("prefix bytes", 4), ("prefix bytes", 2), "direct", "windowed"],
    "window_edge_filtered": [("inflated size", I.INFLATE_WINDOW - 1, "windowed"), ("inflated size", I.INFLATE_WINDOW, "windowed"),
                             ("inflated size", I.INFLATE_WINDOW + 1, "direct")],
    "many_blocks": ["stored raw", "windowed", "direct", ("deflate block", "fixed"), ("deflate block", "dynamic")],
    "dict_none": ["compressed"],
}
for _lv in I.LEVELS:
    for _sn in I.STRATEGIES:
        # (the fixed code's words are at most 9 bits: all of them decode with one probe of the first-level table)
        _EDGES[f"level{_lv}_{_sn}"] = ["compressed"] + ([] if _sn == "huffman" else ["length symbol 285"]) + {
            "default": ["matches", ("deflate block", "dynamic"), "literal/length codes > kInfLBits"],
            "filtered": ["matches", ("deflate block", "dynamic"), "literal/length codes > kInfLBits"],
            "huffman": [("deflate block", "dynamic"), "literal/length codes > kInfLBits"],
            "rle": ["matches", ("deflate block", "dynamic"), "literal/length codes > kInfLBits"],
            "fixed": ["matches", ("deflate block", "fixed")]}[_sn]
_NONE = {f"level{lv}_huffman": ["matches", "length symbol 285"] for lv in I.LEVELS}
_NONE.update({f"level{lv}_fixed": [("deflate block", "dynamic")] for lv in I.LEVELS})
_NONE["wbits9"] = [("max distance", "> 512")]


@pytest.mark.parametrize("name", sorted(I.JOBS))
def test_case_reaches_its_edges(name):
    _need_ref()
    c = _census(name)
    print(name, dict(c))
    _all_positive({k: c[k] for k in _EDGES[name]}, name)
    assert all(c[k] == 0 for k in _NONE.get(name, [])), (name, dict(c))
    if name.endswith("_rle"):  # Z_RLE: every match repeats the byte before it
        assert all(ds == 0 for _, b in I.blocks(I.case(name)["ref"]["inputs"]) if b["census"] for ds in b["census"]["dsyms"]), name


def test_every_edge_is_reached_by_some_case():
    """the whole family together: distance symbols 28 / 29, stored lengths 65535, code words past both first-level tables, 3- and
    4-byte size prefixes, length symbol 285, both sides of the window"""
    _need_ref()
    total = collections.Counter()
    for name in sorted(I.JOBS):
        total.update(_census(name))
    want = [("distance symbol", 28), ("distance symbol", 29), ("stored length", 65535), "literal/length codes > kInfLBits",
            "distance codes > kInfDBits", ("prefix bytes", 2), ("prefix bytes", 3), ("prefix bytes", 4),
            "length symbol 285", "windowed", "direct", ("deflate block", "stored"), ("deflate block", "fixed"), ("deflate block", "dynamic")]
    _all_positive({k: total[k] for k in want}, "all inflate cases")


@pytest.mark.parametrize("name", sorted(I.JOBS))
def test_walker_agrees_with_zlib_on_every_block(name):
    _need_ref()
    n = 0
    for data in I.case(name)["ref"]["inputs"]:
        bl, ix = I.table_census(data)
        for b in bl:
            if b["ctype"] == 2:
                stream = data[b["off"] + b["prefix"]:b["off"] + b["size"]]
                assert b["payload"] == zlib.decompress(stream, -15), (name, b["index"])
                n += 1
        if ix["ctype"] == 2:
            io, isz = sstfmt.parse_footer(data)["index"]
            _, p = sstfmt.varint(data, io)
            assert ix["payload"] == zlib.decompress(data[p:io + isz], -15), (name, "index block")
    assert n > 0, name


def test_walker_refuses_malformed_streams():
    good = zlib.compress(b"compaction level block " * 40, 6, -15)
    assert I.walk(good)[0] == b"compaction level block " * 40
    for bad in (b"\x07", good[:len(good) // 2], bytes([0x01, 0x05, 0x00, 0xfb, 0xff]) + b"abc", b"\x06\x00"):
        with pytest.raises(I.DeflateError):
            I.walk(bad)


def test_many_blocks_gives_every_warp_a_second_pass():
    """the pairs (b, next) of compressed blocks one inflate warp takes back to back, at the grid of a 132-SM and a 114-SM part: windowed
    then direct, direct then windowed, dynamic then fixed, and a raw block in the warp's slots between two compressed ones; plus the
    passes of the verify warps"""
    _need_ref()
    bl = [b for _, b in I.blocks(I.case("many_blocks")["ref"]["inputs"])]
    nblk = len(bl)
    ncomp = sum(b["ctype"] == 2 for b in bl)
    counts = {"compressed blocks over 2 x 64 x 132": ncomp - 2 * 64 * 132}
    # the compressed index blocks are inflated on the host: each is larger than 32 KiB and was written with window_bits -15
    for d in I.case("many_blocks")["ref"]["inputs"]:
        ix = I.table_census(d)[1]
        counts["compressed index blocks > 32 KiB"] = counts.get("compressed index blocks > 32 KiB", 0) + (ix["ctype"] == 2 and ix["u"] > 32768)
    for sms in I.SM_COUNTS:
        T = I.inflate_stride(nblk, sms)
        V = I.verify_stride(nblk, sms)
        pairs = collections.Counter()
        for w in range(T):
            seq = list(range(w, nblk, T))
            comp = [i for i in seq if bl[i]["ctype"] == 2]
            if len(comp) >= 2:
                pairs["warps with two compressed blocks"] += 1
            for a, b in zip(comp, comp[1:]):
                ka, kb = ("windowed" if bl[a]["windowed"] else "direct"), ("windowed" if bl[b]["windowed"] else "direct")
                pairs[(ka, kb)] += 1
                if bl[a]["census"]["types"][-1] == 2 and bl[b]["census"]["types"][0] == 1:
                    pairs[("dynamic", "fixed")] += 1
                if b - a > T:
                    pairs["raw slot between two compressed blocks"] += 1
        assert pairs["warps with two compressed blocks"] == T, (sms, pairs["warps with two compressed blocks"], T)
        for k in [("windowed", "direct"), ("direct", "windowed"), ("windowed", "windowed"), ("dynamic", "fixed"),
                  "raw slot between two compressed blocks"]:
            counts[(sms, "SMs") + ((k,) if isinstance(k, str) else k)] = pairs[k]
        assert nblk >= 2 * V, (sms, nblk, V)  # every verify warp's loop runs at least twice
        vwarps = sum(1 for w in range(V) if sum(bl[i]["ctype"] == 2 for i in range(w, nblk, V)) >= 2)
        counts[(sms, "SMs", "verify warps with two compressed blocks")] = vwarps
    _all_positive(counts, "many_blocks")


@pytest.mark.parametrize("name", sorted(I.JOBS))
def test_oracle_reproduces_the_reference(name):
    _need_ref()
    c = I.case(name)
    files, metas, st = H.oracle_compact(c["params"], c["ref"]["inputs"])
    assert files == c["ref"]["outputs"], name
    for k in H.STAT_KEYS:
        assert getattr(st, k) == c["ref"]["manifest"]["stats"][k], (name, k)


def test_range_twin_skips_compressed_blocks():
    _need_ref()
    import decode_cases as D
    c = I.case("many_blocks_range")
    p = c["params"]
    skipped = 0
    for d in c["ref"]["inputs"]:
        kept = set(D.kept_blocks(d, p.range_start, p.range_end))
        skipped += sum(1 for b in I.table_census(d)[0] if b["ctype"] == 2 and b["index"] not in kept)
    _all_positive({"compressed blocks outside the range": skipped}, "many_blocks_range")


def test_dictionary_job_writes_a_dictionary_and_its_twin_does_not():
    _need_ref()
    def meta(d):  # (the data blocks of a dictionary table only inflate with the dictionary: read the metaindex alone)
        return [k.decode() for k, _, _ in sstfmt.block_entries(sstfmt.read_block(d, sstfmt.parse_footer(d)["metaindex"])[0])]
    with_dict = [meta(d) for d in I.case("dict_16k")["ref"]["inputs"]]
    without = [meta(d) for d in I.case("dict_none")["ref"]["inputs"]]
    assert all("rocksdb.compression_dict" in m for m in with_dict)
    assert not any("rocksdb.compression_dict" in m for m in without)


@pytest.mark.parametrize("name", sorted(I.REFUSALS))
def test_refusals_patch_one_block(name):
    _need_ref()
    base, what, value, _ = I.REFUSALS[name]
    ins, (f, b) = I.patched(base, what, value)
    orig = I.case(base)["ref"]["inputs"]
    assert [len(x) for x in ins] == [len(x) for x in orig]
    assert [i for i in range(len(ins)) if ins[i] != orig[i]] == [f]
    d, off, size = ins[f], b["off"], b["size"]
    diff = [j for j in range(len(d)) if d[j] != orig[f][j]]
    assert diff and off <= diff[0] and diff[-1] < off + size + 5, (name, diff[:4], off, size)
    ck = H.oracle().orc_block_checksum(H.CKSUM[I.case(base)["params"].checksum], d[off:off + size], size, d[off + size])
    stored = int.from_bytes(d[off + size + 1:off + size + 5], "little")
    assert (ck == stored) == (what != "checksum"), name
    if what == "ctype":
        assert d[off + size] == value
    if what == "u":
        u, _ = sstfmt.varint(d, off)
        assert u == (b["u"] + int(value) if isinstance(value, str) else value), name
    if base == "many_blocks":  # the patched block sits in the second pass of every verify warp
        nblk = len(I.blocks(orig))
        gi = sum(len(I.table_census(x)[0]) for x in orig[:f]) + b["index"]
        assert all(gi >= I.verify_stride(nblk, s) for s in I.SM_COUNTS), gi
