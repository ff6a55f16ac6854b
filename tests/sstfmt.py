"""Minimal pure-Python BlockBasedTable reader used by the tests to inspect SST files
(footer / metaindex / properties / index / data blocks).  Test helper only.
Layout follows SURVEY.md Appendix A (reference: table/format.cc:191-259, table/block_based/block_builder.cc:21-32)."""
import struct

MAGIC = 0x88E241B785F4CFF7


def varint(b, p):
    x = 0
    s = 0
    while True:
        c = b[p]
        p += 1
        x |= (c & 0x7F) << s
        if c < 0x80:
            return x, p
        s += 7


def zigzag(x):
    return (x >> 1) ^ -(x & 1)


def parse_footer(data):
    f = data[-53:]
    magic = struct.unpack_from("<Q", f, 45)[0]
    assert magic == MAGIC, hex(magic)
    cksum_type = f[0]
    p = 1
    mo, p = varint(f, p)
    ms, p = varint(f, p)
    io, p = varint(f, p)
    isz, p = varint(f, p)
    fv = struct.unpack_from("<I", f, 41)[0]
    return dict(checksum_type=cksum_type, metaindex=(mo, ms), index=(io, isz), format_version=fv)


def block_entries(block, value_delta=False):
    """Yield (key, value_bytes, shared) for a block payload (without the 5-byte trailer)."""
    nr = struct.unpack_from("<I", block, len(block) - 4)[0] & 0x7FFFFFFF
    end = len(block) - 4 - 4 * nr
    p = 0
    key = b""
    out = []
    while p < end:
        shared, p = varint(block, p)
        non_shared, p = varint(block, p)
        if value_delta:
            key = key[:shared] + block[p:p + non_shared]
            p += non_shared
            out.append((key, p, shared))
            # caller decodes the value at offset p
            if shared == 0:
                _, p = varint(block, p)
                _, p = varint(block, p)
            else:
                _, p = varint(block, p)
        else:
            vlen, p = varint(block, p)
            key = key[:shared] + block[p:p + non_shared]
            p += non_shared
            out.append((key, bytes(block[p:p + vlen]), shared))
            p += vlen
    return out


def read_block(data, handle):
    """payload (inflated when the block is stored with kZlibCompression: varint32 size + raw deflate, util/compression.h:834-924),
    compression type byte, stored checksum"""
    off, sz = handle
    payload, ctype = data[off:off + sz], data[off + sz]
    if ctype == 2:
        import zlib
        usize, p = varint(payload, 0)
        # (one inflate call over the whole announced size, as the reference's Zlib_Uncompress makes: a stream written with
        #  window_bits -15 then reads back under -14 -- in smaller steps its matches past 16 KiB fall outside the window)
        payload = zlib.decompress(payload[p:], -14, max(usize, 1))
        assert len(payload) == usize
    else:
        assert ctype == 0, f"block compression type {ctype}"
    return payload, ctype, struct.unpack_from("<I", data, off + sz + 1)[0]


def parse_sst(data):
    """Return dict(footer, metaindex{name:(off,size)}, properties{name:bytes}, index[(sepkey,(off,size))], entries[(ikey,value)])."""
    ft = parse_footer(data)
    mblock, _, _ = read_block(data, ft["metaindex"])
    meta = {}
    for k, v, _ in block_entries(mblock):
        o, p = varint(v, 0)
        s, p = varint(v, p)
        meta[k.decode()] = (o, s)
    props = {}
    if "rocksdb.properties" in meta:
        pblock, _, _ = read_block(data, meta["rocksdb.properties"])
        for k, v, _ in block_entries(pblock):
            props[k.decode()] = v
    iblock, _, _ = read_block(data, ft["index"])
    index = []
    prev = None
    if ft["format_version"] < 4:  # index values are plain block handles (no delta encoding, IndexValue::EncodeTo format.cc:102-118)
        for k, v, _ in block_entries(iblock):
            o, q = varint(v, 0)
            s, q = varint(v, q)
            index.append((k, (o, s)))
    for k, p, shared in (block_entries(iblock, value_delta=True) if ft["format_version"] >= 4 else []):
        if shared == 0:
            o, p = varint(iblock, p)
            s, p = varint(iblock, p)
        else:
            d, p = varint(iblock, p)
            s = prev[1] + zigzag(d)
            o = prev[0] + prev[1] + 5
        prev = (o, s)
        index.append((k, (o, s)))
    entries = []
    for _, h in index:
        blk, ctype, _ = read_block(data, h)
        assert ctype in (0, 2)  # (read_block inflates kZlibCompression)
        for k, v, _ in block_entries(blk):
            entries.append((k, v))
    return dict(footer=ft, metaindex=meta, properties=props, index=index, entries=entries)


def prop_u64(props, name):
    return varint(props[name], 0)[0]
