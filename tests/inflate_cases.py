"""Compressed input tables for the device's inflate path (block_usize_kernel, verify_compressed_kernel and inflate_blocks_kernel in
csrc/decode.cu, the decoder of csrc/inflate_rules.h; the host inflater of compressed index blocks in csrc/api.cu), written by the
compiled reference under every shape of zlib CompressionOptions a user can set.

Every table comes from oracle/_ref/ref_compact_zlib (tests/native/ref_compact_zlib.cc: the reference driver with the zlib level,
strategy, window bits, ratio limit and dictionary size of the job's input files).  Where block contents matter, the blocks are planned
with decode_cases' `_Table`, so the reference cuts where the plan says.

`walk(stream)` is a small raw-DEFLATE decoder (RFC 1951) written for the tests alone: tests/test_inflate_cases_cpu.py checks it against
zlib on every block, and it reports per block what the device's decoder branches on (`table_census`).  `case(name)` -> dict(ref,
params, opts); `REFUSALS` are patched copies of accepted inputs with the error code the device must answer."""
import collections
import copy
import functools
import os
import random
import struct

import decode_cases as D
import helpers as H
import sstfmt

REF_ZLIB_BIN = os.path.join(H.ROOT, "oracle", "_ref", "ref_compact_zlib")
REF_ZLIB_B200_BIN = os.path.join(H.ROOT, "oracle", "_ref", "ref_compact_zlib_b200")  # + the B200 executor plugin

INFLATE_WINDOW = D.INFLATE_WINDOW
INF_LBITS = D._constant("inflate_rules.h", "kInfLBits")
INF_DBITS = D._constant("inflate_rules.h", "kInfDBits")
INFLATE_WARPS = D._constant("decode.cu", "kInflateWarps")
# the dispatch and the grid rules below are restated from these lines; if one changes, this module must change with it
D._require("decode.cu", "const bool windowed = u <= kInflateWindow;",
           "if (compressed_prefix(p, size, &u, &h) && u >= 4) s = (u + 5 + 15) & ~15u;",
           "if (c == 0 || u > 0x7fffffffull) return false;",
           "for (uint32_t b = blockIdx.x * kInflateWarps + w; b < nblk; b += gridDim.x * kInflateWarps) {",
           "for (uint32_t b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; b < nblk; b += (gridDim.x * blockDim.x) >> 5) {",
           "unsigned g = (nblk + 7) / 8; if (g > (unsigned)sms * 8) g = (unsigned)sms * 8;",
           "verify_compressed_kernel<<<g, 256, 0, st>>>",
           "unsigned grid = (nblk + kInflateWarps - 1) / kInflateWarps; if (grid > (unsigned)sms * 3u) grid = (unsigned)sms * 3u;")
D._require("inflate_rules.h", "const int de = ds < 4 ? 0 : (ds >> 1) - 1;", "if (l != 0 && l <= b.cnt) {")
SM_COUNTS = (132, 114)  # H100 SXM5 and H100 PCIe


def inflate_stride(nblk, sms):
    """warps of inflate_blocks_kernel: the distance between two blocks one warp inflates back to back"""
    return min((nblk + INFLATE_WARPS - 1) // INFLATE_WARPS, 3 * sms) * INFLATE_WARPS


def verify_stride(nblk, sms):
    """warps of verify_compressed_kernel (CTAs of 256 threads)"""
    return min((nblk + 7) // 8, 8 * sms) * 8


# ------------------------------------------------------------------------------------------------ DEFLATE walker
_LBASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
_LEXT = [0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0]
_DBASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193,
          12289, 16385, 24577]
_DEXT = [0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13]
_CL_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]


class DeflateError(ValueError):
    pass


def _table(lengths, complete=True):
    """canonical code of `lengths` as one lookup table over the next `bits` stream bits (LSB first): entry (symbol << 4) | length, 0
    where no code word starts.  An incomplete code is only legal with a single code word (zlib's inflate_table)"""
    bits = max(lengths, default=0)
    if bits == 0:
        return [0], 0
    count = collections.Counter(lengths)
    left = 1
    for ln in range(1, bits + 1):
        left = (left << 1) - count[ln]
        if left < 0:
            raise DeflateError("over-subscribed code")
    if complete and left and sum(count[ln] for ln in range(1, bits + 1)) != 1:
        raise DeflateError("incomplete code")
    nxt, code = {}, 0
    for ln in range(1, bits + 1):
        code = (code + count[ln - 1] if ln > 1 else 0) << 1
        nxt[ln] = code
    tab = [0] * (1 << bits)
    for s, ln in enumerate(lengths):
        if ln:
            c = nxt[ln]
            nxt[ln] += 1
            r = int(format(c, "0%db" % ln)[::-1], 2)
            tab[r::1 << ln] = [(s << 4) | ln] * (1 << (bits - ln))
    return tab, bits


_FIXED = None


def _fixed():
    global _FIXED
    if _FIXED is None:
        _FIXED = (_table([8] * 144 + [9] * 112 + [7] * 24 + [8] * 8), _table([5] * 30, complete=False))  # (30 of the 32 five-bit codes)
    return _FIXED


def walk(stream):
    """inflates a raw deflate stream: (bytes, census) -- census: block types, stored lengths, the longest literal/length and distance
    code words decoded, how many were longer than the device's first-level tables reach, distance symbols used, length symbol 285"""
    data = bytes(stream) + bytes(8)
    nbits = 8 * len(stream)
    out = bytearray()
    c = dict(types=[], stored=[], lmax=0, dmax=0, long_l=0, long_d=0, dsyms=collections.Counter(), sym285=0, maxdist=0)
    pos = 0  # bit position

    def bits(n):
        nonlocal pos
        v = (int.from_bytes(data[pos >> 3:(pos >> 3) + 4], "little") >> (pos & 7)) & ((1 << n) - 1)
        pos += n
        return v

    def sym(tab, tb):
        nonlocal pos
        e = tab[(int.from_bytes(data[pos >> 3:(pos >> 3) + 4], "little") >> (pos & 7)) & ((1 << tb) - 1)]
        if e == 0:
            raise DeflateError("no code word")
        pos += e & 15
        return e >> 4, e & 15

    while True:
        last, typ = bits(1), bits(2)
        c["types"].append(typ)
        if typ == 0:
            pos = (pos + 7) & ~7
            ln, nln = bits(16), bits(16)
            if ln != (~nln & 0xFFFF):
                raise DeflateError("stored LEN / NLEN")
            out += data[pos >> 3:(pos >> 3) + ln]
            pos += 8 * ln
            c["stored"].append(ln)
        elif typ in (1, 2):
            if typ == 1:
                (lt, lb), (dt, db) = _fixed()
            else:
                nlen, ndist, ncode = bits(5) + 257, bits(5) + 1, bits(4) + 4
                if nlen > 286 or ndist > 30:
                    raise DeflateError("too many codes")
                cl = [0] * 19
                for i in range(ncode):
                    cl[_CL_ORDER[i]] = bits(3)
                ct, cb = _table(cl)
                lens = []
                while len(lens) < nlen + ndist:
                    s, _ = sym(ct, cb)
                    if s < 16:
                        lens.append(s)
                    elif s == 16:
                        if not lens:
                            raise DeflateError("repeat without a length")
                        lens += [lens[-1]] * (3 + bits(2))
                    else:
                        lens += [0] * ((3 + bits(3)) if s == 17 else (11 + bits(7)))
                if len(lens) != nlen + ndist or lens[256] == 0:
                    raise DeflateError("code lengths")
                lt, lb = _table(lens[:nlen])
                dt, db = _table(lens[nlen:])
            while True:
                s, ln = sym(lt, lb)
                c["lmax"] = max(c["lmax"], ln)
                c["long_l"] += ln > INF_LBITS
                if s < 256:
                    out.append(s)
                    continue
                if s == 256:
                    break
                s -= 257
                if s >= 29:
                    raise DeflateError("length symbol")
                c["sym285"] += s == 28
                length = _LBASE[s] + bits(_LEXT[s])
                ds, dl = sym(dt, db)
                if ds >= 30:
                    raise DeflateError("distance symbol")
                c["dmax"] = max(c["dmax"], dl)
                c["long_d"] += dl > INF_DBITS
                c["dsyms"][ds] += 1
                dist = _DBASE[ds] + bits(_DEXT[ds])
                if dist > len(out):
                    raise DeflateError("distance too far back")
                c["maxdist"] = max(c["maxdist"], dist)
                if length <= dist:
                    out += out[-dist:len(out) - dist + length]
                else:
                    for _ in range(length):
                        out.append(out[-dist])
        else:
            raise DeflateError("block type 3")
        if pos > nbits:
            raise DeflateError("stream ends early")
        if last:
            return bytes(out), c


@functools.lru_cache(maxsize=None)
def table_census(data):
    """every data block of a table: dict(index, off, size, ctype, prefix, u, windowed, payload, census) -- census None for a block
    stored raw; plus the index block's: (ctype, u, inflated index block)"""
    t = sstfmt.parse_sst(data)
    out = []
    for i, (_, (off, size)) in enumerate(t["index"]):
        ctype = data[off + size]
        b = dict(index=i, off=off, size=size, ctype=ctype, prefix=0, u=size, windowed=None, census=None)
        if ctype == 2:
            u, p = sstfmt.varint(data, off)
            payload, cen = walk(data[p:off + size])
            if len(payload) != u:
                raise DeflateError(f"block {i} inflates to {len(payload)} bytes, announces {u}")
            b.update(prefix=p - off, u=u, windowed=u <= INFLATE_WINDOW, census=cen, payload=payload)
        out.append(b)
    io, isz = t["footer"]["index"]
    ix = dict(ctype=data[io + isz], u=isz, wbits=None)
    if ix["ctype"] == 2:
        u, p = sstfmt.varint(data, io)
        ix["u"] = u
        ix["payload"], ix["census"] = walk(data[p:io + isz])
    return out, ix


def blocks(ref_inputs):
    """(file, block) in the job's global block order (inputs in the order they are added, blocks in file order)"""
    return [(f, b) for f, d in enumerate(ref_inputs) for b in table_census(d)[0]]


# ------------------------------------------------------------------------------------------------ jobs
LEVELS = (1, 6, 9)
STRATEGIES = {"default": 0, "filtered": 1, "huffman": 2, "rle": 3, "fixed": 4}


def _mixed(rnd, n):
    """mostly word soup, with stretches of random bytes (rare literals get long code words) and runs of one byte (matches of 258)"""
    out = bytearray()
    while len(out) < n:
        r = rnd.random()
        out += rnd.randbytes(rnd.randint(4, 40)) if r < 0.25 else rnd.randbytes(1) * 300 if r < 0.28 else D._texty(rnd, rnd.randint(20, 200))
    return bytes(out[:n])


def _run(ks, t_entries, ops):
    for entries in t_entries:
        for k, v in entries:
            ops.put(k[:-8], v)
    ops.flush()


def _planned(ks, rnd, bs, nblk, fill, tag, sizes=()):
    """blocks of about bs bytes (or of the planned sizes first) filled by fill(rnd, n)"""
    t = D._Table(16, block_size=bs, deviation=10, fill=fill)
    keys = iter(sorted(ks.key(tag) for _ in range(200 * (nblk + len(sizes)))))

    def entry(n):
        return H.ikey(next(keys), 1, D.VALUE), fill(rnd, n)
    for size in sizes:
        es = []
        while D.block_estimate(es, 16) < 2000:
            es.append(entry(rnd.randint(20, 200)))
        t.add(es + [entry(0)], ("size", size))
    lim = (bs * 90 + 99) // 100
    for _ in range(nblk):
        es = []
        while True:
            e = entry(rnd.randint(20, min(400, bs // 2)))
            if D.block_estimate(es + [e], 16) > lim:
                break
            es.append(e)
        t.add(es + [entry(0)], ("min",))
    planned, _ = t.plan(rnd)
    return [e for e, _ in planned]


def _strategy_job(level, strategy):
    ks = D._Keys(100 + 10 * level + strategy)
    ops = H.Ops()
    for run in range(2):
        _run(ks, _planned(ks, ks.rnd, 4096, 24, _mixed if run else D._texty, 9 + run), ops)
    return ops, dict(zlib_level=level, zlib_strategy=strategy)


def _wbits_job(wbits):
    """64 KiB blocks (-15) or 4 KiB blocks (-9): a random 300-byte chunk that repeats 17-32 KiB later behind compressible filler, so
    the only match for it lies past 16 KiB (distance symbols 28 and 29)"""
    ks = D._Keys(200 - wbits)
    rnd = ks.rnd
    ops = H.Ops()
    if wbits == -15:
        for run in range(2):
            keys = sorted(ks.key(20 + run) for _ in range(40))
            for k in keys:
                v = bytearray()
                for gap in (rnd.randint(17 << 10, 24 << 10), rnd.randint(24 << 10, 31 << 10)):
                    chunk = rnd.randbytes(300)
                    v += chunk + D._texty(rnd, gap - 300) + chunk
                ops.put(k, bytes(v))
            ops.flush()
        return ops, dict(zlib_window_bits=-15, block_size=65536)
    for run in range(2):
        _run(ks, _planned(ks, rnd, 4096, 30, _mixed, 20 + run), ops)
    return ops, dict(zlib_window_bits=wbits)


def _stored_job():
    """level 0: deflate_stored writes stored blocks of at most 65535 bytes; a ratio limit of 2048 bytes per KiB keeps them"""
    ks = D._Keys(300)
    rnd = ks.rnd
    ops = H.Ops()
    for run in range(2):
        for k in sorted(ks.key(30 + run) for _ in range(12)):
            ops.put(k, rnd.randbytes(rnd.choice((65535 - 40, 70000, 140000, rnd.randint(100, 3000)))))
        ops.flush()
    return ops, dict(zlib_level=0, max_compressed_bytes_per_kb=2048, block_size=65536)


def _half_random_job():
    """64 KiB blocks, half random and half text: zlib ends a dynamic block and stores the random half"""
    ks = D._Keys(310)
    rnd = ks.rnd
    ops = H.Ops()
    for run in range(2):
        for k in sorted(ks.key(31 + run) for _ in range(16)):
            ops.put(k, rnd.randbytes(32 << 10) + D._texty(rnd, 32 << 10) if rnd.random() < 0.5 else D._texty(rnd, 32 << 10) + rnd.randbytes(32 << 10))
        ops.flush()
    return ops, dict(block_size=65536)


def _big_value_job():
    """one value of about 2.5 MiB of text (a 4-byte size prefix, the direct path) among small ones"""
    ks = D._Keys(320)
    rnd = ks.rnd
    ops = H.Ops()
    keys = sorted(ks.key(32) for _ in range(40))
    for i, k in enumerate(keys):
        ops.put(k, D._texty(rnd, (5 << 19) + 12345 if i == 20 else rnd.randint(10, 300)))
    ops.flush()
    for k in sorted(ks.key(32) for _ in range(40)):
        ops.put(k, D._texty(rnd, rnd.randint(10, 300)))
    ops.flush()
    return ops, dict()


def _window_edge_job():
    """planned inflated sizes on both sides of the window, written with the filtered strategy"""
    ks = D._Keys(330)
    ops = H.Ops()
    sizes = [s for s in (INFLATE_WINDOW - 1, INFLATE_WINDOW, INFLATE_WINDOW + 1) for _ in range(3)]
    for run in range(2):
        _run(ks, _planned(ks, ks.rnd, 4096, 6, D._texty, 33 + run, sizes), ops)
    return ops, dict(zlib_strategy=1, zlib_level=9)


MANY_BLOCKS_COMPRESSED = 2 * 64 * max(SM_COUNTS) + 1200


def _many_blocks_job():
    """1 KiB blocks, more than 2 x 64 x 132 of them compressed: every inflate warp and every verify warp of a 132-SM part takes
    several passes.  Among them: blocks of random bytes (stored raw: ctype 0), blocks of one repeated byte (a fixed-code stream), and
    blocks larger than the window (the direct path), spread over the whole job.  Written at -15, so every index block is a
    compressed block of more than 32 KiB for the host inflater."""
    ks = D._Keys(340)
    rnd = ks.rnd
    ops = H.Ops()
    total = int(MANY_BLOCKS_COMPRESSED * 1.12)
    nrun = 4
    for run in range(nrun):
        keys = iter(sorted(ks.key(40 + run) for _ in range(6 * total // nrun)))
        t = D._Table(16, block_size=1024, deviation=10, fill=D._texty)
        for _ in range(total // nrun):
            r = rnd.random()
            if r < 0.08:  # random bytes: stored raw
                t.add([(H.ikey(next(keys), 1, D.VALUE), rnd.randbytes(n)) for n in (rnd.randint(20, 300), 1024)], None)
            elif r < 0.12:  # one repeated byte
                t.add([(H.ikey(next(keys), 1, D.VALUE), bytes([rnd.randrange(256)]) * 1100)], None)
            elif r < 0.135:  # larger than the window
                t.add([(H.ikey(next(keys), 1, D.VALUE), D._texty(rnd, rnd.randint(INFLATE_WINDOW + 1, 3 * INFLATE_WINDOW)))], None)
            else:
                t.add([(H.ikey(next(keys), 1, D.VALUE), D._texty(rnd, rnd.randint(30, 200))) for _ in range(rnd.randint(1, 4))] +
                      [(H.ikey(next(keys), 1, D.VALUE), b"")], ("min",))
        planned, _ = t.plan(rnd)
        _run(ks, [e for e, _ in planned], ops)
    return ops, dict(zlib_window_bits=-15, block_size=1024, target_file_size=64 << 20)


def _dict_job(dict_bytes):
    ks = D._Keys(350)
    ops = H.Ops()
    for run in range(2):
        _run(ks, _planned(ks, ks.rnd, 4096, 12, D._texty, 50 + run), ops)
    return ops, dict(max_dict_bytes=dict_bytes)


JOBS = {
    **{f"level{lv}_{sn}": (lambda lv=lv, s=s: _strategy_job(lv, s)) for lv in LEVELS for sn, s in STRATEGIES.items()},
    "wbits9": lambda: _wbits_job(-9),
    "wbits15": lambda: _wbits_job(-15),
    "stored_level0": _stored_job,
    "half_random": _half_random_job,
    "big_value": _big_value_job,
    "window_edge_filtered": _window_edge_job,
    "many_blocks": _many_blocks_job,
    "dict_none": lambda: _dict_job(0),
}
REFUSED_JOBS = {"dict_16k": lambda: _dict_job(16384)}
CASES = sorted(JOBS) + ["many_blocks_range"]


def have_ref():
    return os.path.exists(REF_ZLIB_BIN)


def _opts(extra):
    opts = dict(target_file_size=1 << 20, input_compression="zlib", block_size=4096, index_compression=1)
    opts.update(extra)
    return opts


@functools.lru_cache(maxsize=None)
def case(name):
    """dict(ref, params, opts): the compiled reference's run (the inputs it wrote and its outputs) and the job parameters"""
    if name.endswith("_range"):
        c = case(name[:-len("_range")])
        p = copy.copy(c["params"])
        keys = sorted({k[:-8] for d in c["ref"]["inputs"] for k, _ in sstfmt.parse_sst(d)["entries"]})
        p.range_start, p.range_end = keys[len(keys) // 5], keys[4 * len(keys) // 5]
        return dict(c, params=p)
    ops, extra = {**JOBS, **REFUSED_JOBS}[name]()
    opts = _opts(extra)
    ref = H.run_reference(ops, binary=REF_ZLIB_BIN, **opts)
    return dict(ref=ref, params=H.params_from_reference(ref), opts=opts, ops=ops)


# ------------------------------------------------------------------------------------------------ refusals
def _set_u(block, prefix, u):
    """the stored block with its size prefix replaced by u, written in at least `prefix` bytes (zero-padded varint) -- the deflate
    stream is cut where a longer prefix needs room; the size checks refuse the block before it is inflated"""
    w = max(prefix, D.varint_len(u))
    enc = bytes(((u >> (7 * i)) & 0x7F) | (0x80 if i + 1 < w else 0) for i in range(w))
    return enc + block[prefix:len(block) - (w - prefix)]


def _rechecksum(data, off, size, ck):
    L = H.oracle()
    data[off + size + 1:off + size + 5] = struct.pack("<I", L.orc_block_checksum(H.CKSUM[ck], bytes(data[off:off + size]), size, data[off + size]))


def patched(base, what, value):
    """the inputs of case `base` with one compressed block patched, its checksum recomputed: what = "ctype" (the type byte),
    "u" (the announced size: an int, or "+1" / "-1" against the real stream), or "checksum" (the block's checksum flipped, nothing
    else).  The block is the last compressed block of the job (the second pass of every warp in many_blocks)."""
    c = case(base)
    ins = [bytearray(d) for d in c["ref"]["inputs"]]
    f, b = [(f, b) for f, b in blocks(c["ref"]["inputs"]) if b["ctype"] == 2][-1]
    d, off, size = ins[f], b["off"], b["size"]
    ck = c["params"].checksum
    if what == "ctype":
        d[off + size] = value
    elif what == "u":
        u = b["u"] + int(value) if isinstance(value, str) else value
        d[off:off + size] = _set_u(bytes(d[off:off + size]), b["prefix"], u)
    elif what == "checksum":
        d[off + size + 1] ^= 0x01
        return [bytes(x) for x in ins], (f, b)
    _rechecksum(d, off, size, ck)
    return [bytes(x) for x in ins], (f, b)


REFUSALS = {  # name -> (base case, what, value, error name)
    "ctype1": ("level6_default", "ctype", 1, "ERR_NOT_SUPPORTED"),
    "ctype4": ("level6_default", "ctype", 4, "ERR_NOT_SUPPORTED"),
    "ctype7": ("level6_default", "ctype", 7, "ERR_NOT_SUPPORTED"),
    "u3": ("level6_default", "u", 3, "ERR_CORRUPTION"),
    "u_plus1": ("level6_default", "u", "+1", "ERR_CORRUPTION"),
    "u_minus1": ("level6_default", "u", "-1", "ERR_CORRUPTION"),
    "u_over_2g": ("level6_default", "u", 0x80000000, "ERR_CORRUPTION"),
    "u_plus1_direct": ("wbits15", "u", "+1", "ERR_CORRUPTION"),
    "u_minus1_direct": ("wbits15", "u", "-1", "ERR_CORRUPTION"),
    "checksum_second_pass": ("many_blocks", "checksum", None, "ERR_CORRUPTION"),
}
