"""Input tables for the decode stage (index_decode_kernel, block_decode_fused_kernel, inflate_blocks_kernel in csrc/decode.cu), each
built to sit on one of the decoder's branches.

The decoder stages a data block in shared memory only when the block, its trailer and its 16-byte phase fit the staging slice; it
rebuilds keys one entry per lane only when the block has at most kDecRows restart intervals of at most kDecRowLen entries and every
entry header fits eight bytes; it scans 1, 2 or 3 key words depending on the largest `shared` of a pair of rows.  Everything else goes
to a lane-per-interval slow path.  Compressed blocks are inflated into a 16-byte aligned arena, through a shared-memory window when
they fit it.  Blocks outside a sub-job's key range are skipped (size 0), and the look-back over skipped blocks resolves at every
32nd block.  Index blocks with a restart interval other than 1 are walked by one thread.

Uncompressed tables come from the oracle's table builder (pinned byte for byte to the reference): `_Table` plans every block's
entries and exact size, the builder cuts where the plan says (block_size_deviation 0, or the reference's 10 % rule), and `_Table.build`
checks the result with sstfmt.  Compressed tables are written by the compiled reference itself (oracle/_ref/ref_compact) from the
same plans, because the arena path must see what the reference really writes.

`case(name)` -> dict(inputs, params); `table_blocks(data)` restates the dispatch for every block of a table;
tests/test_decode_cases_cpu.py proves from it that each case reaches the edges it exists for."""
import copy
import functools
import os
import random
import re
import struct

import helpers as H
import sstfmt

_CSRC = os.path.join(H.ROOT, "toplingdb_b200", "csrc")


def _src(path):
    with open(os.path.join(_CSRC, path)) as f:
        return f.read()


def _constant(path, name):
    m = re.search(r"constexpr[^;]*?\b%s\s*=\s*(\d+)\s*[;,]" % name, _src(path))
    assert m, f"{name} not found in {path}"
    return int(m.group(1))


def _require(path, *patterns):
    text = re.sub(r"\s+", " ", _src(path))
    for p in patterns:
        assert re.sub(r"\s+", " ", p) in text, f"{path} no longer contains `{p}`: restate the dispatch in tests/decode_cases.py"


DEC_SLICE = _constant("decode.cu", "kDecSlice")
DEC_ROWS = _constant("decode.cu", "kDecRows")
DEC_ROW_LEN = _constant("decode.cu", "kDecRowLen")
INFLATE_WINDOW = _constant("decode.cu", "kInflateWindow")
META_VLEN_BITS = _constant("common.cuh", "kMetaVlenBits")
MAX_VLEN = (1 << META_VLEN_BITS) - 1
LOOKBACK_STRIDE = 32
# the conditions below are restated from these lines; if one changes, this module must change with it
_require("decode.cu", "kDecVecs = kDecSlice / 16", "nvec = (shift + size + 5 + 15) >> 4", "nvec <= (uint32_t)kDecVecs - 3 && size >= 8",
         "nr > (uint32_t)kDecRows", "c > (uint32_t)kDecRowLen", "if (k >= 8 || sft > 28)", "ok && v[2] <= kMetaVlenMask",
         "else if (mx <= 8) scan_key_maps<1>", "else if (mx <= 16) scan_key_maps<2>", "else scan_key_maps<3>",
         "const bool windowed = u <= kInflateWindow;", "(b & 31u) == 31u", "if (nr != fd.nblocks)")
_require("range_rules.h", "if (has_start && range_key_cmp(sep, start) < 0) return false;",
         "if (has_end && has_prev && range_key_cmp(prev_sep, end) >= 0) return false;")
# largest shift + size that is staged: (shift + size + 5 + 15) >> 4 <= kDecVecs - 3
STAGE_LIMIT = 16 * (DEC_SLICE // 16 - 3) - 5
VALUE, DELETION, SINGLE_DELETION = 1, 0, 7


# ------------------------------------------------------------------------------------------------ restated dispatch
def varint_len(x):
    n = 1
    while x >= 128:
        x >>= 7
        n += 1
    return n


def parse_block(payload):
    """restart intervals of a data block: rows = [[(offset, shared, non_shared, vlen, header bytes)]] and the decoded entries"""
    nr = struct.unpack_from("<I", payload, len(payload) - 4)[0] & 0x7FFFFFFF
    data_end = len(payload) - 4 - 4 * nr
    rs = list(struct.unpack_from("<%dI" % nr, payload, data_end))
    rows = []
    for j, r0 in enumerate(rs):
        r1 = rs[j + 1] if j + 1 < nr else data_end
        row, q = [], r0
        while q < r1:
            sh, p = sstfmt.varint(payload, q)
            ns, p = sstfmt.varint(payload, p)
            vl, p = sstfmt.varint(payload, p)
            row.append((q, sh, ns, vl, p - q))
            q = p + ns + vl
        rows.append(row)
    return rows, [(k, v) for k, v, _ in sstfmt.block_entries(payload)]


def block_path(size, shift, rows):
    """(path, reason) the decoder takes for a block of `size` bytes whose first byte sits `shift` bytes past a 16-byte boundary"""
    if shift + size > STAGE_LIMIT or size < 8:
        return "slow", "not staged"
    if len(rows) == 0 or len(rows) > DEC_ROWS:
        return "slow", "restart intervals"
    if any(hdr > 8 or vl > MAX_VLEN for row in rows for _, _, _, vl, hdr in row):
        return "slow", "header"
    if any(len(row) > DEC_ROW_LEN for row in rows):
        return "slow", "interval length"
    return "fast", ""


def scan_width(mx):
    """key words the fast path scans for a pair of rows whose largest `shared` is mx"""
    return 0 if mx == 0 else 1 if mx <= 8 else 2 if mx <= 16 else 3


def index_info(data):
    t = sstfmt.parse_sst(data)
    payload, _, _ = sstfmt.read_block(data, t["footer"]["index"])
    nr = struct.unpack_from("<I", payload, len(payload) - 4)[0] & 0x7FFFFFFF
    user_key = sstfmt.prop_u64(t["properties"], "rocksdb.index.key.is.user.key") if "rocksdb.index.key.is.user.key" in t["properties"] else 0
    shared = [sh for _, _, sh in sstfmt.block_entries(payload, value_delta=t["footer"]["format_version"] >= 4)]
    return dict(nr=nr, nblocks=len(t["index"]), parallel=nr == len(t["index"]), user_key=bool(user_key), shared=shared,
                fv=t["footer"]["format_version"])


@functools.lru_cache(maxsize=256)
def table_blocks(data):
    """every data block of a table with what the decoder does with it: file offset, stored size, phase, compression, inflated size,
    restart intervals, entries and (path, reason) -- "arena-fast" / "arena-slow" for inflated blocks, which sit 16-byte aligned"""
    t = sstfmt.parse_sst(data)
    out = []
    for i, (sep, (off, size)) in enumerate(t["index"]):
        payload, ctype, _ = sstfmt.read_block(data, (off, size))
        rows, entries = parse_block(payload)
        shift = 0 if ctype == 2 else off % 16
        path, why = block_path(len(payload), shift, rows)
        out.append(dict(index=i, off=off, size=size, usize=len(payload), ctype=ctype, phase=off % 16, rows=rows, entries=entries, sep=sep,
                        path=("arena-" + path) if ctype == 2 else path, why=why))
    return out


def kept_blocks(data, start, end):
    """indices of the blocks a job with key range [start, end) decodes (index_decode_kernel: restart interval 1 and a separator of
    at most 16 user-key bytes, compared as block_may_touch_range does; everything else is kept)"""
    blocks = table_blocks(data)
    info = index_info(data)
    if (start is None and end is None) or not info["parallel"]:
        return list(range(len(blocks)))

    def sep(b):
        s = b["sep"] if info["user_key"] else b["sep"][:-8]
        return s if len(s) <= 16 else None
    kept = []
    for j, b in enumerate(blocks):
        s = sep(b)
        prev = sep(blocks[j - 1]) if j > 0 else None
        skip = s is not None and (j == 0 or prev is not None) and (
            (start is not None and s < start) or (end is not None and j > 0 and prev >= end))
        if not skip:
            kept.append(j)
    return kept


def located_entries(data, blocks=None):
    """entries of the given blocks (default: all) with where each one sits: (entries, [dict(block, offset, phase, path)])"""
    tb = table_blocks(data)
    entries, where = [], []
    for j in (range(len(tb)) if blocks is None else blocks):
        b = tb[j]
        offs = [e[0] for row in b["rows"] for e in row]
        for (k, v), o in zip(b["entries"], offs):
            entries.append((k, v))
            where.append(dict(block=j, offset=o, phase=b["phase"], path=b["path"] + (f" ({b['why']})" if b["why"] else "")))
    return entries, where


# ------------------------------------------------------------------------------------------------ planned tables
def block_estimate(entries, ri):
    """BlockBuilder::CurrentSizeEstimate after adding entries: the finished block's size"""
    n, prev = 0, b""
    for i, (k, v) in enumerate(entries):
        sh = 0
        if i % ri:
            while sh < min(len(k), len(prev)) and k[sh] == prev[sh]:
                sh += 1
        n += varint_len(sh) + varint_len(len(k) - sh) + varint_len(len(v)) + len(k) - sh + len(v)
        prev = k
    return n + 4 * ((len(entries) + ri - 1) // ri) + 4


class _Table:
    """One table as a list of planned blocks.  A block is [(internal key, value)]; the value of its last entry (the closer) is filled
    to `fill` bytes by `spec`: ("min",) the block just reaches block_size; ("size", n) the block is exactly n bytes; ("phase", q) the
    smallest size at least block_size that puts the NEXT block at file offset = q (mod 16); None leaves it as given.  The builder cuts
    a block when it reaches block_size, and -- with a deviation -- in front of an entry that would overshoot once the block is past
    the deviation limit (FlushBlockBySizePolicy); every block but its closer stays under both, so the cuts are the planned ones."""

    def __init__(self, ri, block_size=None, deviation=0, fill=None):
        self.ri, self.block_size, self.deviation = ri, block_size, deviation
        self.fill = fill or (lambda rnd, n: rnd.randbytes(n))
        self.blocks = []

    def add(self, entries, spec=("min",)):
        self.blocks.append((list(entries), spec))

    def _limits(self):
        bs = self.block_size or max(1, max(block_estimate(e[:-1], self.ri) for e, _ in self.blocks) + 1)
        lim = (bs * (100 - self.deviation) + 99) // 100 if self.deviation else bs
        return bs, min(lim, bs - 1) if self.deviation else bs - 1

    def plan(self, rnd):
        """resolved blocks ([(ikey, value)]) and their sizes; raises if a plan cannot be met"""
        bs, cap = self._limits()
        off, out = 0, []
        for entries, spec in self.blocks:
            # (the estimate only grows: the whole prefix under the cap means every state before the closer is)
            assert len(entries) == 1 or block_estimate(entries[:-1], self.ri) <= cap, "prefix would be cut"
            k, v = entries[-1]
            if spec is not None:
                base = block_estimate(entries[:-1] + [(k, b"")], self.ri) - 1
                if spec[0] == "min":  # (a value length at a varint boundary skips one size: take the next)
                    want = [max(bs, base + 1) + i for i in range(4)]
                elif spec[0] == "size":
                    want = [spec[1]]
                else:
                    first = max(bs, base + 1)
                    want = [first + ((spec[1] - (off + first + 5)) % 16) + 16 * t for t in range(4)]
                n = None
                for w in want:
                    for ln in range(1, 6):
                        if w - base - ln >= 0 and varint_len(w - base - ln) == ln:
                            n = w - base - ln
                            break
                    if n is not None:
                        break
                assert n is not None, ("no value length gives", spec)
                v = self.fill(rnd, n)
            entries = entries[:-1] + [(k, v)]
            size = block_estimate(entries, self.ri)
            assert size >= bs, (size, bs)
            if spec is not None and spec[0] == "size":
                assert size == spec[1], (size, spec)
            out.append((entries, size))
            off += size + 5
        return out, bs

    def build(self, rnd, **params):
        planned, bs = self.plan(rnd)
        p = H.Params(block_size=bs, block_size_deviation=self.deviation, block_restart_interval=self.ri, **params)
        data = H.oracle_build_sst(p, H.kvstream(kv for entries, _ in planned for kv in entries))
        got = table_blocks(data)
        assert [(b["usize"], len(b["entries"])) for b in got] == [(s, len(e)) for e, s in planned], "the builder cut elsewhere"
        return data


class _Keys:
    """unique sequence numbers and ascending 16-byte user keys for one job"""

    def __init__(self, seed):
        self.rnd = random.Random(seed)
        self.used = set()
        self.n = 0

    def seq(self, lo=1000, hi=1 << 40):
        while True:
            s = self.rnd.randrange(lo, hi)
            if s not in self.used:
                self.used.add(s)
                return s

    def key(self, prefix=0):
        self.n += self.rnd.randint(1, 9)
        return struct.pack(">QQ", prefix, (self.n << 24) | self.rnd.randrange(1 << 24))

    def entry(self, prefix=0, vlen=None, t=VALUE):
        v = b"" if t != VALUE else self.rnd.randbytes(self.rnd.randint(0, 40) if vlen is None else vlen)
        return H.ikey(self.key(prefix), self.seq(), t), v

    def mixed(self, prefix, n, vlens=(0, 8, 40)):
        """n entries, one in eight a tombstone and one in sixteen a SingleDelete"""
        out = []
        for _ in range(n):
            r = self.rnd.random()
            out.append(self.entry(prefix, self.rnd.choice(vlens), DELETION if r < 0.125 else SINGLE_DELETION if r < 0.19 else VALUE))
        return out


def _params(**kw):
    kw.setdefault("max_output_file_size", 256 << 10)
    kw.setdefault("file_creation_times", [7, 8, 9])
    return H.Params(**kw)


# ------------------------------------------------------------------------------------------------ staging_limit
STAGING_EXTRA = (DEC_SLICE, DEC_SLICE + 1, 5000, 9000, 40000, 70000)


def _staging_limit(ri, fv, checksum):
    ks = _Keys(11 + ri)
    t = _Table(ri)
    for q in range(16):
        for size in (STAGE_LIMIT - q, STAGE_LIMIT + 1 - q):
            t.add(ks.mixed(1, ks.rnd.randint(1, 3)) + [ks.entry(1, 0)], ("phase", q))
            t.add(ks.mixed(1, ks.rnd.randint(12, 24)) + [ks.entry(1, 0)], ("size", size))
    for size in STAGING_EXTRA:
        t.add(ks.mixed(1, 2) + [ks.entry(1, 0)], ("phase", ks.rnd.randrange(16)))
        t.add(ks.mixed(1, 20) + [ks.entry(1, 0)], ("size", size))
    t.add(ks.mixed(1, 5) + [ks.entry(1, 0)])
    # a second run over the same key range with ordinary blocks, so the merge interleaves
    u = _Table(ri, block_size=2048, deviation=0)
    for _ in range(60):
        u.add(ks.mixed(1, 10) + [ks.entry(1, 0)])
    inputs = [tb.build(ks.rnd, format_version=fv, checksum=checksum) for tb in (t, u)]
    return inputs, _params(format_version=fv, checksum=checksum)


# ------------------------------------------------------------------------------------------------ rows
ROW_COUNTS = (1, 16, 17, 32, 33, 64, 65)


def _rows(ri):
    """one table per restart-interval count: blocks of nr intervals whose last interval is full or one entry short; short user keys
    and empty values keep nr = 16 (and 17) intervals of 16 (17) entries inside the staging slice"""
    ks = _Keys(30 + ri)
    inputs = []
    for nr in ROW_COUNTS:
        t = _Table(ri)
        for rep in range(2):
            for short in ((False, True) if ri > 1 else (False,)):
                n = nr * ri - (1 if short else 0)
                es = []
                for _ in range(n):
                    ks.n += ks.rnd.randint(1, 3)
                    r = ks.rnd.random()
                    tp = DELETION if r < 0.1 else SINGLE_DELETION if r < 0.15 else VALUE
                    es.append((H.ikey(struct.pack(">I", (nr << 24) | ks.n), ks.seq(), tp),
                               b"" if tp != VALUE or ks.rnd.random() < 0.7 else ks.rnd.randbytes(2)))
                es[-1] = (H.ikey(es[-1][0][:-8], ks.seq(), VALUE), b"")
                t.add(es)
        inputs.append(t.build(ks.rnd))
    return inputs, _params(block_restart_interval=ri)


# ------------------------------------------------------------------------------------------------ key_words
KEY_WORD_TARGETS = (0, 8, 9, 16, 17, 23)


def _trailer(seq, t):
    return bytearray(struct.pack("<Q", (seq << 8) | t))


def _pair(ks, lead, ua_len, x, mode=None):
    """two internal keys (a, b), a before b, whose longest common prefix is exactly x bytes; a's user key is ua_len bytes starting
    with `lead`.  x past a's user key is reached by versions of one user key (trailers that agree on x - ua_len bytes) or by a user
    key that extends a's with a's own trailer bytes."""
    rnd = ks.rnd
    ua = (bytes([lead]) + rnd.randbytes(ua_len - 1)) if ua_len else b""
    if x < ua_len:
        ua = ua[:x] + bytes([rnd.randrange(0, 255)]) + ua[x + 1:] if x else ua
        ub = ua[:x] + bytes([(ua[x] + 1) if x else lead + 1]) + rnd.randbytes(rnd.randint(0, 16 - x - 1))
        return H.ikey(ua, ks.seq(), rnd.choice((VALUE, VALUE, DELETION, SINGLE_DELETION))), H.ikey(ub, ks.seq(), VALUE)
    j = x - ua_len  # common trailer bytes
    modes = []
    if j <= 7:
        modes.append("versions")
    if ua_len < 16 and 1 <= j <= 8:
        modes.append("extend")
    assert modes and (mode is None or mode in modes), (ua_len, x, mode)
    mode = mode or rnd.choice(modes)
    while True:
        if mode == "versions":
            if j == 0:
                ta, tb = rnd.choice(((VALUE, DELETION), (SINGLE_DELETION, VALUE), (VALUE, SINGLE_DELETION)))
                sa, sb = ks.seq(), ks.seq()
                sa, sb = max(sa, sb), min(sa, sb)
            else:
                ta = tb = rnd.choice((VALUE, VALUE, DELETION))
                sb = rnd.randrange(1000, 1 << 48)
                byte = j - 1  # first seq byte that differs
                cur = (sb >> (8 * byte)) & 0xFF
                if cur == 255:
                    continue
                sa = sb + (rnd.randint(1, 255 - cur) << (8 * byte))
                if sa in ks.used or sb in ks.used:
                    continue
                ks.used.update((sa, sb))
            return H.ikey(ua, sa, ta), H.ikey(ua, sb, tb)
        # extend: ub = ua + Ta[:k]; then b's trailer agrees with Ta[k:] on m bytes
        k = rnd.randint(1, min(j, 16 - ua_len))
        m = j - k  # (<= 8 - k because j <= 8)
        tb_type = rnd.choice((VALUE, DELETION)) if m >= 1 else VALUE
        tbb = _trailer(ks.seq(), tb_type)
        ta = _trailer(ks.seq(), rnd.choice((VALUE, DELETION)))
        for i in range(m):
            ta[k + i] = tbb[i]
        if k + m < 8 and ta[k + m] == tbb[m]:
            ta[k + m] ^= 1
        sa = struct.unpack("<Q", bytes(ta))[0] >> 8
        if sa in ks.used or sa < 1000:
            continue
        ks.used.add(sa)
        return ua + bytes(ta), ua + bytes(ta[:k]) + bytes(tbb)


def _before(a, b):
    """internal key order: user key ascending, then sequence number and type descending"""
    return a[:-8] < b[:-8] or (a[:-8] == b[:-8] and a[-8:][::-1] > b[-8:][::-1])


def _common(a, b):
    n = 0
    while n < min(len(a), len(b)) and a[n] == b[n]:
        n += 1
    return n


def _key_words(seed, slow):
    """restart interval 2: every row is a planted pair, a block is 15 pairs and a closer (16 rows, the fast path) -- or the same
    behind a 5000-byte closer (the slow path).  Rows of a pair share at most X, X running over KEY_WORD_TARGETS and the values between.
    A second table holds versions of 16-byte user keys at restart interval 16: sequence numbers that differ only in a high byte
    (shared = 23) or in the lowest byte (shared = 17)."""
    ks = _Keys(seed)
    rnd = ks.rnd
    inputs = []
    for tbl in range(3):
        t = _Table(2)
        lead, es, pairs, mx = 16, [], 0, 0
        while lead + 2 <= 255:
            if pairs == 0:  # the empty user key: its versions (at the restart point and behind it), or a key made of its trailer bytes
                ua_len, x, mode = 0, (7, 8, 0)[tbl], ("versions", "extend", "versions")[tbl]
            else:
                # the first row of a pair sets the pair's largest `shared`; the second stays at or below it
                x = rnd.choice(KEY_WORD_TARGETS) if pairs % 2 == 0 else rnd.randint(0, mx)
                ua_len, mode = rnd.randint(max(1, x - 8), 16), None
            mx = x
            a, b = _pair(ks, lead, ua_len, x, mode)
            assert _common(a, b) == x and _before(a, b) and (not es or _before(es[-1][0], a)), (a, b, x)
            es += [(a, rnd.randbytes(rnd.choice((0, 3, 9)))), (b, rnd.randbytes(rnd.choice((0, 3, 9))))]
            if a[-8] != VALUE:
                es[-2] = (a, b"")
            if b[-8] != VALUE:
                es[-1] = (b, b"")
            pairs += 1
            lead += 3
            if pairs % 15 == 0 or lead + 2 > 255:
                es.append((H.ikey(bytes([lead - 1]) + rnd.randbytes(4), ks.seq(), VALUE), b""))
                t.add(es, ("size", 5000) if slow else ("min",))
                es = []
        inputs.append(t.build(rnd))
    # versions of hot 16-byte keys, restart interval 16
    t = _Table(16)
    for blk in range(12):
        uk = struct.pack(">QQ", 0xFF00 + blk, rnd.getrandbits(64))
        base = rnd.randrange(1 << 20, 1 << 40)
        if blk % 2 == 0:  # sequence numbers 2^48 apart: only the top trailer byte differs
            seqs = [base + (i << 48) for i in range(1, 40)]
        else:  # consecutive: the lowest sequence byte differs (the type byte does not)
            base &= ~0xFF
            seqs = [base + i for i in range(1, 40)]
        seqs = sorted(seqs, reverse=True)
        ks.used.update(seqs)
        es = [(H.ikey(uk, s, VALUE), rnd.randbytes(rnd.choice((0, 4)))) for s in seqs]
        t.add(es, ("size", 5000) if slow and blk % 4 < 2 else ("min",))
    inputs.append(t.build(rnd))
    return inputs, _params()


# ------------------------------------------------------------------------------------------------ headers
FAST_VLENS = (0, 127, 128)
SLOW_VLENS = (16383, 16384, (1 << 21) - 1, 1 << 21)


def _headers():
    ks = _Keys(51)
    rnd = ks.rnd
    fast = _Table(16)
    for _ in range(40):
        es = []
        for _ in range(rnd.randint(6, 20)):
            r = rnd.random()
            es.append(ks.entry(2, rnd.choice(FAST_VLENS), DELETION if r < 0.15 else SINGLE_DELETION if r < 0.25 else VALUE))
        fast.add(es + [ks.entry(2, 0)])
    slow = _Table(16)
    for i in range(24):
        es = []
        for _ in range(rnd.randint(2, 12)):
            r = rnd.random()
            es.append(ks.entry(2, rnd.choice(FAST_VLENS), DELETION if r < 0.15 else SINGLE_DELETION if r < 0.25 else VALUE))
        big = SLOW_VLENS[i % len(SLOW_VLENS)] if i < 16 else 5000 + i
        slow.add(es + [ks.entry(2, big)], None)
    inputs = [fast.build(rnd), slow.build(rnd)]
    return inputs, _params(max_output_file_size=4 << 20)


def _one_big_value(vlen):
    ks = _Keys(52)
    es = [ks.entry(3, 10) for _ in range(5)] + [ks.entry(3, 0, DELETION)]
    es.append((H.ikey(ks.key(3), ks.seq(), VALUE), random.Random(53).randbytes(vlen)))
    es += [ks.entry(3, 10) for _ in range(5)]
    data = H.oracle_build_sst(H.Params(), H.kvstream(es))
    return [data], _params()


# ------------------------------------------------------------------------------------------------ skipped
# (stretch of skipped blocks in front of a file's first kept block, that block's global index mod 32)
SKIP_TARGETS = [(32, 0), (31, 31), (33, 1), (100, 0), (31, 0), (32, 1), (33, 31), (100, 31), (31, 1), (32, 31), (33, 0), (100, 1)]
RANGE_S = struct.pack(">QQ", 5 << 40, 0)
RANGE_E = struct.pack(">QQ", 6 << 40, 0)


def _skipped(nothing=False):
    """files of three-entry blocks: `lead` blocks below the range, `mid` in it, `trail` at or above its end.  Every file holds the
    range's start key as its first kept key and its end key as the first trailing key, so the skipped blocks are exactly the leading
    ones and all trailing ones but the first (its predecessor's separator lies below the end).  Mid counts put every file's first kept
    block at the planned global index mod 32; a file below the range sits between two of them, and the job ends on skipped blocks."""
    ks = _Keys(61)
    rnd = ks.rnd
    S, E = struct.unpack(">Q", RANGE_S[:8])[0], struct.unpack(">Q", RANGE_E[:8])[0]
    files = []  # (lead, mid, trail)
    g, pending = 0, 0
    for f, (L, r) in enumerate(SKIP_TARGETS):
        a = L - pending
        assert a >= 1 and (g + a) % 32 == r, (f, g, a, r)
        g += a
        nxt = SKIP_TARGETS[f + 1] if f + 1 < len(SKIP_TARGETS) else None
        trail = 0 if f % 3 == 0 else 4 if f % 3 == 1 else 1
        if f + 1 == len(SKIP_TARGETS):
            trail = 6
        empty = 40 if f == 6 else 0  # a whole file below the range after this one
        pend = max(0, trail - 1) + empty
        if nxt:
            mid = 3
            while (g + mid + trail + empty + nxt[0] - pend) % 32 != nxt[1]:
                mid += 1
        else:
            mid = 5
        files.append((a, mid, trail))
        if empty:
            files.append((empty, 0, 0))
        g += mid + trail + empty
        pending = pend
    inputs = []
    for f, (a, mid, trail) in enumerate(files):
        t = _Table(16, block_size=None)

        def blk(keys):
            es = [(H.ikey(k, ks.seq(), VALUE), rnd.randbytes(rnd.randint(0, 30))) for k in keys]
            t.add(es, ("min",))
        for i in range(a):
            base = (S - 1) if mid else (S - 1 - (1 << 20))
            blk([struct.pack(">QQ", base, (f << 40) | ((i * 3 + c) << 8)) for c in range(3)])
        for i in range(mid):
            ks_ = [struct.pack(">QQ", S, (f << 40) | ((i * 3 + c + 1) << 8)) for c in range(3)]
            if i == 0:
                ks_[0] = RANGE_S
            blk(ks_)
        for i in range(trail):
            ks_ = [struct.pack(">QQ", E, (f << 40) | ((i * 3 + c + 1) << 8)) for c in range(3)]
            if i == 0:
                ks_[0] = RANGE_E
            blk(ks_)
        inputs.append(t.build(rnd))
    p = _params()
    if nothing:
        p.range_start, p.range_end = struct.pack(">QQ", 7 << 40, 0), None
    else:
        p.range_start, p.range_end = RANGE_S, RANGE_E
    return inputs, p


# ------------------------------------------------------------------------------------------------ index_walk
INDEX_INTERVALS = (2, 3, 16)


def _index_walk(fv, ranged):
    """per index restart interval one file of many small blocks (walked by one thread); at interval 3 a hot user key spans block
    boundaries, so the separators keep their sequence numbers; a one-block file at interval 16 (one restart point per block: the
    parallel path) and a file at interval 1"""
    ks = _Keys(70 + fv)
    rnd = ks.rnd
    inputs = []
    for ir in (1,) + INDEX_INTERVALS:
        es = []
        ks.n = 0  # the files overlap in key order
        for i in range(600):
            es.append(ks.entry(4, rnd.choice((0, 8, 30))))
            if ir == 3 and i % 150 == 75:  # a hot user key: 40 versions over several 256-byte blocks
                uk = ks.key(4)
                es += [(H.ikey(uk, s, VALUE), rnd.randbytes(8)) for s in sorted((ks.seq() for _ in range(40)), reverse=True)]
        inputs.append(H.oracle_build_sst(H.Params(block_size=256, index_block_restart_interval=ir, format_version=fv), H.kvstream(es)))
    ks.n = 1500
    es = [ks.entry(4, 8) for _ in range(20)]
    inputs.append(H.oracle_build_sst(H.Params(block_size=4096, index_block_restart_interval=16, format_version=fv), H.kvstream(es)))
    p = _params(format_version=fv)
    if ranged:
        keys = sorted({k[:-8] for d in inputs[:1] for k, _ in sstfmt.parse_sst(d)["entries"]})
        p.range_start, p.range_end = keys[len(keys) // 4], keys[3 * len(keys) // 4]
    return inputs, p


# ------------------------------------------------------------------------------------------------ inflate (reference-written)
_WORDS = [b"compaction", b"level", b"block", b"table", b"restart", b"varint", b"checksum", b"footer", b"index", b"merge", b"snapshot"]


def _texty(rnd, n):
    out = bytearray()
    while len(out) < n:
        out += rnd.choice(_WORDS) + b" "
    return bytes(out[:n])


# (block_size, restart_interval, format_version, checksum, index_compression)
INFLATE_CONFIGS = {
    "inflate_4k_ri16_fv5": (4096, 16, 5, "xxh3", 1),
    "inflate_4k_ri1_fv4": (4096, 1, 4, "crc32c", 0),
    "inflate_4k_ri32_fv3": (4096, 32, 3, "xxh3", 1),
    "inflate_1k_ri16_fv5": (1024, 16, 5, "crc32c", 0),
    "inflate_16k_ri32_fv4": (16384, 32, 4, "xxh3", 1),
    "inflate_16k_ri16_fv3": (16384, 16, 3, "crc32c", 0),
    "inflate_64k_ri1_fv3": (65536, 1, 3, "crc32c", 1),
    "inflate_64k_ri16_fv5": (65536, 16, 5, "xxh3", 0),
}
# planned inflated block sizes at 4 KiB blocks: both sides of the fast path's limit and of the inflate window
INFLATE_TARGETS = (STAGE_LIMIT - 1, STAGE_LIMIT, STAGE_LIMIT + 1, INFLATE_WINDOW - 1, INFLATE_WINDOW, INFLATE_WINDOW + 1, 6500, 9000)


def _inflate_plan(name):
    """the ops script and options for the reference: three flushes (inputs) of planned blocks -- word soup that compresses, and
    stretches of random bytes that the builder stores raw"""
    bs, ri, fv, ck, ic = INFLATE_CONFIGS[name]
    ks = _Keys(80 + bs + ri + fv)
    rnd = ks.rnd
    ops = H.Ops()
    plans = []
    for run in range(3):
        t = _Table(ri, block_size=bs, deviation=10, fill=_texty)
        keys = iter(sorted(ks.key(8 + run) for _ in range(6000)))

        def entry(n, raw):
            return H.ikey(next(keys), 1, VALUE), (rnd.randbytes(n) if raw else _texty(rnd, n))
        nblk = 0
        if bs == 4096:
            for target in INFLATE_TARGETS:
                for _ in range(2):
                    es = []
                    while block_estimate(es, ri) < 2000:
                        es.append(entry(rnd.randint(20, 200), False))
                    t.add(es + [entry(0, False)], ("size", target))
                    nblk += 1
        while nblk < {1024: 60, 4096: 40, 16384: 10, 65536: 5}[bs]:
            raw = (nblk // (8 if bs <= 4096 else 2)) % 3 == 1  # a stretch of blocks that do not compress
            es = []
            lim = (bs * 90 + 99) // 100
            while True:
                e = entry(rnd.randint(20, min(400, bs // 2)) if rnd.random() < 0.9 else rnd.randint(bs // 2, bs), raw)
                if block_estimate(es + [e], ri) > lim:
                    break
                es.append(e)
            t.add(es + [entry(0, raw)], ("min",))
            nblk += 1
        planned, _ = t.plan(rnd)
        plans.append(planned)
        for entries, _ in planned:
            for k, v in entries:
                ops.put(k[:-8], v)
        ops.flush()
    opts = dict(target_file_size=1 << 20, input_compression="zlib", block_size=bs, restart_interval=ri, format_version=fv, checksum=ck,
                index_compression=ic)
    return ops, opts, plans


@functools.lru_cache(maxsize=None)
def inflate_case(name):
    """dict(ref, params, plans): the compiled reference's run (inputs it wrote and its outputs); needs oracle/_ref"""
    if name.endswith("_range"):
        c = inflate_case(name[:-len("_range")])
        ref, p = c["ref"], copy.copy(c["params"])
        keys = sorted({k[:-8] for d in ref["inputs"] for k, _ in sstfmt.parse_sst(d)["entries"]})
        p.range_start, p.range_end = keys[len(keys) // 3], keys[2 * len(keys) // 3]
        return dict(c, params=p)
    ops, opts, plans = _inflate_plan(name)
    ref = H.run_reference(ops, **opts)
    return dict(ref=ref, params=H.params_from_reference(ref), plans=plans)


# ------------------------------------------------------------------------------------------------ registry
CASES = {
    "staging_limit": lambda: _staging_limit(16, 5, "xxh3"),
    "staging_limit_crc32c_fv4": lambda: _staging_limit(4, 4, "crc32c"),
    **{f"rows_ri{ri}": (lambda ri=ri: _rows(ri)) for ri in (1, 15, 16, 17, 32)},
    "key_words": lambda: _key_words(41, False),
    "key_words_slow": lambda: _key_words(42, True),
    "headers": _headers,
    "skipped": lambda: _skipped(False),
    "skipped_nothing_kept": lambda: _skipped(True),
    **{f"index_walk_fv{fv}": (lambda fv=fv: _index_walk(fv, False)) for fv in (3, 4, 5)},
    **{f"index_walk_fv{fv}_range": (lambda fv=fv: _index_walk(fv, True)) for fv in (3, 4, 5)},
}
BIG_VALUE_CASES = {"headers_vlen_max": MAX_VLEN, "headers_vlen_too_long": MAX_VLEN + 1}
INFLATE_CASES = sorted(INFLATE_CONFIGS) + ["inflate_4k_ri16_fv5_range"]


@functools.lru_cache(maxsize=None)
def case(name):
    """dict(inputs, params): a built case (CASES, BIG_VALUE_CASES) or a reference-written one (INFLATE_CASES)"""
    if name in INFLATE_CASES:
        c = inflate_case(name)
        return dict(inputs=c["ref"]["inputs"], params=c["params"])
    if name in BIG_VALUE_CASES:
        inputs, p = _one_big_value(BIG_VALUE_CASES[name])
    else:
        inputs, p = CASES[name]()
    return dict(inputs=inputs, params=p)


@functools.lru_cache(maxsize=None)
def expected(name):
    """the case with the oracle's job over it: files, metas, stats"""
    c = case(name)
    files, metas, stats = H.oracle_compact(c["params"], c["inputs"])
    return dict(c, files=files, metas=metas, stats=stats)
