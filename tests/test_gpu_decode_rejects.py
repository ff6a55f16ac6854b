"""The decoder's rejection classes: malformed or unsupported input tables and the status and error words each one ends in.

Which error bits a block raises decides between ERR_NOT_SUPPORTED (the job goes back to the CPU) and ERR_CORRUPTION (a failed
compaction), so every class is pinned on a block staged in shared memory (fast path) and on one that is not (slow path), where both
exist.  Tables come from the oracle's builder with checksum type none; each case then rewrites bytes of one data block (or of the index
block) in place, so sizes, offsets and entry counts stay what the builder wrote and the intended fault is the only one.

The CPU tests prove that each rewritten block reaches the path it is meant for (decode_cases.block_path, as in
test_decode_cases_cpu.py); the GPU test runs the job and compares the status and the exact set of error words."""
import struct

import pytest

import decode_cases as D
import helpers as H
import sstfmt

CORRUPT, IRREGULAR = "corrupt-block", "restart-intervals-of-unequal-length"
KEY_TOO_LONG, VALUE_TOO_LONG = "user-key-longer-than-16-bytes", "value>=128MiB"
BAD_TYPE = "value-type-outside-{Value,Deletion,SingleDeletion}"
TYPE_MERGE = 2

# (block_size, restart interval, value length, entries): small blocks that are staged; blocks larger than the staging slice; small
# blocks of more than kDecRows restart intervals (staged, then the slow path)
SHAPES = {"staged": (512, 4, 20, 100), "unstaged": (6000, 4, 200, 120), "staged_many_rows": (1024, 1, 20, 100)}


def _uk(i):
    return struct.pack(">QQ", 7, i << 8)


def _table(shape, **kw):
    bs, ri, vlen, n = SHAPES[shape]
    es = [(H.ikey(_uk(i), 1000 + i), bytes((i + t) & 0x7F for t in range(vlen))) for i in range(n)]
    p = H.Params(block_size=bs, block_size_deviation=0, block_restart_interval=ri, checksum="none", **kw)
    return bytearray(H.oracle_build_sst(p, H.kvstream(es)))


def _block(data, j=1):
    """(file offset, payload, restart offsets, rows) of data block j"""
    off, size = sstfmt.parse_sst(bytes(data))["index"][j][1]
    payload = bytes(data[off:off + size])
    nr = struct.unpack_from("<I", payload, size - 4)[0] & 0x7FFFFFFF
    rs = list(struct.unpack_from("<%dI" % nr, payload, size - 4 - 4 * nr))
    rows, _ = D.parse_block(payload)
    return off, payload, rs, rows


def _put_restarts(data, j, rs):
    off, payload, _, _ = _block(data, j)
    struct.pack_into("<%dI" % len(rs), data, off + len(payload) - 4 - 4 * len(rs), *rs)


def _rewrite_entry(data, j, row, i, shared=None, non_shared=None, vlen=None, hdr=None):
    """entry i of restart interval `row` of block j with other header fields; bytes after the header stay where they are"""
    off, _, _, rows = _block(data, j)
    q, sh, ns, vl, h = rows[row][i]
    new = hdr if hdr is not None else (_varint(sh if shared is None else shared) + _varint(ns if non_shared is None else non_shared)
                                       + _varint(vl if vlen is None else vlen))
    assert len(new) == h, "the header keeps its length"
    data[off + q:off + q + h] = new


def _varint(x):
    out = bytearray()
    while x >= 0x80:
        out.append((x & 0x7F) | 0x80)
        x >>= 7
    out.append(x)
    return bytes(out)


def _long_key(data, restart):
    """one more key byte taken from the value: a 17-byte user key at a restart point or behind one"""
    _, _, _, rows = _block(data)
    i = 0 if restart else 1
    _, sh, ns, vl, _ = rows[1][i]
    _rewrite_entry(data, 1, 1, i, non_shared=ns + 1, vlen=vl - 1)


def _merge_type(data):
    off, _, _, rows = _block(data)
    q, sh, ns, vl, h = rows[1][1]
    data[off + q + h + ns - 8] = TYPE_MERGE


def _padded_header(data):
    """shared and non_shared as five-byte varints (GetVarint32Ptr reads them): a header longer than 8 bytes, the value 8 bytes shorter"""
    off, _, _, rows = _block(data)
    q, sh, ns, vl, h = rows[1][1]
    pad = lambda x: bytes([x | 0x80, 0x80, 0x80, 0x80, 0x00])  # noqa: E731
    hdr = pad(sh) + pad(ns) + _varint(vl - 8)
    assert len(hdr) == h + 8
    a = off + q
    data[a:a + h + ns + vl] = hdr + data[a + h:a + h + ns] + data[a + h + ns + 8:a + h + ns + vl]


def _swap_restarts(data):
    _, _, rs, _ = _block(data)
    rs[1], rs[2] = rs[2], rs[1]
    _put_restarts(data, 1, rs)


def _past_interval(data):
    _, _, _, rows = _block(data)
    _, sh, ns, vl, _ = rows[0][-1]
    _rewrite_entry(data, 1, 0, len(rows[0]) - 1, vlen=vl + 1)


def _irregular(data):
    _, _, rs, _ = _block(data)
    rs[2] = rs[3]  # interval 1 holds two intervals' entries, interval 2 none
    _put_restarts(data, 1, rs)


def _handle_past_end(data):
    """block 0's size in the index grows to the largest value of its varint length, past the end of the file"""
    t = sstfmt.parse_sst(bytes(data))
    io, _ = t["footer"]["index"]
    p = io
    shared, p = sstfmt.varint(data, p)
    ns, p = sstfmt.varint(data, p)
    assert shared == 0
    p += ns
    _, p = sstfmt.varint(data, p)
    size, e = sstfmt.varint(data, p)
    n = e - p
    assert (1 << (7 * n)) - 1 + 5 > len(data)
    data[p:e] = bytes([0xFF] * (n - 1) + [0x7F])


MUTATIONS = {
    "long_key_at_restart": lambda d: _long_key(d, True),
    "long_key_behind_restart": lambda d: _long_key(d, False),
    "merge_type": _merge_type,
    "padded_header": _padded_header,
    "restarts_out_of_order": _swap_restarts,
    "entry_past_its_interval": _past_interval,
    "irregular_intervals": _irregular,
}
# (case, shape) -> (status, error words) of the job.  A block the decoder drops contributes no entries, and the merge over the run that
# lost them reports key-order/partition as well
KEY_ORDER = "key-order/partition"
CASES = {
    ("long_key_at_restart", "staged"): ("NOT_SUPPORTED", {KEY_TOO_LONG}),
    ("long_key_at_restart", "unstaged"): ("NOT_SUPPORTED", {KEY_TOO_LONG}),
    ("long_key_behind_restart", "staged"): ("NOT_SUPPORTED", {KEY_TOO_LONG}),
    ("long_key_behind_restart", "unstaged"): ("NOT_SUPPORTED", {KEY_TOO_LONG}),
    ("merge_type", "staged"): ("NOT_SUPPORTED", {BAD_TYPE}),
    ("merge_type", "unstaged"): ("NOT_SUPPORTED", {BAD_TYPE}),
    ("padded_header", "staged"): ("CORRUPTION", {CORRUPT}),
    ("padded_header", "unstaged"): ("CORRUPTION", {CORRUPT}),
    ("restarts_out_of_order", "staged"): ("CORRUPTION", {CORRUPT, KEY_ORDER}),
    ("restarts_out_of_order", "unstaged"): ("CORRUPTION", {CORRUPT, IRREGULAR, KEY_ORDER}),
    ("entry_past_its_interval", "staged"): ("CORRUPTION", {CORRUPT, KEY_ORDER}),
    ("entry_past_its_interval", "staged_many_rows"): ("CORRUPTION", {CORRUPT, IRREGULAR, KEY_ORDER}),
    ("entry_past_its_interval", "unstaged"): ("CORRUPTION", {CORRUPT, IRREGULAR, KEY_ORDER}),
    # (the decoder raises the irregular bit alone; the merge's key-order bit makes the job a corruption)
    ("irregular_intervals", "unstaged"): ("CORRUPTION", {IRREGULAR, KEY_ORDER}),
}
# (index_block_restart_interval, error words).  The sequential walk goes on from the rejected handle (offset 0, size 4), so the next
# delta-encoded handles point into the wrong bytes and the block decoder reports what it finds there as well
INDEX_CASES = {"handle_past_end_parallel_index": (1, {CORRUPT, KEY_ORDER}),
               "handle_past_end_sequential_index": (4, {CORRUPT, KEY_ORDER, "compressed-block"})}


def _case(name, shape):
    data = _table(shape)
    MUTATIONS[name](data)
    return bytes(data)


def _index_case(name):
    """(the table, the table with block 0's handle past the end of the file)"""
    data = _table("staged", index_block_restart_interval=INDEX_CASES[name][0])
    bad = bytearray(data)
    _handle_past_end(bad)
    return bytes(data), bytes(bad)


def _params(ri):
    return H.Params(block_restart_interval=ri, checksum="none", file_creation_times=[7])


# ------------------------------------------------------------------------------------------------ CPU: each case is on its path
def _path(data, j=1):
    off, payload, rs, _ = _block(data, j)
    staged = off % 16 + len(payload) <= D.STAGE_LIMIT
    return staged, len(rs)


@pytest.mark.parametrize("name,shape", sorted(CASES))
def test_reject_case_reaches_its_path(name, shape):
    data = _case(name, shape)
    staged, nr = _path(data)
    assert staged == (shape != "unstaged"), (name, shape)
    assert (nr > D.DEC_ROWS) == (shape == "staged_many_rows"), (name, shape, nr)
    off, payload, rs, rows = _block(data)
    if name.startswith("long_key") or name == "merge_type" or name == "padded_header":
        row = rows[1]
        i = 0 if name == "long_key_at_restart" else 1
        q, sh, ns, vl, h = row[i]
        assert (q == rs[1]) == (i == 0) and (sh == 0) == (i == 0)
        if name.startswith("long_key"):
            assert sh + ns == 16 + 1 + 8
        elif name == "merge_type":
            assert payload[q + h + ns - 8] == TYPE_MERGE
        else:
            assert h > 8 and sh + ns <= 24 and vl <= D.MAX_VLEN
        want = ("slow", "header") if name == "padded_header" else ("fast", "")
        assert D.block_path(len(payload), off % 16, rows) == (want if shape == "staged" else ("slow", "not staged"))
    elif name == "restarts_out_of_order":
        assert rs[1] > rs[2]
    elif name == "entry_past_its_interval":
        q, sh, ns, vl, h = rows[0][-1]
        assert q + h + ns + vl == rs[1] + 1
    elif name == "irregular_intervals":
        assert rs[2] == rs[3] and len(set(len(r) for r in rows[:-1])) > 1


@pytest.mark.parametrize("name", sorted(INDEX_CASES))
def test_index_case_reaches_its_path(name):
    data, bad = _index_case(name)
    info = D.index_info(data)  # (sstfmt reads every handle: the intact table)
    assert info["parallel"] == (INDEX_CASES[name][0] == 1) and info["nblocks"] > 1
    assert len(bad) == len(data) and sum(a != b for a, b in zip(data, bad)) >= 1


def test_value_of_2_to_the_27_bytes_is_on_the_slow_path():
    data = D.case("headers_vlen_too_long")["inputs"][0]
    big = [b for b in D.table_blocks(data) if max(vl for row in b["rows"] for *_, vl, _ in row) == D.MAX_VLEN + 1]
    assert len(big) == 1 and big[0]["path"] == "slow" and big[0]["why"] == "not staged"


# ------------------------------------------------------------------------------------------------ GPU: status and error words
def _reject(params, inputs):
    from gpu_harness import run_product
    import toplingdb_b200 as T
    with pytest.raises(T.B200cError) as ei:
        run_product(params, inputs)
    msg = str(ei.value)
    assert "device reported:" in msg, msg
    code = {T.native.ERR_NOT_SUPPORTED: "NOT_SUPPORTED", T.native.ERR_CORRUPTION: "CORRUPTION"}.get(ei.value.code, ei.value.code)
    return code, set(msg.split("device reported:", 1)[1].split())


@pytest.mark.gpu
@pytest.mark.parametrize("name,shape", sorted(CASES))
def test_decoder_rejects_with_its_status_and_words(name, shape):
    assert _reject(_params(SHAPES[shape][1]), [_case(name, shape)]) == CASES[(name, shape)]


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(INDEX_CASES))
def test_index_handle_past_the_file_is_corrupt(name):
    assert _reject(_params(SHAPES["staged"][1]), [_index_case(name)[1]]) == ("CORRUPTION", INDEX_CASES[name][1])


@pytest.mark.gpu
def test_value_of_2_to_the_27_bytes_is_not_supported():
    c = D.case("headers_vlen_too_long")
    assert _reject(c["params"], c["inputs"]) == ("NOT_SUPPORTED", {VALUE_TOO_LONG})
