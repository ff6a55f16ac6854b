"""toplingdb_b200/csrc/inflate_rules.h (the raw DEFLATE decoder of the device's block decompression and of the host's compressed index
blocks) compiled for the host and checked against zlib: streams of all three block types (stored, fixed, dynamic Huffman) as the
reference's Zlib_Compress writes them (util/compression.h:746-826: raw deflate, window_bits -14), long matches, the 16 KiB window limit,
and malformed input (truncated streams, random bytes, output larger than the announced size) which must be refused, never overrun.
Also the varint32 size prefix in front of the stream, which both sides read with inf_size_prefix."""
import ctypes as C
import os
import random
import subprocess
import zlib

import pytest

import helpers as H

ROOT = H.ROOT


@pytest.fixture(scope="module")
def sim(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("inf") / "inflate_rules_sim.so")
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-std=c++17", "-I" + os.path.join(ROOT, "toplingdb_b200", "csrc"),
                           os.path.join(ROOT, "tests", "native", "inflate_rules_sim.cc"), "-o", so])
    L = C.CDLL(so)
    L.inflate_sim.restype = C.c_long
    L.inflate_sim.argtypes = [C.c_char_p, C.c_uint32, C.c_char_p, C.c_uint32]
    L.size_prefix_sim.restype = C.c_int
    L.size_prefix_sim.argtypes = [C.c_char_p, C.c_uint32, C.POINTER(C.c_uint64)]
    return L


def _deflate(data, level=-1, strategy=zlib.Z_DEFAULT_STRATEGY, wbits=-14):
    c = zlib.compressobj(level, zlib.DEFLATED, wbits, 8, strategy)
    return c.compress(data) + c.flush()


def _inflate(sim, comp, cap):
    dst = C.create_string_buffer(cap + 16)
    n = sim.inflate_sim(comp, len(comp), dst, cap)
    return n, dst.raw[:max(n, 0)], dst.raw[cap:]


def _samples():
    rnd = random.Random(11)
    yield b""
    yield b"a"
    yield b"abc" * 5000                                   # long matches at a short distance
    yield bytes(rnd.randrange(256) for _ in range(5000))  # incompressible: stored blocks / literals only
    yield bytes(rnd.choice(b"ab") for _ in range(20000))  # two symbols: very short codes
    yield b"".join(b"key%08d" % i + bytes([rnd.randrange(4)]) * 20 for i in range(3000))  # what a data block looks like
    base = bytes(rnd.randrange(256) for _ in range(300))
    yield base + bytes(16000) + base + bytes(20000) + base  # matches just inside / outside a 16 KiB window
    yield bytes(70000)                                     # run of one byte: distance 1, maximal lengths


@pytest.mark.parametrize("level,strategy", [(0, zlib.Z_DEFAULT_STRATEGY), (1, zlib.Z_DEFAULT_STRATEGY), (-1, zlib.Z_DEFAULT_STRATEGY),
                                            (9, zlib.Z_DEFAULT_STRATEGY), (6, zlib.Z_FIXED), (6, zlib.Z_HUFFMAN_ONLY), (6, zlib.Z_RLE)])
def test_streams_of_every_block_type_inflate_to_the_original(sim, level, strategy):
    for data in _samples():
        comp = _deflate(data, level, strategy)
        n, got, guard = _inflate(sim, comp, len(data))
        assert n == len(data) and got == data, (level, strategy, len(data))
        assert guard == bytes(16)
        if data:
            assert _inflate(sim, comp, len(data) - 1)[0] == -1  # one byte short: refused, nothing behind the buffer touched


def test_malformed_streams_are_refused(sim):
    rnd = random.Random(3)
    data = b"".join(b"key%08d" % i + b"v" * 30 for i in range(2000))
    comp = _deflate(data)
    for cut in (0, 1, 2, 5, len(comp) // 2, len(comp) - 1):
        n, _, guard = _inflate(sim, comp[:cut], len(data))
        assert n == -1 and guard == bytes(16), cut
    bad = 0
    for _ in range(300):  # random bytes: whatever they decode to, the output buffer is never overrun
        junk = bytes(rnd.randrange(256) for _ in range(rnd.randrange(1, 200)))
        n, _, guard = _inflate(sim, junk, 4096)
        assert guard == bytes(16)
        bad += n == -1
    assert bad > 200
    # a flipped bit somewhere in a valid stream: either an error or different bytes, never a crash
    for pos in range(0, len(comp), max(1, len(comp) // 64)):
        c2 = bytearray(comp)
        c2[pos] ^= 0x10
        n, got, guard = _inflate(sim, bytes(c2), len(data))
        assert guard == bytes(16) and (n == -1 or n <= len(data))


def test_agrees_with_zlib_on_random_streams(sim):
    rnd = random.Random(7)
    for _ in range(200):
        n = rnd.randrange(0, 9000)
        alphabet = rnd.randrange(1, 257)
        data = bytes(rnd.randrange(alphabet) for _ in range(n))
        if rnd.random() < 0.5 and n > 100:  # splice in repeats
            k = rnd.randrange(10, 100)
            data = data[:n // 2] + data[:k] * rnd.randrange(1, 20) + data[n // 2:]
        comp = _deflate(data, rnd.choice([0, 1, 6, 9]), rnd.choice([zlib.Z_DEFAULT_STRATEGY, zlib.Z_FIXED, zlib.Z_FILTERED]))
        got_n, got, _ = _inflate(sim, comp, len(data))
        assert got_n == len(data) and got == zlib.decompress(comp, -14)


def _varint(u):
    out = bytearray()
    while u >= 128:
        out.append(u & 127 | 128)
        u >>= 7
    return bytes(out + bytes([u]))


def _prefix(sim, data, size=None):
    u = C.c_uint64(0xdead)
    n = sim.size_prefix_sim(data, len(data) if size is None else size, C.byref(u))
    return n, u.value if n else None


def test_size_prefix_reads_one_to_five_bytes_within_the_block(sim):
    for u in (0, 1, 4, 8, 127, 128, 6144, 16383, 16384, (1 << 21) - 1, 1 << 21, (1 << 28) - 1, 1 << 28, 0x7fffffff, 1 << 31,
              (1 << 32) - 1, (1 << 35) - 1):
        enc = _varint(u)
        assert _prefix(sim, enc + b"\x01\x02") == (len(enc), u), u  # (the stream behind the prefix is not read)
        assert _prefix(sim, enc + b"\x01", len(enc) - 1) == (0, None), u  # cut by the block's end
    for enc in (b"\x80" * 5 + b"\x01", b"\xff" * 6, b"\x80\x80\x80\x80\x80"):  # no end within the first five bytes
        assert _prefix(sim, enc) == (0, None), enc
    assert _prefix(sim, b"", 0) == (0, None)
    assert _prefix(sim, b"\x85\x80\x80\x80\x00") == (5, 5)  # zero-padded: five bytes, as the reference's GetVarint32 reads them
