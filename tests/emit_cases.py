"""Jobs for the data-block emit stage (encode_emit_kernel, encode_emit_long_kernel and emit_block_warp in csrc/encode.cu).

The launcher picks the kernel by the mean on-disk bytes per entry (the staged kernel up to 64, the long kernel above).  In a block
of at most kEmitMaxEntries entries that fits the warp's image slot, lane l writes entries [3l, 3l + 3): the values of a group of
three that are all <= 32 bytes leave through the kernel's short-value load (16-byte chunks in the staged kernel, 4-byte words in
the long one), otherwise a value of <= 64 bytes is copied by its lane and a longer one by the whole warp.  Every other block goes to
emit_block_warp, built in the slot when it fits there and straight in the file image when it does not.  The jobs below put blocks,
lane groups and values on each of those paths:
- kernel selection: the cases of every other group once per kernel (filler entries behind the case's own steer the mean), and two
  jobs whose data blocks total exactly 64 n and 64 n + 1 bytes;
- values of 0 and 1-32 bytes at every source phase mod 16; 33-64-byte values at every phase, also beside short ones in one group;
  65-600-byte values of every length mod 4, one and two 512-byte passes;
- restart intervals 1, 16, 128 (mask) and 3, 17 (divide), 128 with one restart per block;
- blocks of 96 and 97 entries; blocks whose payload + 53 bytes equals the image slot and exceeds it by one, at the lower clamp
  (5632 bytes), a middle slot and the upper clamp (24 KiB);
- emit_block_warp in the slot and in the file image, under both restart-interval paths;
- xxh3 blocks of <= 240 and > 240 payload bytes, crc32c;
- the seven compaction jobs that mix fallback blocks with the emit kernels' own.

`build(name) -> (params, data)`: data is ("kv", entries) for a job through b200c_job_encode_kv (values at arena + off + klen in
one cudaMalloc'ed arena, so the case sets every value's source phase mod 16) and ("compact", inputs) for a compaction job.
tests/test_emit_cases_cpu.py proves from the oracle's output layout that each case reaches the paths it is named for."""
import functools
import os
import random
import re
import struct

import helpers as H

_CSRC = os.path.join(H.ROOT, "toplingdb_b200", "csrc")
ENCODE = open(os.path.join(_CSRC, "encode.cu")).read()


def _constant(name):
    m = re.search(r"constexpr\s+int\s+%s\s*=\s*(\d+)\s*;" % name, ENCODE)
    assert m, f"{name} not found in encode.cu"
    return int(m.group(1))


PER_LANE = _constant("kEmitPerLane")
assert "constexpr int kEmitMaxEntries = 32 * kEmitPerLane;" in ENCODE
MAX_ENTRIES = 32 * PER_LANE
# encode_emit_slice: block_size * 5 / 4 + 512, rounded up to 256, clamped to [5632, 24 KiB]
assert re.search(r"uint32_t s = block_size \+ block_size / 4 \+ 512;\s*s = \(s \+ 255\) & ~255u;\s*if \(s < 5632\) s = 5632;\s*"
                 r"if \(s > 24 \* 1024\) s = 24 \* 1024;", ENCODE)
SLOT_MIN, SLOT_MAX = 5632, 24 * 1024
# the emit kernels' fit rule, emit_block_warp's slot rule and the launcher's kernel selection
# emit_block_fits: body + 4 nrest + 4 (= the payload) + 5 + 32 + 16 <= slot; payload + FIT_OVER > slot leaves the fast path
assert "return body + 4ull * nrest + 4 + 5 + 32 + 16 <= slot_bytes;" in ENCODE
FIT_OVER = 5 + 32 + 16
assert "const bool staged = payload + 5 + 16 <= slot_bytes;" in ENCODE
assert "const bool long_entries = data_bytes > 64 * m.n;" in ENCODE
BIG = 1 << 30


def slot_bytes(block_size):
    s = (block_size + block_size // 4 + 512 + 255) & ~255
    return min(max(s, SLOT_MIN), SLOT_MAX)


def arena_phases(entries):
    """source phase (mod 16) of every value in b200c_job_encode_kv's arena: key and value bytes back to back from a 256-byte
    aligned start"""
    out, o = [], 0
    for k, v in entries:
        out.append((o + len(k)) % 16)
        o += len(k) + len(v)
    return out


class _Keys:
    """internal keys in increasing order: a 2-byte counter, then filler up to the wanted user-key length (2..16)"""

    def __init__(self, seed):
        self.c, self.rnd = 0, random.Random(seed)

    def next(self, ulen):
        assert 2 <= ulen <= 16 and self.c < 1 << 16
        k = struct.pack(">H", self.c) + bytes(self.rnd.choice(b"ab") for _ in range(ulen - 2))
        self.c += 1
        return H.ikey(k, self.c)


def _place(specs, seed, keys=None):
    """specs: [(value length, source phase mod 16 or None)] -> entries whose values sit at those phases in the arena.  The key length
    sets the phase; when the phase needs a 9-byte key (user key of 1 byte), a 10-byte key with an empty value goes in front."""
    rnd = random.Random(seed)
    keys = keys or _Keys(seed)
    out, o = [], 0
    for vlen, ph, *ulen in specs:  # (a third element fixes the user-key length)
        if ulen:
            ulen = ulen[0]
        elif ph is None:
            ulen = rnd.randint(2, 16)
        else:
            need = (ph - o - 8) % 16
            if need == 1:
                out.append((keys.next(2), b""))
                o += 10
                need = (ph - o - 8) % 16
            ulen = need if need >= 2 else need + 16
        k = keys.next(ulen)
        out.append((k, rnd.randbytes(vlen)))
        o += len(k) + vlen
    return out, keys


def _steer(entries, keys, kernel, seed):
    """entries behind the case's own that put the job's mean entry on the kernel's side of 64 bytes (with a margin the CPU test
    checks against the oracle's layout)"""
    rnd = random.Random(seed)
    est = lambda: sum(len(k) + len(v) + 4 for k, v in entries) * 1.1 + 64
    while (est() > 56 * len(entries)) if kernel == "staged" else (est() < 72 * len(entries)):
        entries.append((keys.next(8), b"" if kernel == "staged" else rnd.randbytes(2000)))
    return entries


def _classes(n, classes, seed):
    rnd = random.Random(seed)
    return [(rnd.randint(*rnd.choice(classes)), rnd.randrange(16)) for _ in range(n)]


def _short(seed):
    specs = [(v, ph) for v in range(33) for ph in range(16)]
    random.Random(seed).shuffle(specs)
    return specs


def _per_lane(seed):
    rnd = random.Random(seed)
    specs = [(rnd.randint(33, 64), i % 16) for i in range(320)] + [(rnd.randint(0, 32), rnd.randrange(16)) for _ in range(320)]
    rnd.shuffle(specs)
    return specs


def _warp(seed):
    rnd = random.Random(seed)
    specs = [(65 + 4 * rnd.randrange(134) + i % 4, i // 4 % 16) for i in range(192)]  # 65..600, every length and phase mod 4
    specs += [(rnd.randint(513, 600), rnd.randrange(16)) for _ in range(16)]            # two 512-byte passes
    rnd.shuffle(specs)
    return specs


MIXED = ((0, 0), (1, 32), (33, 64), (65, 300))
UNIFORM = dict(block_size_deviation=0)

# name -> (params, entries builder(seed) -> specs); every one runs once per kernel ("<name>_staged", "<name>_long")
_KV = {
    "short": (dict(block_size=1024), _short),
    "per_lane": (dict(block_size=2048), _per_lane),
    "warp": (dict(block_size=4096), _warp),
    "checksum_xxh3": (dict(block_size=256, checksum="xxh3"), lambda s: _classes(600, MIXED[:3], s)),
    "checksum_crc32c": (dict(block_size=256, checksum="crc32c"), lambda s: _classes(600, MIXED[:3], s)),
    # emit_block_warp: 16 KiB blocks of ~170 entries in the slot, one value larger than the largest slot in the file image
    "block_warp_r3": (dict(block_size=16384, block_restart_interval=3), lambda s: _classes(1500, MIXED, s) + [(30000, 5)]),
    "block_warp_r16": (dict(block_size=16384, block_restart_interval=16), lambda s: _classes(1500, MIXED, s) + [(30000, 5)]),
}
for _r in (1, 3, 16, 17, 128):  # 128: one restart per block
    _KV[f"restart{_r}"] = (dict(block_size=1024, block_restart_interval=_r), lambda s: _classes(500, MIXED, s))
# with restart interval 1 and deviation 0 every block holds the first k entries whose payload (27 bytes each + 4) reaches block_size
for _k in (MAX_ENTRIES, MAX_ENTRIES + 1):
    _KV[f"entries{_k}"] = (dict(block_size=4 + 27 * _k, block_restart_interval=1, **UNIFORM), lambda s, k=_k: [(4, None, 8)] * (3 * k))
# blocks whose payload + FIT_OVER equals the slot and exceeds it by one: the block size of each slot class, small values in front
FIT_BLOCK_SIZES = {"fit_min": 4096, "fit_mid": 8192, "fit_max": 20000}
for _n, _b in FIT_BLOCK_SIZES.items():
    _KV[_n] = (dict(block_size=_b, **UNIFORM), None)

CASES = [f"{n}_{k}" for n in _KV for k in ("staged", "long")] + ["select_64n", "select_64n_plus_1"] + \
    [f"fallback_r{r}_{c}" for r in (1, 16) for c in ("xxh3", "crc32c")] + \
    [f"small_v{lo}-{hi}" for lo, hi in ((0, 0), (1, 32), (33, 64), (65, 127), (128, 300))]


def layout(data):
    """one oracle file -> [(offset, payload bytes, [(key, value)])] of its data blocks"""
    import sstfmt
    out = []
    for _, h in sstfmt.parse_sst(data)["index"]:
        payload, _, _ = sstfmt.read_block(data, h)
        out.append((h[0], h[1], [(k, v) for k, v, _ in sstfmt.block_entries(payload)]))
    return out


def _oracle_blocks(p, entries):
    return layout(H.oracle_build_sst(p, H.kvstream(entries)))


def _fit_entries(p, seed):
    """for each target payload slot - FIT_OVER and one more: a block of small entries below block_size, then one entry whose value
    brings the payload to the target (solved against the oracle)"""
    rnd = random.Random(seed)
    slot = slot_bytes(p.block_size)
    small = p.block_size // 80
    k = int(p.block_size * 0.8) // (small + 20)
    assert k < MAX_ENTRIES
    keys, groups = _Keys(seed), []
    for target in (slot - FIT_OVER, slot - FIT_OVER + 1):
        g = [(keys.next(8), rnd.randbytes(small)) for _ in range(k)]
        g.append((keys.next(8), rnd.randbytes(target - (small + 20) * k)))
        groups.append(g)
    for _ in range(8):
        entries = [e for g in groups for e in g]
        blocks, done = _oracle_blocks(p, entries), True
        for g, target in zip(groups, (slot - FIT_OVER, slot - FIT_OVER + 1)):
            size = next(b[1] for b in blocks if b[2][-1][0] == g[-1][0])
            if size != target:
                done = False
                g[-1] = (g[-1][0], g[-1][1][:len(g[-1][1]) + target - size] + rnd.randbytes(max(0, target - size)))
        if done:
            return entries, keys
    raise AssertionError("fit case did not converge")


def _select_entries(p, extra, seed):
    """entries whose data blocks total exactly 64 n + extra bytes: one value of a few hundred bytes absorbs the difference"""
    rnd = random.Random(seed)
    entries, _ = _place([(rnd.randint(25, 45), None) for _ in range(2000)], seed)
    mid = len(entries) // 2
    entries[mid] = (entries[mid][0], rnd.randbytes(4000))
    for _ in range(16):
        d = 64 * len(entries) + extra - sum(b[1] + 5 for b in _oracle_blocks(p, entries))
        if d == 0:
            return entries
        entries[mid] = (entries[mid][0], rnd.randbytes(len(entries[mid][1]) + d))
    raise AssertionError("selection case did not converge")


def _compaction_runs(seed, classes, big, nruns=3, n=3000):
    rnd = random.Random(seed)
    runs, seq = [], 1
    for r in range(nruns):
        dedup = {}
        for k in sorted(rnd.sample(range(nruns * n * 4), n)):
            # variable-length user keys (4..16 bytes) so that shared prefixes and restart points vary
            kb = struct.pack(">QQ", k >> 2, (k * 0x9E3779B97F4A7C15) & ((1 << 64) - 1))[:4 + (k % 13)]
            lo, hi = rnd.choice(classes)
            dedup[kb] = (kb + struct.pack("<Q", (seq << 8) | 1), rnd.randbytes(rnd.randint(lo, hi)))
            seq += 1
        run = [dedup[kb] for kb in sorted(dedup)]
        if big and r == 0:
            i = len(run) // 2
            run[i] = (run[i][0], rnd.randbytes(30000))  # larger than the largest image slot
        runs.append(run)
    return list(reversed(runs))  # newest run first


@functools.lru_cache(maxsize=None)
def build(name):
    seed = sum(map(ord, name))
    if name.startswith(("fallback_", "small_")):
        classes = ((0, 0), (1, 32), (33, 64), (65, 127), (128, 300))
        if name.startswith("fallback_"):
            r, ck = name[len("fallback_r"):].split("_")
            p = H.Params(bottommost_level=True, block_size=16384, block_restart_interval=int(r), checksum=ck)
            runs = _compaction_runs(31 + int(r), classes, big=True)
        else:
            lo, hi = map(int, name[len("small_v"):].split("-"))
            p = H.Params(bottommost_level=True, block_size=1024, block_restart_interval=16, checksum="xxh3")
            runs = _compaction_runs(7 + lo, ((lo, hi),), big=False)
        return p, ("compact", tuple(H.oracle_build_sst(H.Params(), H.kvstream(r)) for r in runs))
    if name.startswith("select_"):
        p = H.Params(block_size=4096, max_output_file_size=BIG)
        return p, ("kv", tuple(_select_entries(p, int(name == "select_64n_plus_1"), seed)))
    base, kernel = name.rsplit("_", 1)
    params, specs = _KV[base]
    p = H.Params(max_output_file_size=BIG, **params)
    entries, keys = _fit_entries(p, seed) if specs is None else _place(specs(seed), seed)
    return p, ("kv", tuple(_steer(entries, keys, kernel, seed)))
