"""Data blocks that the emit kernels leave to their fallback builder (more than 96 entries, or larger than a warp's image slot) and the
same value shapes in small blocks that the kernels build themselves: whole jobs through the C ABI against the CPU oracle.  The value
lengths cover every copy path of the block builders: empty, 1-32 bytes, 33-64, 65-127, 128-300, and one value larger than the 24 KiB
image slot, so that its block is written straight into the file image (block_builder.cc:97-253, block_based_table_builder.cc:1277-1378)."""
import random
import struct

import pytest

import helpers as H

pytestmark = pytest.mark.gpu

CLASSES = ((0, 0), (1, 32), (33, 64), (65, 127), (128, 300))
BIG_VALUE = 30000  # larger than the largest image slot (24 KiB)


def _runs(seed, classes, big, nruns=3, n=3000):
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
            run[i] = (run[i][0], rnd.randbytes(BIG_VALUE))
        runs.append(run)
    return list(reversed(runs))  # newest run first


def _check(p, runs):
    from gpu_harness import run_product
    inputs = [H.oracle_build_sst(H.Params(), H.kvstream(r)) for r in runs]
    want, wmetas, wst = H.oracle_compact(p, inputs)
    files, metas, st = run_product(p, inputs)
    assert [len(f) for f in files] == [len(o) for o in want]
    for i, (a, b) in enumerate(zip(files, want)):
        assert a == b, f"output {i} differs at byte {next(j for j in range(len(a)) if a[j] != b[j])}"
    for k in H.STAT_KEYS:
        assert getattr(st, k) == getattr(wst, k), k
    for m, om in zip(metas, wmetas):
        assert (m.file_size, m.num_entries, m.num_data_blocks) == (om.file_size, om.num_entries, om.num_data_blocks)


@pytest.mark.parametrize("ri", (1, 16))
@pytest.mark.parametrize("ck", ("xxh3", "crc32c"))
def test_fallback_blocks_match_oracle(ri, ck):
    """16 KiB blocks of ~170 entries with values of every length class mixed, and one block that overflows the image slot"""
    p = H.Params(bottommost_level=True, block_size=16384, block_restart_interval=ri, checksum=ck)
    _check(p, _runs(31 + ri, CLASSES, big=True))


@pytest.mark.parametrize("cls", CLASSES, ids=lambda c: f"v{c[0]}-{c[1]}")
def test_small_blocks_match_oracle(cls):
    """1 KiB blocks (at most 96 entries: built by the emit kernels themselves) with values of one length class"""
    p = H.Params(bottommost_level=True, block_size=1024, block_restart_interval=16, checksum="xxh3")
    _check(p, _runs(7 + cls[0], (cls,), big=False))
