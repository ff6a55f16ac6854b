"""The product's output-file cut rules with the fixed-prefix partitioner's events as a second event source
(toplingdb_b200/csrc/gp_rules.h: gp_next_event / gp_block_cut / gp_size_cut, the code the encoder's stitch walk runs on the device)
compiled for the host and driven over the block layout of finished jobs (tests/native/partition_rules_sim.cc).  They must cut exactly
where the oracle did (synthetic and random shapes) and where the unmodified reference did.  CPU only: the host-logic half of
test_gpu_partitioner.py."""
import bisect
import ctypes as C
import os
import random
import subprocess

import pytest

import gp_cases
import helpers as H
import partition_cases as PC
import sstfmt

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def sim(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("part") / "partition_rules_sim.so")
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-std=c++17", "-I" + os.path.join(ROOT, "toplingdb_b200", "csrc"),
                           os.path.join(ROOT, "tests", "native", "partition_rules_sim.cc"), "-o", so])
    L = C.CDLL(so)
    L.partition_rules_sim.restype = C.c_int64
    return L


def _layout(files):
    """output files -> (user keys of all entries, blocks [(first entry, count, flushed bytes before, last of file)], file starts)"""
    ukeys, blocks, starts = [], [], []
    for data in files:
        t = sstfmt.parse_sst(data)
        starts.append(len(ukeys))
        hs = [h for _, h in t["index"]]
        for i, h in enumerate(hs):
            payload, _, _ = sstfmt.read_block(data, h)
            ents = list(sstfmt.block_entries(payload))
            blocks.append((len(ukeys), len(ents), h[0], i == len(hs) - 1))
            ukeys += [k[:-8] for k, _, _ in ents]
    return ukeys, blocks, starts


def _run(sim, p, files):
    """(cuts of the rules, file starts of the layout that the size rule did not make, number of partition events)"""
    ukeys, blocks, starts = _layout(files)
    gps = p.grandparents if p.output_level > 0 else []
    G = len(gps)
    lo = [bisect.bisect_left(ukeys, a) for a, _, _ in gps]
    eq = [bisect.bisect_left(ukeys, b) for _, b, _ in gps]
    hi = [bisect.bisect_right(ukeys, b) for _, b, _ in gps]
    same = [int(i + 1 < G and gps[i + 1][0] == gps[i][1]) for i in range(G)]
    pev = PC.prefix_events(ukeys, p.sst_partitioner_prefix_len) if p.output_level > 0 else []
    u64 = lambda v: (C.c_uint64 * max(1, len(v)))(*v)
    target = p.target_output_file_size or p.max_output_file_size
    cap = 2 * G + 2 + len(pev)
    cuts = (C.c_uint64 * cap)()
    n = sim.partition_rules_sim(C.c_uint32(G), u64(lo), u64(eq), u64(hi), u64([s for _, _, s in gps]), (C.c_uint8 * max(1, G))(*same),
                                C.c_uint32(int(p.level_compaction_dynamic_file_size)), C.c_uint64(p.max_compaction_bytes or 25 * target),
                                C.c_uint64(target), u64(pev), C.c_uint32(len(pev)),
                                C.c_uint64(p.max_output_file_size if p.output_level > 0 else (1 << 64) - 1), C.c_uint64(len(ukeys)),
                                C.c_uint64(len(blocks)), u64([b[0] for b in blocks]), (C.c_uint32 * len(blocks))(*[b[1] for b in blocks]),
                                u64([b[2] for b in blocks]), (C.c_uint8 * len(blocks))(*[int(b[3]) for b in blocks]), cuts, C.c_uint64(cap))
    assert n >= 0, f"rules disagree with the layout at block {-n - 1}"
    size_cut = {blocks[i + 1][0] for i, b in enumerate(blocks[:-1]) if b[3] and b[2] >= p.max_output_file_size}
    return list(cuts[:n]), [s for s in starts[1:] if s not in size_cut], len(pev)


@pytest.mark.parametrize("plen", PC.LENS)
@pytest.mark.parametrize("name", ["dynamic_mixed", "static_file_size", "small_max_compaction_bytes", "short_boundary_keys",
                                  "shared_boundaries_snapshots"])
def test_rules_cut_where_the_oracle_does_with_grandparents(sim, name, plen):
    p, inputs = gp_cases.build(**gp_cases.CASES[name])
    p.sst_partitioner_prefix_len = plen
    files, _, _ = PC.oracle_compact(p, inputs)
    got, want, nev = _run(sim, p, files)
    assert got == want
    assert nev > 0 or plen < 15  # (the first bytes of these keys take few values)


@pytest.mark.parametrize("seed", range(12))
def test_rules_cut_where_the_oracle_does_on_random_streams(sim, seed):
    """random event positions, runs of consecutive events, events on and next to size cuts, with and without grandparents"""
    rnd = random.Random(seed)
    n = rnd.choice([500, 3000, 9000])
    events = set()
    while len(events) < rnd.randint(1, 60):
        e = rnd.randrange(1, n)
        events.update(range(e, min(n, e + rnd.choice([1, 1, 2, 5]))))
    p, inputs = PC.stream_job(n, events, vlen=rnd.choice([8, 60, 300]), seed=seed,
                              max_output_file_size=rnd.choice([3000, 20000, 64 << 20]))
    if seed % 3 == 0:
        keys = PC.stream_keys(n, events)
        picks = sorted(rnd.sample(range(n), 8))
        p.grandparents = [(keys[picks[i]], keys[picks[i + 1]], rnd.choice([4000, 40000])) for i in range(0, 8, 2)]
        p.level_compaction_dynamic_file_size = seed % 2 == 0
        p.bottommost_level = False
    files, _, _ = PC.oracle_compact(p, inputs)
    got, want, nev = _run(sim, p, files)
    assert got == want and nev == len(events)


@pytest.mark.parametrize("plen", PC.LENS)
@pytest.mark.parametrize("case", ["basic", "drops_at_prefix_changes", "grandparents", "grandparents_static", "size_meets_partition",
                                  "output_level0"])
def test_rules_cut_where_the_reference_does(sim, case, plen):
    if not PC.have_ref():
        pytest.skip("oracle/_ref/ref_compact_partition not built (needs /root/reference)")
    ops, opts = PC.SCENARIOS[case]()
    ref = PC.run_reference(ops, plen, **opts)
    p = PC.params_from_reference(ref, plen)
    got, want, _ = _run(sim, p, ref["outputs"])
    assert got == want
