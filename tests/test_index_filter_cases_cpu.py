"""The index and filter jobs (tests/index_filter_cases.py) reach the edges they are named for: proved from the oracle's output files
without a GPU.  Separators are classified by a Python FindShortestSeparator that must reproduce every index key the oracle wrote;
the kernel conditions restated here are read out of csrc/encode.cu and csrc/common.cuh, so a change to them fails this file rather
than silently moving a case off its edge."""
import collections
import functools
import os
import struct

import pytest

import helpers as H
import index_filter_cases as C
import sstfmt

ENCODE = open(os.path.join(C.plan_cases._CSRC, "encode.cu")).read()
COMMON = open(os.path.join(C.plan_cases._CSRC, "common.cuh")).read()
assert "if (d < nul - 1 || (uint32_t)s[d] + 1 < (uint32_t)l[d]) {" in ENCODE
assert "sep = KeyRec{hi, lo, (kMaxSeq << 8) | 0x16, tn, 1};" in ENCODE
assert "p = first_nonzero_byte(~hi & a.x & ~b.x, ~lo & a.y & ~b.y);" in ENCODE and "if (p == 16) return false;  // all 0xff" in ENCODE
assert "const uint64_t nb_blocks = (len - 1) / 1024;" in COMMON and "for (; n + 8 <= nb_blocks; n += 8) {" in COMMON
assert "if (len <= 240) return xxh3_64_short(in, (uint32_t)len);" in COMMON
SEEK_TRAILER = struct.pack("<Q", (H.MAX_SEQ << 8) | 0x16)  # kMaxSequenceNumber, kValueTypeForSeek


@functools.lru_cache(maxsize=None)
def _job(name):
    p, inputs = C.build(name)
    files, metas, st = H.oracle_compact(p, inputs)
    return p, files, metas, [C.table_layout(f) for f in files]


def _varint_len(v):
    n = 1
    while v >= 128:
        v >>= 7
        n += 1
    return n


def separator_census(files, lays):
    """(branches Counter, [(file has sequence numbers in its index, shortened separators in it)]).  Asserts that the Python
    FindShortestSeparator yields exactly the index key the oracle wrote for every block."""
    branches, per_file = collections.Counter(), []
    for data, lay in zip(files, lays):
        edges = []
        for _, h in lay["index"]:
            ents = sstfmt.block_entries(sstfmt.read_block(data, h)[0])
            edges.append((ents[0][0], ents[-1][0]))
        want, has_seq, shortened = [], False, 0
        for b, (_, last) in enumerate(edges):
            if b + 1 == len(edges):
                want.append(last)
                continue
            nxt = edges[b + 1][0]
            if last[:-8] == nxt[:-8]:
                has_seq = True
                branches["equal"] += 1
                want.append(last)
                continue
            sep, branch = C.shortest_separator(last[:-8], nxt[:-8])
            branches[branch] += 1
            if sep != last[:-8]:
                shortened += 1
                want.append(sep + SEEK_TRAILER)
            else:
                want.append(last)
        got = [k for k, _ in lay["index"]]
        want = [k if has_seq else k[:-8] for k in want]
        assert got == want, f"index keys differ from FindShortestSeparator: {[(g.hex(), w.hex()) for g, w in zip(got, want) if g != w][:3]}"
        per_file.append((has_seq, shortened))
    return branches, per_file


SEP_BRANCHES = ({"empty", "prefix", "equal", "before_last@0", "before_last@7", "before_last@8", "last_byte@7", "last_byte@15", "ff_tail0"}
                | {f"ff_run{r}" for r in range(15)} | {f"ff_tail{r}" for r in range(1, 16)})


@pytest.mark.parametrize("name", [n for n in C.CASES if n.startswith("sep_")])
def test_separator_cases_reach_every_branch(name):
    p, files, metas, lays = _job(name)
    branches, per_file = separator_census(files, lays)
    print(f"{name}: {len(files)} files, boundaries per branch {dict(sorted(branches.items()))}, (has seq, shortened) per file {per_file}")
    assert all(len(lay["index"]) == m.num_data_blocks for lay, m in zip(lays, metas))
    missing = SEP_BRANCHES - set(branches)
    assert not missing, f"branches not reached: {sorted(missing)}"
    seq = [s for s, _ in per_file]
    assert any(seq) and not all(seq), "no file with and one without sequence numbers in its index"
    assert any(a != b for a, b in zip(seq, seq[1:])), "files with and without sequence numbers are not neighbours"
    assert any(s and n for s, n in per_file), "no shortened separator (kMaxSequenceNumber) in a file that keeps sequence numbers"


@pytest.mark.parametrize("name", C.SLOW)
def test_handles_cross_every_varint_width(name):
    """SLOW: about 400 MB of values"""
    p, files, metas, lays = _job(name)
    assert len(files) == 1
    off_w = collections.Counter(_varint_len(h[0]) for _, h in lays[0]["index"])
    size_w = collections.Counter(_varint_len(h[1]) for _, h in lays[0]["index"])
    print(f"{name}: offset varint widths {dict(sorted(off_w.items()))}, size varint widths {dict(sorted(size_w.items()))}")
    assert set(off_w) == {1, 2, 3, 4, 5} and set(size_w) == {1, 2, 3, 4}


def _xxh3_shape(n):
    """(full 1024-byte blocks summed by file_block_contrib_kernel, passes of the eight-block fold, stripes of the last block)"""
    if n <= 240:
        return "short"
    nb = (n - 1) // 1024
    return nb, nb // 8, ((n - 1) - 1024 * nb) // 64


@pytest.mark.parametrize("name", [n for n in C.CASES if n.startswith("index_len_")])
def test_index_blocks_have_the_exact_lengths(name):
    p, files, metas, lays = _job(name)
    lens = [C.index_block_len(f) for f in files]
    print(f"{name}: index block lengths {lens}, XXH3 shapes {[_xxh3_shape(n) for n in lens]}, blocks {[m.num_data_blocks for m in metas]}")
    assert tuple(lens) == C.CASES[name]["lengths"]


def _filters(files, lays):
    return [C.filter_block(f, lay) for f, lay in zip(files, lays)]


def _slices(bits):
    return -(-bits // C.SLICE)


@pytest.mark.parametrize("name", [n for n in C.CASES if n.startswith("filter_")])
def test_filter_cases(name):
    p, files, metas, lays = _job(name)
    fb = _filters(files, lays)
    assert all(fb), "a file without a filter block"
    slices = [_slices(b) for _, b, _ in fb]
    phases = sorted({o % 16 for o, _, _ in fb})
    probes = sorted({k for _, _, k in fb})
    entries = [sstfmt.prop_u64(lay["properties"], "rocksdb.num.entries") for lay in lays]
    fentries = [sstfmt.prop_u64(lay["properties"], "rocksdb.num.filter_entries") for lay in lays]
    starts_inside = sum(1 for a, b in zip(metas, metas[1:]) if bytes(a.largest[:a.largest_len - 8]) == bytes(b.smallest[:b.smallest_len - 8]))
    print(f"{name}: {len(files)} files, filter bits {[b for _, b, _ in fb][:12]}, slices per file {slices[:12]}, phases {len(phases)} of 16, "
          f"probes {probes}, entries {sum(entries)}, filter entries {sum(fentries)}, files starting inside a key's versions {starts_inside}")
    assert probes == [C.num_probes(p.bloom_millibits_per_key)]
    bits = [b for _, b, _ in fb]
    if name == "filter_slice1":
        assert bits == [C.SLICE]
    elif name == "filter_slice1_64":
        assert bits == [C.SLICE + 64]
    elif name == "filter_slice2":
        assert bits == [2 * C.SLICE]
    elif name == "filter_slice8":
        assert len(files) == 1 and slices[0] >= 7 and bits[0] % C.SLICE
    elif name == "filter_slices_per_file":
        assert len(set(slices)) >= 2 and max(slices) >= 7 and min(slices) == 1
    elif name == "filter_phases":
        assert len(phases) == 16, phases
    elif name.startswith("filter_len_64x"):
        m = int(name.rsplit("x", 1)[1])
        assert bits == [64 * m] and files[0][fb[0][0] + 64 * m + 5] == 0  # filter block of 64 m + 5 bytes, then its trailer
    elif name.startswith("filter_probes_"):
        mb = int(name.rsplit("_", 1)[1])
        assert mb == p.bloom_millibits_per_key and (C.num_probes(mb) != C.num_probes(mb + 1) or C.num_probes(mb) != C.num_probes(mb - 1))
    elif name == "filter_key_lengths":
        ents, _ = C._filter_data(*C.CASES[name]["data"])
        lens = collections.Counter(len(k) - 8 for k, _ in ents)
        print(f"user keys per length {dict(sorted(lens.items()))}")
        assert len(files) == 1 and set(lens) == set(range(17)) and slices[0] >= 2
    elif name == "filter_hot_keys":
        assert len(files) == 1 and slices[0] >= 2 and entries[0] - fentries[0] >= 50 * 29
    elif name == "filter_cut_in_versions":
        assert starts_inside >= 1 and sum(entries) > sum(fentries)
    else:
        raise KeyError(name)


def test_probe_thresholds_change_the_probe_count():
    got = {}
    for lim in C.PROBE_LIMITS:
        got[lim] = tuple(C.filter_block(f)[2] for mb in (lim, lim + 1) for f in _job(f"filter_probes_{mb}")[1])
    print(f"probes at each threshold and one past it: {got}")
    assert all(a != b for a, b in got.values())


@pytest.mark.parametrize("name", ["files_max", "files_max_filter", "files_over"])
def test_file_count_cases(name):
    p, files, metas, lays = _job(name)
    print(f"{name}: {len(files)} files (kMaxOutFiles {C.MAX_FILES}), entries per file {sorted({m.num_entries for m in metas})}")
    assert len(files) == C.CASES[name]["nfiles"]
    assert all(bool(C.filter_block(f, lay)) == bool(p.bloom_millibits_per_key) for f, lay in zip(files[:50], lays))


# ---------------------------------------------------------------------------------------------------- the reference writes the same
def _ref_or_skip():
    if not H.have_ref():
        pytest.skip("oracle/_ref missing")


@pytest.mark.ref
@pytest.mark.parametrize("name", ["sep_v3_crc32c", "sep_v5_xxh3"])
def test_reference_writes_the_separator_keys_as_the_oracle_does(name):
    _ref_or_skip()
    p, _ = C.build(name)
    ents, snaps = C._separator_data()
    ops = H.Ops()
    by_seq = sorted(ents, key=lambda e: struct.unpack("<Q", e[0][-8:])[0])
    for ik, v in by_seq:  # the DB assigns sequence numbers in write order: the hot key's snapshots fall between its versions
        ops.put(ik[:-8], v)
        if struct.unpack("<Q", ik[-8:])[0] >> 8 in snaps:
            ops.snapshot()
    ops.flush()
    ref = H.run_reference(ops, block_size=64, restart_interval=1, format_version=p.format_version, checksum=p.checksum,
                          target_file_size=p.max_output_file_size)
    q = H.params_from_reference(ref)
    files, _, _ = H.oracle_compact(q, ref["inputs"])
    assert len(ref["outputs"]) >= 3 and files == ref["outputs"]
    lays = [C.table_layout(f) for f in files]
    branches, per_file = separator_census(files, lays)
    print(f"reference: {len(files)} files, branches {dict(sorted(branches.items()))}, per file {per_file}")
    assert SEP_BRANCHES - {"equal"} <= set(branches)


@pytest.mark.ref
def test_reference_writes_a_two_slice_filter_as_the_oracle_does():
    _ref_or_skip()
    ents, _ = C._filter_data(*C.CASES["filter_slice2"]["data"])
    ops = H.Ops()
    for ik, v in ents:
        ops.put(ik[:-8], v)
    ops.flush()
    ref = H.run_reference(ops, bloom_bits=50)
    q = H.params_from_reference(ref)
    files, _, _ = H.oracle_compact(q, ref["inputs"])
    assert files == ref["outputs"]
    fb = [C.filter_block(f) for f in files]
    print(f"reference: filter bits {[b for _, b, _ in fb]}, probes {[k for _, _, k in fb]}")
    assert [b for _, b, _ in fb] == [2 * C.SLICE]
