"""The fixed-prefix SST partitioner (SstPartitionerFixedPrefixFactory, db/compaction/sst_partitioner.cc, checked by
CompactionOutputs::ShouldStopBefore in front of the size and grandparent rules, compaction_outputs.cc:231-300) restated in the CPU
oracle (partition_cases.oracle_compact) and pinned against the compiled reference: files, FileMetaData and statistics byte-exact for every prefix length in
partition_cases.LENS.  Host-compiled device rules: tests/test_partition_rules_host.py; device: tests/test_gpu_partitioner.py."""
import pytest

import helpers as H
import partition_cases as PC
import sstfmt

needs_ref = pytest.mark.skipif(not PC.have_ref(), reason="oracle/_ref/ref_compact_partition not built (needs /root/reference)")
SUB_STATS = ("num_input_deletion_records", "num_expired_deletion_records", "num_records_replaced", "total_input_raw_key_bytes",
             "total_input_raw_value_bytes")


def _ukeys(files):
    return [ik[:-8] for f in files for ik, _ in sstfmt.parse_sst(f)["entries"]]


def _file_starts(files):
    starts, k = [], 0
    for f in files:
        starts.append(k)
        k += len(sstfmt.parse_sst(f)["entries"])
    return starts


def _meta_tuple(m):
    return (m.file_size, m.smallest_seqno, m.largest_seqno, m.num_entries, m.num_deletions, m.raw_key_size, m.raw_value_size,
            m.num_data_blocks, bytes(m.smallest[:m.smallest_len]), bytes(m.largest[:m.largest_len]))


def _ref_meta_tuple(data):
    t = sstfmt.parse_sst(data)
    pr = t["properties"]
    ents = t["entries"]
    seqs = [int.from_bytes(ik[-8:], "little") >> 8 for ik, _ in ents]
    return (len(data), min(seqs), max(seqs), sstfmt.prop_u64(pr, "rocksdb.num.entries"), sstfmt.prop_u64(pr, "rocksdb.deleted.keys"),
            sstfmt.prop_u64(pr, "rocksdb.raw.key.size"), sstfmt.prop_u64(pr, "rocksdb.raw.value.size"),
            sstfmt.prop_u64(pr, "rocksdb.num.data.blocks"), ents[0][0], ents[-1][0])


@needs_ref
@pytest.mark.parametrize("plen", PC.LENS)
@pytest.mark.parametrize("case", [c for c in PC.SCENARIOS if c != "subcompactions"])
def test_oracle_partitions_files_where_the_reference_does(case, plen):
    ops, opts = PC.SCENARIOS[case]()
    ref = PC.run_reference(ops, plen, **opts)
    man = ref["manifest"]
    p = PC.params_from_reference(ref, plen)
    files, metas, st = PC.oracle_compact(p, ref["inputs"])
    assert [len(f) for f in files] == [len(f) for f in ref["outputs"]]
    assert files == ref["outputs"]
    assert [_meta_tuple(m) for m in metas] == [_ref_meta_tuple(o) for o in ref["outputs"]]
    for k in H.STAT_KEYS:
        assert getattr(st, k) == man["stats"][k], k
    # every partition event of the output stream starts a file; L0 outputs are never partitioned
    ukeys = _ukeys(files)
    events = set(PC.prefix_events(ukeys, plen))
    starts = set(_file_starts(files))
    if man["output_level"] == 0:
        assert len(files) == 1 and events
    else:
        assert events <= starts and len(files) >= len(events) + 1
    if case == "grandparents" or case == "grandparents_static":
        assert len(man["grandparents"]) >= 2 and man["level_compaction_dynamic_file_size"] == (case == "grandparents")


@needs_ref
@pytest.mark.parametrize("plen", PC.LENS)
def test_oracle_partitions_each_subcompaction_like_the_reference(plen):
    """every sub-compaction has its own CompactionOutputs: its first entry starts a file whatever the key before the range was"""
    ops, opts = PC.subcompactions()
    ref = PC.run_reference(ops, plen, **opts)
    ranges = H.subcompaction_ranges(ref)
    assert len(ranges) >= 2, "the reference did not split this job"
    props = [sstfmt.parse_sst(o)["properties"] for o in ref["outputs"]]
    k = 0
    for start, end, rstats in ranges:
        p = PC.params_from_reference(ref, plen)
        p.range_start, p.range_end = start, end
        nfiles = len(PC.oracle_compact(p, ref["inputs"])[0])
        p.file_creation_times = [sstfmt.prop_u64(q, "rocksdb.file.creation.time") for q in props[k:k + nfiles]] or [0]
        files, _, st = PC.oracle_compact(p, ref["inputs"])
        want = ref["outputs"][k:k + nfiles]
        assert H.sizes_without_file_number(files) == H.sizes_without_file_number(want)
        for got, exp in zip(files, want):
            tg, te = sstfmt.parse_sst(got), sstfmt.parse_sst(exp)
            assert tg["entries"] == te["entries"]
            io, isz = tg["footer"]["index"]
            assert got[:io + isz + 5] == exp[:io + isz + 5]
        for key in SUB_STATS:
            assert getattr(st, key) == rstats[key], key
        k += nfiles
    assert k == len(ref["outputs"])


def test_oracle_partitioner_edges_without_the_reference():
    """short keys, the empty key and len 0 on a hand-made stream: "ab" vs "abc" cuts at len 3, not at len 2; len 0 never cuts"""
    keys = [b"", b"a", b"ab", b"abc", b"abd", b"b"]
    kv = [(H.ikey(k, 10 + i), b"v") for i, k in enumerate(keys)]
    inp = H.oracle_build_sst(H.Params(), H.kvstream(kv))
    for plen, want in [(0, []), (1, [1, 5]), (2, [1, 2, 5]), (3, [1, 2, 3, 4, 5]), (17, [1, 2, 3, 4, 5])]:
        p = H.Params()
        p.sst_partitioner_prefix_len = plen
        files, _, _ = PC.oracle_compact(p, [inp])
        assert _file_starts(files)[1:] == want, plen
        assert PC.prefix_events(keys, plen) == want
        p.output_level = 0
        assert len(PC.oracle_compact(p, [inp])[0]) == 1
