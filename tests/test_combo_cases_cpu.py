"""The jobs of combo_cases.py reach what they claim, without a GPU: the covering array holds every allowed pair of factor levels, and in
every job each optional part changes something -- shown from the checker's outputs, sstfmt and the job rebuilt without that part.
Then the combined checker against the live reference on the combinations the reference driver can express."""
import collections
import functools

import pytest

import combo_cases as C
import decode_cases as D
import helpers as H
import partition_cases as PC
import sstfmt


def _skip_without_reference(name):
    if C.needs_reference(name) and not H.have_ref():
        pytest.skip("oracle/_ref not built (needs /root/reference)")


def test_pairwise_coverage():
    allowed = C.all_pairs()
    covered = set().union(*(C.row_pairs(r) for r in C.rows()))
    for a, b, why in C.EXCLUDED:
        print(f"excluded: {a[0]}={a[1]} with {b[0]}={b[1]}: {why}")
        assert not any(r[a[0]] == a[1] and r[b[0]] == b[1] for r in C.rows())
    print(f"pairwise coverage: {len(allowed & covered)} of {len(allowed)} allowed pairs in {len(C.rows())} jobs")
    assert allowed <= covered
    kept = [r for r in C.rows() if r["output_level"] == 0 and (r["prefix_len"] or r["grandparents"] != "none")]
    assert kept, "output level 0 with a partitioner or grandparents must stay in the array"


def _user_keys(files):
    return [ik[:-8] for f in files for ik, _ in sstfmt.parse_sst(f)["entries"]]


def _in_range(k, p):
    return (p.range_start is None or k >= p.range_start) and (p.range_end is None or k < p.range_end)


@functools.lru_cache(maxsize=None)
def census(name):
    """per factor the count that shows it acting in this job; None where the level is off or cannot act (output level 0 ignores the
    partitioner and the cuts; a 16-byte partitioner already starts a file at every user key, leaving a grandparent nothing to cut)"""
    e = C.expected(name)
    row, p, inputs = e["row"], e["params"], e["inputs"]
    out = {}
    outs = {ik for f in e["files"] for ik, _ in sstfmt.parse_sst(f)["entries"]}
    tables = [sstfmt.parse_sst(d) for d in inputs]
    in_entries = [ik for t in tables for ik, _ in t["entries"]]
    out["filter"] = e["stats"].num_record_drop_user if row["filter"] != "none" else None
    if row["snapshots"]:  # versions per user key beyond those of the job without snapshots (sequence numbers may be zeroed either way)
        with_ = collections.Counter(_user_keys(e["files"]))
        without = collections.Counter(_user_keys(C.variant(name, snapshots=[])[0]))
        out["snapshots"] = sum(max(0, n - without[k]) for k, n in with_.items())
    else:
        out["snapshots"] = None
    if row["single_delete"]:
        sds = [ik for ik in in_entries if ik[-8] == C.SINGLE_DELETION and _in_range(ik[:-8], p)]
        out["single_delete"] = sum(1 for ik in sds if ik not in outs)
    else:
        out["single_delete"] = None
    starts = {sstfmt.parse_sst(f)["entries"][0][0] for f in e["files"][1:]}
    if row["grandparents"] != "none" and row["output_level"] == 1 and row["prefix_len"] != 16:
        other = {sstfmt.parse_sst(f)["entries"][0][0] for f in C.variant(name, grandparents=[])[0][1:]}
        out["grandparents"] = len(starts - other)
    else:
        out["grandparents"] = None
    if row["prefix_len"] and row["output_level"] == 1:
        out["partition"] = len(PC.prefix_events(_user_keys(e["files"]), row["prefix_len"]))
    else:
        out["partition"] = None
    kept = [D.kept_blocks(d, p.range_start, p.range_end) for d in inputs]
    blocks = [D.table_blocks(d) for d in inputs]
    ukeys = [ik[:-8] for ik in in_entries]

    def skipped(start, end):
        return sum(len(b) - len(D.kept_blocks(d, start, end)) for b, d in zip(blocks, inputs))
    # per bounded side: entries clipped, data blocks skipped
    out["range_start"] = (sum(1 for k in ukeys if k < p.range_start), skipped(p.range_start, None)) if p.range_start is not None else None
    out["range_end"] = (sum(1 for k in ukeys if k >= p.range_end), skipped(None, p.range_end)) if p.range_end is not None else None
    if row["inputs"] == "zlib":
        comp_kept = sum(1 for b, k in zip(blocks, kept) for j in k if b[j]["ctype"] == 2)
        comp_skipped = sum(1 for b, k in zip(blocks, kept) for j, x in enumerate(b) if x["ctype"] == 2 and j not in k)
        out["zlib"] = (comp_kept, comp_skipped) if row["range"] != "none" else (comp_kept,)
    else:
        out["zlib"] = None
    out["bloom"] = sum(1 for f in e["files"] if "fullfilter.rocksdb.BuiltinBloomFilter" in sstfmt.parse_sst(f)["metaindex"]) \
        if row["bloom"] else None
    out["level_files"] = sum(1 for lv in e["levels"] if lv) if row["runs"] == "l0+level" else None
    return out


@pytest.mark.parametrize("name", C.names() + [C.REFUSAL_TWIN])
def test_engagement_census(name):
    _skip_without_reference(name)
    e = C.expected(name)
    row, st = e["row"], e["stats"]
    c = census(name)
    shown = ", ".join(f"{k}={v}" for k, v in c.items() if v is not None)
    print(f"{name}: {st.num_input_records} entries in, {st.num_output_records} out, {len(e['files'])} files; {shown}")
    for k, v in c.items():
        if v is not None:
            assert min(v if isinstance(v, tuple) else (v,)) >= 1, (k, v)
    if row["bloom"]:
        assert c["bloom"] == len(e["files"])  # every file has its filter block
    # sizes: two merge tiles inside any range; at least two files at output level 1
    assert st.num_input_records > C.MERGE_TILE
    if row["output_level"] == 1:
        assert len(e["files"]) >= 2
    # the hot key's versions span data blocks of the run that holds them: that run's index keeps sequence numbers
    assert any(not D.index_info(d)["user_key"] for d in e["inputs"])


@pytest.mark.parametrize("name", sorted(C.BIG))
def test_big_jobs_cut_on_both_sides_of_a_stitch_group_boundary(name):
    """the output inside the range spans more than one stitch group (kEncTile * kEncGroupTiles entries), and partition or grandparent
    cuts fall inside the groups on both sides of a group boundary"""
    e = C.expected(name)
    ukeys = _user_keys(e["files"])
    n = len(ukeys)
    starts, k = [], 0
    for f in e["files"]:
        starts.append(k)
        k += len(sstfmt.parse_sst(f)["entries"])
    no_gp = {sstfmt.parse_sst(f)["entries"][0][0] for f in C.variant(name, grandparents=[])[0]}
    first = [sstfmt.parse_sst(f)["entries"][0][0] for f in e["files"]]
    gp_cuts = {s for s, ik in zip(starts[1:], first[1:]) if ik not in no_gp}
    part = set(PC.prefix_events(ukeys, 2))
    cuts = sorted(gp_cuts | part)
    G = C.STITCH_GROUP
    both = [b for b in range(G, n, G) if any(b - G <= c < b for c in cuts) and any(b <= c < b + G for c in cuts)]
    print(f"{name}: {n} output entries, {len(part)} partition and {len(gp_cuts)} grandparent cuts; group boundaries cut on both "
          f"sides: {both}")
    assert n > G and both and gp_cuts and part


def test_census_totals():
    """every factor acts in at least one job (the per-job test asserts each job; this prints the totals)"""
    tot = collections.Counter()
    for n in C.names():
        if C.needs_reference(n) and not H.have_ref():
            continue
        for k, v in census(n).items():
            if v is not None:
                tot[k] += 1
    print("jobs in which each part acts: " + ", ".join(f"{k} {v}" for k, v in sorted(tot.items())))
    assert set(tot) == {"filter", "snapshots", "single_delete", "grandparents", "partition", "range_start", "range_end", "bloom",
                        "level_files"} | ({"zlib"} if H.have_ref() else set())
    print(f"{len(C.rows())} jobs of the covering array, {len(C.BIG)} jobs over a stitch group")


# ------------------------------------------------------------------------------------------------ against the live reference
needs_part_ref = pytest.mark.skipif(not PC.have_ref(), reason="oracle/_ref/ref_compact_partition not built (needs /root/reference)")


def _meta(m):
    return (m.file_size, m.num_entries, m.num_deletions, m.num_data_blocks, bytes(m.smallest[:m.smallest_len]), bytes(m.largest[:m.largest_len]))


def _ref_meta(data):
    t = sstfmt.parse_sst(data)
    pr = t["properties"]
    return (len(data), sstfmt.prop_u64(pr, "rocksdb.num.entries"), sstfmt.prop_u64(pr, "rocksdb.deleted.keys"),
            sstfmt.prop_u64(pr, "rocksdb.num.data.blocks"), t["entries"][0][0], t["entries"][-1][0])


@needs_part_ref
@pytest.mark.parametrize("name", sorted(C.REF_COMBOS))
def test_checker_matches_the_reference_on_combinations(name):
    ops, opts, plen = C.ref_combo(name)
    ref = PC.run_reference(ops, plen, **opts)
    man = ref["manifest"]
    if opts.get("max_subcompactions", 1) > 1:
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
                assert sstfmt.parse_sst(got)["entries"] == sstfmt.parse_sst(exp)["entries"]
                io, isz = sstfmt.parse_sst(got)["footer"]["index"]
                assert got[:io + isz + 5] == exp[:io + isz + 5]  # data, filter and index blocks
            for key in ("num_input_deletion_records", "num_expired_deletion_records", "num_records_replaced",
                        "total_input_raw_key_bytes", "total_input_raw_value_bytes"):
                assert getattr(st, key) == rstats[key], key
            k += nfiles
        assert k == len(ref["outputs"])
        print(f"{name}: {len(ranges)} sub-compactions, {k} files agree")
        return
    p = PC.params_from_reference(ref, plen)
    files, metas, st = PC.oracle_compact(p, ref["inputs"])
    assert [len(f) for f in files] == [len(f) for f in ref["outputs"]]
    assert files == ref["outputs"]
    assert [_meta(m) for m in metas] == [_ref_meta(o) for o in ref["outputs"]]
    for key in H.STAT_KEYS:
        assert getattr(st, key) == man["stats"][key], key
    if "grandparents" in opts or opts.get("mode") == "range":
        assert len(man["grandparents"]) >= 2
    print(f"{name}: {len(files)} files, {st.num_output_records} entries agree; {len(man['snapshots'])} snapshots, "
          f"{len(man.get('grandparents', []))} grandparents")
