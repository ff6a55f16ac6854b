"""The fixed-prefix SST partitioner on the device (GPU box).  partition_events_kernel lists the merged entries in front of which
SstPartitionerFixedPrefix::ShouldPartition (db/compaction/sst_partitioner.cc) cuts, and the encoder's stitch walk and block list
meet them as a second event source of gp_rules.h, in front of the size and grandparent rules (CompactionOutputs::ShouldStopBefore,
compaction_outputs.cc:231-300).  Checked byte for byte against
 (a) the unmodified reference on the jobs of partition_cases.SCENARIOS, for every prefix length in partition_cases.LENS;
 (b) the CPU oracle (pinned to the reference in test_oracle_partitioner.py) on synthetic streams whose events sit on the walk's edges:
     tile and stitch-group boundaries, a block's first and last entry, runs of consecutive events, size and grandparent cuts, the
     largest number of events the file records hold, key-range sub-jobs, host- and device-resident inputs;
 (c) the reference DB running its jobs through the B200 executor plugin with the partitioner set."""
import os
import random

import pytest

try:
    import torch  # noqa: F401
except Exception:  # pragma: no cover
    torch = None

import helpers as H
import partition_cases as PC
import sstfmt
import toplingdb_b200 as T

pytestmark = pytest.mark.gpu

KENC_TILE = 4096
KENC_GROUP = 16 * KENC_TILE
KMAX_OUT_FILES = 4096


def _first_diff(a, b):
    return next((j for j in range(min(len(a), len(b))) if a[j] != b[j]), min(len(a), len(b)))


def _same_files(got, want):
    assert [len(f) for f in got] == [len(f) for f in want]
    for i, (a, b) in enumerate(zip(got, want)):
        assert a == b, f"output {i} differs at byte {_first_diff(a, b)}"


def _blocks(files):
    """[(first entry, entries, file index)] of every data block, and the first entry of every file"""
    blocks, starts, k = [], [], 0
    for fi, data in enumerate(files):
        starts.append(k)
        t = sstfmt.parse_sst(data)
        for _, h in t["index"]:
            payload, _, _ = sstfmt.read_block(data, h)
            c = len(list(sstfmt.block_entries(payload)))
            blocks.append((k, c, fi))
            k += c
    return blocks, starts


def _check_stream(p, inputs, events, device_inputs=False):
    from gpu_harness import run_product
    want, wmetas, wst = PC.oracle_compact(p, inputs)
    _, starts = _blocks(want)
    assert set(events) <= set(starts), "an event does not start a file in the oracle's layout"
    files, metas, st = run_product(p, inputs, device_inputs=device_inputs, sst_partitioner_prefix_len=p.sst_partitioner_prefix_len)
    _same_files(files, want)
    for m, w in zip(metas, wmetas):
        assert (m.num_entries, m.num_deletions, m.raw_key_size, m.raw_value_size, m.num_data_blocks) == \
               (w.num_entries, w.num_deletions, w.raw_key_size, w.raw_value_size, w.num_data_blocks)
    for k in H.STAT_KEYS:
        assert getattr(st, k) == getattr(wst, k), k
    return want


# ---------------------------------------------------------------- (a) against the reference
@pytest.mark.parametrize("plen", PC.LENS)
@pytest.mark.parametrize("case", [c for c in PC.SCENARIOS if c != "subcompactions"])
def test_device_partitions_like_the_reference(case, plen):
    from gpu_harness import run_product
    if not PC.have_ref():
        pytest.fail("oracle/_ref/ref_compact_partition missing: run __graft_entry__.build() where /root/reference exists")
    ops, opts = PC.SCENARIOS[case]()
    ref = PC.run_reference(ops, plen, **opts)
    man = ref["manifest"]
    p = PC.params_from_reference(ref, plen)
    files, metas, st = run_product(p, ref["inputs"], sst_partitioner_prefix_len=plen)
    _same_files(files, ref["outputs"])
    for k in H.STAT_KEYS:
        assert getattr(st, k) == man["stats"][k], k
    for m, want in zip(metas, man["outputs"]):
        assert (m.file_size, m.num_entries, m.num_deletions) == (want["size"], want["num_entries"], want["num_deletions"])
        assert bytes(m.smallest_ikey[: m.smallest_ikey_len - 8]).hex() == want["smallestkey"]
        assert bytes(m.largest_ikey[: m.largest_ikey_len - 8]).hex() == want["largestkey"]


@pytest.mark.parametrize("plen", [1, 3, 16])
def test_sub_jobs_partition_each_key_range_like_the_reference(plen):
    """key-range sub-jobs (b200c_job_create_sub) over the reference's own sub-compaction ranges: each range starts fresh"""
    from gpu_harness import job_from_params
    if not PC.have_ref():
        pytest.fail("oracle/_ref/ref_compact_partition missing: run __graft_entry__.build() where /root/reference exists")
    ops, opts = PC.subcompactions()
    ref = PC.run_reference(ops, plen, **opts)
    ranges = H.subcompaction_ranges(ref)
    assert len(ranges) >= 2
    p = PC.params_from_reference(ref, plen)
    parent = job_from_params(p, sst_partitioner_prefix_len=plen)
    for i, data in enumerate(ref["inputs"]):
        parent.add_input(data, level=0, file_number=i)
    props = [sstfmt.parse_sst(o)["properties"] for o in ref["outputs"]]
    k = 0
    for start, end, _ in ranges:
        q = PC.params_from_reference(ref, plen)
        q.range_start, q.range_end, q.sst_partitioner_prefix_len = start, end, plen
        nfiles = len(PC.oracle_compact(q, ref["inputs"])[0])
        fct = [sstfmt.prop_u64(x, "rocksdb.file.creation.time") for x in props[k:k + nfiles]] or [0]
        sub = parent.sub_job(range_start=start, range_end=end, file_creation_times=fct)
        sub.run()
        got = sub.outputs()
        sub.close()
        want = ref["outputs"][k:k + nfiles]
        assert len(got) == len(want)
        for a, b in zip(got, want):  # concurrent sub-compactions number their files from one counter: compare all but the properties
            ta, tb = sstfmt.parse_sst(a), sstfmt.parse_sst(b)
            assert ta["entries"] == tb["entries"]
            io, isz = ta["footer"]["index"]
            assert a[:io + isz + 5] == b[:io + isz + 5]
        k += nfiles
    assert k == len(ref["outputs"])
    parent.close()


# ---------------------------------------------------------------- (b) synthetic streams against the oracle
@pytest.mark.parametrize("device_inputs", [False, True])
@pytest.mark.parametrize("fmax", [64 << 20, 300 << 10])
def test_events_on_and_next_to_tile_and_group_boundaries(device_inputs, fmax):
    n = KENC_GROUP + 3 * KENC_TILE
    events = set()
    for b in (KENC_TILE, 2 * KENC_TILE, 5 * KENC_TILE, KENC_GROUP, KENC_GROUP + KENC_TILE):
        events.update((b - 1, b, b + 1))
    events.update((KENC_GROUP - 2, KENC_GROUP + 2 * KENC_TILE))
    p, inputs = PC.stream_job(n, events, vlen=8, seed=1, max_output_file_size=fmax)
    _check_stream(p, inputs, sorted(events), device_inputs=device_inputs)


def test_events_on_the_first_and_last_entry_of_a_block():
    """each event is placed on the layout the earlier ones left: alternately on a block's first entry (the open block ends whole
    in front of it) and on its last entry (the block is cut short by one entry)"""
    n, events = 4000, []
    for j in range(10):
        p, inputs = PC.stream_job(n, events, vlen=60, seed=2)
        blocks, _ = _blocks(PC.oracle_compact(p, inputs)[0])
        last = events[-1] if events else 0
        b = [x for x in blocks if x[0] > last + 1][2]
        events.append(b[0] if j % 2 == 0 else b[0] + b[1] - 1)
    p, inputs = PC.stream_job(n, events, vlen=60, seed=2)
    _check_stream(p, inputs, events)


def test_consecutive_events_give_one_entry_files():
    events = list(range(100, 112)) + [777, 778] + list(range(KENC_TILE - 3, KENC_TILE + 3))
    p, inputs = PC.stream_job(6000, events, vlen=60, seed=3)
    want = _check_stream(p, inputs, events)
    assert sum(1 for f in want if len(sstfmt.parse_sst(f)["entries"]) == 1) >= 15


def test_events_where_the_size_rule_cuts():
    """an event on the entry behind the size cut (both rules ask for the same cut) and on the entry whose Add flushed the block that
    reached the limit (the partitioner is checked first: the file ends in front of that entry)"""
    n, fmax, events = 6000, 20000, []
    for j in range(8):
        p, inputs = PC.stream_job(n, events, vlen=60, seed=4, max_output_file_size=fmax)
        _, starts = _blocks(PC.oracle_compact(p, inputs)[0])
        last = events[-1] if events else 0
        s = [x for x in starts if x > last + 2 and x not in events][1]
        events.append(s if j % 2 == 0 else s - 1)
    p, inputs = PC.stream_job(n, events, vlen=60, seed=4, max_output_file_size=fmax)
    _check_stream(p, inputs, events)


def test_events_where_a_grandparent_rule_cuts():
    n, events = 12000, []
    rnd = random.Random(5)
    picks = sorted(rnd.sample(range(n), 24))

    def job(ev):
        p, inputs = PC.stream_job(n, ev, vlen=60, seed=5, target_output_file_size=40 << 10, max_output_file_size=80 << 10)
        ks = PC.stream_keys(n, ev)
        p.grandparents = [(ks[picks[i]], ks[picks[i + 1]], 30 << 10) for i in range(0, 24, 2)]
        p.bottommost_level = False
        return p, inputs

    for _ in range(5):
        p, inputs = job(events)
        blocks, starts = _blocks(PC.oracle_compact(p, inputs)[0])
        size = {blocks[i + 1][0] for i in range(len(blocks) - 1) if blocks[i + 1][2] != blocks[i][2] and blocks[i][1] == 1}
        last = events[-1] if events else 0
        gp = [s for s in starts if s > last and s not in events and s not in size]
        if not gp:
            break
        events.append(gp[0])
    assert len(events) >= 3, "the grandparent rules cut too rarely to place events on their cuts"
    p, inputs = job(events)
    _check_stream(p, inputs, events)


def test_the_most_events_the_file_records_hold():
    """k events give k + 1 files: kMaxOutFiles - 1 events fill the device's file records exactly, one more is refused before any
    file is written"""
    from gpu_harness import run_product
    n = 2 * KMAX_OUT_FILES
    events = list(range(2, n, 2))
    assert len(events) == KMAX_OUT_FILES - 1
    p, inputs = PC.stream_job(n, events, vlen=8, seed=6)
    want = _check_stream(p, inputs, events)
    assert len(want) == KMAX_OUT_FILES
    n += 2
    events = list(range(2, n, 2))
    assert len(events) == KMAX_OUT_FILES
    p, inputs = PC.stream_job(n, events, vlen=8, seed=6)
    with pytest.raises(T.B200cError) as ei:
        run_product(p, inputs, sst_partitioner_prefix_len=p.sst_partitioner_prefix_len)
    assert ei.value.code == T.native.ERR_NOT_SUPPORTED


def test_level0_output_and_zero_length_ignore_the_events():
    events = [10, 500, KENC_TILE]
    for level, plen in ((0, PC.PLEN), (1, 0)):
        p, inputs = PC.stream_job(9000, events, vlen=30, seed=7)
        p.output_level, p.sst_partitioner_prefix_len = level, plen
        want = _check_stream(p, inputs, [])
        assert len(want) == 1


@pytest.mark.parametrize("device_inputs", [False, True])
def test_sub_jobs_over_key_ranges_of_a_synthetic_stream(device_inputs):
    from gpu_harness import job_from_params
    n = 3 * KENC_TILE
    events = sorted(random.Random(8).sample(range(1, n), 300))
    p, inputs = PC.stream_job(n, events, vlen=40, seed=8, max_output_file_size=64 << 10)
    keys = PC.stream_keys(n, events)
    bounds = [None, keys[events[40]], keys[events[41] + 3], keys[KENC_TILE], None]
    parent = job_from_params(p, sst_partitioner_prefix_len=PC.PLEN)
    keep = []
    for i, data in enumerate(inputs):
        if device_inputs:
            t = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
            keep.append(t)
            parent.add_input(t, level=0, file_number=i)
        else:
            parent.add_input(data, level=0, file_number=i)
    for a, b in zip(bounds[:-1], bounds[1:]):
        p.range_start, p.range_end = a, b
        want, _, _ = PC.oracle_compact(p, inputs)
        sub = parent.sub_job(range_start=a, range_end=b)
        sub.run()
        got = sub.outputs()
        sub.close()
        _same_files(got, want)
    parent.close()


# ---------------------------------------------------------------- (c) the reference DB through the executor plugin
@pytest.mark.parametrize("case,plen", [("basic", 1), ("basic", 16), ("drops_at_prefix_changes", 3), ("grandparents", 8),
                                       ("size_meets_partition", 2), ("subcompactions", 3), ("bloom", 15)])
def test_reference_db_partitions_through_b200_executor(case, plen):
    if not (os.path.exists(PC.REF_PART_BIN) and os.path.exists(PC.REF_PART_B200_BIN)):
        pytest.fail("oracle/_ref/ref_compact_partition(_b200) missing: run __graft_entry__.build() where /root/reference exists")
    ops, opts = PC.SCENARIOS[case]()
    want = PC.run_reference(ops, plen, **opts)
    got = PC.run_reference(ops, plen, binary=PC.REF_PART_B200_BIN, executor="b200", **opts)
    gm, wm = got["manifest"], want["manifest"]
    assert gm["executor"] == "B200Compact" and wm["executor"] == "local"
    assert gm["remote_compact_read_bytes"] > 0, "compaction did not take the RunRemote/B200 branch"
    assert (gm["scan_count"], gm["scan_digest"]) == (wm["scan_count"], wm["scan_digest"])
    for data in got["outputs"]:  # the partitioner's promise: no output file spans two prefixes
        assert len({ik[:-8][:plen] for ik, _ in sstfmt.parse_sst(data)["entries"]}) == 1
    if opts.get("max_subcompactions", 1) > 1:
        # the executor splits the job at its own range boundaries (b200c_job_plan_ranges), not at GenSubcompactionBoundaries', and
        # every range starts a file: only the DB's contents and the entry count are the same
        assert sum(m["num_entries"] for m in gm["outputs"]) == sum(m["num_entries"] for m in wm["outputs"])
        return
    assert len(got["outputs"]) == len(want["outputs"])
    for k in ("smallest_seqno", "largest_seqno", "num_entries", "num_deletions", "smallestkey", "largestkey"):
        assert [m[k] for m in gm["outputs"]] == [m[k] for m in wm["outputs"]], k
    assert H.sizes_without_file_number(got["outputs"]) == H.sizes_without_file_number(want["outputs"])
    for g, w in zip(got["outputs"], want["outputs"]):
        tg, tw = sstfmt.parse_sst(g), sstfmt.parse_sst(w)
        assert tg["entries"] == tw["entries"]
        assert [g[h[0]:h[0] + h[1] + 5] for _, h in tg["index"]] == [w[h[0]:h[0] + h[1] + 5] for _, h in tw["index"]]
    for k in H.STAT_KEYS:
        assert gm["stats"][k] == wm["stats"][k], k
