"""The merge cases (merge_cases.py; their edges are proven by test_merge_cases_cpu.py) on the device, through the C ABI:
 (a) stage level: run(until=2), then the merged records and values against the oracle's compaction iterator entry by entry, and the
     stage's statistics -- a failure names the first entry that differs, so it points at the merge kernels and at a key;
 (b) job level on the same inputs: every output file byte for byte against the oracle, all statistics and the per-file metadata.  This
     is what sees merge_sizes_fix_kernel (a wrong encoded size or shared-prefix length for a tile's first survivor corrupts the block)
     and the tile statistics that end up in the properties block; 64 KiB files and, in one parametrisation, 512-byte blocks make a hot
     key's neighbourhood span many of both;
 (c) hot keys with device-resident inputs (value references then point into caller memory) and as key-range sub-jobs whose boundaries
     are hot user keys, so that a run is clipped next to thousands of versions of the boundary key.
Every job runs once."""
import collections
import copy

import pytest

try:  # a fresh box can take minutes to page torch in: do it at collection time, outside any per-test timeout
    import torch  # noqa: F401
except Exception:  # pragma: no cover
    torch = None

import helpers as H
import merge_cases as M

pytestmark = pytest.mark.gpu

SMALL_BLOCKS = ["hot_keys", "tombstone_tails", "filtered_heads_empty_value", "filtered_heads_ttl", "prefix_ties", "fan_in_17"]


def _assert_job(files, metas, st, want, wmetas, wst, label):
    assert [len(f) for f in files] == [len(f) for f in want], label
    for i, (a, b) in enumerate(zip(files, want)):
        assert a == b, f"{label}: output {i} differs at byte {next(j for j in range(len(a)) if a[j] != b[j])}"
    for k in H.STAT_KEYS + ("num_record_drop_user",):
        assert getattr(st, k) == getattr(wst, k), (label, k)
    for i, (m, om) in enumerate(zip(metas, wmetas)):
        assert (m.file_size, m.num_entries, m.num_deletions, m.raw_key_size, m.raw_value_size, m.num_data_blocks, m.smallest_seqno,
                m.largest_seqno) == (om.file_size, om.num_entries, om.num_deletions, om.raw_key_size, om.raw_value_size, om.num_data_blocks,
                                     om.smallest_seqno, om.largest_seqno), (label, i)
        assert bytes(m.smallest_ikey[:m.smallest_ikey_len]) == bytes(om.smallest[:om.smallest_len]), (label, i)
        assert bytes(m.largest_ikey[:m.largest_ikey_len]) == bytes(om.largest[:om.largest_len]), (label, i)


@pytest.mark.parametrize("name", sorted(M.CASES))
def test_merge_stage_matches_oracle_on_merge_cases(name):
    from gpu_harness import assert_merged_matches, job_from_params
    e = M.expected(name)
    job = job_from_params(e["params"])
    for i, d in enumerate(e["inputs"]):
        job.add_input(d, file_number=i)
    job.run(until=2)
    assert_merged_matches(job, e["records"], name)
    st = job.stats()
    for k in M.STAGE_STAT_KEYS:
        assert getattr(st, k) == getattr(e["stage_stats"], k), (name, k)
    assert st.num_input_records == len(e["order"])
    job.close()


@pytest.mark.parametrize("name", sorted(M.CASES))
def test_job_matches_oracle_on_merge_cases(name):
    from gpu_harness import run_product
    e = M.expected(name)
    files, metas, st = run_product(e["params"], e["inputs"])
    _assert_job(files, metas, st, e["files"], e["metas"], e["stats"], name)
    if e["params"].compaction_filter != "none":
        assert st.num_record_drop_user > 0


@pytest.mark.parametrize("name", SMALL_BLOCKS)
def test_job_matches_oracle_on_merge_cases_with_small_blocks(name):
    """512-byte blocks: a tile's first survivor is far more often the first entry of a block or the entry behind a restart point"""
    from gpu_harness import run_product
    e = M.expected(name)
    p = copy.copy(e["params"])
    p.block_size, p.block_restart_interval = 512, 4
    want, wmetas, wst = H.oracle_compact(p, e["inputs"])
    files, metas, st = run_product(p, e["inputs"])
    _assert_job(files, metas, st, want, wmetas, wst, name)


@pytest.mark.parametrize("name", ["hot_keys", "filtered_heads_ttl"])
def test_device_resident_inputs_on_merge_cases(name):
    """the TTL filter reads the stamp through the value reference, which points into the caller's device memory here"""
    from gpu_harness import run_product
    e = M.expected(name)
    files, metas, st = run_product(e["params"], e["inputs"], device_inputs=True)
    _assert_job(files, metas, st, e["files"], e["metas"], e["stats"], name)


def test_hot_keys_as_sub_jobs_cut_at_hot_user_keys():
    from gpu_harness import job_from_params
    e = M.expected("hot_keys")
    p = e["params"]
    hot = sorted(uk for uk, c in collections.Counter(uk for uk, *_ in e["order"]).items() if c >= min(M.HOT_VERSIONS))
    assert len(hot) == len(M.HOT_VERSIONS)
    parent = job_from_params(p)
    for i, d in enumerate(e["inputs"]):
        parent.add_input(d, level=0, file_number=i)
    planned = parent.plan_ranges(4, min_range_bytes=16 << 10)
    # the planner's own boundaries and the hot keys: a range that starts at a hot key owns all its versions, the one in front none
    bounds = sorted(set(planned) | set(hot))
    ranges = list(zip([None] + bounds, bounds + [None]))
    subs = [parent.sub_job(range_start=a, range_end=b, first_file_number=1000 * (i + 1)) for i, (a, b) in enumerate(ranges)]
    total_in = total_out = 0
    for i, ((a, b), j) in enumerate(zip(ranges, subs)):
        j.run()
        q = copy.copy(p)
        q.range_start, q.range_end, q.first_file_number = a, b, 1000 * (i + 1)
        want, wmetas, wst = H.oracle_compact(q, e["inputs"])
        st = j.stats()
        _assert_job(j.outputs(), [j.output_meta(x) for x in range(j.output_count())], st, want, wmetas, wst, ("hot_keys", a, b))
        total_in += st.num_input_records
        total_out += st.num_output_records
    assert (total_in, total_out) == (e["stats"].num_input_records, e["stats"].num_output_records)  # the ranges partition the job
    for j in subs:
        j.close()
    parent.close()
