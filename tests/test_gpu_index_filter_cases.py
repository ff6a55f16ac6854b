"""The index and filter jobs (tests/index_filter_cases.py) through the C ABI against the CPU oracle: output files, statistics and file
metadata, a failure naming the region of the first differing byte (gpu_harness.describe_first_difference); a subset with
device-resident inputs; a separator job and a two-slice filter through b200c_job_encode_kv (the B200TableBuilder path) against the
oracle's table builder; the launches the XXH3 checksums of the index and filter blocks add; exactly kMaxOutFiles output files, and
one more refused with ERR_NOT_SUPPORTED.  The handles_* jobs hold about
400 MB of values each and dominate the runtime."""
import copy

import pytest

import helpers as H
import index_filter_cases as C
import sstfmt

pytestmark = pytest.mark.gpu

JOBS = [n for n in C.CASES if n != "files_over"]
DEVICE_INPUTS = ["sep_v5_xxh3", "index_len_multi_crc32c", "filter_slice8", "filter_phases", "filter_cut_in_versions", "files_max_filter",
                 "handles_v5"]


def _same_files(name, files, want):
    from gpu_harness import describe_first_difference
    assert [len(f) for f in files] == [len(w) for w in want], f"{name}: file sizes differ"
    for i, (a, b) in enumerate(zip(files, want)):
        assert a == b, f"{name}: output {i} of {len(want)} differs at " + describe_first_difference(a, b)


def _check(name, device_inputs=False):
    from gpu_harness import run_product
    p, inputs = C.build(name)
    want, wmetas, wst = H.oracle_compact(p, inputs)
    files, metas, st = run_product(p, inputs, device_inputs=device_inputs)
    _same_files(name, files, want)
    for k in H.STAT_KEYS:
        assert getattr(st, k) == getattr(wst, k), k
    for m, om in zip(metas, wmetas):
        assert (m.file_size, m.num_entries, m.num_deletions, m.num_data_blocks, m.smallest_seqno, m.largest_seqno) == \
            (om.file_size, om.num_entries, om.num_deletions, om.num_data_blocks, om.smallest_seqno, om.largest_seqno)


@pytest.mark.parametrize("name", JOBS)
def test_job_matches_oracle_on_index_filter_cases(name):
    _check(name)


@pytest.mark.parametrize("name", DEVICE_INPUTS)
def test_device_resident_inputs(name):
    _check(name, device_inputs=True)


@pytest.mark.parametrize("name", ["sep_v4_crc32c", "filter_slice2"])
def test_table_builder_path_matches_the_oracle_builder(name):
    from gpu_harness import job_from_params
    p, inputs = C.build(name)
    entries = [e for f in H.oracle_compact(p, inputs)[0] for e in sstfmt.parse_sst(f)["entries"]]
    p.max_output_file_size = C.BIG
    want = H.oracle_build_sst(p, H.kvstream(entries))
    job = job_from_params(p)
    try:
        job.encode_kv(entries)
        files = job.outputs()
    finally:
        job.close()
    _same_files(name, files, [want])


@pytest.mark.parametrize("name, blocks", [("filter_phases", 2), ("sep_v5_xxh3", 1)])
def test_xxh3_adds_one_contribution_launch_per_checksummed_block(name, blocks):
    """file_block_contrib_kernel runs only for XXH3: once over the index blocks and, with a filter policy, once over the filter blocks"""
    from gpu_harness import run_product
    p, inputs = C.build(name)
    launches = {}
    for ck in ("xxh3", "crc32c"):
        q = copy.copy(p)
        q.checksum = ck
        launches[ck] = run_product(q, inputs)[2].kernel_launches
    print(f"{name}: kernel launches {launches}")
    assert launches["xxh3"] - launches["crc32c"] == blocks, launches


def test_one_file_more_than_the_limit_is_refused():
    from gpu_harness import run_product
    import toplingdb_b200 as T
    p, inputs = C.build("files_over")
    with pytest.raises(T.B200cError) as ei:
        run_product(p, inputs)
    assert ei.value.code == T.native.ERR_NOT_SUPPORTED, str(ei.value)
    assert f"more-than-{C.MAX_FILES}-output-files" in str(ei.value)
