"""The decode cases (decode_cases.py; their edges are proven by test_decode_cases_cpu.py) on the device, through the C ABI:
 (a) stage level: run(until=1), then every run's decoded keys and values against sstfmt's entries of the blocks the decoder is expected
     to keep (all of them, or for a key range the blocks index_decode_kernel keeps) -- a failure names the block, the entry's offset in
     it, the block's phase and the path the decoder should have taken; then the merge stage against the oracle's compaction iterator
     over the entries in range;
 (b) job level on the same inputs: every output file byte for byte, the statistics and the per-file metadata against the oracle's job
     (and, for reference-written inputs, against the reference's own outputs); a value of 2^27 bytes is refused with ERR_NOT_SUPPORTED;
 (c) a subset with device-resident inputs, and the index_walk inputs as sub-jobs over planned key ranges.
Every job runs once."""
import copy

import pytest

try:  # a fresh box can take minutes to page torch in: do it at collection time, outside any per-test timeout
    import torch  # noqa: F401
except Exception:  # pragma: no cover
    torch = None

import decode_cases as D
import helpers as H
import sstfmt

pytestmark = pytest.mark.gpu

STAGE_CASES = sorted(D.CASES) + ["headers_vlen_max"] + D.INFLATE_CASES
DEVICE_INPUTS = ["staging_limit", "staging_limit_crc32c_fv4", "key_words_slow", "headers", "skipped", "inflate_4k_ri16_fv5",
                 "inflate_4k_ri16_fv5_range"]


def _case(name):
    if name in D.INFLATE_CASES and not H.have_ref():
        pytest.fail("oracle/_ref missing: run __graft_entry__.build() where /root/reference exists")
    return D.case(name)


def _assert_job(files, metas, st, want, wmetas, wst, label):
    assert [len(f) for f in files] == [len(f) for f in want], label
    for i, (a, b) in enumerate(zip(files, want)):
        assert a == b, f"{label}: output {i} differs at byte {next(j for j in range(len(a)) if a[j] != b[j])}"
    for k in H.STAT_KEYS:
        assert getattr(st, k) == getattr(wst, k), (label, k)
    for i, (m, om) in enumerate(zip(metas, wmetas)):
        assert (m.file_size, m.num_entries, m.num_deletions, m.raw_key_size, m.raw_value_size, m.num_data_blocks, m.smallest_seqno,
                m.largest_seqno) == (om.file_size, om.num_entries, om.num_deletions, om.raw_key_size, om.raw_value_size, om.num_data_blocks,
                                     om.smallest_seqno, om.largest_seqno), (label, i)
        assert bytes(m.smallest_ikey[:m.smallest_ikey_len]) == bytes(om.smallest[:om.smallest_len]), (label, i)
        assert bytes(m.largest_ikey[:m.largest_ikey_len]) == bytes(om.largest[:om.largest_len]), (label, i)


def _in_range(p, uk):
    return (p.range_start is None or uk >= p.range_start) and (p.range_end is None or uk < p.range_end)


def _merged_want(p, inputs):
    merged = []
    for r, d in enumerate(inputs):
        for ik, v in sstfmt.parse_sst(d)["entries"]:
            if _in_range(p, ik[:-8]):
                merged.append((ik[:-8], -int.from_bytes(ik[-8:], "little"), r, ik, v))
    merged.sort(key=lambda x: x[:3])
    out, _ = H.oracle_citer(p, H.kvstream((x[3], x[4]) for x in merged))
    return H.parse_kvstream(out)


@pytest.mark.parametrize("name", STAGE_CASES)
def test_decode_stage_matches_the_tables_on_decode_cases(name):
    from gpu_harness import assert_decoded_matches, assert_merged_matches, job_from_params
    c = _case(name)
    p = c["params"]
    job = job_from_params(p)
    for i, d in enumerate(c["inputs"]):
        job.add_input(d, file_number=i)
    job.run(until=1)
    for r, d in enumerate(c["inputs"]):
        kept = D.kept_blocks(d, p.range_start, p.range_end)
        entries, where = D.located_entries(d, kept)
        assert all(any(k[:-8] == ik[:-8] for ik, _ in entries) for k, _ in sstfmt.parse_sst(d)["entries"] if _in_range(p, k[:-8]))
        assert_decoded_matches(job, r, entries, name, where)
    job.close()
    job = job_from_params(p)
    for i, d in enumerate(c["inputs"]):
        job.add_input(d, file_number=i)
    job.run(until=2)
    assert_merged_matches(job, _merged_want(p, c["inputs"]), name)
    job.close()


@pytest.mark.parametrize("name", STAGE_CASES)
def test_job_matches_oracle_on_decode_cases(name):
    from gpu_harness import run_product
    _case(name)
    e = D.expected(name)
    files, metas, st = run_product(e["params"], e["inputs"])
    _assert_job(files, metas, st, e["files"], e["metas"], e["stats"], name)
    if name in D.INFLATE_CONFIGS:  # the compiled reference's own outputs of the same job
        assert files == D.inflate_case(name)["ref"]["outputs"], name


def test_value_of_2_to_the_27_bytes_is_refused():
    from gpu_harness import run_product
    import toplingdb_b200 as T
    c = D.case("headers_vlen_too_long")
    with pytest.raises(T.B200cError) as ei:
        run_product(c["params"], c["inputs"])
    assert ei.value.code == T.native.ERR_NOT_SUPPORTED


@pytest.mark.parametrize("name", DEVICE_INPUTS)
def test_device_resident_inputs_on_decode_cases(name):
    """device images are 16-byte aligned (checked by the library), so every block keeps its file phase; host images are copied into
    a fresh cudaMalloc buffer, whose base is 256-byte aligned -- the phases of both runs are the file offsets mod 16"""
    from gpu_harness import run_product
    _case(name)
    e = D.expected(name)
    files, metas, st = run_product(e["params"], e["inputs"], device_inputs=True)
    _assert_job(files, metas, st, e["files"], e["metas"], e["stats"], name)


@pytest.mark.parametrize("fv", [3, 4, 5])
def test_index_walk_as_sub_jobs(fv):
    from gpu_harness import job_from_params
    e = D.expected(f"index_walk_fv{fv}")
    p = e["params"]
    parent = job_from_params(p)
    for i, d in enumerate(e["inputs"]):
        parent.add_input(d, level=0, file_number=i)
    bounds = parent.plan_ranges(4, min_range_bytes=4 << 10)
    assert len(bounds) >= 2, bounds
    ranges = list(zip([None] + bounds, bounds + [None]))
    subs = [parent.sub_job(range_start=a, range_end=b, first_file_number=1000 * (i + 1)) for i, (a, b) in enumerate(ranges)]
    total_in = total_out = 0
    for i, ((a, b), j) in enumerate(zip(ranges, subs)):
        j.run()
        q = copy.copy(p)
        q.range_start, q.range_end, q.first_file_number = a, b, 1000 * (i + 1)
        want, wmetas, wst = H.oracle_compact(q, e["inputs"])
        st = j.stats()
        _assert_job(j.outputs(), [j.output_meta(x) for x in range(j.output_count())], st, want, wmetas, wst, (fv, a, b))
        total_in += st.num_input_records
        total_out += st.num_output_records
    assert (total_in, total_out) == (e["stats"].num_input_records, e["stats"].num_output_records)
    for j in subs:
        j.close()
    parent.close()
