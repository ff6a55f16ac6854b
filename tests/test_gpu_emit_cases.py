"""The emit stage's jobs (tests/emit_cases.py) on the device against the CPU oracle: the b200c_job_encode_kv jobs against the oracle's
table builder (file bytes and file metadata), the compaction jobs against the oracle's whole job (files, statistics, file metadata).
A failure names the region of the first differing byte (gpu_harness.describe_first_difference)."""
import pytest

import helpers as H
import emit_cases as C
import sstfmt

pytestmark = pytest.mark.gpu


def _same_files(name, files, want):
    from gpu_harness import describe_first_difference
    assert [len(f) for f in files] == [len(w) for w in want], f"{name}: file sizes differ"
    for i, (a, b) in enumerate(zip(files, want)):
        assert a == b, f"{name}: output {i} of {len(want)} differs at " + describe_first_difference(a, b)


@pytest.mark.parametrize("name", C.CASES)
def test_emit_case_matches_oracle(name):
    from gpu_harness import job_from_params, run_product
    p, (kind, data) = C.build(name)
    if kind == "compact":
        want, wmetas, wst = H.oracle_compact(p, list(data))
        files, metas, st = run_product(p, list(data))
        _same_files(name, files, want)
        for k in H.STAT_KEYS:
            assert getattr(st, k) == getattr(wst, k), k
        for m, om in zip(metas, wmetas):
            assert (m.file_size, m.num_entries, m.num_deletions, m.num_data_blocks, m.smallest_seqno, m.largest_seqno) == \
                (om.file_size, om.num_entries, om.num_deletions, om.num_data_blocks, om.smallest_seqno, om.largest_seqno)
        return
    want = H.oracle_build_sst(p, H.kvstream(data))
    job = job_from_params(p)
    try:
        job.encode_kv(list(data))
        files = job.outputs()
        metas = [job.output_meta(i) for i in range(job.output_count())]
    finally:
        job.close()
    _same_files(name, files, [want])
    seqs = [int.from_bytes(k[-8:], "little") >> 8 for k, _ in data]
    m = metas[0]
    assert (m.file_size, m.num_entries, m.num_data_blocks, m.smallest_seqno, m.largest_seqno) == \
        (len(want), len(data), len(sstfmt.parse_sst(want)["index"]), min(seqs), max(seqs))
