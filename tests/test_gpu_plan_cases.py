"""The block-cut planner's jobs (tests/plan_cases.py) through the C ABI against the CPU oracle: output bytes, statistics and file
metadata; the job whose smallest entry puts the block-chain candidate count past kEncHalo is refused with ERR_NOT_SUPPORTED."""
import pytest

import helpers as H
import plan_cases as P

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", [n for n in P.CASES if n != "hc_over_halo"])
def test_job_matches_oracle_on_plan_cases(name):
    from gpu_harness import run_product
    p, inputs = P.build(name)
    want, wmetas, wst = H.oracle_compact(p, inputs)
    files, metas, st = run_product(p, inputs)
    assert [len(f) for f in files] == [len(o) for o in want]
    for i, (a, b) in enumerate(zip(files, want)):
        assert a == b, f"output {i} differs at byte {next(j for j in range(len(a)) if a[j] != b[j])}"
    for k in H.STAT_KEYS:
        assert getattr(st, k) == getattr(wst, k), k
    for m, om in zip(metas, wmetas):
        assert (m.file_size, m.num_entries, m.num_deletions, m.num_data_blocks) == \
            (om.file_size, om.num_entries, om.num_deletions, om.num_data_blocks)


def test_candidate_count_past_the_halo_is_refused():
    from gpu_harness import run_product
    import toplingdb_b200 as T
    p, inputs = P.build("hc_over_halo")
    with pytest.raises(T.B200cError) as ei:
        run_product(p, inputs)
    assert ei.value.code == T.native.ERR_NOT_SUPPORTED
