"""The SingleDelete cases (sd_cases.py; their edges are proven by test_sd_cases_cpu.py) on the device, through the C ABI:
 (a) stage level: run(until=2), the merged records and values against the oracle's compaction iterator entry by entry, and the stage's
     statistics; a failure names the tile that holds the first differing key and the moves of the boundaries around it;
 (b) job level: every output file byte for byte against the oracle, all statistics (num_record_drop_user included) and the per-file
     metadata; 512-byte blocks over the moves and the empty last tile;
 (c) refusals (ERR_NOT_SUPPORTED) next to their accepted twins, the same inputs without one entry: the tests pin the limits;
 (d) the decoder's SingleDelete flag from each of its paths, device-resident inputs under the TTL filter, sub-jobs cut at SingleDelete
     keys, and -- at the device's own size -- tile boundaries that the partition resolves as the second of a warp's chunk."""
import collections
import copy
import struct

import numpy as np
import pytest

try:  # a fresh box can take minutes to page torch in: do it at collection time, outside any per-test timeout
    import torch
except Exception:  # pragma: no cover
    torch = None

import helpers as H
import merge_cases as M
import sd_cases as S
from test_gpu_merge_cases import _assert_job

pytestmark = pytest.mark.gpu
SMALL_BLOCKS = ["moves_one_run", "moves_spread", "empty_last_tile_r1", "empty_last_tile_r32"]


def _T():
    import toplingdb_b200 as T
    return T


def _stage_label(job, e, name):
    """the case, and the tile that holds the first key where the device and the oracle part"""
    from gpu_harness import parse_key_recs
    recs = parse_key_recs(job.debug(_T().native.DBG_MERGED_KEYS))
    for (uk, tr, _), (ik, _) in zip(recs, e["records"]):
        if uk + struct.pack("<Q", tr) != ik:
            return f"{name}, {S.where(e, min(uk, ik[:-8]))}"
    return name


@pytest.mark.parametrize("name", sorted(S.CASES))
def test_merge_stage_matches_oracle_on_sd_cases(name):
    from gpu_harness import assert_merged_matches, job_from_params
    e = S.expected(name)
    job = job_from_params(e["params"])
    for i, d in enumerate(e["inputs"]):
        job.add_input(d, file_number=i)
    job.run(until=2)
    assert_merged_matches(job, e["records"], _stage_label(job, e, name))
    st = job.stats()
    for k in M.STAGE_STAT_KEYS:
        assert getattr(st, k) == getattr(e["stage_stats"], k), (name, k)
    assert st.num_input_records == len(e["order"])
    job.close()


@pytest.mark.parametrize("name", sorted(S.CASES))
def test_job_matches_oracle_on_sd_cases(name):
    from gpu_harness import run_product
    e = S.expected(name)
    files, metas, st = run_product(e["params"], e["inputs"])
    _assert_job(files, metas, st, e["files"], e["metas"], e["stats"], name)
    if e["params"].compaction_filter != "none":
        assert st.num_record_drop_user > 0


@pytest.mark.parametrize("name", SMALL_BLOCKS)
def test_job_matches_oracle_on_sd_cases_with_small_blocks(name):
    from gpu_harness import run_product
    e = S.expected(name)
    p = copy.copy(e["params"])
    p.block_size, p.block_restart_interval = 512, 4
    want, wmetas, wst = H.oracle_compact(p, e["inputs"])
    files, metas, st = run_product(p, e["inputs"])
    _assert_job(files, metas, st, want, wmetas, wst, name)


@pytest.mark.parametrize("name", sorted(S.REFUSED))
def test_refused_next_to_its_accepted_twin(name):
    """one entry more than the limit is refused with ERR_NOT_SUPPORTED; the same inputs without it are compacted as the oracle does"""
    from gpu_harness import run_product
    T = _T()
    e = S.expected(name)
    with pytest.raises(T.B200cError) as ei:
        run_product(e["params"], e["inputs"])
    assert ei.value.code == T.native.ERR_NOT_SUPPORTED, ei.value
    twin = S.expected(name + "_minus_one")
    assert sum(map(len, twin["runs"])) == sum(map(len, e["runs"])) - 1
    files, metas, st = run_product(twin["params"], twin["inputs"])
    _assert_job(files, metas, st, twin["files"], twin["metas"], twin["stats"], name + "_minus_one")


@pytest.mark.parametrize("name", S.FLAG_CASES)
def test_single_delete_flag_from_every_decoder_path(name):
    """the job's only SingleDelete lies in a block the decoder takes by the named path; had that path not raised the flag, the plain
    merge variant would keep the SingleDelete (test_sd_cases_cpu.py proves the records would differ)"""
    from gpu_harness import run_product
    if name == "flag_zlib" and not H.have_ref():
        pytest.skip("oracle/_ref not built (needs /root/reference)")
    c = S.flag_case(name)
    want, wmetas, wst = H.oracle_compact(c["params"], c["inputs"])
    files, metas, st = run_product(c["params"], c["inputs"])
    _assert_job(files, metas, st, want, wmetas, wst, f"{name}: run {c['run']} block {c['block']} ({c['path']})")
    if c["ref"] is not None:
        assert files == c["ref"]["outputs"]


@pytest.mark.parametrize("name", ["sd_filter_ttl_bottom", "sd_filter_ttl_nonbottom"])
def test_device_resident_inputs_on_sd_cases(name):
    """the serial walk's TTL verdict reads the stamp through the value reference, which points into the caller's device memory here"""
    from gpu_harness import run_product
    e = S.expected(name)
    files, metas, st = run_product(e["params"], e["inputs"], device_inputs=True)
    _assert_job(files, metas, st, e["files"], e["metas"], e["stats"], name)
    assert st.num_record_drop_user > 0


def test_sub_jobs_cut_at_single_delete_keys():
    """range boundaries on SingleDelete keys of 20 versions (a range that starts there owns them all), and a range of plain keys only
    inside a job that holds SingleDeletes"""
    from gpu_harness import job_from_params
    e = S.expected("subjob_keys")
    p, order = e["params"], e["order"]
    groups = collections.defaultdict(list)
    for uk, _, t, _, _ in order:
        groups[uk].append(t)
    sd20 = sorted(uk for uk, ts in groups.items() if len(ts) == S.SUBJOB_VERSIONS and M.SINGLE_DELETION in ts)
    assert len(sd20) >= 4
    keys = sorted(groups)
    # the longest stretch of keys without a SingleDelete: a range over its middle third
    best, start = (0, 0), 0
    for i, uk in enumerate(keys + [None]):
        if uk is None or M.SINGLE_DELETION in groups[uk]:
            best = max(best, (i - start, start))
            start = i + 1
    n, a = best
    plain = (keys[a + n // 3], keys[a + 2 * n // 3])
    assert n >= 500
    bounds = sorted(set(sd20) | set(plain))
    ranges = list(zip([None] + bounds, bounds + [None]))
    assert plain in ranges
    parent = job_from_params(p)
    for i, d in enumerate(e["inputs"]):
        parent.add_input(d, level=0, file_number=i)
    subs = [parent.sub_job(range_start=lo, range_end=hi, first_file_number=1000 * (i + 1)) for i, (lo, hi) in enumerate(ranges)]
    total_in = total_out = 0
    for i, ((lo, hi), j) in enumerate(zip(ranges, subs)):
        j.run()
        q = copy.copy(p)
        q.range_start, q.range_end, q.first_file_number = lo, hi, 1000 * (i + 1)
        want, wmetas, wst = H.oracle_compact(q, e["inputs"])
        st = j.stats()
        _assert_job(j.outputs(), [j.output_meta(x) for x in range(j.output_count())], st, want, wmetas, wst, ("subjob_keys", lo, hi))
        total_in += st.num_input_records
        total_out += st.num_output_records
    assert (total_in, total_out) == (e["stats"].num_input_records, e["stats"].num_output_records)
    for j in subs:
        j.close()
    parent.close()


def _device_stream(keys, vals):
    """the merge stage's debug columns as a kv stream (helpers.kvstream format), built in slices: 16-byte user keys, values of 0 or 8
    bytes"""
    rec = np.frombuffer(keys, dtype=[("hi", "<u8"), ("lo", "<u8"), ("tr", "<u8"), ("ulen", "<u4"), ("vlen", "<u4")])
    assert (rec["ulen"] == 16).all() and np.isin(rec["vlen"], (0, 8)).all()
    vlen = rec["vlen"].astype(np.int64)
    voff = np.concatenate([[0], np.cumsum(vlen)[:-1]])
    varr = np.frombuffer(vals, dtype=np.uint8)
    out = []
    for c in range(0, len(rec), 1 << 21):
        r, m = rec[c:c + (1 << 21)], min(1 << 21, len(rec) - c)
        row = np.zeros((m, 40), dtype=np.uint8)
        row[:, 0:4] = np.array([24], dtype="<u4").view(np.uint8)
        row[:, 4:8] = r["vlen"].astype("<u4").view(np.uint8).reshape(m, 4)
        row[:, 8:16] = r["hi"].astype(">u8").view(np.uint8).reshape(m, 8)
        row[:, 16:24] = r["lo"].astype(">u8").view(np.uint8).reshape(m, 8)
        row[:, 24:32] = r["tr"].astype("<u8").view(np.uint8).reshape(m, 8)
        has = np.flatnonzero(vlen[c:c + m] == 8)
        row[has, 32:40] = varr[voff[c:c + m][has][:, None] + np.arange(8)]
        out.append(row[np.arange(40)[None, :] < (32 + vlen[c:c + m])[:, None]].tobytes())
    return b"".join(out), voff + 32 * np.arange(len(rec)), rec


def test_merge_stage_on_chunked_boundaries_at_the_device_size():
    """case 10: enough entries that launch_merge_partition gives every partition warp two boundaries on this device; moves of 32, 1 and 0
    on the second boundary of a chunk and on consecutive boundaries, in one chunk and across two"""
    from gpu_harness import job_from_params
    T = _T()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    J = S.chunked_job(sms)
    job = job_from_params(J["params"])
    for i, d in enumerate(J["inputs"]):
        job.add_input(d, file_number=i)
    job.run(until=2)
    got, offs, rec = _device_stream(job.debug(T.native.DBG_MERGED_KEYS), job.debug(T.native.DBG_MERGED_VALUES))
    st = job.stats()
    job.close()
    want = J["want"]
    if got != want:
        m = min(len(got), len(want))
        diff = np.flatnonzero(np.frombuffer(got, np.uint8, m) != np.frombuffer(want, np.uint8, m))
        j = int(diff[0]) if len(diff) else m
        r = int(np.searchsorted(offs, j, side="right")) - 1
        kid = int(rec["hi"][min(r, len(rec) - 1)])
        cuts = S.chunked_cuts(J)
        t = S.tile_of(cuts, int(np.searchsorted(J["kid"], kid)))
        pytest.fail(f"{sms} SMs, chunk {S.chunk_of(J['ntiles'], sms)}: merged stream differs at byte {j} of {len(want)} (device "
                    f"{len(got)}), output entry {r} (key id {kid}) in tile {t}: boundary {t} moved {cuts[t]['move']}, boundary {t + 1} "
                    f"moved {cuts[t + 1]['move']}")
    for k in M.STAGE_STAT_KEYS:
        assert getattr(st, k) == getattr(J["stage_stats"], k), k
    assert st.num_input_records == J["n"]
