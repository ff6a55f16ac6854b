"""The device against the checker on the jobs of combo_cases.py: optional parts switched on together (files byte for byte, statistics,
file metadata; with paranoid_file_checks the same files as without), independent jobs of different shapes in flight at once from 4 and
8 threads, buffers handed from one job to the next job of another shape, sub-jobs of two parents at once, and the reference DB through
the executor plugin with several options at once."""
import os
import threading

import pytest

try:
    import torch  # noqa: F401
except Exception:  # pragma: no cover
    torch = None

import combo_cases as C
import helpers as H
import partition_cases as PC
import sstfmt
from gpu_harness import describe_first_difference, job_from_params

pytestmark = pytest.mark.gpu


def _names():
    return C.names() + [C.REFUSAL_TWIN]


def _usable(name):
    return not C.needs_reference(name) or H.have_ref()


def _job(c, **extra):
    """an unrun job of the case (every input added), and what keeps its inputs alive; a host-deferred case is a sub-job of a parent
    whose inputs are uploaded range by range"""
    p, kw = c["params"], dict(c["extras"], **extra)
    res = c["residency"]
    keep = []
    parent = job_from_params(p, **kw) if res == "deferred" else None
    job = parent or job_from_params(p, **kw)
    for i, (data, lvl) in enumerate(zip(c["inputs"], c["levels"])):
        if res == "device":
            t = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
            keep.append(t)
            job.add_input(t, level=lvl, file_number=i)
        else:
            job.add_input(data, level=lvl, file_number=i, deferred=res == "deferred")
    if parent is not None:
        parent.upload_by_ranges([b for b in (p.range_start, p.range_end) if b is not None])
        job = parent.sub_job(range_start=p.range_start, range_end=p.range_end)
        keep.append(parent)
    return job, keep


def _result(job):
    return job.outputs(), [job.output_meta(i) for i in range(job.output_count())], job.stats()


def run_case(c, **extra):
    job, keep = _job(c, **extra)
    try:
        job.run()
        return _result(job)
    finally:
        job.close()
        for k in keep:
            if hasattr(k, "close"):
                k.close()


def _meta(m):
    return (m.file_size, m.num_entries, m.num_deletions, m.num_data_blocks, bytes(m.smallest_ikey[:m.smallest_ikey_len]),
            bytes(m.largest_ikey[:m.largest_ikey_len]))


def _want_meta(m):
    return (m.file_size, m.num_entries, m.num_deletions, m.num_data_blocks, bytes(m.smallest[:m.smallest_len]), bytes(m.largest[:m.largest_len]))


def assert_matches(name, got):
    e = C.expected(name)
    files, metas, st = got
    assert len(files) == len(e["files"]), f"{name}: {len(files)} files, the checker wrote {len(e['files'])}"
    for i, (g, w) in enumerate(zip(files, e["files"])):
        assert g == w, f"{name}: file {i}: {describe_first_difference(g, w)}"
    for k in H.STAT_KEYS + ("num_record_drop_user",):
        assert getattr(st, k) == getattr(e["stats"], k), (name, k)
    assert [_meta(m) for m in metas] == [_want_meta(m) for m in e["metas"]], name


@pytest.mark.parametrize("name", _names())
def test_job_matches_the_checker(name):
    if not _usable(name):
        pytest.skip("oracle/_ref not built: the zlib inputs are written by the reference")
    c = C.build(name)
    got = run_case(c)
    assert_matches(name, got)
    if c["extras"]["paranoid_file_checks"]:  # the read-back changes nothing
        assert run_case(c, paranoid_file_checks=0)[0] == got[0]
    else:
        assert run_case(c, paranoid_file_checks=1)[0] == got[0]


def test_write_conflict_snapshot_with_single_deletes_is_refused_beside_its_twin():
    import toplingdb_b200 as T
    if not H.have_ref():
        pytest.skip("oracle/_ref not built: the zlib inputs are written by the reference")
    with pytest.raises(T.B200cError) as ei:
        run_case(C.build(C.REFUSAL))
    assert ei.value.code == T.native.ERR_NOT_SUPPORTED
    assert_matches(C.REFUSAL_TWIN, run_case(C.build(C.REFUSAL_TWIN)))


def _all_expected():
    names = [n for n in _names() if _usable(n)]
    for n in names:
        C.expected(n)
    return names


def _run_in_threads(names, nthreads):
    """every job once, from nthreads threads, one handle per job; the results by name"""
    import queue
    todo = queue.Queue()
    for n in names:
        todo.put(n)
    got, errs = {}, []

    def worker():
        while True:
            try:
                n = todo.get_nowait()
            except queue.Empty:
                return
            try:
                got[n] = run_case(C.build(n))
            except Exception as ex:  # noqa: BLE001
                errs.append((n, ex))
    ths = [threading.Thread(target=worker) for _ in range(nthreads)]
    for t in ths:
        t.start()
    for t in ths:
        t.join()
    assert not errs, errs
    return got


@pytest.mark.parametrize("nthreads", [4, 8])
def test_jobs_of_different_shapes_at_once(nthreads):
    names = _all_expected()
    got = _run_in_threads(names, nthreads)
    for n in names:
        assert_matches(n, got[n])


def test_cached_buffers_of_another_shape():
    """the jobs one after the other from the largest to the smallest: the buffer cache hands a cached buffer to a request between half
    its size and its size, so each job mostly runs in buffers that a slightly larger job of another shape held and did not clear; then
    one handle runs twice with another job run on another handle in between"""
    names = sorted(_all_expected(), key=lambda n: C.expected(n)["stats"].num_input_records)
    for n in reversed(names):
        assert_matches(n, run_case(C.build(n)))
    small, large = names[0], names[-1]
    job, keep = _job(C.build(small))
    job.run()
    assert_matches(small, _result(job))
    assert_matches(large, run_case(C.build(large)))
    job.run()
    assert_matches(small, _result(job))
    job.close()


def _sub_jobs(parent_case, ranged):
    """a parent over the inputs of parent_case, host-deferred and uploaded range by range, with one sub-job per ranged case"""
    c = C.build(parent_case)
    parent = job_from_params(c["params"], **c["extras"])
    for i, (data, lvl) in enumerate(zip(c["inputs"], c["levels"])):
        parent.add_input(data, level=lvl, file_number=i, deferred=True)
    bounds = sorted({b for n in ranged for b in (C.build(n)["params"].range_start, C.build(n)["params"].range_end) if b is not None})
    parent.upload_by_ranges(bounds)
    subs = []
    for n in ranged:
        q = C.build(n)["params"]
        subs.append((n, parent.sub_job(range_start=q.range_start, range_end=q.range_end, **_sub_params(q), **C.build(n)["extras"])))
    return parent, subs


def _sub_params(q):
    return dict(output_level=q.output_level, bottommost_level=q.bottommost_level, format_version=q.format_version, checksum=q.checksum,
                snapshots=list(q.snapshots), compaction_filter=q.compaction_filter, ttl=q.ttl, ttl_now=q.now,
                grandparents=list(q.grandparents), level_compaction_dynamic_file_size=int(q.level_compaction_dynamic_file_size),
                max_compaction_bytes=q.max_compaction_bytes, bloom_millibits_per_key=q.bloom_millibits_per_key,
                first_file_number=q.first_file_number, file_creation_times=list(q.file_creation_times))


def _share_inputs(a, b):
    ca, cb = C.build(a), C.build(b)
    return ca["inputs"] == cb["inputs"] and ca["levels"] == cb["levels"]


def test_ranged_jobs_as_sub_jobs_of_shared_parents_at_once():
    """every ranged job runs as a sub-job of a parent over its inputs (pipelined upload): the ranged jobs over one set of inputs share
    one parent, and the sub-jobs of all parents run at the same time"""
    ranged = [n for n in _all_expected() if C.build(n)["params"].range_start is not None or C.build(n)["params"].range_end is not None]
    groups = []
    for n in ranged:
        for g in groups:
            if _share_inputs(g[0], n):
                g.append(n)
                break
        else:
            groups.append([n])
    groups.sort(key=len, reverse=True)
    assert len(groups) >= 2 and len(groups[0]) >= 2
    parents, subs = [], []
    for g in groups:
        parent, s = _sub_jobs(g[0], g)
        parents.append(parent)
        subs += s
    errs = []

    def run(j):
        try:
            j.run()
        except Exception as ex:  # noqa: BLE001
            errs.append(ex)
    ths = [threading.Thread(target=run, args=(j,)) for _, j in subs]
    for t in ths:
        t.start()
    for t in ths:
        t.join()
    assert not errs, errs
    for n, j in subs:
        assert_matches(n, _result(j))
        j.close()
    for p in parents:
        p.close()


# ------------------------------------------------------------------------------------------------ the reference DB through the plugin
def test_reference_db_with_several_options_through_the_executor():
    """partitioner, Bloom filter, max_subcompactions = 4, paranoid_file_checks and DB::CompactRange over grandparents at once, SingleDeletes
    and snapshots in the script: the same DB contents as the reference's own CPU run"""
    if not (PC.have_ref() and os.path.exists(PC.REF_PART_B200_BIN)):
        pytest.fail("oracle/_ref/ref_compact_partition(_b200) missing: run __graft_entry__.build() where /root/reference exists")
    ops, opts, plen = C.ref_combo("grandparents_subcompactions_bloom_paranoid_p2")
    want = PC.run_reference(ops, plen, **opts)
    got = PC.run_reference(ops, plen, binary=PC.REF_PART_B200_BIN, executor="b200", **opts)
    gm, wm = got["manifest"], want["manifest"]
    assert gm["executor"] == "B200Compact" and gm["remote_compact_read_bytes"] > 0
    assert len(wm["subcompactions"]) >= 2, "the reference did not split this job"
    assert len(wm["grandparents"]) >= 2
    assert (gm["scan_count"], gm["scan_digest"]) == (wm["scan_count"], wm["scan_digest"])
    for k in H.STAT_KEYS:
        assert gm["stats"][k] == wm["stats"][k], k
    # the executor plans its own key ranges (b200c_job_plan_ranges), so the files of a range may be cut elsewhere than the
    # reference's: the same entries in order, every file's count as its properties state, and a sorted, non-overlapping level
    ge = [sstfmt.parse_sst(f) for f in got["outputs"]]
    assert [e for t in ge for e in t["entries"]] == [e for f in want["outputs"] for e in sstfmt.parse_sst(f)["entries"]]
    assert all(sstfmt.prop_u64(t["properties"], "rocksdb.num.entries") == len(t["entries"]) for t in ge)
    assert all(a["entries"][-1][0][:-8] < b["entries"][0][0][:-8] for a, b in zip(ge, ge[1:]))
