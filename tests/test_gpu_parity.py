"""GPU parity tests (run with -m gpu on an H100): the CUDA path, called through the C ABI, against
 (a) the committed output files of the unmodified reference (tests/golden), (b) the CPU oracle on seeded inputs,
 (c) per-stage oracles (decode, merge) so a failure points at one kernel."""
import random
import struct

import pytest

try:  # a fresh box can take minutes to page torch in: do it at collection time, outside any per-test timeout
    import torch  # noqa: F401
except Exception:  # pragma: no cover
    torch = None

import helpers as H
import scenarios as S
import sstfmt

pytestmark = pytest.mark.gpu


def _T():
    import toplingdb_b200 as T
    return T


def test_device_block_checksums_match_oracle():
    T = _T()
    L = H.oracle()
    rnd = random.Random(11)
    bufs = [rnd.randbytes(n) for n in list(range(0, 260, 7)) + [1023, 1024, 1025, 2048, 4000, 4096, 4097, 5000, 20000, 100001]]
    bufs += [b"This is a short block!", b"This is a long block!" * 100]
    for kind in ("xxh3", "crc32c"):
        for last in (0, 1, 7):
            got = T.block_checksums(kind, bufs, last)
            want = [L.orc_block_checksum(H.CKSUM[kind], b, len(b), last) for b in bufs]
            bad = [(len(b), g, w) for b, g, w in zip(bufs, got, want) if g != w]
            assert not bad, (kind, last, bad[:5])
    # reference known answers (table/table_test.cc:2303-2389)
    got = T.block_checksums("xxh3", [b"This is a short block!", b"This is a long block!" * 100], 0)
    assert [struct.pack("<I", v).hex().upper() for v in got] == ["B37FB5E6", "FA2D482E"]
    got = T.block_checksums("crc32c", [b"This is a short block!", b"This is a long block!" * 100], 0)
    assert [struct.pack("<I", v).hex().upper() for v in got] == ["583F0355", "943EF0AB"]


@pytest.mark.parametrize("case", [c for c in H.golden_cases() if c != "long_keys"])
def test_decode_stage_matches_oracle(case):
    from gpu_harness import job_from_params, parse_key_recs
    T = _T()
    g = H.load_golden(case)
    p = H.params_from_reference(g)
    job = job_from_params(p)
    for d in g["inputs"]:
        job.add_input(d)
    job.run(until=1)
    for r, data in enumerate(g["inputs"]):
        want = sstfmt.parse_sst(data)["entries"]
        recs = parse_key_recs(job.debug(T.native.DBG_DECODED_KEYS, r))
        vals = job.debug(T.native.DBG_DECODED_VALUES, r)
        assert len(recs) == len(want)
        off = 0
        for (uk, tr, vlen), (ik, v) in zip(recs, want):
            assert uk + struct.pack("<Q", tr) == ik
            assert vals[off:off + vlen] == v
            off += vlen
    job.close()


def _expected_merged(p, inputs):
    entries = []
    for r, data in enumerate(inputs):
        for ik, v in sstfmt.parse_sst(data)["entries"]:
            entries.append((ik[:-8], -struct.unpack("<Q", ik[-8:])[0], r, ik, v))
    entries.sort(key=lambda e: (e[0], e[1], e[2]))
    kv = H.kvstream((e[3], e[4]) for e in entries)
    out, st = H.oracle_citer(p, kv)
    return H.parse_kvstream(out), st


@pytest.mark.parametrize("case", [c for c in H.golden_cases() if c != "long_keys"])
def test_merge_stage_matches_oracle(case):
    from gpu_harness import assert_merged_matches, job_from_params
    g = H.load_golden(case)
    p = H.params_from_reference(g)
    want, _ = _expected_merged(p, g["inputs"])
    job = job_from_params(p)
    for d in g["inputs"]:
        job.add_input(d)
    job.run(until=2)
    assert_merged_matches(job, want, case)
    job.close()


@pytest.mark.parametrize("case", [c for c in H.golden_cases() if c != "long_keys"])
@pytest.mark.parametrize("device_inputs", [False, True])
def test_full_job_matches_reference_fixture(case, device_inputs):
    from gpu_harness import run_product
    g = H.load_golden(case)
    p = H.params_from_reference(g)
    files, metas, st = run_product(p, g["inputs"], device_inputs=device_inputs)
    assert [len(f) for f in files] == [len(o) for o in g["outputs"]]
    for i, (a, b) in enumerate(zip(files, g["outputs"])):
        assert a == b, f"{case}: output {i} differs at byte {next(j for j in range(len(a)) if a[j] != b[j])}"
    for k in H.STAT_KEYS:
        assert getattr(st, k) == g["manifest"]["stats"][k], k
    for m, want in zip(metas, g["manifest"]["outputs"]):
        assert (m.file_size, m.num_entries, m.num_deletions) == (want["size"], want["num_entries"], want["num_deletions"])
        assert (m.smallest_seqno, m.largest_seqno) == (want["smallest_seqno"], want["largest_seqno"])
        assert bytes(m.smallest_ikey[: m.smallest_ikey_len - 8]).hex() == want["smallestkey"]
        assert bytes(m.largest_ikey[: m.largest_ikey_len - 8]).hex() == want["largestkey"]


def test_long_keys_are_rejected_not_mangled():
    from gpu_harness import run_product
    T = _T()
    g = H.load_golden("long_keys")
    p = H.params_from_reference(g)
    with pytest.raises(T.B200cError) as ei:
        run_product(p, g["inputs"])
    assert ei.value.code == T.native.ERR_NOT_SUPPORTED


def _oracle_inputs(runs, p_in):
    return [H.oracle_build_sst(p_in, H.kvstream(r)) for r in runs]


@pytest.mark.parametrize("seed,nruns,n,vlen,bottom,target", [
    (1, 8, 20000, 32, True, 1 << 20), (2, 16, 6000, 256, True, 2 << 20), (3, 4, 30000, 100, False, 512 << 10),
    (4, 3, 5000, 0, True, 64 << 10), (5, 33, 1500, 40, True, 256 << 10), (6, 2, 50000, 8, False, 300 << 10),
    (7, 5, 4000, 3000, True, 4 << 20)])
def test_seeded_jobs_match_oracle(seed, nruns, n, vlen, bottom, target):
    """inputs built by the oracle's table builder (itself pinned to the reference), larger than the fixtures:
    many tiles, many output files, wide fan-in, empty / large values"""
    from gpu_harness import run_product
    rnd = random.Random(seed)
    universe = n * nruns
    runs, seq = [], 1
    for r in range(nruns):
        keys = sorted(rnd.sample(range(universe // 2), n))
        run = []
        for k in keys:
            kb = struct.pack(">QQ", k >> 3, (k * 0x9E3779B97F4A7C15) & ((1 << 64) - 1)) if seed % 2 else struct.pack(">QQ", 0, k)
            t = 0 if rnd.random() < 0.1 else 1
            run.append((kb + struct.pack("<Q", (seq << 8) | t), b"" if t == 0 else rnd.randbytes(vlen)))
            seq += 1
        run.sort(key=lambda e: e[0][:-8])
        runs.append(run)
    inputs = _oracle_inputs(list(reversed(runs)), H.Params())  # newest run first
    p = H.Params(bottommost_level=bottom, max_output_file_size=target, file_creation_times=[7, 8, 9])
    want, wmetas, wst = H.oracle_compact(p, inputs)
    files, metas, st = run_product(p, inputs)
    assert [len(f) for f in files] == [len(o) for o in want]
    assert files == want
    for k in ("num_output_records", "num_records_replaced", "num_expired_deletion_records", "num_input_deletion_records",
              "total_input_raw_key_bytes", "total_input_raw_value_bytes"):
        assert getattr(st, k) == getattr(wst, k), k


def test_edge_single_entry_and_empty_result():
    from gpu_harness import run_product
    for case in ("tiny", "all_deleted"):
        g = H.load_golden(case)
        p = H.params_from_reference(g)
        files, _, _ = run_product(p, g["inputs"])
        assert files == g["outputs"]


def test_corrupt_input_is_detected():
    from gpu_harness import run_product
    T = _T()
    g = H.load_golden("basic_bottommost")
    p = H.params_from_reference(g)
    bad = bytearray(g["inputs"][0])
    bad[1000] ^= 0x40
    with pytest.raises(T.B200cError) as ei:
        run_product(p, [bytes(bad)] + g["inputs"][1:])
    assert ei.value.code == T.native.ERR_CORRUPTION


@pytest.mark.parametrize("case", ["filter_empty_value", "filter_empty_value_nonbottom", "ttl_filter", "ttl_filter_nonbottom"])
def test_in_kernel_compaction_filter_counts_like_the_oracle(case):
    """RemoveEmptyValueCompactionFilter / TtlCompactionFilter (DBWithTTL) applied inside the merge kernel (compaction_iterator.cc:579-584, :385-391): output
    bytes are covered by the fixture tests above; CompactionIterationStats::num_record_drop_user is not part of
    CompactionJobStats, so it is checked against the oracle."""
    from gpu_harness import run_product
    g = H.load_golden(case)
    p = H.params_from_reference(g)
    assert p.compaction_filter in ("remove_empty_value", "ttl")
    files, _, st = run_product(p, g["inputs"])
    ofiles, _, ost = H.oracle_compact(p, g["inputs"])
    assert files == ofiles == g["outputs"]
    assert st.num_record_drop_user == ost.num_record_drop_user > 0
    # the same inputs without the filter give different files: the rule really ran
    p.compaction_filter = "none"
    files2, _, st2 = run_product(p, g["inputs"])
    assert st2.num_record_drop_user == 0 and files2 != files


def test_level_runs_lift_the_file_cap():
    """MakeInputIterator gives every L0 file its own child and every deeper level ONE LevelIterator over its disjoint, ordered files
    (db/version_set.cc:1076,7311-7352).  Two L0 files + 100 L1 files + 40 L2 files = 142 files but 4 sorted runs: the device takes the
    job (round 1 refused more than 64 files); the oracle merges the same files as 142 runs, which yields the same stream because the
    files of a level do not overlap."""
    from gpu_harness import run_product
    T = _T()
    rnd = random.Random(77)
    seq = [1]

    def make_run(keys, delete_frac=0.1):
        out = []
        for k in keys:
            t = 0 if rnd.random() < delete_frac else 1
            out.append((struct.pack(">QQ", 1, k) + struct.pack("<Q", (seq[0] << 8) | t), b"" if t == 0 else rnd.randbytes(40)))
            seq[0] += 1
        return out

    universe = 60000
    l2_keys = sorted(rnd.sample(range(universe), 24000))
    l1_keys = sorted(rnd.sample(range(universe), 20000))
    l2 = make_run(l2_keys)
    l1 = make_run(l1_keys)
    l0b = make_run(sorted(rnd.sample(range(universe), 3000)))
    l0a = make_run(sorted(rnd.sample(range(universe), 3000)))  # newest

    def split(run, n):
        per = (len(run) + n - 1) // n
        return [run[i:i + per] for i in range(0, len(run), per)]

    files = [l0a, l0b] + split(l1, 100) + split(l2, 40)
    levels = [0, 0] + [1] * 100 + [2] * 40
    assert len(files) == 142 and len(levels) == 142
    inputs = [H.oracle_build_sst(H.Params(), H.kvstream(f)) for f in files]
    p = H.Params(bottommost_level=True, max_output_file_size=256 << 10, output_level=2, file_creation_times=[5])
    want, _, wst = H.oracle_compact(p, inputs)
    files_out, _, st = run_product(p, inputs, levels=levels)
    assert files_out == want
    for k in H.STAT_KEYS:
        assert getattr(st, k) == getattr(wst, k), k
    # the same files all declared L0 are 142 runs: still refused
    with pytest.raises(T.B200cError) as ei:
        run_product(p, inputs)
    assert ei.value.code == T.native.ERR_NOT_SUPPORTED
    # files of one level that are out of order are reported, not merged wrongly
    bad_inputs = [inputs[0], inputs[1], inputs[3], inputs[2]] + inputs[4:]
    with pytest.raises(T.B200cError) as ei:
        run_product(p, bad_inputs, levels=levels)
    assert ei.value.code == T.native.ERR_CORRUPTION
