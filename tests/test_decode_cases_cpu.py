"""The decode cases (decode_cases.py) without a GPU: proof that every case sits on the edges it exists for, and that its tables are
legal tables.

 (a) every table reads the same in sstfmt and in the oracle's reader; the tables the oracle's builder wrote are read by the reference's
     stock reader as well (oracle/_ref/ref_sst_check: every block checksum verified, the whole file scanned);
 (b) per family, the decoder's dispatch restated from sstfmt's block parse and from the limits read out of csrc/decode.cu and
     csrc/common.cuh (decode_cases.table_blocks): the blocks on each side of every edge are counted and every count must be >= 1.  If a
     change of a limit or of a generator moves a case off its edge, this file fails -- the GPU test would otherwise pass while testing
     nothing.  The counts are in every assertion message."""
import collections
import json
import os
import subprocess

import pytest

import decode_cases as D
import helpers as H
import sstfmt

TOOL = os.path.join(H.ROOT, "oracle", "_ref", "ref_sst_check")
ALL_BUILT = sorted(D.CASES) + sorted(D.BIG_VALUE_CASES)


def _blocks(name):
    return [b for d in D.case(name)["inputs"] for b in D.table_blocks(d)]


def _need_ref():
    if not H.have_ref():
        pytest.skip("oracle/_ref not built (needs /root/reference)")


def _all_positive(counts, label):
    assert counts and min(counts.values()) >= 1, f"{label}: {dict(counts)}"
    print(label, dict(counts))


@pytest.mark.parametrize("name", ALL_BUILT + D.INFLATE_CASES)
def test_tables_read_the_same_in_sstfmt_and_the_oracle(name):
    if name in D.INFLATE_CASES:
        _need_ref()
    for data in D.case(name)["inputs"]:
        entries = sstfmt.parse_sst(data)["entries"]
        kv, n = H.oracle_sst_to_kv(data)
        assert n == len(entries) and H.parse_kvstream(kv) == entries, name
        assert [e for b in D.table_blocks(data) for e in b["entries"]] == entries


@pytest.mark.parametrize("name", ALL_BUILT)
def test_the_reference_reads_the_built_tables(name, tmp_path):
    if not os.path.exists(TOOL):
        pytest.skip("oracle/_ref not built (needs /root/reference)")
    for i, data in enumerate(D.case(name)["inputs"]):
        path = tmp_path / f"{i:06d}.sst"
        path.write_bytes(data)
        out = json.loads(subprocess.check_output([TOOL, str(path)], text=True))
        assert out["dumper_entries"] == out["num_entries"] == len(sstfmt.parse_sst(data)["entries"]), (name, i)
        assert out["num_data_blocks"] == len(D.table_blocks(data)), (name, i)


def test_staging_limit_blocks_sit_on_both_sides_at_every_phase():
    counts = collections.Counter()
    for name in ("staging_limit", "staging_limit_crc32c_fv4"):
        for b in _blocks(name):
            edge = b["phase"] + b["usize"] - D.STAGE_LIMIT
            if edge in (0, 1):
                counts[(name, "phase %d" % b["phase"], "limit" if edge == 0 else "limit + 1", b["path"])] += 1
            if b["usize"] >= D.DEC_SLICE:
                counts[(name, "at least the slice", b["path"])] += 1
        for q in range(16):
            for edge, path in ((0, "fast"), (1, "slow")):
                counts.setdefault((name, "phase %d" % q, "limit" if edge == 0 else "limit + 1", path), 0)
        counts.setdefault((name, "at least the slice", "slow"), 0)
    _all_positive(counts, "staging_limit")
    assert not any(k[-1] == "slow" and k[2] == "limit" or k[-1] == "fast" and k[2] == "limit + 1" for k in counts if len(k) == 4 and counts[k])
    sizes = {b["usize"] for n in ("staging_limit", "staging_limit_crc32c_fv4") for b in _blocks(n)}
    assert set(D.STAGING_EXTRA) <= sizes, sorted(s for s in sizes if s >= D.DEC_SLICE)


@pytest.mark.parametrize("ri", [1, 15, 16, 17, 32])
def test_rows_reach_the_interval_limits(ri):
    name = f"rows_ri{ri}"
    assert D.case(name)["params"].block_restart_interval == ri
    counts = collections.Counter()
    for b in _blocks(name):
        nr = len(b["rows"])
        last = len(b["rows"][-1])
        counts[("nr", nr, "full" if last == ri else "short")] += 1
        counts[("path", b["path"], b["why"])] += 1
    want = [("nr", nr, "full") for nr in D.ROW_COUNTS] + ([("nr", nr, "short") for nr in D.ROW_COUNTS] if ri > 1 else [])
    if ri <= D.DEC_ROW_LEN:  # up to 16 intervals of up to 16 entries stay on the fast path, 17 intervals leave it
        want += [("path", "fast", ""), ("path", "slow", "restart intervals")]
    else:
        want += [("path", "slow", "interval length")]
    _all_positive({k: counts[k] for k in want}, name)
    # the edges themselves: nr = 16 decoded fast and nr = 17 in a block small enough to be staged (ri <= 16)
    if ri <= D.DEC_ROW_LEN:
        edge = collections.Counter((len(b["rows"]), b["path"]) for b in _blocks(name) if b["why"] != "not staged")
        _all_positive({(16, "fast"): edge[(16, "fast")], (17, "slow"): edge[(17, "slow")]}, name + " nr edge")


def test_key_words_cover_every_scan_width():
    pairs = collections.Counter()
    ulens = collections.Counter()
    slow_past_16 = 0
    for name in ("key_words", "key_words_slow"):
        for b in _blocks(name):
            rows = b["rows"]
            if b["path"] == "slow":
                slow_past_16 += sum(1 for row in rows for _, sh, _, _, _ in row if sh > 16)
            if b["path"] == "fast":
                for r0 in range(0, len(rows), 2):
                    mx = max(sh for row in rows[r0:r0 + 2] for _, sh, _, _, _ in row)
                    pairs[("max shared", mx)] += 1
                    pairs[("scan words", D.scan_width(mx))] += 1
            for row in rows:
                for i, (k, _) in enumerate(_row_keys(b, row)):
                    ulens[("restart" if i == 0 else "behind", len(k) - 8)] += 1
    want = {("max shared", x): pairs[("max shared", x)] for x in D.KEY_WORD_TARGETS}
    want.update({("scan words", w): pairs[("scan words", w)] for w in range(4)})
    want["slow path entries sharing more than 16 bytes"] = slow_past_16
    _all_positive(want, "key_words")
    _all_positive({k: ulens[k] for k in [(p, n) for p in ("restart", "behind") for n in range(17)]}, "key_words user-key lengths")


def _row_keys(b, row):
    offs = [o for o, *_ in row]
    flat = [o for r in b["rows"] for o, *_ in r]
    return [b["entries"][flat.index(o)] for o in offs]


def test_key_words_shared_runs_past_the_user_key():
    """shared = ulen + 7 (versions whose sequence numbers differ in a high byte) and shared past the previous user key (a key that
    extends its predecessor's user key with the predecessor's trailer bytes)"""
    counts = collections.Counter()
    for name in ("key_words", "key_words_slow"):
        for b in _blocks(name):
            prev = None
            for row in b["rows"]:
                for i, ((k, _), (_, sh, _, _, _)) in enumerate(zip(_row_keys(b, row), row)):
                    if i and prev is not None:
                        if k[:-8] == prev[:-8] and sh == len(k) - 8 + 7:
                            counts[("versions, shared = ulen + 7", b["path"])] += 1
                        if len(k) - 8 > len(prev) - 8 and k[:len(prev) - 8] == prev[:-8] and sh > len(prev) - 8:
                            counts[("extends the previous user key", b["path"])] += 1
                    prev = k
    _all_positive({k: counts[k] for k in [(w, p) for w in ("versions, shared = ulen + 7", "extends the previous user key")
                                          for p in ("fast", "slow")]}, "key_words past the user key")


def test_headers_cover_every_varint_width_on_both_paths():
    counts = collections.Counter()
    types = collections.Counter()
    for b in _blocks("headers"):
        for row in b["rows"]:
            for _, _, _, vl, _ in row:
                if vl in D.FAST_VLENS + D.SLOW_VLENS:
                    counts[(vl, b["path"])] += 1
        for k, _ in b["entries"]:
            types[(k[-8], b["path"])] += 1
    want = {(v, "fast"): counts[(v, "fast")] for v in D.FAST_VLENS}
    want.update({(v, "slow"): counts[(v, "slow")] for v in D.FAST_VLENS + D.SLOW_VLENS})
    _all_positive(want, "headers")
    _all_positive({(t, p): types[(t, p)] for t in (D.VALUE, D.DELETION, D.SINGLE_DELETION) for p in ("fast", "slow")}, "headers types")
    assert [D.varint_len(v) for v in D.FAST_VLENS + D.SLOW_VLENS] == [1, 1, 2, 2, 3, 3, 4]
    for name, vlen in D.BIG_VALUE_CASES.items():
        got = [vl for b in _blocks(name) for row in b["rows"] for *_, vl, _ in row]
        assert max(got) == vlen and D.varint_len(vlen) == 4, name
    assert D.BIG_VALUE_CASES["headers_vlen_max"] == (1 << D.META_VLEN_BITS) - 1


def _stretches(name):
    """(skipped blocks in front of a kept block, that block's global index mod 32) over the job's global block order, and facts"""
    c = D.case(name)
    p = c["params"]
    flags, file_first, runs_empty = [], [], 0
    for d in c["inputs"]:
        kept = set(D.kept_blocks(d, p.range_start, p.range_end))
        file_first.append(len(flags))
        nb = len(D.table_blocks(d))
        flags += [j in kept for j in range(nb)]
        runs_empty += not kept
    out, run = collections.Counter(), 0
    for g, k in enumerate(flags):
        if k:
            if run:
                out[(run, g % D.LOOKBACK_STRIDE)] += 1
            run = 0
        else:
            run += 1
    return out, flags, runs_empty


def test_skipped_stretches_meet_the_look_back_stride():
    out, flags, empty = _stretches("skipped")
    counts = {(L, r): out[(L, r)] for L, r in D.SKIP_TARGETS}
    long_runs = sum(v for (L, _), v in out.items() if L >= 90)
    _all_positive(dict(counts, long=long_runs, empty_runs=empty, last_block_skipped=int(not flags[-1])), "skipped")
    assert {r for _, r in D.SKIP_TARGETS} == {0, 1, 31}
    out, flags, empty = _stretches("skipped_nothing_kept")
    assert not any(flags) and empty == len(D.case("skipped_nothing_kept")["inputs"])


def test_index_walk_takes_both_index_paths():
    counts = collections.Counter()
    for fv in (3, 4, 5):
        for ranged in ("", "_range"):
            name = f"index_walk_fv{fv}{ranged}"
            c = D.case(name)
            assert (c["params"].range_start is not None) == bool(ranged)
            for d, ir in zip(c["inputs"], (1,) + D.INDEX_INTERVALS + (16,)):  # (the builder's order; the last file has one block)
                info = D.index_info(d)
                assert info["fv"] == fv and info["nr"] == -(-info["nblocks"] // ir), (name, ir, info["nr"], info["nblocks"])
                path = "parallel" if info["parallel"] else "sequential"
                counts[(fv, ranged or "whole", path, "one block" if info["nblocks"] == 1 else "many")] += 1
                if not info["parallel"]:
                    counts[(fv, ranged or "whole", "interval", ir)] += 1
                    if fv >= 4 and any(info["shared"]):
                        counts[(fv, ranged or "whole", "delta-encoded sizes")] += 1
                    if not info["user_key"]:
                        counts[(fv, ranged or "whole", "separators keep the sequence number")] += 1
                if ranged and info["parallel"] and info["nblocks"] > 1:
                    kept = D.kept_blocks(d, c["params"].range_start, c["params"].range_end)
                    counts[(fv, ranged, "parallel blocks skipped")] += info["nblocks"] - len(kept)
    want = []
    for fv in (3, 4, 5):
        for r in ("whole", "_range"):
            want += [(fv, r, "sequential", "many"), (fv, r, "parallel", "one block"), (fv, r, "parallel", "many"),
                     (fv, r, "separators keep the sequence number")] + [(fv, r, "interval", ir) for ir in D.INDEX_INTERVALS]
            if fv >= 4:
                want.append((fv, r, "delta-encoded sizes"))
        want.append((fv, "_range", "parallel blocks skipped"))
    _all_positive({k: counts[k] for k in want}, "index_walk")


def test_inflate_reaches_both_sides_of_the_window():
    _need_ref()
    counts = collections.Counter()
    near = collections.Counter()
    for name in sorted(D.INFLATE_CONFIGS):
        c = D.case(name)
        bs, ri, fv, ck, ic = D.INFLATE_CONFIGS[name]
        man = D.inflate_case(name)["ref"]["manifest"]
        assert (man["block_size"], man["restart_interval"], man["format_version"], man["checksum"]) == (bs, ri, fv, ck)
        for d in c["inputs"]:
            for b in D.table_blocks(d):
                counts[(name, "compressed" if b["ctype"] == 2 else "stored raw")] += 1
                if b["ctype"] == 2:
                    u = b["usize"]
                    side = "<= limit" if u <= D.STAGE_LIMIT else "<= window" if u <= D.INFLATE_WINDOW else "> window"
                    counts[("inflated", side, b["path"])] += 1
                    if u in (D.INFLATE_WINDOW - 1, D.INFLATE_WINDOW, D.INFLATE_WINDOW + 1, D.STAGE_LIMIT, D.STAGE_LIMIT + 1):
                        near[(u, b["path"])] += 1
            assert sstfmt.parse_sst(d)["footer"]["checksum_type"] == H.CKSUM[ck]
    _all_positive(counts, "inflate")
    _all_positive({k: near[k] for k in [(D.INFLATE_WINDOW - 1, "arena-slow"), (D.INFLATE_WINDOW, "arena-slow"),
                                         (D.INFLATE_WINDOW + 1, "arena-slow"), (D.STAGE_LIMIT, "arena-fast"),
                                         (D.STAGE_LIMIT + 1, "arena-slow")]}, "inflate exact sizes")
    # a key range that skips compressed blocks
    c = D.case("inflate_4k_ri16_fv5_range")
    p = c["params"]
    skipped = sum(1 for d in c["inputs"] for b in D.table_blocks(d)
                  if b["ctype"] == 2 and b["index"] not in D.kept_blocks(d, p.range_start, p.range_end))
    _all_positive({"compressed blocks skipped by the range": skipped}, "inflate range")


def test_job_expectations_are_the_oracle_over_the_tables():
    """the job-level expectation of the built cases: the oracle's whole job agrees with its compaction iterator over the merged
    entries (the stage-level expectation of the GPU test)"""
    for name in ("staging_limit", "key_words", "headers", "skipped"):
        e = D.expected(name)
        p = e["params"]
        merged = []
        for r, d in enumerate(e["inputs"]):
            for ik, v in sstfmt.parse_sst(d)["entries"]:
                uk = ik[:-8]
                if (p.range_start is None or uk >= p.range_start) and (p.range_end is None or uk < p.range_end):
                    merged.append((uk, -int.from_bytes(ik[-8:], "little"), r, ik, v))
        merged.sort(key=lambda x: x[:3])
        out, st = H.oracle_citer(p, H.kvstream((x[3], x[4]) for x in merged))
        assert H.parse_kvstream(out) == [kv for f in e["files"] for kv in sstfmt.parse_sst(f)["entries"]], name
        assert st.num_output_records == e["stats"].num_output_records, name
