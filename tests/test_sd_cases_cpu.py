"""The SingleDelete cases (sd_cases.py) without a GPU: proof that every case sits on the edge it exists for, and that the oracle the GPU
tests use is right on them.

 (a) coverage witnesses, from sd_cases.moved_cuts (the partition rule restated, with kMergeTile / kSdSpill / kMaxGroup and the chunk
     rule read out of the sources) over the Python-merged order: moves of every size and the runs they come from, tiles of exactly
     kMergeTile entries, empty tiles, groups of 64 and 65 versions, filtered heads over SingleDeletes by shape, the lane groups of the
     partition warp, boundaries that a warp resolves as the second of its chunk.  Each case prints its census and fails if a witness it
     exists for is missing; refused cases must be refused for their one reason, their twins not at all.
 (b) oracle_citer over the merged stream and oracle_compact over the tables agree on records and statistics.
 (c) compaction filters together with SingleDeletes: the host build of csrc/group_rules.h (the device's serial walk) against the oracle
     on the filtered-head streams, and the oracle against the live reference on a SingleDelete + remove_empty_value write script.  TTL is
     not pinned this way: DBWithTTL::Write passes the batch through a handler without SingleDeleteCF (utilities/ttl/db_ttl_impl.cc),
     whose default SingleDelete does nothing, so the reference DB silently loses the SingleDeletes of a TTL script."""
import collections
import random
import struct

import pytest

import helpers as H
import merge_cases as M
import sd_cases as S
import sstfmt
from test_group_rules_host import sim, walk_stream  # noqa: F401  (sim: the module's fixture)

N = S.NOMINAL


def _groups(order):
    """[(first position, end)] of every user key"""
    out, i = [], 0
    while i < len(order):
        j = i
        while j < len(order) and order[j][0] == order[i][0]:
            j += 1
        out.append((i, j))
        i = j
    return out


def _has_sd(order, i, j):
    return any(order[x][2] == M.SINGLE_DELETION for x in range(i, j))


def census(e):
    order, cuts, nruns = e["order"], e["cuts"], len(e["runs"])
    sizes = S.tile_sizes(cuts)
    c = collections.Counter()
    for b in cuts:
        if b["move"]:
            k = sum(1 for x in b["per_run"] if x)
            c[f"move {b['move']}"] += 1
            c[f"move {b['move']} from {k} runs"] += 1
            c["runs contributing to a move"] += k
            i = b["nominal"] - 1
            while i > 0 and order[i - 1][0] == order[i][0]:
                i -= 1
            if not _has_sd(order, i, b["cut"]):
                c[f"plain key moved {b['move']}"] += 1
    for t, sz in enumerate(sizes):
        if sz == S.TILE:
            c["tiles of kMergeTile"] += 1
        if sz == 0:
            c["empty tiles"] += 1
        if t + 1 < len(cuts) - 1 and cuts[t]["move"] == cuts[t + 1]["move"] == S.SPILL:
            c["tiles between two 32-entry moves"] += 1
        if t > 0 and cuts[t]["move"] == S.SPILL and cuts[t + 1]["move"] == 0 and t + 1 < len(cuts) - 1:
            c["tiles behind a 32-entry move, in front of an unmoved cut"] += 1
    straddling = {(b["nominal"], b["cut"]) for b in cuts if b["move"]}
    for i, j in _groups(order):
        if _has_sd(order, i, j):
            if j - i in (S.MAX_GROUP, S.MAX_GROUP + 1):
                c[f"SingleDelete keys of {j - i} versions"] += 1
                if any(a == j for _, a in straddling) and i < N * (i // N + 1) < j:
                    c[f"SingleDelete keys of {j - i} versions across a cut"] += 1
            if any(i < nom < j for nom, _ in straddling) and e["params"].snapshots and \
                    any(M.stripe_index(e["params"].snapshots, order[x][1]) >= S.SNAP_CACHE for x in range(i, j)):
                c["moved SingleDelete keys with versions past the cached snapshots"] += 1
        elif j - i > S.MAX_GROUP:
            c["plain keys longer than kMaxGroup"] += 1
    if e["params"].compaction_filter != "none":
        c.update(_filtered_shapes(e))
    if nruns <= S.SD_MAX_RUNS:
        c[f"runs {nruns}: {S.lanes_per_run(nruns)} lanes per run, {32 // S.lanes_per_run(nruns) - nruns} idle groups"] += 1
    else:
        c[f"runs {nruns}: more than {S.SD_MAX_RUNS}"] += 1
    return c


def _filtered_shapes(e):
    order, p, snaps = e["order"], e["params"], e["params"].snapshots
    sd_tiles = {S.tile_of(e["cuts"], x) for x in range(len(order)) if order[x][2] == M.SINGLE_DELETION}
    c = collections.Counter()
    for i, j in _groups(order):
        types = [order[x][2] for x in range(i, j)]
        stale = [t == M.VALUE and M.filter_removes(p.compaction_filter, order[x][4]) for x, t in zip(range(i, j), types)]
        if stale[0] and len(types) > 1 and types[1] == M.SINGLE_DELETION:
            same = M.stripe_index(snaps, order[i][1]) == M.stripe_index(snaps, order[i + 1][1])
            c["filtered Put over a SingleDelete, " + ("same stripe" if same else "older stripe")] += 1
            if len(types) > 2 and types[2] == M.VALUE:
                c["filtered Put over a SingleDelete / Put pair"] += 1
        if types[0] == M.SINGLE_DELETION and len(types) > 1 and stale[1]:
            c["SingleDelete over a stale Put"] += 1
        if types == [M.VALUE] and stale[0] and S.tile_of(e["cuts"], i) in sd_tiles:
            c["filtered plain key in a tile with a SingleDelete"] += 1
    return c


def _all(*keys):
    return lambda c: [k for k in keys if c[k] < 1]


REQUIRED = {
    "moves_one_run": _all(*[f"move {m} from 1 runs" for m in (1, 2, 16, 31, 32)], "tiles of kMergeTile", "tiles between two 32-entry moves",
                          "tiles behind a 32-entry move, in front of an unmoved cut"),
    "moves_spread": _all(*[f"move 32 from {k} runs" for k in (1, 2, 3, 8, 16)], "move 31 from 16 runs", "tiles of kMergeTile"),
    "every_boundary_32": lambda c: [] if c["move 32"] == 9 and c["tiles between two 32-entry moves"] == 8 else ["nine 32-entry moves"],
    "alternate_32_0": lambda c: [] if c["move 32"] == 5 and c["tiles of kMergeTile"] == 5 else ["alternating 2048 / 1984 tiles"],
    "empty_last_tile_r1": _all("empty tiles", "move 1"),
    "empty_last_tile_r32": _all("empty tiles", "move 32"),
    "straddle_plain_32": _all("plain key moved 32"),
    "straddle_plain_33_minus_one": _all("plain key moved 32"),
    "spill_33_one_run_minus_one": _all("move 32 from 1 runs"),
    "spill_33_three_runs_minus_one": _all("move 32 from 3 runs"),
    "group_64": _all("SingleDelete keys of 64 versions", "SingleDelete keys of 64 versions across a cut", "plain keys longer than kMaxGroup"),
    "group_65_minus_one": _all("SingleDelete keys of 64 versions"),
    "runs_17_minus_one": _all("runs 16: 2 lanes per run, 0 idle groups"),
    "snaps_17": _all("moved SingleDelete keys with versions past the cached snapshots", "move 32"),
    "snaps_40": _all("moved SingleDelete keys with versions past the cached snapshots"),
}
for _k in ("empty_value_bottom", "empty_value_nonbottom", "ttl_bottom", "ttl_nonbottom"):
    REQUIRED["sd_filter_" + _k] = _all("filtered Put over a SingleDelete, same stripe", "filtered Put over a SingleDelete, older stripe",
                                        "filtered Put over a SingleDelete / Put pair", "SingleDelete over a stale Put",
                                        "filtered plain key in a tile with a SingleDelete", "move 1")
for _k in (1, 2, 3, 5, 9, 16):
    REQUIRED[f"moves_runs_{_k}"] = _all(f"move 32 from {_k} runs", "move 1 from 1 runs",
                                         f"runs {_k}: {S.lanes_per_run(_k)} lanes per run, {32 // S.lanes_per_run(_k) - _k} idle groups")
REQUIRED.update({"spill_33_one_run": _all("move 33 from 1 runs"), "spill_33_three_runs": _all("move 33 from 3 runs"),
                 "straddle_plain_33": _all("plain key moved 33"), "group_65": _all("SingleDelete keys of 65 versions"),
                 "runs_17": _all("runs 17: more than 16")})
REFUSED_FOR = {"spill_33_one_run": "spill", "spill_33_three_runs": "spill", "straddle_plain_33": "spill", "group_65": "group",
               "runs_17": "runs"}


@pytest.mark.parametrize("name", sorted(S.CASES) + sorted(S.REFUSED))
def test_case_sits_on_its_edge(name):
    e = S.expected(name)
    c = census(e)
    print(f"\n{name}: {len(e['order'])} entries, {len(e['runs'])} runs, tiles {S.tile_sizes(e['cuts'])}")
    for k in sorted(c):
        print(f"    {k}: {c[k]}")
    why = S.refusals(e["order"], len(e["runs"]))
    if name in S.REFUSED:
        assert why == [REFUSED_FOR[name]], why
        twin = S.expected(name + "_minus_one")
        assert sum(map(len, twin["runs"])) == sum(map(len, e["runs"])) - 1 and not S.refusals(twin["order"], len(twin["runs"]))
    else:
        assert why == [], why
        assert e["cuts"][-1]["cut"] == len(e["order"]) and all(0 <= x <= S.TILE for x in S.tile_sizes(e["cuts"]))
    if name == "spill_33_three_runs":
        assert sorted(x for b in e["cuts"] for x in b["per_run"] if b["move"] > S.SPILL) == [0, 11, 11, 11]
    if name.startswith("empty_last_tile"):
        assert S.tile_sizes(e["cuts"])[-1] == 0 and len(e["order"]) % N == int(name.split("_r")[1])
    if name.startswith("sd_filter"):
        assert e["stats"].num_record_drop_user > 0
    missing = REQUIRED.get(name, lambda c: [])(c)
    assert not missing, (missing, dict(c))


def test_the_cases_cover_every_move_size_and_tile_shape():
    total = collections.Counter()
    for name in S.CASES:
        total.update(census(S.expected(name)))
    print("\nall cases:", dict(sorted(total.items())))
    for k in [f"move {m}" for m in (1, 2, 16, 31, 32)] + ["tiles of kMergeTile", "empty tiles", "SingleDelete keys of 64 versions"]:
        assert total[k] >= 1, k
    assert {S.lanes_per_run(k) for k in (1, 2, 3, 5, 9, 16)} == {16, 8, 4, 2}


@pytest.mark.parametrize("sms", [132, 114])
def test_chunked_boundaries_move_as_the_second_of_a_chunk(sms):
    """case 10 at the size where launch_merge_partition gives each warp two boundaries (H100 SXM: 132 SMs, H100 PCIe: 114)"""
    L = S.chunked_layout(sms)
    cuts = S.chunked_cuts(L)
    chunk = S.chunk_of(L["ntiles"], sms)
    assert chunk == 2 and S.chunk_of(L["ntiles"] - 64 - 1, sms) == 1
    moves = {b["b"]: b["move"] for b in cuts}
    assert {b: m for b, m in moves.items() if m} == {b: m for b, m in L["planned"].items() if m}
    c = collections.Counter()
    for b in cuts[1:-1]:
        pos = "second" if b["b"] % chunk == 1 else "first"
        c[f"{pos} of a chunk, move {b['move'] if b['move'] in (0, 1, S.SPILL) else 'other'}"] += 1
        nxt = cuts[b["b"] + 1]
        if b["move"] and nxt["move"]:
            c["consecutive moves, " + ("in one chunk" if pos == "first" else "across two chunks")] += 1
        if b["move"] and pos == "first":
            # a warp starts the next boundary's brackets from this cut; they are too short if it kept the split before the move.  That
            # shows when the run that moved also fills the next tile: its adv exceeds the other runs' entries in [cut, next nominal)
            r = max(range(S.CHUNK_RUNS), key=lambda x: b["per_run"][x])
            others = sum(1 for x in range(b["cut"], nxt["nominal"]) if L["run"][x] != r)
            if b["per_run"][r] > others:
                c["moved first boundary whose run fills the rest of the chunk's next tile"] += 1
    print(f"\n{sms} SMs: {L['n']} entries, {L['ntiles']} tiles, chunk {chunk}:", dict(sorted(c.items())))
    for k in ("second of a chunk, move 32", "second of a chunk, move 1", "second of a chunk, move 0", "consecutive moves, in one chunk",
              "consecutive moves, across two chunks", "moved first boundary whose run fills the rest of the chunk's next tile"):
        assert c[k] >= 1, k
    assert S.lanes_per_run(S.CHUNK_RUNS) == 8


@pytest.mark.parametrize("name", sorted(S.CASES))
def test_stage_and_job_expectations_agree(name):
    e = S.expected(name)
    entries = [kv for f in e["files"] for kv in sstfmt.parse_sst(f)["entries"]]
    assert entries == e["records"]
    for k in M.STAGE_STAT_KEYS:
        assert getattr(e["stage_stats"], k) == getattr(e["stats"], k), k
    assert e["stats"].num_input_records == len(e["order"])
    assert [sstfmt.parse_sst(t)["entries"] for t in e["inputs"]] == e["runs"]


@pytest.mark.parametrize("name", S.FLAG_CASES)
def test_the_only_single_delete_sits_on_the_named_decoder_path(name):
    if name == "flag_zlib" and not H.have_ref():
        pytest.skip("oracle/_ref not built (needs /root/reference)")
    c = S.flag_case(name)
    want = {"flag_fast_path": "fast", "flag_slow_path": "slow", "flag_last_block_of_oldest_run": "fast", "flag_zlib": "arena-fast"}[name]
    assert c["path"] == want, c["path"]
    if name == "flag_last_block_of_oldest_run":
        assert c["run"] == len(c["inputs"]) - 1 and c["block"] == c["nblocks"] - 1
    # the SingleDelete changes the output: kept like a Put (what the plain merge variant would do), the records differ
    stream = sorted(((ik, v) for d in c["inputs"] for ik, v in sstfmt.parse_sst(d)["entries"]),
                    key=lambda e: (e[0][:-8], -int.from_bytes(e[0][-8:], "little")))
    as_put = [(ik[:-8] + bytes([M.VALUE]) + ik[-7:], v) if ik[-8] == M.SINGLE_DELETION else (ik, v) for ik, v in stream]
    got, _ = H.oracle_citer(c["params"], H.kvstream(stream))
    plain, _ = H.oracle_citer(c["params"], H.kvstream(as_put))
    assert len(H.parse_kvstream(got)) < len(H.parse_kvstream(plain))
    if c["ref"] is not None:  # the oracle reproduces the reference on the reference-written inputs
        files, _, st = H.oracle_compact(c["params"], c["inputs"])
        assert files == c["ref"]["outputs"]
        for k in H.STAT_KEYS:
            assert getattr(st, k) == c["ref"]["manifest"]["stats"][k], k


@pytest.mark.parametrize("name", [n for n in S.CASES if n.startswith("sd_filter")])
def test_serial_walk_with_filters_matches_the_oracle(sim, name):  # noqa: F811
    """csrc/group_rules.h compiled for the host, over the filtered-head streams with the filter's verdict on each key's newest version"""
    e = S.expected(name)
    p = e["params"]
    stream = [(H.ikey(uk, q, t), v) for uk, q, t, _, v in e["order"]]
    got, cnt = walk_stream(sim, p, stream)
    assert got == e["records"]
    st = e["stage_stats"]
    assert (cnt[0], cnt[1], cnt[3]) == (st.num_records_replaced, st.num_expired_deletion_records, st.num_record_drop_user)
    assert walk_stream.examined_key_bytes == st.total_input_raw_key_bytes
    assert st.num_record_drop_user > 0


def _sd_filter_script(seed, nonbottom):
    """Put / SingleDelete / empty Put over four flushes with snapshots: empty newest Puts over SingleDeletes of older flushes, over
    SingleDelete / Put pairs, SingleDeletes over empty Puts; keys without a SingleDelete take Put / Delete"""
    rnd = random.Random(seed)
    ops = H.Ops()
    if nonbottom:
        for k in (0, 1 << 40):
            ops.put(struct.pack(">QQ", 0, k), b"base")
        ops.flush()
        ops.compact_all_to(6)
    sd_keys = set(rnd.sample(range(1, 800), 400))
    for r in range(4):
        for k in sorted(rnd.sample(range(1, 800), 300)):
            key = struct.pack(">QQ", 0, k)
            x = rnd.random()
            if k in sd_keys:
                if x < 0.35:
                    ops.single_delete(key)
                    if rnd.random() < 0.3:  # Put again in the same flush: an (empty) Put over a SingleDelete
                        ops.put(key, b"" if rnd.random() < 0.5 else rnd.randbytes(8))
                else:
                    ops.put(key, b"" if x < 0.7 else rnd.randbytes(rnd.randint(1, 30)))
            elif x < 0.1:
                ops.delete(key)
            else:
                ops.put(key, b"" if x < 0.4 else rnd.randbytes(rnd.randint(1, 30)))
        ops.flush()
        if r in (0, 2):
            ops.snapshot()
    return ops, dict(target_file_size=24 << 10, filter="remove_empty_value")


@pytest.mark.skipif(not H.have_ref(), reason="oracle/_ref not built (needs /root/reference)")
@pytest.mark.parametrize("nonbottom", [False, True])
@pytest.mark.parametrize("seed", [31, 32])
def test_oracle_matches_the_reference_with_single_deletes_and_a_filter(seed, nonbottom):
    ops, opts = _sd_filter_script(seed, nonbottom)
    ref = H.run_reference(ops, **opts)
    entries = [ik for d in ref["inputs"] for ik, _ in sstfmt.parse_sst(d)["entries"]]
    assert sum(1 for ik in entries if ik[-8] == M.SINGLE_DELETION) > 50
    p = H.params_from_reference(ref)
    assert p.compaction_filter == "remove_empty_value"
    files, metas, st = H.oracle_compact(p, ref["inputs"])
    assert files == ref["outputs"]
    for k in H.STAT_KEYS:  # (the reference's manifest does not report num_record_drop_user)
        assert getattr(st, k) == ref["manifest"]["stats"][k], k
    assert st.num_record_drop_user > 0
    for m, want in zip(metas, ref["manifest"]["outputs"]):
        assert (m.file_size, m.num_entries, m.num_deletions) == (want["size"], want["num_entries"], want["num_deletions"])
