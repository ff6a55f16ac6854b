"""The merge cases (merge_cases.py) without a GPU: proof that every case sits on the edge it exists for, and that the two oracle
expectations the GPU tests use are one.

 (a) coverage witnesses, computed from the Python-merged order, the snapshot list and the tile size read out of csrc/kernels.h: the
     counts of positions that take the kernel's boundary paths.  If a change of tile size or generator moves the inputs off an edge,
     this file fails -- the GPU test would otherwise pass while testing nothing.  Every assertion message carries the counts.
 (b) H.oracle_citer over the merged stream (the stage expectation) and H.oracle_compact over the built tables (the job expectation)
     give the same records and statistics.

The compiled reference is not run on these cases: its write-script driver writes through the DB, and a flush itself drops the versions
a newer one in the same snapshot stripe hides, so no script yields a run with thousands of same-stripe versions of one key or a
filtered head followed by same-stripe versions in the same run.  The oracle these tests rely on is pinned to the reference by
test_oracle_vs_reference.py, test_oracle_golden.py and the compaction-iterator vectors of test_oracle_kat.py."""
import collections

import pytest

import helpers as H
import merge_cases as M
import sstfmt

N = M.NOMINAL


def _case(name):
    e = M.expected(name)
    return e, e["order"], e["params"].snapshots


def _same_group(order, snaps, a, b):
    return order[a][0] == order[b][0] and M.stripe_index(snaps, order[a][1]) == M.stripe_index(snaps, order[b][1])


def _boundary_groups(order, snaps):
    """[(o, head)]: tile-first positions whose (user key, stripe) group starts in front of the tile, with the group's head position"""
    out = []
    for o in range(N, len(order), N):
        if _same_group(order, snaps, o - 1, o):
            h = o - 1
            while h > 0 and _same_group(order, snaps, h - 1, o):
                h -= 1
            out.append((o, h))
    return out


def _kept(e):
    return {(ik[:-8], int.from_bytes(ik[-8:], "little")) for ik, _ in e["records"]}


@pytest.mark.parametrize("name", ["hot_keys", "hot_keys_nonbottom"])
def test_hot_keys_make_whole_tiles_depend_on_the_tile_in_front(name):
    e, order, snaps = _case(name)
    assert len(snaps) == 20
    groups = [(o, h) for o, h in _boundary_groups(order, snaps) if M.stripe_index(snaps, order[o][1]) != 0]
    heads = collections.Counter(order[h][2] for _, h in groups)
    # tiles that lie inside one user key from their first to their last position
    inside = sum(1 for b in range(N, len(order) - N + 1, N) if order[b - 1][0] == order[b][0] == order[b + N - 1][0])
    hot = collections.Counter(uk for uk, *_ in order).most_common(len(M.HOT_VERSIONS))
    counts = dict(boundary_groups=len(groups), tombstone_heads=heads[M.DELETION], value_heads=heads[M.VALUE], tiles_inside_a_key=inside,
                  hot=sorted(c for _, c in hot), tiles=(len(order) + N - 1) // N)
    assert len(groups) >= 8 and heads[M.DELETION] >= 3 and heads[M.VALUE] >= 3 and inside >= 5, counts
    assert sorted(c for _, c in hot) == sorted(M.HOT_VERSIONS), counts
    for uk, _ in hot:  # many versions per run, in every run; snapshots inside the key's sequence range
        per_run = collections.Counter(r for k, _, _, r, _ in order if k == uk)
        seqs = [q for k, q, *_ in order if k == uk]
        assert len(per_run) == len(e["runs"]) and min(per_run.values()) >= 300, per_run
        assert sum(1 for s in snaps if min(seqs) < s < max(seqs)) >= 18, counts
    # same-stripe followers of a bottommost tombstone newer than the earliest snapshot are stepped over without touching a counter
    silent, head_type = 0, None
    for o in range(len(order)):
        if o == 0 or not _same_group(order, snaps, o - 1, o):
            head_type = order[o][2]
        elif head_type == M.DELETION and M.stripe_index(snaps, order[o][1]) != 0:
            silent += 1
    if e["params"].bottommost_level:
        assert silent >= 1000 and e["stats"].total_input_raw_key_bytes == sum(len(uk) + 8 for uk, *_ in order) - 24 * silent, (silent, counts)
    else:
        assert e["stats"].total_input_raw_key_bytes == sum(len(uk) + 8 for uk, *_ in order)


@pytest.mark.parametrize("name,nsnap", [("snap_edges_15", 15), ("snap_edges_16", 16), ("snap_edges_17", 17), ("snap_edges_40", 40),
                                        ("snap_edges_below_all", 1), ("snap_edges_above_all", 1)])
def test_snap_edges_reach_past_the_cached_snapshots(name, nsnap):
    e, order, snaps = _case(name)
    assert len(snaps) == nsnap and snaps == sorted(snaps)
    idx = [M.stripe_index(snaps, q) for _, q, *_ in order]
    stripe_uncached = sum(1 for i in idx if M.SNAP_CACHE <= i < nsnap)  # the stripe's own snapshot is read from global memory
    prev_uncached = sum(1 for i in idx if i - 1 >= M.SNAP_CACHE)        # ... the one in front of it
    hidden_uncached = sum(1 for o in range(1, len(order)) if idx[o] >= M.SNAP_CACHE and _same_group(order, snaps, o - 1, o))
    counts = dict(stripe_uncached=stripe_uncached, prev_uncached=prev_uncached, hidden_uncached=hidden_uncached, top=max(idx),
                  above_all=sum(1 for i in idx if i == nsnap))
    if nsnap > M.SNAP_CACHE:
        assert stripe_uncached >= 100 and prev_uncached >= 100 and hidden_uncached >= 10, counts
    else:
        assert stripe_uncached == 0 and prev_uncached == 0, counts
    if name == "snap_edges_below_all":
        assert set(idx) == {1}, counts
    elif name == "snap_edges_above_all":
        assert set(idx) == {0}, counts
    else:
        assert counts["above_all"] >= 100 and idx.count(0) >= 100, counts


def test_tombstone_tails_leave_the_tile_unresolved():
    e, order, snaps = _case("tombstone_tails")
    kept = _kept(e)
    outcome = collections.Counter()
    for o, (uk, q, t, _, _) in enumerate(order):
        if t != M.DELETION or q <= snaps[0] or (o > 0 and _same_group(order, snaps, o - 1, o)):
            continue
        si = M.stripe_index(snaps, q)
        end = min((o // N + 1) * N, len(order))
        if all(order[x][0] == uk and order[x][1] > snaps[si - 1] for x in range(o + 1, end)):  # the in-tile scan finds no answer
            later = end < len(order) and order[end][0] == uk
            outcome[("kept" if (uk, (q << 8) | t) in kept else "dropped", "versions behind the tile" if later else "none behind")] += 1
    assert sum(outcome.values()) >= 2 * len(M.TAIL_SHAPES), outcome
    assert outcome[("kept", "versions behind the tile")] >= 6 and outcome[("dropped", "versions behind the tile")] >= 4 and \
        outcome[("dropped", "none behind")] >= 2, outcome
    assert outcome[("kept", "none behind")] == 0, outcome


@pytest.mark.parametrize("kind", ["empty_value", "ttl"])
def test_filtered_heads_straddle_tile_boundaries(kind):
    e, order, snaps = _case("filtered_heads_" + kind)
    p = e["params"]
    seen = collections.Counter()
    for o, h in _boundary_groups(order, snaps):
        uk, q, t, _, v = order[h]
        stale = t == M.VALUE and M.filter_removes(p.compaction_filter, v)
        first = h == 0 or order[h - 1][0] != uk
        where = "earliest stripe" if M.stripe_index(snaps, q) == 0 else "later stripe"
        seen[("turned" if stale and first else "stale but not first" if stale else "not stale", where)] += 1
    assert seen[("turned", "later stripe")] >= 6 and seen[("stale but not first", "later stripe")] >= 6 and \
        seen[("not stale", "later stripe")] >= 2 and seen[("turned", "earliest stripe")] >= 2, seen
    assert e["stats"].num_record_drop_user >= 1000, e["stats"].num_record_drop_user
    if kind == "ttl":  # values shorter than the stamp are in the stream and are left alone
        assert sum(1 for *_, t, _, v in order if t == M.VALUE and 0 < len(v) < 4) >= 100


def test_prefix_ties_occur_between_runs_and_at_tile_boundaries():
    e, order, snaps = _case("prefix_ties")
    pad = lambda k: k.ljust(M.MAX_USER_KEY, b"\x00")  # noqa: E731
    ties = [o for o in range(1, len(order)) if order[o - 1][0] != order[o][0] and pad(order[o - 1][0]) == pad(order[o][0])]
    across = sum(1 for o in ties if order[o - 1][3] != order[o][3])
    at_boundary = sum(1 for o in ties if o % N == 0)
    last_byte = sum(1 for o in range(1, len(order)) if len(order[o][0]) == M.MAX_USER_KEY and order[o - 1][0] != order[o][0] and
                    order[o - 1][0][:-1] == order[o][0][:-1])
    keys = {uk for uk, *_ in order}
    counts = dict(ties=len(ties), across_runs=across, at_tile_boundary=at_boundary, last_byte_only=last_byte, keys=len(keys),
                  tiles=(len(order) + N - 1) // N)
    assert len(ties) >= 1000 and across >= 500 and at_boundary >= 1 and last_byte >= 100, counts
    assert {b"", b"ab", b"ab\x00", b"ab\x00\x00", b"\x00" * M.MAX_USER_KEY} <= keys and max(map(len, keys)) == M.MAX_USER_KEY
    # a tie pair whose first key is hidden-free: both keys survive, so dropping the length from a comparison changes the output
    kept_keys = {uk for uk, _ in _kept(e)}
    assert sum(1 for o in ties if order[o - 1][0] in kept_keys and order[o][0] in kept_keys) >= 500, counts


@pytest.mark.parametrize("name,lens", [("fan_in_16", [1500] * 16), ("fan_in_17", [1400] * 17), ("fan_in_33", [750] * 33),
                                       ("fan_in_64", [400] * 64), ("fan_in_uneven", [1, 63, 200000, 64, 65]),
                                       ("fan_in_disjoint", [3000] * 8)])
def test_fan_in_shapes(name, lens):
    e, order, _ = _case(name)
    stride, max_runs = M._constant("merge.cu", "kPartStride"), M._constant("kernels.h", "kMaxRuns")
    assert [len(r) for r in e["runs"]] == lens and len(lens) <= max_runs
    runs_per_tile = [len({order[x][3] for x in range(b, min(b + N, len(order)))}) for b in range(0, len(order), N)]
    counts = dict(tiles=len(runs_per_tile), fewest_runs_in_a_tile=min(runs_per_tile), most=max(runs_per_tile))
    assert len(runs_per_tile) >= 8, counts
    if name == "fan_in_64":
        assert len(lens) == max_runs
    if name == "fan_in_uneven":  # runs shorter than, as long as and just longer than the partition's sample stride
        assert {1, stride - 1, stride, stride + 1} <= set(lens) and max(lens) == 200000 and max(runs_per_tile) >= 3, counts
    elif name == "fan_in_disjoint":  # no interleaving: a tile takes from one run, or from two where it crosses from a run to the next
        assert max(runs_per_tile) <= 2 and runs_per_tile.count(1) >= 4, counts
        first = [order[b][3] for b in range(0, len(order), N)]
        assert first != sorted(first), first  # the runs' key ranges are not in run order
    else:
        assert min(runs_per_tile) == len(lens), counts  # every tile draws on every run


@pytest.mark.parametrize("name,total", [("tile_sizes_nominal_minus_1", N - 1), ("tile_sizes_nominal", N), ("tile_sizes_nominal_plus_1", N + 1),
                                        ("tile_sizes_two_tiles", 2 * N), ("tile_sizes_one_entry", 1)])
def test_tile_size_totals(name, total):
    e, order, _ = _case(name)
    assert len(order) == total == e["stats"].num_input_records


@pytest.mark.parametrize("name", sorted(M.CASES))
def test_stage_and_job_expectations_agree(name):
    e = M.expected(name)
    entries = [kv for f in e["files"] for kv in sstfmt.parse_sst(f)["entries"]]
    assert len(entries) == len(e["records"])
    assert entries == e["records"]
    for k in M.STAGE_STAT_KEYS:
        assert getattr(e["stage_stats"], k) == getattr(e["stats"], k), k
    assert e["stats"].num_input_records == len(e["order"])
    # the inputs really are what the case describes: the tables decode to the runs
    assert [sstfmt.parse_sst(t)["entries"] for t in e["inputs"][:2]] == e["runs"][:2]
