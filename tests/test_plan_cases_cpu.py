"""The block-cut planner's jobs (tests/plan_cases.py) still reach the branches they are named for: proved from the oracle's output
layout, without a GPU.  The window and launcher conditions restated here are read out of csrc/encode.cu and csrc/api.cu, so a change
to them fails this file rather than silently moving a case off its branch."""
import bisect
import os

import pytest

import helpers as H
import plan_cases as P

ENCODE = open(os.path.join(P._CSRC, "encode.cu")).read()
API = open(os.path.join(P._CSRC, "api.cu")).read()
# build_window's per-class scan; every other restart interval takes the Hillis-Steele scan
assert "if ((R & (R - 1)) == 0 && R <= 32 && kEncThreads % R == 0) {" in ENCODE
# the launcher's choice of the 64-bit window
assert "if (((uint64_t)max_s1 + 64) * (uint64_t)(kW + 1) < (1ull << 32))" in ENCODE
assert "uint64_t hop = (uint64_t)(P.block_size - 1) / std::max<uint32_t>(min_s1, 1) + 3;" in API
assert "if (hop > (uint64_t)kEncHalo) return fail(B200C_ERR_NOT_SUPPORTED" in API


def _job(name):
    p, inputs = P.build(name)
    files, _, _ = H.oracle_compact(p, inputs)
    entries, layout = P.layout(files)
    return p, entries, layout


def _descended_groups(layout, n, events=()):
    """groups the stitch walk descends into: a file ends, a grandparent boundary is crossed or the stream ends on the chain from the
    first block start at or behind the group start to the first one at or behind its end"""
    starts = [b[0] for f in layout for b in f] + [n]
    last = [f[-1][0] + f[-1][1] - 1 for f in layout]
    out = set()
    for g in range((n + P.GROUP - 1) // P.GROUP):
        a = starts[bisect.bisect_left(starts, g * P.GROUP)]
        x = starts[bisect.bisect_left(starts, min((g + 1) * P.GROUP, n))]
        if x >= n or any(a <= y <= x for y in last) or any(a < e <= x for e in events):
            out.add(g)
    return out


@pytest.mark.parametrize("name", ["restart3_dev0", "restart64_dev0", "restart3_dev10"])
def test_restart_cases_take_the_generic_scan(name):
    p, entries, layout = _job(name)
    R = p.block_restart_interval
    assert not ((R & (R - 1)) == 0 and R <= 32), "takes the per-class scan"
    blocks = [b for f in layout for b in f]
    multi = sum(1 for b in blocks if b[1] > R)
    assert multi, "no block holds more than one restart interval"
    # the payload is what CurrentSizeEstimate() said at the flush; under deviation 0 only the size rule cuts (next_block, LIM == 0)
    full = [b[3] >= p.block_size for f in layout for b in f[:-1]]
    if p.block_size_deviation == 0:
        assert all(full)
    else:
        assert not all(full), "BlockAlmostFull never cut a block"
    print(f"{name}: {len(blocks)} blocks, {multi} with several restarts, {len(layout)} files")


@pytest.mark.parametrize("name", ["end_tile_first", "end_tile_last", "end_group_first", "end_inside_group", "last_file_one_entry"])
def test_file_ends_where_the_case_says(name):
    p, entries, layout = _job(name)
    y = P.CASES[name]["end"]
    first = layout[0]
    assert first[-1][:2] == (y, 1) and first[-1][2] >= p.max_output_file_size, "not the size rule's single-entry block"
    assert all(b[1] == first[0][1] for b in first[:-1]), "data blocks of unequal entry counts"
    desc = _descended_groups(layout, len(entries))
    if name == "end_tile_first":
        assert y % P.TILE == 0 and y % P.GROUP != 0
    elif name == "end_tile_last":
        assert y % P.TILE == P.TILE - 1
    elif name == "end_group_first":
        assert y % P.GROUP == 0 and y // P.GROUP - 1 in desc  # the group in front descends: its exit is the file's last entry
    elif name == "end_inside_group":
        g = y // P.GROUP
        assert y % P.TILE and y // P.TILE % (P.GROUP // P.TILE) not in (0, P.GROUP // P.TILE - 1)
        assert g in desc and not desc & set(range(g)), f"groups walked tile by tile: {sorted(desc)}"
    else:
        assert len(layout) == 2 and layout[1] == [(len(entries) - 1, 1, 0, layout[1][0][3])]
    print(f"{name}: file 0 ends on entry {y}; groups descended into {sorted(desc)} of {(len(entries) + P.GROUP - 1) // P.GROUP}")


def test_one_block_files():
    p, entries, layout = _job("one_block_files")
    assert 100 < len(layout) <= P._constant("kernels.h", "kMaxOutFiles")
    for f in layout[:-1]:
        assert len(f) == 2 and f[1][1] == 1, f


@pytest.mark.parametrize("name", ["hc_at_halo", "hc_over_halo"])
def test_candidate_count_at_the_halo(name):
    p, entries, layout = _job(name)
    hc = (p.block_size - 1) // max(P.min_s1(entries), 1) + 3
    assert hc == P.CASES[name]["hc"] and P.CASES[name]["hc"] - P.HALO in (0, 1)
    assert max(b[1] for f in layout for b in f) > P.HALO // 2  # the blocks are as long as the window allows


def test_wide_window():
    p, entries, layout = _job("wide_window")
    prev, mx = b"", 0
    for k, v in entries:
        sh = next((i for i in range(min(len(k), len(prev))) if k[i] != prev[i]), min(len(k), len(prev)))
        mx = max(mx, P.entry_size(sh, len(k), len(v)))
        prev = k
    assert (mx + 64) * (P.WINDOW + 1) >= 1 << 32, "narrow window"


def test_grandparent_events_in_skipped_groups():
    p, entries, layout = _job("gp_in_skipped_groups")
    ukeys = [k[:-8] for k, _ in entries]
    events = set()
    for lo, hi, _ in p.grandparents:
        events |= {bisect.bisect_left(ukeys, lo), bisect.bisect_left(ukeys, hi), bisect.bisect_right(ukeys, hi)}
    assert len(layout) >= 2, "no grandparent cut"
    assert all(f[-1][2] < p.max_output_file_size for f in layout), "a size cut"
    only_gp = _descended_groups(layout, len(entries), events) - _descended_groups(layout, len(entries))
    assert only_gp, "every group with a boundary is walked tile by tile anyway"
    print(f"groups descended into only for a grandparent boundary: {sorted(only_gp)}; {len(layout)} files")
