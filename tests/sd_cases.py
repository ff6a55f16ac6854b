"""Adversarial inputs for the SingleDelete (kTypeSingleDeletion) path of the merge stage (csrc/merge.cu).

When an input holds a SingleDelete (the decoder raises kFlagHasSingleDelete), merge_partition_grouped_kernel moves every tile cut that
would split a user key forward behind that key, by at most kSdSpill entries summed over the runs (more refuses the job), and the kSD
variant of merge_tiles_kernel walks every key that holds a SingleDelete serially (sd_walk_tile: at most kMaxGroup versions, with the
compaction filter's verdict on the newest version).  Jobs with more than 16 runs are refused.  The cases below sit on those edges: moves
of 1 ... 32 entries from one run and spread over up to 16 runs, tiles of exactly kMergeTile entries, an empty last tile, groups of 64 and
65 versions, filtered heads over SingleDeletes, 16 and 17 runs, snapshots beyond the cached sixteen, and -- at the device's size --
boundaries that a partition warp resolves as the second of its chunk.

`build(name) -> (runs, params)` as in merge_cases.py (runs newest first, every one sorted); `moved_cuts` restates the partition rule so
that tests/test_sd_cases_cpu.py can prove each case sits on its edge and the GPU tests can name the boundary and tile of a failure.
Refused jobs (REFUSED) each have an accepted twin, `<name>_minus_one`: the same inputs without one entry."""
import bisect
import functools
import os
import random
import re
import struct

import numpy as np

import helpers as H
import merge_cases as M
from merge_cases import DELETION, NOW, SEQ_HI, SINGLE_DELETION, TTL, VALUE

_CSRC = M._CSRC


def _src(path):
    with open(os.path.join(_CSRC, path)) as f:
        return re.sub(r"\s+", " ", f.read())


TILE = M._constant("kernels.h", "kMergeTile")
SPILL = M._constant("kernels.h", "kSdSpill")
NOMINAL = M.NOMINAL
MAX_GROUP = M._constant("merge.cu", "kMaxGroup")
SNAP_CACHE = M.SNAP_CACHE
assert NOMINAL == TILE - SPILL
# the partition rule restated below (moved_cuts, chunk_of, lanes_per_run); if one of these lines changes, this module must change with it
_PART = _src("merge.cu")
for _p in ("while (lo < nrun && adv <= (uint32_t)kSdSpill) {", "if (tadv > (uint32_t)kSdSpill && lane == 0) atomicOr(err, (uint32_t)kErrGroupTooLong);",
           "if (n > kMaxGroup) { atomicOr(err, (uint32_t)kErrGroupTooLong);", "unsigned warps = (unsigned)(ntiles + 1);",
           "uint32_t chunk = (uint32_t)((warps + wave - 1) / wave);", "if (chunk < 1) chunk = 1;",
           "const uint64_t b0 = ((uint64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * chunk;",
           "uint32_t kp2 = 2; // at most 16 lanes per run while (kp2 < nruns) kp2 <<= 1;",
           "while ((kp2 << (gshift + 1)) <= 32) gshift++;"):
    assert _p in _PART, f"merge.cu no longer contains `{_p}`: restate the partition rule in tests/sd_cases.py"
_m = re.search(r"const unsigned wave = \(unsigned\)sms \* (\d+)u; .*? if \(chunk > (\d+)\) chunk = \2;", _PART)
assert _m, "the chunk rule of launch_merge_partition changed: restate it in tests/sd_cases.py"
WARPS_PER_SM, MAX_CHUNK = int(_m.group(1)), int(_m.group(2))
_m = re.search(r"constexpr uint32_t kPartGroupedMaxRuns = (\d+);", _PART)
assert _m and "if (nruns <= kPartGroupedMaxRuns) { uint32_t kp2 = 2;" in _PART and "SingleDeletes with more than 16 runs stay on the CPU" in _PART
SD_MAX_RUNS = int(_m.group(1))


def chunk_of(ntiles, sms):
    """boundaries per partition warp (launch_merge_partition): warp w resolves boundaries chunk * w ... chunk * w + chunk - 1"""
    wave = sms * WARPS_PER_SM
    return max(1, min(MAX_CHUNK, (ntiles + 1 + wave - 1) // wave))


def lanes_per_run(nruns):
    """lanes of the partition warp that search one run (16, 8, 4, 2 for 1-2, 3-4, 5-8, 9-16 runs); groups past nruns idle"""
    kp2 = 2
    while kp2 < nruns:
        kp2 <<= 1
    return 32 // kp2


def ntiles_of(n):
    return (n + NOMINAL - 1) // NOMINAL


def _moved(n, nruns, ukey_at, run_at):
    out = []
    for b in range(ntiles_of(n) + 1):
        d = min(b * NOMINAL, n)
        e, per = d, [0] * nruns
        if 0 < d < n:
            k = ukey_at(d - 1)
            while e < n and ukey_at(e) == k:
                per[run_at(e)] += 1
                e += 1
        out.append(dict(b=b, nominal=d, cut=e, move=e - d, per_run=per))
    return out


def moved_cuts(order, nruns):
    """the partition in SingleDelete mode: for every tile boundary b = 0 ... ntiles the nominal rank min(b * kMergeNominal, n), the cut
    after the move (behind the last version of the user key that straddles the nominal rank) and the move per run.  Tile t is
    [cut(t), cut(t + 1)).  A move of more than kSdSpill entries refuses the job."""
    return _moved(len(order), nruns, lambda i: order[i][0], lambda i: order[i][3])


def tile_sizes(cuts):
    return [cuts[i + 1]["cut"] - cuts[i]["cut"] for i in range(len(cuts) - 1)]


def tile_of(cuts, pos):
    """the tile that holds merged position pos"""
    return bisect.bisect_right([c["cut"] for c in cuts], pos) - 1


def refusals(order, nruns):
    """why the device refuses the job (empty: it takes it): moves past kSdSpill, SingleDelete keys with more than kMaxGroup versions,
    more than 16 runs"""
    why = []
    if not any(t == SINGLE_DELETION for _, _, t, _, _ in order):
        return why
    if nruns > SD_MAX_RUNS:
        why.append("runs")
    if any(c["move"] > SPILL for c in moved_cuts(order, nruns)):
        why.append("spill")
    i = 0
    while i < len(order):
        j = i
        while j < len(order) and order[j][0] == order[i][0]:
            j += 1
        if j - i > MAX_GROUP and any(order[x][2] == SINGLE_DELETION for x in range(i, j)):
            why.append("group")
            break
        i = j
    return why


# ------------------------------------------------------------------------------------------------ building blocks
def _versions(s, n, sd=True, seqs=None):
    """n versions of one user key, newest first: Put / SingleDelete mixed with at least one SingleDelete in front of the oldest (sd), or
    Put / Delete (not sd: a key that holds both breaks the SingleDelete contract)"""
    seqs = sorted(seqs or (s.seq() for _ in range(n)), reverse=True)
    if sd:
        types = [s.rnd.choice((VALUE, VALUE, SINGLE_DELETION)) for _ in range(n)]
        if SINGLE_DELETION not in types[:max(1, n - 1)]:
            types[s.rnd.randrange(max(1, n - 1))] = SINGLE_DELETION
    else:
        types = [DELETION if s.rnd.random() < 0.1 else VALUE for _ in range(n)]
    return [(q, t, s.value()) for q, t in zip(seqs, types)]


def _spread(n, runs):
    """the runs of n versions dealt over `runs` in turn (32 over 3 runs: 11 + 11 + 10)"""
    return [runs[i % len(runs)] for i in range(n)]


def _straddle(s, b, front, behind, runs, sd=True):
    """a user key with `front` versions in front of nominal boundary b and `behind` versions behind it, those in `runs` (dealt in turn);
    the ones in front go to random runs"""
    s.pad_to(b * NOMINAL - front)
    vs = _versions(s, front + behind, sd)
    s.add(s.key(), [v + (s.rnd.randrange(s.nruns),) for v in vs[:front]] + [v + (r,) for v, r in zip(vs[front:], _spread(behind, runs))])
    return s.keys[-1][0]


def _clean(s, b):
    """no user key straddles nominal boundary b: its cut does not move"""
    s.pad_to(b * NOMINAL)


def _sd_inside(s, n, room=0, sd=True):
    """a SingleDelete key (sd) of n versions that lies inside a tile, with at least `room` ordinary entries in front of it"""
    s.ordinary(room)
    if (s.pos % NOMINAL) + n >= NOMINAL - 4:
        s.pad_to((s.pos // NOMINAL + 1) * NOMINAL + 100)
    s.add(s.key(), _versions(s, n, sd))
    return s.keys[-1][0]


def _params(**kw):
    kw.setdefault("bottommost_level", True)
    kw.setdefault("snapshots", M._even_snapshots(3))
    return M._params(**kw)


def _job(s, **kw):
    return s.runs(), _params(**kw)


# ------------------------------------------------------------------------------------------------ 1. moves
def _moves_one_run():
    """moves of 1, 2, 16, 31 and 32 entries, each from one run; 32 behind an unmoved cut (a 2048-entry tile), behind a 32-entry move
    (2016) and in front of an unmoved cut (1984)"""
    s = M._Stream(9001, 4)
    for b, (move, run) in enumerate([(1, 0), (2, 1), (16, 2), (31, 3), (0, 0), (32, 0), (32, 1), (0, 0), (32, 3)], start=1):
        if move:
            _straddle(s, b, s.rnd.randint(1, 12), move, [run])
        else:
            _clean(s, b)
        s.ordinary(300)
    s.ordinary(700)
    return _job(s)


def _moves_spread():
    """moves spread over 2, 3, 8 and 16 runs"""
    s = M._Stream(9002, 16)
    plan = [(32, 2), (32, 3), (32, 8), (32, 16), (0, 0), (31, 16), (16, 8), (2, 2), (32, 1), (3, 3), (17, 16), (0, 0)]
    for b, (move, k) in enumerate(plan, start=1):
        if move:
            _straddle(s, b, s.rnd.randint(1, 20), move, s.rnd.sample(range(16), k))
        else:
            _clean(s, b)
        _sd_inside(s, s.rnd.randint(2, 30), 200)
    s.ordinary(500)
    return _job(s)


# ------------------------------------------------------------------------------------------------ 2. refused moves (and their twins)
def _spill(seed, nruns, runs, behind):
    s = M._Stream(seed, nruns)
    _sd_inside(s, 10, 400)
    _straddle(s, 1, 5, 20, [0])
    s.ordinary(400)
    key = _straddle(s, 2, 7, behind, runs)
    s.ordinary(900)
    return s, key


def _refuse_spill_one_run():
    s, key = _spill(9003, 3, [1], SPILL + 1)
    return _job(s) + (key,)


def _refuse_spill_three_runs():
    """11 + 11 + 11: no run passes kSdSpill on its own"""
    s, key = _spill(9004, 4, [0, 2, 3], SPILL + 1)
    return _job(s) + (key,)


# ------------------------------------------------------------------------------------------------ 3. moves at every boundary
def _every_boundary(alternate):
    s = M._Stream(9005 + alternate, 5)
    for b in range(1, 10):
        if alternate and b % 2 == 0:
            _clean(s, b)
        else:
            _straddle(s, b, s.rnd.randint(1, 30), SPILL, s.rnd.sample(range(5), s.rnd.randint(1, 3)))
        _sd_inside(s, s.rnd.randint(2, 12), 100)
    s.pad_to(10 * NOMINAL - 50)
    return _job(s)


# ------------------------------------------------------------------------------------------------ 4. empty last tile
def _empty_last_tile(r):
    """n = 3 kMergeNominal + r: the key that straddles boundary 3 owns the last r entries, so the last tile is empty"""
    s = M._Stream(9007 + r, 3)
    _straddle(s, 1, 4, 9, [2])
    _sd_inside(s, 20, 300)
    _straddle(s, 3, s.rnd.randint(1, 40 - r), r, [0, 1, 2])
    return _job(s)


# ------------------------------------------------------------------------------------------------ 5. a straddling key without a SingleDelete
def _straddle_plain(behind):
    """the cut moves behind every user key in SingleDelete mode, not only behind the keys that hold one: the documented cost"""
    s = M._Stream(9009, 4)
    _sd_inside(s, 12, 500)
    _straddle(s, 1, 3, 2, [1])
    s.ordinary(200)
    key = _straddle(s, 2, 10, behind, [0, 3], sd=False)
    s.ordinary(600)
    return s, key


def _refuse_straddle_plain():
    s, key = _straddle_plain(SPILL + 1)
    return _job(s) + (key,)


# ------------------------------------------------------------------------------------------------ 6. group size
def _group_64():
    """a SingleDelete key of exactly kMaxGroup versions inside a tile, one that straddles a nominal cut (32 in front, 32 behind), and a
    plain key of 200 versions (not walked serially)"""
    s = M._Stream(9010, 4)
    _sd_inside(s, MAX_GROUP, 500)
    _sd_inside(s, 200, 300, sd=False)
    _straddle(s, 2, MAX_GROUP // 2, MAX_GROUP - MAX_GROUP // 2, [1, 2])
    _sd_inside(s, MAX_GROUP - 1, 300)
    s.ordinary(600)
    return _job(s)


def _refuse_group_65():
    s = M._Stream(9011, 4)
    key = _sd_inside(s, MAX_GROUP + 1, 700)
    s.ordinary(1500)
    return _job(s) + (key,)


# ------------------------------------------------------------------------------------------------ 7. filtered heads over SingleDeletes
# (user key versions, newest first) whose newest version the compaction filter may remove:
#   same_stripe    stale Put, SingleDelete in the same stripe (and maybe an older Put)
#   older_stripe   stale Put, SingleDelete in an older stripe
#   over_pair      stale Put, SingleDelete, Put
#   sd_newest      SingleDelete, stale Put (the filter looks at the newest version only: it must not apply)
#   plain          a key without a SingleDelete whose only version is stale, in a tile that holds one
FILTER_SHAPES = ("same_stripe", "older_stripe", "over_pair", "sd_newest", "plain")


def _stripe_range(snaps, si):
    return (snaps[si - 1] + 1 if si else 10), (snaps[si] if si < len(snaps) else SEQ_HI - 1)


def _sd_filtered(kind, bottommost):
    rnd = random.Random(9100 + (kind == "ttl") * 2 + bottommost)
    if kind == "remove_empty_value":
        fresh, stale = (lambda: rnd.randbytes(rnd.choice((8, 40)))), (lambda: b"")
    else:  # values shorter than the 4-byte stamp are left alone
        fresh = lambda: rnd.randbytes(rnd.choice((0, 2, 8))) + (struct.pack("<I", NOW - rnd.randint(0, 10)) if rnd.random() < 0.9 else b"")  # noqa: E731
        stale = lambda: rnd.randbytes(rnd.choice((0, 8))) + struct.pack("<I", NOW - TTL - rnd.randint(1, 5000))  # noqa: E731
    s = M._Stream(9100 + bottommost, 5, value=lambda: stale() if rnd.random() < 0.2 else fresh())
    snaps = M._even_snapshots(5)

    def q(si):
        return s.seq(*_stripe_range(snaps, si))
    for rep in range(40):
        for shape in FILTER_SHAPES:
            si = rnd.randrange(6)
            if shape == "same_stripe":
                lo, hi = _stripe_range(snaps, si)
                a = s.seq((lo + hi) // 2, hi + 1)
                vs = [(a, VALUE, stale()), (s.seq(lo, a), SINGLE_DELETION, b"")]
                if rnd.random() < 0.5:
                    vs.append((s.seq(10, vs[1][0]), VALUE, fresh()))
            elif shape == "older_stripe":
                si = max(si, 1)
                vs = [(q(si), VALUE, stale()), (q(rnd.randrange(si)), SINGLE_DELETION, b"")]
            elif shape == "over_pair":
                seqs = sorted((q(rnd.randrange(6)) for _ in range(3)), reverse=True)
                vs = [(seqs[0], VALUE, stale()), (seqs[1], SINGLE_DELETION, b""), (seqs[2], VALUE, fresh())]
            elif shape == "sd_newest":
                seqs = sorted((q(rnd.randrange(6)) for _ in range(2)), reverse=True)
                vs = [(seqs[0], SINGLE_DELETION, b""), (seqs[1], VALUE, stale())]
            else:
                vs = [(q(si), VALUE, stale())]
            if rnd.random() < 0.3 and shape != "plain":  # more history under the head, all Put / SingleDelete
                older = [s.seq(10, min(v[0] for v in vs)) for _ in range(rnd.randint(1, 4))]
                vs += [(x, t, fresh()) for x, t, _ in _versions(s, len(older), seqs=older)]
            b = s.pos // NOMINAL + 1
            if rep % 8 == 7 and b * NOMINAL - s.pos > len(vs):  # now and then the shape straddles a tile boundary: its cut moves
                s.pad_to(b * NOMINAL - rnd.randint(1, len(vs) - 1) if len(vs) > 1 else b * NOMINAL - 1)
            s.add(s.key(), vs)
            s.ordinary(rnd.randint(5, 40))
    s.ordinary(300)
    return s.runs(), _params(bottommost_level=bottommost, snapshots=snaps, compaction_filter=kind, ttl=TTL, now=NOW)




# ------------------------------------------------------------------------------------------------ 8. run counts
def _moves_runs(nruns):
    """moves spread over every run of the job (and over one), for every lane-group width of the partition warp"""
    s = M._Stream(9200 + nruns, nruns)
    for b in range(1, 5):
        runs = list(range(nruns)) if b % 2 else [s.rnd.randrange(nruns)]
        _straddle(s, b, s.rnd.randint(1, 20), [SPILL, max(1, min(SPILL, 2 * nruns)), SPILL - 1, 1][b - 1], runs)
        _sd_inside(s, s.rnd.randint(2, 40), 300)
    s.ordinary(400)
    return _job(s)


def _refuse_runs_17():
    """17 runs: the last one holds a single entry (the twin without it has 16)"""
    s = M._Stream(9217, 16)
    _straddle(s, 1, 10, 16, list(range(16)))
    _sd_inside(s, 30, 300)
    s.ordinary(1500)
    runs, p = _job(s)
    extra = H.ikey(s.key(), s.seq(), VALUE)
    return runs + [[(extra, b"x")]], p, extra[:-8]


# ------------------------------------------------------------------------------------------------ 9. snapshots beyond the cache
def _snaps(n):
    s = M._Stream(9300 + n, 5)
    jitter = SEQ_HI // (n + 1) // 4
    snaps = [q + random.Random(2020 + q).randrange(-jitter, jitter) for q in M._even_snapshots(n)]
    for b in range(1, 8):
        _straddle(s, b, s.rnd.randint(10, 30), s.rnd.randint(1, SPILL), s.rnd.sample(range(5), s.rnd.randint(1, 5)))
        for _ in range(6):
            _sd_inside(s, s.rnd.randint(8, MAX_GROUP), 150)
    s.ordinary(500)
    return _job(s, snapshots=snaps)


# ------------------------------------------------------------------------------------------------ sub-jobs
SUBJOB_VERSIONS = 20


def _subjob_keys():
    """SingleDelete keys of 20 versions that serve as key-range boundaries, and a stretch of plain keys (no SingleDelete)"""
    s = M._Stream(9400, 4)
    for b in range(1, 3):
        _straddle(s, b, 10, 10, [0, 3])
        _sd_inside(s, SUBJOB_VERSIONS, 400)
    s.ordinary(3000)  # plain keys only
    s.add(s.key(), _versions(s, SUBJOB_VERSIONS))
    s.ordinary(800)
    return _job(s)


CASES = {
    "moves_one_run": _moves_one_run,
    "moves_spread": _moves_spread,
    "every_boundary_32": lambda: _every_boundary(False),
    "alternate_32_0": lambda: _every_boundary(True),
    "empty_last_tile_r1": lambda: _empty_last_tile(1),
    "empty_last_tile_r32": lambda: _empty_last_tile(SPILL),
    "straddle_plain_32": lambda: _job(_straddle_plain(SPILL)[0]),
    "group_64": _group_64,
    "sd_filter_empty_value_bottom": lambda: _sd_filtered("remove_empty_value", True),
    "sd_filter_empty_value_nonbottom": lambda: _sd_filtered("remove_empty_value", False),
    "sd_filter_ttl_bottom": lambda: _sd_filtered("ttl", True),
    "sd_filter_ttl_nonbottom": lambda: _sd_filtered("ttl", False),
    **{f"moves_runs_{k}": (lambda k=k: _moves_runs(k)) for k in (1, 2, 3, 5, 9, 16)},
    "snaps_17": lambda: _snaps(SNAP_CACHE + 1),
    "snaps_40": lambda: _snaps(40),
    "subjob_keys": _subjob_keys,
}
# refused jobs: (runs, params, user key of the entry whose removal makes the job acceptable -- its oldest version)
REFUSED = {
    "spill_33_one_run": _refuse_spill_one_run,
    "spill_33_three_runs": _refuse_spill_three_runs,
    "straddle_plain_33": _refuse_straddle_plain,
    "group_65": _refuse_group_65,
    "runs_17": _refuse_runs_17,
}


def _minus_one(runs, ukey):
    """the runs without the oldest version of ukey (an empty run is dropped)"""
    hits = [(struct.unpack("<Q", ik[-8:])[0] >> 8, r, i) for r, run in enumerate(runs) for i, (ik, _) in enumerate(run) if ik[:-8] == ukey]
    _, r, i = min(hits)
    out = [list(run) for run in runs]
    del out[r][i]
    return [run for run in out if run]


for _name, _fn in REFUSED.items():
    CASES[_name + "_minus_one"] = (lambda fn=_fn: (lambda x: (_minus_one(x[0], x[2]), x[1]))(fn()))


def build(name):
    if name in REFUSED:
        return REFUSED[name]()[:2]
    return CASES[name]()


@functools.lru_cache(maxsize=None)
def expected(name):
    """the case with its tables and both oracle expectations (as merge_cases.expected); refused cases carry no expectation"""
    runs, p = build(name)
    order = M.merged_order(runs)
    inputs = M.tables(runs)
    e = dict(runs=runs, params=p, order=order, inputs=inputs, cuts=moved_cuts(order, len(runs)))
    if name in REFUSED:
        return e
    out, stage_stats = H.oracle_citer(p, H.kvstream((H.ikey(uk, q, t), v) for uk, q, t, _, v in order))
    files, metas, stats = H.oracle_compact(p, inputs)
    return dict(e, records=H.parse_kvstream(out), stage_stats=stage_stats, files=files, metas=metas, stats=stats)


def where(e, ukey):
    """'tile t (boundary b moved m)' for the tile that holds ukey's first version -- for failure messages"""
    order, cuts = e["order"], e["cuts"]
    i = bisect.bisect_left([x[0] for x in order], ukey)
    t = tile_of(cuts, i)
    return f"tile {t} of {len(cuts) - 1} [{cuts[t]['cut']}, {cuts[t + 1]['cut']}), boundary {t} moved {cuts[t]['move']}, " \
           f"boundary {t + 1} moved {cuts[t + 1]['move']}"


# ------------------------------------------------------------------------------------------------ 10. chunked boundaries (device size)
CHUNK_RUNS = 3
CHUNK_REGION = 3 * NOMINAL + 17  # runs own long stretches of the key space in turn, so the run a cut moves in fills the next tile
# (move at boundary 2c + off for off = 0, 1, 2, 3): moves on the second boundary of a chunk of two, on consecutive boundaries in one
# chunk and across two chunks
CHUNK_PATTERNS = [(0, 32, 0, 0), (0, 1, 0, 0), (32, 32, 0, 0), (0, 32, 32, 0), (1, 32, 0, 0), (32, 0, 0, 0), (32, 1, 32, 1),
                  (0, 0, 0, 0), (32, 32, 32, 32), (0, 32, 1, 0)]
CHUNK_EVERY = 24  # a pattern every 24 boundaries


def chunked_layout(sms, seed=9500):
    """the merged order of a job large enough that launch_merge_partition gives every warp 2 boundaries on a device with `sms` SMs, as
    numpy columns: key id (a user key per id), seq, type, run, value length; plus the planned moves {boundary: move}"""
    ntiles = sms * WARPS_PER_SM + 64
    assert chunk_of(ntiles, sms) == 2
    n = ntiles * NOMINAL - 1000
    rng = np.random.default_rng(seed)
    kid = np.arange(n, dtype=np.int64)
    seq = rng.integers(1000, 1 << 40, n, dtype=np.int64)
    typ = np.where(rng.random(n) < 0.01, DELETION, np.where(rng.random(n) < 0.01, SINGLE_DELETION, VALUE)).astype(np.uint8)
    region = np.arange(n) // CHUNK_REGION
    run = (region % CHUNK_RUNS).astype(np.uint8)
    mixed = region % 5 == 4  # one stretch in five interleaves all runs
    run[mixed] = rng.integers(0, CHUNK_RUNS, int(mixed.sum()))
    planned = {}
    for p in range(0, ntiles - 8, CHUNK_EVERY):
        pat = CHUNK_PATTERNS[(p // CHUNK_EVERY) % len(CHUNK_PATTERNS)]
        for off, move in enumerate(pat):
            b = p + 2 + off
            planned[b] = move
            if not move:
                continue
            front = int(rng.integers(1, MAX_GROUP - move + 1)) if move < MAX_GROUP else 0
            a, z = b * NOMINAL - front, b * NOMINAL + move
            kid[a:z] = a
            seq[a:z] = int(rng.integers(1 << 41, 1 << 42)) - np.arange(z - a) * 3
            t = np.where(rng.random(z - a) < 0.35, SINGLE_DELETION, VALUE).astype(np.uint8)
            t[0] = SINGLE_DELETION
            typ[a:z] = t
            run[a:z] = run[z]  # the run that holds the entry behind the moved cut
    vlen = np.where((typ == VALUE) & (rng.random(n) < 0.7), 8, 0).astype(np.int64)
    return dict(n=n, ntiles=ntiles, kid=kid, seq=seq, typ=typ, run=run, vlen=vlen, planned=planned, seed=seed)


def chunked_cuts(L):
    kid, run = L["kid"], L["run"]
    return _moved(L["n"], CHUNK_RUNS, lambda i: int(kid[i]), lambda i: int(run[i]))


def _ukeys(kid):
    """16-byte user keys as an (n, 16) uint8 array: big-endian id, then a scrambled word"""
    k = np.empty((len(kid), 2), dtype=">u8")
    k[:, 0] = kid
    k[:, 1] = (kid.astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15)) & np.uint64((1 << 64) - 1)
    return k.view(np.uint8).reshape(-1, 16)


def kv_records(L, sel, values):
    """the kv stream (helpers.kvstream format) of the merged positions `sel` (ascending) with 16-byte user keys"""
    out = []
    for c in range(0, len(sel), 1 << 21):
        s = sel[c:c + (1 << 21)]
        m = len(s)
        rec = np.zeros((m, 40), dtype=np.uint8)
        rec[:, 0:4] = np.array([24], dtype="<u4").view(np.uint8)
        rec[:, 4:8] = L["vlen"][s].astype("<u4").view(np.uint8).reshape(m, 4)
        rec[:, 8:24] = _ukeys(L["kid"][s])
        rec[:, 24:32] = ((L["seq"][s].astype(np.uint64) << np.uint64(8)) | L["typ"][s].astype(np.uint64)).astype("<u8").view(np.uint8).reshape(m, 8)
        rec[:, 32:40] = values[s]
        keep = np.arange(40)[None, :] < (32 + L["vlen"][s])[:, None]
        out.append(rec[keep].tobytes())
    return b"".join(out)


def chunked_job(sms, seed=9500):
    """the layout, its tables (one per run) and the oracle's compaction iterator over the merged stream"""
    L = chunked_layout(sms, seed)
    values = np.random.default_rng(seed + 1).integers(0, 256, (L["n"], 8), dtype=np.uint8)
    p = H.Params(bottommost_level=True, snapshots=[1 << 39, (1 << 41) + (1 << 40)])
    inputs = [H.oracle_build_sst(H.Params(), kv_records(L, np.flatnonzero(L["run"] == r), values)) for r in range(CHUNK_RUNS)]
    out, st = H.oracle_citer(p, kv_records(L, np.arange(L["n"]), values))
    return dict(L, params=p, inputs=inputs, want=out, stage_stats=st)


# ------------------------------------------------------------------------------------------------ the decoder's SingleDelete flag
# kFlagHasSingleDelete alone selects the kSD merge variant; the decoder raises it on its fast path, on its slow path and for inflated
# blocks.  In each job below the job's only SingleDelete lies in a block the decoder takes by the named path, and it changes the
# output (bottommost, no snapshot: it cancels the Put under it, or goes as a dangling tombstone): a path that failed to raise the flag
# would send the job through the plain variant, which keeps a SingleDelete like a Put.
FLAG_CASES = ("flag_fast_path", "flag_slow_path", "flag_last_block_of_oldest_run", "flag_zlib")


def _flag_tables(name):
    import decode_cases as D
    ks = D._Keys(9600 + FLAG_CASES.index(name))
    newer = [ks.entry(0, ks.rnd.choice((0, 8, 24, 40))) for _ in range(700)]
    older = [ks.entry(0, ks.rnd.choice((0, 8, 24, 40))) for _ in range(700)]
    older.sort(key=lambda e: e[0][:-8])
    if name == "flag_last_block_of_oldest_run":  # a dangling SingleDelete behind every other key
        older.append((H.ikey(ks.key(0), ks.seq(), SINGLE_DELETION), b""))
        target, sd_run = older[-1][0], 1
    else:  # the SingleDelete sits in the middle of the newer run, the Put it cancels in the older one
        uk = newer[350][0][:-8]
        put = ks.seq(1000, 1 << 30)
        newer[350] = (H.ikey(uk, ks.seq(1 << 31, 1 << 40), SINGLE_DELETION), b"")
        older.append((H.ikey(uk, put, VALUE), b"cancelled"))
        older.sort(key=lambda e: e[0][:-8])
        target, sd_run = newer[350][0], 0
    ri = 17 if name == "flag_slow_path" else 16
    tables = [H.oracle_build_sst(H.Params(block_restart_interval=ri), H.kvstream(sorted(r, key=lambda e: e[0][:-8]))) for r in (newer, older)]
    return tables, H.Params(bottommost_level=True, max_output_file_size=64 << 10), target, sd_run


def _flag_zlib():
    """written by the reference: three flushes of compressible values; the second one holds the SingleDelete of a key of the first"""
    import decode_cases as D
    rnd = random.Random(9700)
    ops = H.Ops()
    keys = [struct.pack(">QQ", 1, k) for k in sorted(rnd.sample(range(1, 1 << 30), 3000))]
    victim = keys[0::3][400]
    for run in range(3):
        for k in keys[run::3]:
            ops.put(k, D._texty(rnd, rnd.randint(20, 200)))
        if run == 1:
            ops.single_delete(victim)
        ops.flush()
    return H.run_reference(ops, target_file_size=1 << 20, input_compression="zlib"), victim


@functools.lru_cache(maxsize=None)
def flag_case(name):
    """dict(inputs, params, run, block, path, ref): the job, the run and block that hold its only SingleDelete, and the decoder's path
    for that block (decode_cases.table_blocks); ref: the reference's run for the zlib case (needs oracle/_ref)"""
    import decode_cases as D
    ref = None
    if name == "flag_zlib":
        ref, uk = _flag_zlib()
        inputs, p = ref["inputs"], H.params_from_reference(ref)
    else:
        inputs, p, target, _ = _flag_tables(name)
        uk = target[:-8]
    found = [(r, b["index"], b["path"]) for r, data in enumerate(inputs) for b in D.table_blocks(data)
             for k, _ in b["entries"] if k[-8] == SINGLE_DELETION]
    assert len(found) == 1, found
    r, blk, path = found[0]
    return dict(inputs=inputs, params=p, run=r, block=blk, path=path, nblocks=len(D.table_blocks(inputs[r])), ref=ref, ukey=uk)
