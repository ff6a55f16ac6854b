"""Adversarial inputs for the merge stage (merge_partition_*_kernel, merge_tiles_kernel, merge_sizes_fix_kernel in csrc/merge.cu).

The kernel restates CompactionIterator::NextFromInput (db/compaction/compaction_iterator.cc:475-1087) per merged position, with the
predecessor taken from the tile or from the tile in front, and leaves the tile for three slow paths.  The jobs below are built so
that those pieces decide the result: user keys with thousands of versions (every entry of several consecutive tiles depends on the
tile in front), more snapshots than the kernel caches in shared memory, bottommost tombstones whose older versions lie behind the
end of their tile, compaction-filtered heads of groups that straddle a tile boundary, user keys that tie on the zero-padded 16-byte
prefix, wide and uneven fan-in, and totals at the edges of the tile size.

`build(name) -> (runs, params)`: runs = sorted [(internal key, value)] lists, newest first; a run may hold many versions of one user
key (a flush under snapshots writes that).  Everything is seeded.  The streams are laid out in user-key order, so the merged position
of every version is known while it is placed; tests/test_merge_cases_cpu.py proves from the merged order that each case still sits on
the edge it exists for."""
import bisect
import functools
import os
import random
import re
import struct

import helpers as H

_CSRC = os.path.join(H.ROOT, "toplingdb_b200", "csrc")


def _constant(path, name):
    m = re.search(r"constexpr\s+\w+\s+%s\s*=\s*(\d+)\s*;" % name, open(os.path.join(_CSRC, path)).read())
    assert m, f"{name} not found in {path}"
    return int(m.group(1))


# tiles are cut every kMergeNominal = kMergeTile - kSdSpill merged entries; the first kSnapCache snapshots live in shared memory
assert re.search(r"kMergeNominal\s*=\s*kMergeTile\s*-\s*kSdSpill\s*;", open(os.path.join(_CSRC, "kernels.h")).read())
NOMINAL = _constant("kernels.h", "kMergeTile") - _constant("kernels.h", "kSdSpill")
SNAP_CACHE = _constant("merge.cu", "kSnapCache")
MAX_USER_KEY = 16
SEQ_HI = 1 << 22
TTL, NOW = 1000, 1_000_000
DELETION, VALUE, SINGLE_DELETION = 0, 1, 7
# what the compaction iterator and the whole job count alike.  num_input_records is not among them: the job sums the input files' entry
# counts (UpdateCompactionInputStatsHelper, compaction_job.cc:2383-2396), the iterator counts the entries it stepped on.
STAGE_STAT_KEYS = tuple(k for k in H.STAT_KEYS if k != "num_input_records") + ("num_record_drop_user",)


def stripe_index(snaps, seq):
    """index of the earliest snapshot that sees seq (len(snaps): none does); the snapshot in front of it is the stripe's prev"""
    return bisect.bisect_left(snaps, seq)


def merged_order(runs):
    """[(user key, seq, type, run, value)] in the order the merge produces: user key, newest first, lower run index on a tie"""
    out = []
    for r, run in enumerate(runs):
        for ik, v in run:
            tr = struct.unpack("<Q", ik[-8:])[0]
            out.append((ik[:-8], tr >> 8, tr & 0xff, r, v))
    out.sort(key=lambda e: (e[0], -e[1], e[3]))
    return out


def tables(runs):
    return [H.oracle_build_sst(H.Params(), H.kvstream(r)) for r in runs]


def _params(**kw):
    kw.setdefault("max_output_file_size", 64 << 10)  # a hot key spans files as well as tiles
    kw.setdefault("file_creation_times", [7, 8, 9])
    return H.Params(**kw)


class _Stream:
    """A job laid out in user-key order: `pos` is the merged position of the next version added."""

    def __init__(self, seed, nruns, value=None):
        self.rnd = random.Random(seed)
        self.nruns = nruns
        self.used = set()
        self.keys = []
        self.pos = 0
        self.next_id = 1
        self.value = value or (lambda: self.rnd.randbytes(self.rnd.choice((0, 8, 40))))

    def seq(self, lo=10, hi=SEQ_HI):
        """an unused sequence number in [lo, hi)"""
        while True:
            s = self.rnd.randrange(lo, hi)
            if s not in self.used:
                self.used.add(s)
                return s

    def key(self):
        """the next 16-byte user key: ascending, with both prefix words and the last bytes varying"""
        i = self.next_id
        self.next_id += self.rnd.randint(1, 3)
        return struct.pack(">QQ", i >> 8, ((i & 255) << 56) | ((i * 0x9E3779B97F4A7C15) & ((1 << 56) - 1)))

    def add(self, ukey, versions):
        """versions: [(seq, type, value)] or [(seq, type, value, run)], any order; a version without a run goes to a random one.
        Tombstones (Deletion, SingleDeletion) are stored without a value."""
        assert len(ukey) <= MAX_USER_KEY and (not self.keys or self.keys[-1][0] < ukey)
        vs = sorted(versions, key=lambda v: -v[0])
        assert len({v[0] for v in vs}) == len(vs) and all(v[1] in (DELETION, VALUE, SINGLE_DELETION) for v in vs)
        self.keys.append((ukey, [(v[0], v[1], v[2] if v[1] == VALUE else b"", v[3] if len(v) > 3 else self.rnd.randrange(self.nruns))
                                 for v in vs]))
        self.pos += len(vs)

    def ordinary(self, n, max_versions=3):
        """n entries of ordinary keys: one to max_versions versions each, one in ten a tombstone"""
        while n > 0:
            nv = min(n, self.rnd.randint(1, max_versions))
            self.add(self.key(), [(self.seq(), DELETION if self.rnd.random() < 0.1 else VALUE, self.value()) for _ in range(nv)])
            n -= nv

    def pad_to(self, pos):
        assert pos >= self.pos, (pos, self.pos)
        self.ordinary(pos - self.pos)

    def next_boundary(self, room):
        """the first tile boundary that leaves at least `room` positions for ordinary keys in front of it"""
        return ((self.pos + room) // NOMINAL + 1) * NOMINAL

    def runs(self):
        runs = [[] for _ in range(self.nruns)]
        for ukey, vs in self.keys:  # keys ascending, versions newest first: every run comes out sorted
            for s, t, v, r in vs:
                runs[r].append((H.ikey(ukey, s, t), v))
        return [r for r in runs if r]


def _even_snapshots(n):
    return [SEQ_HI // (n + 1) * (i + 1) for i in range(n)]


# ------------------------------------------------------------------------------------------------ hot keys
HOT_VERSIONS = (7000, 3000, 10000, 4500)


def _hot_keys(bottommost):
    s = _Stream(101, 6)
    snaps = sorted(s.rnd.sample(range(1000, SEQ_HI - 1000), 20))
    flip = 0
    for nver in HOT_VERSIONS:
        s.ordinary(s.rnd.randint(300, 900))
        seqs = sorted((s.seq() for _ in range(nver)), reverse=True)
        types = [DELETION if s.rnd.random() < 0.1 else VALUE for _ in range(nver)]
        # the head of every (key, stripe) group that reaches over a tile boundary is a tombstone and a value in turn: followers of a
        # bottommost tombstone newer than the earliest snapshot are skipped silently, followers of a value count as replaced
        for i in range(1, nver):
            st = stripe_index(snaps, seqs[i])
            if (s.pos + i) % NOMINAL == 0 and stripe_index(snaps, seqs[i - 1]) == st:
                h = i
                while h > 0 and stripe_index(snaps, seqs[h - 1]) == st:
                    h -= 1
                types[h] = flip
                flip ^= 1
        s.add(s.key(), [(q, t, s.rnd.randbytes(s.rnd.choice((0, 8, 40)))) for q, t in zip(seqs, types)])
    s.ordinary(500)
    return s.runs(), _params(bottommost_level=bottommost, snapshots=snaps)


# ------------------------------------------------------------------------------------------------ snapshot counts
def _snap_edges(snapshots):
    s = _Stream(202, 4)
    s.ordinary(20000, max_versions=8)
    if isinstance(snapshots, int):  # jittered around an even spread, so that every stripe, the last one included, holds entries
        jitter = SEQ_HI // (snapshots + 1) // 4
        snapshots = [q + random.Random(2020 + q).randrange(-jitter, jitter) for q in _even_snapshots(snapshots)]
    return s.runs(), _params(bottommost_level=True, snapshots=snapshots)


# ------------------------------------------------------------------------------------------------ tombstones at a tile's end
# what follows a bottommost tombstone that is newer than the earliest snapshot and sits in the last positions of a tile:
#   lead      versions of the key in newer stripes, in front of the tombstone
#   same      versions in the tombstone's own stripe (hidden; the in-tile scan for an older stripe's version runs over them)
#   same_tail how many of them still lie in the tombstone's tile
#   older     a version at or below the stripe's previous snapshot exists (the tombstone stays) or not (it goes)
TAIL_SHAPES = [
    dict(lead=0, same=0, same_tail=0, older=True),
    dict(lead=0, same=3, same_tail=0, older=False),
    dict(lead=0, same=0, same_tail=0, older=False),  # the key's only version
    dict(lead=0, same=5, same_tail=3, older=True),
    dict(lead=2, same=0, same_tail=0, older=True),
    dict(lead=0, same=NOMINAL + 50, same_tail=0, older=True),  # the older version lies two tiles on
    dict(lead=0, same=NOMINAL + 50, same_tail=0, older=False),
    dict(lead=1, same=4, same_tail=2, older=False),
]


def _tombstone_tails():
    s = _Stream(303, 5)
    snaps = _even_snapshots(5)
    for rep in range(2):
        for shape in TAIL_SHAPES:
            si = s.rnd.randint(1, 5 if shape["lead"] == 0 else 4)  # the tombstone's stripe: never the earliest
            lo, hi = snaps[si - 1] + 1, (snaps[si] if si < 5 else SEQ_HI - 1)
            tomb = s.seq((lo + hi) // 2, hi + 1)
            vs = [(s.seq(hi + 1, SEQ_HI), VALUE, s.value()) for _ in range(shape["lead"])]
            vs.append((tomb, DELETION, b""))
            vs += [(s.seq(lo, tomb), VALUE, s.value()) for _ in range(shape["same"])]
            if shape["older"]:
                vs += [(s.seq(10, lo), s.rnd.choice((VALUE, VALUE, DELETION)), s.value()) for _ in range(s.rnd.randint(1, 2))]
            b = s.next_boundary(300)
            s.pad_to(b - 1 - shape["same_tail"] - shape["lead"])  # the tombstone's tile ends with it and its same_tail followers
            s.add(s.key(), vs)
    s.ordinary(400)
    return s.runs(), _params(bottommost_level=True, snapshots=snaps)


# ------------------------------------------------------------------------------------------------ filtered heads
# a (user key, stripe) group that straddles a tile boundary, bottommost, under a compaction filter:
#   newer   an unfiltered version in a newer stripe exists: the group's head is not the key's first version and is NOT turned
#   stale   the head's value is one the filter removes (empty / expired); as the key's first version it becomes a tombstone
#   in_tile versions of the group in front of the boundary (the head among them)
#   behind  versions of the group behind the boundary
#   stripe  0: the earliest stripe (the turned head is an obsolete tombstone), else random among the later ones
HEAD_SHAPES = [
    dict(newer=False, stale=True, in_tile=1, behind=3, stripe=1),
    dict(newer=True, stale=True, in_tile=1, behind=3, stripe=1),
    dict(newer=False, stale=True, in_tile=3, behind=2, stripe=1),
    dict(newer=True, stale=True, in_tile=2, behind=4, stripe=1),
    dict(newer=False, stale=False, in_tile=2, behind=3, stripe=1),
    dict(newer=False, stale=True, in_tile=2, behind=3, stripe=0),
    dict(newer=False, stale=True, in_tile=1, behind=NOMINAL + 30, stripe=1),  # the group covers the whole next tile
    dict(newer=True, stale=True, in_tile=1, behind=NOMINAL + 30, stripe=1),
]


def filter_removes(kind, value):
    """the built-in filters: RemoveEmptyValueCompactionFilter; DBWithTTL's (trailing fixed32 write time + ttl < now)"""
    if kind == "remove_empty_value":
        return len(value) == 0
    return len(value) >= 4 and struct.unpack("<I", value[-4:])[0] + TTL < NOW


def _filtered_heads(kind):
    rnd = random.Random(4040)
    if kind == "remove_empty_value":
        fresh, stale = (lambda: rnd.randbytes(rnd.choice((8, 40)))), (lambda: b"")
    else:  # values shorter than the 4-byte stamp are left alone
        fresh = lambda: rnd.randbytes(rnd.choice((0, 2, 8))) + (struct.pack("<I", NOW - rnd.randint(0, 10)) if rnd.random() < 0.9 else b"")  # noqa: E731
        stale = lambda: rnd.randbytes(rnd.choice((0, 8))) + struct.pack("<I", NOW - TTL - rnd.randint(1, 5000))  # noqa: E731
    s = _Stream(404, 5, value=lambda: stale() if rnd.random() < 0.2 else fresh())
    snaps = _even_snapshots(5)
    for rep in range(2):
        for shape in HEAD_SHAPES:
            si = rnd.randint(1, 4) if shape["stripe"] else 0
            lo, hi = (snaps[si - 1] + 1 if si else 10), snaps[si]
            head = s.seq((lo + hi) // 2, hi + 1)
            vs = [(s.seq(snaps[4] + 1, SEQ_HI), VALUE, fresh())] if shape["newer"] else []
            vs.append((head, VALUE, stale() if shape["stale"] else fresh()))
            vs += [(s.seq(lo, head), VALUE, s.value()) for _ in range(shape["in_tile"] - 1 + shape["behind"])]
            if si and rep:  # the turned head stays only if an older stripe holds a version
                vs.append((s.seq(10, lo), VALUE, fresh()))
            b = s.next_boundary(300)
            s.pad_to(b - shape["in_tile"] - (1 if shape["newer"] else 0))
            s.add(s.key(), vs)
    s.ordinary(400)
    return s.runs(), _params(bottommost_level=True, snapshots=snaps, compaction_filter=kind, ttl=TTL, now=NOW)


# ------------------------------------------------------------------------------------------------ prefix ties
def _prefix_ties():
    s = _Stream(505, 5)
    keys = {b""}
    for _ in range(600):  # k, k + \x00, k + \x00\x00, ... up to 16 bytes: equal zero-padded prefix, different length
        base = bytes(s.rnd.choice(b"\x00\x01ab\xff") for _ in range(s.rnd.randint(1, 9)))
        keys.update(base + b"\x00" * i for i in range(MAX_USER_KEY + 1 - len(base)) if s.rnd.random() < 0.6)
    keys.update((b"ab", b"ab\x00", b"ab\x00\x00", b"\x00" * MAX_USER_KEY))
    for _ in range(40):  # 16-byte keys that differ in the last byte only
        stem = s.rnd.randbytes(MAX_USER_KEY - 1)
        keys.update(stem + bytes([c]) for c in s.rnd.sample(range(256), 4))
    for k in sorted(keys):
        s.add(k, [(s.seq(), DELETION if s.rnd.random() < 0.15 else VALUE, s.value()) for _ in range(s.rnd.randint(1, 6))])
    return s.runs(), _params(bottommost_level=True, snapshots=_even_snapshots(3))


# ------------------------------------------------------------------------------------------------ fan-in
def _sampled_runs(seed, lens, universe, disjoint=False):
    """run r holds lens[r] distinct keys drawn from the universe (disjoint: from its own slice of it, the slices dealt out of key
    order); run 0 is the newest: its sequence numbers lie above those of run 1, and so on"""
    rnd = random.Random(seed)
    band = SEQ_HI // len(lens)
    assert band >= max(lens)
    slices = list(range(len(lens)))
    rnd.shuffle(slices)
    runs = []
    for r, n in enumerate(lens):
        pool = range(universe) if not disjoint else range(slices[r] * universe // len(lens), (slices[r] + 1) * universe // len(lens))
        seqs = rnd.sample(range((len(lens) - 1 - r) * band + 10, (len(lens) - r) * band), n)
        run = []
        for k, q in zip(sorted(rnd.sample(pool, n)), seqs):
            t = DELETION if rnd.random() < 0.1 else VALUE
            run.append((H.ikey(struct.pack(">QQ", k >> 6, (k * 0x9E3779B97F4A7C15) & ((1 << 64) - 1) if k & 1 else k), q, t),
                        b"" if t == DELETION else rnd.randbytes(rnd.choice((0, 8, 40)))))
        run.sort(key=lambda e: e[0][:-8])
        runs.append(run)
    return runs


def _fan_in(lens, disjoint=False):
    universe = max(max(lens) * 3 // 2, sum(lens) // 3) if not disjoint else sum(lens) * 2
    return _sampled_runs(606 + len(lens), lens, universe, disjoint), _params(bottommost_level=True, snapshots=_even_snapshots(3))


# ------------------------------------------------------------------------------------------------ totals at the tile size
def _tile_sizes(total):
    s = _Stream(707, 3 if total >= 3 else 1)
    s.ordinary(total)
    return s.runs(), _params(bottommost_level=True, snapshots=_even_snapshots(2))


CASES = {
    "hot_keys": lambda: _hot_keys(True),
    "hot_keys_nonbottom": lambda: _hot_keys(False),
    "snap_edges_15": lambda: _snap_edges(SNAP_CACHE - 1),
    "snap_edges_16": lambda: _snap_edges(SNAP_CACHE),
    "snap_edges_17": lambda: _snap_edges(SNAP_CACHE + 1),
    "snap_edges_40": lambda: _snap_edges(40),
    "snap_edges_below_all": lambda: _snap_edges([5]),  # one snapshot below every sequence number
    "snap_edges_above_all": lambda: _snap_edges([SEQ_HI + 5]),  # ... and one above every one
    "tombstone_tails": _tombstone_tails,
    "filtered_heads_empty_value": lambda: _filtered_heads("remove_empty_value"),
    "filtered_heads_ttl": lambda: _filtered_heads("ttl"),
    "prefix_ties": _prefix_ties,
    "fan_in_16": lambda: _fan_in([1500] * 16),
    "fan_in_17": lambda: _fan_in([1400] * 17),
    "fan_in_33": lambda: _fan_in([750] * 33),
    "fan_in_64": lambda: _fan_in([400] * 64),
    "fan_in_uneven": lambda: _fan_in([1, 63, 200000, 64, 65]),
    "fan_in_disjoint": lambda: _fan_in([3000] * 8, disjoint=True),
    "tile_sizes_nominal_minus_1": lambda: _tile_sizes(NOMINAL - 1),
    "tile_sizes_nominal": lambda: _tile_sizes(NOMINAL),
    "tile_sizes_nominal_plus_1": lambda: _tile_sizes(NOMINAL + 1),
    "tile_sizes_two_tiles": lambda: _tile_sizes(2 * NOMINAL),
    "tile_sizes_one_entry": lambda: _tile_sizes(1),
}


def build(name):
    return CASES[name]()


@functools.lru_cache(maxsize=None)
def expected(name):
    """the case with its tables and both oracle expectations: the compaction iterator over the merged stream (stage level) and the
    whole job over the tables"""
    runs, p = build(name)
    order = merged_order(runs)
    out, stage_stats = H.oracle_citer(p, H.kvstream((H.ikey(uk, q, t), v) for uk, q, t, _, v in order))
    inputs = tables(runs)
    files, metas, stats = H.oracle_compact(p, inputs)
    return dict(runs=runs, params=p, order=order, inputs=inputs, records=H.parse_kvstream(out), stage_stats=stage_stats, files=files,
                metas=metas, stats=stats)
