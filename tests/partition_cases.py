"""Jobs for the fixed-prefix SST partitioner (SstPartitionerFixedPrefixFactory(len): an output file ends in front of every output entry
whose user key, truncated to len bytes, differs from the previous output entry's; SstPartitionerFixedPrefix::ShouldPartition,
db/compaction/sst_partitioner.cc, checked first by CompactionOutputs::ShouldStopBefore, compaction_outputs.cc:231-300).

The CPU checker is `oracle_compact` below, and the reference runs through `run_reference` (oracle/_ref/ref_compact_partition, the
reference driver with the partitioner options, tests/native/ref_compact_partition.cc).  A job's prefix length is the attribute
`sst_partitioner_prefix_len` of its helpers.Params (absent: no partitioner).

Two kinds of jobs:
  - write scripts for the compiled reference (`SCENARIOS`): user keys from a small tree whose prefixes of 1, 2, 3, 8, 15 and 16
    bytes each take a few values, so every prefix length in LENS cuts a different, bounded number of times; plus keys shorter than
    the prefix and the empty key;
  - synthetic single-run jobs (`stream_job`) whose events sit on chosen merged entries, for the device walk's edges."""
import bisect
import copy
import os
import random
import struct

import helpers as H
import sstfmt
from helpers import Ops

LENS = (1, 2, 3, 8, 15, 16, 17)
REF_PART_BIN = os.path.join(H.ROOT, "oracle", "_ref", "ref_compact_partition")
REF_PART_B200_BIN = os.path.join(H.ROOT, "oracle", "_ref", "ref_compact_partition_b200")  # + the B200 executor plugin


def have_ref():
    return os.path.exists(REF_PART_BIN)


def run_reference(ops, plen, binary=None, **opts):
    """helpers.run_reference with NewSstPartitionerFixedPrefixFactory(plen) on the column family; the Params of the result carry plen"""
    return H.run_reference(ops, binary=binary or REF_PART_BIN, partitioner_prefix_len=plen, **opts)


def params_from_reference(ref, plen):
    p = H.params_from_reference(ref)
    p.sst_partitioner_prefix_len = plen
    return p


def output_user_keys(files):
    return [ik[:-8] for f in files for ik, _ in sstfmt.parse_sst(f)["entries"]]


def oracle_compact(p, inputs):
    """helpers.oracle_compact with the fixed-prefix partitioner of p.sst_partitioner_prefix_len.

    The partitioner decides on the output stream, which the cut rules do not change: the job without it gives the output user keys,
    and with them the events.  Each stretch between two events is then the oracle's job clipped to the key range [event key, next
    event key), numbered on from the files in front of it.  That is exactly the partitioned job: a partition cut starts a file with
    nothing flushed, and leaves the grandparent state what a range's first key leaves it (UpdateGrandparentBoundaryInfo has crossed
    every boundary up to the key, GetCurrentKeyGrandparentOverlappedBytes of the key, no boundary counted as switched); the
    compaction iterator keeps no state across user keys, and an event always lies on a user-key change.  Statistics add up over the
    stretches.  No partitioner for L0 outputs (compaction_outputs.cc:793-795)."""
    plen = getattr(p, "sst_partitioner_prefix_len", 0)
    whole = H.oracle_compact(p, inputs)
    if not plen or p.output_level == 0:
        return whole
    ukeys = output_user_keys(whole[0])
    bounds = [ukeys[e] for e in prefix_events(ukeys, plen)]
    if not bounds:
        return whole
    files, metas, st = [], [], H.OrcStats()
    fct = list(p.file_creation_times)
    for a, b in zip([p.range_start] + bounds, bounds + [p.range_end]):
        q = copy.copy(p)
        k = len(files)
        q.range_start, q.range_end = a, b
        q.first_file_number = p.first_file_number + k
        q.file_creation_times = fct[k:] if k < len(fct) else fct[-1:]
        f, m, s = H.oracle_compact(q, inputs)
        files += f
        metas += m
        for name, _ in H.OrcStats._fields_:
            setattr(st, name, getattr(st, name) + getattr(s, name))
    return files, metas, st


def tree_key(rnd):
    return (bytes([rnd.choice(b"abc"), rnd.choice(b"xy"), rnd.choice(b"01")]) +
            rnd.choice([b"\x00" * 5, b"mmmmm", b"\xff\xff\xff\xff\xfe"]) + rnd.choice([b"\x00" * 7, b"ttttttt"]) +
            rnd.choice([b"", b"\x01", b"z"]))


SHORT_KEYS = [b"", b"a", b"ax", b"ax0", b"ax1", b"b", b"by0", b"by0mmmmm", b"cx1\x00\x00\x00\x00\x00"]


def universe(rnd, n):
    return sorted({tree_key(rnd) for _ in range(n)} | set(SHORT_KEYS))


def prefix_events(ukeys, plen):
    """entries e >= 1 of an output stream in front of which the partitioner cuts"""
    return [e for e in range(1, len(ukeys)) if ukeys[e][:plen] != ukeys[e - 1][:plen]] if plen else []


def _runs(ops, rnd, keys, nruns, per_run, vlen, del_frac):
    for _ in range(nruns):
        for k in sorted(rnd.sample(keys, min(per_run, len(keys)))):
            if rnd.random() < del_frac:
                ops.delete(k)
            else:
                ops.put(k, rnd.randbytes(vlen if not callable(vlen) else vlen(rnd)))
        ops.flush()


def basic(seed=31):
    rnd = random.Random(seed)
    ops = Ops()
    _runs(ops, rnd, universe(rnd, 600), 3, 150, lambda r: r.randint(10, 300), 0.1)
    return ops, dict(target_file_size=32 << 10)


def drops_at_prefix_changes(seed=32):
    """bottommost: the first key of every 3-byte prefix group is overwritten (its old version is dropped) or deleted (the tombstone is
    dropped), so the merged input has entries at prefix changes that the output does not: the cut follows the output stream"""
    rnd = random.Random(seed)
    ops = Ops()
    keys = universe(rnd, 600)
    for k in keys:
        ops.put(k, rnd.randbytes(40))
    ops.flush()
    firsts = [k for i, k in enumerate(keys) if i == 0 or k[:3] != keys[i - 1][:3]] + [k for k in keys if len(k) == 16][::5]
    for k in sorted(set(firsts)):
        if rnd.random() < 0.5:
            ops.delete(k)
        else:
            ops.put(k, rnd.randbytes(50))
    ops.flush()
    _runs(ops, rnd, keys, 1, 80, 30, 0.3)
    return ops, dict(target_file_size=64 << 10)


def output_level0(seed=33):
    ops, _ = basic(seed)
    return ops, dict(target_file_size=8 << 10, output_level=0)


def grandparents(seed=34, dynamic=1):
    """DB::CompactRange builds the job: L0 -> L1 with the L2 files (cut small by the set-up compaction) as grandparents"""
    rnd = random.Random(seed)
    ops = Ops()
    keys = universe(rnd, 600)
    for k in keys:
        ops.put(k, rnd.randbytes(400))
    ops.flush()
    ops.compact_all_to(2)
    _runs(ops, rnd, keys, 3, 120, 400, 0.05)
    return ops, dict(mode="range", target_file_size=64 << 10, setup_file_size=16 << 10, dynamic_file_size=dynamic)


def grandparents_static(seed=35):
    return grandparents(seed, dynamic=0)


def subcompactions(seed=36):
    """large values: enough input bytes for GenSubcompactionBoundaries to split the job over few distinct keys"""
    rnd = random.Random(seed)
    ops = Ops()
    _runs(ops, rnd, universe(rnd, 600), 4, 160, 2000, 0.05)
    return ops, dict(target_file_size=64 << 10, max_subcompactions=3)


def bloom(seed=37):
    ops, opts = basic(seed)
    return ops, dict(opts, bloom_bits=10)


def size_meets_partition(seed=38):
    """max_output_file_size of a few blocks: size cuts fall on, and next to, partition events"""
    rnd = random.Random(seed)
    ops = Ops()
    _runs(ops, rnd, universe(rnd, 800), 3, 200, lambda r: r.randint(100, 700), 0.05)
    return ops, dict(target_file_size=6 << 10)


SCENARIOS = dict(basic=basic, drops_at_prefix_changes=drops_at_prefix_changes, output_level0=output_level0, grandparents=grandparents,
                 grandparents_static=grandparents_static, subcompactions=subcompactions, bloom=bloom,
                 size_meets_partition=size_meets_partition)


# ---------------------------------------------------------------- synthetic single-run jobs with events on chosen entries
PLEN = 2  # the prefix is a 2-byte group number: up to 65536 groups


def stream_keys(n, events):
    """n 16-byte user keys in order; entry e starts a new 2-byte prefix exactly when e is in `events`"""
    ev = sorted(events)
    return [struct.pack(">H", bisect.bisect_right(ev, i)) + struct.pack(">Q", i) + b"\0" * 6 for i in range(n)]


def stream_job(n, events, vlen=60, seed=0, **params):
    """one sorted run of n puts (bottommost: the merged output is the input, entry for entry) with partition events at `events`"""
    rnd = random.Random(seed)
    kv = [(H.ikey(k, 1 + i), rnd.randbytes(vlen)) for i, k in enumerate(stream_keys(n, events))]
    inp = H.oracle_build_sst(H.Params(), H.kvstream(kv))
    p = H.Params(output_level=1, bottommost_level=True, file_creation_times=[7, 8, 9], **params)
    p.sst_partitioner_prefix_len = PLEN
    return p, [inp]
