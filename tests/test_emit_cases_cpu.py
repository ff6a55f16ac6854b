"""The emit stage's jobs (tests/emit_cases.py) still reach the paths they are named for: proved from the oracle's output layout and
the jobs' inputs, without a GPU.  The constants, the slot formula, the two fit rules and the kernel selection restated here are read
out of csrc/encode.cu (emit_cases), so a change to them fails this file rather than silently moving a case off its path.

Per data block: more than kEmitMaxEntries entries or payload + 53 > slot -> emit_block_warp (in the slot when payload + 21 <= slot,
else in the file image); otherwise the kernel builds it, lane l taking entries [3l, 3l + 3): a group whose values are all <= 32
bytes takes the short-value load, else values of 1..64 bytes the per-lane copy and longer ones the warp-wide copy."""
import collections
import functools

import pytest

import helpers as H
import emit_cases as C

KERNELS = ("staged", "long")


@functools.lru_cache(maxsize=None)
def census(name):
    """every block and value of the case's outputs, tagged with the path the emit stage takes for it"""
    p, (kind, data) = C.build(name)
    files = H.oracle_compact(p, list(data))[0] if kind == "compact" else [H.oracle_build_sst(p, H.kvstream(data))]
    layouts = [C.layout(f) for f in files]
    n = sum(len(b[2]) for lay in layouts for b in lay)
    data_bytes = sum(b[1] + 5 for lay in layouts for b in lay)
    phases = C.arena_phases(data) if kind == "kv" else None
    R, slot = p.block_restart_interval, C.slot_bytes(p.block_size)
    rpath = "mask" if R & (R - 1) == 0 else "divide"
    out = dict(kernel="long" if data_bytes > 64 * n else "staged", n=n, data_bytes=data_bytes, blocks=[], values=[])
    e = 0
    for lay in layouts:
        for off, payload, ents in lay:
            E = len(ents)
            nrest = (E + R - 1) // R
            if E <= C.MAX_ENTRIES and payload + C.FIT_OVER <= slot:
                path = "fast"
            else:
                path = "warp_slot" if payload + 5 + 16 <= slot else "warp_image"
            out["blocks"].append(dict(path=path, E=E, nrest=nrest, payload=payload, dphase=off % 16, rpath=rpath, slot=slot,
                                      fit=payload + C.FIT_OVER - slot, ck=p.checksum))
            for g in range(0, E, C.PER_LANE):
                group = [len(v) for _, v in ents[g:g + C.PER_LANE]]
                for i, vl in enumerate(group):
                    a = phases[e + g + i] if phases else None
                    if path != "fast":
                        how = path
                    elif max(group) <= 32:
                        how = "short"
                    else:
                        how = "lane" if vl <= 64 else "warp_copy"
                    out["values"].append(dict(how=how, vl=vl, a=a, rpath=rpath))
            e += E
    return out


def _of(kernel, prefix=""):
    return [census(n) for n in C.CASES if n.startswith(prefix) and census(n)["kernel"] == kernel]


@pytest.mark.parametrize("name", C.CASES)
def test_case_takes_its_kernel(name):
    c = census(name)
    if name.endswith(KERNELS):
        assert c["kernel"] == name.rsplit("_", 1)[1]
    elif name.startswith("select_"):
        assert c["data_bytes"] == 64 * c["n"] + (name == "select_64n_plus_1")
        assert c["kernel"] == ("long" if name == "select_64n_plus_1" else "staged")
    paths = collections.Counter(b["path"] for b in c["blocks"])
    hows = collections.Counter(v["how"] for v in c["values"])
    print(f"{name}: {c['kernel']} kernel, {c['n']} entries, {c['data_bytes']} data bytes; blocks {dict(paths)}; values {dict(hows)}")


@pytest.mark.parametrize("kernel", KERNELS)
def test_short_values_at_every_phase(kernel):
    vals = [v for c in _of(kernel, "short_") for v in c["values"] if v["how"] == "short"]
    assert {v["vl"] for v in vals} == set(range(33))
    assert {v["a"] for v in vals if v["vl"]} == set(range(16))  # staged: every a & 8, a & 4, a & 3; long: every a & 3
    assert {(v["vl"], v["a"]) for v in vals if v["vl"] in (1, 32)} == {(vl, a) for vl in (1, 32) for a in range(16)}


@pytest.mark.parametrize("kernel", KERNELS)
def test_per_lane_copies(kernel):
    vals = [v for c in _of(kernel, "per_lane_") for v in c["values"] if v["how"] == "lane"]
    assert {v["a"] % 4 for v in vals if v["vl"] > 32} == set(range(4))
    assert any(0 < v["vl"] <= 32 for v in vals), "no short value in a group with a 33-64-byte one"


@pytest.mark.parametrize("kernel", KERNELS)
def test_warp_copies(kernel):
    vals = [v for c in _of(kernel, "warp_") for v in c["values"] if v["how"] == "warp_copy"]
    assert {v["vl"] % 4 for v in vals} == set(range(4)) and {v["a"] % 4 for v in vals} == set(range(4))
    assert {(v["vl"] + 3) // 4 > 128 for v in vals} == {False, True}, "one and two 512-byte passes"
    assert any(v["vl"] >= 128 for v in vals), "no value-length varint of two bytes"


@pytest.mark.parametrize("kernel", KERNELS)
def test_restart_paths(kernel):
    blocks = [b for c in _of(kernel, "restart") for b in c["blocks"] if b["path"] == "fast"]
    for rpath in ("mask", "divide"):
        assert any(b["rpath"] == rpath and b["nrest"] > 1 for b in blocks), rpath
    assert any(b["nrest"] == 1 and b["E"] > 1 for b in blocks), "no block of one restart"
    hows = {v["how"] for c in _of(kernel, "restart") for v in c["values"]}
    assert {"short", "lane", "warp_copy"} <= hows


@pytest.mark.parametrize("kernel", KERNELS)
def test_destination_phases(kernel):
    assert {b["dphase"] for c in _of(kernel) for b in c["blocks"] if b["path"] == "fast"} == set(range(16))


@pytest.mark.parametrize("kernel", KERNELS)
def test_fit_rule(kernel):
    blocks = [b for c in _of(kernel) for b in c["blocks"]]
    assert any(b["E"] == C.MAX_ENTRIES and b["path"] == "fast" for b in blocks)
    assert any(b["E"] == C.MAX_ENTRIES + 1 and b["path"] != "fast" for b in blocks)
    slots = {C.slot_bytes(bs) for bs in C.FIT_BLOCK_SIZES.values()}
    assert C.SLOT_MIN in slots and C.SLOT_MAX in slots and len(slots) == 3
    for slot in slots:
        at = {b["fit"]: b["path"] for b in blocks if b["slot"] == slot and b["E"] <= C.MAX_ENTRIES}
        assert at.get(0) == "fast" and at.get(1) == "warp_slot", f"slot {slot}: {sorted(at.items())[-4:]}"
        print(f"{kernel}: slot {slot}: payload {slot - C.FIT_OVER} -> {at[0]}, payload {slot - C.FIT_OVER + 1} -> {at[1]}")


@pytest.mark.parametrize("kernel", KERNELS)
def test_block_warp_paths(kernel):
    vals = [v for c in _of(kernel, "block_warp_") for v in c["values"]]
    for how in ("warp_slot", "warp_image"):
        for rpath in ("mask", "divide"):
            lens = [v["vl"] for v in vals if v["how"] == how and v["rpath"] == rpath]
            assert any(vl <= 32 for vl in lens) and any(32 < vl <= 64 for vl in lens) and any(vl > 64 for vl in lens), (how, rpath)


@pytest.mark.parametrize("kernel", KERNELS)
def test_checksums(kernel):
    blocks = [b for c in _of(kernel, "checksum_") for b in c["blocks"] if b["path"] == "fast"]
    assert {b["payload"] <= 240 for b in blocks if b["ck"] == "xxh3"} == {False, True}
    assert any(b["ck"] == "crc32c" for b in blocks)


def test_compaction_cases():
    for name in C.CASES:
        if name.startswith("fallback_"):
            assert {"warp_slot", "warp_image"} <= {b["path"] for b in census(name)["blocks"]}, name
        elif name.startswith("small_"):
            assert {b["path"] for b in census(name)["blocks"]} == {"fast"}, name
