"""The inflate cases (inflate_cases.py; their edges are proven by test_inflate_cases_cpu.py) on the device, through the C ABI:
 (a) decode stage, run by run: the decoded entries against the tables' entries, block by block -- a failure names the block, its
     inflated size u, the path (windowed / direct / stored raw) and the pass of the inflate warp that took it;
 (b) the whole job against the reference's outputs, statistics and file metadata, with host-resident and device-resident inputs;
 (c) the refusals (dictionary, patched type bytes, patched sizes, a flipped checksum in a verify warp's second pass) with their error
     codes and no outputs, each next to its accepted twin;
 (d) one option set through the reference DB and the same driver with the B200 executor plugin."""
import os

import pytest

try:  # a fresh box can take minutes to page torch in: do it at collection time, outside any per-test timeout
    import torch  # noqa: F401
except Exception:  # pragma: no cover
    torch = None

import decode_cases as D
import helpers as H
import inflate_cases as I
import sstfmt
import toplingdb_b200 as T

pytestmark = pytest.mark.gpu


def _case(name):
    if not I.have_ref():
        pytest.fail("oracle/_ref/ref_compact_zlib missing: run __graft_entry__.build() where /root/reference exists")
    c = I.case(name)
    if name.startswith("many_blocks"):  # every warp of the grid must take a second pass on this device
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        ncomp = sum(b["ctype"] == 2 for _, b in I.blocks(c["ref"]["inputs"]))
        assert ncomp > 64 * sms, (ncomp, sms)
    return c


def _where(inputs, sms):
    """per run: the decoded entries and, per entry, the block, u, path and inflate-warp pass that produced it"""
    nblk = len(I.blocks(inputs))
    stride = I.inflate_stride(nblk, sms)
    g = 0
    out = []
    for d in inputs:
        cen = I.table_census(d)[0]
        entries, where = [], []
        for b in cen:
            for k, v, _ in sstfmt.block_entries(b["payload"] if b["ctype"] == 2 else sstfmt.read_block(d, (b["off"], b["size"]))[0]):
                entries.append((k, v))
                path = "stored raw" if b["ctype"] != 2 else ("windowed" if b["windowed"] else "direct")
                where.append(dict(block=b["index"], offset=f"- (u {b['u']})", phase=b["off"] % 16,
                                  path=f"{path}, inflate pass {(g + b['index']) // stride + 1}"))
        g += len(cen)
        out.append((entries, where))
    return out


@pytest.mark.parametrize("name", I.CASES)
def test_decode_stage_matches_the_tables(name):
    from gpu_harness import assert_decoded_matches, job_from_params
    c = _case(name)
    p, inputs = c["params"], c["ref"]["inputs"]
    job = job_from_params(p)
    for i, d in enumerate(inputs):
        job.add_input(d, file_number=i)
    job.run(until=1)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for r, (d, (entries, where)) in enumerate(zip(inputs, _where(inputs, sms))):
        kept = set(D.kept_blocks(d, p.range_start, p.range_end))
        sel = [i for i, w in enumerate(where) if w["block"] in kept]
        assert_decoded_matches(job, r, [entries[i] for i in sel], name, [where[i] for i in sel])
    job.close()


def _assert_job(files, metas, st, want, wmetas, wst, label):
    assert [len(f) for f in files] == [len(f) for f in want], label
    for i, (a, b) in enumerate(zip(files, want)):
        assert a == b, f"{label}: output {i} differs at byte {next(j for j in range(len(a)) if a[j] != b[j])}"
    for k in H.STAT_KEYS:
        assert getattr(st, k) == getattr(wst, k), (label, k)
    for i, (m, om) in enumerate(zip(metas, wmetas)):
        assert (m.file_size, m.num_entries, m.num_deletions, m.raw_key_size, m.raw_value_size, m.num_data_blocks, m.smallest_seqno,
                m.largest_seqno) == (om.file_size, om.num_entries, om.num_deletions, om.raw_key_size, om.raw_value_size, om.num_data_blocks,
                                     om.smallest_seqno, om.largest_seqno), (label, i)


@pytest.mark.parametrize("device_inputs", [False, True])
@pytest.mark.parametrize("name", I.CASES)
def test_job_matches_the_reference(name, device_inputs):
    from gpu_harness import run_product
    c = _case(name)
    p, inputs = c["params"], c["ref"]["inputs"]
    want, wmetas, wst = H.oracle_compact(p, inputs)
    if p.range_start is None:
        assert want == c["ref"]["outputs"], name  # (the oracle is the reference on the whole job)
        man = c["ref"]["manifest"]
        assert [(o["size"], o["num_entries"], o["num_deletions"]) for o in man["outputs"]] == \
            [(m.file_size, m.num_entries, m.num_deletions) for m in wmetas], name
    files, metas, st = run_product(p, inputs, device_inputs=device_inputs)
    _assert_job(files, metas, st, want, wmetas, wst, name)


def _refused(p, inputs, code, **extra):
    from gpu_harness import job_from_params
    job = job_from_params(p, **extra)
    for i, d in enumerate(inputs):
        job.add_input(d, level=0, file_number=i)
    with pytest.raises(T.B200cError) as ei:
        job.run()
    assert ei.value.code == getattr(T.native, code), (ei.value.code, str(ei.value))
    with pytest.raises(T.B200cError):
        job.outputs()
    job.close()


def test_dictionary_inputs_are_refused_and_their_twin_runs():
    from gpu_harness import run_product
    c = _case("dict_16k")
    _refused(c["params"], c["ref"]["inputs"], "ERR_NOT_SUPPORTED")
    t = _case("dict_none")
    files, _, _ = run_product(t["params"], t["ref"]["inputs"])
    assert files == t["ref"]["outputs"]


@pytest.mark.parametrize("verify", [1, 0])
@pytest.mark.parametrize("name", sorted(I.REFUSALS))
def test_patched_blocks_are_refused(name, verify):
    from gpu_harness import run_product
    base, what, value, code = I.REFUSALS[name]
    c = _case(base)
    ins, _ = I.patched(base, what, value)
    if what == "checksum" and not verify:  # the stream is intact: without the check the job is the reference's
        files, _, _ = run_product(c["params"], ins, verify_input_checksums=0)
        assert files == c["ref"]["outputs"], name
        return
    _refused(c["params"], ins, code, verify_input_checksums=verify)
    files, _, _ = run_product(c["params"], c["ref"]["inputs"], verify_input_checksums=verify)  # the accepted twin
    assert files == c["ref"]["outputs"], name


def test_reference_db_compacts_through_the_b200_executor():
    if not (os.path.exists(I.REF_ZLIB_BIN) and os.path.exists(I.REF_ZLIB_B200_BIN)):
        pytest.fail("oracle/_ref/ref_compact_zlib(_b200) missing: run __graft_entry__.build() where /root/reference exists")
    c = _case("level9_filtered")
    ops, opts = c["ops"], c["opts"]
    want = H.run_reference(ops, binary=I.REF_ZLIB_BIN, **opts)
    got = H.run_reference(ops, binary=I.REF_ZLIB_B200_BIN, executor="b200", **opts)
    gm, wm = got["manifest"], want["manifest"]
    assert gm["executor"] == "B200Compact" and gm["remote_compact_read_bytes"] > 0
    assert (gm["scan_count"], gm["scan_digest"]) == (wm["scan_count"], wm["scan_digest"])
    assert H.sizes_without_file_number(got["outputs"]) == H.sizes_without_file_number(want["outputs"])
    assert [e for f in got["outputs"] for e in sstfmt.parse_sst(f)["entries"]] == \
        [e for f in want["outputs"] for e in sstfmt.parse_sst(f)["entries"]]
    for k in H.STAT_KEYS:
        assert gm["stats"][k] == wm["stats"][k], k


def test_verification_adds_exactly_the_verify_launch():
    """stats.kernel_launches of a zlib job: verify_input_checksums adds the one launch of the verify kernel and nothing else"""
    from gpu_harness import run_product
    c = _case("level6_default")
    launches = {v: run_product(c["params"], c["ref"]["inputs"], verify_input_checksums=v)[2].kernel_launches for v in (1, 0)}
    assert launches[1] == launches[0] + 1, launches
