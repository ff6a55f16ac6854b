"""The B200 executor plugin takes jobs of column families that set the stock fixed-prefix SST partitioner
(SstPartitionerFixedPrefixFactory, read through its registered option "length") and passes the prefix length to the device as
b200c_params::sst_partitioner_prefix_len; WhyLocal() in toplingdb_b200/plugin/b200_compaction_executor.cc decides it from the options
alone, so the routing is checked on the CPU (B200C_PLUGIN_TRACE)."""
import os
import subprocess
import tempfile

import pytest

import helpers as H
import partition_cases as PC
import scenarios as S

pytestmark = pytest.mark.skipif(not os.path.exists(PC.REF_PART_B200_BIN), reason="oracle/_ref/ref_compact_partition_b200 not built")


def _trace(ops, opts):
    with tempfile.TemporaryDirectory(prefix="b200c_route_") as d:
        with open(os.path.join(d, "ops.bin"), "wb") as f:
            f.write(ops.bytes())
        args = [PC.REF_PART_B200_BIN, os.path.join(d, "ops.bin"), os.path.join(d, "w"), "executor=b200"] + [f"{k}={v}" for k, v in opts.items()]
        r = subprocess.run(args, capture_output=True, text=True, env=dict(os.environ, B200C_PLUGIN_TRACE="1"))
        assert r.returncode == 0, r.stderr[-2000:]
    lines = [ln for ln in r.stderr.splitlines() if ln.startswith("B200Compact: job ")]
    assert lines, "the executor factory was never asked"
    return [ln.split(": ", 2)[2] for ln in lines]


@pytest.mark.parametrize("plen", [1, 3, 8, 16, 17])
@pytest.mark.parametrize("case", ["basic", "grandparents", "subcompactions"])
def test_fixed_prefix_partitioner_jobs_are_device_eligible(case, plen):
    ops, opts = PC.SCENARIOS[case]()
    for why in _trace(ops, dict(opts, partitioner_prefix_len=plen)):
        assert why.startswith("device-eligible"), why


def test_cfg3_with_a_partitioner_is_device_eligible():
    ops, opts = S.ALL["cfg3_mini"]()
    for why in _trace(ops, dict(opts, partitioner_prefix_len=4)):
        assert why.startswith("device-eligible"), why
