"""CPU: what ptxas made of the tensor-core convolution kernel (conv_tc_kernel), read from the built library and the
ptxas log that the build writes next to the objects (no GPU needed).

Every instantiation must keep its wgmma instructions asynchronous: ptxas serialises them (C7510 / C7511 / C7520) when
they sit behind run-time branches, when MMAs of different shapes share accumulator registers on some path, or when the
registers run short - and then waits for each MMA before the next one issues (one WARPGROUP.DEPBAR per HGMMA in the
SASS), which leaves the main loop's multi-stage pipelining without effect.  The plain (TMA) variants also split the
register file between the producer warpgroup and the consumer warpgroups with setmaxnreg: that needs the kernel to
start with 168 registers per thread (2 * 128 * 232 + 128 * 40 of 65 536), and they must not spill."""
import os
import re
import shutil
import subprocess

import pytest

from orientedreppoints_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOG = os.path.join(ROOT, "orientedreppoints_b200", "lib", "obj", "dense_tc.ptxas.log")
# conv_tc_kernel<BN, OUT_F32, DEFORM, ...>
NAME = re.compile(r"conv_tc_kernelILi(\d+)ELb([01])ELb([01])E")


def _log():
    if not os.path.exists(LOG):
        pytest.fail("no ptxas log at %s: build the library first (python -m orientedreppoints_b200.build)" % LOG)
    return open(LOG).read()


def _kernels(log):
    """mangled name -> {'deform', 'regs', 'spill_stores', 'spill_loads'} from the ptxas -v records"""
    out, cur = {}, None
    for line in log.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            cur = m.group(1) if NAME.search(m.group(1)) else None
            if cur:
                out[cur] = {"deform": NAME.search(cur).group(3) == "1"}
            continue
        if cur is None:
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m:
            out[cur]["spill_stores"], out[cur]["spill_loads"] = int(m.group(1)), int(m.group(2))
        m = re.search(r"Used (\d+) registers", line)
        if m:
            out[cur]["regs"] = int(m.group(1))
            cur = None
    return out


def test_every_instantiation_is_reported():
    ks = _kernels(_log())
    assert len(ks) >= 30, sorted(ks)
    assert any(k["deform"] for k in ks.values()) and any(not k["deform"] for k in ks.values())
    for name, k in ks.items():
        assert "regs" in k and "spill_stores" in k, name


def test_no_serialised_wgmma():
    bad = [line for line in _log().splitlines()
           if "wgmma.mma_async instructions are serialized" in line and NAME.search(line)]
    assert not bad, "\n".join(bad)


def test_plain_variants_do_not_spill_and_start_with_168_registers():
    for name, k in _kernels(_log()).items():
        if k["deform"]:
            continue
        assert (k["spill_stores"], k["spill_loads"]) == (0, 0), (name, k)
        assert k["regs"] == 168, (name, k)


def test_sass_keeps_mmas_in_flight():
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    sass = subprocess.run([tool, "-sass", _lib.LIB_PATH], capture_output=True, text=True).stdout
    counts, fn = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            fn = m.group(1) if NAME.search(m.group(1)) else None
            if fn:
                counts[fn] = [0, 0]
            continue
        if fn is None:
            continue
        if "HGMMA" in line:
            counts[fn][0] += 1
        if "WARPGROUP.DEPBAR" in line:
            counts[fn][1] += 1
    for name, (hgmma, depbar) in counts.items():
        # a serialised kernel waits after every MMA (depbar == hgmma); a pipelined one only at stage releases and drains
        assert hgmma >= 12 and 2 * depbar < hgmma, (name, hgmma, depbar)
    assert len(counts) >= 30, sorted(counts)
