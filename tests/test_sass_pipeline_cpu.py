"""The fused forward's wgmma stream is pipelined in the compiled library.

ptxas serialises every wgmma of a kernel (a full WARPGROUP.DEPBAR after each HGMMA) when the code between two of them
calls a function, branches divergently or lacks registers.  This disassembles the built library and checks that each
field_tc_kernel instance and prune_tc_kernel, which runs the same scene trunk, wait with one group still in flight
(gsb0, 0x1) and wait for all groups only rarely (about once per layer), not after every HGMMA.
"""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "object_nerf_b200", "libonerf_sm90.so")


def _cuobjdump():
    exe = shutil.which("cuobjdump")
    if exe is None:
        for home in (os.environ.get("CUDA_HOME"), os.environ.get("CUDA_PATH"), "/usr/local/cuda"):
            cand = os.path.join(home, "bin", "cuobjdump") if home else None
            if cand and os.path.exists(cand):
                return cand
    return exe


def _wait_counts():
    exe = _cuobjdump()
    if exe is None:
        pytest.skip("cuobjdump not found (CUDA toolkit bin/ not on PATH): cannot disassemble the library")
    assert os.path.exists(LIB), f"{LIB} is missing: build the library first (__graft_entry__.build())"
    sass = subprocess.run([exe, "-sass", LIB], check=True, capture_output=True, text=True).stdout
    counts, fn = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            fn = m.group(1) if re.search("field_tc_kernel|prune_tc_kernel", m.group(1)) else None
            if fn:
                counts[fn] = {"hgmma": 0, "wait_all": 0, "wait_one": 0}
            continue
        if fn is None:
            continue
        c = counts[fn]
        if re.search(r"\bHGMMA\.", line):
            c["hgmma"] += 1
        if "WARPGROUP.DEPBAR.LE gsb0, 0x0" in line:
            c["wait_all"] += 1
        if "WARPGROUP.DEPBAR.LE gsb0, 0x1" in line:
            c["wait_one"] += 1
    return counts


def test_field_tc_kernel_wgmma_is_pipelined():
    counts = _wait_counts()
    # field_tc_kernel<VOXEL, DUMP> in {false, true}^2, and prune_tc_kernel
    assert len(counts) == 5, sorted(counts)
    for fn, c in counts.items():
        assert c["hgmma"] > 0, (fn, c)
        assert c["wait_one"] > 0, (fn, c)                  # per-stage waits leave a group in flight
        assert 4 * c["wait_all"] <= c["hgmma"], (fn, c)    # full waits at layer ends, not after every HGMMA
