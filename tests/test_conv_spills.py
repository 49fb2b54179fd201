"""The wgmma convolution's hot instances must not spill registers: the MMA warpgroups hold up to 128 fp32 accumulators
each (setmaxnreg), and a spill there puts local-memory traffic into the K loop.  Compiles conv_umma.cu for sm_90a with
-Xptxas -v (no GPU needed)."""
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "raft-ncup_b200", "csrc")

# (BN, epilogue class): plain layers, the GRU z|r gates, and the 128-column GRU q gate -- the update block's layers
SPILL_FREE = [(128, 0), (64, 0), (32, 0), (128, 1), (64, 1), (128, 2)]


def _spills(tmp_path):
    from rnc.build import ARCH, nvcc_path
    cmd = [nvcc_path(), *ARCH, "-O3", "-std=c++17", "-lineinfo", "--expt-relaxed-constexpr", "-Xptxas", "-v", "-I",
           os.path.join(ROOT, "include"), "-I", CSRC, "-c", os.path.join(CSRC, "conv_umma.cu"), "-o", str(tmp_path / "c.o")]
    out = subprocess.run(cmd, capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    res, fn = {}, None
    for line in (out.stdout + out.stderr).splitlines():
        m = re.search(r"Function properties for _ZN3rnc4umma16conv_umma_kernelILi(\d+)ELi(\d+)E", line)
        if m:
            fn = (int(m.group(1)), int(m.group(2)))
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and fn is not None:
            res[fn] = (int(m.group(1)), int(m.group(2)))
            fn = None
    return res


def test_update_block_conv_instances_do_not_spill(tmp_path):
    try:
        from rnc.build import nvcc_path
        nvcc_path()
    except RuntimeError:
        pytest.skip("nvcc not available")
    res = _spills(tmp_path)
    assert len(res) == 12, res
    bad = {k: v for k, v in res.items() if k in SPILL_FREE and v != (0, 0)}
    assert not bad, f"conv_umma_kernel<BN, EC> spills (stores, loads bytes): {bad}"
