"""Register budget of the tensor-core edge kernels (no GPU): compiled for sm_90a with ``-Xptxas -v``, every
``edge_{fwd,bwd}_tc_kernel`` instance runs 512 threads per CTA, so it must fit 128 registers per thread with no spill
stores or loads.  A spill inside the warp-specialised schedules of the <= 64-row tiles costs a local-memory round trip
in every phase that holds rows across a hand-off."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
INSTANCES = [f"edge_{d}_tc_kernel<{r}>" for d in ("fwd", "bwd") for r in (32, 64, 96, 128)]


def _mangled(name):
    d, r = re.fullmatch(r"edge_(fwd|bwd)_tc_kernel<(\d+)>", name).groups()
    return f"_ZN2vb18edge_{d}_tc_kernelILi{r}EEEvNS_10EdgeTcArgsE"


@pytest.mark.skipif(shutil.which(NVCC) is None and not os.path.exists(NVCC), reason="nvcc not available")
def test_edge_tc_kernels_fit_128_registers_without_spills(tmp_path):
    from ai2bmd_b200 import build
    out = subprocess.run([NVCC, "-Xptxas=-v", *build.NVCC_FLAGS, "-o", str(tmp_path / "lib.so"),
                          os.path.join(build.CSRC, "engine.cu")], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-4000:]
    lines = out.stderr.splitlines()
    report = {}
    for i, line in enumerate(lines):
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            info = " ".join(lines[i + 1:i + 5])
            regs = re.search(r"Used (\d+) registers", info)
            spill = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", info)
            report[m.group(1)] = (int(regs.group(1)), int(spill.group(1)), int(spill.group(2)))
    for name in INSTANCES:
        assert _mangled(name) in report, f"{name} not compiled"
        regs, st, ld = report[_mangled(name)]
        assert regs <= 128 and st == 0 and ld == 0, f"{name}: {regs} registers, spill stores {st} B, loads {ld} B"
