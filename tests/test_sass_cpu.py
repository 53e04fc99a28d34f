"""Static check of the built library (no GPU needed: cuobjdump disassembles the sm_90a cubin in-tree).  The hot kernels must really be
wgmma / TMA / mbarrier code — a build that silently fell back to mma.sync-era code or started spilling would still pass the numerical
tests, only slower."""
import os
import re
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "hr-viton_b200", "libhrviton_sm100.so")
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"

pytestmark = pytest.mark.skipif(not (os.path.exists(SO) and os.path.exists(CUOBJDUMP)), reason="needs the built library and cuobjdump")


@pytest.fixture(scope="module")
def sass():
    out = subprocess.run([CUOBJDUMP, "-sass", SO], capture_output=True, text=True, check=True).stdout
    funcs, cur = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            funcs[cur] = []
        elif cur is not None:
            m = re.search(r"/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", line)
            if m:
                funcs[cur].append(m.group(1))
    return funcs


def _one(funcs, needle, flavour_f16=False):
    names = [n for n in funcs if needle in n and (("hrv_f16" in n) == flavour_f16)]
    assert names, needle
    return names


@pytest.mark.parametrize("f16", [False, True])
def test_conv_kernels_are_wgmma_tma(sass, f16):
    for needle in ("conv_wgmma_kernelILi64", "conv_wgmma_kernelILi128", "conv_wgrad_kernelILi64", "conv_wgrad_kernelILi128"):
        for n in _one(sass, needle, f16):
            ops = sass[n]
            assert any(o.startswith("HGMMA") for o in ops), (n, "no wgmma")
            assert any(o.startswith("UTMALDG") for o in ops), (n, "no TMA tensor load")
            assert any(o.startswith("SYNCS") for o in ops), (n, "no mbarrier")
            assert not any(o.startswith("HMMA") for o in ops), (n, "legacy tensor-core instructions")


def test_no_register_spills():
    out = subprocess.run([CUOBJDUMP, "--dump-resource-usage", SO], capture_output=True, text=True, check=True).stdout
    rows = re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+)", out)
    assert rows, "no resource-usage rows"
    hot = [(f, int(r), int(s)) for f, r, s in rows if re.search(r"conv_(wgmma|wgrad)_kernel", f)]
    assert len(hot) >= 8
    for f, regs, stack in hot:
        assert stack == 0, (f, "stack frame %d B: local-memory spills in a hot kernel" % stack)
        assert regs <= 112, (f, regs)  # 2 CTAs of 288 threads per SM: at most 65536 / 576 registers per thread
