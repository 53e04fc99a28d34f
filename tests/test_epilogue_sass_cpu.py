"""Static check of the built library (no GPU needed): the forward convolution kernels write their outputs through the staged epilogue,
i.e. with 128-bit global stores, in every instance (N tile 64 / 128; bf16, fp16 and fp32 storage)."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "hr-viton_b200", "libhrviton_sm100.so")
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"

pytestmark = pytest.mark.skipif(not (os.path.exists(SO) and os.path.exists(CUOBJDUMP)), reason="needs the built library and cuobjdump")


def test_conv_kernels_store_16_byte_vectors():
    out = subprocess.run([CUOBJDUMP, "-sass", SO], capture_output=True, text=True, check=True).stdout
    stores, cur = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            if re.search(r"conv_(wgmma|tf32x3)_kernel", cur):
                stores[cur] = 0
        elif cur in stores and re.search(r"\bSTG\.E\.128\b", line):
            stores[cur] += 1
    assert len(stores) == 6, sorted(stores)  # conv_wgmma_kernel<64|128> x (bf16, fp16), conv_tf32x3_kernel<64|128>
    for name, n in stores.items():
        assert n > 0, (name, "no 128-bit global stores")
