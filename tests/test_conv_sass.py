"""The strip and fused up-sampling convolution kernels issue their wgmma chains asynchronously.

ptxas serialises a chain (each HGMMA followed by its own WARPGROUP.DEPBAR) when it has to move an accumulator
register between two wgmmas: a branch it takes for divergent, a code path merged into the chain, an unrolled
remainder loop, or one accumulator used by wgmmas of two widths (conv_tc.cu, strip_pair_mma). Nothing fails then,
the kernels only run at a fraction of the tensor-core rate, so this reads the compiled library's SASS: every
conv_strip_kernel and conv_up2_kernel must wait for fewer wgmma groups than it issues wgmmas. Needs cuobjdump
from the CUDA toolkit that built the library, no GPU.
"""
import os
import re
import shutil
import subprocess

import pytest

from v2e_b200 import build as _build


def _cuobjdump():
    nvcc = _build._nvcc()
    cand = os.path.join(os.path.dirname(nvcc), "cuobjdump") if os.path.isabs(nvcc) else None
    return cand if cand and os.path.exists(cand) else shutil.which("cuobjdump")


def _counts():
    lib = _build.build()
    tool = _cuobjdump()
    if tool is None:
        pytest.skip("cuobjdump not found")
    sass = subprocess.run([tool, "-sass", lib], check=True, capture_output=True, text=True).stdout
    counts, cur = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1) if ("conv_strip_kernel" in m.group(1) or "conv_up2_kernel" in m.group(1)) else None
            if cur:
                counts[cur] = [0, 0]
            continue
        if cur:
            if "HGMMA" in line:
                counts[cur][0] += 1
            elif "WARPGROUP.DEPBAR" in line:
                counts[cur][1] += 1
    return counts


def test_strip_and_up2_kernels_chain_their_wgmmas():
    counts = _counts()
    assert any("conv_strip_kernel" in k for k in counts) and any("conv_up2_kernel" in k for k in counts)
    serial = {k: v for k, v in counts.items() if v[1] >= v[0] or v[0] == 0}
    assert not serial, "wgmma chains serialised (HGMMA, DEPBAR): %r" % serial
