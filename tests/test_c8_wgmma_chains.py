"""conv_c8_kernel issues each k-step as one wgmma chain: ptxas compiles every instantiation without injecting a
warpgroup.arrive between its wgmma instructions (C7519) and without spilling.

With a k-step shape known only at run time, ptxas keeps the accumulators live across the issue loops and puts a
`warpgroup.arrive` before every wgmma, so each MMA closed its own group. Needs nvcc (no GPU): compiles se_conv_c8.cu for
sm_90a with the library's flags.
"""
import os
import re
import shutil
import subprocess

import pytest

from sketchedit_b200 import build


def _nvcc():
    try:
        nvcc = build._nvcc()
    except RuntimeError:
        return None
    return nvcc if os.path.isabs(nvcc) or shutil.which(nvcc) else None


@pytest.mark.skipif(_nvcc() is None, reason="nvcc not available")
def test_conv_c8_chains_have_no_injected_arrive(tmp_path):
    src = os.path.join(build.CSRC, "se_conv_c8.cu")
    flags = [f for f in build.NVCC_FLAGS if not f.startswith("--use_fast_math")]   # as build.build() compiles
    cmd = [_nvcc()] + flags + ["-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "c8.o")]
    out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert out.returncode == 0, out.stdout
    log = out.stdout
    injected = [l for l in log.splitlines() if "C7519" in l and "conv_c8_kernel" in l]
    assert not injected, "\n".join(injected[:5])
    # "Function properties for <name>" is followed by "... N bytes spill stores, M bytes spill loads"
    spills, fn = {}, None
    for line in log.splitlines():
        m = re.search(r"Function properties for (\w+)", line)
        if m:
            fn = m.group(1)
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and fn and "conv_c8_kernel" in fn:
            spills[fn] = int(m.group(1)) + int(m.group(2))
            fn = None
    assert len(spills) >= 20, log[-2000:]
    assert not [k for k, n in spills.items() if n], spills
