"""Compile-time resources of the persistent conv-stack kernel (csrc/conv_stack.cu), read from the built library with cuobjdump.

Both instantiations run 512 threads at one CTA per SM, so each thread has 128 registers.  The layer loop holds up to 32 activations, a
64 x 64 fp32 accumulator fragment (32 registers) and two sets of A fragments at once; when that does not fit, the overflow goes to local
memory, which the slice loop touches several times per layer.  The layer loops of both instantiations are spill-free.  A small frame
remains: a few kernel-lifetime scalars that the FC head's peak pushes out once per launch and, in the single-slice kernel, part of the
activations held across the statistics exchange between layers.  The bound keeps it that small.
"""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "samplenet_b200", "lib", "libsamplenet_b200.so")
MAX_STACK_BYTES = 32


def _cuobjdump():
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    return exe if os.path.exists(exe) else None


@pytest.mark.skipif(not os.path.exists(LIB), reason="libsamplenet_b200.so has not been built")
@pytest.mark.skipif(_cuobjdump() is None, reason="cuobjdump is not available")
def test_conv_stack_kernel_frames_stay_small():
    out = subprocess.run([_cuobjdump(), "-res-usage", LIB], capture_output=True, text=True, check=True).stdout
    found = {}
    lines = out.splitlines()
    for i, line in enumerate(lines):
        m = re.search(r"Function (_ZN3snb17conv_stack_kernelILb([01])EEE\S*):", line)
        if m:
            res = dict(re.findall(r"(\w+(?:\[\d+\])?):(\d+)", lines[i + 1]))
            found["multi" if m.group(2) == "1" else "single"] = {k: int(v) for k, v in res.items()}
    assert set(found) == {"multi", "single"}, out[:2000]
    for name, res in found.items():
        assert res["REG"] <= 128, (name, res)   # __launch_bounds__(512, 1)
        assert res["STACK"] <= MAX_STACK_BYTES, (name, res)
