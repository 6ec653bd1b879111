"""The queue kernels' register budget, read from ptxas at compile time (no GPU).

ptxas allocates the parser warp and the mover warps of a queue kernel together: a change in the parser can make
the movers' inner loops spill.  Each of the five queue kernels must stay within 128 registers (OIM_MIN_BLOCKS 2),
a 120-byte stack frame and no spill traffic.
"""
from __future__ import annotations

import os
import re
import subprocess

from oim_b200 import build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
QUEUE_KERNELS = ["oim_lun_queue_kernel", "oim_lun_queue_mirror_kernel", "oim_lun_vring_kernel",
                 "oim_lun_shared_queue_kernel", "oim_lun_shared_queue_mirror_kernel"]


def test_queue_kernels_stay_within_the_register_budget(tmp_path):
    src = os.path.join(ROOT, "oim_b200", "csrc", "lun_kernel.cu")
    r = subprocess.run([build.NVCC, *[f for f in build.FLAGS if f != "-shared"], "-Xptxas", "-v", "-c", src,
                        "-o", str(tmp_path / "lun_kernel.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    for name in QUEUE_KERNELS:
        m = re.search(rf"Function properties for _ZN6oimgpu\d+{name}E\S*\n"
                      r"\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads\n"
                      r"ptxas info\s*: Used (\d+) registers", r.stderr)
        assert m, f"no ptxas report for {name}:\n{r.stderr[-3000:]}"
        stack, stores, loads, regs = map(int, m.groups())
        assert regs <= 128 and stores == 0 and loads == 0 and stack <= 120, (name, m.group(0))
    # #284: a reference bound to null; #177: a variable declared and never used
    diags = re.findall(r"lun_kernel\.cu\(\d+\): warning #(?:284|177)-D: .*", r.stderr)
    assert not diags, "\n".join(diags)
