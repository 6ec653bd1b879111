"""Check and repair of an 8 GiB mirror with 2 and 4 replicas on one GPU (oimgpu_bdev_mirror_check), a few seeded
differences each.  Each call is timed with CUDA events (the call ends in a synchronise of the stream it runs on) and
reported as bytes read (replicas x range) per second, against the H100 SXM's 3.35 TB/s of HBM3.  A repair call checks
first and then copies the differing blocks, so it reads the same bytes.  Prints the card and its power limit, then one
JSON line per (replicas, mode)."""
import json
import statistics
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, ".")
from oim_b200 import build, lib  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
BS = 4096
NB = (8 << 30) // BS
DIFFS = 16
REPS = 5

print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv"], capture_output=True, text=True).stdout.strip())
build.build()
torch.zeros(1, device="cuda:0")
lib.init([0])
rng = np.random.default_rng(1)


def seed(name, nrep):
    for b in rng.choice(NB, size=DIFFS, replace=False):
        lib.bdev_write_raw(name, int(b) * BS + 100, rng.integers(1, 256, size=8, dtype=np.uint8), replica=int(rng.integers(1, nrep)))


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / 1e3, out


try:
    for nrep in (2, 4):
        name = lib.construct_mirror_bdev(NB, BS, [0] * nrep, name=f"bench{nrep}")
        try:
            lib.mirror_check(name)                     # warm-up: module load, the stream-ordered pool
            for mode in ("check", "repair"):
                secs = []
                for _ in range(REPS):
                    seed(name, nrep)
                    s, res = timed(lambda: lib.mirror_check(name, repair=mode == "repair"))
                    assert res["mismatched_blocks"] > 0 and res["repaired_blocks"] == (res["mismatched_blocks"] if mode == "repair" else 0)
                    secs.append(s)
                    if mode == "check":
                        lib.mirror_check(name, repair=True)
                assert lib.mirror_check(name)["mismatched_blocks"] == 0
                t = statistics.median(secs)
                rate = nrep * NB * BS / t
                print(json.dumps({"replicas": nrep, "mode": mode, "range_gib": NB * BS / 2**30, "median_ms": round(1e3 * t, 2),
                                  "min_ms": round(1e3 * min(secs), 2), "read_tb_per_s": round(rate / 1e12, 3),
                                  "of_hbm_peak": round(rate / HBM_BYTES_PER_S, 3)}))
        finally:
            lib.delete_bdev(name)
finally:
    lib.fini()
