#!/usr/bin/env python
"""Incremental volume images on one GPU: save_bdev_image_delta / apply_bdev_image_delta of an 8 GiB dense volume with
4 KiB blocks after 0 %, 0.1 %, 1 % and 10 % of its granules changed, next to a full save_bdev_image of the same volume,
into the directory given (default: the temporary directory; run it on tmpfs and on a local disk).

Per change rate, the median of 3 calls, then one more under the profiler:
  save_delta    the call's time: the stall a guest on the volume sees
  apply         the call's time on a copy holding the parent content
  scan          oim_image_delta_scan_kernel's time in one save_delta, from a torch.profiler trace, and its share of
                3.35 TB/s (it reads every byte of the store once)
and once, a full save_bdev_image of the dense volume.  The card's name and power limit are read in the same run.
  python tools/image_delta_bench.py /dev/shm"""
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

NB, BS = 2 << 20, 4096
HBM = 3.35e12
RUNS = 3
RATES = (0.0, 0.001, 0.01, 0.1)


def kernel_ms(fn):
    """device time of the delta kernels during fn(), from a profiler trace"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {"delta_scan": 0.0, "move": 0.0, "delta_zero": 0.0}
    for e in prof.key_averages():
        for k in out:
            if f"oim_image_{k}_kernel" in e.key:
                out[k] += e.device_time_total / 1e3      # us -> ms
    return out


def main():
    import torch
    from oim_b200 import build, lib
    d = (sys.argv[1:] or [tempfile.gettempdir()])[0]
    build.build()
    torch.zeros(1, device="cuda:0")
    card = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    print(f"{card}, power limit {power}; {NB * BS >> 30} GiB dense volume, {BS}-byte blocks, {d}, median of {RUNS}")
    lib.init([0])
    rng = np.random.default_rng(1)
    tag = f"oim-delta-bench-{os.getpid()}"
    paths = []

    def path(name):
        paths.append(os.path.join(d, f"{tag}-{name}"))
        return paths[-1]
    src = lib.construct_malloc_bdev(NB, BS, name="delta-src", device=0)
    dst = lib.construct_malloc_bdev(NB, BS, name="delta-dst", device=0)
    try:
        chunk = rng.integers(1, 256, size=64 << 20, dtype=np.uint8)
        for off in range(0, NB * BS, chunk.size):
            lib.bdev_write_raw(src, off, chunk)
        t0 = time.perf_counter()
        full = lib.bdev_image_save(src, path("full.img"))
        t1 = time.perf_counter()
        print(f"full save_bdev_image (untracked): {full['data_bytes'] >> 20} MiB, {(t1 - t0) * 1e3:.1f} ms", flush=True)
        lib.bdev_image_load(dst, paths[-1])
        lib.bdev_image_track(src)
        t0 = time.perf_counter()
        lib.bdev_image_save(src, path("tracked.img"))
        t1 = time.perf_counter()
        print(f"full save_bdev_image (tracked):   {(t1 - t0) * 1e3:.1f} ms", flush=True)
        for p in paths:
            os.unlink(p)
        paths.clear()
        piece = rng.integers(1, 256, size=BS, dtype=np.uint8)
        for rate in RATES:
            save_t, apply_t, scan, info = [], [], [], None
            for i in range(RUNS + 1):
                for g in rng.choice(NB, size=int(NB * rate), replace=False):
                    piece[:8] = rng.integers(1, 256, size=8, dtype=np.uint8)
                    lib.bdev_write_raw(src, int(g) * BS, piece)
                p = path(f"{rate}-{i}.delta")
                t0 = time.perf_counter()
                if i == RUNS:
                    k = kernel_ms(lambda: lib.bdev_image_save_delta(src, p))
                    scan.append(k["delta_scan"])
                else:
                    info = lib.bdev_image_save_delta(src, p)
                t1 = time.perf_counter()
                lib.bdev_image_apply_delta(dst, p)
                t2 = time.perf_counter()
                os.unlink(p)
                paths.clear()
                if i < RUNS:
                    save_t.append(t1 - t0)
                apply_t.append(t2 - t1)
            assert lib.bdev_digest(dst) == lib.bdev_digest(src)
            s, a = statistics.median(save_t), statistics.median(apply_t)
            print(f"{rate * 100:5.1f} % changed: {info['data_bytes'] / 2**20:.0f} MiB in {info['nextents']} runs; "
                  f"save_delta {s * 1e3:.1f} ms, apply {a * 1e3:.1f} ms; "
                  f"scan {scan[0]:.2f} ms ({NB * BS / (scan[0] / 1e3) / HBM if scan[0] else 0:.2f} of 3.35 TB/s)", flush=True)
    finally:
        for p in paths:
            if os.path.exists(p):
                os.unlink(p)
        lib.delete_bdev(src)
        lib.delete_bdev(dst)
        lib.fini()


if __name__ == "__main__":
    main()
