#!/usr/bin/env python
"""Volume images on one GPU: save_bdev_image / load_bdev_image of an 8 GiB volume with 4 KiB blocks, empty, with 1 % of
its granules scattered, and dense, into each directory given (run it on tmpfs and on a local disk).

Per density and directory, the median of 5 calls after a warm-up:
  save / load   the call's time (for save, the stall a guest on the volume sees)
  GB/s          the image's data bytes over the call's time
  scan+pack     the scan and gather kernels of one save, from a torch.profiler trace (CUDA events of the kernels),
                and the scan's share of 3.35 TB/s (it reads every byte of the store once)
The card's name and power limit are read in the same run.
  python tools/image_bench.py /dev/shm /var/tmp"""
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
RUNS = 5


def fill(lib, name, density, rng):
    if density == "empty":
        return
    if density == "dense":
        chunk = rng.integers(1, 256, size=64 << 20, dtype=np.uint8)
        for off in range(0, NB * BS, chunk.size):
            lib.bdev_write_raw(name, off, chunk)
        return
    piece = rng.integers(1, 256, size=BS, dtype=np.uint8)
    for g in rng.choice(NB, size=NB // 100, replace=False):
        lib.bdev_write_raw(name, int(g) * BS, piece)


def kernel_ms(lib, name, path):
    """scan and gather kernel time of one save, from a profiler trace"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        lib.bdev_image_save(name, path)
        torch.cuda.synchronize()
    os.unlink(path)
    out = {"scan": 0.0, "move": 0.0}
    for e in prof.key_averages():
        for k in out:
            if f"oim_image_{k}_kernel" in e.key:
                out[k] += e.device_time_total / 1e3      # us -> ms
    return out


def main():
    import torch
    from oim_b200 import build, lib
    dirs = sys.argv[1:] or [tempfile.gettempdir()]
    build.build()
    torch.zeros(1, device="cuda:0")
    card = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    print(f"{card}, power limit {power}; {NB * BS >> 30} GiB volume, {BS}-byte blocks, median of {RUNS} after a warm-up")
    lib.init([0])
    rng = np.random.default_rng(1)
    try:
        for density in ("empty", "1%", "dense"):
            src = lib.construct_malloc_bdev(NB, BS, name="img-src", device=0)
            dst = lib.construct_malloc_bdev(NB, BS, name="img-dst", device=0)
            try:
                fill(lib, src, density, rng)
                for d in dirs:
                    path = os.path.join(d, f"oim-image-bench-{os.getpid()}.img")
                    save_t, load_t = [], []
                    try:
                        for i in range(RUNS + 1):
                            t0 = time.perf_counter()
                            info = lib.bdev_image_save(src, path)
                            t1 = time.perf_counter()
                            lib.bdev_image_load(dst, path)
                            t2 = time.perf_counter()
                            os.unlink(path)
                            if i:
                                save_t.append(t1 - t0)
                                load_t.append(t2 - t1)
                    except OSError as e:        # e.g. a tmpfs too small for the dense image
                        print(f"{density:>5} {d}: {e}", flush=True)
                        if os.path.exists(path):
                            os.unlink(path)
                        continue
                    assert lib.bdev_digest(dst) == lib.bdev_digest(src)
                    k = kernel_ms(lib, src, path)
                    s, l_ = statistics.median(save_t), statistics.median(load_t)
                    gb = info["data_bytes"] / 1e9
                    print(f"{density:>5} {d}: data {info['data_bytes'] / 2**20:.0f} MiB in {info['nextents']} extents; "
                          f"save {s * 1e3:.1f} ms ({gb / s:.2f} GB/s), load {l_ * 1e3:.1f} ms ({gb / l_:.2f} GB/s); "
                          f"scan {k['scan']:.2f} ms ({NB * BS / (k['scan'] / 1e3) / HBM if k['scan'] else 0:.2f} of 3.35 TB/s), "
                          f"gather {k['move']:.2f} ms", flush=True)
            finally:
                lib.delete_bdev(src)
                lib.delete_bdev(dst)
    finally:
        lib.fini()


if __name__ == "__main__":
    main()
