"""Measure the oimgpu bdev module against the reference's Malloc bdev, both under the reference's own bdev layer.

Three arms, each on one SPDK thread (integration/spdk/bdev_oimgpu_driver.c, perf mode):
  oimgpu          the oimgpu bdev module: store in HBM, one oim_bio_kernel launch per poller tick
  malloc+oimgpu   Malloc bdev on the oimgpu copy engine: store in host memory, one kernel per iovec
  malloc+memcpy   Malloc bdev on SPDK's memcpy engine: the CPU reference
Workloads: 4 KiB random read and random write at queue depth 32 and 128, 128 KiB sequential write at queue depth 32
(what bdevperf users run for small-block IOPS and large-block throughput).  Each runs `--seconds` after a one-second
warm-up, timed with the host clock.  Prints one JSON line, with the GPU's name and power limit read in the same run.

    python tools/bdev_module_bench.py [--seconds 10]
"""
import argparse
import json
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DRIVER = os.path.join(ROOT, "oracle", "_ref", "spdk", "bdev_oimgpu_driver")

ARMS = {"oimgpu": ("oimgpu", {}), "malloc+oimgpu": ("malloc", {}), "malloc+memcpy": ("malloc", {"OIMGPU_COPY_ENGINE": "off"})}
WORKLOADS = [("randread", 4096, 32), ("randread", 4096, 128), ("randwrite", 4096, 32), ("randwrite", 4096, 128),
             ("write", 131072, 32)]


def gpu_info() -> dict:
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True)
    name, limit = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": limit}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=10.0)
    a = ap.parse_args()
    if not os.path.exists(DRIVER):
        raise SystemExit(f"{DRIVER} not built: run __graft_entry__.build() where the reference tree is")
    out = {**gpu_info(), "seconds": a.seconds, "results": []}
    for rw, size, qd in WORKLOADS:
        for arm, (bdev, env) in ARMS.items():
            r = subprocess.run([DRIVER, "--bdev", bdev, "perf", rw, str(size), str(qd), str(a.seconds)],
                               capture_output=True, text=True, env={**os.environ, **env}, timeout=a.seconds + 120)
            if r.returncode != 0:
                raise SystemExit(f"{arm} {rw} {size} qd{qd} failed:\n{r.stdout[-1000:]}{r.stderr[-1000:]}")
            res = json.loads(r.stdout.strip().splitlines()[-1])
            out["results"].append({"arm": arm, "rw": rw, "io_bytes": size, "qd": qd, "iops": round(res["iops"]),
                                   "gbps": round(res["gbps"], 3), "launches": res["launches"]})
    print(json.dumps(out))


if __name__ == "__main__":
    main()
