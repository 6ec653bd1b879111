"""Moving the imported replica of a 2-way mirror to another store (oimgpu_bdev_mirror_replace_remote) at 1 GiB and
8 GiB: the new store is exported by a second process on the same GPU as replica 0, and on a second GPU where there is
one.  Reports, per (placement, size):
- the whole call, timed on the host around it (it returns after a stream synchronise): the stall a guest sees;
- the copy alone: the same copy kernel over the same bytes, from replica 0 to a store of this process on the new
  store's GPU, timed with CUDA events on a session's stream, and its GB/s against the H100 SXM's 3.35 TB/s of HBM3
  (a copy reads and writes every byte, so 2 x size bytes cross HBM on one GPU).
Prints the card and its power limit, then one JSON line per (placement, size)."""
import json
import multiprocessing as mp
import statistics
import subprocess
import sys
import time

sys.path.insert(0, ".")
from oim_b200 import build, lib  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
BS = 4096
REPS = 5


def exporter(conn, device):
    """a second process: two Malloc bdevs of the size asked for on `device`, exported"""
    from oim_b200 import lib as olib
    olib.init([device])
    try:
        while True:
            cmd = conn.recv()
            if cmd[0] == "make":
                nb = cmd[1]
                conn.send([olib.bdev_export_store(olib.construct_malloc_bdev(nb, BS, name=f"x{nb}-{k}", device=device))
                           for k in range(2)])
            elif cmd[0] == "drop":
                for k in range(2):
                    olib.delete_bdev(f"x{cmd[1]}-{k}")
                conn.send("ok")
            else:
                break
    finally:
        olib.fini()


def main():
    print(subprocess.run(["nvidia-smi", "--query-gpu=index,name,power.limit", "--format=csv"], capture_output=True,
                         text=True).stdout.strip())
    build.build()
    import torch
    ngpu = torch.cuda.device_count()
    if ngpu < 1:
        sys.exit("no CUDA device: nothing to measure")
    lib.init(list(range(min(ngpu, 2))))
    ctx = mp.get_context("spawn")
    try:
        for target in range(min(ngpu, 2)):
            conn, child = ctx.Pipe()
            p = ctx.Process(target=exporter, args=(child, target), daemon=True)
            p.start()
            try:
                for gib in (1, 8):
                    nb = (gib << 30) // BS
                    conn.send(("make", nb))
                    ha, hb = conn.recv()
                    name = lib.construct_mirror_bdev_remote(nb, BS, 0, [ha], name=f"bench{gib}")
                    dst = lib.construct_malloc_bdev(nb, BS, name=f"copy{gib}", device=target)
                    lib.construct_vhost_scsi_controller("bench")
                    lib.add_vhost_scsi_lun("bench", 0, name)
                    try:
                        calls, copies = [], []
                        handles = [hb, ha]
                        for k in range(REPS + 1):               # the first of each: warm-up
                            t0 = time.perf_counter()
                            lib.mirror_replace_remote(name, 1, handles[k % 2])
                            t1 = time.perf_counter()
                            if k:
                                calls.append(t1 - t0)
                        src, to = lib.get_bdevs(name)[0]["device_ptr"], lib.get_bdevs(dst)[0]["device_ptr"]
                        with lib.Lun("bench", 0, num_queues=1, queue_size=64) as lun:
                            t = lib.Timer()
                            try:
                                for k in range(REPS + 1):
                                    t.start(lun)
                                    lun.copy(to, src, nb * BS)
                                    t.stop(lun)
                                    ms = t.elapsed_ms()
                                    if k:
                                        copies.append(ms / 1e3)
                            finally:
                                t.close()
                        assert lib.mirror_check(name)["mismatched_blocks"] == 0
                        call, copy = statistics.median(calls), statistics.median(copies)
                        nbytes = nb * BS
                        print(json.dumps({"replica0_gpu": 0, "new_store_gpu": target, "size_gib": gib,
                                          "replace_call_ms": round(1e3 * call, 2), "replace_call_min_ms": round(1e3 * min(calls), 2),
                                          "copy_ms": round(1e3 * copy, 2), "copy_gb_per_s": round(nbytes / copy / 1e9, 1),
                                          "copy_hbm_share": round(2 * nbytes / copy / HBM_BYTES_PER_S, 3) if target == 0 else None}))
                    finally:
                        lib.remove_vhost_scsi_target("bench", 0)
                        lib.remove_vhost_controller("bench")
                        lib.delete_bdev(name)
                        lib.delete_bdev(dst)
                        conn.send(("drop", nb))
                        conn.recv()
            finally:
                conn.send(("quit",))
                p.join(60)
    finally:
        lib.fini()


if __name__ == "__main__":
    main()
