"""Check and repair of a mirrored bdev (oimgpu_bdev_mirror_check, oim_b200/csrc/mirror_check.cu; the daemon's
check_mirror_bdev) compared with a numpy model of the contract.

`model_check` states what a check reports: the blocks of the range in which any replica differs from replica 0 by at
least one byte, as runs in LBA order, cut after `max_ranges` runs (then `truncated`), and every differing block
counted.  A repair leaves every replica equal to replica 0 over the blocks the check marked and nowhere else.

CPU: the model on hand-made cases, the kernels' ptxas report, the C ABI's refusals and the daemon's answers without a
GPU.  GPU (one H100, every replica on cuda:0): seeded differences at block sizes 512, 520, 4096 and 4097 with 2-4
replicas, over the whole device and sub-ranges; repair; a check and a repair next to a running resident poller; a
replica another process exports; the refusals; the daemon's method; and one 8 GiB mirror."""
import base64
import errno
import glob
import os
import re
import subprocess
import threading

import numpy as np
import pytest

from oim_b200 import abi, build, lib, traces
from test_daemon_mirror import daemons, rpc  # noqa: F401  (daemons: the daemon fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MAX_RANGES = 64                 # what check_mirror_bdev returns at most


# ---- the model ------------------------------------------------------------------------------------------------

def model_check(replicas, block_size, off, n, max_ranges=MAX_RANGES):
    """replicas: whole stores (uint8 arrays) -> what a check of blocks [off, off + n) reports"""
    st = np.stack([np.asarray(r)[off * block_size:(off + n) * block_size] for r in replicas]).reshape(len(replicas), n, block_size)
    blocks = off + np.nonzero((st[1:] != st[0]).any(axis=(0, 2)))[0]
    runs = []
    for b in blocks.tolist():
        if runs and runs[-1][0] + runs[-1][1] == b:
            runs[-1][1] += 1
        else:
            runs.append([b, 1])
    return {"blocks_checked": n, "mismatched_blocks": len(blocks), "ranges": [tuple(r) for r in runs[:max_ranges]],
            "truncated": len(runs) > max_ranges, "blocks": blocks}


def model_repair(replicas, block_size, blocks):
    for b in blocks:
        for r in replicas[1:]:
            r[b * block_size:(b + 1) * block_size] = replicas[0][b * block_size:(b + 1) * block_size]


def _stores(nrep, nb, bs, fill=7):
    return [np.full(nb * bs, fill, dtype=np.uint8) for _ in range(nrep)]


def test_model_first_and_last_byte_of_a_block():
    bs, nb = 512, 8
    reps = _stores(2, nb, bs)
    reps[1][3 * bs] ^= 1                    # first byte of block 3
    reps[1][5 * bs + bs - 1] ^= 1           # last byte of block 5
    m = model_check(reps, bs, 0, nb)
    assert (m["mismatched_blocks"], m["ranges"], m["truncated"]) == (2, [(3, 1), (5, 1)], False)
    assert model_check(reps, bs, 4, 4)["ranges"] == [(5, 1)]
    assert model_check(reps, bs, 0, 3)["mismatched_blocks"] == 0
    reps[1][4 * bs - 1] ^= 1                # last byte of block 3: blocks 3 and 5 stay two runs, 4 is equal
    assert model_check(reps, bs, 0, nb)["ranges"] == [(3, 1), (5, 1)]
    reps[1][4 * bs] ^= 1                    # first byte of block 4: one run
    assert model_check(reps, bs, 0, nb)["ranges"] == [(3, 3)]


def test_model_vector_straddling_two_520_byte_blocks():
    """the 16-byte vector at bytes 512..527 holds the end of block 0 and the start of block 1 (520): a difference in
    one of its bytes marks exactly the block that owns it"""
    bs, nb = 520, 4
    for pos, want in ((519, [(0, 1)]), (520, [(1, 1)]), (512, [(0, 1)]), (527, [(1, 1)])):
        reps = _stores(2, nb, bs)
        reps[1][pos] ^= 0x80
        assert model_check(reps, bs, 0, nb)["ranges"] == want, pos
    reps = _stores(2, nb, bs)
    reps[1][519] ^= 1
    reps[1][520] ^= 1
    assert model_check(reps, bs, 0, nb)["ranges"] == [(0, 2)]
    assert model_check(reps, bs, 1, 3)["ranges"] == [(1, 1)]


def test_model_one_of_four_replicas_and_the_range_cut():
    bs, nb = 4096, 300
    reps = _stores(4, nb, bs)
    reps[2][10 * bs + 100] = 0
    m = model_check(reps, bs, 0, nb)
    assert (m["mismatched_blocks"], m["ranges"]) == (1, [(10, 1)])
    reps[0][11 * bs] = 1                    # replica 0 differs from all the others
    assert model_check(reps, bs, 0, nb)["ranges"] == [(10, 2)]
    reps = _stores(3, nb, bs)
    for k in range(100):                    # 100 runs of one block, every third block
        reps[1 + k % 2][3 * k * bs] ^= 1
    m = model_check(reps, bs, 0, nb)
    assert (m["mismatched_blocks"], len(m["ranges"]), m["truncated"]) == (100, 64, True)
    assert m["ranges"][-1] == (3 * 63, 1)
    m = model_check(reps, bs, 0, nb, max_ranges=100)
    assert (len(m["ranges"]), m["truncated"]) == (100, False)
    model_repair(reps, bs, m["blocks"])
    assert model_check(reps, bs, 0, nb)["mismatched_blocks"] == 0


# ---- CPU: the kernels, the C ABI and the daemon without a GPU -------------------------------------------------------

def test_mirror_check_kernels_compile_for_sm90a_without_spills(tmp_path):
    src = os.path.join(ROOT, "oim_b200", "csrc", "mirror_check.cu")
    r = subprocess.run([build.NVCC, *[f for f in build.FLAGS if f != "-shared"], "-Xptxas", "-v", "-c", src,
                        "-o", str(tmp_path / "mirror_check.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    for k in ("oim_mirror_check_kernel", "oim_mirror_repair_kernel"):
        m = re.search(rf"Compiling entry function '(\S*{k}\S*)' for 'sm_90a'.*?(\d+) bytes stack frame, (\d+) bytes spill stores, "
                      r"(\d+) bytes spill loads", r.stderr, re.S)
        assert m and m.group(3) == "0" and m.group(4) == "0", (k, r.stderr[-3000:])
    sass = subprocess.run(["/usr/local/cuda/bin/cuobjdump", "-sass", build.build()], capture_output=True, text=True).stdout
    for k in ("oim_mirror_check_kernel", "oim_mirror_repair_kernel"):
        assert re.search(rf"Function : \S*{k}", sass), k


def test_mirror_check_struct_matches_c(tmp_path):
    probe = tmp_path / "probe.c"
    probe.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "oimgpu.h"\n'
                     'int main(void){printf("%zu %zu %zu %zu\\n",sizeof(struct oimgpu_mirror_check),'
                     "offsetof(struct oimgpu_mirror_check,repaired_blocks),offsetof(struct oimgpu_mirror_check,nranges),"
                     "offsetof(struct oimgpu_mirror_check,truncated));return 0;}\n")
    exe = tmp_path / "probe"
    subprocess.run(["cc", "-I", os.path.join(ROOT, "include"), str(probe), "-o", str(exe)], check=True)
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    d = abi.mirror_check_dtype
    assert got == [d.itemsize, d.fields["repaired_blocks"][1], d.fields["nranges"][1], d.fields["truncated"][1]]


def test_mirror_check_abi_without_gpu():
    L = lib.load()
    out = np.zeros(1, dtype=abi.mirror_check_dtype)
    ranges = np.zeros(8, dtype=np.uint64)
    assert L.oimgpu_bdev_mirror_check(b"x", 0, 1, 0, ranges.ctypes.data, 4, None) == -errno.EINVAL
    assert L.oimgpu_bdev_mirror_check(b"x", 0, 1, 0, None, 4, out.ctypes.data) == -errno.EINVAL
    if glob.glob("/dev/nvidia[0-9]*"):
        return      # below: a library that never found a GPU
    assert L.oimgpu_bdev_mirror_check(b"x", 0, 1, 0, None, 0, out.ctypes.data) == -errno.ENODEV
    assert L.oimgpu_init_control_only() == 0
    try:
        name = lib.construct_mirror_bdev(64, 512, [0, 0], name="CtlMirror")
        for nm in (name, "nope"):
            assert L.oimgpu_bdev_mirror_check(nm.encode(), 0, 64, 1, ranges.ctypes.data, 4, out.ctypes.data) == -errno.ENODEV
    finally:
        lib.fini()


def test_check_mirror_bdev_without_a_gpu(daemons):
    s = daemons("ours", ["--control-only"])
    rpc(s, "construct_mirror_bdev", {"num_blocks": 64, "block_size": 512, "replicas": 2, "name": "M"})
    nodev = {"code": -32602, "message": "No such device"}
    for p in ({"name": "M"}, {"name": "M", "repair": True}, {"name": "M", "offset_blocks": 8, "num_blocks": 8}, {"name": "nope"}):
        assert rpc(s, "check_mirror_bdev", p) == {"error": nodev}, p
    bad = {"code": -32602, "message": "Invalid parameters"}
    for p in ({}, {"offset_blocks": 0}, {"name": 1}, {"name": "M", "repair": 1}, {"name": "M", "offset_blocks": -1},
              {"name": "M", "num_blocks": "8"}, {"name": "M", "num_blocks": 0.5}, {"name": "M", "x": 1}, None):
        assert rpc(s, "check_mirror_bdev", p) == {"error": bad}, p
    cfg = rpc(s, "get_subsystem_config", {"name": "bdev"})
    assert [x["method"] for x in cfg] == ["set_bdev_options", "construct_mirror_bdev"]


# ---- GPU ----------------------------------------------------------------------------------------------------

def _seed(rng, reps, bs, nb, count):
    """`count` differences of 1-40 bytes at random places of random replicas (replica 0 included), and the edge cases:
    the first and the last byte of a block, a piece across a block boundary"""
    def put(r, pos, nbytes):
        nbytes = min(nbytes, reps[r].size - pos)
        reps[r][pos:pos + nbytes] ^= rng.integers(1, 256, size=nbytes, dtype=np.uint8)
        return r, pos, nbytes
    nrep = len(reps)
    out = [put(nrep - 1, 5 * bs, 1), put(1, 9 * bs - 1, 1), put(nrep - 1, 13 * bs - 3, 6)]
    for _ in range(count):
        out.append(put(int(rng.integers(0, nrep)), int(rng.integers(0, nb * bs)), int(rng.integers(1, 41))))
    return out


def _assert_equal_model(got, want, what):
    for k in ("blocks_checked", "mismatched_blocks", "ranges", "truncated"):
        assert got[k] == want[k], f"{what}: {k} {got[k]!r} != model {want[k]!r}"


CASES = [(bs, r) for bs in (512, 520, 4096, 4097) for r in (2, 3, 4)]


@pytest.mark.gpu
@pytest.mark.parametrize("bs,nrep", CASES, ids=[f"bs{b}-r{r}" for b, r in CASES])
def test_check_and_repair_match_the_model(gpu, bs, nrep):
    nb = 1536
    rng = np.random.default_rng(bs * 10 + nrep)
    name = gpu.construct_mirror_bdev(nb, bs, [0] * nrep, name=f"chk{bs}r{nrep}")
    try:
        base = traces.pattern_bytes(7, 0, nb * bs)
        reps = [base.copy() for _ in range(nrep)]
        gpu.bdev_write_raw(name, 0, base, replica=0)
        got = gpu.mirror_check(name)
        assert (got["mismatched_blocks"], got["ranges"]) == (nb, [(0, nb)]), "zeroed replicas next to the pattern: every block"
        for r in range(1, nrep):
            gpu.bdev_write_raw(name, 0, base, replica=r)
        assert gpu.mirror_check(name) == {"blocks_checked": nb, "mismatched_blocks": 0, "repaired_blocks": 0,
                                          "ranges": [], "truncated": False}
        for r, pos, n in _seed(rng, reps, bs, nb, 150):
            gpu.bdev_write_raw(name, pos, reps[r][pos:pos + n], replica=r)
        windows = [(0, nb), (1, nb - 1), (0, nb - 1), (5, 1), (8, 1), (12, 2), (100, 700), (nb - 1, 1), (nb, 0)]
        windows += [(int(a), int(rng.integers(0, nb - a + 1))) for a in rng.integers(0, nb, size=4)]
        for off, n in windows:
            for mr in (MAX_RANGES, 3, 0):
                got = gpu.mirror_check(name, off, n, max_ranges=mr)
                _assert_equal_model(got, model_check(reps, bs, off, n, mr), f"[{off}, +{n}) max_ranges {mr}")
                assert got["repaired_blocks"] == 0
        assert model_check(reps, bs, 0, nb)["truncated"], "the seeds make more runs than one call returns"
        # repair a sub-range: only its blocks change, and only in replicas 1..
        d0 = gpu.bdev_digest(name, 0)
        off, n = 200, 600
        want = model_check(reps, bs, off, n)
        got = gpu.mirror_check(name, off, n, repair=True)
        _assert_equal_model(got, want, "repair of a sub-range")
        assert got["repaired_blocks"] == want["mismatched_blocks"] > 0
        model_repair(reps, bs, want["blocks"])
        for r in range(nrep):
            bad = np.nonzero(gpu.bdev_read_raw(name, 0, nb * bs, replica=r) != reps[r])[0]
            assert not len(bad), f"replica {r} after the sub-range repair differs from the model at {bad[:8]} (block {bad[:1] // bs})"
        _assert_equal_model(gpu.mirror_check(name), model_check(reps, bs, 0, nb), "after the sub-range repair")
        # the whole device
        got = gpu.mirror_check(name, repair=True)
        assert got["repaired_blocks"] == got["mismatched_blocks"] == model_check(reps, bs, 0, nb)["mismatched_blocks"]
        assert gpu.bdev_digest(name, 0) == d0, "a repair changed replica 0"
        for r in range(1, nrep):
            assert gpu.bdev_digest(name, r) == d0, f"replica {r} after the repair"
        assert gpu.mirror_check(name)["mismatched_blocks"] == 0
    finally:
        gpu.delete_bdev(name)


@pytest.mark.gpu
def test_mirror_check_refusals(gpu):
    import socket
    plain = gpu.construct_malloc_bdev(64, 512, name="chkplain", device=0)
    name = gpu.construct_mirror_bdev(64, 512, [0, 0], name="chkrefuse")
    try:
        for call, rc in ((lambda: gpu.mirror_check(plain), -errno.ENOTSUP),
                         (lambda: gpu.mirror_check("nope"), -errno.ENODEV),
                         (lambda: gpu.mirror_check(name, 0, 65), -errno.EINVAL),
                         (lambda: gpu.mirror_check(name, 65, 0), -errno.EINVAL),
                         (lambda: gpu.mirror_check(name, 60, 5), -errno.EINVAL),
                         (lambda: gpu.mirror_check(name, 1, (1 << 64) - 1), -errno.EINVAL)):
            with pytest.raises(gpu.OimGpuError) as e:
                call()
            assert e.value.rc == rc
        assert gpu.mirror_check(name, 64, 0)["blocks_checked"] == 0
        # an NBD export serving the mirror: -EBUSY while it runs, a check again once it ended
        a, b = socket.socketpair()
        a.settimeout(20)
        rc = []

        def serve():
            rc.append(gpu.load().oimgpu_nbd_serve(name.encode(), b.fileno()))
            b.close()
        th = threading.Thread(target=serve, daemon=True)
        th.start()
        try:
            flush = (0x25609513).to_bytes(4, "big") + (3).to_bytes(4, "big") + b"chkflush" + bytes(12)
            a.sendall(flush)                            # answered: the export is in its loop
            reply = b""
            while len(reply) < 16:
                reply += a.recv(16 - len(reply))
            assert reply[:8] == bytes([0x67, 0x44, 0x66, 0x98, 0, 0, 0, 0]) and reply[8:] == b"chkflush"
            with pytest.raises(gpu.OimGpuError) as e:
                gpu.mirror_check(name)
            assert e.value.rc == -errno.EBUSY
        finally:
            a.close()
            th.join(20)
        assert rc == [0]
        assert gpu.mirror_check(name)["mismatched_blocks"] == 0
    finally:
        gpu.delete_bdev(name)
        gpu.delete_bdev(plain)


@pytest.mark.gpu
@pytest.mark.timeout(120)
def test_check_and_repair_next_to_a_resident_poller(gpu):
    """a controller-wide session with a resident poller serves a 2-way mirror.  Writes go in, a replica is changed
    behind the session's back, and a check and a repair run from another thread: the poller is parked and comes back,
    the writes that follow reach both replicas, and both end equal to the model of every write"""
    import torch
    from test_mirror import _io
    from test_multi_target import Controller
    c = Controller(gpu, only={3}, mirrors={3: [0, 0]})
    name, nb = c.names[3], c.sizes[3][0]
    want = traces.pattern_bytes(7 + 3, 0, nb * 512)
    buf = torch.zeros(4096, dtype=torch.uint8).pin_memory()
    try:
        with gpu.Lun(c.ctrlr, -1, num_queues=1, queue_size=64) as lun:
            lun.start_poller(idle_timeout_ms=4000)
            try:
                for k, lba in enumerate((40, 300, 1000)):
                    payload = traces.pattern_bytes(5000 + k, 0, 4096)
                    buf.numpy()[:] = payload
                    cp = _io(lun, 3, lba, 8, True, buf.data_ptr())
                    assert (cp["response"], cp["status"]) == (abi.S_OK, 0)
                    want[lba * 512:(lba + 8) * 512] = payload
                junk = np.full(700, 0xA5, dtype=np.uint8)
                gpu.bdev_write_raw(name, 2000 * 512 + 100, junk, replica=1)     # blocks 2000 and 2001
                box = {}

                def run():
                    try:
                        box["check"] = gpu.mirror_check(name)
                        box["repair"] = gpu.mirror_check(name, repair=True)
                    except Exception as e:          # noqa: BLE001  (reported below)
                        box["error"] = e
                th = threading.Thread(target=run)
                th.start()
                th.join(60)
                assert not th.is_alive() and "error" not in box, box.get("error")
                assert box["check"]["ranges"] == [(2000, 2)] and box["check"]["mismatched_blocks"] == 2
                assert box["repair"]["repaired_blocks"] == 2
                assert lun.poller_running(), "the poller did not come back after the check"
                payload = traces.pattern_bytes(6000, 0, 4096)
                buf.numpy()[:] = payload
                cp = _io(lun, 3, 2000, 8, True, buf.data_ptr())
                assert (cp["response"], cp["status"]) == (abi.S_OK, 0)
                want[2000 * 512:2008 * 512] = payload
                buf.numpy()[:] = 0
                assert _io(lun, 3, 300, 8, False, buf.data_ptr())["status"] == 0
                assert (buf.numpy() == want[300 * 512:308 * 512]).all(), "a read after the check returned other bytes"
                assert lun.poller_running()
            finally:
                lun.stop_poller()
            # the first start and the restarts after the check and the repair
            assert lun.iostat()["kernel_launches"] == 3
        for r in (0, 1):
            bad = np.nonzero(gpu.bdev_read_raw(name, 0, nb * 512, replica=r) != want)[0]
            assert not len(bad), f"replica {r} differs from the model of the writes at {len(bad)} bytes, first {bad[:8]}"
        assert gpu.mirror_check(name)["mismatched_blocks"] == 0
    finally:
        c.close()


def _exporter(conn, nb, bs):
    """another process on cuda:0: a Malloc bdev it exports; "write" changes its own store, "read" returns it"""
    from oim_b200 import lib as olib
    olib.init([0])
    try:
        nm = olib.construct_malloc_bdev(nb, bs, name="chkexport", device=0)
        olib.bdev_write_raw(nm, 0, traces.pattern_bytes(9, 0, nb * bs))
        conn.send(olib.bdev_export_store(nm))
        while True:
            cmd = conn.recv()
            if cmd[0] == "write":
                olib.bdev_write_raw(nm, cmd[1], np.frombuffer(cmd[2], dtype=np.uint8))
                conn.send("ok")
            elif cmd[0] == "read":
                conn.send(olib.bdev_read_raw(nm, 0, nb * bs).tobytes())
            else:
                break
        olib.delete_bdev(nm)
        conn.send("done")
    finally:
        olib.fini()


@pytest.mark.gpu
@pytest.mark.timeout(240)
def test_imported_replica_written_by_its_own_process(gpu):
    import multiprocessing as mp
    nb, bs = 8192, 520
    init = traces.pattern_bytes(9, 0, nb * bs)
    ctx = mp.get_context("spawn")
    conn, child_conn = ctx.Pipe()
    p = ctx.Process(target=_exporter, args=(child_conn, nb, bs), daemon=True)
    p.start()
    name = None
    try:
        assert conn.poll(120), "the exporting process sent no handle"
        name = gpu.construct_mirror_bdev_remote(nb, bs, 0, [conn.recv()], name="chkimport")
        # replica 0 is new and zeroed: the mirror is inconsistent from the start, everywhere
        got = gpu.mirror_check(name, max_ranges=4)
        assert (got["mismatched_blocks"], got["ranges"], got["truncated"]) == (nb, [(0, nb)], False)
        gpu.bdev_write_raw(name, 0, init, replica=0)
        assert gpu.mirror_check(name)["mismatched_blocks"] == 0
        want = init.copy()
        for pos, n in ((100 * bs + 7, 3), (4000 * bs - 1, 2), (nb * bs - 1, 1)):
            piece = (want[pos:pos + n] ^ 0x5A).astype(np.uint8)
            conn.send(("write", pos, piece.tobytes()))
            assert conn.recv() == "ok"
            want[pos:pos + n] = piece
        m = model_check([init, want], bs, 0, nb)
        assert m["ranges"] == [(100, 1), (3999, 2), (nb - 1, 1)]
        _assert_equal_model(gpu.mirror_check(name), m, "difference written by the exporter")
        got = gpu.mirror_check(name, repair=True)
        assert got["repaired_blocks"] == 4
        conn.send(("read",))
        assert (np.frombuffer(conn.recv(), dtype=np.uint8) == init).all(), "the exporter's store is not replica 0's after the repair"
        assert gpu.mirror_check(name)["mismatched_blocks"] == 0
        gpu.delete_bdev(name)
        name = None
        conn.send(("quit",))
        assert conn.poll(60) and conn.recv() == "done"
        p.join(60)
        assert p.exitcode == 0
    finally:
        if name is not None:
            gpu.delete_bdev(name)
        p.join(5)
        if p.is_alive():
            p.kill()
            p.join(10)


@pytest.mark.gpu
def test_check_mirror_bdev_through_the_daemon(gpu, daemons):
    s = daemons("ours", ["--gpus", "0"])
    nb, bs = 4096, 4096
    assert rpc(s, "construct_mirror_bdev", {"num_blocks": nb, "block_size": bs, "replicas": 2, "name": "vol7"}) == "vol7"
    clean = {"name": "vol7", "replicas": 2, "offset_blocks": 0, "num_blocks": nb, "mismatched_blocks": 0,
             "repaired_blocks": 0, "mismatches": [], "truncated": False}
    assert rpc(s, "check_mirror_bdev", {"name": "vol7"}) == clean
    handle = base64.b64decode(rpc(s, "export_bdev_store", {"name": "vol7", "replica": 1}))
    local = gpu.construct_mirror_bdev_remote(nb, bs, 0, [handle], name="chkdaemon")
    try:
        gpu.bdev_write_raw(local, 17 * bs + 4000, np.full(bs, 0xEE, dtype=np.uint8), replica=1)    # blocks 17, 18
        gpu.bdev_write_raw(local, 4095 * bs + 4095, np.ones(1, dtype=np.uint8), replica=1)       # the last byte
        want = dict(clean, mismatched_blocks=3, mismatches=[{"offset_blocks": 17, "num_blocks": 2},
                                                             {"offset_blocks": 4095, "num_blocks": 1}])
        assert rpc(s, "check_mirror_bdev", {"name": "vol7"}) == want
        assert rpc(s, "check_mirror_bdev", {"name": "vol7", "offset_blocks": 18, "num_blocks": 100}) == \
            dict(clean, offset_blocks=18, num_blocks=100, mismatched_blocks=1, mismatches=[{"offset_blocks": 18, "num_blocks": 1}])
        assert rpc(s, "check_mirror_bdev", {"name": "vol7", "offset_blocks": nb + 1}) == \
            {"error": {"code": -32602, "message": "Invalid argument"}}
        assert rpc(s, "check_mirror_bdev", {"name": "vol7", "repair": True}) == dict(want, repaired_blocks=3)
        assert rpc(s, "check_mirror_bdev", {"name": "vol7"}) == clean
        assert (gpu.bdev_read_raw(local, 0, nb * bs, replica=1) == 0).all(), "the repair did not copy replica 0's zeros"
        many = np.zeros(nb * bs, dtype=np.uint8)
        many[np.arange(100) * 3 * bs] = 1                  # 100 runs
        gpu.bdev_write_raw(local, 0, many, replica=1)
        got = rpc(s, "check_mirror_bdev", {"name": "vol7"})
        assert (got["mismatched_blocks"], len(got["mismatches"]), got["truncated"]) == (100, 64, True)
        assert got["mismatches"][-1] == {"offset_blocks": 189, "num_blocks": 1}
    finally:
        gpu.delete_bdev(local)
    cfg = [x["method"] for x in rpc(s, "get_subsystem_config", {"name": "bdev"})]
    assert cfg == ["set_bdev_options", "construct_mirror_bdev"]
    assert rpc(s, "delete_bdev", {"name": "vol7"}) is True
    assert rpc(s, "check_mirror_bdev", {"name": "vol7"}) == {"error": {"code": -32602, "message": "No such device"}}


@pytest.mark.gpu
@pytest.mark.timeout(280)
def test_eight_gib_mirror_with_sparse_differences(gpu):
    """a size a host copy is too slow for: 8 GiB per replica, differences in both replicas, the last block included"""
    import time
    bs = 4096
    nb = (8 << 30) // bs
    name = gpu.construct_mirror_bdev(nb, bs, [0, 0], name="chk8g")
    try:
        rng = np.random.default_rng(8)
        blocks = sorted(set(int(b) for b in rng.choice(nb - 2, size=90, replace=False)) | {nb - 1})
        for k, blk in enumerate(blocks):
            off = int(rng.integers(0, bs - 8))
            gpu.bdev_write_raw(name, blk * bs + off, rng.integers(1, 256, size=8, dtype=np.uint8), replica=k % 2)
        runs = []
        for b in blocks:
            if runs and runs[-1][0] + runs[-1][1] == b:
                runs[-1][1] += 1
            else:
                runs.append([b, 1])
        t0 = time.perf_counter()
        got = gpu.mirror_check(name)
        t1 = time.perf_counter()
        assert got["mismatched_blocks"] == len(blocks)
        assert got["ranges"] == [tuple(r) for r in runs[:MAX_RANGES]] and got["truncated"] == (len(runs) > MAX_RANGES)
        got = gpu.mirror_check(name, nb - 2, 2, repair=True)
        assert got["ranges"][-1] == (nb - 1, 1)
        d0 = gpu.bdev_digest(name, 0)
        got = gpu.mirror_check(name, repair=True)
        assert got["repaired_blocks"] == len(blocks) - 1
        assert gpu.bdev_digest(name, 1) == d0 == gpu.bdev_digest(name, 0)
        assert gpu.mirror_check(name)["mismatched_blocks"] == 0
        print(f"check of 2 x 8 GiB: {1e3 * (t1 - t0):.1f} ms")
    finally:
        gpu.delete_bdev(name)
