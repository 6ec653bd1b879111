"""Moving an imported replica of a mirror to another process's store while the mirror is served
(oimgpu_bdev_mirror_replace_remote, lib.mirror_replace_remote, the daemon's replace_mirror_replica).

After the call the new store holds replica 0's bytes, every later write reaches it and none reaches the old one, and
nothing else about the bdev changes: its counters, uuid, listing and configuration dump (with the new handle).

CPU: the C ABI's refusals without a device, and the daemon's replies under --control-only.
GPU (cuda:0; one test also cuda:1): content at block sizes 512, 4096 and 4097 on 2- and 4-way mirrors written through a
session; a VM through the vhost-user socket with the replace between two halves of its trace, launch per kick and
with the resident poller; a controller-wide session that reaches the mirror as a peer target and a session that does
not reach it; the refusals; the documented drain sequence over three daemons with save and restore; and a new store on
a second GPU."""
import base64
import errno
import glob
import json
import os
import socket
import struct
import sys
import threading
import time

import numpy as np
import pytest

from oim_b200 import abi, traces, vring
from oim_b200 import vhost_user_master as vu
from test_daemon_mirror import (BAD, IOSTAT, RING, UUID, daemons, masked, mirror_entry, oracle_run,  # noqa: F401
                                provision_mirror, qring, replica_digests, rpc, vm_trace)
from test_vhost_user import handshake, small_ring

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NODEV = {"code": -32602, "message": "No such device"}


# ---- CPU ------------------------------------------------------------------------------------------------------------

def test_replace_abi_without_gpu():
    from oim_b200 import lib
    L = lib.load()
    h = bytes(64)
    assert L.oimgpu_bdev_mirror_replace_remote(None, 1, h) == -errno.EINVAL
    assert L.oimgpu_bdev_mirror_replace_remote(b"x", 1, None) == -errno.EINVAL
    with pytest.raises(ValueError):
        lib.mirror_replace_remote("x", 1, bytes(63))
    if glob.glob("/dev/nvidia[0-9]*"):
        return      # below: a library that never found a GPU
    assert L.oimgpu_bdev_mirror_replace_remote(b"x", 1, h) == -errno.ENODEV
    assert L.oimgpu_init_control_only() == 0
    try:
        name = lib.construct_mirror_bdev(64, 512, [0, 0], name="CtlMirror")
        for nm in (name, "nope"):
            for rep in (0, 1, 2):
                assert L.oimgpu_bdev_mirror_replace_remote(nm.encode(), rep, h) == -errno.ENODEV
    finally:
        lib.fini()


def test_replace_mirror_replica_without_a_gpu(daemons):
    s = daemons("ours", ["--control-only"])
    rpc(s, "construct_malloc_bdev", {"num_blocks": 64, "block_size": 512, "name": "Plain"})
    rpc(s, "construct_mirror_bdev", {"num_blocks": 64, "block_size": 512, "replicas": 2, "name": "M", "uuid": UUID})
    cfg = rpc(s, "get_subsystem_config", {"name": "bdev"})
    bdevs = rpc(s, "get_bdevs")
    handle = base64.b64encode(bytes(range(64))).decode()
    ok = {"name": "M", "replica": 1, "remote_replica": handle}
    for p in (ok, dict(ok, name="nope"), dict(ok, name="Plain"), dict(ok, replica=0), dict(ok, replica=7)):
        assert rpc(s, "replace_mirror_replica", p) == {"error": NODEV}, p
    for p in ({}, None, {"name": "M"}, {"name": "M", "replica": 1}, {"replica": 1, "remote_replica": handle},
              dict(ok, name=1), dict(ok, replica="1"), dict(ok, replica=1.5), dict(ok, replica=1 << 40),
              dict(ok, remote_replica=7), dict(ok, remote_replica=[handle]), dict(ok, remote_replica="not base64!"),
              dict(ok, remote_replica=handle[:-4]), dict(ok, remote_replica=handle + "="),
              dict(ok, remote_replica=base64.b64encode(bytes(65)).decode()),
              dict(ok, remote_replica=base64.b64encode(bytes(48)).decode()), dict(ok, bogus=1)):
        raw = s.call("replace_mirror_replica", p)
        assert json.loads(raw)["error"] == BAD, (p, raw)
    assert rpc(s, "get_subsystem_config", {"name": "bdev"}) == cfg
    assert rpc(s, "get_bdevs") == bdevs


# ---- GPU: helpers ---------------------------------------------------------------------------------------------------

def _exporter(conn, devices):
    """another process: makes Malloc bdevs on request and answers with their IPC handles; digests and deletes them"""
    from oim_b200 import lib as olib
    olib.init(devices)
    try:
        conn.send("ready")
        while True:
            cmd = conn.recv()
            try:
                if cmd[0] == "make":
                    _, nm, nb, bs, dev, seed = cmd
                    olib.construct_malloc_bdev(nb, bs, name=nm, device=dev)
                    if seed is not None:
                        olib.bdev_write_raw(nm, 0, traces.pattern_bytes(seed, 0, nb * bs))
                    conn.send(olib.bdev_export_store(nm))
                elif cmd[0] == "digest":
                    conn.send(olib.bdev_digest(cmd[1]))
                elif cmd[0] == "delete":
                    olib.delete_bdev(cmd[1])
                    conn.send("ok")
                else:
                    break
            except Exception as e:              # noqa: BLE001  (raised in the test process)
                conn.send(("error", repr(e)))
        conn.send("done")
    finally:
        olib.fini()


class Exporter:
    def __init__(self, devices):
        import multiprocessing as mp
        ctx = mp.get_context("spawn")
        self.conn, child = ctx.Pipe()
        self.p = ctx.Process(target=_exporter, args=(child, devices), daemon=True)
        self.p.start()
        assert self.conn.poll(120) and self.conn.recv() == "ready", "the exporting process did not start"

    def ask(self, *cmd):
        self.conn.send(cmd)
        assert self.conn.poll(120), f"no answer to {cmd[0]}"
        r = self.conn.recv()
        if isinstance(r, tuple) and r and r[0] == "error":
            raise RuntimeError(f"exporter: {cmd[0]}: {r[1]}")
        return r

    def make(self, name, nb, bs, device=0, seed=None) -> bytes:
        return self.ask("make", name, nb, bs, device, seed)

    def digest(self, name):
        return tuple(self.ask("digest", name))

    def stop(self):
        if self.p.is_alive():
            try:
                self.conn.send(("quit",))
                self.conn.poll(60) and self.conn.recv()
            except (BrokenPipeError, EOFError):
                pass
        self.p.join(30)
        if self.p.is_alive():
            self.p.kill()
            self.p.join(10)


@pytest.fixture()
def exporters():
    """start exporting processes; they stop after the test, when its importing mirrors are gone"""
    made = []

    def start(devices=(0,)):
        e = Exporter(list(devices))
        made.append(e)
        return e
    yield start
    for e in reversed(made):
        e.stop()


def _rw(lun, target, lba, nblk, bs, write, addr):
    b = abi.Batch(target)
    (b.write if write else b.read)(lba, nblk, [(addr, nblk * bs)], tag=lba + 1)
    cp = lun.run(*b.arrays())[0]
    assert (cp["response"], cp["status"]) == (abi.S_OK, 0), cp


def _write(lun, target, want, buf, lba, nblk, bs, seed):
    payload = traces.pattern_bytes(seed, 0, nblk * bs)
    buf.numpy()[:nblk * bs] = payload
    _rw(lun, target, lba, nblk, bs, True, buf.data_ptr())
    want[lba * bs:(lba + nblk) * bs] = payload


def _writes(lun, target, want, buf, nb, bs, rng, count):
    top = max(1, min(64, (1 << 20) // bs))
    for k in range(count):
        n = int(rng.integers(1, top + 1))
        lba = 0 if k == 0 else nb - n if k == 1 else int(rng.integers(0, nb - n + 1))
        _write(lun, target, want, buf, lba, n, bs, int(rng.integers(1, 1 << 30)))


def _pinned(nbytes):
    import torch
    return torch.zeros(nbytes, dtype=torch.uint8).pin_memory()


def _refused(gpu, rc, *args):
    with pytest.raises(gpu.OimGpuError) as e:
        gpu.mirror_replace_remote(*args)
    assert e.value.rc == rc, (args[:2], e.value.rc)


def _replica_info(gpu, name, r):
    import ctypes as C
    d, i = C.c_int(-1), C.c_int(-1)
    assert gpu.load().oimgpu_bdev_replica_info(name.encode(), r, C.byref(d), C.byref(i)) == 0
    return d.value, i.value


# ---- GPU: content ---------------------------------------------------------------------------------------------------

CONTENT = [(bs, r) for r in (2, 4) for bs in (512, 4096, 4097)]


@pytest.mark.gpu
@pytest.mark.timeout(240)
@pytest.mark.parametrize("bs,nrep", CONTENT, ids=[f"bs{b}-r{r}" for b, r in CONTENT])
def test_replaced_replica_holds_replica_0_and_takes_the_writes(gpu, exporters, bs, nrep):
    nb = 2048
    rng = np.random.default_rng(bs * 10 + nrep)
    ex = exporters()
    olds = [f"old{r}" for r in range(1, nrep)]
    handles = [ex.make(nm, nb, bs) for nm in olds]
    fresh = ex.make("fresh", nb, bs, seed=77)          # junk the copy must overwrite
    ctrlr, name = f"rpl{bs}r{nrep}", f"rplm{bs}r{nrep}"
    gpu.construct_mirror_bdev_remote(nb, bs, 0, handles, name=name)
    gpu.construct_vhost_scsi_controller(ctrlr)
    gpu.add_vhost_scsi_lun(ctrlr, 0, name)
    buf = _pinned(1 << 20)
    want = np.zeros(nb * bs, dtype=np.uint8)
    r = nrep - 1
    try:
        with gpu.Lun(ctrlr, 0, num_queues=1, queue_size=64) as lun:
            _writes(lun, 0, want, buf, nb, bs, rng, 12)
            before = {k: gpu.get_bdevs(name)[0][k] for k in ("uuid", "claimed", "num_blocks", "block_size", "replicas")}
            stat = gpu.get_bdevs_iostat(name)
            gpu.mirror_replace_remote(name, r, fresh)
            assert {k: gpu.get_bdevs(name)[0][k] for k in before} == before
            assert gpu.get_bdevs_iostat(name) == stat, "the replace changed the bdev's counters"
            assert _replica_info(gpu, name, r) == (0, 1)
            d = gpu.digest_host(want)
            assert ex.digest("fresh") == d, "the new store does not hold replica 0's bytes"
            assert gpu.bdev_digest(name, r) == d == gpu.bdev_digest(name, 0)
            assert gpu.mirror_check(name)["mismatched_blocks"] == 0
            d_old = ex.digest(olds[r - 1])
            _writes(lun, 0, want, buf, nb, bs, rng, 8)
            buf.numpy()[:] = 0
            _rw(lun, 0, 0, 1, bs, False, buf.data_ptr())
            assert (buf.numpy()[:bs] == want[:bs]).all()
        d = gpu.digest_host(want)
        assert ex.digest("fresh") == d, "a write after the replace missed the new store"
        assert ex.digest(olds[r - 1]) == d_old, "a write after the replace reached the old store"
        for k in range(1, nrep - 1):
            assert ex.digest(olds[k - 1]) == d, f"replica {k}"
        assert gpu.bdev_digest(name, 0) == d
        assert gpu.mirror_check(name)["mismatched_blocks"] == 0
    finally:
        gpu.remove_vhost_scsi_target(ctrlr, 0)
        gpu.remove_vhost_controller(ctrlr)
        gpu.delete_bdev(name)


# ---- GPU: a VM through the daemon -----------------------------------------------------------------------------------

def vm_run_split(s, rq, seed, between):
    """a VM with one request queue: the first half of `rq` is published and drained, `between()` runs while the VM
    stays connected, then the rest -> (image, guest memory after, used elements)"""
    img = vring.build_image(rq, ring_size=RING, seed=seed, mutate=False)
    assert img.meta["placed"] == len(rq)
    ram = vu.GuestRam(img.arena.size)
    ram.mem[:] = img.arena
    cq, eq = small_ring(0), small_ring(1)
    for r in (cq, eq):
        ram.mem[r[0]:r[0] + 8192] = 0
    avail, used = qring(0)
    ram.mem[avail:avail + 16384] = 0
    heads = np.asarray(img.heads[:len(rq)], dtype="<u2")
    ram.mem[avail + 4:avail + 4 + 2 * len(heads)] = heads.view(np.uint8)
    queues = [vu.Queue(0, 16, *cq[:3]), vu.Queue(1, 16, *eq[:3]), vu.Queue(2, RING, img.desc_off, avail, used)]
    m = vu.Master(s.sock("scsi0"))
    try:
        handshake(m, ram, img, queues)
        time.sleep(0.3)
        q = queues[2]
        for upto in (len(rq) // 2, len(rq)):
            ram.mem[avail + 2:avail + 4] = np.frombuffer(struct.pack("<H", upto), np.uint8)
            q.notify()
            q.wait_used(ram, upto)
            if upto < len(rq):
                between()
        time.sleep(0.1)
        assert int(ram.mem[used + 2:used + 4].view("<u2")[0]) == len(rq), "more used elements than requests"
        u = ram.mem[used + 4:used + 4 + 8 * len(rq)].view(vring.used_elem_dtype)
        out = sorted((int(i), int(ln)) for i, ln in u)
        mem = ram.mem.copy()
        for x in queues:
            m.get_vring_base(x.index)
        return img, mem, out
    finally:
        m.close()
        for x in queues:
            x.close()
        ram.close()


@pytest.mark.gpu
@pytest.mark.timeout(300)
@pytest.mark.parametrize("mode,bs", [("kick", 512), ("poller", 4096)])
def test_replace_in_the_middle_of_a_vm(gpu, oracles, daemons, mode, bs):
    """daemon B exports replica 1 of A's mirror, daemon C the store it moves to; the replace comes between the two
    halves of the VM's trace.  The VM sees what the C restatement computes for the whole trace, each request completes
    once, the counters count each once, and A's replica 0 and C's store end equal to the restatement's store"""
    seed = 900 + bs
    rq_by_q, nb = vm_trace(bs, 1, seed)
    rq = rq_by_q[0]
    b = daemons("b", ["--gpus", "0"])
    c = daemons("c", ["--gpus", "0"])
    a = daemons("a", ["--gpus", "0"] + (["--poller"] if mode == "poller" else []))
    assert rpc(b, "construct_malloc_bdev", {"num_blocks": nb, "block_size": bs, "name": "r1"}) == "r1"
    assert rpc(c, "construct_malloc_bdev", {"num_blocks": nb, "block_size": bs, "name": "r1b"}) == "r1b"
    old, new = rpc(b, "export_bdev_store", {"name": "r1"}), rpc(c, "export_bdev_store", {"name": "r1b"})
    name = provision_mirror(a, nb, bs, remote_replicas=[old], uuid=UUID)
    done = []

    def between():
        assert rpc(a, "replace_mirror_replica", {"name": name, "replica": 1, "remote_replica": new}) is True
        done.append(rpc(a, "get_bdevs_iostat", {"name": name})[1])
    img, mem, used = vm_run_split(a, rq, seed, between)
    assert done, "the replace did not run"
    wimg, wused, wstore, wstat = oracle_run(oracles, [rq], nb, bs, seed)
    assert len(used) == len(rq) == len({i for i, _ in used}), "a request was lost or completed twice"
    assert used == wused, "used elements differ from the checker's"
    bad = np.nonzero(masked(img, mem, 1) != masked(wimg, wimg.arena, 1))[0]
    assert not len(bad), f"guest memory differs from the checker's at {len(bad)} bytes, first {bad[:8]}"
    want = {k: wstat[k] for k in IOSTAT}
    deadline = time.time() + 10
    while True:
        st = rpc(a, "get_bdevs_iostat", {"name": name})[1]
        got = {k: st[k] for k in IOSTAT}
        if got == want or time.time() > deadline:
            break
        time.sleep(0.05)
    assert got == want, f"get_bdevs_iostat {got}, the checker counted {want}"
    assert 0 < done[0]["num_write_ops"] + done[0]["num_read_ops"] < want["num_write_ops"] + want["num_read_ops"], \
        "the replace did not fall between requests"
    digest = gpu.digest_host(wstore)
    assert replica_digests(gpu, a, name, 1, nb, bs) == [digest], "A's replica 0 differs from the checker's store"
    assert replica_digests(gpu, c, "r1b", 1, nb, bs) == [digest], "the new replica differs from the checker's store"
    assert rpc(a, "check_mirror_bdev", {"name": name})["mismatched_blocks"] == 0
    assert rpc(b, "delete_bdev", {"name": "r1"}) is True           # the old exporter may go first now
    assert rpc(a, "remove_vhost_scsi_target", {"ctrlr": "scsi0", "scsi_target_num": 0}) is True
    assert rpc(a, "delete_bdev", {"name": name}) is True
    assert rpc(c, "delete_bdev", {"name": "r1b"}) is True


# ---- GPU: sessions that reach the mirror as a peer, and sessions that do not ---------------------------------------

@pytest.mark.gpu
@pytest.mark.timeout(180)
def test_peer_target_session_and_an_unrelated_session_are_held_and_resume(gpu, exporters):
    """a controller-wide session reaches the mirror as target 3; a session of another controller on the same GPU does
    not reach it.  Both run resident pollers, both are parked for the replace and restarted, and the controller-wide
    session's writes afterwards land in the new store only"""
    nb, bs = 4096, 512
    ex = exporters()
    old = ex.make("old", nb, bs)
    fresh = ex.make("fresh", nb, bs, seed=5)
    name = gpu.construct_mirror_bdev_remote(nb, bs, 0, [old], name="rplpeer")
    plain = gpu.construct_malloc_bdev(nb, bs, name="rplplain0", device=0)
    other = gpu.construct_malloc_bdev(nb, bs, name="rplother", device=0)
    gpu.construct_vhost_scsi_controller("rplwide")
    gpu.add_vhost_scsi_lun("rplwide", 0, plain)
    gpu.add_vhost_scsi_lun("rplwide", 3, name)
    gpu.construct_vhost_scsi_controller("rplalone")
    gpu.add_vhost_scsi_lun("rplalone", 0, other)
    want, want_other = np.zeros(nb * bs, np.uint8), np.zeros(nb * bs, np.uint8)
    buf = _pinned(1 << 20)
    try:
        with gpu.Lun("rplwide", -1, num_queues=1, queue_size=64) as wide, \
                gpu.Lun("rplalone", 0, num_queues=1, queue_size=64) as alone:
            wide.start_poller(idle_timeout_ms=4000)
            alone.start_poller(idle_timeout_ms=4000)
            try:
                for k, lba in enumerate((40, 300, nb - 8)):
                    _write(wide, 3, want, buf, lba, 8, bs, 3000 + k)
                    _write(alone, 0, want_other, buf, lba, 8, bs, 4000 + k)
                d_old = ex.digest("old")
                gpu.mirror_replace_remote(name, 1, fresh)
                assert wide.poller_running() and alone.poller_running(), "a poller did not come back"
                for k, lba in enumerate((41, 1000)):
                    _write(wide, 3, want, buf, lba, 8, bs, 5000 + k)
                    _write(alone, 0, want_other, buf, lba, 8, bs, 6000 + k)
                buf.numpy()[:] = 0
                _rw(wide, 3, 300, 8, bs, False, buf.data_ptr())
                assert (buf.numpy()[:8 * bs] == want[300 * bs:308 * bs]).all()
                assert wide.poller_running() and alone.poller_running()
            finally:
                wide.stop_poller()
                alone.stop_poller()
            assert wide.iostat()["kernel_launches"] == 2 and alone.iostat()["kernel_launches"] == 2, \
                "each poller: the first start and one restart after the replace"
        d = gpu.digest_host(want)
        assert ex.digest("fresh") == d == gpu.bdev_digest(name, 0) == gpu.bdev_digest(name, 1)
        assert ex.digest("old") == d_old, "a write after the replace reached the old store"
        assert gpu.bdev_digest(other, 0) == gpu.digest_host(want_other)
    finally:
        for c, t in (("rplwide", 0), ("rplwide", 3), ("rplalone", 0)):
            gpu.remove_vhost_scsi_target(c, t)
        gpu.remove_vhost_controller("rplwide")
        gpu.remove_vhost_controller("rplalone")
        for nm in (name, plain, other):
            gpu.delete_bdev(nm)


# ---- GPU: refusals --------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.timeout(180)
def test_replace_refusals(gpu, exporters):
    nb, bs = 1024, 512
    ex = exporters()
    h1, h2 = ex.make("a1", nb, bs), ex.make("a2", nb, bs)
    plain = gpu.construct_malloc_bdev(nb, bs, name="rplrefplain", device=0)
    local = gpu.construct_mirror_bdev(nb, bs, [0, 0], name="rplreflocal")
    name = gpu.construct_mirror_bdev_remote(nb, bs, 0, [h1, h2], name="rplref")
    gpu.construct_vhost_scsi_controller("rplref")
    gpu.add_vhost_scsi_lun("rplref", 0, name)
    want = np.zeros(nb * bs, np.uint8)
    buf = _pinned(1 << 20)
    try:
        h3 = ex.make("a3", nb, bs)
        _refused(gpu, -errno.ENOTSUP, local, 1, h3)
        _refused(gpu, -errno.ENOTSUP, plain, 1, h3)
        _refused(gpu, -errno.ENODEV, "nope", 1, h3)
        for rep in (0, 3, -1):
            _refused(gpu, -errno.EINVAL, name, rep, h3)
        _refused(gpu, -errno.EINVAL, name, 1, h1)          # the handle the replica has
        _refused(gpu, -errno.EINVAL, name, 1, h2)          # another replica's
        with gpu.Lun("rplref", 0, num_queues=1, queue_size=64) as lun:
            _write(lun, 0, want, buf, 10, 16, bs, 1)
            _refused(gpu, -errno.EIO, name, 1, bytes(range(64)))     # not a handle: nothing changes
            assert _replica_info(gpu, name, 1) == (0, 1)
            _write(lun, 0, want, buf, 500, 16, bs, 2)
        d = gpu.digest_host(want)
        assert ex.digest("a1") == ex.digest("a2") == gpu.bdev_digest(name, 0) == d, "the mirror after a refused replace"
        assert ex.digest("a3") == gpu.digest_host(np.zeros(nb * bs, np.uint8)), "a refused replace wrote the new store"
        # an NBD export serving the mirror: -EBUSY while it runs, a replace once it ended
        a, b = socket.socketpair()
        a.settimeout(20)
        rc = []

        def serve():
            rc.append(gpu.load().oimgpu_nbd_serve(name.encode(), b.fileno()))
            b.close()
        th = threading.Thread(target=serve, daemon=True)
        th.start()
        try:
            a.sendall((0x25609513).to_bytes(4, "big") + (3).to_bytes(4, "big") + b"rplflush" + bytes(12))
            reply = b""
            while len(reply) < 16:
                reply += a.recv(16 - len(reply))
            assert reply[8:] == b"rplflush"              # answered: the export is in its loop
            _refused(gpu, -errno.EBUSY, name, 1, h3)
        finally:
            a.close()
            th.join(20)
        assert rc == [0]
        gpu.mirror_replace_remote(name, 1, h3)
        assert ex.digest("a3") == d and gpu.mirror_check(name)["mismatched_blocks"] == 0
        _refused(gpu, -errno.EINVAL, name, 2, h3)          # now replica 1's
    finally:
        gpu.remove_vhost_scsi_target("rplref", 0)
        gpu.remove_vhost_controller("rplref")
        for nm in (name, local, plain):
            gpu.delete_bdev(nm)


# ---- GPU: the documented drain sequence -----------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.timeout(300)
def test_drain_sequence_through_three_daemons(gpu, daemons):
    """INTEGRATION.md 3c: vol7 on gpu0.sock mirrors onto vol7-r1 of gpu1.sock; vol7-r1b is made on gpu2.sock and
    replaces it; then gpu1.sock deletes vol7-r1 while the mirror lives.  A saved configuration restores the mirror
    onto the new store in a fresh daemon"""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import oimcfg
    nb, bs = 8192, 4096
    gpu1, gpu2, gpu0 = daemons("gpu1", ["--gpus", "0"]), daemons("gpu2", ["--gpus", "0"]), daemons("gpu0", ["--gpus", "0"])
    assert rpc(gpu1, "construct_malloc_bdev", {"num_blocks": nb, "block_size": bs, "name": "vol7-r1"}) == "vol7-r1"
    old = rpc(gpu1, "export_bdev_store", {"name": "vol7-r1"})
    assert rpc(gpu0, "construct_mirror_bdev", {"name": "vol7", "num_blocks": nb, "block_size": bs, "uuid": UUID,
                                               "remote_replicas": [old]}) == "vol7"
    local = gpu.construct_mirror_bdev_remote(nb, bs, 0, [base64.b64decode(rpc(gpu0, "export_bdev_store", {"name": "vol7"}))],
                                             name="vol7-writer")
    try:
        gpu.bdev_write_raw(local, 0, traces.pattern_bytes(70, 0, nb * bs), replica=1)       # vol7's replica 0
    finally:
        gpu.delete_bdev(local)
    assert rpc(gpu0, "check_mirror_bdev", {"name": "vol7", "repair": True})["repaired_blocks"] == nb
    listing = rpc(gpu0, "get_bdevs", {"name": "vol7"})
    # on gpu2.sock
    assert rpc(gpu2, "construct_malloc_bdev", {"num_blocks": nb, "block_size": bs, "name": "vol7-r1b"}) == "vol7-r1b"
    new = rpc(gpu2, "export_bdev_store", {"name": "vol7-r1b"})
    # on gpu0.sock: refusals first, then the move
    assert rpc(gpu0, "replace_mirror_replica", {"name": "vol7", "replica": 1, "remote_replica": old}) == \
        {"error": {"code": -32602, "message": "Invalid argument"}}
    assert rpc(gpu0, "replace_mirror_replica", {"name": "vol7", "replica": 2, "remote_replica": new}) == \
        {"error": {"code": -32602, "message": "Invalid argument"}}
    assert rpc(gpu0, "replace_mirror_replica", {"name": "vol7", "replica": 1,
                                                "remote_replica": base64.b64encode(bytes(range(64))).decode()}) == \
        {"error": {"code": -32602, "message": "Input/output error"}}
    assert rpc(gpu0, "replace_mirror_replica", {"name": "vol7", "replica": 1, "remote_replica": new}) is True
    assert rpc(gpu0, "get_bdevs", {"name": "vol7"}) == listing
    assert listing[0]["driver_specific"] == mirror_entry([(0, False), (0, True)])
    clean = rpc(gpu0, "check_mirror_bdev", {"name": "vol7"})
    assert (clean["mismatched_blocks"], clean["mismatches"]) == (0, [])
    # on gpu1.sock: the old exporter goes before the mirror
    assert rpc(gpu1, "delete_bdev", {"name": "vol7-r1"}) is True
    assert rpc(gpu0, "check_mirror_bdev", {"name": "vol7"})["mismatched_blocks"] == 0
    assert replica_digests(gpu, gpu2, "vol7-r1b", 1, nb, bs) == [gpu.digest_host(traces.pattern_bytes(70, 0, nb * bs))]
    cfg = [x for x in rpc(gpu0, "get_subsystem_config", {"name": "bdev"}) if x["method"] == "construct_mirror_bdev"]
    assert cfg == [{"method": "construct_mirror_bdev", "params": {"name": "vol7", "num_blocks": nb, "block_size": bs,
                                                                  "uuid": UUID, "remote_replicas": [new]}}]
    saved = oimcfg.save(oimcfg.Rpc(gpu0.rpc))
    fresh = daemons("fresh", ["--gpus", "0"])
    rf = oimcfg.Rpc(fresh.rpc)
    oimcfg.load(rf, json.loads(json.dumps(saved)))
    assert rpc(fresh, "get_bdevs", {"name": "vol7"}) == listing
    assert [x for x in rpc(fresh, "get_subsystem_config", {"name": "bdev"}) if x["method"] == "construct_mirror_bdev"] == cfg
    assert rpc(fresh, "delete_bdev", {"name": "vol7"}) is True
    assert rpc(gpu0, "delete_bdev", {"name": "vol7"}) is True
    assert rpc(gpu2, "delete_bdev", {"name": "vol7-r1b"}) is True


# ---- GPU: a new store on a second GPU -------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.timeout(240)
def test_new_replica_on_a_second_gpu(gpu, exporters):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    nb, bs = 1 << 16, 4096
    ex0, ex1 = exporters([0]), exporters([1])
    old = ex0.make("old", nb, bs)
    fresh = ex1.make("fresh", nb, bs, device=1, seed=3)
    name = gpu.construct_mirror_bdev_remote(nb, bs, 0, [old], name="rpl2gpu")
    gpu.construct_vhost_scsi_controller("rpl2gpu")
    gpu.add_vhost_scsi_lun("rpl2gpu", 0, name)
    rng = np.random.default_rng(2)
    want = np.zeros(nb * bs, np.uint8)
    buf = _pinned(1 << 20)
    try:
        with gpu.Lun("rpl2gpu", 0, num_queues=1, queue_size=64) as lun:
            _writes(lun, 0, want, buf, nb, bs, rng, 10)
            gpu.mirror_replace_remote(name, 1, fresh)
            assert _replica_info(gpu, name, 1) == (0, 1), "the replica is reached from replica 0's GPU"
            assert ex1.digest("fresh") == gpu.digest_host(want)
            _writes(lun, 0, want, buf, nb, bs, rng, 6)
        d = gpu.digest_host(want)
        assert ex1.digest("fresh") == d == gpu.bdev_digest(name, 0)
        assert gpu.mirror_check(name)["mismatched_blocks"] == 0
    finally:
        gpu.remove_vhost_scsi_target("rpl2gpu", 0)
        gpu.remove_vhost_controller("rpl2gpu")
        gpu.delete_bdev(name)
