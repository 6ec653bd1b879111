"""The oimgpu bdev module (integration/spdk/bdev_oimgpu.c): a bdev in SPDK's own bdev layer whose store is an oimgpu
bdev in HBM, served by oim_bio_kernel through a block-I/O channel (include/oimgpu.h, oimgpu_bio_chan).

The driver (integration/spdk/bdev_oimgpu_driver.c) links the reference's bdev layer, Malloc bdev and thread library;
the reference's Malloc bdev on the memcpy engine is the checker for every byte and status of the module.  The
channel itself is also driven from Python through the C ABI."""
import contextlib
import ctypes as C
import errno
import glob
import json
import os
import re
import signal
import socket
import subprocess
import time

import numpy as np
import pytest

from oim_b200 import abi, build, lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DRIVER = os.path.join(ROOT, "oracle", "_ref", "spdk", "bdev_oimgpu_driver")
MEMCPY = {"OIMGPU_COPY_ENGINE": "off"}


def _driver():
    if os.path.isdir("/root/reference/vendor/github.com/spdk/spdk"):
        build.build()
        r = subprocess.run(["make", "-s", "-C", os.path.join(ROOT, "integration", "spdk")], capture_output=True, text=True)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    if not os.path.exists(DRIVER):
        pytest.skip("oracle/_ref/spdk/bdev_oimgpu_driver not built (needs the reference tree at build time)")
    return DRIVER


def _run(bdev, *args, env=None, timeout=240):
    r = subprocess.run([_driver(), "--bdev", bdev, *map(str, args)], capture_output=True, text=True, timeout=timeout,
                       env={**os.environ, **(env or {})})
    assert r.returncode == 0, r.stdout[-1500:] + r.stderr[-1500:]
    return r.stdout.strip().splitlines()[-1]


# ---- CPU: RPCs and config on a control-only library ----------------------------------------------------------

class _Rpc:
    def __init__(self, path):
        self.s = socket.socket(socket.AF_UNIX, socket.SOCK_STREAM)
        t0 = time.time()
        while True:
            try:
                self.s.connect(path)
                break
            except (ConnectionRefusedError, FileNotFoundError):
                assert time.time() - t0 < 10
                time.sleep(0.01)
        self.id = 0

    def call(self, method, params=None):
        self.id += 1
        req = {"jsonrpc": "2.0", "method": method, "id": self.id}
        if params is not None:
            req["params"] = params
        self.s.sendall((json.dumps(req) + "\n").encode())
        buf = b""
        while True:
            buf += self.s.recv(1 << 20)
            try:
                return json.loads(buf)
            except ValueError:
                continue


class _Server:
    def __init__(self, sock_dir, name):
        self.path = os.path.join(sock_dir, name)
        self.p = subprocess.Popen([_driver(), "--bdev", "oimgpu", "rpc", self.path], stdout=subprocess.PIPE,
                                  stderr=subprocess.PIPE, text=True, env={**os.environ, **MEMCPY, "OIMGPU_CONTROL_ONLY": "1"})
        self.c = _Rpc(self.path)

    def close(self):
        self.p.send_signal(signal.SIGTERM)
        self.p.communicate(timeout=20)


@pytest.fixture()
def server(sock_tmp):
    s = _Server(sock_tmp, "a.sock")
    yield s
    s.close()


def _strip(b):
    return {k: v for k, v in b.items() if k not in ("name", "uuid", "product_name")}


def test_construct_oimgpu_bdev_replies_equal_construct_malloc_bdev(server):
    c = server.c
    u = "7f3d2c1a-0000-4000-8000-000000000001"
    cases = [
        {"num_blocks": 0, "block_size": 512},
        {"num_blocks": 16, "block_size": 512, "uuid": "not-a-uuid"},
        {"num_blocks": 16},
        {"block_size": 512},
        {"name": 7, "num_blocks": 16, "block_size": 512},
    ]
    for p in cases:
        want = c.call("construct_malloc_bdev", p)
        got = c.call("construct_oimgpu_bdev", p)
        assert "error" in want and got["error"] == want["error"], (p, got, want)
    assert c.call("construct_oimgpu_bdev", None)["error"] == c.call("construct_malloc_bdev", None)["error"]
    # success returns the name; a name in use (either module's) is refused the same way
    assert c.call("construct_oimgpu_bdev", {"name": "G0", "num_blocks": 2048, "block_size": 4096, "uuid": u})["result"] == "G0"
    assert c.call("construct_malloc_bdev", {"name": "M0", "num_blocks": 2048, "block_size": 4096})["result"] == "M0"
    for name in ("G0", "M0"):
        p = {"name": name, "num_blocks": 16, "block_size": 512}
        assert c.call("construct_oimgpu_bdev", p)["error"] == c.call("construct_malloc_bdev", p)["error"]
    g = c.call("get_bdevs", {"name": "G0"})["result"][0]
    m = c.call("get_bdevs", {"name": "M0"})["result"][0]
    assert g["product_name"] == "OimGpu disk" and m["product_name"] == "Malloc disk" and g["uuid"] == u
    assert _strip(g) == _strip(m)
    # auto name
    assert c.call("construct_oimgpu_bdev", {"num_blocks": 8, "block_size": 512})["result"] == "OimGpu0"
    # delete: true, then the bdev is gone; unknown names and missing params as delete_malloc_bdev
    assert c.call("delete_oimgpu_bdev", {"name": "G0"})["result"] is True
    assert c.call("get_bdevs", {"name": "G0"})["error"]["code"] == -32602
    for p in ({"name": "nope"}, {}, None):
        assert c.call("delete_oimgpu_bdev", p)["error"] == c.call("delete_malloc_bdev", p)["error"]
    # a bdev of the other module is not this module's to delete
    assert c.call("delete_oimgpu_bdev", {"name": "M0"})["result"] == c.call("delete_malloc_bdev", {"name": "OimGpu0"})["result"] is False


def test_config_emits_construct_oimgpu_bdev_and_replays(sock_tmp):
    specs = [("Cfg0", 1024, 512, "7f3d2c1a-0000-4000-8000-00000000000a"), ("Cfg1", 100, 520, "7f3d2c1a-0000-4000-8000-00000000000b")]
    out = _run("oimgpu", "config", *[":".join(map(str, s)) for s in specs], env={**MEMCPY, "OIMGPU_CONTROL_ONLY": "1"})
    cfg = json.loads(out)
    calls = [x for x in cfg if x["method"] == "construct_oimgpu_bdev"]
    assert [c["params"] for c in calls] == [{"name": n, "num_blocks": nb, "block_size": bs, "uuid": u} for n, nb, bs, u in specs]
    a, b = _Server(sock_tmp, "a.sock"), _Server(sock_tmp, "b.sock")
    try:
        for n, nb, bs, u in specs:
            a.c.call("construct_oimgpu_bdev", {"name": n, "num_blocks": nb, "block_size": bs, "uuid": u})
        for x in cfg:
            if x["method"] != "set_bdev_options":
                assert "result" in b.c.call(x["method"], x["params"])
        assert a.c.call("get_bdevs")["result"] == b.c.call("get_bdevs")["result"]
    finally:
        a.close()
        b.close()


# ---- CPU: the C ABI without a GPU ---------------------------------------------------------------------------

def test_bio_chan_abi_without_gpu():
    L = lib.load()
    h = C.c_void_p()
    cpl = np.zeros(4, dtype=abi.bio_cpl_dtype)
    assert L.oimgpu_bio_chan_open(None, C.byref(h)) == -errno.EINVAL
    assert L.oimgpu_bio_chan_open(b"x", None) == -errno.EINVAL
    assert L.oimgpu_bio_chan_submit(None, None, 0, None, 0) == -errno.EINVAL
    assert L.oimgpu_bio_chan_poll(None, cpl.ctypes.data, 4) == -errno.EINVAL
    assert L.oimgpu_bio_chan_close(None) == -errno.EINVAL
    assert L.oimgpu_bio_chan_launches(None) == 0
    if glob.glob("/dev/nvidia[0-9]*"):
        return      # below: a library that never found a GPU
    assert L.oimgpu_bio_chan_open(b"x", C.byref(h)) == -errno.ENODEV
    assert L.oimgpu_init_control_only() == 0
    try:
        lib.construct_malloc_bdev(16, 512, name="CtlOnly0")
        assert L.oimgpu_bio_chan_open(b"CtlOnly0", C.byref(h)) == -errno.ENODEV
    finally:
        lib.fini()


def test_bio_kernel_compiles_for_sm90a_without_spills(tmp_path):
    src = os.path.join(ROOT, "oim_b200", "csrc", "bio_chan.cu")
    r = subprocess.run([build.NVCC, *[f for f in build.FLAGS if f != "-shared"], "-Xptxas", "-v", "-c", src,
                        "-o", str(tmp_path / "bio.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    m = re.search(r"Compiling entry function '(\S*oim_bio_kernel\S*)' for 'sm_90a'.*?(\d+) bytes spill stores, (\d+) bytes spill loads",
                  r.stderr, re.S)
    assert m and m.group(2) == "0" and m.group(3) == "0", r.stderr[-3000:]
    sass = subprocess.run(["/usr/local/cuda/bin/cuobjdump", "-sass", build.build()], capture_output=True, text=True).stdout
    assert re.search(r"Function : \S*oim_bio_kernel", sass)


# ---- GPU: the module under SPDK's bdev layer ------------------------------------------------------------------

@pytest.mark.gpu
def test_bdevio_cases_on_the_oimgpu_bdev_module():
    out = json.loads(_run("oimgpu", "bdevio"))
    assert out["failed"] == 0 and out["cases"] >= 50
    assert out["launches"] > 0 and out["engine_ops"] == 0, out


FUZZ = [(seed, bs) for seed in range(1, 13) for bs in (512, 4096, 520)]


@pytest.mark.gpu
@pytest.mark.parametrize("seed,bs", FUZZ, ids=[f"seed{s}-bs{b}" for s, b in FUZZ])
def test_fuzz_equals_malloc_on_the_memcpy_engine(seed, bs):
    got = json.loads(_run("oimgpu", "fuzz", seed, bs))
    want = json.loads(_run("malloc", "fuzz", seed, bs, env=MEMCPY))
    assert got["status"] == want["status"]
    assert got["reads"] == want["reads"]
    assert got["device"] == want["device"]
    assert "F" in got["status"] and "R" in got["status"]
    # many I/Os per launch: one poller tick sends a whole round
    assert 0 < got["launches"] < len(got["status"]) and got["engine_ops"] == 0


@pytest.mark.gpu
@pytest.mark.parametrize("seed,bs", [(21, 512), (22, 4096), (23, 520)])
def test_two_spdk_threads_equal_the_reference(seed, bs):
    got = json.loads(_run("oimgpu", "fuzz", seed, bs, 2))
    want = json.loads(_run("malloc", "fuzz", seed, bs, 2, env=MEMCPY))
    assert (got["status"], got["reads"], got["device"]) == (want["status"], want["reads"], want["device"])


# ---- GPU: the channel through the C ABI ---------------------------------------------------------------------

def _bios(*rows):
    b = np.zeros(len(rows), dtype=abi.bio_dtype)
    for i, (op, off, nb, start, cnt) in enumerate(rows):
        b[i] = (off, nb, op, start, cnt, 0, i)
    return b


def _host(n, fill=0):
    """n bytes of host memory starting on a page of their own, with no other buffer in their last page"""
    raw = np.full(n + 3 * 4096, fill, dtype=np.uint8)
    off = (-raw.ctypes.data) % 4096
    return raw[off:off + n]


@contextlib.contextmanager
def _registered(*arrays):
    """_host buffers registered for the GPU for the duration (oimgpu_mem_register, whole pages): the channel then
    pins nothing of this process's heap that a later pageable copy could straddle"""
    L = lib.load()
    for a in arrays:
        assert L.oimgpu_mem_register(a.ctypes.data, (a.nbytes + 4095) // 4096 * 4096) == 0
    try:
        yield
    finally:
        for a in arrays:
            L.oimgpu_mem_unregister(a.ctypes.data)


def _iovs(pieces):
    v = np.zeros(max(1, len(pieces)), dtype=abi.iov_dtype)
    for i, (a, n) in enumerate(pieces):
        v[i]["addr"], v[i]["len"] = a, n
    return v


@pytest.mark.gpu
@pytest.mark.parametrize("bs", [512, 520])
def test_alignment_sweep_keeps_guard_bytes(gpu, bs):
    """every client address mod 16 x byte lengths around a 4 KiB unit: the iovec of that length sits at that
    address, the rest of the bio's bytes in a second iovec; write, read back, guards untouched"""
    nb_dev = 4096
    name = gpu.construct_malloc_bdev(nb_dev, bs, name=f"BioAlign{bs}")
    rng = np.random.default_rng(bs)
    lengths = [1, 15, 16, 17, 4095, 4096, 4097, 3 * 4096 + 77]
    size = 2 * (3 * 4096 + 77) + 3 * bs + 128
    src, dst = _host(size), _host(size)
    try:
        with _registered(src, dst), gpu.BioChan(name) as ch:
            lba = 0
            for mod in range(16):
                for n in lengths:
                    nblk = (n + bs - 1) // bs + 1
                    total = nblk * bs
                    src[:] = rng.integers(0, 256, size, dtype=np.uint8)
                    dst[:] = 0xA5
                    base_s, base_d = src.ctypes.data, dst.ctypes.data
                    sa = ((base_s + 15) & ~15) - base_s + mod      # index of the element whose address is mod 16
                    da = ((base_d + 15) & ~15) - base_d + mod
                    wr = _iovs([(base_s + sa, n), (base_s + sa + n + 3, total - n)])
                    rd = _iovs([(base_d + da, n), (base_d + da + n + 3, total - n)])
                    ch.submit(_bios((abi.BIO_WRITE, lba, nblk, 0, 2)), wr)
                    ch.submit(_bios((abi.BIO_READ, lba, nblk, 0, 2)), rd)
                    c = ch.wait(2)
                    assert (c["status"] == 0).all()
                    want = np.concatenate([src[sa:sa + n], src[sa + n + 3:sa + n + 3 + total - n]])
                    assert (gpu.bdev_read_raw(name, lba * bs, total) == want).all(), (mod, n)
                    assert (dst[da:da + n] == src[sa:sa + n]).all() and (dst[da + n + 3:da + total + 3] == want[n:]).all()
                    guard = np.ones(size, dtype=bool)
                    guard[da:da + n] = False
                    guard[da + n + 3:da + total + 3] = False
                    assert (dst[guard] == 0xA5).all(), (mod, n)
                    lba = (lba + nblk) % (nb_dev - 64)
            assert ch.launches > 0
    finally:
        gpu.delete_bdev(name)


@pytest.mark.gpu
def test_exactly_the_bios_bytes_move_and_bad_bios_move_nothing(gpu):
    bs, nb = 512, 256
    name = gpu.construct_malloc_bdev(nb, bs, name="BioEdge")
    try:
        gpu.bdev_write_raw(name, 0, np.full(nb * bs, 0x11, dtype=np.uint8))
        src, dst = _host(4 * bs, 0x77), _host(4 * bs, 0x33)
        with _registered(src, dst), gpu.BioChan(name) as ch:
            # iovecs holding more than the bio: exactly num_blocks x block_size bytes move, both ways
            ch.submit(_bios((abi.BIO_WRITE, 10, 2, 0, 1), (abi.BIO_READ, 20, 2, 1, 1)),
                      _iovs([(src.ctypes.data, 4 * bs), (dst.ctypes.data, 4 * bs)]))
            assert (ch.wait(2)["status"] == 0).all()
            store = gpu.bdev_read_raw(name, 0, nb * bs)
            assert (store[10 * bs:12 * bs] == 0x77).all() and (store[12 * bs:] != 0x77).all()
            assert (dst[:2 * bs] == 0x11).all() and (dst[2 * bs:] == 0x33).all()
            before = gpu.bdev_read_raw(name, 0, nb * bs)
            bad = np.zeros(6, dtype=abi.bio_dtype)
            bad[0] = (nb - 1, 2, abi.BIO_WRITE, 0, 1, 0, 0)          # past the end
            bad[1] = (0, 1, 7, 0, 1, 0, 1)                           # bad op
            bad[2] = (0, 1, abi.BIO_WRITE, 1, 1, 0, 2)               # iovec beyond the table
            bad[3] = (0, 8, abi.BIO_WRITE, 0, 1, 0, 3)               # iovecs sum to fewer bytes
            bad[4] = (2 ** 64 - 1, 2, abi.BIO_UNMAP, 0, 0, 0, 4)     # wraps
            bad[5] = (0, 1, abi.BIO_READ, 0, 1, 1, 5)                # reserved flags
            ch.submit(bad, _iovs([(src.ctypes.data, 4 * bs)]))
            c = ch.wait(6)
            assert list(c["tag"]) == list(range(6)) and (c["status"] == -errno.EINVAL).all()
            assert (gpu.bdev_read_raw(name, 0, nb * bs) == before).all()
            # WRITE_ZEROES and UNMAP fill with 0x00
            ch.submit(_bios((abi.BIO_WRITE_ZEROES, 0, 3, 0, 0), (abi.BIO_UNMAP, 100, 5, 0, 0)), _iovs([]))
            assert (ch.wait(2)["status"] == 0).all()
            store = gpu.bdev_read_raw(name, 0, nb * bs)
            assert (store[:3 * bs] == 0).all() and (store[100 * bs:105 * bs] == 0).all() and store[3 * bs] == 0x11
    finally:
        gpu.delete_bdev(name)


@pytest.mark.gpu
def test_overlapping_bios_in_one_batch_take_effect_in_order(gpu):
    bs = 4096
    name = gpu.construct_malloc_bdev(64, bs, name="BioOrder")
    try:
        a, b = _host(8 * bs, 0xAA), _host(8 * bs, 0xBB)
        r1, r2, r3 = _host(12 * bs), _host(4 * bs), _host(4 * bs)
        with _registered(a, b, r1, r2, r3), gpu.BioChan(name) as ch:
            l0 = ch.launches
            # W[0,8) A; R[0,12) after it; W[4,12) B; R[40,44) (no conflict); W[8,10) zeroes; R[6,10)
            ch.submit(_bios((abi.BIO_WRITE, 0, 8, 0, 1), (abi.BIO_READ, 0, 12, 1, 1), (abi.BIO_WRITE, 4, 8, 2, 1),
                            (abi.BIO_READ, 40, 4, 3, 1), (abi.BIO_WRITE_ZEROES, 8, 2, 0, 0), (abi.BIO_READ, 6, 4, 4, 1)),
                      _iovs([(a.ctypes.data, 8 * bs), (r1.ctypes.data, 12 * bs), (b.ctypes.data, 8 * bs),
                             (r3.ctypes.data, 4 * bs), (r2.ctypes.data, 4 * bs)]))
            assert (ch.wait(6)["status"] == 0).all()
            assert ch.launches - l0 == 5        # W | R | W R(40) | Z | R
        assert (r1[:8 * bs] == 0xAA).all() and (r1[8 * bs:] == 0).all()
        assert (r2[:2 * bs] == 0xBB).all() and (r2[2 * bs:] == 0).all()
        store = gpu.bdev_read_raw(name, 0, 12 * bs)
        assert (store[:4 * bs] == 0xAA).all() and (store[4 * bs:8 * bs] == 0xBB).all()
        assert (store[8 * bs:10 * bs] == 0).all() and (store[10 * bs:] == 0xBB).all()
    finally:
        gpu.delete_bdev(name)


@pytest.mark.gpu
def test_lifecycle_busy_mirror_refused_close_waits(gpu):
    import torch
    name = gpu.construct_malloc_bdev(1 << 17, 4096, name="BioLife")      # 512 MiB
    try:
        ch = gpu.BioChan(name)
        with pytest.raises(lib.OimGpuError) as e:
            gpu.delete_bdev(name)
        assert e.value.rc == -errno.EBUSY
        src = torch.full((1 << 29,), 0x5C, dtype=torch.uint8, device="cuda:0")
        ch.submit(_bios((abi.BIO_WRITE, 0, 1 << 17, 0, 1)), _iovs([(src.data_ptr(), 1 << 29)]))
        ch.close()                      # returns once the write is done
        d = gpu.bdev_digest(name)
        assert d == gpu.digest_host(np.full(1 << 29, 0x5C, dtype=np.uint8))
    finally:
        gpu.delete_bdev(name)
    m = gpu.construct_mirror_bdev(64, 512, [0, 0], name="BioMirror")     # two replicas on one GPU: still a mirror
    try:
        with pytest.raises(lib.OimGpuError) as e:
            gpu.BioChan(m)
        assert e.value.rc == -errno.ENOTSUP
    finally:
        gpu.delete_bdev(m)


@pytest.mark.gpu
@pytest.mark.parametrize("bs", [512, 4096])
def test_bio_channel_and_scsi_session_see_the_same_volume(gpu, bs):
    """written through a bio channel, read through an oimgpu_lun session with READ(16); and the reverse"""
    nb = 1024
    name = gpu.construct_malloc_bdev(nb, bs, name=f"BioScsi{bs}")
    ctrlr = f"bio_scsi_{bs}"
    gpu.construct_vhost_scsi_controller(ctrlr)
    gpu.add_vhost_scsi_lun(ctrlr, 0, name)
    rng = np.random.default_rng(bs)
    n = 64 * bs
    data, back, data2, back2 = _host(n), _host(n), _host(n), _host(n + 3)
    data[:] = rng.integers(0, 256, n, dtype=np.uint8)
    data2[:] = data[::-1]
    try:
        with _registered(data, back, data2, back2), gpu.Lun(ctrlr, 0) as lun:
            with gpu.BioChan(name) as ch:
                ch.submit(_bios((abi.BIO_WRITE, 100, 64, 0, 3)),
                          _iovs([(data.ctypes.data, 1000), (data.ctypes.data + 1000, 7), (data.ctypes.data + 1007, n - 1007)]))
                assert ch.wait(1)["status"][0] == 0
            batch = abi.Batch(0)
            batch.read(100, 64, [(back.ctypes.data, n)], opcode=abi.READ_16)
            c = lun.run(*batch.arrays())
            assert c[0]["status"] == 0 and (back == data).all()
            # the reverse: WRITE(16) through the session, read through a channel
            batch = abi.Batch(0)
            batch.write(300, 64, [(data2.ctypes.data, n)], opcode=abi.WRITE_16)
            assert lun.run(*batch.arrays())[0]["status"] == 0
            with gpu.BioChan(name) as ch:
                ch.submit(_bios((abi.BIO_READ, 300, 64, 0, 1)), _iovs([(back2.ctypes.data + 3, n)]))
                assert ch.wait(1)["status"][0] == 0
            assert (back2[3:] == data2).all()
    finally:
        gpu.remove_vhost_scsi_target(ctrlr, 0)
        gpu.remove_vhost_controller(ctrlr)
        gpu.delete_bdev(name)
