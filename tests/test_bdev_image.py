"""Volume images (oimgpu_bdev_image_save / _load, oim_b200/csrc/bdev_image.cu; the daemon's save_bdev_image and
load_bdev_image; tools/oimcfg.py --images) compared with a numpy model of the format.

`model_image` states the file a store must give: the 4096-byte header, the table of the maximal runs of 4 KiB granules
that hold a non-zero byte (the last one cut at the end of the store), then the runs' bytes.  The format is canonical,
so a save is compared with the model byte for byte.

CPU: the model on hand-built stores, the kernels' ptxas report, the struct layout, the C ABI's and the daemon's answers
without a GPU.  GPU (one H100): round trips at block sizes 512, 520, 4096 and 4097 at three densities, a load over
existing data, a payload of several staging chunks, 2- and 4-way mirrors and a mirror with a replica in another
process, a save between the two halves of a VM's trace (launch per kick and resident poller), every refusal, the
daemon's methods, a daemon restart through oimcfg.py --images, and one 8 GiB volume."""
import base64
import errno
import glob
import json
import os
import re
import socket
import struct
import subprocess
import sys
import threading
import time

import numpy as np
import pytest

from oim_b200 import abi, build, lib, traces
from test_daemon_mirror import IOSTAT, daemons, masked, oracle_run, replica_digests, rpc, vm_trace  # noqa: F401
from test_mirror_replace import vm_run_split

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GRANULE = 4096
UUID = "0123abcd-4567-89ef-0123-456789abcdef"
HEADER = struct.Struct("<8sIIQIIQQQQ36s")


# ---- the model ------------------------------------------------------------------------------------------------

def model_extents(store):
    """the maximal runs of granules holding a non-zero byte -> [(offset_bytes, len_bytes)]"""
    size = store.size
    ngran = (size + GRANULE - 1) // GRANULE
    pad = np.zeros(ngran * GRANULE, dtype=np.uint8)
    pad[:size] = store
    nz = np.concatenate([[False], pad.reshape(ngran, GRANULE).any(axis=1), [False]])
    edges = np.nonzero(nz[1:] != nz[:-1])[0]
    return [(int(s) * GRANULE, min(int(e) * GRANULE, size) - int(s) * GRANULE) for s, e in zip(edges[::2], edges[1::2])]


def model_digest(store):
    """oimgpu_bdev_digest over the whole store, the last word zero-padded"""
    pad = np.zeros((store.size + 7) // 8 * 8, dtype=np.uint8)
    pad[:store.size] = store
    return lib.digest_host(pad)


def model_image(store, block_size, uuid=UUID) -> bytes:
    store = np.asarray(store, dtype=np.uint8)
    assert store.size % block_size == 0
    ext = model_extents(store)
    data = b"".join(store[o:o + n].tobytes() for o, n in ext)
    d = model_digest(store)
    head = HEADER.pack(b"OIMGPUIM", 1, block_size, store.size // block_size, GRANULE, 0, len(ext), len(data), d[0], d[1],
                       uuid.encode())
    table = b"".join(struct.pack("<QQ", o, n) for o, n in ext)
    return head.ljust(4096, b"\0") + table.ljust((len(table) + 4095) // 4096 * 4096, b"\0") + data


def parse_image(blob: bytes):
    """-> (header fields, extents, store) of an image"""
    magic, ver, bs, nb, gran, res, n, data_bytes, d0, d1, uuid = HEADER.unpack_from(blob)
    ext = [struct.unpack_from("<QQ", blob, 4096 + 16 * i) for i in range(n)]
    pos = 4096 + (16 * n + 4095) // 4096 * 4096
    store = np.zeros(nb * bs, dtype=np.uint8)
    for o, ln in ext:
        store[o:o + ln] = np.frombuffer(blob, np.uint8, ln, pos)
        pos += ln
    assert pos == len(blob)
    return {"magic": magic, "version": ver, "block_size": bs, "num_blocks": nb, "granule_bytes": gran, "reserved": res,
            "nextents": n, "data_bytes": data_bytes, "digest": (d0, d1), "uuid": uuid.decode()}, ext, store


def content(kind, nb, bs, seed):
    """a store of nb x bs bytes: empty, a few scattered pieces (edges of granules and of the store included), or dense"""
    rng = np.random.default_rng(seed)
    size = nb * bs
    s = np.zeros(size, dtype=np.uint8)
    if kind == "dense":
        s[:] = rng.integers(0, 256, size=size, dtype=np.uint8)
        s[s == 0] = 1
    elif kind == "sparse":
        for pos, n in [(0, 1), (GRANULE - 1, 2), (3 * GRANULE, GRANULE), (size - 1, 1)]:
            s[pos:pos + n] = 0x5A
        for pos in rng.integers(0, size, size=40):
            n = int(rng.integers(1, 200))
            s[pos:pos + n] = rng.integers(1, 256, size=min(n, size - pos), dtype=np.uint8)
    return s


def test_model_runs_are_maximal_and_not_adjacent():
    s = np.zeros(10 * GRANULE, dtype=np.uint8)
    s[GRANULE + 5] = 1                      # granule 1
    s[2 * GRANULE] = 1                      # granule 2: joins 1
    s[5 * GRANULE - 1] = 1                  # granule 4
    s[9 * GRANULE] = 1                      # granule 9, the last
    assert model_extents(s) == [(GRANULE, 2 * GRANULE), (4 * GRANULE, GRANULE), (9 * GRANULE, GRANULE)]
    assert model_extents(np.zeros(3 * GRANULE, np.uint8)) == []
    assert model_extents(np.ones(3 * GRANULE, np.uint8)) == [(0, 3 * GRANULE)]
    blob = model_image(s, 512)
    assert len(blob) == 4096 + 4096 + 4 * GRANULE
    h, ext, back = parse_image(blob)
    assert (h["nextents"], h["data_bytes"], ext) == (3, 4 * GRANULE, model_extents(s)) and (back == s).all()


@pytest.mark.parametrize("bs,nb", [(520, 17), (4097, 3), (520, 1)])
def test_model_partial_last_granule(bs, nb):
    """a store whose size is not a multiple of 4096: the last run ends at the end of the store"""
    size = bs * nb
    assert size % GRANULE
    s = np.zeros(size, dtype=np.uint8)
    s[-1] = 7
    ext = model_extents(s)
    last = (size - 1) // GRANULE * GRANULE
    assert ext == [(last, size - last)]
    s[:] = 3
    assert model_extents(s) == [(0, size)]
    h, ext, back = parse_image(model_image(s, bs))
    assert (h["block_size"], h["num_blocks"], h["data_bytes"]) == (bs, nb, size) and (back == s).all()


def test_model_digest_with_an_odd_tail():
    """the digest's last word is zero-padded: the digest of the 13-byte store equals the position-keyed sums written
    out by hand"""
    s = np.arange(1, 14, dtype=np.uint8)
    mask = (1 << 64) - 1

    def mix(z):
        z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & mask
        z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & mask
        return z ^ (z >> 31)
    w = [int.from_bytes(bytes(s[:8]), "little"), int.from_bytes(bytes(s[8:]) + b"\0\0\0", "little")]
    want = (sum(x * (2 * i + 1) for i, x in enumerate(w)) & mask, sum(mix(x ^ i) for i, x in enumerate(w)) & mask)
    assert model_digest(s) == want
    h, _, _ = parse_image(model_image(np.resize(s, 13 * 40), 13))
    assert h["digest"] == model_digest(np.resize(s, 13 * 40))


# ---- CPU: the kernels, the C ABI and the daemon without a GPU -------------------------------------------------------

def test_image_kernels_compile_for_sm90a_without_spills(tmp_path):
    src = os.path.join(ROOT, "oim_b200", "csrc", "bdev_image.cu")
    r = subprocess.run([build.NVCC, *[f for f in build.FLAGS if f != "-shared"], "-Xptxas", "-v", "-c", src,
                        "-o", str(tmp_path / "bdev_image.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    for k in ("oim_image_scan_kernel", "oim_image_move_kernel"):
        m = re.search(rf"Compiling entry function '(\S*{k}\S*)' for 'sm_90a'.*?(\d+) bytes stack frame, (\d+) bytes spill stores, "
                      r"(\d+) bytes spill loads", r.stderr, re.S)
        assert m and m.group(2) == "0" and m.group(3) == "0" and m.group(4) == "0", (k, r.stderr[-3000:])
    sass = subprocess.run(["/usr/local/cuda/bin/cuobjdump", "-sass", build.build()], capture_output=True, text=True).stdout
    for k in ("oim_image_scan_kernel", "oim_image_move_kernel"):
        assert re.search(rf"Function : \S*{k}", sass), k


def test_image_info_struct_matches_c(tmp_path):
    probe = tmp_path / "probe.c"
    probe.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "oimgpu.h"\n'
                     "#define O(f) offsetof(struct oimgpu_image_info, f)\n"
                     'int main(void){printf("%zu %zu %zu %zu %zu\\n",sizeof(struct oimgpu_image_info),O(file_bytes),'
                     "O(block_size),O(granule_bytes),O(uuid));return 0;}\n")
    exe = tmp_path / "probe"
    subprocess.run(["cc", "-I", os.path.join(ROOT, "include"), str(probe), "-o", str(exe)], check=True)
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    d = abi.image_info_dtype
    assert got == [d.itemsize] + [d.fields[f][1] for f in ("file_bytes", "block_size", "granule_bytes", "uuid")]


def test_image_abi_without_gpu(tmp_path):
    L = lib.load()
    out = np.zeros(1, dtype=abi.image_info_dtype)
    p = str(tmp_path / "x.img").encode()
    for fn in (L.oimgpu_bdev_image_save, L.oimgpu_bdev_image_load):
        assert fn(None, p, out.ctypes.data) == -errno.EINVAL
        assert fn(b"x", None, out.ctypes.data) == -errno.EINVAL
        assert fn(b"x", p, None) == -errno.EINVAL
    if glob.glob("/dev/nvidia[0-9]*"):
        return      # below: a library that never found a GPU
    for fn in (L.oimgpu_bdev_image_save, L.oimgpu_bdev_image_load):
        assert fn(b"x", p, out.ctypes.data) == -errno.ENODEV
    assert L.oimgpu_init_control_only() == 0
    try:
        name = lib.construct_malloc_bdev(64, 512, name="CtlImage")
        for nm in (name, "nope"):
            for fn in (L.oimgpu_bdev_image_save, L.oimgpu_bdev_image_load):
                assert fn(nm.encode(), p, out.ctypes.data) == -errno.ENODEV
    finally:
        lib.fini()
    assert not os.path.exists(p)


def test_image_methods_without_a_gpu(daemons, tmp_path):
    s = daemons("ours", ["--control-only"])
    rpc(s, "construct_malloc_bdev", {"num_blocks": 64, "block_size": 512, "name": "V"})
    nodev = {"code": -32602, "message": "No such device"}
    bad = {"code": -32602, "message": "Invalid parameters"}
    for m in ("save_bdev_image", "load_bdev_image"):
        for p in ({"name": "V", "path": str(tmp_path / "v.img")}, {"name": "nope", "path": str(tmp_path / "n.img")}):
            assert rpc(s, m, p) == {"error": nodev}, (m, p)
        for p in ({}, {"name": "V"}, {"path": "/x"}, {"name": 1, "path": "/x"}, {"name": "V", "path": 2},
                  {"name": "V", "path": "/x", "x": 1}, None):
            assert rpc(s, m, p) == {"error": bad}, (m, p)
    assert not os.listdir(tmp_path)
    cfg = rpc(s, "get_subsystem_config", {"name": "bdev"})
    assert [x["method"] for x in cfg] == ["set_bdev_options", "construct_malloc_bdev"]


# ---- GPU ----------------------------------------------------------------------------------------------------

def _read(path):
    with open(path, "rb") as f:
        return f.read()


def _info_of(blob):
    h, _, _ = parse_image(blob)
    return {"num_blocks": h["num_blocks"], "block_size": h["block_size"], "granule_bytes": GRANULE,
            "nextents": h["nextents"], "data_bytes": h["data_bytes"], "file_bytes": len(blob), "uuid": h["uuid"]}


def _refused(call, rc):
    with pytest.raises(lib.OimGpuError) as e:
        call()
    assert e.value.rc == rc, (e.value.rc, rc)


ROUND = [(bs, kind) for bs in (512, 520, 4096, 4097) for kind in ("empty", "sparse", "dense")]


@pytest.mark.gpu
@pytest.mark.parametrize("bs,kind", ROUND, ids=[f"bs{b}-{k}" for b, k in ROUND])
def test_round_trip_matches_the_model(gpu, tmp_path, bs, kind):
    nb = 2000 if bs < 4096 else 700
    s = content(kind, nb, bs, seed=bs + len(kind))
    src = gpu.construct_malloc_bdev(nb, bs, name=f"src{bs}{kind}", uuid=UUID, device=0)
    dst = gpu.construct_malloc_bdev(nb, bs, name=f"dst{bs}{kind}", device=0)
    try:
        gpu.bdev_write_raw(src, 0, s)
        want = model_image(s, bs)
        info = gpu.bdev_image_save(src, tmp_path / "a.img")
        got = _read(tmp_path / "a.img")
        assert len(got) == len(want) and got[:4096] == want[:4096], "header differs from the model's"
        assert got == want, "table or data differs from the model's"
        assert info == _info_of(want)
        assert gpu.bdev_image_save(src, tmp_path / "b.img") == info
        assert _read(tmp_path / "b.img") == got, "two saves of the same content differ"
        assert gpu.bdev_image_load(dst, tmp_path / "a.img") == info
        assert (gpu.bdev_read_raw(dst, 0, nb * bs) == s).all()
        if (nb * bs) % 8 == 0:
            assert gpu.bdev_digest(dst) == gpu.bdev_digest(src) == model_digest(s)
    finally:
        gpu.delete_bdev(src)
        gpu.delete_bdev(dst)


@pytest.mark.gpu
def test_load_over_existing_data_leaves_the_holes_zero(gpu, tmp_path):
    nb, bs = 3000, 520
    s = content("sparse", nb, bs, seed=5)
    p = tmp_path / "s.img"
    p.write_bytes(model_image(s, bs))
    name = gpu.construct_malloc_bdev(nb, bs, name="over", device=0)
    try:
        gpu.bdev_write_raw(name, 0, np.full(nb * bs, 0xAB, dtype=np.uint8))
        info = gpu.bdev_image_load(name, p)
        assert info["uuid"] == UUID
        assert (gpu.bdev_read_raw(name, 0, nb * bs) == s).all()
    finally:
        gpu.delete_bdev(name)


@pytest.mark.gpu
@pytest.mark.timeout(240)
def test_payload_of_several_staging_chunks(gpu, tmp_path):
    """160 MiB of 4097-byte blocks with a hole every few granules: the extents cross the 64 MiB chunk boundaries"""
    nb, bs = 40000, 4097
    rng = np.random.default_rng(11)
    s = rng.integers(1, 256, size=nb * bs, dtype=np.uint8)
    gran = s[:nb * bs // GRANULE * GRANULE].reshape(-1, GRANULE)
    gran[rng.random(len(gran)) < 0.1] = 0
    src = gpu.construct_malloc_bdev(nb, bs, name="chunks", uuid=UUID, device=0)
    dst = gpu.construct_malloc_bdev(nb, bs, name="chunks2", device=0)
    try:
        gpu.bdev_write_raw(src, 0, s)
        want = model_image(s, bs)
        info = gpu.bdev_image_save(src, tmp_path / "c.img")
        assert info["data_bytes"] > 2 * (64 << 20) and info["nextents"] > 1000
        assert _read(tmp_path / "c.img") == want
        gpu.bdev_image_load(dst, tmp_path / "c.img")
        assert (gpu.bdev_read_raw(dst, 0, nb * bs) == s).all()
    finally:
        gpu.delete_bdev(src)
        gpu.delete_bdev(dst)


@pytest.mark.gpu
@pytest.mark.parametrize("nrep", [2, 4])
def test_mirrors_save_replica_0_and_load_every_replica(gpu, tmp_path, nrep):
    nb, bs = 1500, 4096
    s = content("sparse", nb, bs, seed=nrep)
    src = gpu.construct_mirror_bdev(nb, bs, [0] * nrep, name=f"msrc{nrep}")
    dst = gpu.construct_mirror_bdev(nb, bs, [0] * nrep, name=f"mdst{nrep}")
    try:
        gpu.bdev_write_raw(src, 0, s, replica=0)
        for r in range(1, nrep):                # the other replicas differ: a save reads replica 0 only
            gpu.bdev_write_raw(src, 0, np.full(nb * bs, r, dtype=np.uint8), replica=r)
        for r in range(nrep):
            gpu.bdev_write_raw(dst, 0, np.full(nb * bs, 0x77, dtype=np.uint8), replica=r)
        uuid = gpu.get_bdevs(src)[0]["uuid"]
        gpu.bdev_image_save(src, tmp_path / "m.img")
        assert _read(tmp_path / "m.img") == model_image(s, bs, uuid)
        gpu.bdev_image_load(dst, tmp_path / "m.img")
        for r in range(nrep):
            assert gpu.bdev_digest(dst, r) == model_digest(s), f"replica {r}"
        assert gpu.mirror_check(dst)["mismatched_blocks"] == 0
    finally:
        gpu.delete_bdev(src)
        gpu.delete_bdev(dst)


@pytest.mark.gpu
@pytest.mark.timeout(180)
def test_load_into_a_mirror_with_a_replica_in_another_process(gpu, daemons, tmp_path):
    nb, bs = 2048, 4096
    s = content("dense", nb, bs, seed=3)
    s[100 * GRANULE:900 * GRANULE] = 0
    p = tmp_path / "r.img"
    p.write_bytes(model_image(s, bs))
    b = daemons("b", ["--gpus", "0"])
    assert rpc(b, "construct_malloc_bdev", {"num_blocks": nb, "block_size": bs, "name": "r1"}) == "r1"
    h = base64.b64decode(rpc(b, "export_bdev_store", {"name": "r1"}))
    name = gpu.construct_mirror_bdev_remote(nb, bs, 0, [h], name="remote-mirror")
    try:
        gpu.bdev_write_raw(name, 0, np.full(nb * bs, 9, dtype=np.uint8), replica=1)
        gpu.bdev_image_load(name, p)
        assert gpu.bdev_digest(name, 0) == gpu.bdev_digest(name, 1) == model_digest(s)
        assert gpu.mirror_check(name)["mismatched_blocks"] == 0
    finally:
        gpu.delete_bdev(name)
    assert replica_digests(gpu, b, "r1", 1, nb, bs) == [model_digest(s)]


@pytest.mark.gpu
@pytest.mark.timeout(300)
@pytest.mark.parametrize("mode,bs", [("kick", 512), ("poller", 4096)])
def test_save_in_the_middle_of_a_vm(gpu, oracles, daemons, tmp_path, mode, bs):
    """a save comes between the two halves of a VM's trace while the VM stays connected: the image is the volume as
    the first half left it (its digest is the store's, read right after, and it loads back into that), and the second
    half then completes as the C restatement computes for the whole trace"""
    seed = 700 + bs
    rq_by_q, nb = vm_trace(bs, 1, seed)
    rq = rq_by_q[0]
    a = daemons("a", ["--gpus", "0"] + (["--poller"] if mode == "poller" else []))
    assert rpc(a, "construct_malloc_bdev", {"num_blocks": nb, "block_size": bs, "name": "Vol", "uuid": UUID}) == "Vol"
    assert rpc(a, "construct_vhost_scsi_controller", {"ctrlr": "scsi0"}) is True
    assert rpc(a, "add_vhost_scsi_lun", {"ctrlr": "scsi0", "scsi_target_num": 0, "bdev_name": "Vol"}) == 0
    done = []

    def between():
        path = str(tmp_path / "mid.img")
        rep = rpc(a, "save_bdev_image", {"name": "Vol", "path": path})
        assert rep["name"] == "Vol" and rep["uuid"] == UUID, rep
        done.append((rep, rpc(a, "get_bdevs_iostat", {"name": "Vol"})[1], replica_digests(gpu, a, "Vol", 1, nb, bs)[0]))
    img, mem, used = vm_run_split(a, rq, seed, between)
    assert done, "the save did not run"
    rep, stat, digest = done[0]
    blob = _read(tmp_path / "mid.img")
    h, _, store = parse_image(blob)
    assert h["digest"] == digest == model_digest(store), "the image is not the volume between the two halves"
    assert blob == model_image(store, bs)
    assert rep["file_bytes"] == len(blob) and rep["extents"] == h["nextents"]
    assert 0 < stat["num_write_ops"] + stat["num_read_ops"], "the save came before any request"
    wimg, wused, wstore, wstat = oracle_run(oracles, [rq], nb, bs, seed)
    assert stat["num_write_ops"] + stat["num_read_ops"] < wstat["num_write_ops"] + wstat["num_read_ops"]
    assert used == wused, "used elements differ from the checker's"
    bad = np.nonzero(masked(img, mem, 1) != masked(wimg, wimg.arena, 1))[0]
    assert not len(bad), f"guest memory differs from the checker's at {len(bad)} bytes, first {bad[:8]}"
    deadline = time.time() + 10
    while True:
        st = rpc(a, "get_bdevs_iostat", {"name": "Vol"})[1]
        got = {k: st[k] for k in IOSTAT}
        if got == {k: wstat[k] for k in IOSTAT} or time.time() > deadline:
            break
        time.sleep(0.05)
    assert got == {k: wstat[k] for k in IOSTAT}, "the save was counted, or the second half was not served"
    assert replica_digests(gpu, a, "Vol", 1, nb, bs) == [gpu.digest_host(wstore)]
    local = gpu.construct_malloc_bdev(nb, bs, name="mid-copy", device=0)
    try:
        gpu.bdev_image_load(local, tmp_path / "mid.img")
        assert gpu.bdev_digest(local) == digest
    finally:
        gpu.delete_bdev(local)


def _nbd_export(gpu, name):
    """an NBD export serving `name` until the returned socket is closed -> (socket, thread, rc list)"""
    a, b = socket.socketpair()
    a.settimeout(20)
    rc = []

    def serve():
        rc.append(gpu.load().oimgpu_nbd_serve(name.encode(), b.fileno()))
        b.close()
    th = threading.Thread(target=serve, daemon=True)
    th.start()
    a.sendall((0x25609513).to_bytes(4, "big") + (3).to_bytes(4, "big") + b"imgflush" + bytes(12))
    reply = b""
    while len(reply) < 16:
        reply += a.recv(16 - len(reply))
    assert reply[8:] == b"imgflush"             # answered: the export is in its loop
    return a, th, rc


@pytest.mark.gpu
@pytest.mark.timeout(180)
def test_image_refusals(gpu, tmp_path):
    nb, bs = 1000, 512
    s = content("sparse", nb, bs, seed=9)
    name = gpu.construct_malloc_bdev(nb, bs, name="refuse", uuid=UUID, device=0)
    other = gpu.construct_malloc_bdev(nb + 1, bs, name="refuse-geo", device=0)
    bs4k = gpu.construct_malloc_bdev(nb * bs // 4096, 4096, name="refuse-bs", device=0)
    try:
        gpu.bdev_write_raw(name, 0, s)
        good = tmp_path / "good.img"
        gpu.bdev_image_save(name, good)
        blob = _read(good)
        # save: never over an existing file, and not while an NBD export or a bio channel serves the bdev
        _refused(lambda: gpu.bdev_image_save(name, good), -errno.EEXIST)
        assert _read(good) == blob
        _refused(lambda: gpu.bdev_image_save("nope", tmp_path / "n.img"), -errno.ENODEV)
        _refused(lambda: gpu.bdev_image_save(name, tmp_path / "no-dir" / "x.img"), -errno.ENOENT)
        sock, th, rc = _nbd_export(gpu, name)
        try:
            _refused(lambda: gpu.bdev_image_save(name, tmp_path / "nbd.img"), -errno.EBUSY)
            _refused(lambda: gpu.bdev_image_load(name, good), -errno.EBUSY)
        finally:
            sock.close()
            th.join(20)
        assert rc == [0]
        with gpu.BioChan(name):
            _refused(lambda: gpu.bdev_image_save(name, tmp_path / "bio.img"), -errno.EBUSY)
            _refused(lambda: gpu.bdev_image_load(name, good), -errno.EBUSY)
        assert not os.path.exists(tmp_path / "nbd.img") and not os.path.exists(tmp_path / "bio.img")
        # load: every malformed image is refused before a store is touched
        _refused(lambda: gpu.bdev_image_load(other, good), -errno.EINVAL)
        _refused(lambda: gpu.bdev_image_load(bs4k, good), -errno.EINVAL)
        h, ext, _ = parse_image(blob)
        assert len(ext) >= 3
        table = 4096

        def variant(tag, b):
            p = tmp_path / f"{tag}.img"
            p.write_bytes(bytes(b))
            return p
        bad = [variant("magic", b"X" + blob[1:]), variant("version", blob[:8] + struct.pack("<I", 2) + blob[12:]),
               variant("short", blob[:-1]), variant("long", blob + b"\0"), variant("header-only", blob[:100])]
        o1, n1 = ext[1]
        for tag, e in (("overlap", (ext[0][0], n1)), ("adjacent", (ext[0][0] + ext[0][1], n1)),
                       ("range", (nb * bs // GRANULE * GRANULE + GRANULE, n1)), ("unaligned", (o1 + 8, n1))):
            b = bytearray(blob)
            b[table + 16:table + 32] = struct.pack("<QQ", *e)
            bad.append(variant(tag, b))
        d0 = gpu.bdev_digest(name)
        for p in bad:
            _refused(lambda: gpu.bdev_image_load(name, p), -errno.EINVAL)
            assert gpu.bdev_digest(name) == d0, f"{p.name}: the bdev changed"
        _refused(lambda: gpu.bdev_image_load(name, tmp_path / "missing.img"), -errno.ENOENT)
        # a flipped data byte loads, and is caught by the digest
        b = bytearray(blob)
        b[-1] ^= 0x10
        _refused(lambda: gpu.bdev_image_load(name, variant("flipped", b)), -errno.EIO)
        gpu.bdev_image_load(name, good)
        assert (gpu.bdev_read_raw(name, 0, nb * bs) == s).all()
    finally:
        for nm in (name, other, bs4k):
            gpu.delete_bdev(nm)


@pytest.mark.gpu
@pytest.mark.timeout(180)
def test_image_methods_through_the_daemon(gpu, daemons, tmp_path):
    nb, bs = 4096, 4096
    s = content("sparse", nb, bs, seed=21)
    d = daemons("ours", ["--gpus", "0"])
    assert rpc(d, "construct_malloc_bdev", {"num_blocks": nb, "block_size": bs, "name": "A", "uuid": UUID}) == "A"
    assert rpc(d, "construct_malloc_bdev", {"num_blocks": nb, "block_size": bs, "name": "B"}) == "B"
    local = gpu.construct_mirror_bdev_remote(nb, bs, 0, [base64.b64decode(rpc(d, "export_bdev_store", {"name": "A"}))],
                                             name="A-writer")
    try:
        gpu.bdev_write_raw(local, 0, s, replica=1)
    finally:
        gpu.delete_bdev(local)
    path = str(tmp_path / "a.img")
    want = model_image(s, bs)
    shape = {"name": "A", "path": path, "block_size": bs, "num_blocks": nb, "uuid": UUID,
             "extents": len(model_extents(s)), "data_bytes": len(want) - 4096 - (16 * len(model_extents(s)) + 4095) // 4096 * 4096,
             "file_bytes": len(want)}
    assert rpc(d, "save_bdev_image", {"name": "A", "path": path}) == shape
    assert _read(path) == want
    assert rpc(d, "save_bdev_image", {"name": "A", "path": path}) == {"error": {"code": -32602, "message": "File exists"}}
    assert rpc(d, "load_bdev_image", {"name": "B", "path": path}) == {**shape, "name": "B"}
    assert replica_digests(gpu, d, "B", 1, nb, bs) == [model_digest(s)]
    assert rpc(d, "load_bdev_image", {"name": "B", "path": path + ".x"}) == \
        {"error": {"code": -32602, "message": "No such file or directory"}}
    assert rpc(d, "construct_vhost_scsi_controller", {"ctrlr": "scsi0"}) is True
    assert rpc(d, "add_vhost_scsi_lun", {"ctrlr": "scsi0", "scsi_target_num": 0, "bdev_name": "B"}) == 0
    cfg = rpc(d, "get_subsystem_config", {"name": "bdev"}) + rpc(d, "get_subsystem_config", {"name": "vhost"})
    assert not [x for x in cfg if "image" in x["method"]]


@pytest.mark.gpu
@pytest.mark.timeout(300)
def test_restart_through_oimcfg_images(gpu, daemons, tmp_path):
    """oimcfg.py save --images, the daemon stops, a fresh one starts, oimcfg.py load --images: every bdev - a plain
    volume, a 2-way mirror and an empty volume - has its old uuid and digest, and is attached again"""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import oimcfg
    nb, bs = 4096, 4096
    old = daemons("old", ["--gpus", "0"])
    assert rpc(old, "construct_malloc_bdev", {"num_blocks": nb, "block_size": bs, "name": "plain", "uuid": UUID}) == "plain"
    assert rpc(old, "construct_mirror_bdev", {"num_blocks": nb, "block_size": 520 * 8, "name": "mir", "replicas": 2}) == "mir"
    assert rpc(old, "construct_malloc_bdev", {"num_blocks": 64, "block_size": 512, "name": "empty"}) == "empty"
    assert rpc(old, "construct_vhost_scsi_controller", {"ctrlr": "scsi0"}) is True
    assert rpc(old, "add_vhost_scsi_lun", {"ctrlr": "scsi0", "scsi_target_num": 0, "bdev_name": "plain"}) == 0
    for nm, seed in (("plain", 1), ("mir", 2)):
        local = gpu.construct_mirror_bdev_remote(nb, 4096, 0, [base64.b64decode(rpc(old, "export_bdev_store", {"name": nm}))],
                                                 name="writer")
        try:
            gpu.bdev_write_raw(local, 0, content("sparse", nb, 4096, seed), replica=1)
        finally:
            gpu.delete_bdev(local)
    assert rpc(old, "check_mirror_bdev", {"name": "mir", "repair": True})["repaired_blocks"] > 0
    listing = rpc(old, "get_bdevs")
    digests = {b["name"]: replica_digests(gpu, old, b["name"], len(b.get("driver_specific", {}).get("mirror", {}).get("replicas", [0])),
                                          b["num_blocks"], b["block_size"]) for b in listing}
    images = tmp_path / "images"
    images.mkdir()
    saved = json.loads(json.dumps(oimcfg.save(oimcfg.Rpc(old.rpc), str(images))))
    assert sorted(os.listdir(images)) == ["empty.img", "mir.img", "plain.img"]
    old.close()
    fresh = daemons("fresh", ["--gpus", "0"])
    oimcfg.load(oimcfg.Rpc(fresh.rpc), saved, str(images))
    assert rpc(fresh, "get_bdevs") == listing
    for b in listing:
        n = len(b.get("driver_specific", {}).get("mirror", {}).get("replicas", [0]))
        assert replica_digests(gpu, fresh, b["name"], n, b["num_blocks"], b["block_size"]) == digests[b["name"]], b["name"]
    assert rpc(fresh, "check_mirror_bdev", {"name": "mir"})["mismatched_blocks"] == 0
    assert [c["backend_specific"]["scsi"][0]["luns"][0]["bdev_name"] for c in rpc(fresh, "get_vhost_controllers")] == ["plain"]


@pytest.mark.gpu
@pytest.mark.timeout(300)
def test_eight_gib_sparse_volume(gpu, tmp_path):
    nb, bs = 2 << 20, 4096
    size = nb * bs
    rng = np.random.default_rng(8)
    src = gpu.construct_malloc_bdev(nb, bs, name="big", uuid=UUID, device=0)
    dst = gpu.construct_malloc_bdev(nb, bs, name="big2", device=0)
    try:
        gpu.bdev_write_raw(dst, 0, np.full(64 << 20, 1, dtype=np.uint8))        # a load zeroes what the image does not hold
        pieces = [(size - 4096, traces.pattern_bytes(3, 0, 4096)), (1 << 30, traces.pattern_bytes(4, 0, 48 << 20))]
        for g in rng.choice(nb, size=500, replace=False):
            pieces.append((int(g) * bs + int(rng.integers(0, bs - 64)), rng.integers(1, 256, size=64, dtype=np.uint8)))
        for off, data in pieces:
            gpu.bdev_write_raw(src, off, data)
        t0 = time.perf_counter()
        info = gpu.bdev_image_save(src, tmp_path / "big.img")
        t1 = time.perf_counter()
        granules = {off // GRANULE for off, _ in pieces[2:]} | {(size - 4096) // GRANULE}
        granules |= set(range((1 << 30) // GRANULE, ((1 << 30) + (48 << 20)) // GRANULE))
        assert info["data_bytes"] == GRANULE * len(granules)
        assert os.path.getsize(tmp_path / "big.img") == info["file_bytes"]
        gpu.bdev_image_load(dst, tmp_path / "big.img")
        t2 = time.perf_counter()
        assert gpu.bdev_digest(dst) == gpu.bdev_digest(src)
        print(f"8 GiB, {info['data_bytes'] >> 20} MiB of data in {info['nextents']} extents: save {t1 - t0:.3f} s, "
              f"load {t2 - t1:.3f} s")
    finally:
        gpu.delete_bdev(src)
        gpu.delete_bdev(dst)
