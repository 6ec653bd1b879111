"""The bdev registry's record of who uses a bdev and where its stores live.

A bdev that an NBD export, a bio channel or a session's target uses is not deleted, and a failed delete leaves the
controllers' targets where they were.  While anything uses the bdev, a disabled histogram reads as -EFAULT, as the
reference's per-channel histogram does.  A mirror whose import fails gives its own store's bytes back, so that placement
by rule (device -1: the GPU with the fewest bytes) is not skewed by a store that no longer exists."""
import contextlib
import errno
import socket
import struct
import threading

import pytest

pytestmark = pytest.mark.gpu

NB, BS = 4096, 512


def recv_exact(sock, n):
    buf = b""
    while len(buf) < n:
        chunk = sock.recv(n - len(buf))
        assert chunk, "the NBD export closed the connection"
        buf += chunk
    return buf


@contextlib.contextmanager
def nbd_export(lib, name):
    """oimgpu_nbd_serve on one end of a socketpair, in a thread.  Enters once the export has answered a FLUSH, so that
    it holds the bdev; leaving closes the other end, which ends the export."""
    a, b = socket.socketpair()
    a.settimeout(20)
    rc = []

    def serve():
        rc.append(lib.load().oimgpu_nbd_serve(name.encode(), b.fileno()))
        b.close()

    th = threading.Thread(target=serve, daemon=True)
    th.start()
    try:
        a.sendall(struct.pack(">IIQQI", 0x25609513, 3, 7, 0, 0))     # struct nbd_request: NBD_CMD_FLUSH, handle 7
        assert recv_exact(a, 16) == struct.pack(">IIQ", 0x67446698, 0, 7)
        yield
    finally:
        a.close()
        th.join(20)
    assert not th.is_alive() and rc == [0]


def hold(lib, holder, name, ctrlr):
    if holder == "nbd":
        return nbd_export(lib, name)
    if holder == "bio_chan":
        return lib.BioChan(name)
    return lib.Lun(ctrlr, -1)        # a controller-wide session: the bdev is one of its peer targets


def targets(lib, ctrlr):
    return [t["luns"][0]["bdev_name"] for t in lib.get_vhost_controllers(ctrlr)[0]["backend_specific"]["scsi"]]


@contextlib.contextmanager
def bdev_on_controller(lib, name, ctrlr):
    lib.construct_malloc_bdev(NB, BS, name=name, device=0)
    lib.construct_vhost_scsi_controller(ctrlr)
    try:
        lib.add_vhost_scsi_lun(ctrlr, 0, name)
        yield
    finally:
        if name in [b["name"] for b in lib.get_bdevs()]:
            lib.delete_bdev(name)
        lib.remove_vhost_controller(ctrlr)


@pytest.mark.parametrize("holder", ["nbd", "bio_chan"])
def test_delete_is_refused_while_the_bdev_is_held(gpu, holder):
    """refused before any target is taken apart, next to a controller-wide session whose peer target would let go"""
    name, ctrlr = f"reg_{holder}", f"reg_{holder}.ctl"
    with bdev_on_controller(gpu, name, ctrlr), gpu.Lun(ctrlr, -1):
        before = gpu.get_bdevs()
        with hold(gpu, holder, name, ctrlr):
            with pytest.raises(gpu.OimGpuError) as e:
                gpu.delete_bdev(name)
            assert e.value.rc == -errno.EBUSY
            assert targets(gpu, ctrlr) == [name]
            assert gpu.get_bdevs() == before
        gpu.delete_bdev(name)
        assert targets(gpu, ctrlr) == []
        assert name not in [b["name"] for b in gpu.get_bdevs()]


@pytest.mark.parametrize("holder", ["nbd", "bio_chan", "peer"])
def test_disabled_histogram_reads_efault_while_the_bdev_is_held(gpu, holder):
    name, ctrlr = f"hist_{holder}", f"hist_{holder}.ctl"
    with bdev_on_controller(gpu, name, ctrlr):
        assert not gpu.get_bdev_histogram(name).any()
        with hold(gpu, holder, name, ctrlr):
            with pytest.raises(gpu.OimGpuError) as e:
                gpu.get_bdev_histogram(name)
            assert e.value.rc == -errno.EFAULT
        assert not gpu.get_bdev_histogram(name).any()


@pytest.fixture(scope="module")
def gpu2():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from oim_b200 import build, lib
    build.build()
    for d in (0, 1):
        torch.zeros(1, device=f"cuda:{d}")
    lib.fini()
    lib.init([0, 1])
    yield lib
    lib.fini()
    lib.init([0])           # what the session-wide `gpu` fixture set up: the modules after this one rely on it


def test_failed_import_gives_its_store_back(gpu2):
    with pytest.raises(gpu2.OimGpuError) as e:
        gpu2.construct_mirror_bdev_remote(NB, BS, 0, [bytes(gpu2.IPC_HANDLE_BYTES)], name="reg_ipc")   # a handle of zeros
    assert e.value.rc == -errno.EIO
    name = gpu2.construct_malloc_bdev(NB, BS, device=-1)
    try:
        assert gpu2.get_bdevs(name)[0]["device"] == 0     # both GPUs hold no bytes: the tie goes to the first
    finally:
        gpu2.delete_bdev(name)
