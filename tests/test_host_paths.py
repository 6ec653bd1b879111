"""Host paths of the C ABI next to a resident poller (GPU only): host-array batches through the poller's rings, the
error codes of that path, and control calls that park and restart the pollers of other sessions.  Every poller arms
the idle watchdog, and every call that waits for the GPU runs in a daemon thread with a deadline."""
import ctypes
import errno
import threading

import numpy as np
import pytest

import util
from oim_b200 import abi, traces

pytestmark = pytest.mark.gpu
WATCHDOG_MS = 8000


def _blocking(fn, timeout=60):
    """fn() in a daemon thread; fails instead of hanging when it does not return"""
    out = {}
    th = threading.Thread(target=lambda: out.setdefault("rc", fn()), daemon=True)
    th.start()
    th.join(timeout)
    assert not th.is_alive(), "call did not return"
    return out["rc"]


def _setup(gpu, name, nb):
    gpu.construct_malloc_bdev(nb, 512, name=name, device=0)
    gpu.construct_vhost_scsi_controller(name + ".ctl")
    gpu.add_vhost_scsi_lun(name + ".ctl", 0, name)
    gpu.bdev_write_raw(name, 0, traces.pattern_bytes(7, 0, nb * 512))


def _teardown(gpu, name):
    gpu.remove_vhost_scsi_target(name + ".ctl", 0)
    gpu.remove_vhost_controller(name + ".ctl")
    gpu.delete_bdev(name)


def _oracle(oracles, t, host, nb):
    with oracles.PortOracle(nb) as o:
        o.store[:] = traces.pattern_bytes(7, 0, o.store.size)
        oa = host.copy()
        want = o.submit(t.reqs, t.bind(oa.ctypes.data))
        return want, oa, o.store.copy()


def _submit_batch(gpu, lun, nq, per_q, reqs, iovs, cpls):
    return gpu.load().oimgpu_submit_batch(lun.h, nq, per_q, reqs.ctypes.data, iovs.ctypes.data, len(iovs),
                                          cpls.ctypes.data, abi.MEM_HOST)


@pytest.mark.timeout(180)
def test_poller_host_batch_matches_oracle(gpu, oracles):
    """oimgpu_submit_and_wait with host arrays while the poller is resident: every queue's requests index one SG table
    of the call, so their ranges start past 0 and are rebased onto each ring; 32-slot rings wrap many times"""
    import torch
    nb, nq, k, rounds = 1 << 16, 4, 24, 10
    t = traces.partitioned_queues(nq, k * rounds, nb, pattern="randrw", read_pct=60, io_blocks=8, sg="pages")
    host = np.zeros(t.arena_bytes, dtype=np.uint8)
    traces.fill_arena(host, t)
    want, want_arena, want_store = _oracle(oracles, t, host, nb)
    _setup(gpu, "hp0", nb)
    try:
        arena = torch.from_numpy(host.copy()).pin_memory()
        iovs = np.ascontiguousarray(t.bind(arena.data_ptr()))
        got = np.zeros(len(t.reqs), dtype=abi.cpl_dtype)
        rebased = 0
        with gpu.Lun("hp0.ctl", 0, num_queues=nq, queue_size=32) as lun:
            lun.start_poller(idle_timeout_ms=WATCHDOG_MS)
            try:
                for r in range(rounds):
                    idx = np.concatenate([np.arange(q * k * rounds + r * k, q * k * rounds + (r + 1) * k) for q in range(nq)])
                    reqs = np.ascontiguousarray(t.reqs[idx])
                    rebased += int((reqs["iov_start"].reshape(nq, k).min(axis=1) > 0).sum())
                    cpls = np.zeros(len(reqs), dtype=abi.cpl_dtype)
                    rc = _blocking(lambda: gpu.load().oimgpu_submit_and_wait(
                        lun.h, nq, k, reqs.ctypes.data, iovs.ctypes.data, len(iovs), cpls.ctypes.data, abi.MEM_HOST))
                    assert rc == 0, f"round {r}: rc {rc}"
                    got[idx] = cpls
                assert lun.poller_running()
            finally:
                lun.stop_poller()
            assert lun.iostat()["kernel_launches"] == 1, "the resident kernel served every round"
        assert rebased >= nq * rounds - 1, "per-queue SG ranges should start past 0"
        util.assert_cpls_equal(got, want, t.reqs)
        assert (arena.numpy() == want_arena).all(), "client buffers"
        assert (gpu.bdev_read_raw("hp0", 0, nb * 512) == want_store).all(), "store"
    finally:
        _teardown(gpu, "hp0")


@pytest.mark.timeout(120)
def test_poller_host_batch_error_codes(gpu):
    """-EINVAL (SG index past the table), -EAGAIN (ring full), -E2BIG (SG span past the ring's SG table) from the
    poller branch of oimgpu_submit_batch, and -EBUSY from a kick with caller-owned device arrays pending"""
    import torch
    nb, qs = 1 << 14, 32
    t = traces.uniform_trace(qs, nb, io_blocks=8, pattern="randread", seed=5)
    _setup(gpu, "hp1", nb)
    try:
        arena = torch.zeros(t.arena_bytes, dtype=torch.uint8).pin_memory()
        iovs = np.ascontiguousarray(t.bind(arena.data_ptr()))
        cpls = np.zeros(qs, dtype=abi.cpl_dtype)
        with gpu.Lun("hp1.ctl", 0, num_queues=2, queue_size=qs) as lun:
            iov_cap = max(1024, qs * 8)
            lun.start_poller(idle_timeout_ms=WATCHDOG_MS)
            try:
                bad = np.ascontiguousarray(t.reqs[:1].copy())
                bad["iov_start"] = len(iovs)
                assert _submit_batch(gpu, lun, 1, 1, bad, iovs, cpls) == -errno.EINVAL
                wide = np.zeros(iov_cap + 1, dtype=abi.iov_dtype)
                span = np.ascontiguousarray(t.reqs[:2].copy())
                span["iov_start"] = [0, iov_cap]
                span["iovcnt"] = 1
                assert _submit_batch(gpu, lun, 1, 2, span, wide, cpls) == -errno.E2BIG
                full = np.ascontiguousarray(t.reqs)
                assert _submit_batch(gpu, lun, 1, qs, full, iovs, cpls) == 1      # one doorbell rung
                assert _submit_batch(gpu, lun, 1, 1, full[:1], iovs, cpls) == -errno.EAGAIN
                assert len(_blocking(lambda: lun.poll(0, qs, wait=True))) == qs
                d = torch.zeros(4096, dtype=torch.uint8, device="cuda:0")
                lun.submit_device(1, d.data_ptr(), 1, d.data_ptr(), d.data_ptr())
                with pytest.raises(gpu.OimGpuError) as e:
                    lun.kick()
                assert e.value.rc == -errno.EBUSY
                assert lun.poller_running()
            finally:
                lun.stop_poller()
    finally:
        _teardown(gpu, "hp1")


@pytest.mark.timeout(180)
def test_park_sites_keep_a_resident_poller(gpu, oracles):
    """histogram disable, delete_bdev of an unrelated bdev (with and without a histogram), mem_unregister and a session
    open that fails with -ENOMEM park the resident poller of another session and bring it back, and bdev_digest of an
    unrelated bdev on its GPU does not stop it; afterwards it still serves a trace bit-exactly"""
    import torch
    nb, nq, rounds = 1 << 16, 2, 4
    t = traces.partitioned_queues(nq, 32 * rounds, nb, pattern="randrw", read_pct=60, io_blocks=8)
    host = np.zeros(t.arena_bytes, dtype=np.uint8)
    traces.fill_arena(host, t)
    want, want_arena, want_store = _oracle(oracles, t, host, nb)
    _setup(gpu, "pk0", nb)
    gpu.construct_malloc_bdev(1024, 512, name="pk1", device=0)
    gpu.construct_malloc_bdev(1024, 512, name="pk2", device=0)
    gpu.construct_malloc_bdev(1024, 512, name="pk3", device=0)
    gpu.construct_vhost_scsi_controller("pk1.ctl")
    gpu.add_vhost_scsi_lun("pk1.ctl", 0, "pk1")
    try:
        arena = torch.from_numpy(host.copy()).pin_memory()
        iovs = t.bind(arena.data_ptr())
        per_q = 32 * rounds
        got = np.zeros(len(t.reqs), dtype=abi.cpl_dtype)
        buf = np.zeros((1 << 20) + 4096, dtype=np.uint8)
        reg = buf[-buf.ctypes.data % 4096:][:1 << 20]            # page-aligned, pageable
        with gpu.Lun("pk0.ctl", 0, num_queues=nq, queue_size=64) as lun:
            lun.start_poller(idle_timeout_ms=WATCHDOG_MS)
            try:
                gpu.enable_bdev_histogram("pk1", True)
                _blocking(lambda: gpu.enable_bdev_histogram("pk1", False))
                _blocking(lambda: gpu.delete_bdev("pk2"))
                gpu.mem_register(reg)
                _blocking(lambda: gpu.mem_unregister(reg))
                gpu.enable_bdev_histogram("pk3", True)
                _blocking(lambda: gpu.delete_bdev("pk3"))
                _blocking(lambda: gpu.bdev_digest("pk1"))
                h = ctypes.c_void_p()
                # terabytes of kick staging: refused, and the half-open session is taken apart
                assert _blocking(lambda: gpu.load().oimgpu_lun_open(b"pk1.ctl", 0, 0xFFFFFFFF, 64, ctypes.byref(h))) \
                    == -errno.ENOMEM
                assert lun.poller_running()
                for r in range(rounds):
                    for q in range(nq):
                        lo = q * per_q + r * 32
                        part = t.reqs[lo:lo + 32].copy()
                        i0 = int(part["iov_start"][0])
                        part["iov_start"] -= np.uint32(i0)
                        lun.submit(q, part, iovs[i0:i0 + 32])
                    assert lun.kick() == nq                   # doorbells, not launches
                    for q in range(nq):
                        c = _blocking(lambda: lun.poll(q, 32, wait=True))
                        assert len(c) == 32
                        got[q * per_q + r * 32:q * per_q + r * 32 + 32] = c
                assert lun.poller_running()
            finally:
                lun.stop_poller()
            assert lun.iostat()["kernel_launches"] == 6, "five parks, each followed by a restart"
        util.assert_cpls_equal(got, want, t.reqs)
        assert (arena.numpy() == want_arena).all(), "client buffers"
        assert (gpu.bdev_read_raw("pk0", 0, nb * 512) == want_store).all(), "store"
    finally:
        _teardown(gpu, "pk0")
        _teardown(gpu, "pk1")


@pytest.mark.timeout(120)
def test_session_survives_a_refused_host_batch(gpu, oracles):
    """a host-array batch whose staging arrays cannot be allocated (128 GiB of request slots) is refused with -ENOMEM
    before the caller's arrays are read; the same session then serves a batch as the oracle does"""
    import torch
    nb, nq, k = 1 << 14, 4, 32
    t = traces.partitioned_queues(nq, k, nb, pattern="randrw", read_pct=60, io_blocks=8)
    host = np.zeros(t.arena_bytes, dtype=np.uint8)
    traces.fill_arena(host, t)
    with oracles.PortOracle(nb) as o:                          # the same batch, twice
        o.store[:] = traces.pattern_bytes(7, 0, o.store.size)
        want_arena = host.copy()
        want_first = o.submit(t.reqs, t.bind(want_arena.ctypes.data))
        want = o.submit(t.reqs, t.bind(want_arena.ctypes.data))
        want_store = o.store.copy()
    _setup(gpu, "hp2", nb)
    try:
        arena = torch.from_numpy(host.copy()).pin_memory()
        iovs = np.ascontiguousarray(t.bind(arena.data_ptr()))
        reqs = np.ascontiguousarray(t.reqs)
        with gpu.Lun("hp2.ctl", 0, num_queues=nq, queue_size=64) as lun:
            def batch():
                cpls = np.zeros(len(reqs), dtype=abi.cpl_dtype)
                rc = _blocking(lambda: gpu.load().oimgpu_submit_and_wait(
                    lun.h, nq, k, reqs.ctypes.data, iovs.ctypes.data, len(iovs), cpls.ctypes.data, abi.MEM_HOST))
                assert rc == 0, f"rc {rc}"
                return cpls
            util.assert_cpls_equal(batch(), want_first, t.reqs)
            one = np.zeros(1, dtype=abi.req_dtype)
            assert _submit_batch(gpu, lun, 1, 1 << 31, one, np.zeros(1, dtype=abi.iov_dtype),
                                 np.zeros(1, dtype=abi.cpl_dtype)) == -errno.ENOMEM
            util.assert_cpls_equal(batch(), want, t.reqs)
        assert (arena.numpy() == want_arena).all(), "client buffers"
        assert (gpu.bdev_read_raw("hp2", 0, nb * 512) == want_store).all(), "store"
    finally:
        _teardown(gpu, "hp2")
