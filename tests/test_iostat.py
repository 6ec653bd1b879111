"""get_bdevs_iostat counters and get_bdev_histogram tallies, as the reference's bdev layer keeps them
(_spdk_bdev_io_complete, S/lib/bdev/bdev.c:3233-3258): per completed bdev_io, the histogram tallies every one
whatever its type and status, the counters book successful reads, writes and unmaps only.  One SCSI request can
make no bdev_io (refused before submission), one (READ, WRITE, the FLUSH of SYNCHRONIZE CACHE) or one per applied
UNMAP descriptor.

CPU: the restatement's counters against the compiled reference's own spdk_bdev_get_device_stat and histogram.
GPU: the kernel's counters (lun.iostat, get_bdevs_iostat) and histogram against the reference, on every path."""
import numpy as np
import pytest

import util
from oim_b200 import abi, traces, vring
from test_multi_target import TARGETS, Controller, multi_trace, run_session
from test_oracle import GOLDEN, HostBuf, load_golden, run_bdevio
from test_vring import VQ_KERNELS, make_requests

COUNTERS = ("num_read_ops", "bytes_read", "num_write_ops", "bytes_written", "num_unmap_ops", "bytes_unmapped")
# get_bdevs_iostat's fields that add up over a bdev's lifetime (everything lun.iostat reports but kernel_launches)
LIFETIME = ("num_read_ops", "num_write_ops", "num_unmap_ops", "num_other_ops", "bytes_read", "bytes_written",
            "bytes_unmapped", "num_errors", "read_latency_ns", "write_latency_ns", "unmap_latency_ns")
FUZZ_SEEDS = (200, 203, 207, 211)


# ---- traces -------------------------------------------------------------------------------------------------

def edge_trace(nb: int, block_size: int = 512, target: int = 0) -> traces.Trace:
    """one of each request that books something other than one I/O, or nothing at all; SG addresses are arena
    offsets.  Repeated twice, so that the trace is more than one pass (shared kernels)."""
    bs = block_size
    b = abi.Batch(target)
    pay = []
    top = [0]

    def buf(n: int) -> int:
        off = top[0]
        top[0] += (max(n, 1) + 4095) // 4096 * 4096
        return off

    def sg(n: int) -> list:
        return [(buf(n), n)]

    def unmap(descs, sg_len=None):
        pl = abi.unmap_param_list(descs)
        off = buf(len(pl))
        pay.append((off, pl))
        b.add(abi.cdb_unmap(len(pl)), abi.DIR_TO_DEV, [(off, len(pl) if sg_len is None else sg_len)])

    def sync(opcode, lba, n):
        b.add(abi.cdb_sync(opcode, lba, n), abi.DIR_FROM_DEV, [])

    big = abi.MAX_XFER_BYTES // bs + 1
    for _ in range(2):
        b.read(0, 8, sg(8 * bs))                                    # plain ones, for contrast
        b.write(64, 8, sg(8 * bs))
        b.read(8, 0, [])                                            # 0 blocks
        b.read(8, 0, sg(bs), opcode=abi.READ_16)
        b.write(8, 0, sg(bs))
        b.read(nb, 1, sg(bs))                                       # out of range
        b.write(nb - 1, 2, sg(2 * bs), opcode=abi.WRITE_16)
        b.read(0, big, sg(big * bs), opcode=abi.READ_16)            # over 4 MiB
        b.read(16, 8, sg(bs))                                       # SG shorter than the transfer
        b.write(16, 8, sg(bs))
        b.read(32, 1, sg(8 * bs))                                   # SG longer than the transfer
        b.write(32, 1, sg(8 * bs))
        b.read(40, 1, sg(bs + 188))                                 # SG not a whole number of blocks
        b.read(48, 4, [])                                           # a transfer with no SG at all
        b.write(48, 4, [])
        b.read(56, 2, [(buf(bs), bs), (buf(bs), 0), (buf(bs), bs)])
        unmap([])                                                   # 0, 1 and 256 descriptors
        unmap([(100, 4)])
        unmap([(1000 + 2 * i, 1) for i in range(256)])
        unmap([(300, 0), (301, 2), (310, 0)])                       # zero-length descriptors are skipped
        unmap([(5, 0), (6, 0)])
        unmap([(400, 2), (nb - 1, 4), (420, 2)])                    # fails mid-list: the first stays applied
        unmap([(nb, 1), (10, 1)])                                   # fails at once
        unmap([(200, 1)], sg_len=6)                                 # parameter list shorter than its header
        unmap([(nb - 8, 8), (0, 8)])
        sync(abi.SYNCHRONIZE_CACHE_10, 0, 8)
        sync(abi.SYNCHRONIZE_CACHE_16, 100, 1)
        sync(abi.SYNCHRONIZE_CACHE_10, 16, 0)                       # count 0: to the end of the device
        sync(abi.SYNCHRONIZE_CACHE_16, nb - 4, 0)
        sync(abi.SYNCHRONIZE_CACHE_16, nb, 0)                       # count 0 at the end: nothing to flush
        sync(abi.SYNCHRONIZE_CACHE_10, nb, 1)                       # out of range
        sync(abi.SYNCHRONIZE_CACHE_16, nb - 2, 4)
        b.read(0, 1, sg(bs), lun=abi.virtio_lun(target + 1 if target < 7 else 0))  # no device there
        lun = abi.virtio_lun(target)
        lun[0] = 2
        b.read(0, 1, sg(bs), lun=lun)                               # not a single-level LUN address
        b.read(0, 1, sg(bs), lun=abi.virtio_lun(target, 1))         # LUN 1: the null LUN
        b.read(0, 1, [(int(traces.NULL_ADDR_FLAG), bs)])            # untranslatable SG: invalid request
        b.add(abi.cdb_read_capacity(True), abi.DIR_FROM_DEV, sg(32))
        b.add(np.zeros(abi.CDB_SIZE, dtype=np.uint8), abi.DIR_FROM_DEV, [])   # TEST UNIT READY
    reqs, iovs = b.arrays()
    t = traces.Trace(reqs, iovs, top[0], f"edge{bs}")
    t.meta["param_payloads"] = pay
    return t


def named_traces():
    """(id, trace, num_blocks, block_size, removed) of every single-target trace the counters are checked on"""
    out = []
    for p in GOLDEN:
        t, z = load_golden(p)
        out.append((t.name[:-4], t, int(z["num_blocks"]), 512, bool(z["removed"])))
    for s in FUZZ_SEEDS:
        nb = 32768
        out.append((f"fuzz{s}", traces.fuzz_trace(300, nb, seed=s, max_io_blocks=[8, 64, 300][s % 3]), nb, 512, False))
    out.append(("alignment_sweep", traces.alignment_sweep(65536), 65536, 512, False))
    out.append(("edge512", edge_trace(16384), 16384, 512, False))
    out.append(("edge520", edge_trace(16384, 520), 16384, 520, False))
    out.append(("edge_removed", edge_trace(16384), 16384, 512, True))
    return out


TRACES = {x[0]: x[1:] for x in named_traces()}


def replay(cls, t, nb, block_size=512, removed=False):
    """-> (cpls, iostat of the target) after replaying `t` on a checker"""
    with cls(nb, block_size) as o:
        o.store[:] = traces.pattern_bytes(7, 0, o.store.size)
        if removed:
            o.set_removed(0, True)
        arena = np.zeros(t.arena_bytes, dtype=np.uint8)
        traces.fill_arena(arena, t)
        cpls = o.submit(t.reqs, t.bind(arena.ctypes.data))
        return cpls, o.iostat()


def failed(cpls) -> int:
    """num_errors as the kernel books it: every request that did not complete GOOD"""
    ok = (cpls["resp_valid"] == 1) & (cpls["response"] == abi.S_OK) & (cpls["status"] == abi.STATUS_GOOD)
    return int((~ok).sum())


def need_ref(oracles):
    if not oracles.ref_available():
        pytest.skip("oracle/_ref not built here (no reference sources)")
    if not oracles.ref_available(iostat=True):
        pytest.skip("oracle/_ref was built before its counters were exported, and there are no reference sources to rebuild it")


def diffs(got: dict, want: dict, keys) -> list:
    return [f"{k}: got {got[k]} want {want[k]}" for k in keys if got[k] != want[k]]


# ---- CPU: the restatement against the reference ----------------------------------------------------------------

@pytest.mark.parametrize("name", list(TRACES))
def test_restatement_iostat_matches_reference(oracles, name):
    need_ref(oracles)
    t, nb, bs, removed = TRACES[name]
    wc, want = replay(oracles.RefOracle, t, nb, bs, removed)
    gc, got = replay(oracles.PortOracle, t, nb, bs, removed)
    util.assert_cpls_equal(gc, wc, t.reqs, name)
    assert got == want, diffs(got, want, want)


def test_edge_trace_books_what_the_reference_books(oracles):
    """the edge trace reaches every booking rule: UNMAP per descriptor, FLUSH in the histogram only, refusals nowhere"""
    need_ref(oracles)
    t, nb, bs, _ = TRACES["edge512"]
    _, st = replay(oracles.RefOracle, t, nb, bs)
    # per copy: 1 + 256 + 1 + 1 (before the failing one) + 2 descriptors applied; 4 flushes
    assert st["num_unmap_ops"] == 2 * 261
    assert st["bytes_unmapped"] == 2 * (4 + 256 + 2 + 2 + 16) * bs
    ios = st["num_read_ops"] + st["num_write_ops"] + st["num_unmap_ops"]
    assert st["bdev_ios"] == ios + 2 * 4, "one tally per bdev_io, the SYNCHRONIZE CACHE flushes included"
    _, st = replay(oracles.RefOracle, t, nb, bs, removed=True)
    assert st == dict.fromkeys(st, 0), "a hot-removed target is never reached"


@pytest.mark.parametrize("seed", range(700, 704))
@pytest.mark.parametrize("kind", ["fuzz", "primary"])
def test_restatement_iostat_matches_reference_per_target(oracles, seed, kind):
    need_ref(oracles)
    t = multi_trace(seed, kind=kind)
    per = {}
    for cls in (oracles.RefOracle, oracles.PortOracle):
        with cls(TARGETS[1], 512, 1) as o:
            o.store[:] = traces.pattern_bytes(7, 0, o.store.size)
            for k in (3, 6):
                o.add_target(k, TARGETS[k])[:] = traces.pattern_bytes(7 + k, 0, TARGETS[k] * 512)
            arena = np.zeros(t.arena_bytes, dtype=np.uint8)
            traces.fill_arena(arena, t)
            o.submit(t.reqs, t.bind(arena.ctypes.data))
            per[cls.__name__] = {k: o.iostat(k) for k in TARGETS}
    assert per["PortOracle"] == per["RefOracle"]
    if kind == "fuzz":
        assert all(per["RefOracle"][k]["bdev_ios"] > 0 for k in TARGETS), "every device took I/O"


def test_restatement_iostat_matches_reference_on_bdevio(oracles):
    need_ref(oracles)
    nb = 65536
    out = {}
    for cls in (oracles.RefOracle, oracles.PortOracle):
        with cls(nb) as o:
            run_bdevio(o.submit, HostBuf, nb)
            out[cls.__name__] = o.iostat()
    assert out["PortOracle"] == out["RefOracle"]
    assert out["RefOracle"]["num_unmap_ops"] == 4


# ---- GPU: the kernel against the reference ---------------------------------------------------------------------

def checker(oracles):
    """the compiled reference where its library exports the counters, the restatement pinned to it otherwise"""
    return oracles.RefOracle if oracles.ref_available(iostat=True) else oracles.PortOracle


def check_counts(got: dict, want: dict, want_cpls, what: str, histogram: bool = True):
    """lun.iostat (+ histogram total) against the reference's bdev; num_errors against its completions"""
    bad = diffs(got, want, COUNTERS)
    if got["num_errors"] != failed(want_cpls):
        bad.append(f"num_errors: got {got['num_errors']} want {failed(want_cpls)}")
    if histogram and got["histogram_total"] != want["bdev_ios"]:
        bad.append(f"histogram tallies: got {got['histogram_total']} want {want['bdev_ios']} bdev_ios")
    assert not bad, f"{what}: " + "; ".join(bad)


@pytest.mark.gpu
@pytest.mark.parametrize("kernel,name", util.kernel_cases(list(TRACES)))
def test_cuda_iostat_matches_reference(gpu, oracles, kernel, name):
    """every trace in ONE launch of each queue-kernel variant: counters, errors and histogram tallies"""
    t, nb, bs, removed = TRACES[name]
    wc, want = replay(checker(oracles), t, nb, bs, removed)
    gc, _, _, got = util.run_cuda(gpu, t, nb, block_size=bs, removed=removed, kernel=kernel, histogram=True)
    util.assert_cpls_equal(gc, wc, t.reqs, f"{kernel}:{name}")
    check_counts(got, want, wc, f"{kernel}:{name}")


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", util.KERNELS)
def test_cuda_iostat_lun_removed(gpu, kernel):
    """a LUN being torn down aborts every request before a bdev_io exists (spdk_scsi_task_process_abort)"""
    t, nb, bs, _ = TRACES["edge512"]
    _, _, _, got = util.run_cuda(gpu, t, nb, block_size=bs, lun_removed=True, kernel=kernel, histogram=True)
    assert all(got[k] == 0 for k in COUNTERS) and got["histogram_total"] == 0, got
    assert got["num_errors"] == len(t.reqs)


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", list(VQ_KERNELS))
@pytest.mark.parametrize("seed", [420, 421, 1422])
def test_cuda_iostat_virtqueue(gpu, oracles, kernel, seed):
    """the guest's own rings: the kernel walks them, the counters must come out the same"""
    import torch
    nb, rq = 32768, make_requests(seed, contiguous=seed >= 1000)
    ring = 1024
    with checker(oracles)(nb) as o:
        o.store[:] = traces.pattern_bytes(7, 0, o.store.size)
        img = vring.build_image(rq, ring_size=ring, seed=seed, contiguous=seed >= 1000)
        o.vq_process(img)
        want = o.iostat()
        used = img.used_in_order(None, 0, img.used_entries()[0])
    name = f"ios{seed}{kernel}"
    gpu.construct_malloc_bdev(nb, 512, name=name, device=0)
    gpu.construct_vhost_scsi_controller(f"{name}.ctl")
    gpu.add_vhost_scsi_lun(f"{name}.ctl", 0, name)
    try:
        gpu.bdev_write_raw(name, 0, traces.pattern_bytes(7, 0, nb * 512))
        gpu.enable_bdev_histogram(name, True)
        with util.environ(**VQ_KERNELS[kernel]), gpu.Lun(f"{name}.ctl", 0, num_queues=1, queue_size=32) as lun:
            img = vring.build_image(rq, ring_size=ring, seed=seed, contiguous=seed >= 1000)
            dev = torch.from_numpy(img.arena).to("cuda:0")
            base = dev.data_ptr()
            lun.set_mem_table(img.region_table(base))
            lun.vq_attach(0, base + img.desc_off, base + img.avail_off, base + img.used_off, img.ring_size, 0, 0)
            assert lun.vq_kick() == 1
            lun.sync()
            lun.vq_detach(0)
            got = lun.iostat()
            got["histogram_total"] = int(gpu.get_bdev_histogram(name).sum())
        bad = diffs(got, want, COUNTERS)
        if got["histogram_total"] != want["bdev_ios"]:
            bad.append(f"histogram tallies: got {got['histogram_total']} want {want['bdev_ios']}")
        assert not bad, f"{kernel}: " + "; ".join(bad)
        # every used element of length 0 is an invalid request, and so is counted as an error
        assert got["num_errors"] >= int((used["len"] == 0).sum())
    finally:
        gpu.remove_vhost_scsi_target(f"{name}.ctl", 0)
        gpu.remove_vhost_controller(f"{name}.ctl")
        gpu.delete_bdev(name)


@pytest.mark.gpu
@pytest.mark.timeout(180)
@pytest.mark.parametrize("how", ["doorbell", "batch"])
def test_cuda_iostat_resident_poller(gpu, oracles, how):
    """a resident poller flushes its counters when it leaves: after stop_poller they match the reference.
    doorbell: ring slots + kick; batch: host arrays through oimgpu_submit_and_wait"""
    import torch
    nb, k = 32768, 32
    t = traces.fuzz_trace(320, nb, seed=4711, max_io_blocks=64)
    wc, want = replay(checker(oracles), t, nb)
    name = f"iosp{how}"
    gpu.construct_malloc_bdev(nb, 512, name=name, device=0)
    gpu.construct_vhost_scsi_controller(f"{name}.ctl")
    gpu.add_vhost_scsi_lun(f"{name}.ctl", 0, name)
    try:
        gpu.bdev_write_raw(name, 0, traces.pattern_bytes(7, 0, nb * 512))
        gpu.enable_bdev_histogram(name, True)
        host = np.zeros(t.arena_bytes, dtype=np.uint8)
        traces.fill_arena(host, t)
        arena = torch.from_numpy(host).pin_memory()
        iovs = np.ascontiguousarray(t.bind(arena.data_ptr()))
        got_cpls = np.zeros(len(t.reqs), dtype=abi.cpl_dtype)
        with gpu.Lun(f"{name}.ctl", 0, num_queues=1, queue_size=64) as lun:
            lun.start_poller(idle_timeout_ms=8000)
            try:
                for lo in range(0, len(t.reqs), k):
                    part = t.reqs[lo:lo + k].copy()
                    i0 = int(part["iov_start"][0])
                    part["iov_start"] -= np.uint32(i0)
                    hi = int(part["iov_start"][-1] + part["iovcnt"][-1])
                    sub = np.ascontiguousarray(iovs[i0:i0 + max(hi, 1)])
                    if how == "doorbell":
                        lun.submit(0, part, sub)
                        assert lun.kick() == 1
                        got_cpls[lo:lo + k] = lun.poll(0, k, wait=True)
                    else:
                        cpls = np.zeros(k, dtype=abi.cpl_dtype)
                        rc = gpu.load().oimgpu_submit_and_wait(lun.h, 1, k, part.ctypes.data, sub.ctypes.data, len(sub),
                                                              cpls.ctypes.data, abi.MEM_HOST)
                        assert rc == 0, rc
                        got_cpls[lo:lo + k] = cpls
            finally:
                lun.stop_poller()
            got = lun.iostat()
            got["histogram_total"] = int(gpu.get_bdev_histogram(name).sum())
            assert got["kernel_launches"] == 1, "the resident kernel served every round"
        util.assert_cpls_equal(got_cpls, wc, t.reqs, how)
        check_counts(got, want, wc, how)
    finally:
        gpu.remove_vhost_scsi_target(f"{name}.ctl", 0)
        gpu.remove_vhost_controller(f"{name}.ctl")
        gpu.delete_bdev(name)


@pytest.mark.gpu
@pytest.mark.parametrize("home", [1, -1])
def test_cuda_iostat_per_target(gpu, oracles, home):
    """one controller, three devices behind the same queues: each device's counters, peer bookings included,
    and get_bdevs_iostat of each bdev while the session is open"""
    t = multi_trace(741, n=400)
    c = Controller(gpu)
    try:
        with oracles.PortOracle(TARGETS[1], 512, 1) as o:
            o.store[:] = traces.pattern_bytes(7, 0, o.store.size)
            for k in (3, 6):
                o.add_target(k, TARGETS[k])[:] = traces.pattern_bytes(7 + k, 0, TARGETS[k] * 512)
            arena = np.zeros(t.arena_bytes, dtype=np.uint8)
            traces.fill_arena(arena, t)
            o.submit(t.reqs, t.bind(arena.ctypes.data))
            want = {k: o.iostat(k) for k in TARGETS}
        for k in TARGETS:
            gpu.enable_bdev_histogram(c.names[k], True)
        _, _, stats = run_session(gpu, c, home, t)
        for k in TARGETS:
            bad = diffs(stats[k], want[k], COUNTERS)
            hist = int(gpu.get_bdev_histogram(c.names[k]).sum())
            if hist != want[k]["bdev_ios"]:
                bad.append(f"histogram tallies: got {hist} want {want[k]['bdev_ios']}")
            life = gpu.get_bdevs_iostat(c.names[k])
            bad += diffs(life, stats[k], [f for f in LIFETIME if f != "num_errors"])
            assert not bad, f"target {k}: " + "; ".join(bad)
    finally:
        c.close()


@pytest.mark.gpu
def test_cuda_get_bdevs_iostat_adds_up_over_a_lifetime(gpu):
    """get_bdevs_iostat of a bdev = the sessions that are gone + the ones that are open, every counter including
    the three latency sums; a bdev reached as another session's peer target counts there too"""
    import torch
    nb = 32768
    gpu.construct_malloc_bdev(nb, 512, name="life0", device=0)
    gpu.construct_malloc_bdev(nb, 512, name="life1", device=0)
    gpu.construct_vhost_scsi_controller("life.ctl")
    gpu.add_vhost_scsi_lun("life.ctl", 0, "life0")
    gpu.add_vhost_scsi_lun("life.ctl", 2, "life1")
    try:
        def session(seed, home, peer_too=False):
            t = traces.fuzz_trace(200, nb, seed=seed, max_io_blocks=64, target=home)
            if peer_too:                             # half of the well-formed requests to the other device
                ok = t.reqs["lun"][:, 0] == 1
                t.reqs["lun"][ok & (np.arange(len(t.reqs)) % 2 == 1), 1] = 2 - home
            host = np.zeros(t.arena_bytes, dtype=np.uint8)
            traces.fill_arena(host, t)
            dev = torch.from_numpy(host).to("cuda:0")
            with gpu.Lun("life.ctl", home, num_queues=1, queue_size=1024) as lun:
                lun.run(t.reqs, t.bind(dev.data_ptr()))
                torch.cuda.synchronize()
                own = lun.iostat()
                peer = lun.iostat(2 - home)
                during = gpu.get_bdevs_iostat(f"life{home // 2}"), gpu.get_bdevs_iostat(f"life{1 - home // 2}")
            return own, peer, during

        def plus(a, b):
            return {f: a[f] + b[f] for f in LIFETIME}

        zero = dict.fromkeys(LIFETIME, 0)
        own1, _, (d0, _) = session(11, 0)
        assert own1["num_read_ops"] and own1["num_unmap_ops"] and own1["read_latency_ns"] and own1["unmap_latency_ns"]
        assert {f: d0[f] for f in LIFETIME} == plus(zero, own1), "open session: get_bdevs_iostat = lun.iostat"
        after1 = gpu.get_bdevs_iostat("life0")
        assert {f: after1[f] for f in LIFETIME} == plus(zero, own1), "closing the session keeps the totals"
        own2, _, (d0, _) = session(12, 0)
        assert {f: d0[f] for f in LIFETIME} == plus(own1, own2), "second session, open"
        after2 = gpu.get_bdevs_iostat("life0")
        assert {f: after2[f] for f in LIFETIME} == plus(own1, own2), "two sessions in sequence add up"
        # life1 reached through a session whose home is life0: the peer's counters land on life1
        own3, peer3, (d0, d1) = session(13, 0, peer_too=True)
        assert peer3["num_read_ops"] + peer3["num_write_ops"] > 0
        assert {f: d0[f] for f in LIFETIME} == plus(plus(own1, own2), own3)
        assert {f: d1[f] for f in LIFETIME} == plus(zero, peer3), "peer target, open"
        after3 = gpu.get_bdevs_iostat("life1")
        assert {f: after3[f] for f in LIFETIME} == plus(zero, peer3), "peer target, closed"
        # and the same bdev as a home device afterwards adds to it
        own4, _, (d1, _) = session(14, 2)
        assert {f: d1[f] for f in LIFETIME} == plus(peer3, own4)
    finally:
        gpu.remove_vhost_scsi_target("life.ctl", 0)
        gpu.remove_vhost_scsi_target("life.ctl", 2)
        gpu.remove_vhost_controller("life.ctl")
        gpu.delete_bdev("life0")
        gpu.delete_bdev("life1")
