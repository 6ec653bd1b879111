"""Persistent mode: the resident reactor kernel served by doorbells (GPU only).  Every test arms the
kernel's idle watchdog so a failing assertion cannot leave a spinning kernel behind."""
import time

import numpy as np
import pytest

import util
from oim_b200 import abi, traces, vring
from test_vring import VQ_KERNELS, VQ_MIRROR_KERNELS

pytestmark = pytest.mark.gpu
WATCHDOG_MS = 4000
# the resident kernel a single guest ring of 256 runs on: the shared-queue kernel (default); with
# OIMGPU_NO_SHARED_QUEUES=1 oim_lun_vring_kernel, where mover warp 0 publishes; with OIMGPU_NO_VRING_KERNEL=1 as well,
# oim_lun_queue_kernel, where the parser publishes
POLLER_VARIANTS = VQ_KERNELS
# the two mirror kernels resident, on two and three replicas on cuda:0: variant -> (environment, replicas)
MIRROR_POLLER_VARIANTS = {f"{k}-r{r}": (env, r) for r in (2, 3) for k, env in VQ_MIRROR_KERNELS.items()}
POLLER_CASES = {**{k: (env, 1) for k, env in POLLER_VARIANTS.items()}, **MIRROR_POLLER_VARIANTS}


def _shared(variant: str) -> bool:
    """whether the variant's resident kernel shares the queues a pass at a time (shared_launches)"""
    return variant == "shared" or variant.startswith("mirror-shared")


def _setup(gpu, name, nb, replicas=1):
    if replicas > 1:
        gpu.construct_mirror_bdev(nb, 512, [0] * replicas, name=name)
        assert gpu.get_bdevs(name)[0]["replicas"] == replicas
    else:
        gpu.construct_malloc_bdev(nb, 512, name=name, device=0)
    gpu.construct_vhost_scsi_controller(name + ".ctl")
    gpu.add_vhost_scsi_lun(name + ".ctl", 0, name)
    for r in range(replicas):
        gpu.bdev_write_raw(name, 0, traces.pattern_bytes(7, 0, nb * 512), replica=r)


def _check_replicas(gpu, name, nb, replicas, want_store):
    for r in range(replicas):
        bad = np.nonzero(gpu.bdev_read_raw(name, 0, nb * 512, replica=r) != want_store)[0]
        assert not len(bad), f"replica {r} of {replicas} differs from the oracle at {len(bad)} bytes, first {bad[:8]}"


def _teardown(gpu, name):
    gpu.remove_vhost_scsi_target(name + ".ctl", 0)
    gpu.remove_vhost_controller(name + ".ctl")
    gpu.delete_bdev(name)


@pytest.mark.timeout(120)
def test_poller_serves_ring_doorbells(gpu, oracles):
    """closed loop, qd=32 per queue: submit 32, ring the doorbell, wait for the completion counter"""
    _ring_doorbells(gpu, oracles, "pl0", {}, 1, 64)


@pytest.mark.timeout(120)
@pytest.mark.parametrize("variant", list(MIRROR_POLLER_VARIANTS))
def test_poller_serves_ring_doorbells_on_a_mirror(gpu, oracles, variant):
    """the same on a mirror, with rings of 256 so that the resident mirror-shared kernel has CTAs to share them"""
    env, replicas = MIRROR_POLLER_VARIANTS[variant]
    _ring_doorbells(gpu, oracles, f"plm{variant}", env, replicas, 256, shared=_shared(variant))


def _ring_doorbells(gpu, oracles, name, env, replicas, queue_size, shared=None):
    import torch
    nb, nq, rounds = 1 << 16, 4, 12
    t = traces.partitioned_queues(nq, 32 * rounds, nb, pattern="randrw", read_pct=60, io_blocks=8)
    host = np.zeros(t.arena_bytes, dtype=np.uint8)
    traces.fill_arena(host, t)
    with oracles.PortOracle(nb) as o:
        o.store[:] = traces.pattern_bytes(7, 0, o.store.size)
        oa = host.copy()
        want = o.submit(t.reqs, t.bind(oa.ctypes.data))
        want_store = o.store.copy()
    _setup(gpu, name, nb, replicas)
    try:
        arena = torch.from_numpy(host.copy()).pin_memory()
        iovs = t.bind(arena.data_ptr())
        per_q = 32 * rounds
        got = np.zeros(len(t.reqs), dtype=abi.cpl_dtype)
        with util.environ(**env), gpu.Lun(name + ".ctl", 0, num_queues=nq, queue_size=queue_size) as lun:
            assert lun.start_poller(idle_timeout_ms=WATCHDOG_MS) >= nq      # workers: one per queue, more when they share queues
            if shared is not None:
                assert lun.shared_launches == shared, f"the resident kernel {'does not share' if shared else 'shares'} the queues"
            launches_before = None
            try:
                for r in range(rounds):
                    for q in range(nq):
                        lo = q * per_q + r * 32
                        part = t.reqs[lo:lo + 32].copy()
                        i0 = int(part["iov_start"][0])
                        part["iov_start"] -= np.uint32(i0)
                        lun.submit(q, part, iovs[i0:i0 + 32])
                    assert lun.kick() == nq                   # doorbells, not launches
                    for q in range(nq):
                        c = lun.poll(q, 32, wait=True)
                        assert len(c) == 32
                        got[q * per_q + r * 32:q * per_q + r * 32 + 32] = c
                assert lun.poller_running()
            finally:
                lun.stop_poller()
            stats = lun.iostat()
        assert stats["kernel_launches"] == 1, "one resident kernel served every round"
        util.assert_cpls_equal(got, want, t.reqs)
        assert (arena.numpy() == oa).all()
        _check_replicas(gpu, name, nb, replicas, want_store)
    finally:
        _teardown(gpu, name)


@pytest.mark.timeout(120)
def test_poller_serves_guest_virtqueue(gpu, oracles):
    """a guest image in pinned memory: the 'guest' publishes avail->idx in two steps, the resident
    kernel answers through the used ring without any host call"""
    import torch
    nb = 32768
    t = traces.fuzz_trace(48, nb, seed=77, max_io_blocks=16, arena_bytes=8 << 20, include_malformed=False)
    a0 = np.zeros(t.arena_bytes, dtype=np.uint8)
    traces.fill_arena(a0, t)
    rq = vring.requests_from_trace(t, a0)
    img = vring.build_image(rq, ring_size=256, seed=3, mutate=False)
    n = img.meta["placed"]
    assert n == 48
    ref = vring.build_image(rq, ring_size=256, seed=3, mutate=False)
    with oracles.PortOracle(nb) as o:
        o.store[:] = traces.pattern_bytes(7, 0, o.store.size)
        o.vq_process(ref)
        want_store = o.store.copy()
    _setup(gpu, "pv0", nb)
    try:
        guest = torch.from_numpy(img.arena.copy()).pin_memory()
        g = guest.numpy()
        avail_idx = g[img.avail_off + 2:img.avail_off + 4].view("<u2")
        used_idx = g[img.used_off + 2:img.used_off + 4].view("<u2")
        avail_idx[0] = 0                                       # nothing published yet
        base = guest.data_ptr()
        with gpu.Lun("pv0.ctl", 0, num_queues=1, queue_size=32) as lun:
            lun.set_mem_table(img.region_table(base))
            lun.vq_attach(0, base + img.desc_off, base + img.avail_off, base + img.used_off, img.ring_size, 0, 0)
            lun.start_poller(idle_timeout_ms=WATCHDOG_MS)
            try:
                for target in (20, n):
                    avail_idx[0] = target                      # the guest's "kick" is just this store
                    deadline = time.time() + 20
                    while int(used_idx[0]) != target and time.time() < deadline:
                        time.sleep(0.0005)
                    assert int(used_idx[0]) == target, f"used->idx stuck at {int(used_idx[0])}"
            finally:
                lun.stop_poller()
            la, lu = lun.vq_detach(0)
        assert (la, lu) == (n, n)
        got = img.masked(g.copy())
        assert (got == ref.masked(ref.arena)).all()
        assert (gpu.bdev_read_raw("pv0", 0, nb * 512) == want_store).all()
    finally:
        _teardown(gpu, "pv0")


@pytest.mark.timeout(60)
def test_poller_watchdog_and_busy_errors(gpu):
    import errno
    _setup(gpu, "pw0", 4096)
    try:
        with gpu.Lun("pw0.ctl", 0, num_queues=2, queue_size=32) as lun:
            lun.start_poller(idle_timeout_ms=300)
            with pytest.raises(gpu.OimGpuError) as e:
                lun.iostat()                                   # would need to drain the stream
            assert e.value.rc == -errno.EBUSY
            t0 = time.time()
            while lun.poller_running() and time.time() - t0 < 10:
                time.sleep(0.01)
            assert not lun.poller_running(), "idle watchdog did not fire"
            lun.stop_poller()
            assert lun.iostat()["kernel_launches"] == 1
    finally:
        _teardown(gpu, "pw0")


@pytest.mark.gpu
@pytest.mark.timeout(180)
def test_poller_guest_reuses_ring_and_buffers(gpu, oracles):
    """What a real guest does all day under a resident kernel: the SAME descriptor slots, request headers,
    indirect tables and data buffers are rewritten by the CPU with different contents round after round,
    with nothing but the avail index as a signal.  Every round must see the new contents, never what
    the GPU read from those addresses in an earlier round."""
    import torch
    nb, rounds = 32768, 6
    imgs, refs = [], []
    with oracles.PortOracle(nb) as o:
        o.store[:] = traces.pattern_bytes(7, 0, o.store.size)
        la = lu = 0
        for r in range(rounds):
            t = traces.fuzz_trace(40, nb, seed=900 + r, max_io_blocks=32, arena_bytes=8 << 20, include_malformed=False)
            a0 = np.zeros(t.arena_bytes, dtype=np.uint8)
            traces.fill_arena(a0, t)
            rq = vring.requests_from_trace(t, a0)
            # same seed -> same ring slots, header / table / buffer addresses in every round; different requests
            img = vring.build_image(rq, ring_size=256, seed=3, mutate=False, pattern_seed=0x5EED + r)
            ref = vring.build_image(rq, ring_size=256, seed=3, mutate=False, pattern_seed=0x5EED + r)
            assert img.meta["placed"] == 40
            o.vq_process(ref)                                      # each image is a fresh ring for the oracle
            imgs.append(img)
            refs.append(ref)
        want_store = o.store.copy()
    _setup(gpu, "pv1", nb)
    try:
        guest = torch.from_numpy(imgs[0].arena.copy()).pin_memory()
        g = guest.numpy()
        img0 = imgs[0]
        avail_idx = g[img0.avail_off + 2:img0.avail_off + 4].view("<u2")
        used_idx = g[img0.used_off + 2:img0.used_off + 4].view("<u2")
        avail_idx[0] = 0
        base = guest.data_ptr()
        with gpu.Lun("pv1.ctl", 0, num_queues=1, queue_size=32) as lun:
            lun.set_mem_table(img0.region_table(base))
            lun.vq_attach(0, base + img0.desc_off, base + img0.avail_off, base + img0.used_off, img0.ring_size, 0, 0)
            lun.start_poller(idle_timeout_ms=WATCHDOG_MS)
            try:
                done = 0
                for r in range(rounds):
                    img = imgs[r]
                    if r:
                        # the guest rewrites its memory in place: everything except the ring indices, then
                        # the avail ring entries at the positions the next 40 heads go to
                        keep_a, keep_u = int(avail_idx[0]), int(used_idx[0])
                        lo, hi = img.avail_off, img.used_off + 4 + 8 * img.ring_size
                        g[:lo] = img.arena[:lo]
                        g[hi:] = img.arena[hi:]
                        ring = g[img.avail_off + 4:img.avail_off + 4 + 2 * img.ring_size].view("<u2")
                        src = img.arena[img.avail_off + 4:img.avail_off + 4 + 2 * img.ring_size].view("<u2")
                        for k in range(40):
                            ring[(keep_a + k) % img.ring_size] = src[k]
                        assert (int(avail_idx[0]), int(used_idx[0])) == (keep_a, keep_u)
                    done += 40
                    avail_idx[0] = done
                    deadline = time.time() + 20
                    while int(used_idx[0]) != done and time.time() < deadline:
                        time.sleep(0.0005)
                    assert int(used_idx[0]) == done, f"round {r}: used->idx stuck at {int(used_idx[0])}"
                    # everything outside the two rings equals what the oracle left for this round's image
                    want = refs[r].arena
                    lo, hi = img.avail_off, img.used_off + 4 + 8 * img.ring_size
                    assert (g[:lo] == want[:lo]).all(), f"round {r}: guest memory differs at {np.nonzero(g[:lo] != want[:lo])[0][:8]}"
                    assert (g[hi:] == want[hi:]).all(), f"round {r}: guest memory differs at {hi + np.nonzero(g[hi:] != want[hi:])[0][:8]}"
            finally:
                lun.stop_poller()
        assert (gpu.bdev_read_raw("pv1", 0, nb * 512) == want_store).all()
    finally:
        _teardown(gpu, "pv1")


@pytest.mark.gpu
@pytest.mark.timeout(120)
@pytest.mark.parametrize("resident", [False, True])
def test_slot_ring_passes_that_straddle_the_ring_end(gpu, oracles, resident):
    """Submissions of uneven size on one 64-slot ring: passes start at slot 16, 48 (-> wraps to 16), ... so a pass's
    slots lie in two pieces of the ring - the TMA unit fetches them with two bulk copies (lun_kernel.cu issue_fetch).
    Launch per kick and resident poller; results equal the oracle's sequential execution."""
    import torch
    nb = 1 << 15
    sizes = [16, 32, 32, 7, 32, 25, 32, 32, 1, 31, 32, 32]
    n = sum(sizes)
    t = traces.uniform_trace(n, nb, io_blocks=8, pattern="randrw", read_pct=50, seed=91, lba_span=4096)
    host = np.zeros(t.arena_bytes, dtype=np.uint8)
    traces.fill_arena(host, t)
    with oracles.PortOracle(nb) as o:
        o.store[:] = traces.pattern_bytes(7, 0, o.store.size)
        oa = host.copy()
        want = o.submit(t.reqs, t.bind(oa.ctypes.data))
        want_store = o.store.copy()
    name = "wrap1" if resident else "wrap0"
    _setup(gpu, name, nb)
    try:
        arena = torch.from_numpy(host.copy()).pin_memory()
        iovs = t.bind(arena.data_ptr())
        got = []
        with gpu.Lun(name + ".ctl", 0, num_queues=1, queue_size=64) as lun:
            if resident:
                lun.start_poller(idle_timeout_ms=WATCHDOG_MS)
            try:
                lo = 0
                for k in sizes:
                    part = t.reqs[lo:lo + k].copy()
                    i0 = int(part["iov_start"][0])
                    part["iov_start"] -= np.uint32(i0)
                    lun.submit(0, part, iovs[i0:i0 + k])
                    lun.kick()
                    c = lun.poll(0, k, wait=True)
                    assert len(c) == k
                    got.append(c)
                    lo += k
            finally:
                if resident:
                    lun.stop_poller()
        util.assert_cpls_equal(np.concatenate(got), want, t.reqs)
        assert (arena.numpy() == oa).all()
        assert (gpu.bdev_read_raw(name, 0, nb * 512) == want_store).all()
    finally:
        _teardown(gpu, name)


def _wait_used(used_idx, target, what, timeout_s=20.0):
    deadline = time.time() + timeout_s
    while int(used_idx[0]) != target and time.time() < deadline:
        time.sleep(0.0005)
    assert int(used_idx[0]) == target, f"{what}: used->idx is {int(used_idx[0])} after {timeout_s:.0f} s, expected {target}"


@pytest.mark.timeout(180)
@pytest.mark.parametrize("variant", list(POLLER_CASES))
def test_poller_guest_ring_across_the_index_wrap(gpu, oracles, variant):
    """test_poller_guest_reuses_ring_and_buffers from cursor 65536 - 100: rounds of 40 requests carry avail->idx and
    used->idx across the 16-bit wrap and the ring's end under the resident kernel.  After stop_poller the cursors
    vq_detach returns are the oracle's, mod 2^16."""
    import torch
    nb, rounds, per, R = 32768, 5, 40, 256
    start = 65536 - 100
    imgs, refs, cur = [], [], []
    with oracles.PortOracle(nb) as o:
        o.store[:] = traces.pattern_bytes(7, 0, o.store.size)
        la = lu = start
        for r in range(rounds):
            t = traces.fuzz_trace(per, nb, seed=950 + r, max_io_blocks=32, arena_bytes=8 << 20, include_malformed=False)
            a0 = np.zeros(t.arena_bytes, dtype=np.uint8)
            traces.fill_arena(a0, t)
            rq = vring.requests_from_trace(t, a0)
            kw = dict(ring_size=R, seed=3, mutate=False, pattern_seed=0x5EED + r, start_avail=la, start_used=lu)
            img, ref = vring.build_image(rq, **kw), vring.build_image(rq, **kw)
            assert img.meta["placed"] == per
            cur.append((la, lu))
            n, la, lu = o.vq_process(ref, la, lu)
            assert n == per
            imgs.append(img)
            refs.append(ref)
        want_store = o.store.copy()
        want_cursors = (la, lu)
    assert want_cursors == ((start + rounds * per) & 0xFFFF,) * 2
    name = f"pvw{variant}"
    env, replicas = POLLER_CASES[variant]
    _setup(gpu, name, nb, replicas)
    try:
        img0 = imgs[0]
        guest = torch.from_numpy(img0.arena.copy()).pin_memory()
        g = guest.numpy()
        avail_idx = g[img0.avail_off + 2:img0.avail_off + 4].view("<u2")
        used_idx = g[img0.used_off + 2:img0.used_off + 4].view("<u2")
        avail_idx[0] = start                                   # nothing published yet
        base = guest.data_ptr()
        lo, hi = img0.avail_off, img0.used_off + 4 + 8 * R
        with util.environ(**env), gpu.Lun(f"{name}.ctl", 0, num_queues=1, queue_size=32) as lun:
            lun.set_mem_table(img0.region_table(base))
            lun.vq_attach(0, base + img0.desc_off, base + img0.avail_off, base + img0.used_off, R, start, start)
            shared = lun.shared_launches
            lun.start_poller(idle_timeout_ms=WATCHDOG_MS)
            try:
                assert lun.shared_launches - shared == _shared(variant), f"the poller is not the {variant} kernel"
                for r in range(rounds):
                    img, (la, lu) = imgs[r], cur[r]
                    if r:
                        # the guest rewrites its memory in place, then the avail entries of this round's window
                        g[:lo] = img.arena[:lo]
                        g[hi:] = img.arena[hi:]
                        ring = g[img.avail_off + 4:img.avail_off + 4 + 2 * R].view("<u2")
                        src = img.arena[img.avail_off + 4:img.avail_off + 4 + 2 * R].view("<u2")
                        pos = (la + np.arange(per)) & (R - 1)
                        ring[pos] = src[pos]
                    assert int(used_idx[0]) == lu
                    avail_idx[0] = (la + per) & 0xFFFF
                    _wait_used(used_idx, (lu + per) & 0xFFFF, f"round {r} (from {la},{lu})")
                    used = img.used_in_order(g, lu, per)
                    assert [int(i) for i in used["id"]] == img.heads, f"round {r}: used elements out of ring order"
                    assert sorted((int(i), int(l)) for i, l in used) == \
                        sorted((int(i), int(l)) for i, l in refs[r].used_in_order(None, lu, per)), f"round {r}: used elements"
                    want = refs[r].arena
                    assert (g[:lo] == want[:lo]).all(), f"round {r}: guest memory differs at {np.nonzero(g[:lo] != want[:lo])[0][:8]}"
                    assert (g[hi:] == want[hi:]).all(), f"round {r}: guest memory differs at {hi + np.nonzero(g[hi:] != want[hi:])[0][:8]}"
            finally:
                lun.stop_poller()
            assert lun.vq_detach(0) == want_cursors
            assert lun.iostat()["kernel_launches"] == 1, "one resident kernel served every round"
        _check_replicas(gpu, name, nb, replicas, want_store)
    finally:
        _teardown(gpu, name)


def _spin_us(us: float) -> None:
    t = time.perf_counter() + us * 1e-6
    while time.perf_counter() < t:
        pass


@pytest.mark.timeout(180)
@pytest.mark.parametrize("variant", list(POLLER_CASES))
def test_poller_guest_publishes_while_a_batch_moves(gpu, oracles, variant):
    """A Linux guest bumps avail->idx for every request it adds, so the resident kernel finds new requests on a ring
    while the batch before them is still moving.  First 32 READs of 1 MiB into guest memory (pinned host memory:
    around a millisecond of PCIe traffic, estimated), then the rest of a fuzz trace one request at a time - avail
    entry, then avail->idx + 1, tens of microseconds apart - including writes to the blocks the READs read.  From
    cursor 65536 - 50, so the batches also cross the 16-bit wrap.  Everything equals the oracle's single pass over the
    same image: used->idx, the used elements in ring order, guest memory, store, and the cursors after stop."""
    import torch
    nb, R, big = 32768, 256, 2048
    start = 65536 - 50
    rng = np.random.default_rng(61)
    reads = []
    for k in range(32):
        cdb = np.zeros(32, dtype=np.uint8)
        c = abi.cdb_rw(abi.READ_10, int(rng.integers(0, nb - big)), big)
        cdb[:len(c)] = c
        reads.append({"cdb": cdb, "dir": abi.DIR_FROM_DEV, "lun": abi.virtio_lun(0), "tag": 0x7000 + k,
                      "sg": [big * 512], "payload": None})
    t = traces.fuzz_trace(96, nb, seed=62, max_io_blocks=64, arena_bytes=8 << 20, include_malformed=False)
    a0 = np.zeros(t.arena_bytes, dtype=np.uint8)
    traces.fill_arena(a0, t)
    rq = reads + vring.requests_from_trace(t, a0)
    n = len(rq)
    kw = dict(ring_size=R, seed=4, mutate=False, all_indirect=True, data_bytes=48 << 20, start_avail=start, start_used=start)
    img, ref = vring.build_image(rq, **kw), vring.build_image(rq, **kw)
    assert img.meta["placed"] == n
    end = (start + n) & 0xFFFF
    with oracles.PortOracle(nb) as o:
        o.store[:] = traces.pattern_bytes(7, 0, o.store.size)
        assert o.vq_process(ref, start, start) == (n, end, end)
        want_store = o.store.copy()
    name = f"pvs{variant}"
    env, replicas = POLLER_CASES[variant]
    _setup(gpu, name, nb, replicas)
    try:
        guest = torch.from_numpy(img.arena.copy()).pin_memory()
        g = guest.numpy()
        avail_idx = g[img.avail_off + 2:img.avail_off + 4].view("<u2")
        used_idx = g[img.used_off + 2:img.used_off + 4].view("<u2")
        ring = g[img.avail_off + 4:img.avail_off + 4 + 2 * R].view("<u2")
        pos = (start + np.arange(n)) & (R - 1)
        ring[pos[32:]] = (ring[pos[32:]] + 1) % R             # not yet written by the guest: wrong heads
        avail_idx[0] = start
        base = guest.data_ptr()
        with util.environ(**env), gpu.Lun(f"{name}.ctl", 0, num_queues=1, queue_size=32) as lun:
            lun.set_mem_table(img.region_table(base))
            lun.vq_attach(0, base + img.desc_off, base + img.avail_off, base + img.used_off, R, start, start)
            shared = lun.shared_launches
            lun.start_poller(idle_timeout_ms=WATCHDOG_MS)
            try:
                assert lun.shared_launches - shared == _shared(variant), f"the poller is not the {variant} kernel"
                avail_idx[0] = (start + 32) & 0xFFFF               # the 32 large READs
                for k in range(32, n):
                    _spin_us(30)
                    ring[pos[k]] = img.heads[k]                    # the avail entry, then the index that publishes it
                    avail_idx[0] = (start + k + 1) & 0xFFFF
                _wait_used(used_idx, end, f"{n} requests published one by one from {start}")
            finally:
                lun.stop_poller()
            cursors = lun.vq_detach(0)
            assert lun.iostat()["kernel_launches"] == 1, "one resident kernel served the whole stream"
        used = img.used_in_order(g, start, n)
        assert [int(i) for i in used["id"]] == img.heads, "used elements out of ring order"
        assert sorted((int(i), int(l)) for i, l in used) == sorted((int(i), int(l)) for i, l in ref.used_in_order(None, start, n))
        assert img.used_untouched(g, start, n), "a used element outside the published window was written"
        got, want = img.masked(g.copy()), ref.masked(ref.arena)
        assert (got == want).all(), f"guest memory differs at {np.nonzero(got != want)[0][:8]}"
        assert cursors == (end, end)
        _check_replicas(gpu, name, nb, replicas, want_store)
    finally:
        _teardown(gpu, name)
