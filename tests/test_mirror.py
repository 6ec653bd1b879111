"""Config 5: R-way mirrored bdev, write fan-out over NVLink by P2P stores from the mover warps.
No reference implementation exists (S/lib/bdev/raid is RAID0 only); parity = every replica's content
equals the single-bdev oracle's after the same write trace (SURVEY.md 8(c)).  Both replicas on one GPU
([0, 0]) run the same mirror kernels without NVLink, so the fan-out is checked on a single GPU too.

Beyond that one shape: 3 and 4 replicas, mirrors as peer targets of a controller (home elsewhere and controller-wide,
slot rings and a guest virtqueue), hot-plug that changes the kernel variant, replicas imported from another process,
and the digest the bench's replica parity rests on.  The resident poller, NBD and several queues on a mirror are in
test_poller.py, test_nbd.py and test_shared_queues.py."""
import numpy as np
import pytest

import util
from oim_b200 import abi, traces, vring

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gpu2():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs (gpurun --gpus 2)")
    from oim_b200 import build, lib
    build.build()
    for d in (0, 1):
        torch.zeros(1, device=f"cuda:{d}")
    lib.fini()
    lib.init([0, 1])
    yield lib
    lib.fini()
    lib.init([0])           # what the session-wide `gpu` fixture set up: the modules after this one rely on it


def test_mirror_write_fanout_matches_oracle(gpu2, oracles):
    """replicas on cuda:0 and cuda:1: the fan-out by P2P stores"""
    _write_fanout(gpu2, oracles, [0, 1])


def test_mirror_write_fanout_on_one_gpu(gpu, oracles):
    """both replicas on cuda:0: the mirror kernels and their byte-granular mover without a second GPU"""
    _write_fanout(gpu, oracles, [0, 0])


def _write_fanout(lib, oracles, devices):
    import torch
    nb = 1 << 16
    t = traces.fuzz_trace(600, nb, seed=515, max_io_blocks=128, arena_bytes=32 << 20, include_malformed=False)
    want = util.run_oracle(oracles.PortOracle, t, nb)
    name = lib.construct_mirror_bdev(nb, 512, devices, name="mir0")
    lib.construct_vhost_scsi_controller("mir.ctl")
    lib.add_vhost_scsi_lun("mir.ctl", 0, name)
    try:
        init = traces.pattern_bytes(7, 0, nb * 512)
        for rep in (0, 1):
            lib.bdev_write_raw(name, 0, init, replica=rep)
        assert lib.get_bdevs(name)[0]["replicas"] == 2
        host = np.zeros(t.arena_bytes, dtype=np.uint8)
        traces.fill_arena(host, t)
        dev = torch.from_numpy(host).to("cuda:0")
        with util.environ(**util.kernel_env("mirror-shared")), lib.Lun("mir.ctl", 0, num_queues=1, queue_size=1024) as lun:
            assert lun.device == 0
            cpls = lun.run(t.reqs, t.bind(dev.data_ptr()))
            assert lun.iostat()["kernel_launches"] == 1 and lun.shared_launches == 1, "one shared launch of the mirror kernel"
        util.assert_cpls_equal(cpls, want[0], t.reqs)
        assert (dev.cpu().numpy() == want[1]).all()
        for rep in (0, 1):
            got = lib.bdev_read_raw(name, 0, nb * 512, replica=rep)
            assert (got == want[2]).all(), f"replica {rep} differs from the oracle store"
    finally:
        lib.remove_vhost_scsi_target("mir.ctl", 0)
        lib.remove_vhost_controller("mir.ctl")
        lib.delete_bdev(name)


# ---- three and four replicas ------------------------------------------------------------------------------------

def _mirror_trace(name: str, nb: int) -> traces.Trace:
    """'sweep': traces.alignment_sweep (every (client, store) skew through move_unit<true>'s compact path); 'fuzzN':
    the fuzzer's adversarial trace (UNMAP, malformed requests, ragged SG lists) with seed N"""
    if name == "sweep":
        return traces.alignment_sweep(nb)
    seed = int(name[4:])
    t = traces.fuzz_trace(500, nb, seed=seed, max_io_blocks=[64, 300][seed % 2], arena_bytes=16 << 20)
    assert (t.reqs["cdb"][:, 0] == abi.UNMAP).any()
    return t


def _compare(got, want, t, what):
    util.assert_cpls_equal(got[0], want[0], t.reqs, what)
    bad = np.nonzero(got[1] != want[1])[0]
    assert not len(bad), f"{what}: client arena differs at {len(bad)} bytes, first {bad[:8]}"
    bad = np.nonzero(got[2] != want[2])[0]
    assert not len(bad), f"{what}: store differs at {len(bad)} bytes, first {bad[:8]}"


@pytest.mark.parametrize("name", ["fuzz521", "fuzz522", "sweep"])
@pytest.mark.parametrize("replicas", [3, 4])
@pytest.mark.parametrize("kernel", util.MIRROR_KERNELS)
def test_mirror_replicas_match_oracle(gpu, oracles, kernel, replicas, name):
    """replicas 3 and 4 on cuda:0 (mirror_unit's loop past replica 1): one launch; completions, client bytes and
    replica 0 equal the oracle's, every other replica equals replica 0 (util.run_cuda)"""
    nb = 65536
    t = _mirror_trace(name, nb)
    want = util.run_oracle(oracles.PortOracle, t, nb)
    got = util.run_cuda(gpu, t, nb, kernel=kernel, replicas=replicas)
    _compare(got, want, t, f"{kernel}, {replicas} replicas, {name}")


@pytest.mark.parametrize("bs", (4097, 1 << 20), ids=lambda bs: f"{bs >> 20}M" if bs >= 1 << 20 else str(bs))
@pytest.mark.parametrize("kernel", util.MIRROR_KERNELS)
def test_mirror_four_replicas_at_block_size_edges(gpu, oracles, kernel, bs):
    """traces.block_size_trace on four replicas: transfers up to the 4 MiB limit, fills over 1 MiB, UNMAP extents
    in blocks of a size that is not a power of two"""
    from test_block_sizes import blocks, make_trace, want
    t = make_trace(bs, "edges")
    w = want(oracles, bs, "edges")
    got = util.run_cuda(gpu, t, blocks(bs), block_size=bs, kernel=kernel, replicas=4)
    _compare(got, w, t, f"{kernel}, 4 replicas, block size {bs}")


def test_mirror_with_five_replicas_is_refused(gpu):
    import errno
    with pytest.raises(gpu.OimGpuError) as e:
        gpu.construct_mirror_bdev(64, 512, [0] * 5, name="mir5")
    assert e.value.rc == -errno.EINVAL
    assert "mir5" not in [b["name"] for b in gpu.get_bdevs()]


# ---- mirrors as targets of a controller -------------------------------------------------------------------------
# Every vhost-user connection is a controller-wide session (target -1): the only way a VM reaches a mirror is as a
# peer target, whose writes fan out through LunCtx::peer (emit_segments, move_seg_unit, scsi_unmap).

IO_COUNTERS = ("num_read_ops", "num_write_ops", "num_unmap_ops", "num_other_ops", "bytes_read", "bytes_written",
               "bytes_unmapped", "num_errors")
# target -> devices of its replicas
CTRLR_MIRRORS = {"m3": {3: [0, 0, 0]}, "m1m3": {1: [0, 0], 3: [0, 0, 0]}}


def _controller_run(gpu, c, home, t, side):
    """one launch of the whole multi-target trace on `side` (exclusive / shared) through a session with home
    target `home`; -> cpls, client arena, {target: iostat}"""
    import torch
    host = np.zeros(t.arena_bytes, dtype=np.uint8)
    traces.fill_arena(host, t)
    dev = torch.from_numpy(host).to("cuda:0")
    with util.environ(**util.kernel_env(side)), gpu.Lun(c.ctrlr, home, num_queues=1, queue_size=32) as lun:
        cpls = util._run_device_arrays(lun, t.reqs, t.bind(dev.data_ptr()))
        stats = {k: lun.iostat(k) for k in c.sizes}
        assert stats[1]["kernel_launches"] == 1
        assert lun.shared_launches == (side == "shared"), f"the launch was not on the {side} side"
    return cpls, dev.cpu().numpy(), stats


@pytest.mark.parametrize("side", ["exclusive", "shared"])
@pytest.mark.parametrize("home", [1, 3, -1])
@pytest.mark.parametrize("seed,mirrors", [(760, "m3"), (761, "m1m3"), (762, "m1m3")])
def test_mirror_targets_of_a_controller_match_oracle(gpu, oracles, seed, mirrors, home, side):
    """target 3 a mirror of three replicas, target 1 a mirror of two or plain, target 6 plain; sessions at home on
    the plain target, on the mirror and controller-wide.  Every replica of every target equals the oracle's store,
    and each target's counters count every I/O once: they equal those of the same trace on plain bdevs."""
    from test_multi_target import Controller, multi_trace, run_oracle
    t = multi_trace(seed)
    c = Controller(gpu, mirrors=CTRLR_MIRRORS[mirrors])
    try:
        wc, wa, ws, _ = run_oracle(oracles.PortOracle, t, c.names, c.ids())
        gc, ga, stats = _controller_run(gpu, c, home, t, side)
        what = f"home {home}, {side}, mirrors {CTRLR_MIRRORS[mirrors]}"
        util.assert_cpls_equal(gc, wc, t.reqs, what)
        assert (ga == wa).all(), f"{what}: client memory differs at {np.nonzero(ga != wa)[0][:8]}"
        for (k, r), st in c.replica_stores().items():
            bad = np.nonzero(st != ws[k])[0]
            assert not len(bad), f"{what}: target {k} replica {r} differs from the oracle at {len(bad)} bytes, first {bad[:8]}"
    finally:
        c.close()
    plain = Controller(gpu)
    try:
        _, _, plain_stats = _controller_run(gpu, plain, home, t, side)
    finally:
        plain.close()
    for k in stats:
        got = {n: stats[k][n] for n in IO_COUNTERS}
        assert got == {n: plain_stats[k][n] for n in IO_COUNTERS}, f"target {k}: counters on mirrors {got} vs plain {plain_stats[k]}"
    assert stats[3]["num_write_ops"] > 0 and stats[3]["num_unmap_ops"] + stats[1]["num_unmap_ops"] > 0


@pytest.mark.parametrize("kernel", util.MIRROR_KERNELS)
def test_mirror_targets_through_a_controller_wide_virtqueue(gpu, oracles, kernel):
    """a guest virtio ring on a controller-wide session: WRITEs and UNMAPs to the peer mirrors fan out to every replica"""
    import torch
    from test_multi_target import TARGETS, Controller, multi_trace
    from test_vring import VQ_MIRROR_KERNELS
    t = multi_trace(732, n=96)
    assert ((t.reqs["cdb"][:, 0] == abi.UNMAP) & (t.reqs["lun"][:, 1] == 3)).sum() >= 2, "UNMAPs to the 3-way mirror"
    a0 = np.zeros(t.arena_bytes, dtype=np.uint8)
    traces.fill_arena(a0, t)
    rq = vring.requests_from_trace(t, a0)
    img = vring.build_image(rq, ring_size=1024, seed=9, mutate=False)
    assert img.meta["placed"] == len(rq)
    c = Controller(gpu, mirrors={1: [0, 0], 3: [0, 0, 0]})
    try:
        with oracles.PortOracle(TARGETS[1], 512, 1) as o:
            o.store[:] = traces.pattern_bytes(7, 0, o.store.size)
            for k in (3, 6):
                o.add_target(k, TARGETS[k])[:] = traces.pattern_bytes(7 + k, 0, TARGETS[k] * 512)
            ref_img = vring.build_image(rq, ring_size=1024, seed=9, mutate=False)
            n, la, lu = o.vq_process(ref_img)
            want_mem = ref_img.masked(ref_img.arena)
            want_stores = {1: o.store.copy(), 3: o.stores[3].copy(), 6: o.stores[6].copy()}
        dev = torch.from_numpy(img.arena).to("cuda:0")
        with util.environ(**VQ_MIRROR_KERNELS[kernel]), gpu.Lun(c.ctrlr, -1, num_queues=1, queue_size=32) as lun:
            base = dev.data_ptr()
            lun.set_mem_table(img.region_table(base))
            lun.vq_attach(0, base + img.desc_off, base + img.avail_off, base + img.used_off, img.ring_size, 0, 0)
            assert lun.vq_kick() == 1
            lun.sync()
            assert lun.vq_detach(0) == (la, lu)
            assert lun.iostat(3)["kernel_launches"] == 1
            assert lun.shared_launches == (kernel == "mirror-shared"), f"the launch was not the {kernel} kernel"
        got = img.masked(dev.cpu().numpy())
        assert (got == want_mem).all(), f"guest memory differs at {np.nonzero(got != want_mem)[0][:8]}"
        for (k, r), st in c.replica_stores().items():
            assert (st == want_stores[k]).all(), f"target {k} replica {r} differs from the oracle"
    finally:
        c.close()


# ---- hot-plug that changes the kernel variant -------------------------------------------------------------------

def _io(lun, target, lba, nblk, write, addr):
    b = abi.Batch(target)
    (b.write if write else b.read)(lba, nblk, [(addr, nblk * 512)], tag=lba + 1)
    return lun.run(*b.arrays())[0]


def _unmap(lun, target, extents, buf):
    """UNMAP of `extents` [(lba, blocks)]; the parameter list goes to the start of pinned tensor `buf`"""
    plist = abi.unmap_param_list(extents)
    buf.numpy()[:len(plist)] = plist
    b = abi.Batch(target)
    b.add(abi.cdb_unmap(len(plist)), abi.DIR_TO_DEV, [(buf.data_ptr(), len(plist))], tag=0x4242)
    return lun.run(*b.arrays())[0]


@pytest.mark.timeout(120)
def test_mirror_hot_plugged_under_a_resident_poller(gpu):
    """a controller-wide session on a controller whose only target is plain runs the plain poller kernel.  Attaching
    a mirror must park it and restart it as the mirror kernel (a plain kernel ignores Segment::mirror: writes would
    reach replica 0 only).  Writes and UNMAPs to the mirror reach both replicas; after the detach the bdev can go."""
    import torch
    from test_multi_target import Controller
    c = Controller(gpu, only={1}, mirrors={3: [0, 0]})
    buf = torch.zeros(8192, dtype=torch.uint8).pin_memory()
    parm = torch.zeros(512, dtype=torch.uint8).pin_memory()
    nb3 = c.sizes[3][0]
    want = traces.pattern_bytes(7 + 3, 0, nb3 * 512)
    payload = traces.pattern_bytes(4343, 0, 4096)
    try:
        with gpu.Lun(c.ctrlr, -1, num_queues=1, queue_size=64) as lun:
            lun.start_poller(idle_timeout_ms=4000)
            try:
                assert _io(lun, 1, 16, 8, False, buf.data_ptr())["status"] == 0
                assert _io(lun, 3, 16, 8, False, buf.data_ptr())["response"] == abi.S_BAD_TARGET
                c.attach(3)
                assert lun.poller_running(), "the poller did not come back after the mirror was attached"
                buf.numpy()[:4096] = payload
                cp = _io(lun, 3, 40, 8, True, buf.data_ptr())
                assert (cp["response"], cp["status"]) == (abi.S_OK, 0)
                want[40 * 512:48 * 512] = payload
                cp = _unmap(lun, 3, [(100, 4), (200, 3)], parm)
                assert (cp["response"], cp["status"]) == (abi.S_OK, 0)
                want[100 * 512:104 * 512] = 0
                want[200 * 512:203 * 512] = 0
                buf.numpy()[:] = 0x11
                assert _io(lun, 3, 36, 16, False, buf.data_ptr())["status"] == 0
                assert (buf.numpy() == want[36 * 512:52 * 512]).all(), "a read after the write returned other bytes"
                assert _io(lun, 3, 96, 16, False, buf.data_ptr())["status"] == 0
                assert (buf.numpy() == want[96 * 512:112 * 512]).all(), "a read after the UNMAP returned other bytes"
                c.detach(3)
                assert _io(lun, 3, 16, 8, False, buf.data_ptr())["response"] == abi.S_BAD_TARGET
                assert _io(lun, 1, 24, 8, False, buf.data_ptr())["status"] == 0
                assert lun.poller_running()
            finally:
                lun.stop_poller()
            # the first start, the restart on the attach (other kernel variant), the restart on the detach
            assert lun.iostat()["kernel_launches"] == 3
            for r in (0, 1):
                got = gpu.bdev_read_raw(c.names[3], 0, nb3 * 512, replica=r)
                bad = np.nonzero(got != want)[0]
                assert not len(bad), f"replica {r} of the hot-plugged mirror differs at {len(bad)} bytes, first {bad[:8]}"
            gpu.delete_bdev(c.names[3])                        # no longer pinned by the session
            gpu.construct_malloc_bdev(nb3, 512, name=c.names[3], device=0)
    finally:
        c.close()


@pytest.mark.timeout(240)
def test_mirror_attached_while_a_plain_launch_is_in_flight(gpu):
    """A launch of the plain kernel is still moving a long prefix of large READs when a mirror is attached as
    target 3.  WRITEs to target 3 behind the prefix answer BAD_TARGET (the launch never saw the target) or GOOD -
    and then they are on both replicas: a plain kernel must never serve a mirror.  (Before the attach waited for
    the launch in flight, all 64 writes answered GOOD and reached replica 0 only.  Now it waits, so they answer
    BAD_TARGET; the test checks that the attach really came while the prefix was moving.)"""
    import time

    import torch
    from test_multi_target import Controller
    nread, big, nw = 4096, 8192, 64                    # 4096 READs of 4 MiB from target 1, then 64 WRITEs of 4 KiB
    c = Controller(gpu, only={1}, mirrors={3: [0, 0]})
    nb1 = c.sizes[1][0]
    init3 = traces.pattern_bytes(7 + 3, 0, c.sizes[3][0] * 512)
    payload = traces.pattern_bytes(4545, 0, nw * 4096)
    rng = np.random.default_rng(77)
    b = abi.Batch(1)
    for k in range(nread):
        b.read(int(rng.integers(0, nb1 - big + 1)), big, [(0, big * 512)], tag=k)
    for k in range(nw):
        b.write(16 * k, 8, [(big * 512 + 4096 * k, 4096)], tag=0x3000 + k, lun=abi.virtio_lun(3))
    reqs, iovs = b.arrays()
    arena = np.zeros(big * 512 + nw * 4096, dtype=np.uint8)
    arena[big * 512:] = payload
    try:
        dev = torch.from_numpy(arena).to("cuda:0")
        iovs["addr"] += np.uint64(dev.data_ptr())
        d_reqs = torch.from_numpy(reqs.view(np.uint8).copy()).to("cuda:0")
        d_iovs = torch.from_numpy(iovs.view(np.uint8).copy()).to("cuda:0")
        d_cpls = torch.zeros(len(reqs) * abi.cpl_dtype.itemsize, dtype=torch.uint8, device="cuda:0")
        torch.cuda.synchronize()
        with util.environ(**util.kernel_env("exclusive")), gpu.Lun(c.ctrlr, -1, num_queues=1, queue_size=32) as lun:
            c.attach(3)                                # the session allocates target 3's context once, here
            c.detach(3)
            stream = torch.cuda.ExternalStream(gpu.load().oimgpu_lun_stream(lun.h), device="cuda:0")
            lun.submit_device(0, d_reqs.data_ptr(), len(reqs), d_iovs.data_ptr(), d_cpls.data_ptr())
            t0 = time.perf_counter()
            lun.kick()
            in_flight = not stream.query()
            t1 = time.perf_counter()
            c.attach(3)
            t2 = time.perf_counter()
            lun.sync()
            t3 = time.perf_counter()
            launches, shared = lun.iostat()["kernel_launches"], lun.shared_launches
        cpls = np.frombuffer(d_cpls.cpu().numpy().tobytes(), dtype=abi.cpl_dtype)
        assert (cpls["status"][:nread] == 0).all() and (cpls["response"][:nread] == abi.S_OK).all()
        w = cpls[nread:]
        good = (w["response"] == abi.S_OK) & (w["status"] == abi.STATUS_GOOD)
        absent = w["response"] == abi.S_BAD_TARGET
        print(f"attach {1e3 * (t1 - t0):.1f} ms after the kick, took {1e3 * (t2 - t1):.1f} ms; launch done after "
              f"{1e3 * (t3 - t0):.1f} ms; target-3 writes: {int(good.sum())} GOOD, {int(absent.sum())} BAD_TARGET")
        assert (good | absent).all(), f"target-3 writes answered other than GOOD or BAD_TARGET: {w[~(good | absent)][:2]}"
        want = init3.copy()
        for k in np.nonzero(good)[0]:
            want[16 * k * 512:(16 * k + 8) * 512] = payload[4096 * k:4096 * (k + 1)]
        for r in (0, 1):
            got = gpu.bdev_read_raw(c.names[3], 0, init3.size, replica=r)
            bad = np.nonzero(got != want)[0]
            assert not len(bad), (f"replica {r}: {len(bad)} bytes differ from the GOOD writes, first at block "
                                  f"{bad[0] // 512} ({int(good.sum())} writes GOOD)")
        assert (launches, shared) == (1, 0), "one launch of the plain kernel on the exclusive side"
        assert in_flight and t2 - t1 > 0.02, "the launch had (nearly) ended before the attach: the prefix is too short"
    finally:
        c.close()


# ---- replicas imported from another process (CUDA IPC) ----------------------------------------------------------

def _store_process(conn, device: int, nb: int, bs: int):
    """The other process of a cross-process mirror (what bench.py --gpus N runs per GPU): two Malloc bdevs on
    `device` whose stores it exports; then it answers "read" with both stores, "init" by rewriting them with the
    initial pattern, and "quit" by deleting them."""
    from oim_b200 import lib
    lib.init([device])
    try:
        names = [lib.construct_malloc_bdev(nb, bs, name=f"ipcstore{r}", device=device) for r in (1, 2)]
        init = traces.pattern_bytes(7, 0, nb * bs)
        for n in names:
            lib.bdev_write_raw(n, 0, init)
        conn.send([lib.bdev_export_store(n) for n in names])
        while True:
            cmd = conn.recv()
            if cmd == "read":
                conn.send([lib.bdev_read_raw(n, 0, nb * bs).tobytes() for n in names])
            elif cmd == "init":
                for n in names:
                    lib.bdev_write_raw(n, 0, init)
                conn.send("ok")
            else:
                break
        for n in names:
            lib.delete_bdev(n)
        conn.send("done")
    finally:
        lib.fini()


def _serve(lib, bname, t, kernel):
    """one launch of `kernel` for trace t on the existing bdev `bname` (target 0 of a controller of its own)"""
    import torch
    cname = f"{bname}.ctl"
    lib.construct_vhost_scsi_controller(cname)
    lib.add_vhost_scsi_lun(cname, 0, bname)
    try:
        host = np.zeros(t.arena_bytes, dtype=np.uint8)
        traces.fill_arena(host, t)
        dev = torch.from_numpy(host).to("cuda:0")
        torch.cuda.synchronize()
        with util.environ(**util.kernel_env(kernel)), lib.Lun(cname, 0, num_queues=1, queue_size=32) as lun:
            cpls = util._run_device_arrays(lun, t.reqs, t.bind(dev.data_ptr()))
            assert lun.iostat()["kernel_launches"] == 1
            assert lun.shared_launches == (kernel in util.SHARED_KERNELS), f"the launch was not the {kernel} kernel"
        return cpls, dev.cpu().numpy()
    finally:
        lib.remove_vhost_scsi_target(cname, 0)
        lib.remove_vhost_controller(cname)


@pytest.mark.timeout(280)
@pytest.mark.parametrize("child_device", [0, 1], ids=["one-gpu", "two-gpus"])
def test_mirror_imported_replicas_match_oracle(gpu, oracles, child_device):
    """construct_mirror_bdev_remote: replica 0 here, replicas 1 and 2 another process's stores opened by CUDA IPC
    handle.  Every replica equals the oracle: read here through the mapping, read by the other process from its own
    store, and by bdev_digest.  Deleting the mirror closes the mapping and leaves the other process's stores intact."""
    import errno
    import multiprocessing as mp

    import torch
    if child_device >= torch.cuda.device_count():
        pytest.skip("needs 2 GPUs")
    nb = 65536
    init = traces.pattern_bytes(7, 0, nb * 512)
    ctx = mp.get_context("spawn")
    conn, child_conn = ctx.Pipe()
    p = ctx.Process(target=_store_process, args=(child_conn, child_device, nb, 512), daemon=True)
    p.start()
    name = None
    try:
        assert conn.poll(120), "the store process sent no handles"
        handles = conn.recv()
        assert len(handles) == 2 and all(len(h) == gpu.IPC_HANDLE_BYTES for h in handles)
        with pytest.raises(gpu.OimGpuError) as e:
            gpu.construct_mirror_bdev_remote(nb, 512, 0, handles * 2, name="ipcmir")       # five replicas
        assert e.value.rc == -errno.EINVAL
        for peers in ([bytes(gpu.IPC_HANDLE_BYTES)], [handles[0], bytes(gpu.IPC_HANDLE_BYTES)]):
            with pytest.raises(gpu.OimGpuError) as e:
                gpu.construct_mirror_bdev_remote(nb, 512, 0, peers, name="ipcmir")          # a handle of zeros
            assert e.value.rc == -errno.EIO
        assert "ipcmir" not in [b["name"] for b in gpu.get_bdevs()], "a failed import left the bdev behind"
        name = gpu.construct_mirror_bdev_remote(nb, 512, 0, handles, name="ipcmir")     # the name is free again
        assert gpu.get_bdevs(name)[0]["replicas"] == 3
        with pytest.raises(gpu.OimGpuError) as e:
            gpu.bdev_export_store(name, 1)                 # an imported replica is not this process's to export
        assert e.value.rc == -errno.EINVAL
        assert len(gpu.bdev_export_store(name, 0)) == gpu.IPC_HANDLE_BYTES
        for kernel in util.MIRROR_KERNELS:
            for tname in ("fuzz523", "sweep"):
                what = f"{kernel}, {tname}"
                t = _mirror_trace(tname, nb)
                want = util.run_oracle(oracles.PortOracle, t, nb)
                for r in range(3):
                    gpu.bdev_write_raw(name, 0, init, replica=r)
                cpls, arena = _serve(gpu, name, t, kernel)
                util.assert_cpls_equal(cpls, want[0], t.reqs, what)
                assert (arena == want[1]).all(), f"{what}: client memory differs at {np.nonzero(arena != want[1])[0][:8]}"
                for r in range(3):
                    bad = np.nonzero(gpu.bdev_read_raw(name, 0, nb * 512, replica=r) != want[2])[0]
                    assert not len(bad), f"{what}: replica {r} read through the mapping differs at {len(bad)} bytes, first {bad[:8]}"
                conn.send("read")
                for r, b in enumerate(conn.recv(), start=1):
                    got = np.frombuffer(b, dtype=np.uint8)
                    bad = np.nonzero(got != want[2])[0]
                    assert not len(bad), f"{what}: replica {r} read by its own process differs at {len(bad)} bytes, first {bad[:8]}"
                d = gpu.digest_host(want[2])
                for r in range(3):
                    assert gpu.bdev_digest(name, r) == d, f"{what}: digest of replica {r}"
        gpu.delete_bdev(name)                              # closes the mapping
        name = None
        conn.send("read")
        for r, b in enumerate(conn.recv(), start=1):
            assert (np.frombuffer(b, dtype=np.uint8) == want[2]).all(), f"store of replica {r} changed when the mirror went"
        conn.send("quit")
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


# ---- the digest the bench's mirror parity rests on --------------------------------------------------------------

def _grid_step_words() -> int:
    """words one grid-stride step of oim_digest_kernel covers: sm_count x 4 CTAs x 256 threads"""
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count * 4 * 256


def test_digest_device_matches_digest_host(gpu):
    """random data: 8 and 16 bytes, one grid-stride step -1 / 0 / +1 words, over 1 GiB; start addresses 8 mod 16"""
    import torch
    step = _grid_step_words()
    rng = np.random.default_rng(88)
    for nwords in (1, 2, 3, step - 1, step, step + 1, 2 * step + 5, (1 << 27) + 3):
        host = rng.integers(0, 1 << 63, size=nwords + 2, dtype=np.int64).view(np.uint8)
        dev = torch.from_numpy(host).to("cuda:0")
        for skew in (0, 8):
            data = host[skew:skew + 8 * nwords]
            assert (dev.data_ptr() + skew) % 16 == skew
            got = gpu.digest_device(0, dev.data_ptr() + skew, 8 * nwords)
            assert got == gpu.digest_host(data), f"{nwords} words at address {skew} mod 16"
        del dev


def test_bdev_digest_windows_and_refusals(gpu):
    import errno
    nb = 4096
    size = nb * 512
    name = gpu.construct_mirror_bdev(nb, 512, [0, 0], name="dgst0")
    try:
        data = np.random.default_rng(89).integers(0, 256, size=size, dtype=np.uint8)
        for r in (0, 1):
            gpu.bdev_write_raw(name, 0, data, replica=r)
        for r in (0, 1):
            assert gpu.bdev_digest(name, r) == gpu.digest_host(data)
            for off, n in ((8, size - 8), (size - 8, 8), (4096 + 8, size - 4096 - 8), (1000, 808)):
                assert gpu.bdev_digest(name, r, off, n) == gpu.digest_host(data[off:off + n]), f"window {off}+{n}"
        for off, n in ((0, 12), (4, 8), (size - 8, 16), (size + 8, 0)):
            with pytest.raises(gpu.OimGpuError) as e:
                gpu.bdev_digest(name, 0, off, n)
            assert e.value.rc == -errno.EINVAL, f"window {off}+{n}"
        with pytest.raises(gpu.OimGpuError) as e:
            gpu.bdev_digest(name, 2)
        assert e.value.rc == -errno.EINVAL
    finally:
        gpu.delete_bdev(name)


def test_digest_changes_with_any_byte_and_with_word_order(gpu):
    """both halves of the digest change when one byte changes (64 random positions) and when two distinct words
    swap places: a digest blind to position or content would let the bench's replica parity pass on wrong data"""
    import torch
    nwords = _grid_step_words() + 77
    rng = np.random.default_rng(90)
    host = rng.integers(0, 1 << 63, size=nwords, dtype=np.int64).view(np.uint8).copy()
    dev = torch.from_numpy(host).to("cuda:0")
    base = gpu.digest_device(0, dev.data_ptr(), host.size)
    assert base == gpu.digest_host(host)
    for pos in rng.choice(host.size, size=64, replace=False):
        pos = int(pos)
        old = int(host[pos])
        host[pos] = old ^ (1 << int(rng.integers(0, 8)))
        dev[pos] = int(host[pos])
        got = gpu.digest_device(0, dev.data_ptr(), host.size)
        assert got == gpu.digest_host(host)
        assert got[0] != base[0] and got[1] != base[1], f"a changed byte at {pos} left a half of the digest as it was"
        host[pos] = old
        dev[pos] = old
    w = host.view(np.uint64)
    for i, j in ((0, 1), (5, nwords - 1), (nwords // 2, nwords // 2 + _grid_step_words() // 3)):
        assert w[i] != w[j]
        sw = w.copy()
        sw[[i, j]] = sw[[j, i]]
        d = torch.from_numpy(sw.view(np.uint8)).to("cuda:0")
        got = gpu.digest_device(0, d.data_ptr(), host.size)
        assert got == gpu.digest_host(sw)
        assert got[0] != base[0] and got[1] != base[1], f"swapping words {i} and {j} left a half of the digest as it was"
