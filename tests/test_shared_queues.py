"""Queue sharing (KickHeader::shared, lun_kernel.cuh QShare): with fewer queues than the GPU holds CTAs, the CTAs
take a queue's requests a pass at a time.  The reference runs a queue's requests strictly one after the other
(process_requestq -> spdk_scsi_lun_execute_tasks, S/lib/vhost/vhost_scsi.c:690-741, S/lib/scsi/lun.c:163-211), so
whatever the interleaving across CTAs, every byte must equal the sequential result."""
import numpy as np
import pytest

import util
from oim_b200 import abi, traces

pytestmark = pytest.mark.gpu


def _oracle(oracles, t, nb, seed=7):
    o = oracles.PortOracle(nb)
    o.store[:] = traces.pattern_bytes(seed, 0, o.store.size)
    arena = np.zeros(t.arena_bytes, dtype=np.uint8)
    traces.fill_arena(arena, t)
    cpls = o.submit(t.reqs, t.bind(arena.ctypes.data))
    store = o.store.copy()
    o.close()
    return cpls, arena, store


def _make_bdev(gpu, name, nb, replicas):
    if replicas > 1:
        gpu.construct_mirror_bdev(nb, 512, [0] * replicas, name=name)
        assert gpu.get_bdevs(name)[0]["replicas"] == replicas
    else:
        gpu.construct_malloc_bdev(nb, 512, name=name, device=0)


def _run_batch(gpu, name, t, nb, nq, per_q, seed=7, kernel="shared", replicas=1):
    """one oimgpu_submit_batch launch: queue q <- requests [q*per_q, (q+1)*per_q), everything in HBM.
    kernel="exclusive": with OIMGPU_NO_SHARED_QUEUES=1 (one CTA per queue).  replicas > 1: on a mirror with that
    many replicas on cuda:0; every replica must end up equal to replica 0, whose store is returned"""
    import torch
    _make_bdev(gpu, name, nb, replicas)
    gpu.construct_vhost_scsi_controller(name + ".ctl")
    gpu.add_vhost_scsi_lun(name + ".ctl", 0, name)
    try:
        for r in range(replicas):
            gpu.bdev_write_raw(name, 0, traces.pattern_bytes(seed, 0, nb * 512), replica=r)
        host = np.zeros(t.arena_bytes, dtype=np.uint8)
        traces.fill_arena(host, t)
        dev = torch.from_numpy(host).to("cuda:0")
        d_reqs = torch.from_numpy(t.reqs.view(np.uint8).copy()).cuda()
        d_iovs = torch.from_numpy(t.bind(dev.data_ptr()).view(np.uint8).copy()).cuda()
        d_cpls = torch.zeros(len(t.reqs) * 48, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        with util.environ(**util.kernel_env(kernel)), gpu.Lun(name + ".ctl", 0, num_queues=nq, queue_size=32) as lun:
            lun.submit_batch(nq, per_q, d_reqs.data_ptr(), d_iovs.data_ptr(), len(t.iovs), d_cpls.data_ptr(), abi.MEM_DEVICE)
            lun.sync()
            shared = lun.shared_launches
            stats = lun.iostat()
        assert stats["kernel_launches"] == 1
        cpls = np.frombuffer(d_cpls.cpu().numpy().tobytes(), dtype=abi.cpl_dtype)
        store = gpu.bdev_read_raw(name, 0, nb * 512)
        for r in range(1, replicas):
            bad = np.nonzero(gpu.bdev_read_raw(name, 0, nb * 512, replica=r) != store)[0]
            assert not len(bad), f"replica {r} of {replicas} differs from replica 0 at {len(bad)} bytes, first {bad[:8]}"
        return cpls, dev.cpu().numpy(), store, shared, stats
    finally:
        gpu.remove_vhost_scsi_target(name + ".ctl", 0)
        gpu.remove_vhost_controller(name + ".ctl")
        gpu.delete_bdev(name)


@pytest.mark.parametrize("nq,per_q,read_pct", [(1, 8192, 100), (1, 4096, 60), (3, 4096, 50), (7, 2048, 70), (40, 512, 90)])
def test_shared_queues_match_sequential_result(gpu, oracles, nq, per_q, read_pct):
    """few deep queues, each hammering a SMALL LBA window (every pass collides with its neighbours: RAW, WAW and
    WAR pairs across the CTAs that share the queue)"""
    _shared_queues(gpu, oracles, nq, per_q, read_pct, 1)


@pytest.mark.parametrize("replicas", [2, 3])
@pytest.mark.parametrize("nq,per_q,read_pct", [(3, 4096, 50), (7, 2048, 70)])
def test_shared_queues_on_a_mirror_match_sequential_result(gpu, oracles, nq, per_q, read_pct, replicas):
    """the same on a mirror: the shared mirror kernel's cross-CTA hazards, with every replica equal to the
    sequential result"""
    _shared_queues(gpu, oracles, nq, per_q, read_pct, replicas)


def _shared_queues(gpu, oracles, nq, per_q, read_pct, replicas):
    window = 4096                                   # blocks per queue: 512 distinct 4 KiB slots for thousands of requests
    nb = max(1 << 16, nq * window)
    parts = [traces.uniform_trace(per_q, nb, io_blocks=8, pattern="randrw", read_pct=read_pct, lba_lo=q * window,
                                  lba_span=window, seed=900 + q) for q in range(nq)]
    stride = parts[0].meta["stride"]
    reqs = np.concatenate([p.reqs for p in parts])
    iovs = np.concatenate([p.iovs for p in parts])
    for q in range(nq):
        sl = slice(q * per_q, (q + 1) * per_q)
        reqs["iov_start"][sl] += np.uint32(q * per_q)
        reqs["tag"][sl] += np.uint64(q * per_q)
        iovs["addr"][sl] += np.uint64(q * per_q * stride)
    t = traces.Trace(reqs, iovs, nq * per_q * stride, f"shared-{nq}x{per_q}")
    want = _oracle(oracles, t, nb)
    got = _run_batch(gpu, f"shq{nq}_{read_pct}_{replicas}", t, nb, nq, per_q, replicas=replicas)
    assert got[3] == 1, "the launch did not take the shared-queue path"
    util.assert_cpls_equal(got[0], want[0], t.reqs)
    assert (got[1] == want[1]).all(), "read payloads differ from the sequential result"
    assert (got[2] == want[2]).all(), "store differs from the sequential result"
    reads = int((t.reqs["dir"] == abi.DIR_FROM_DEV).sum())
    assert got[4]["num_read_ops"] == reads and got[4]["num_write_ops"] == nq * per_q - reads


@pytest.mark.parametrize("kernel,seed", util.kernel_cases([31, 32, 33], kernels=("shared", "exclusive")))
def test_shared_queue_fuzz_every_opcode(gpu, oracles, seed, kernel):
    """the adversarial trace (UNMAP, control payloads, malformed requests, ragged SG lists) on ONE queue in one launch:
    shared by the CTAs a pass at a time, and (exclusive) the whole queue on one CTA"""
    nb = 1 << 15
    t = traces.fuzz_trace(3000, nb, seed=seed, max_io_blocks=96, arena_bytes=64 << 20)
    n = len(t.reqs) // 32 * 32
    t = traces.Trace(t.reqs[:n].copy(), t.iovs, t.arena_bytes, t.name, t.meta)
    want = _oracle(oracles, t, nb)
    got = _run_batch(gpu, f"shfz{seed}{kernel}", t, nb, 1, n, kernel=kernel)
    assert got[3] == (kernel == "shared"), f"the launch did not take the {kernel} path"
    util.assert_cpls_equal(got[0], want[0], t.reqs)
    assert (got[1] == want[1]).all() and (got[2] == want[2]).all()


def test_cross_queue_write_after_write_is_one_of_the_legal_outcomes(gpu):
    """Queues are mutually unordered (as for any multi-queue block device; the reference interleaves them in an order
    that depends on poller timing).  What IS guaranteed: every word of the block is from the LAST write of one of
    the queues, never from an earlier write of a queue that wrote the LBA again."""
    _cross_queue_waw(gpu, "waw0", 1)


@pytest.mark.parametrize("replicas", [2, 3])
def test_cross_queue_write_after_write_on_a_mirror(gpu, replicas):
    """The same on a mirror, plus slots that only one queue writes.  Each replica on its own obeys the per-word rule.
    The replicas may differ from each other in the words two queues wrote at the same time (each replica's stores of
    two racing warps land in their own order); a slot that one queue alone wrote is the same on every replica."""
    _cross_queue_waw(gpu, f"wawm{replicas}", replicas, solo=64)


def _cross_queue_waw(gpu, name, replicas, solo=0):
    """every queue writes each of `slots` shared 4 KiB slots `rounds` times in its own random order; slot
    slots + k (k < solo) is written `rounds` times by queue k % nq only.  Returns nothing: asserts on every replica."""
    import torch
    nb, slots, nq = 1 << 14, 256, 4
    rounds = 8                                      # every queue writes every slot `rounds` times, in its own random order
    rng = np.random.default_rng(5)
    per_q = slots * rounds + solo // nq * rounds
    b = abi.Batch(0)
    last = np.zeros((nq, slots + solo), dtype=np.int64)     # request index of queue q's last write to the slot
    off = 0
    for q in range(nq):
        mine = np.arange(slots + q, slots + solo, nq)
        order = np.concatenate([rng.permutation(np.concatenate([np.arange(slots), mine])) for _ in range(rounds)])
        for k, sl in enumerate(order):
            i = q * per_q + k
            b.write(int(sl) * 8, 8, [(off, 4096)])
            last[q, sl] = i
            off += 4096
    reqs, iovs = b.arrays()
    assert len(reqs) == nq * per_q
    t = traces.Trace(reqs, iovs, off, "waw")
    arena = np.zeros(off, dtype=np.uint8)
    arena.view(np.uint64)[:] = np.repeat(np.arange(nq * per_q, dtype=np.uint64), 512) * np.uint64(0x9E3779B97F4A7C15) + np.uint64(1)
    ctl = name + ".ctl"
    _make_bdev(gpu, name, nb, replicas)
    gpu.construct_vhost_scsi_controller(ctl)
    gpu.add_vhost_scsi_lun(ctl, 0, name)
    try:
        dev = torch.from_numpy(arena).to("cuda:0")
        d_reqs = torch.from_numpy(t.reqs.view(np.uint8).copy()).cuda()
        d_iovs = torch.from_numpy(t.bind(dev.data_ptr()).view(np.uint8).copy()).cuda()
        d_cpls = torch.zeros(len(t.reqs) * 48, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        with gpu.Lun(ctl, 0, num_queues=nq, queue_size=32) as lun:
            lun.submit_batch(nq, per_q, d_reqs.data_ptr(), d_iovs.data_ptr(), len(t.iovs), d_cpls.data_ptr(), abi.MEM_DEVICE)
            lun.sync()
        c = np.frombuffer(d_cpls.cpu().numpy().tobytes(), dtype=abi.cpl_dtype)
        assert not c["status"].any()
        with np.errstate(over="ignore"):
            legal = last.astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15) + np.uint64(1)      # [nq, slots + solo]
        stores = [gpu.bdev_read_raw(name, 0, (slots + solo) * 4096, replica=r).view(np.uint64).reshape(slots + solo, 512)
                  for r in range(replicas)]
        for r, store in enumerate(stores):
            shared = store[:slots]
            # Two queues writing one block at the same time are two warps storing 16-byte vectors side by side: the
            # block may end up with vectors of both (the reference, one reactor, would leave one whole request; NVMe
            # promises no more than this beyond its atomic write unit).  What must hold for EVERY word: it is from the
            # LAST write of one of the queues.
            ok = np.zeros(shared.shape, dtype=bool)
            for q in range(nq):
                ok |= shared == legal[q, :slots][:, None]
            assert ok.all(), f"replica {r}: {int((~ok).sum())} words are not from the last write of any queue (an overwritten write survived)"
            for k in range(solo):
                q = k % nq
                assert (store[slots + k] == legal[q, slots + k]).all(), f"replica {r}: slot {slots + k}, written by queue {q} alone"
            torn = int((shared != shared[:, :1]).any(axis=1).sum())
            print(f"cross-queue WAW, replica {r}: {torn} of {slots} blocks hold vectors of more than one queue's last write")
        for r in range(1, replicas):
            differ = stores[r] != stores[0]
            assert not differ[slots:].any(), f"replica {r}: a slot one queue alone wrote differs from replica 0"
            print(f"cross-queue WAW: replica {r} differs from replica 0 in {int(differ.sum())} of {slots * 512} words "
                  f"of the slots the queues share")
    finally:
        gpu.remove_vhost_scsi_target(ctl, 0)
        gpu.remove_vhost_controller(ctl)
        gpu.delete_bdev(name)


def test_sg_lengths_that_wrap_32_bits_are_an_invalid_request(gpu):
    """ADVICE r1: two SG elements of 2 GiB + (2 GiB + 4 KiB) sum to 4 KiB in 32 bits (the reference's `len += desc->len`,
    vhost_scsi.c:573,596).  Every length check would pass on the wrapped value and the movers would then run over
    4 GiB of HBM.  Here the request is invalid: used element of length 0, response untouched, nothing moved."""
    import torch
    nb = 1 << 14
    name = "wrap0"
    gpu.construct_malloc_bdev(nb, 512, name=name, device=0)
    gpu.construct_vhost_scsi_controller("wrap.ctl")
    gpu.add_vhost_scsi_lun("wrap.ctl", 0, name)
    try:
        init = traces.pattern_bytes(3, 0, nb * 512)
        gpu.bdev_write_raw(name, 0, init)
        buf = torch.zeros(1 << 20, dtype=torch.uint8, device="cuda:0")
        for write in (False, True):
            b = abi.Batch(0)
            (b.write if write else b.read)(0, 8, [(0, 0x80000000), (4096, 0x80001000)])
            (b.write if write else b.read)(8, 8, [(8192, 4096)])        # a good one behind it
            reqs, iovs = b.arrays()
            iovs = iovs.copy()
            iovs["addr"] += np.uint64(buf.data_ptr())
            with gpu.Lun("wrap.ctl", 0, num_queues=1, queue_size=32) as lun:
                cpls = lun.run(reqs, iovs)
            assert cpls["used_len"][0] == 0 and cpls["resp_valid"][0] == 0, "wrapped SG sum was not rejected"
            assert cpls["status"][1] == 0 and cpls["resp_valid"][1] == 1
            torch.cuda.synchronize()
        got = gpu.bdev_read_raw(name, 0, nb * 512)
        want = init.copy()
        want[8 * 512:16 * 512] = buf[8192:8192 + 4096].cpu().numpy()        # the good write (it wrote what the good read fetched)
        assert (got == want).all(), "the rejected request touched the store"
    finally:
        gpu.remove_vhost_scsi_target("wrap.ctl", 0)
        gpu.remove_vhost_controller("wrap.ctl")
        gpu.delete_bdev(name)


def test_sharing_follows_the_sessions_read_write_mix(gpu, oracles):
    """Sharing pays for read-dominated sessions only (a write-hot queue is left to its home CTA): the kernels count what
    they served, and the launch shape follows the recent mix - shared, then one CTA per queue once writes dominate,
    then shared again when they stop.  Results equal the oracle's either way."""
    import torch
    nb, nq, per_q = 1 << 16, 4, 2048
    name = "mix0"
    gpu.construct_malloc_bdev(nb, 512, name=name, device=0)
    gpu.construct_vhost_scsi_controller("mix.ctl")
    gpu.add_vhost_scsi_lun("mix.ctl", 0, name)
    o = oracles.PortOracle(nb)
    try:
        init = traces.pattern_bytes(7, 0, nb * 512)
        gpu.bdev_write_raw(name, 0, init)
        o.store[:] = init
        shapes = []
        with gpu.Lun("mix.ctl", 0, num_queues=nq, queue_size=32) as lun:
            for step, pattern in enumerate(["randrw", "randrw", "randread", "randread", "randread"]):
                t = traces.partitioned_queues(nq, per_q, nb, pattern=pattern, read_pct=50, io_blocks=8, seed=40 + step)
                host = np.zeros(t.arena_bytes, dtype=np.uint8)
                traces.fill_arena(host, t, 0x5EED + step)
                oa = host.copy()
                want = o.submit(t.reqs, t.bind(oa.ctypes.data))
                dev = torch.from_numpy(host).to("cuda:0")
                d_reqs = torch.from_numpy(t.reqs.view(np.uint8).copy()).cuda()
                d_iovs = torch.from_numpy(t.bind(dev.data_ptr()).view(np.uint8).copy()).cuda()
                d_cpls = torch.zeros(len(t.reqs) * 48, dtype=torch.uint8, device="cuda")
                torch.cuda.synchronize()
                before = lun.shared_launches
                lun.submit_batch(nq, per_q, d_reqs.data_ptr(), d_iovs.data_ptr(), len(t.iovs), d_cpls.data_ptr(), abi.MEM_DEVICE)
                lun.sync()
                shapes.append(lun.shared_launches - before)
                got = np.frombuffer(d_cpls.cpu().numpy().tobytes(), dtype=abi.cpl_dtype)
                util.assert_cpls_equal(got, want, t.reqs, f"step {step}")
                assert (dev.cpu().numpy() == oa).all(), f"step {step}: payload"
        assert (gpu.bdev_read_raw(name, 0, nb * 512) == o.store).all()
        # launch 0: no history -> shared; 1: writes seen -> one CTA per queue; 2: still write-hot (its own reads are only
        # known afterwards); 3, 4: reads dominate the recent window -> shared again
        assert shapes == [1, 0, 0, 1, 1], shapes
    finally:
        o.close()
        gpu.remove_vhost_scsi_target("mix.ctl", 0)
        gpu.remove_vhost_controller("mix.ctl")
        gpu.delete_bdev(name)
