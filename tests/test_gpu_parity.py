"""The parity tests proper: the CUDA path (through the C ABI) against the oracle, bit for bit.

Run on an H100: python -m pytest tests -m gpu.  The reference sources need not exist there; the
checkers are the C restatement (compiled on the machine) and, where build() produced it, the
prebuilt oracle/_ref/liboim_ref.so, plus the golden vectors committed under tests/golden/.
"""
import os

import numpy as np
import pytest

import util
from oim_b200 import abi, traces
from test_oracle import GOLDEN, bdevio_cases, load_golden, run_bdevio  # noqa: F401

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("kernel,mem,path", util.kernel_cases([(m, p) for p in GOLDEN for m in ("device", "host")],
                                                                ids=lambda v: f"{v[0]}-{os.path.basename(v[1])}"))
def test_cuda_matches_reference_golden_vectors(gpu, path, mem, kernel):
    t, z = load_golden(path)
    cpls, arena, store, _ = util.run_cuda(gpu, t, int(z["num_blocks"]), mem=mem, removed=bool(z["removed"]), kernel=kernel)
    util.assert_cpls_equal(cpls, z["cpls"], t.reqs, f"cuda[{kernel}, {mem}]:{t.name}")
    assert util.sha(arena) == str(z["arena_sha"]), "client buffers differ from the reference's"
    assert util.sha(store) == str(z["store_sha"]), "backing store differs from the reference's"


@pytest.mark.parametrize("kernel,seed", util.kernel_cases(range(300, 316), range(300, 304)))
def test_cuda_matches_oracle_on_fuzz(gpu, oracles, kernel, seed):
    """fresh seeded traces: all opcodes, ragged/unaligned/empty SG lists, limits, malformed requests,
    with a hot spot so that RAW/WAW/WAR hazards inside a 32-request pass are common"""
    nb = 32768
    t = traces.fuzz_trace(500, nb, seed=seed, max_io_blocks=[8, 64, 300, 1024][seed % 4],
                          arena_bytes=(8 << 20) if seed % 4 < 3 else (48 << 20))
    want = util.run_oracle(oracles.PortOracle, t, nb)
    got = util.run_cuda(gpu, t, nb, mem="device" if seed % 2 else "host", kernel=kernel)
    util.assert_cpls_equal(got[0], want[0], t.reqs, f"seed {seed}")
    assert (got[1] == want[1]).all(), f"client arena differs at {np.nonzero(got[1] != want[1])[0][:8]}"
    assert (got[2] == want[2]).all(), f"store differs at {np.nonzero(got[2] != want[2])[0][:8]}"
    if oracles.ref_available():         # the compiled reference itself, when it travelled to the box
        ref = util.run_oracle(oracles.RefOracle, t, nb)
        util.assert_cpls_equal(got[0], ref[0], t.reqs, f"seed {seed} vs reference")
        assert (got[1] == ref[1]).all() and (got[2] == ref[2]).all()


@pytest.mark.parametrize("kernel,seed", util.kernel_cases(range(340, 348), range(340, 344)))
def test_cuda_sg_elements_that_continue_each_other(gpu, oracles, kernel, seed):
    """SG lists cut from ONE client buffer at arbitrary bytes (with zero-length elements and gaps in between): the
    kernel moves a run of elements that continue each other in client memory as one segment (lun_kernel.cu
    parse_request / emit_segments), the reference copies element by element (bdev_malloc.c:180-189) - same bytes"""
    nb = 32768
    t = traces.fuzz_trace(400, nb, seed=seed, max_io_blocks=[8, 64, 300, 1024][seed % 4], contiguous=True,
                          arena_bytes=(8 << 20) if seed % 4 < 3 else (48 << 20))
    checker = oracles.RefOracle if oracles.ref_available() and seed % 2 else oracles.PortOracle
    want = util.run_oracle(checker, t, nb)
    got = util.run_cuda(gpu, t, nb, mem="device" if seed % 2 else "host", kernel=kernel)
    util.assert_cpls_equal(got[0], want[0], t.reqs, f"seed {seed}")
    assert (got[1] == want[1]).all(), f"client arena differs at {np.nonzero(got[1] != want[1])[0][:8]}"
    assert (got[2] == want[2]).all(), f"store differs at {np.nonzero(got[2] != want[2])[0][:8]}"


def test_cuda_hazards_same_lba_chain(gpu, oracles):
    """32 requests of one pass all on the same blocks: W,R,W,R,... must serialise exactly (shared kernel)"""
    _hazards_same_lba_chain(gpu, oracles, "shared")


@pytest.mark.parametrize("kernel", util.OTHER_KERNELS)
def test_cuda_hazards_same_lba_chain_on(gpu, oracles, kernel):
    _hazards_same_lba_chain(gpu, oracles, kernel)


def _hazards_same_lba_chain(gpu, oracles, kernel):
    nb = 4096
    b = abi.Batch(0)
    off = 64
    for i in range(64):
        if i % 2 == 0:
            b.write(100, 8, [(off, 4096)])
        else:
            b.read(100 + (i % 3), 4, [(off, 2048)])
        off += 4096
    reqs, iovs = b.arrays()
    t = traces.Trace(reqs, iovs, off + 4096, "chain")
    want = util.run_oracle(oracles.PortOracle, t, nb)
    got = util.run_cuda(gpu, t, nb, kernel=kernel)
    util.assert_cpls_equal(got[0], want[0], t.reqs)
    assert (got[1] == want[1]).all() and (got[2] == want[2]).all()


@pytest.mark.parametrize("kernel,shape", util.kernel_cases(["hot4k", "sub_granule", "mixed_sizes"]))
def test_cuda_hazard_signatures(gpu, oracles, kernel, shape):
    """the signature filter in front of the exact range check (lun_kernel.cu): conflicts in nearly every pass
    (hot4k), requests that share a 4 KiB granule without overlapping and with overlapping (sub_granule),
    and requests from one block to more than the signature's granule limit (mixed_sizes)"""
    nb = 1 << 15
    rng = np.random.default_rng({"hot4k": 1, "sub_granule": 2, "mixed_sizes": 3}[shape])
    b = abi.Batch(0)
    off = 4096
    for i in range(1500):
        if shape == "hot4k":
            lba, n = int(rng.integers(0, 48)) * 8, 8                      # 48 hot slots
        elif shape == "sub_granule":
            lba, n = int(rng.integers(0, 256)), int(rng.integers(1, 5))  # 512 B .. 2 KiB inside a few granules
        else:
            n = int(rng.choice([1, 8, 64, 256, 300, 1024]))
            lba = int(rng.integers(0, 2048 - n))
        if rng.random() < 0.45:
            b.write(lba, n, [(off, n * 512)])
        else:
            b.read(lba, n, [(off, n * 512)])
        off += n * 512
    reqs, iovs = b.arrays()
    t = traces.Trace(reqs, iovs, off + 4096, shape)
    want = util.run_oracle(oracles.PortOracle, t, nb)
    for _ in range(2):
        got = util.run_cuda(gpu, t, nb, kernel=kernel)
        util.assert_cpls_equal(got[0], want[0], t.reqs)
        assert (got[1] == want[1]).all(), f"client memory differs at {np.nonzero(got[1] != want[1])[0][:8]}"
        assert (got[2] == want[2]).all(), f"store differs at {np.nonzero(got[2] != want[2])[0][:8]}"


def test_cuda_hazards_two_passes_apart(gpu, oracles):
    """movers are not in lock-step: while one is still busy with a 4 MiB write of pass p, the others run
    through pass p+1 (unrelated small reads) and reach pass p+2, which reads what pass p writes.  Shared kernel:
    the passes usually land on different CTAs."""
    _hazards_two_passes_apart(gpu, oracles, "shared")


@pytest.mark.parametrize("kernel", util.OTHER_KERNELS)
def test_cuda_hazards_two_passes_apart_on(gpu, oracles, kernel):
    """exclusive / mirror: one CTA runs the three passes back to back (waves, drain between passes)"""
    _hazards_two_passes_apart(gpu, oracles, kernel)


def _hazards_two_passes_apart(gpu, oracles, kernel):
    nb = 1 << 16
    b = abi.Batch(0)
    off = 4096
    big = 8192                                           # blocks = 4 MiB, the largest transfer
    for rep in range(6):
        base = (rep * 3 * 8192) % (nb - 3 * 8192)
        b.write(base, big, [(off, big * 512)], opcode=abi.WRITE_16)          # pass p: one long write ...
        off += big * 512
        for i in range(31):                                                  # ... padded to a full pass
            b.read(nb - 64 + (i % 8), 1, [(off, 512)])
            off += 512
        for i in range(32):                                                  # pass p+1: unrelated
            b.read(nb - 128 + (i % 8), 1, [(off, 512)])
            off += 512
        for i in range(32):                                                  # pass p+2: reads across the big write
            b.read(base + i * 250, 16, [(off, 8192)])
            off += 8192
    reqs, iovs = b.arrays()
    t = traces.Trace(reqs, iovs, off + 4096, "two-apart")
    want = util.run_oracle(oracles.PortOracle, t, nb)
    for _ in range(3):
        got = util.run_cuda(gpu, t, nb, kernel=kernel)
        util.assert_cpls_equal(got[0], want[0], t.reqs)
        assert (got[1] == want[1]).all(), "a read overtook the write two passes ahead of it"
        assert (got[2] == want[2]).all()


def test_cuda_non_pow2_block_size(gpu, oracles):
    _non_pow2_block_size(gpu, oracles, "shared")


@pytest.mark.parametrize("kernel", util.OTHER_KERNELS)
def test_cuda_non_pow2_block_size_on(gpu, oracles, kernel):
    _non_pow2_block_size(gpu, oracles, kernel)


def _non_pow2_block_size(gpu, oracles, kernel):
    nb, bs = 9000, 520
    t = traces.fuzz_trace(300, nb, block_size=bs, seed=77, max_io_blocks=16)
    want = util.run_oracle(oracles.PortOracle, t, nb, block_size=bs)
    got = util.run_cuda(gpu, t, nb, block_size=bs, kernel=kernel)
    util.assert_cpls_equal(got[0], want[0], t.reqs)
    assert (got[1] == want[1]).all() and (got[2] == want[2]).all()


def _element_at(t, off: int) -> str:
    """which SG element of the trace covers arena offset `off` (for failure messages)"""
    a, n = t.iovs["addr"].astype(np.int64), t.iovs["len"].astype(np.int64)
    hit = np.nonzero((a <= off) & (off < a + n))[0]
    if not len(hit):
        return f"arena byte {off}: in no element (a neighbour was overwritten)"
    j = int(hit[0])
    r = int(np.nonzero((t.reqs["iov_start"] <= j) & (j < t.reqs["iov_start"].astype(np.int64) + t.reqs["iovcnt"]))[0][0])
    return f"arena byte {off}: request {r}, element {j} (address mod 16 = {a[j] % 16}, length {n[j]}, byte {off - a[j]})"


@pytest.mark.parametrize("kernel,mem", util.kernel_cases(["device", "host"], ["device"]))
def test_cuda_alignment_sweep(gpu, oracles, kernel, mem):
    """traces.alignment_sweep through every variant: each (client, store) skew at the byte-granular movers' edge
    lengths (staged pieces, realign cases, prefetched units, the compact path of the mirror kernels) and misaligned
    reads behind writes in the same and the next pass.  The whole client arena and the whole store are compared:
    both hold position-keyed pseudo-random bytes, so a misplaced byte or a stray write next to a buffer shows."""
    nb = 65536
    t = traces.alignment_sweep(nb)
    want = util.run_oracle(oracles.PortOracle, t, nb)
    got = util.run_cuda(gpu, t, nb, mem=mem, kernel=kernel)
    util.assert_cpls_equal(got[0], want[0], t.reqs, f"sweep[{kernel}, {mem}]")
    bad = np.nonzero(got[1] != want[1])[0]
    assert not len(bad), f"client memory differs at {len(bad)} bytes; first: {_element_at(t, int(bad[0]))}"
    bad = np.nonzero(got[2] != want[2])[0]
    assert not len(bad), f"store differs at {len(bad)} bytes, first at byte {bad[:8]}"


class DevBuf:
    """client buffer in HBM (torch tensor: plumbing for device memory only)"""

    def __init__(self, n):
        import torch
        self.t = torch.zeros(max(n, 1), dtype=torch.uint8, device="cuda:0")
        self.addr = self.t.data_ptr()

    def set(self, v):
        import torch
        if hasattr(v, "__len__"):
            self.t[:len(v)] = torch.from_numpy(np.asarray(v, dtype=np.uint8)).to("cuda:0")
        else:
            self.t.fill_(int(v))
        torch.cuda.synchronize()

    def get(self):
        import torch
        torch.cuda.synchronize()
        return self.t.cpu().numpy()


def test_cuda_bdevio_suite(gpu):
    """S/test/bdev/bdevio/bdevio.c:388-800 against an HBM-resident 32 MiB Malloc bdev"""
    nb = 65536
    gpu.construct_malloc_bdev(nb, 512, name="bdevio0", device=0)
    gpu.construct_vhost_scsi_controller("bdevio.ctl")
    gpu.add_vhost_scsi_lun("bdevio.ctl", 0, "bdevio0")
    try:
        with gpu.Lun("bdevio.ctl", 0) as lun:
            run_bdevio(lambda r, i: lun.run(r, i), DevBuf, nb)
    finally:
        gpu.remove_vhost_scsi_target("bdevio.ctl", 0)
        gpu.remove_vhost_controller("bdevio.ctl")
        gpu.delete_bdev("bdevio0")


def test_cuda_multi_queue_partitioned_mixed(gpu, oracles):
    """many queues in one launch; queue q confined to LBA window q; 70/30 r/w (bdevperf.c:484-485)"""
    import torch
    nb, nq, per_q = 1 << 18, 24, 96
    t = traces.partitioned_queues(nq, per_q, nb, pattern="randrw", read_pct=70, io_blocks=8)
    host = np.zeros(t.arena_bytes, dtype=np.uint8)
    traces.fill_arena(host, t)
    want_cpls, want_arena, want_store = None, None, None
    o = oracles.PortOracle(nb)
    o.store[:] = traces.pattern_bytes(7, 0, o.store.size)
    oa = host.copy()
    want_cpls = o.submit(t.reqs, t.bind(oa.ctypes.data))
    want_store = o.store.copy()
    o.close()

    gpu.construct_malloc_bdev(nb, 512, name="mq0", device=0)
    gpu.construct_vhost_scsi_controller("mq.ctl")
    gpu.add_vhost_scsi_lun("mq.ctl", 0, "mq0")
    try:
        gpu.bdev_write_raw("mq0", 0, traces.pattern_bytes(7, 0, nb * 512))
        dev = torch.from_numpy(host).to("cuda:0")
        with gpu.Lun("mq.ctl", 0, num_queues=nq, queue_size=128) as lun:
            iovs = t.bind(dev.data_ptr())
            k = len(iovs) // (nq * per_q)
            for q in range(nq):
                r = t.reqs[q * per_q:(q + 1) * per_q].copy()
                r["iov_start"] -= np.uint32(q * per_q * k)
                lun.submit(q, r, iovs[q * per_q * k:(q + 1) * per_q * k])
            assert lun.kick() == nq
            got = np.concatenate([lun.poll(q, per_q) for q in range(nq)])
            stats = lun.iostat()
        torch.cuda.synchronize()
        util.assert_cpls_equal(got, want_cpls, t.reqs)
        assert (dev.cpu().numpy() == oa).all()
        assert (gpu.bdev_read_raw("mq0", 0, nb * 512) == want_store).all()
        assert stats["num_read_ops"] == t.meta["reads"]
        assert stats["num_write_ops"] == nq * per_q - t.meta["reads"]
        assert stats["bytes_read"] == t.meta["reads"] * 4096
        # latency accounting (get_bdevs_iostat *_latency_ticks): summed per request by the mover warps, in ns;
        # a request cannot complete faster than a memory round trip nor slower than the whole launch took
        for kind, n in (("read", t.meta["reads"]), ("write", nq * per_q - t.meta["reads"])):
            per = stats[f"{kind}_latency_ns"] / n
            assert 300 < per < 50e6, f"{kind}: {per} ns per request"
        assert stats["unmap_latency_ns"] == 0
    finally:
        gpu.remove_vhost_scsi_target("mq.ctl", 0)
        gpu.remove_vhost_controller("mq.ctl")
        gpu.delete_bdev("mq0")


@pytest.mark.parametrize("pin", [False, True])
def test_cuda_host_batch_path(gpu, oracles, pin):
    """oimgpu_submit_and_wait with host arrays (the e2e path): metadata staged by the copy engine,
    payload to/from pinned client buffers; pageable and pinned caller arrays"""
    import torch
    nb, nq, per_q = 1 << 16, 12, 64
    t = traces.partitioned_queues(nq, per_q, nb, pattern="randrw", read_pct=60, io_blocks=8, sg="single")
    host = np.zeros(t.arena_bytes, dtype=np.uint8)
    traces.fill_arena(host, t)
    o = oracles.PortOracle(nb)
    o.store[:] = traces.pattern_bytes(7, 0, o.store.size)
    oa = host.copy()
    want = []                   # two rounds of the same trace on the same store: round 2 reads what round 1 wrote
    for _ in range(2):
        c = o.submit(t.reqs, t.bind(oa.ctypes.data))
        want.append((c.copy(), oa.copy(), o.store.copy()))
    o.close()
    gpu.construct_malloc_bdev(nb, 512, name="hb0", device=0)
    gpu.construct_vhost_scsi_controller("hb.ctl")
    gpu.add_vhost_scsi_lun("hb.ctl", 0, "hb0")
    try:
        gpu.bdev_write_raw("hb0", 0, traces.pattern_bytes(7, 0, nb * 512))
        arena = torch.from_numpy(host.copy()).pin_memory()
        keep = []

        def place(a):
            if not pin:
                return np.ascontiguousarray(a)
            buf = torch.empty(a.nbytes, dtype=torch.uint8).pin_memory()
            keep.append(buf)
            out = buf.numpy().view(a.dtype)
            out[:] = a
            return out
        reqs, iovs = place(t.reqs), place(t.bind(arena.data_ptr()))
        cpls = place(np.zeros(len(t.reqs), dtype=abi.cpl_dtype))
        with gpu.Lun("hb.ctl", 0, num_queues=nq, queue_size=64) as lun:
            for rnd in range(2):    # the second round re-uses the library's staging buffers
                cpls[:] = np.zeros(1, dtype=abi.cpl_dtype)
                rc = gpu.load().oimgpu_submit_and_wait(lun.h, nq, per_q, reqs.ctypes.data, iovs.ctypes.data, len(iovs),
                                                       cpls.ctypes.data, abi.MEM_HOST)
                assert rc == 0
                util.assert_cpls_equal(cpls, want[rnd][0], t.reqs, f"round {rnd}")
                assert (arena.numpy() == want[rnd][1]).all(), f"round {rnd}: client buffers"
                assert (gpu.bdev_read_raw("hb0", 0, nb * 512) == want[rnd][2]).all(), f"round {rnd}: store"
        # an SG index outside the table is an invalid request, not a wild read
        bad = t.reqs[:nq].copy()
        bad["iov_start"] = len(iovs) + 5
        c2 = np.zeros(nq, dtype=abi.cpl_dtype)
        with gpu.Lun("hb.ctl", 0, num_queues=nq, queue_size=64) as lun:
            assert gpu.load().oimgpu_submit_and_wait(lun.h, nq, 1, bad.ctypes.data, iovs.ctypes.data, len(iovs),
                                                     c2.ctypes.data, abi.MEM_HOST) == 0
        assert (c2["used_len"] == 0).all() and (c2["resp_valid"] == 0).all()
    finally:
        gpu.remove_vhost_scsi_target("hb.ctl", 0)
        gpu.remove_vhost_controller("hb.ctl")
        gpu.delete_bdev("hb0")


def test_cuda_latency_histogram(gpu):
    """enable_bdev_histogram / get_bdev_histogram (S/lib/bdev/rpc/bdev_rpc.c:607-790): struct spdk_histogram_data's buckets
    (58 ranges x 128, S/include/spdk/histogram_data.h), one tally per completed bdev_io, by the mover warps.  The trace is
    all good READs and WRITEs - one bdev_io each, and each also in the latency sums - so that the tallies and the sums
    cover the same I/Os (test_iostat.py checks the tallies of every other kind against the reference)"""
    import torch
    from oim_b200.lib import OimGpuError
    nb, n = 1 << 16, 4096
    gpu.construct_malloc_bdev(nb, 512, name="hist0", device=0)
    gpu.construct_vhost_scsi_controller("hist.ctl")
    gpu.add_vhost_scsi_lun("hist.ctl", 0, "hist0")
    try:
        assert gpu.get_bdev_histogram("hist0").sum() == 0            # disabled, nothing open: the empty histogram
        t = traces.uniform_trace(n, nb, io_blocks=8, pattern="randrw", read_pct=50, seed=77)
        dev = torch.zeros(t.arena_bytes, dtype=torch.uint8, device="cuda:0")
        with gpu.Lun("hist.ctl", 0, num_queues=4, queue_size=1024) as lun:
            with pytest.raises(OimGpuError) as e:                    # disabled and in use: the reference's channel has no histogram
                gpu.get_bdev_histogram("hist0")
            assert e.value.rc == -14                                 # EFAULT
            gpu.enable_bdev_histogram("hist0", True)
            parts = t.split_queues(4)
            for q, p in enumerate(parts):
                lun.submit(q, p.reqs, p.bind(dev.data_ptr()))
            lun.kick()
            cpls = np.concatenate([lun.poll(q, len(p.reqs)) for q, p in enumerate(parts)])
            assert not cpls["status"].any()
            h = gpu.get_bdev_histogram("hist0")
            assert int(h.sum()) == n, "one tally per completed bdev_io: here one per request"
            # datapoints are nanoseconds: range r (>= 2) holds values in [2^(r+6), 2^(r+7)); a request on an idle GPU takes
            # between a memory round trip and a few milliseconds
            rng = np.nonzero(h.sum(axis=1))[0]
            assert rng.min() >= 3 and rng.max() <= 20, rng           # 512 ns .. 134 ms
            st = lun.iostat()
            lo = sum(int(h[r, i]) * ((128 + i) << (r - 1) if r >= 1 else i) for r in rng for i in range(128))
            total = st["read_latency_ns"] + st["write_latency_ns"] + st["unmap_latency_ns"]
            assert lo <= total <= lo * 1.02 + n * 2, "bucket lower bounds vs the summed latencies"
            gpu.enable_bdev_histogram("hist0", True)                 # enabling again starts over
            assert gpu.get_bdev_histogram("hist0").sum() == 0
            gpu.enable_bdev_histogram("hist0", False)
            with pytest.raises(OimGpuError):
                gpu.get_bdev_histogram("hist0")
        assert gpu.get_bdev_histogram("hist0").sum() == 0
    finally:
        gpu.remove_vhost_scsi_target("hist.ctl", 0)
        gpu.remove_vhost_controller("hist.ctl")
        gpu.delete_bdev("hist0")


def test_cuda_c2_full_size_sample_matches_oracle(gpu, oracles):
    """BASELINE config 2 at its real size: an 8 GiB bdev holding the position-keyed pattern, 254 x 1024 READ(10)s of 4 KiB at
    `8 * (rng mod 2 097 152)` (the C2 trace of SURVEY 8(d)) over 254 queues, replayed through the oracle on an 8 GiB
    store with the same contents; every completion and every payload byte must agree (per-read digests would hide
    nothing a byte compare shows)."""
    import torch
    nb, seed = 16777216, 0xB2000000
    free, _ = torch.cuda.mem_get_info(0)
    if free < 12 << 30:
        pytest.skip("not enough free HBM")
    nq, per_q = 254, 1024
    n = nq * per_q
    t = traces.uniform_trace(n, nb, io_blocks=8, pattern="randread", seed=seed)
    lbas = np.array([int.from_bytes(bytes(x[2:6]), "big") for x in t.reqs["cdb"]], dtype=np.uint64)
    # the oracle's store: 8 GiB of zero pages of which only the blocks the trace reads are filled in (the rest is never
    # looked at; calloc'ed pages stay uncommitted)
    o = (oracles.RefOracle if oracles.ref_available() else oracles.PortOracle)(nb)     # the compiled reference where it travelled
    words = (lbas[:, None] * np.uint64(64) + np.arange(512, dtype=np.uint64)[None, :]).reshape(-1)     # word index = byte offset / 8
    with np.errstate(over="ignore"):
        pat = traces.mix64((np.uint64(seed) ^ words) * traces.GAMMA + traces.GAMMA)
    o.store.view(np.uint64)[words] = pat
    del words
    oa = np.zeros(t.arena_bytes, dtype=np.uint8)
    want_cpls = o.submit(t.reqs, t.bind(oa.ctypes.data))
    o.close()
    assert (oa.view(np.uint64) == pat).all(), "the oracle itself must return the pattern"
    gpu.construct_malloc_bdev(nb, 512, name="c2big", device=0)
    gpu.construct_vhost_scsi_controller("c2big.ctl")
    gpu.add_vhost_scsi_lun("c2big.ctl", 0, "c2big")
    try:
        store_ptr = gpu.get_bdevs("c2big")[0]["device_ptr"]
        with gpu.Lun("c2big.ctl", 0, num_queues=nq, queue_size=32) as lun:
            # fill the whole device with the pattern on the GPU (same function as traces.pattern_words)
            import bench
            bench.device_pattern_fill(lun, store_ptr, nb * 512, seed, torch)
            dev = torch.zeros(t.arena_bytes, dtype=torch.uint8, device="cuda:0")
            d_reqs = torch.from_numpy(t.reqs.view(np.uint8).copy()).cuda()
            d_iovs = torch.from_numpy(t.bind(dev.data_ptr()).view(np.uint8).copy()).cuda()
            d_cpls = torch.zeros(n * 48, dtype=torch.uint8, device="cuda")
            torch.cuda.synchronize()
            lun.submit_batch(nq, per_q, d_reqs.data_ptr(), d_iovs.data_ptr(), len(t.iovs), d_cpls.data_ptr(), abi.MEM_DEVICE)
            lun.sync()
            st = lun.iostat()
        # the many-queue, many-CTA launch books every read exactly once
        assert st["num_read_ops"] == n and st["bytes_read"] == n * 4096, st
        assert st["num_write_ops"] == st["num_unmap_ops"] == st["num_errors"] == 0, st
        got = np.frombuffer(d_cpls.cpu().numpy().tobytes(), dtype=abi.cpl_dtype)
        util.assert_cpls_equal(got, want_cpls, t.reqs)
        assert (dev.cpu().numpy() == oa).all(), "payload differs from the oracle's at the full device size"
    finally:
        gpu.remove_vhost_scsi_target("c2big.ctl", 0)
        gpu.remove_vhost_controller("c2big.ctl")
        gpu.delete_bdev("c2big")


def test_cuda_full_size_properties(gpu):
    """BASELINE config sizes (8 GiB bdev): size-independent properties instead of a CPU replay.
    write(seeded pattern) -> read back == pattern; random 4 KiB reads return the bytes the position-keyed
    pattern predicts; unmap -> zeros; idempotence of a repeated trace."""
    import torch
    nb = 16777216
    free, _ = torch.cuda.mem_get_info(0)
    if free < 14 << 30:
        pytest.skip("not enough free HBM")
    gpu.construct_malloc_bdev(nb, 512, name="big0", device=0)
    gpu.construct_vhost_scsi_controller("big.ctl")
    gpu.add_vhost_scsi_lun("big.ctl", 0, "big0")
    try:
        nq, per_q = 64, 128
        with gpu.Lun("big.ctl", 0, num_queues=nq, queue_size=1024) as lun:
            def run(t, dev):
                iovs = t.bind(dev.data_ptr())
                k = len(iovs) // (nq * per_q)
                for q in range(nq):
                    r = t.reqs[q * per_q:(q + 1) * per_q].copy()
                    r["iov_start"] -= np.uint32(q * per_q * k)
                    lun.submit(q, r, iovs[q * per_q * k:(q + 1) * per_q * k])
                lun.kick()
                return np.concatenate([lun.poll(q, per_q) for q in range(nq)])
            # 1. 128 KiB sequential writes of a position-keyed pattern over 1 GiB in 32-page SG lists
            wt = traces.partitioned_queues(nq, per_q, nb // 8, pattern="seqwrite", io_blocks=256, sg="pages")
            payload = traces.pattern_bytes(0xC3, 0, wt.arena_bytes)
            dev = torch.from_numpy(payload).to("cuda:0")
            c = run(wt, dev)
            assert (c["status"] == 0).all() and (c["resid"] == 0).all()
            # 2. read the same LBAs back into a second arena with a single-element SG list
            rt = traces.partitioned_queues(nq, per_q, nb // 8, pattern="seqread", io_blocks=256, sg="single")
            back = torch.zeros(rt.arena_bytes, dtype=torch.uint8, device="cuda:0")
            c = run(rt, back)
            assert (c["status"] == 0).all()
            torch.cuda.synchronize()
            assert torch.equal(back, dev), "encode->decode round trip"
            # 3. idempotence: replaying the write trace changes nothing
            run(wt, dev)
            back2 = torch.zeros_like(back)
            run(rt, back2)
            torch.cuda.synchronize()
            assert torch.equal(back2, dev)
            # 4. random 4 KiB reads across the whole 8 GiB: untouched area is zero (fresh Malloc bdev)
            rr = traces.partitioned_queues(nq, per_q, nb, pattern="randread", io_blocks=8)
            lbas = np.array([int.from_bytes(bytes(x[2:6]), "big") for x in rr.reqs["cdb"]])
            out = torch.full((rr.arena_bytes,), 0x5A, dtype=torch.uint8, device="cuda:0")
            c = run(rr, out)
            assert (c["status"] == 0).all()
            torch.cuda.synchronize()
            o = out.cpu().numpy().reshape(-1, 4096)
            untouched = lbas >= nb // 8
            assert (o[untouched] == 0).all()
        store_tail = gpu.bdev_read_raw("big0", (nb - 8) * 512, 4096)
        assert (store_tail == 0).all()
    finally:
        gpu.remove_vhost_scsi_target("big.ctl", 0)
        gpu.remove_vhost_controller("big.ctl")
        gpu.delete_bdev("big0")


def test_cuda_control_plane_errors(gpu):
    """error behaviour of the control entry points = the reference RPCs' (SURVEY.md §8(b))"""
    import errno
    with pytest.raises(gpu.OimGpuError) as e:
        gpu.construct_malloc_bdev(0, 512)                 # bdev_malloc.c:384 "Disk must be more than 0 blocks"
    assert e.value.rc == -errno.EINVAL
    name = gpu.construct_malloc_bdev(2048, 512)
    assert name.startswith("Malloc")                      # auto-name Malloc%d (bdev_malloc.c:412)
    info = gpu.get_bdevs(name)[0]
    assert info["product_name"] == "Malloc disk" and info["num_blocks"] == 2048 and not info["claimed"]
    with pytest.raises(gpu.OimGpuError):
        gpu.get_bdevs("no-such-bdev")
    with pytest.raises(gpu.OimGpuError) as e:
        gpu.add_vhost_scsi_lun("nope", 0, name)
    assert e.value.rc == -errno.ENODEV
    gpu.load().oimgpu_set_socket_dir(b"/some/dir", None)
    gpu.construct_vhost_scsi_controller("cp.ctl")
    with pytest.raises(gpu.OimGpuError) as e:
        gpu.construct_vhost_scsi_controller("cp.ctl")
    assert e.value.rc == -errno.EEXIST
    assert gpu.get_vhost_controllers("/some/dir/cp.ctl")[0]["ctrlr"] == "cp.ctl"   # lookups strip the socket dir (vhost.c:611-628)
    with pytest.raises(gpu.OimGpuError) as e:
        gpu.construct_vhost_scsi_controller("cp2.ctl", cpumask="0x2")     # no core left inside the app mask 0x1
    assert e.value.rc == -errno.EINVAL
    assert gpu.add_vhost_scsi_lun("cp.ctl", 3, name) == 3
    with pytest.raises(gpu.OimGpuError) as e:
        gpu.add_vhost_scsi_lun("cp.ctl", 3, name)
    assert e.value.rc == -errno.EEXIST
    with pytest.raises(gpu.OimGpuError) as e:
        gpu.add_vhost_scsi_lun("cp.ctl", 8, name)
    assert e.value.rc == -errno.EINVAL
    with pytest.raises(gpu.OimGpuError) as e:
        gpu.add_vhost_scsi_lun("cp.ctl", 4, "missing-bdev")
    assert e.value.rc == -errno.EINVAL
    c = gpu.get_vhost_controllers("cp.ctl")[0]
    assert c["cpumask"] == "0x1" and c["socket"] == "/some/dir/cp.ctl"
    assert c["backend_specific"]["scsi"][0]["target_name"] == "Target 3"
    assert c["backend_specific"]["scsi"][0]["luns"] == [{"id": 0, "bdev_name": name}]
    assert not gpu.get_bdevs(name)[0]["claimed"]          # SCSI LUNs open without claiming (lun.c:342)
    with pytest.raises(gpu.OimGpuError) as e:
        gpu.remove_vhost_controller("cp.ctl")             # still has a target -> EBUSY (vhost_scsi.c:837-842)
    assert e.value.rc == -errno.EBUSY
    with gpu.Lun("cp.ctl", 3) as lun:
        assert lun.device == 0
        with pytest.raises(gpu.OimGpuError) as e:
            gpu.delete_bdev(name)                         # a data path is open on it
        assert e.value.rc == -errno.EBUSY
    gpu.delete_bdev(name)                                 # hot-removes the target, as spdk_bdev_unregister does
    assert gpu.get_vhost_controllers("cp.ctl")[0]["backend_specific"]["scsi"] == []
    gpu.remove_vhost_controller("cp.ctl")
    gpu.load().oimgpu_set_socket_dir(b"", None)


COPY_LENGTHS = [1, 15, 16, 17, 2031, 2032, 2033, 2047, 2048, 2049, 4095, 4096, 4097, 3 * 4096 + 1234]
BIG = (5 << 20) + 13                                        # several units per warp and an odd tail


def _slots(cases, n_of):
    """one slot per case in one buffer: 64 guard bytes, the case's range at its offset mod 16, 64 guard bytes"""
    base, out = 0, []
    for c in cases:
        out.append(base + 64)
        base += (64 + 16 + n_of(c) + 64 + 63) // 64 * 64
    return out, base


def test_cuda_copy_engine_level(gpu):
    """B2: struct spdk_copy_engine {copy, fill} on device buffers.  copy: every (destination, source) offset mod 16
    (the 16 realign16 skews of move_unit_unaligned, each with every destination head) at the lengths where the mover's
    cases change, plus a few of several MiB; fill: every destination offset.  The cases sit side by side in one
    buffer between guard bytes of a pseudo-random pattern, and the WHOLE buffer is compared with a numpy replay:
    a wrong byte, a byte out of place or a store past either end of a range fails."""
    import torch
    gpu.construct_malloc_bdev(2048, 512, name="ce0", device=0)
    gpu.construct_vhost_scsi_controller("ce.ctl")
    gpu.add_vhost_scsi_lun("ce.ctl", 0, "ce0")
    try:
        with gpu.Lun("ce.ctl", 0) as lun:
            # copy: (dst offset, src offset, length)
            cases = [(do, so, n) for n in COPY_LENGTHS for do in range(16) for so in range(16)]
            cases += [(0, 0, BIG), (1, 0, BIG), (0, 1, BIG), (3, 11, BIG), (15, 15, BIG), (15, 2, BIG)]
            at, size = _slots(cases, lambda c: c[2])
            src_h = traces.pattern_bytes(0xC0, 0, size).copy()
            dst_h = traces.pattern_bytes(0xD5, 0, size).copy()
            src, dst = torch.from_numpy(src_h).to("cuda:0"), torch.from_numpy(dst_h).to("cuda:0")
            torch.cuda.synchronize()
            want = dst_h.copy()
            for (do, so, n), o in zip(cases, at):
                lun.copy(dst.data_ptr() + o + do, src.data_ptr() + o + so, n)
                want[o + do:o + do + n] = src_h[o + so:o + so + n]
            lun.sync()
            got = dst.cpu().numpy()
            bad = np.nonzero(got != want)[0]
            if len(bad):
                k = max(0, int(np.searchsorted(np.asarray(at) - 64, bad[0], side="right")) - 1)
                raise AssertionError(f"copy: {len(bad)} bytes differ; first at byte {int(bad[0]) - at[k]} of the slot of "
                                     f"(dst mod 16, src mod 16, length) = {cases[k]}")
            assert (src.cpu().numpy() == src_h).all(), "copy wrote into its source"
            # fill: (dst offset, length, value)
            cases = [(do, n, (37 * i + 1) & 0xFF) for i, (do, n) in
                     enumerate((do, n) for n in COPY_LENGTHS + [BIG] for do in range(16))]
            at, size = _slots(cases, lambda c: c[1])
            dst_h = traces.pattern_bytes(0xF1, 0, size).copy()
            dst = torch.from_numpy(dst_h).to("cuda:0")
            torch.cuda.synchronize()
            want = dst_h.copy()
            for (do, n, v), o in zip(cases, at):
                lun.fill(dst.data_ptr() + o + do, v, n)
                want[o + do:o + do + n] = v
            lun.sync()
            bad = np.nonzero(dst.cpu().numpy() != want)[0]
            if len(bad):
                k = max(0, int(np.searchsorted(np.asarray(at) - 64, bad[0], side="right")) - 1)
                raise AssertionError(f"fill: {len(bad)} bytes differ; first at byte {int(bad[0]) - at[k]} of the slot of "
                                     f"(dst mod 16, length, value) = {cases[k]}")
    finally:
        gpu.remove_vhost_scsi_target("ce.ctl", 0)
        gpu.remove_vhost_controller("ce.ctl")
        gpu.delete_bdev("ce0")
