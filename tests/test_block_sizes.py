"""Block sizes from 520 bytes to 4 MiB, and transfers up to the 4 MiB limit (MAX_XFER_BYTES), on every path.

The library takes any block size up to 4 MiB (create_bdev_locked), as the reference's Malloc does.  What depends on
it: the transfer limit (max = MAX_XFER_BYTES // block size blocks), requests over one fill of the movers (1 MiB),
READ(6)/WRITE(6) length 0 (256 blocks), the shift or the division in the range check, where a request starts in the
store mod 16, how dense the hazards of a small device with large blocks are, the control payloads that carry the
block size, and which block size a request to a peer target uses.

Devices hold about 256 MiB: 64 blocks of 4 MiB, 516222 blocks of 520 bytes.
CPU: the restatement against the compiled reference.  GPU: the kernel against the restatement (completions, the whole
client arena, the whole store, the counters), on every queue-kernel variant and both virtqueue kernels."""
import functools

import numpy as np
import pytest

import util
from oim_b200 import abi, traces, vring
import test_iostat
from test_iostat import check_counts, checker, diffs, edge_trace, need_ref
from test_multi_target import Controller, run_session
from test_vring import VQ_KERNELS, make_requests, run_kicks_oracle

POW2 = (1024, 2048, 4096, 8192, 16384, 32768, 1 << 20, 4 << 20)
NON_POW2 = (520, 1000, 4097, 4160)
SIZES = NON_POW2 + POW2
DEV_BYTES = 256 << 20
FUZZ_SEEDS = (901, 902)
TRACE_NAMES = ("edges",) + tuple(f"fuzz{s}" for s in FUZZ_SEEDS)
ALL_VARIANTS = (4096, 4097, 1 << 20)     # every queue-kernel variant; the other sizes: shared and exclusive
COUNTER_SIZES = (4096, 4097, 16384)


def blocks(bs: int) -> int:
    return DEV_BYTES // bs


def bs_id(bs: int) -> str:
    return f"{bs >> 20}M" if bs >= 1 << 20 else str(bs)


@functools.lru_cache(maxsize=4)
def make_trace(bs: int, name: str) -> traces.Trace:
    """block_size_trace, or a fuzz trace whose transfers go just past the limit"""
    nb = blocks(bs)
    if name == "edges":
        return traces.block_size_trace(nb, bs)
    return traces.fuzz_trace(120, nb, block_size=bs, seed=int(name[4:]), max_io_blocks=abi.MAX_XFER_BYTES // bs + 2)


@functools.lru_cache(maxsize=1)
def store_pattern() -> np.ndarray:
    """the initial store of every device here (a prefix of it: the pattern is position-keyed)"""
    return traces.pattern_bytes(7, 0, DEV_BYTES)


def replay(cls, t: traces.Trace, bs: int):
    """-> (cpls, arena, store, iostat) after replaying `t` on a checker's device of blocks(bs) blocks"""
    with cls(blocks(bs), bs) as o:
        o.store[:] = store_pattern()[:o.store.size]
        arena = np.zeros(t.arena_bytes, dtype=np.uint8)
        traces.fill_arena(arena, t)
        cpls = o.submit(t.reqs, t.bind(arena.ctypes.data))
        return cpls, arena, o.store.copy(), o.iostat()


@functools.lru_cache(maxsize=1)
def want(oracles, bs: int, name: str):
    """the restatement's replay, once per (block size, trace): the variants' cases of one trace follow each other"""
    return replay(oracles.PortOracle, make_trace(bs, name), bs)


def compare(got, w, t, what):
    util.assert_cpls_equal(got[0], w[0], t.reqs, what)
    bad = np.nonzero(got[1] != w[1])[0]
    assert not len(bad), f"{what}: client arena differs at {len(bad)} bytes, first {bad[:8]}"
    bad = np.nonzero(got[2] != w[2])[0]
    assert not len(bad), f"{what}: store differs at {len(bad)} bytes, first {bad[:8]}"


# ---- CPU: the restatement against the reference ----------------------------------------------------------------

def need_reference(oracles):
    if not oracles.ref_available():
        pytest.skip("oracle/_ref not built here")


@pytest.mark.parametrize("name", TRACE_NAMES)
@pytest.mark.parametrize("bs", SIZES, ids=bs_id)
def test_restatement_matches_reference(oracles, bs, name):
    need_reference(oracles)
    t = make_trace(bs, name)
    ref = replay(oracles.RefOracle, t, bs)
    got = want(oracles, bs, name)
    compare(got, ref, t, f"{bs}:{name}")
    assert got[3] == ref[3], diffs(got[3], ref[3], ref[3])
    if name == "edges":
        assert (ref[0]["status"] == abi.STATUS_GOOD).sum() > len(t.reqs) // 2


@pytest.mark.parametrize("bs", SIZES, ids=bs_id)
def test_primary_restatement_matches_reference(oracles, bs):
    """INQUIRY (VPD B0: COMPARE AND WRITE length, transfer granularity and limit in blocks), MODE SENSE block
    descriptors, READ CAPACITY at each block size"""
    need_reference(oracles)
    nb, name = blocks(bs), f"Malloc{bs}"
    t = traces.primary_trace(300, seed=bs % 9973)
    with oracles.RefOracle(nb, bs, name=name) as probe:
        dev_id = probe.scsi_dev_id
    ref = util.run_oracle(oracles.RefOracle, t, nb, block_size=bs, name=name)
    got = util.run_oracle(oracles.PortOracle, t, nb, block_size=bs, name=name, scsi_dev_id=dev_id)
    compare(got, ref, t, f"primary {bs}")


def counter_traces():
    return [pytest.param(bs, kind, id=f"{bs_id(bs)}-{kind}") for bs in COUNTER_SIZES for kind in ("edge", "edges")]


def counter_trace(bs, kind):
    nb = blocks(bs)
    return (edge_trace(nb, bs) if kind == "edge" else make_trace(bs, "edges")), nb


@pytest.mark.parametrize("bs,kind", counter_traces())
def test_restatement_iostat_matches_reference(oracles, bs, kind):
    need_ref(oracles)
    t, nb = counter_trace(bs, kind)
    wc, w = test_iostat.replay(oracles.RefOracle, t, nb, bs)
    gc, g = test_iostat.replay(oracles.PortOracle, t, nb, bs)
    util.assert_cpls_equal(gc, wc, t.reqs, f"{bs}:{kind}")
    assert g == w, diffs(g, w, w)
    assert w["num_unmap_ops"] and w["bytes_read"] and w["bytes_written"]


# ---- peers with their own block sizes ----------------------------------------------------------------------------

MIXED = {1: (32768, 512), 3: (8192, 4096), 6: (4096, 4097)}     # target -> (blocks, block size)


def mixed_trace(seed: int) -> traces.Trace:
    """one fuzz trace per target at that target's block size, interleaved request by request into one trace"""
    parts = [traces.fuzz_trace(130, nb, block_size=bs, seed=seed + k, target=k, max_io_blocks=abi.MAX_XFER_BYTES // bs // 16)
             for k, (nb, bs) in MIXED.items()]
    reqs, iovs, pay, base, ibase = [], [], [], 0, 0
    for p in parts:
        r = p.reqs.copy()
        r["iov_start"] += np.uint32(ibase)
        v = p.iovs[:int(p.reqs["iov_start"][-1]) + int(p.reqs["iovcnt"][-1])].copy()
        real = (v["addr"] & traces.NULL_ADDR_FLAG) == 0
        v["addr"][real] += np.uint64(base)
        pay += [(off + base, data) for off, data in p.meta["param_payloads"]]
        reqs.append(r)
        iovs.append(v)
        base += p.arena_bytes
        ibase += len(v)
    key = np.concatenate([np.arange(len(r)) * len(reqs) + k for k, r in enumerate(reqs)])
    all_reqs = np.concatenate(reqs)[np.argsort(key)]                  # round robin over the targets
    all_reqs["tag"] = np.arange(len(all_reqs), dtype=np.uint64)
    t = traces.Trace(all_reqs, np.concatenate(iovs), base, f"mixed-{seed}")
    t.meta["param_payloads"] = pay
    return t


def run_mixed_oracle(cls, t, names=None, ids=None):
    names = names or {}
    (nb1, bs1) = MIXED[1]
    with cls(nb1, bs1, 1, name=names.get(1), scsi_dev_id=(ids or {}).get(1)) as o:
        o.store[:] = traces.pattern_bytes(7, 0, o.store.size)
        for k in (3, 6):
            st = o.add_target(k, *MIXED[k], name=names.get(k), scsi_dev_id=(ids or {}).get(k))
            st[:] = traces.pattern_bytes(7 + k, 0, st.size)
        arena = np.zeros(t.arena_bytes, dtype=np.uint8)
        traces.fill_arena(arena, t)
        cpls = o.submit(t.reqs, t.bind(arena.ctypes.data))
        return (cpls, arena, {k: o.stores[k].copy() for k in MIXED}, {k: o.iostat(k) for k in MIXED},
                {k: o.target_scsi_dev_id(k) for k in MIXED})


def test_mixed_block_size_targets_restatement_matches_reference(oracles):
    need_reference(oracles)
    t = mixed_trace(760)
    names = {k: f"mix{k}" for k in MIXED}
    wc, wa, ws, wstats, sid = run_mixed_oracle(oracles.RefOracle, t, names)
    gc, ga, gs, gstats, _ = run_mixed_oracle(oracles.PortOracle, t, names, sid)
    util.assert_cpls_equal(gc, wc, t.reqs, "mixed block sizes")
    assert (ga == wa).all()
    for k in MIXED:
        assert (gs[k] == ws[k]).all(), f"store of target {k}"
    assert gstats == wstats
    good = (wc["status"] == 0) & (wc["resp_valid"] == 1) & (wc["response"] == abi.S_OK)
    assert all((good & (t.reqs["lun"][:, 1] == k)).sum() > 30 for k in MIXED), "every device took I/O"


# ---- GPU: the kernel against the restatement ---------------------------------------------------------------------

def gpu_cases():
    out = []
    for bs in SIZES:
        for name in TRACE_NAMES:
            for k in (util.KERNELS if bs in ALL_VARIANTS else ("shared", "exclusive")):
                out.append(pytest.param(k, bs, name, id=f"{k}-{bs_id(bs)}-{name}"))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("kernel,bs,name", gpu_cases())
def test_cuda_block_sizes(gpu, oracles, kernel, bs, name):
    """one launch of `kernel`: completions, the whole client arena and the whole store equal the restatement's, the
    counters and the histogram tallies its bdev_ios"""
    t = make_trace(bs, name)
    w = want(oracles, bs, name)
    got = util.run_cuda(gpu, t, blocks(bs), block_size=bs, kernel=kernel, histogram=True)
    compare(got, w, t, f"{kernel}:{bs}:{name}")
    check_counts(got[3], w[3], w[0], f"{kernel}:{bs}:{name}")


@pytest.mark.gpu
def test_cuda_block_sizes_host_memory(gpu, oracles):
    """client buffers in pinned host memory"""
    t = make_trace(4096, "edges")
    got = util.run_cuda(gpu, t, blocks(4096), block_size=4096, mem="host", kernel="shared")
    compare(got, want(oracles, 4096, "edges"), t, "host:4096")


@pytest.mark.gpu
@pytest.mark.parametrize("bs", (4096, 4097))
@pytest.mark.parametrize("kernel", list(VQ_KERNELS))
def test_cuda_vring_block_sizes(gpu, oracles, kernel, bs):
    """guest virtqueues on a device of 4096- and 4097-byte blocks: the virtqueue kernel's register realign path and
    the queue kernel's staged path from every store offset"""
    import torch
    seed, ring, nb = 1424, 256, 16384
    rq = make_requests(seed, nb=nb, block_size=bs)
    w, w_store = run_kicks_oracle(oracles.PortOracle, rq, nb, ring, seed, block_size=bs)
    name = f"vqbs{bs}{kernel}"
    gpu.construct_malloc_bdev(nb, bs, name=name, device=0)
    gpu.construct_vhost_scsi_controller(f"{name}.ctl")
    gpu.add_vhost_scsi_lun(f"{name}.ctl", 0, name)
    try:
        gpu.bdev_write_raw(name, 0, traces.pattern_bytes(7, 0, nb * bs))
        with util.environ(**VQ_KERNELS[kernel]), gpu.Lun(f"{name}.ctl", 0, num_queues=1, queue_size=32) as lun:
            pos = kick = 0
            while pos < len(rq):
                img = vring.build_image(rq[pos:], ring_size=ring, seed=seed * 100 + kick)
                dev = torch.from_numpy(img.arena).to("cuda:0")
                base = dev.data_ptr()
                lun.set_mem_table(img.region_table(base))
                lun.vq_attach(0, base + img.desc_off, base + img.avail_off, base + img.used_off, img.ring_size, 0, 0)
                shared = lun.shared_launches
                assert lun.vq_kick() == 1
                lun.sync()
                assert lun.shared_launches - shared == (kernel == "shared"), f"kick {kick} did not take the {kernel} kernel"
                la, lu = lun.vq_detach(0)
                after = dev.cpu().numpy()
                used = img.used_in_order(after, 0, img.used_entries(after)[0])
                assert (la, lu) == w[kick][2][1:], f"kick {kick}: cursors"
                assert sorted((int(i), int(n)) for i, n in used) == w[kick][1], f"kick {kick}: used elements"
                got = img.masked(after)
                assert (got == w[kick][0]).all(), f"kick {kick}: guest memory differs at {np.nonzero(got != w[kick][0])[0][:8]}"
                pos += img.meta["placed"]
                kick += 1
        assert (gpu.bdev_read_raw(name, 0, nb * bs) == w_store).all()
    finally:
        gpu.remove_vhost_scsi_target(f"{name}.ctl", 0)
        gpu.remove_vhost_controller(f"{name}.ctl")
        gpu.delete_bdev(name)


@pytest.mark.gpu
@pytest.mark.parametrize("bs", (4096, 4097, 16384, 4 << 20), ids=bs_id)
def test_cuda_primary_block_sizes(gpu, oracles, bs):
    """the control payloads that carry the block size, byte for byte"""
    nb, name = blocks(bs), f"Malloc{bs}"
    t = traces.primary_trace(400, seed=bs % 9973)
    w = util.run_oracle(oracles.PortOracle, t, nb, block_size=bs, name=name, scsi_dev_id=0)
    got = util.run_cuda(gpu, t, nb, block_size=bs, name=name)
    util.assert_cpls_equal(got[0], w[0], t.reqs, f"primary {bs}")
    assert (got[1] == w[1]).all(), f"response data differs at {np.nonzero(got[1] != w[1])[0][:8]}"
    if oracles.ref_available():
        with oracles.RefOracle(nb, bs, name=name) as probe:
            dev_id = probe.scsi_dev_id
        if dev_id == 0:
            ref = util.run_oracle(oracles.RefOracle, t, nb, block_size=bs, name=name)
            util.assert_cpls_equal(got[0], ref[0], t.reqs, f"primary {bs} vs reference")
            assert (got[1] == ref[1]).all()


@pytest.mark.gpu
@pytest.mark.parametrize("bs,kind", counter_traces())
def test_cuda_iostat_block_sizes(gpu, oracles, bs, kind):
    """the kernel's counters and histogram tallies against the reference's bdev layer"""
    t, nb = counter_trace(bs, kind)
    wc, w = test_iostat.replay(checker(oracles), t, nb, bs)
    gc, _, _, got = util.run_cuda(gpu, t, nb, block_size=bs, kernel="exclusive", histogram=True)
    util.assert_cpls_equal(gc, wc, t.reqs, f"{bs}:{kind}")
    check_counts(got, w, wc, f"{bs}:{kind}")


@pytest.mark.gpu
def test_cuda_mixed_block_size_targets(gpu, oracles):
    """one session reaches targets of 512-, 4096- and 4097-byte blocks: each request uses its own target's block
    size, store and limits"""
    t = mixed_trace(761)
    c = Controller(gpu, sizes=MIXED)
    try:
        wc, wa, ws, wstats, _ = run_mixed_oracle(oracles.PortOracle, t, c.names, c.ids())
        gc, ga, stats = run_session(gpu, c, 1, t)
        util.assert_cpls_equal(gc, wc, t.reqs, "mixed block sizes")
        assert (ga == wa).all(), f"client memory differs at {np.nonzero(ga != wa)[0][:8]}"
        gs = c.stores()
        for k in MIXED:
            assert (gs[k] == ws[k]).all(), f"store of target {k}"
            bad = diffs(stats[k], wstats[k], ("num_read_ops", "bytes_read", "num_write_ops", "bytes_written",
                                               "num_unmap_ops", "bytes_unmapped"))
            assert not bad, f"target {k}: " + "; ".join(bad)
    finally:
        c.close()
