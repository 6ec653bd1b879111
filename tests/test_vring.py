"""Virtqueue level (SURVEY.md 8(a) a19-a22): real virtio split rings in a guest-memory image.
CPU: the C restatement against the compiled reference.  GPU: the kernel's own ring walk against both."""
import numpy as np
import pytest

import util
from oim_b200 import traces, vring

# the kernels that serve a virtqueue-only kick, and the environment that selects each (liboimgpu.so launch_queue_kernel)
VQ_KERNELS = {
    "shared": {"OIMGPU_NO_SHARED_QUEUES": None, "OIMGPU_SHARE_MAX_QUEUES": None, "OIMGPU_NO_VRING_KERNEL": None},
    # oim_lun_vring_kernel: one CTA per queue, the register realign path (move_unit_unaligned)
    "vring": {"OIMGPU_NO_SHARED_QUEUES": "1", "OIMGPU_NO_VRING_KERNEL": None},
    # oim_lun_queue_kernel in virtqueue mode: what a kick that mixes virtqueues and slot rings runs
    "queue": {"OIMGPU_NO_SHARED_QUEUES": "1", "OIMGPU_NO_VRING_KERNEL": "1"},
}
# a kick on a mirrored bdev: the mirror kernels in virtqueue mode (two replicas on cuda:0)
VQ_MIRROR_KERNELS = {
    "mirror": {"OIMGPU_NO_SHARED_QUEUES": "1", "OIMGPU_SHARE_MAX_QUEUES": None},
    "mirror-shared": {"OIMGPU_NO_SHARED_QUEUES": None, "OIMGPU_SHARE_MAX_QUEUES": None},
}
VQ_ALL_KERNELS = {**VQ_KERNELS, **VQ_MIRROR_KERNELS}
VQ_SHARED = ("shared", "mirror-shared")

# ring cursors (last_avail, last_used) a replay starts from, on a ring of R entries.  A guest is almost never at 0:
# the 16-bit indices wrap every few tens of ms at full rate, and a session resumes wherever SET_VRING_BASE or
# used->idx says.
CURSOR_CASES = {
    "zero": lambda R: (0, 0),                           # control
    "ring-end": lambda R: (R - 7, R - 7),               # the first pass straddles the end of both rings
    "wrap-mid": lambda R: (65536 - 45, 65536 - 45),     # the 16-bit index wraps inside the second pass
    "wrap-pass": lambda R: (65536 - 32, 65536 - 32),    # a pass ends exactly on the wrap
    "split": lambda R: (65530, 1000),                   # the cursors differ: catches one used where the other belongs
}
# the GPU replay's seed for each case (the earlier seeds keep cursor 0 and their ids); ring = [64, 256, 1024][seed % 3]
CURSOR_SEEDS = {440 + k: c for k, c in enumerate(CURSOR_CASES)}


def make_requests(seed: int, n: int = 96, nb: int = 32768, contiguous: bool = False, block_size: int = 512):
    """a fuzz trace as guest requests; at other block sizes the largest transfer keeps its size in bytes, so that a
    kick's data still fits the guest image"""
    mx = max(1, [8, 64, 300][seed % 3] * 512 // block_size)
    t = traces.fuzz_trace(n, nb, block_size=block_size, seed=seed, max_io_blocks=mx, arena_bytes=16 << 20,
                          contiguous=contiguous)
    a0 = np.zeros(t.arena_bytes, dtype=np.uint8)
    traces.fill_arena(a0, t)
    return vring.requests_from_trace(t, a0)


def kick_images(rq, ring_size, seed, mutate=True, contiguous=False, start=None):
    """the guest images a replay of `rq` puts in front of the device, one per kick: [(image, (last_avail, last_used))].
    start=None: every kick is a fresh ring at cursor 0.  Else the first kick is built at `start` and each later one at
    the cursors the kicks before it leave (every consumed avail entry yields one used element)."""
    out = []
    la, lu = start or (0, 0)
    pos = 0
    while pos < len(rq):
        img = vring.build_image(rq[pos:], ring_size=ring_size, seed=seed * 100 + len(out), mutate=mutate,
                                contiguous=contiguous, start_avail=la, start_used=lu)
        out.append((img, (la, lu)))
        n = img.meta["placed"]
        pos += n
        if start is not None:
            la, lu = (la + n) & 0xFFFF, (lu + n) & 0xFFFF
    return out


def run_kicks_oracle(cls, rq, nb, ring_size, seed, mutate=True, contiguous=False, block_size=512, start=None):
    """replay `rq` in as many kicks as the ring needs (start: see kick_images);
    -> [(masked image, sorted used elements, (n, last_avail, last_used) after, used elements outside the written
    window untouched)], store"""
    out = []
    with cls(nb, block_size) as o:
        o.store[:] = traces.pattern_bytes(7, 0, o.store.size)
        for img, (la, lu) in kick_images(rq, ring_size, seed, mutate, contiguous, start):
            n, la2, lu2 = o.vq_process(img, la, lu)
            used = img.used_in_order(None, lu, n)
            out.append((img.masked(img.arena), sorted((int(i), int(l)) for i, l in used), (n, la2, lu2),
                        img.used_untouched(img.arena, lu, n)))
        return out, o.store.copy()


@pytest.mark.parametrize("seed", range(400, 412))
def test_vring_restatement_matches_reference(oracles, seed):
    if not oracles.ref_available():
        pytest.skip("oracle/_ref not built here")
    nb, rq = 32768, make_requests(seed)
    ring = [64, 256, 1024][seed % 3]
    want, want_store = run_kicks_oracle(oracles.RefOracle, rq, nb, ring, seed)
    got, got_store = run_kicks_oracle(oracles.PortOracle, rq, nb, ring, seed)
    assert len(got) == len(want)
    for k, (g, w) in enumerate(zip(got, want)):
        assert g[2] == w[2], f"kick {k}: cursors"
        assert g[1] == w[1], f"kick {k}: used elements"
        assert (g[0] == w[0]).all(), f"kick {k}: guest memory differs at {np.nonzero(g[0] != w[0])[0][:8]}"
    assert (got_store == want_store).all()


def test_vring_broken_avail_index(oracles):
    """avail->idx more than one ring ahead: 'the queue is unrecoverably broken' -> nothing is consumed"""
    rq = make_requests(5, n=8)
    for cls in ([oracles.PortOracle] + ([oracles.RefOracle] if oracles.ref_available() else [])):
        img = vring.build_image(rq, ring_size=64, seed=1, mutate=False)
        img.arena[img.avail_off + 2:img.avail_off + 4] = np.frombuffer(np.uint16(200).tobytes(), np.uint8)
        with cls(32768) as o:
            n, la, lu = o.vq_process(img)
        assert (n, la, lu) == (0, 0, 0) and img.used_entries()[0] == 0


@pytest.mark.parametrize("ring", [64, 256, 1024])
@pytest.mark.parametrize("case", list(CURSOR_CASES))
def test_vring_restatement_matches_reference_from_any_cursor(oracles, case, ring):
    """the replay of test_vring_restatement_matches_reference, started from a cursor pair of CURSOR_CASES and carried
    from kick to kick: avail entries, used elements and both indices cross the ring's end and the 16-bit wrap"""
    if not oracles.ref_available():
        pytest.skip("oracle/_ref not built here")
    seed = 440 + list(CURSOR_CASES).index(case)
    nb, rq = 32768, make_requests(seed)
    start = CURSOR_CASES[case](ring)
    want, want_store = run_kicks_oracle(oracles.RefOracle, rq, nb, ring, seed, start=start)
    got, got_store = run_kicks_oracle(oracles.PortOracle, rq, nb, ring, seed, start=start)
    assert len(got) == len(want)
    for k, (g, w) in enumerate(zip(got, want)):
        assert g[2] == w[2], f"kick {k}: cursors {g[2]} vs {w[2]}"
        assert g[1] == w[1], f"kick {k}: used elements"
        assert w[3] and g[3], f"kick {k}: a used element outside the written window was overwritten"
        assert (g[0] == w[0]).all(), f"kick {k}: guest memory differs at {np.nonzero(g[0] != w[0])[0][:8]}"
    assert sum(w[2][0] for w in want) == len(rq)
    assert want[-1][2][1:] == ((start[0] + len(rq)) & 0xFFFF, (start[1] + len(rq)) & 0xFFFF)
    assert (got_store == want_store).all()


@pytest.mark.parametrize("la", [0, 65536 - 3], ids=["zero", "wrap"])
def test_vring_full_and_broken_ring(oracles, la):
    """avail->idx = last_avail + size (every chain one INDIRECT slot) is a full ring, served in full; one entry more is
    'the queue is unrecoverably broken' (vhost.c:193-198): nothing consumed, cursors, guest memory and store as they
    were.  Both checkers, from cursor 0 and across the 16-bit wrap."""
    R, nb = 64, 32768
    rq = make_requests(6, n=R)
    served = []
    for cls in ([oracles.PortOracle] + ([oracles.RefOracle] if oracles.ref_available() else [])):
        for extra in (0, 1):
            img = vring.build_image(rq, ring_size=R, seed=2, all_indirect=True, start_avail=la, start_used=la)
            assert img.meta["placed"] == R and img.avail_idx == (la + R) & 0xFFFF
            if extra:
                img.arena[img.avail_off + 2:img.avail_off + 4] = np.frombuffer(np.uint16((la + R + extra) & 0xFFFF).tobytes(), np.uint8)
            before = img.arena.copy()
            with cls(nb) as o:
                o.store[:] = traces.pattern_bytes(7, 0, o.store.size)
                n, la2, lu2 = o.vq_process(img, la, la)
                store = o.store.copy()
            if extra:
                assert (n, la2, lu2) == (0, la, la), f"{cls.__name__}: a broken ring was served"
                assert (img.arena == before).all(), f"{cls.__name__}: guest memory changed"
                assert (store == traces.pattern_bytes(7, 0, store.size)).all(), f"{cls.__name__}: store changed"
            else:
                assert (n, la2, lu2) == (R, (la + R) & 0xFFFF, (la + R) & 0xFFFF), f"{cls.__name__}: full ring"
                used = img.used_in_order(None, la, R)
                assert img.used_entries()[0] == (la + R) & 0xFFFF
                served.append((sorted((int(i), int(l)) for i, l in used), img.masked(img.arena), store))
    for s in served[1:]:
        assert s[0] == served[0][0], "used elements"
        assert (s[1] == served[0][1]).all(), f"guest memory differs at {np.nonzero(s[1] != served[0][1])[0][:8]}"
        assert (s[2] == served[0][2]).all(), "store"


def _vq_id(v):
    mem, seed = v
    return f"{mem}-{seed}" + (f"-{CURSOR_SEEDS[seed]}" if seed in CURSOR_SEEDS else "")


def _vq_target(gpu, name, nb, kernel):
    """a bdev (two replicas on cuda:0 for the mirror kernels) behind target 0 of controller name.ctl, holding the
    oracle's initial store"""
    if kernel in VQ_MIRROR_KERNELS:
        gpu.construct_mirror_bdev(nb, 512, [0, 0], name=name)
        assert gpu.get_bdevs(name)[0]["replicas"] == 2
    else:
        gpu.construct_malloc_bdev(nb, 512, name=name, device=0)
    gpu.construct_vhost_scsi_controller(f"{name}.ctl")
    gpu.add_vhost_scsi_lun(f"{name}.ctl", 0, name)
    for rep in _replicas(kernel):
        gpu.bdev_write_raw(name, 0, traces.pattern_bytes(7, 0, nb * 512), replica=rep)


def _replicas(kernel):
    return (0, 1) if kernel in VQ_MIRROR_KERNELS else (0,)


def _vq_teardown(gpu, name):
    gpu.remove_vhost_scsi_target(f"{name}.ctl", 0)
    gpu.remove_vhost_controller(f"{name}.ctl")
    gpu.delete_bdev(name)


@pytest.mark.gpu
@pytest.mark.parametrize("kernel,mem,seed", util.kernel_cases(
    [(m, s) for s in list(range(420, 432)) + [1420, 1421, 1422, 1423] + list(CURSOR_SEEDS) for m in ("device", "host")],
    ids=_vq_id, kernels=list(VQ_ALL_KERNELS)))
def test_cuda_vring_matches_oracle(gpu, oracles, seed, mem, kernel):
    """seeds >= 1000: every request's data descriptors are cuts of one guest buffer - the kernel moves a run of
    descriptors that continue each other as one segment, the reference copies them one by one.  Every kick is one
    launch of `kernel` (the guest buffers sit at random byte offsets: the byte-granular movers of each).
    CURSOR_SEEDS start from their cursor case and carry the cursors from kick to kick.  The even ones keep the ring
    attached: the guest rewrites the same memory with the next image, and the kernel's own ring state carries the
    position.  The odd ones re-attach at the cursors vq_detach returned, as a daemon that stops and starts does."""
    import torch
    contiguous = seed >= 1000
    nb, rq = 32768, make_requests(seed, contiguous=contiguous)
    ring = [64, 256, 1024][seed % 3]
    case = CURSOR_SEEDS.get(seed)
    start = CURSOR_CASES[case](ring) if case else None
    keep_attached = case is not None and seed % 2 == 0
    checker = oracles.RefOracle if oracles.ref_available() and seed % 2 else oracles.PortOracle
    want, want_store = run_kicks_oracle(checker, rq, nb, ring, seed, contiguous=contiguous, start=start)
    images = kick_images(rq, ring, seed, contiguous=contiguous, start=start)
    assert len(images) == len(want)

    name = f"vq{seed}{mem}{kernel}"
    _vq_target(gpu, name, nb, kernel)
    try:
        with util.environ(**VQ_ALL_KERNELS[kernel]), gpu.Lun(f"{name}.ctl", 0, num_queues=2, queue_size=32) as lun:
            dev = None
            for kick, (img, (la0, lu0)) in enumerate(images):
                if keep_attached and dev is not None:
                    # the guest's next requests, written over the same memory (same ring, same regions)
                    if mem == "device":
                        dev.copy_(torch.from_numpy(img.arena))
                    else:
                        dev.numpy()[:] = img.arena
                    torch.cuda.synchronize()
                else:
                    # a fresh guest image, attached at the cursors this kick starts from
                    if mem == "device":
                        dev = torch.from_numpy(img.arena).to("cuda:0")
                    else:
                        dev = torch.from_numpy(img.arena.copy()).pin_memory()
                    torch.cuda.synchronize()
                    base = dev.data_ptr()
                    lun.set_mem_table(img.region_table(base))
                    lun.vq_attach(1, base + img.desc_off, base + img.avail_off, base + img.used_off, img.ring_size, la0, lu0)
                shared = lun.shared_launches
                assert lun.vq_kick() == 1
                lun.sync()
                assert lun.shared_launches - shared == (kernel in VQ_SHARED), f"kick {kick} did not take the {kernel} kernel"
                w = want[kick]
                n = w[2][0]
                if not keep_attached or kick == len(images) - 1:
                    la, lu = lun.vq_detach(1)
                    assert (la, lu) == w[2][1:], f"kick {kick}: cursors {la},{lu} vs {w[2]}"
                after = dev.cpu().numpy() if mem == "device" else dev.numpy().copy()
                used = img.used_in_order(after, lu0, n)
                assert sorted((int(i), int(l)) for i, l in used) == w[1], f"kick {kick}: used elements"
                assert img.used_untouched(after, lu0, n), f"kick {kick}: used elements outside [{lu0}, {lu0}+{n}) written"
                got = img.masked(after)
                assert (got == w[0]).all(), f"kick {kick}: guest memory differs at {np.nonzero(got != w[0])[0][:8]}"
                # the kernel publishes used elements in ring order
                assert [int(i) for i in used["id"]] == img.heads[:n]
            assert lun.iostat()["kernel_launches"] == len(images), "one launch per kick"
        for rep in _replicas(kernel):
            assert (gpu.bdev_read_raw(name, 0, nb * 512, replica=rep) == want_store).all(), f"replica {rep}"
    finally:
        _vq_teardown(gpu, name)


IO_COUNTERS = ("num_read_ops", "num_write_ops", "num_unmap_ops", "num_other_ops", "bytes_read", "bytes_written",
               "bytes_unmapped", "num_errors")


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", list(VQ_ALL_KERNELS))
def test_cuda_vring_full_and_broken_ring(gpu, oracles, kernel):
    """test_vring_full_and_broken_ring on every virtqueue kernel, across the 16-bit wrap: a full ring of INDIRECT
    chains is served in one launch of `kernel`; one entry more consumes nothing - guest memory, store, I/O counters
    and the cursors vq_detach returns are what they were"""
    import torch
    R, nb, la = 64, 32768, 65536 - 3
    rq = make_requests(6, n=R)

    def image(extra):
        img = vring.build_image(rq, ring_size=R, seed=2, all_indirect=True, start_avail=la, start_used=la)
        assert img.meta["placed"] == R
        img.arena[img.avail_off + 2:img.avail_off + 4] = np.frombuffer(np.uint16((la + R + extra) & 0xFFFF).tobytes(), np.uint8)
        return img

    want = image(0)
    with oracles.PortOracle(nb) as o:
        o.store[:] = traces.pattern_bytes(7, 0, o.store.size)
        assert o.vq_process(want, la, la) == (R, (la + R) & 0xFFFF, (la + R) & 0xFFFF)
        want_store = o.store.copy()
    name = f"vqfull{kernel}"
    _vq_target(gpu, name, nb, kernel)
    try:
        with util.environ(**VQ_ALL_KERNELS[kernel]), gpu.Lun(f"{name}.ctl", 0, num_queues=1, queue_size=32) as lun:
            for extra in (1, 0):
                img = image(extra)
                dev = torch.from_numpy(img.arena).to("cuda:0")
                torch.cuda.synchronize()
                base = dev.data_ptr()
                lun.set_mem_table(img.region_table(base))
                lun.vq_attach(0, base + img.desc_off, base + img.avail_off, base + img.used_off, R, la, la)
                before = lun.iostat()
                shared = lun.shared_launches
                assert lun.vq_kick() == 1
                lun.sync()
                served = lun.shared_launches - shared
                after_io = lun.iostat()
                cursors = lun.vq_detach(0)
                after = dev.cpu().numpy()
                if extra:
                    assert cursors == (la, la), f"broken ring: cursors {cursors}"
                    assert (after == img.arena).all(), f"broken ring: guest memory changed at {np.nonzero(after != img.arena)[0][:8]}"
                    assert {k: after_io[k] for k in IO_COUNTERS} == {k: before[k] for k in IO_COUNTERS}
                    for rep in _replicas(kernel):
                        assert (gpu.bdev_read_raw(name, 0, nb * 512, replica=rep) == traces.pattern_bytes(7, 0, nb * 512)).all()
                else:
                    assert served == (kernel in VQ_SHARED), f"the full ring did not take the {kernel} kernel"
                    assert cursors == ((la + R) & 0xFFFF,) * 2
                    used = img.used_in_order(after, la, R)
                    assert sorted((int(i), int(l)) for i, l in used) == \
                        sorted((int(i), int(l)) for i, l in want.used_in_order(None, la, R))
                    assert [int(i) for i in used["id"]] == img.heads
                    got = img.masked(after)
                    w = want.masked(want.arena)
                    assert (got == w).all(), f"full ring: guest memory differs at {np.nonzero(got != w)[0][:8]}"
        for rep in _replicas(kernel):
            assert (gpu.bdev_read_raw(name, 0, nb * 512, replica=rep) == want_store).all(), f"replica {rep}"
    finally:
        _vq_teardown(gpu, name)
