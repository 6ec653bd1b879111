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


def make_requests(seed: int, n: int = 96, nb: int = 32768, contiguous: bool = False, block_size: int = 512):
    """a fuzz trace as guest requests; at other block sizes the largest transfer keeps its size in bytes, so that a
    kick's data still fits the guest image"""
    mx = max(1, [8, 64, 300][seed % 3] * 512 // block_size)
    t = traces.fuzz_trace(n, nb, block_size=block_size, seed=seed, max_io_blocks=mx, arena_bytes=16 << 20,
                          contiguous=contiguous)
    a0 = np.zeros(t.arena_bytes, dtype=np.uint8)
    traces.fill_arena(a0, t)
    return vring.requests_from_trace(t, a0)


def run_kicks_oracle(cls, rq, nb, ring_size, seed, mutate=True, contiguous=False, block_size=512):
    """replay `rq` in as many kicks as the ring needs; -> [(masked image, sorted used entries, cursors)], store"""
    out = []
    with cls(nb, block_size) as o:
        o.store[:] = traces.pattern_bytes(7, 0, o.store.size)
        pos = kick = 0
        while pos < len(rq):
            img = vring.build_image(rq[pos:], ring_size=ring_size, seed=seed * 100 + kick, mutate=mutate, contiguous=contiguous)
            n, la, lu = o.vq_process(img)
            idx, ring = img.used_entries()
            out.append((img.masked(img.arena), sorted((int(i), int(l)) for i, l in ring[:idx]), (n, la, lu)))
            pos += img.meta["placed"]
            kick += 1
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


@pytest.mark.gpu
@pytest.mark.parametrize("kernel,mem,seed", util.kernel_cases(
    [(m, s) for s in list(range(420, 432)) + [1420, 1421, 1422, 1423] for m in ("device", "host")],
    ids=lambda v: f"{v[0]}-{v[1]}", kernels=list(VQ_KERNELS)))
def test_cuda_vring_matches_oracle(gpu, oracles, seed, mem, kernel):
    """seeds >= 1000: every request's data descriptors are cuts of one guest buffer - the kernel moves a run of
    descriptors that continue each other as one segment, the reference copies them one by one.  Every kick is one
    launch of `kernel` (the guest buffers sit at random byte offsets: the byte-granular movers of each)."""
    import torch
    contiguous = seed >= 1000
    nb, rq = 32768, make_requests(seed, contiguous=contiguous)
    ring = [64, 256, 1024][seed % 3]
    checker = oracles.RefOracle if oracles.ref_available() and seed % 2 else oracles.PortOracle
    want, want_store = run_kicks_oracle(checker, rq, nb, ring, seed, contiguous=contiguous)

    name = f"vq{seed}{mem}{kernel}"
    gpu.construct_malloc_bdev(nb, 512, name=name, device=0)
    gpu.construct_vhost_scsi_controller(f"{name}.ctl")
    gpu.add_vhost_scsi_lun(f"{name}.ctl", 0, name)
    try:
        gpu.bdev_write_raw(name, 0, traces.pattern_bytes(7, 0, nb * 512))
        with util.environ(**VQ_KERNELS[kernel]), gpu.Lun(f"{name}.ctl", 0, num_queues=2, queue_size=32) as lun:
            pos = kick = 0
            la = lu = 0
            while pos < len(rq):
                img = vring.build_image(rq[pos:], ring_size=ring, seed=seed * 100 + kick, contiguous=contiguous)
                # each kick is a fresh guest image (cursors restart at 0, as in the oracle replay)
                if mem == "device":
                    dev = torch.from_numpy(img.arena).to("cuda:0")
                else:
                    dev = torch.from_numpy(img.arena.copy()).pin_memory()
                base = dev.data_ptr()
                lun.set_mem_table(img.region_table(base))
                lun.vq_attach(1, base + img.desc_off, base + img.avail_off, base + img.used_off, img.ring_size, 0, 0)
                shared = lun.shared_launches
                assert lun.vq_kick() == 1
                lun.sync()
                assert lun.shared_launches - shared == (kernel == "shared"), f"kick {kick} did not take the {kernel} kernel"
                la, lu = lun.vq_detach(1)
                after = dev.cpu().numpy() if mem == "device" else dev.numpy().copy()
                idx, uring = img.used_entries(after)
                w = want[kick]
                assert (w[2][0], la, lu) == (w[2][0], w[2][1], w[2][2]), f"kick {kick}: cursors {la},{lu} vs {w[2]}"
                assert sorted((int(i), int(l)) for i, l in uring[:idx]) == w[1], f"kick {kick}: used elements"
                got = img.masked(after)
                assert (got == w[0]).all(), f"kick {kick}: guest memory differs at {np.nonzero(got != w[0])[0][:8]}"
                # the kernel publishes used elements in ring order
                assert [int(i) for i in uring[:idx]["id"]] == img.heads[:idx]
                pos += img.meta["placed"]
                kick += 1
            assert lun.iostat()["kernel_launches"] == kick, "one launch per kick"
        assert (gpu.bdev_read_raw(name, 0, nb * 512) == want_store).all()
    finally:
        gpu.remove_vhost_scsi_target(f"{name}.ctl", 0)
        gpu.remove_vhost_controller(f"{name}.ctl")
        gpu.delete_bdev(name)
