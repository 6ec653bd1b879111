"""Config 5: R-way mirrored bdev, write fan-out over NVLink by P2P stores from the mover warps.
No reference implementation exists (S/lib/bdev/raid is RAID0 only); parity = every replica's content
equals the single-bdev oracle's after the same write trace (SURVEY.md 8(c)).  Both replicas on one GPU
([0, 0]) run the same mirror kernels without NVLink, so the fan-out is checked on a single GPU too."""
import numpy as np
import pytest

import util
from oim_b200 import abi, traces

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
