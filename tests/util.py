"""Helpers shared by the parity tests: run one trace through a checker or through the CUDA path."""
from __future__ import annotations

import contextlib
import hashlib
import itertools
import os
import pathlib
import shutil
import tempfile

import numpy as np

from oim_b200 import abi, traces

_seq = itertools.count()


def sha(a: np.ndarray) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def run_oracle(cls, trace: traces.Trace, num_blocks: int, *, block_size: int = 512, store_seed: int | None = 7,
               arena_seed: int = 0x5EED, target: int = 0, removed: bool = False, name: str | None = None,
               scsi_dev_id: int | None = None):
    """-> (cpls, arena, store) after replaying `trace` on a CPU checker (RefOracle / PortOracle).
    name / scsi_dev_id: the identity INQUIRY reports (bdev name, global SCSI device id)."""
    o = cls(num_blocks, block_size, target, name=name, scsi_dev_id=scsi_dev_id)
    try:
        if store_seed is not None:
            o.store[:] = traces.pattern_bytes(store_seed, 0, o.store.size)
        if removed:
            o.set_removed(target, True)
        arena = np.zeros(trace.arena_bytes, dtype=np.uint8)
        traces.fill_arena(arena, trace, arena_seed)
        cpls = o.submit(trace.reqs, trace.bind(arena.ctypes.data))
        return cpls, arena, o.store.copy()
    finally:
        o.close()


@contextlib.contextmanager
def environ(**kv: str | None):
    """set (str) or unset (None) environment variables for the block and restore them afterwards; the library
    reads its launch switches (OIMGPU_NO_SHARED_QUEUES, OIMGPU_NO_VRING_KERNEL, ...) at every kick"""
    old = {k: os.environ.get(k) for k in kv}

    def put(vals):
        for k, v in vals.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    put(kv)
    try:
        yield
    finally:
        put(old)


# The queue-kernel variants a single-queue trace can be pinned to (liboimgpu.so launch_queue_kernel):
#   shared         oim_lun_shared_queue_kernel         the CTAs take the queue a pass at a time
#   exclusive      oim_lun_queue_kernel                one CTA owns the queue (OIMGPU_NO_SHARED_QUEUES=1)
#   mirror         oim_lun_queue_mirror_kernel         two replicas on cuda:0, one CTA per queue
#   mirror-shared  oim_lun_shared_queue_mirror_kernel  two replicas on cuda:0, shared
KERNELS = ("shared", "exclusive", "mirror", "mirror-shared")
SHARED_KERNELS = ("shared", "mirror-shared")
MIRROR_KERNELS = ("mirror", "mirror-shared")
OTHER_KERNELS = KERNELS[1:]     # every variant but the shared kernel, which the unparametrized tests run on


def kernel_env(kernel: str) -> dict:
    """the environment that selects `kernel`'s side of the sharing decision (None = unset)"""
    assert kernel in KERNELS, kernel
    return {"OIMGPU_NO_SHARED_QUEUES": None if kernel in SHARED_KERNELS else "1", "OIMGPU_SHARE_MAX_QUEUES": None}


def kernel_cases(values, mirror_values=None, ids=str, kernels=KERNELS) -> list:
    """pytest parameters (kernel, *value): every value on the plain kernels, `mirror_values` (default: all) on the
    mirror ones.  A tuple value spreads over several arguments.  The shared kernel - the one these traces ran on
    before the variants were pinned - keeps the value's own id (ids(value)); the others prefix it with their name."""
    import pytest
    mirror_values = values if mirror_values is None else mirror_values
    out = []
    for k in kernels:
        for v in (mirror_values if k in MIRROR_KERNELS else values):
            args = v if isinstance(v, tuple) else (v,)
            out.append(pytest.param(k, *args, id=ids(v) if k == "shared" else f"{k}-{ids(v)}"))
    return out


def _ring_fits(trace: traces.Trace) -> int:
    """the smallest ring (power of two, <= 1024 slots) that takes the whole trace in one kick; 0 if none does"""
    n, niov = len(trace.reqs), int(trace.reqs["iovcnt"].astype(np.int64).sum())
    q = 32
    while q < n or max(1024, q * 8) < niov:
        q *= 2
    return q if q <= 1024 else 0


def _run_device_arrays(lun, reqs: np.ndarray, iovs: np.ndarray) -> np.ndarray:
    """one kick of caller-owned request / SG / completion arrays in HBM (oimgpu_submit_device): no ring limit"""
    import torch
    d_reqs = torch.from_numpy(reqs.view(np.uint8).copy()).to("cuda:0")
    d_iovs = torch.from_numpy(np.ascontiguousarray(iovs).view(np.uint8).copy()).to("cuda:0")
    d_cpls = torch.zeros(len(reqs) * abi.cpl_dtype.itemsize, dtype=torch.uint8, device="cuda:0")
    torch.cuda.synchronize()
    lun.submit_device(0, d_reqs.data_ptr(), len(reqs), d_iovs.data_ptr(), d_cpls.data_ptr())
    lun.kick()
    lun.sync()
    return np.frombuffer(d_cpls.cpu().numpy().tobytes(), dtype=abi.cpl_dtype).copy()


def run_cuda(lib, trace: traces.Trace, num_blocks: int, *, block_size: int = 512, store_seed: int | None = 7,
             arena_seed: int = 0x5EED, target: int = 0, mem: str = "device", removed: bool = False,
             queue_size: int = 1024, name: str | None = None, kernel: str | None = None, histogram: bool = False,
             lun_removed: bool = False, replicas: int = 2):
    """Same replay through liboimgpu.so on cuda:0.  mem="device": client buffers in HBM (a torch
    tensor); mem="host": client buffers in pinned, registered host memory.

    kernel (one of KERNELS): serve the whole trace in ONE launch of that queue-kernel variant and fail unless
    the library reports that it did (iostat kernel_launches, Lun.shared_launches).  The ring is sized to hold
    the trace (queue_size is then ignored); a trace longer than a ring goes in as device arrays.  One launch
    also keeps the write-mix switch (a write-hot session stops sharing) from changing the variant mid-trace.
    The mirror variants put `replicas` replicas on cuda:0, write the initial store to each, and check that they all
    end up equal to replica 0.

    histogram: enable the bdev's latency histogram first; stats["histogram_total"] is then its number of tallies.
    lun_removed: the session sees its LUN being torn down (every request aborted)."""
    import torch
    if kernel is not None:
        assert kernel in KERNELS, kernel
        if kernel in SHARED_KERNELS and len(trace.reqs) <= abi.REQS_PER_PASS:
            raise ValueError(f"{len(trace.reqs)} requests are one pass: a launch with one pass is never shared")
    mirror = kernel in MIRROR_KERNELS
    tag = next(_seq)
    bname, cname = name or f"par{tag}", f"parctl{tag}"
    if mirror:
        lib.construct_mirror_bdev(num_blocks, block_size, [0] * replicas, name=bname)
    else:
        lib.construct_malloc_bdev(num_blocks, block_size, name=bname, device=0)
    lib.construct_vhost_scsi_controller(cname)
    lib.add_vhost_scsi_lun(cname, target, bname)
    host_arena = np.zeros(trace.arena_bytes, dtype=np.uint8)
    traces.fill_arena(host_arena, trace, arena_seed)
    ring = _ring_fits(trace) if kernel is not None else queue_size
    try:
        if store_seed is not None:
            init = traces.pattern_bytes(store_seed, 0, num_blocks * block_size)
            for rep in range(replicas if mirror else 1):
                lib.bdev_write_raw(bname, 0, init, replica=rep)
        if mirror:
            assert lib.get_bdevs(bname)[0]["replicas"] == replicas
        if histogram:
            lib.enable_bdev_histogram(bname, True)
        with environ(**(kernel_env(kernel) if kernel is not None else {})), \
                lib.Lun(cname, target, num_queues=1, queue_size=ring or 32) as lun:
            if removed or lun_removed:
                lun.set_removed(removed, lun_removed)
            if mem == "device":
                dev = torch.from_numpy(host_arena).to("cuda:0")
                base = dev.data_ptr()
            else:
                pinned = torch.from_numpy(host_arena.copy()).pin_memory()
                base = pinned.data_ptr()
            torch.cuda.synchronize()
            if ring:
                cpls = lun.run(trace.reqs, trace.bind(base))
            else:
                cpls = _run_device_arrays(lun, trace.reqs, trace.bind(base))
            torch.cuda.synchronize()
            arena = dev.cpu().numpy() if mem == "device" else pinned.numpy().copy()
            stats = lun.iostat()
            if histogram:
                stats["histogram_total"] = int(lib.get_bdev_histogram(bname).sum())
            if kernel is not None:
                assert stats["kernel_launches"] == 1, f"kernel={kernel}: {stats['kernel_launches']} launches, expected 1"
                shared = lun.shared_launches
                assert shared == (kernel in SHARED_KERNELS), f"kernel={kernel}: the launch was {'' if shared else 'not '}shared"
        store = lib.bdev_read_raw(bname, 0, num_blocks * block_size)
        for rep in range(1, replicas if mirror else 1):
            bad = np.nonzero(lib.bdev_read_raw(bname, 0, num_blocks * block_size, replica=rep) != store)[0]
            assert not len(bad), f"kernel={kernel}: replica {rep} of {replicas} differs from replica 0 at {len(bad)} bytes, first {bad[:8]}"
        return cpls, arena, store, stats
    finally:
        lib.remove_vhost_scsi_target(cname, target)
        lib.remove_vhost_controller(cname)
        lib.delete_bdev(bname)


@contextlib.contextmanager
def socket_dir():
    """a fresh directory whose path is short enough for AF_UNIX sockets (sun_path holds 108 bytes): pytest's
    tmp_path lies under $TMPDIR, which may be deep"""
    d = tempfile.mkdtemp(prefix="oim", dir="/tmp")
    try:
        yield pathlib.Path(d)
    finally:
        shutil.rmtree(d, ignore_errors=True)


def assert_cpls_equal(got: np.ndarray, want: np.ndarray, reqs: np.ndarray | None = None, what: str = ""):
    assert len(got) == len(want), f"{what}: {len(got)} completions, expected {len(want)}"
    for f in abi.CPL_PARITY_FIELDS:
        a, b = got[f].reshape(len(got), -1), want[f].reshape(len(want), -1)
        bad = np.nonzero((a != b).any(axis=1))[0]
        if len(bad):
            i = int(bad[0])
            extra = f"\nreq={reqs[i]}" if reqs is not None else ""
            raise AssertionError(f"{what}: completion field '{f}' differs at {len(bad)} requests, first #{i}: "
                                 f"got {got[i]} want {want[i]}{extra}")
