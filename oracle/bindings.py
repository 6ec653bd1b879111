"""ctypes bindings of the two CPU checkers (TEST INFRASTRUCTURE — never imported by oim_b200).

  RefOracle   oracle/_ref/liboim_ref.so — the reference's own SPDK C sources compiled from
              /root/reference (see oracle/Makefile, oracle/ref_driver.c)
  PortOracle  oracle/liboim_oracle.so   — plain-C restatement (oracle/oim_oracle.c)

Both expose: create(num_blocks, block_size, target) / store (numpy view of the backing store) /
submit(reqs, iovs) -> cpls, with SG addresses being host pointers.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from oim_b200.abi import cpl_dtype, iov_dtype, req_dtype

_HERE = os.path.dirname(os.path.abspath(__file__))
REF_SO = os.path.join(_HERE, "_ref", "liboim_ref.so")
PORT_SO = os.path.join(_HERE, "liboim_oracle.so")


def build(verbose: bool = False) -> None:
    """(Re)build whichever checker can be built here (the reference needs /root/reference)."""
    out = subprocess.run(["make", "-C", _HERE, "-j8", "all"], capture_output=True, text=True)
    if out.returncode != 0:
        raise RuntimeError("oracle build failed:\n" + out.stdout[-3000:] + out.stderr[-3000:])
    if verbose:
        print(out.stdout[-2000:])


class _Oracle:
    prefix = ""
    path = ""

    def __init__(self, num_blocks: int, block_size: int = 512, target: int = 0, name: str | None = None,
                 scsi_dev_id: int | None = None):
        if not os.path.exists(self.path):
            raise FileNotFoundError(self.path)
        self.lib = C.CDLL(self.path)
        p = self.prefix
        self._create = getattr(self.lib, p + "_create")
        self._create.restype = C.c_void_p
        self._create.argtypes = [C.c_uint64, C.c_uint32, C.c_int]
        self._destroy = getattr(self.lib, p + "_destroy")
        self._destroy.argtypes = [C.c_void_p]
        self._store = getattr(self.lib, p + "_store")
        self._store.restype = C.c_void_p
        self._store.argtypes = [C.c_void_p]
        self._submit = getattr(self.lib, p + "_submit")
        self._submit.restype = C.c_int
        self._submit.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p]
        self._set_removed = getattr(self.lib, p + "_set_removed")
        self._set_removed.argtypes = [C.c_void_p, C.c_int, C.c_int]
        self._busy = getattr(self.lib, p + "_busy_ns")
        self._busy.restype = C.c_uint64
        self._busy.argtypes = [C.c_void_p, C.c_int]
        if name is None:
            self.h = self._create(num_blocks, block_size, target)
        else:
            cn = getattr(self.lib, p + "_create_named")
            cn.restype = C.c_void_p
            cn.argtypes = [C.c_char_p, C.c_uint64, C.c_uint32, C.c_int]
            self.h = cn(name.encode(), num_blocks, block_size, target)
        if not self.h:
            raise RuntimeError(f"{p}_create failed")
        gid = getattr(self.lib, p + "_scsi_dev_id")
        gid.restype = C.c_int
        gid.argtypes = [C.c_void_p, C.c_int]
        if scsi_dev_id is not None and hasattr(self.lib, p + "_set_identity"):
            si = getattr(self.lib, p + "_set_identity")
            si.argtypes = [C.c_void_p, C.c_char_p, C.c_int]
            si(self.h, (name or "Malloc0").encode(), scsi_dev_id)
        self.scsi_dev_id = gid(self.h, target)
        self.num_blocks, self.block_size, self.target = num_blocks, block_size, target
        addr = self._store(self.h)
        buf = (C.c_uint8 * (num_blocks * block_size)).from_address(addr)
        self.store = np.frombuffer(buf, dtype=np.uint8)

    def submit(self, reqs: np.ndarray, iovs: np.ndarray) -> np.ndarray:
        assert reqs.dtype == req_dtype and iovs.dtype == iov_dtype
        reqs = np.ascontiguousarray(reqs)
        iovs = np.ascontiguousarray(iovs)
        cpls = np.zeros(len(reqs), dtype=cpl_dtype)
        rc = self._submit(self.h, reqs.ctypes.data, len(reqs), iovs.ctypes.data, len(iovs),
                          cpls.ctypes.data)
        if rc != 0:
            raise RuntimeError(f"{self.prefix}_submit rc={rc}")
        return cpls

    def vq_process(self, img, last_avail: int = 0, last_used: int = 0) -> tuple[int, int, int]:
        """run the poller over a guest image's split ring (oim_b200.vring.GuestImage, host memory);
        -> (used elements produced, new last_avail_idx, new last_used_idx)"""
        fn = getattr(self.lib, self.prefix + "_vq_process")
        fn.restype = C.c_int
        fn.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint32, C.c_void_p, C.c_uint32,
                       C.POINTER(C.c_uint16), C.POINTER(C.c_uint16)]
        base = img.arena.ctypes.data
        reg = img.region_table(base)
        la, lu = C.c_uint16(last_avail), C.c_uint16(last_used)
        n = fn(self.h, base + img.desc_off, base + img.avail_off, base + img.used_off, img.ring_size,
               reg.ctypes.data, len(img.regions), C.byref(la), C.byref(lu))
        if n < 0:
            raise RuntimeError(f"{self.prefix}_vq_process rc={n}")
        return n, la.value, lu.value

    def add_target(self, target: int, num_blocks: int, block_size: int = 512, name: str | None = None,
                   scsi_dev_id: int | None = None) -> np.ndarray:
        """one more SCSI device (own Malloc bdev) behind the same queues; -> numpy view of its store.
        The reference assigns the SCSI device id itself (lowest free global slot); the restatement is
        told (scsi_dev_id)."""
        fn = getattr(self.lib, self.prefix + "_add_target")
        fn.restype = C.c_int
        if self.prefix == "oimorc":
            fn.argtypes = [C.c_void_p, C.c_char_p, C.c_int, C.c_uint64, C.c_uint32, C.c_int]
            rc = fn(self.h, name.encode() if name else None, scsi_dev_id or 0, num_blocks, block_size, target)
        else:
            fn.argtypes = [C.c_void_p, C.c_char_p, C.c_uint64, C.c_uint32, C.c_int]
            rc = fn(self.h, name.encode() if name else None, num_blocks, block_size, target)
        if rc != 0:
            raise RuntimeError(f"{self.prefix}_add_target rc={rc}")
        ts = getattr(self.lib, self.prefix + "_target_store")
        ts.restype = C.c_void_p
        ts.argtypes = [C.c_void_p, C.c_int]
        buf = (C.c_uint8 * (num_blocks * block_size)).from_address(ts(self.h, target))
        self.stores = getattr(self, "stores", {self.target: self.store})
        self.stores[target] = np.frombuffer(buf, dtype=np.uint8)
        return self.stores[target]

    def target_scsi_dev_id(self, target: int) -> int:
        gid = getattr(self.lib, self.prefix + "_scsi_dev_id")
        gid.restype = C.c_int
        gid.argtypes = [C.c_void_p, C.c_int]
        return gid(self.h, target)

    IOSTAT_FIELDS = ("num_read_ops", "bytes_read", "num_write_ops", "bytes_written", "num_unmap_ops",
                     "bytes_unmapped", "bdev_ios")

    def iostat(self, target: int | None = None) -> dict:
        """the target bdev's get_bdevs_iostat counters (oimgpu_iostat names) and, as bdev_ios, the total of its
        latency histogram: one tally per completed bdev_io of any type and status"""
        fn = getattr(self.lib, self.prefix + "_iostat")
        fn.restype = C.c_int
        fn.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_uint64)]
        out = (C.c_uint64 * 7)()
        rc = fn(self.h, self.target if target is None else target, out)
        if rc != 0:
            raise RuntimeError(f"{self.prefix}_iostat rc={rc}")
        return dict(zip(self.IOSTAT_FIELDS, (int(v) for v in out)))

    def busy_ns(self, reset: bool = True) -> int:
        """ns spent inside the checker's own request processing (0 = not instrumented: time the call)"""
        return int(self._busy(self.h, int(reset)))

    def set_removed(self, target: int, removed: bool = True) -> None:
        self._set_removed(self.h, target, int(removed))

    @classmethod
    def describe(cls) -> str:
        lib = C.CDLL(cls.path)
        fn = getattr(lib, cls.prefix + "_describe")
        fn.restype = C.c_char_p
        return fn().decode()

    def close(self) -> None:
        if self.h:
            self.store = None
            self.stores = {}
            self._destroy(self.h)
            self.h = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()


class RefOracle(_Oracle):
    prefix, path = "oimref", REF_SO


class PortOracle(_Oracle):
    prefix, path = "oimorc", PORT_SO


def ref_available(*, iostat: bool = False) -> bool:
    """oracle/_ref/liboim_ref.so is there.  iostat=True: and it exports the bdev counters (oimref_iostat).  Where the
    reference sources are absent the library cannot be rebuilt, and one built before that export still serves every
    other comparison; the counter comparisons then fall back to the restatement, which is pinned to the reference's
    counters wherever the reference is present."""
    if not os.path.exists(REF_SO):
        return False
    return not iostat or hasattr(C.CDLL(REF_SO), "oimref_iostat")
