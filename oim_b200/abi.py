"""Wire structures of include/oimgpu.h as numpy dtypes + ctypes, and CDB builders.

Shared by the host-side package, the tests and the oracle bindings so that the CUDA path, the
C restatement and the compiled reference are all fed the very same bytes.

Layouts (asserted against the C side by tests/test_abi.py):
  oimgpu_req  64 B — bytes 0..50 are ``struct virtio_scsi_cmd_req``
                      (reference: /usr/include/linux/virtio_scsi.h, used at
                      S/lib/vhost/vhost_scsi.c:513, 638-641)
  oimgpu_iov  16 B — one iovec of ``spdk_vhost_vring_desc_to_iov`` (S/lib/vhost/vhost.c:461-509)
  oimgpu_cpl  48 B — bytes 8..37 are the head of ``struct virtio_scsi_cmd_resp`` as written by
                      ``spdk_vhost_scsi_task_cpl`` (S/lib/vhost/vhost_scsi.c:311-331)
"""
from __future__ import annotations

import numpy as np

CDB_SIZE = 32
SENSE_SIZE = 18
IOVS_MAX = 129
REQS_PER_PASS = 32
MAX_XFER_BYTES = 4 * 1024 * 1024
RESP_SIZE = 108

DIR_NONE, DIR_TO_DEV, DIR_FROM_DEV = 0, 1, 2
S_OK, S_BAD_TARGET = 0, 3
STATUS_GOOD, STATUS_CHECK_CONDITION = 0x00, 0x02
MEM_DEVICE, MEM_HOST = 0, 1

# sense keys / additional sense codes used on the path (S/include/spdk/scsi_spec.h)
SK_NO_SENSE, SK_ILLEGAL_REQUEST, SK_ABORTED_COMMAND = 0x0, 0x5, 0xB
ASC_NONE = 0x00
ASC_INVALID_OPCODE = 0x20
ASC_LBA_OUT_OF_RANGE = 0x21
ASC_INVALID_FIELD_IN_CDB = 0x24
ASC_LUN_NOT_SUPPORTED = 0x25

# SCSI opcodes decoded by spdk_bdev_scsi_process_block (S/lib/scsi/scsi_bdev.c:1681-1802)
READ_6, WRITE_6 = 0x08, 0x0A
READ_10, WRITE_10 = 0x28, 0x2A
READ_12, WRITE_12 = 0xA8, 0xAA
READ_16, WRITE_16 = 0x88, 0x8A
READ_CAPACITY_10 = 0x25
SERVICE_ACTION_IN_16 = 0x9E
SAI_READ_CAPACITY_16 = 0x10
SYNCHRONIZE_CACHE_10, SYNCHRONIZE_CACHE_16 = 0x35, 0x91
UNMAP = 0x42
INQUIRY = 0x12
TEST_UNIT_READY = 0x00

req_dtype = np.dtype([
    ("lun", "u1", (8,)), ("tag", "<u8"), ("task_attr", "u1"), ("prio", "u1"), ("crn", "u1"),
    ("cdb", "u1", (CDB_SIZE,)), ("dir", "u1"), ("iovcnt", "<u2"), ("flags", "<u2"),
    ("iov_start", "<u4"), ("reserved", "<u4"),
])
iov_dtype = np.dtype([("addr", "<u8"), ("len", "<u4"), ("flags", "<u4")])
cpl_dtype = np.dtype([
    ("tag", "<u8"), ("sense_len", "<u4"), ("resid", "<u4"), ("status_qualifier", "<u2"),
    ("status", "u1"), ("response", "u1"), ("sense", "u1", (SENSE_SIZE,)), ("resp_valid", "u1"),
    ("pad", "u1"), ("used_len", "<u4"), ("data_transferred", "<u4"),
])
assert req_dtype.itemsize == 64 and iov_dtype.itemsize == 16 and cpl_dtype.itemsize == 48

# block-I/O channel (oimgpu_bio_chan): one bio and its completion
BIO_READ, BIO_WRITE, BIO_WRITE_ZEROES, BIO_UNMAP = 0, 1, 2, 3
bio_dtype = np.dtype([("offset_blocks", "<u8"), ("num_blocks", "<u8"), ("op", "<u4"), ("iov_start", "<u4"),
                      ("iovcnt", "<u4"), ("flags", "<u4"), ("tag", "<u8")])
bio_cpl_dtype = np.dtype([("tag", "<u8"), ("status", "<i4"), ("pad", "<u4")])
assert bio_dtype.itemsize == 40 and bio_cpl_dtype.itemsize == 16

# completion fields the reference defines (everything but our bookkeeping extras)
CPL_PARITY_FIELDS = ("tag", "sense_len", "resid", "status_qualifier", "status", "response",
                     "sense", "resp_valid", "used_len")


def virtio_lun(target: int, lun_id: int = 0) -> np.ndarray:
    """8-byte virtio-scsi LUN address: [1, target, lun_hi|0x40, lun_lo, 0...]
    (decoded at S/lib/vhost/vhost_scsi.c:361-387; the 0x40 flat-addressing bit is masked off
    by ``& 0x3FFF`` there, as Linux sets it)."""
    b = np.zeros(8, dtype=np.uint8)
    b[0], b[1] = 1, target
    b[2], b[3] = 0x40 | ((lun_id >> 8) & 0x3F), lun_id & 0xFF
    return b


def _be(value: int, nbytes: int) -> list[int]:
    return list(int(value).to_bytes(nbytes, "big"))


def cdb_rw(opcode: int, lba: int, nblocks: int) -> np.ndarray:
    """READ/WRITE 6/10/12/16 CDB, big-endian fields as decoded at scsi_bdev.c:1693-1727."""
    c = np.zeros(CDB_SIZE, dtype=np.uint8)
    c[0] = opcode
    if opcode in (READ_6, WRITE_6):
        c[1:4] = _be(lba & 0x1FFFFF, 3)
        c[4] = nblocks & 0xFF           # 0 means 256
    elif opcode in (READ_10, WRITE_10):
        c[2:6] = _be(lba, 4)
        c[7:9] = _be(nblocks, 2)
    elif opcode in (READ_12, WRITE_12):
        c[2:6] = _be(lba, 4)
        c[6:10] = _be(nblocks, 4)
    elif opcode in (READ_16, WRITE_16):
        c[2:10] = _be(lba, 8)
        c[10:14] = _be(nblocks, 4)
    else:
        raise ValueError(f"not a READ/WRITE opcode: {opcode:#x}")
    return c


def cdb_sync(opcode: int, lba: int, nblocks: int) -> np.ndarray:
    c = np.zeros(CDB_SIZE, dtype=np.uint8)
    c[0] = opcode
    if opcode == SYNCHRONIZE_CACHE_10:
        c[2:6] = _be(lba, 4)
        c[7:9] = _be(nblocks, 2)
    else:
        c[2:10] = _be(lba, 8)
        c[10:14] = _be(nblocks, 4)
    return c


def cdb_read_capacity(sixteen: bool, alloc_len: int = 32) -> np.ndarray:
    c = np.zeros(CDB_SIZE, dtype=np.uint8)
    if sixteen:
        c[0] = SERVICE_ACTION_IN_16
        c[1] = SAI_READ_CAPACITY_16
        c[10:14] = _be(alloc_len, 4)
    else:
        c[0] = READ_CAPACITY_10
    return c


def cdb_unmap(param_len: int) -> np.ndarray:
    c = np.zeros(CDB_SIZE, dtype=np.uint8)
    c[0] = UNMAP
    c[7:9] = _be(param_len, 2)
    return c


def unmap_param_list(descs: list[tuple[int, int]]) -> np.ndarray:
    """UNMAP parameter list (scsi_bdev.c:1545-1578): BE16 data length @0, BE16 block-descriptor
    length @2, then 16-byte descriptors {BE64 lba, BE32 count, 4 reserved} @8."""
    n = len(descs)
    buf = np.zeros(8 + 16 * n, dtype=np.uint8)
    buf[0:2] = _be(6 + 16 * n, 2)
    buf[2:4] = _be(16 * n, 2)
    for i, (lba, cnt) in enumerate(descs):
        o = 8 + 16 * i
        buf[o:o + 8] = _be(lba, 8)
        buf[o + 8:o + 12] = _be(cnt, 4)
    return buf


class Batch:
    """Builder for one submit call: a request array plus its SG table."""

    def __init__(self, target: int = 0):
        self.target = target
        self._reqs: list[tuple] = []
        self._iovs: list[tuple[int, int]] = []

    def add(self, cdb: np.ndarray, direction: int, iovs: list[tuple[int, int]], *,
            lun: np.ndarray | None = None, tag: int | None = None) -> int:
        idx = len(self._reqs)
        start = len(self._iovs)
        self._iovs.extend((int(a), int(l)) for a, l in iovs)
        self._reqs.append((lun if lun is not None else virtio_lun(self.target),
                           idx if tag is None else tag, cdb, direction, len(iovs), start))
        return idx

    def read(self, lba, nblocks, iovs, opcode=READ_10, **kw):
        return self.add(cdb_rw(opcode, lba, nblocks), DIR_FROM_DEV, iovs, **kw)

    def write(self, lba, nblocks, iovs, opcode=WRITE_10, **kw):
        return self.add(cdb_rw(opcode, lba, nblocks), DIR_TO_DEV, iovs, **kw)

    def arrays(self) -> tuple[np.ndarray, np.ndarray]:
        reqs = np.zeros(len(self._reqs), dtype=req_dtype)
        for i, (lun, tag, cdb, direction, cnt, start) in enumerate(self._reqs):
            r = reqs[i]
            r["lun"], r["tag"], r["cdb"] = lun, tag, cdb
            r["dir"], r["iovcnt"], r["iov_start"] = direction, cnt, start
        iovs = np.zeros(max(1, len(self._iovs)), dtype=iov_dtype)
        for i, (a, l) in enumerate(self._iovs):
            iovs[i]["addr"], iovs[i]["len"] = a, l
        return reqs, iovs

    def __len__(self):
        return len(self._reqs)
