"""ctypes binding of liboimgpu.so (the C ABI in include/oimgpu.h) + thin Python objects.

This is plumbing: every call goes straight to the C ABI.  If the shared library is missing or no
CUDA device is usable the import/`init()` raises — there is no CPU implementation to fall back to.

The Python classes mirror the reference's Go shims in pkg/spdk/spdk.go so tests read like the
reference's (`construct_malloc_bdev`, `add_vhost_scsi_lun`, ...).
"""
from __future__ import annotations

import ctypes as C
import errno
import os

import numpy as np

from . import abi

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("OIM_LIB_PATH") or os.path.join(_HERE, "liboimgpu.so")   # override: tuning builds only


class OimGpuError(OSError):
    def __init__(self, rc: int, what: str):
        super().__init__(-rc, f"{what}: {errno.errorcode.get(-rc, rc)} ({os.strerror(-rc) if rc < 0 else rc})")
        self.rc = rc


class BdevInfo(C.Structure):
    _fields_ = [("name", C.c_char * 64), ("product_name", C.c_char * 32), ("uuid", C.c_char * 40),
                ("num_blocks", C.c_uint64), ("block_size", C.c_uint32), ("claimed", C.c_int32),
                ("device", C.c_int32), ("replicas", C.c_uint32), ("device_ptr", C.c_uint64)]


class TargetInfo(C.Structure):
    _fields_ = [("scsi_dev_num", C.c_int32), ("id", C.c_int32), ("target_name", C.c_char * 16),
                ("lun_id", C.c_int32), ("bdev_name", C.c_char * 64)]


class CtrlrInfo(C.Structure):
    _fields_ = [("ctrlr", C.c_char * 64), ("cpumask", C.c_char * 20), ("delay_base_us", C.c_uint32),
                ("iops_threshold", C.c_uint32), ("socket", C.c_char * 192), ("ntargets", C.c_uint32),
                ("targets", TargetInfo * 8)]


class IoStat(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("num_read_ops", "num_write_ops", "num_unmap_ops", "num_other_ops",
                                          "bytes_read", "bytes_written", "bytes_unmapped", "num_errors",
                                          "kernel_launches", "read_latency_ns", "write_latency_ns", "unmap_latency_ns")]


# every symbol include/oimgpu.h declares: (name, restype, argtypes)
_VP, _U32, _U64, _I = C.c_void_p, C.c_uint32, C.c_uint64, C.c_int
SYMBOLS = [
    ("oimgpu_abi_version", _I, []),
    ("oimgpu_init", _I, [C.POINTER(C.c_int), _I]),
    ("oimgpu_init_control_only", _I, []),
    ("oimgpu_fini", None, []),
    ("oimgpu_device_count", _I, []),
    ("oimgpu_set_socket_dir", _I, [C.c_char_p, C.c_char_p]),
    ("oimgpu_version_string", C.c_char_p, []),
    ("oimgpu_bdev_create_malloc", _I, [C.c_char_p, C.c_char_p, _U64, _U32, _I, C.c_char_p, C.c_size_t]),
    ("oimgpu_bdev_create_rbd", _I, [C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, _U32, _U64, _I, C.c_char_p, C.c_size_t]),
    ("oimgpu_bdev_create_mirror", _I, [C.c_char_p, _U64, _U32, C.POINTER(C.c_int), _I, C.c_char_p, C.c_size_t]),
    ("oimgpu_bdev_export_store", _I, [C.c_char_p, _I, _VP]),
    ("oimgpu_bdev_create_mirror_remote", _I, [C.c_char_p, _U64, _U32, _I, _VP, _I, C.c_char_p, C.c_size_t]),
    ("oimgpu_bdev_create_mirror_uuid", _I, [C.c_char_p, C.c_char_p, _U64, _U32, C.POINTER(C.c_int), _I, C.c_char_p, C.c_size_t]),
    ("oimgpu_bdev_create_mirror_remote_uuid", _I, [C.c_char_p, C.c_char_p, _U64, _U32, _I, _VP, _I, C.c_char_p, C.c_size_t]),
    ("oimgpu_bdev_replica_info", _I, [C.c_char_p, _I, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    ("oimgpu_bdev_mirror_replace_remote", _I, [C.c_char_p, _I, _VP]),
    ("oimgpu_bdev_digest", _I, [C.c_char_p, _I, _U64, _U64, C.POINTER(C.c_uint64)]),
    ("oimgpu_digest_device", _I, [_I, _VP, _U64, C.POINTER(C.c_uint64)]),
    ("oimgpu_bdev_mirror_check", _I, [C.c_char_p, _U64, _U64, _I, _VP, _U32, _VP]),
    ("oimgpu_bdev_image_save", _I, [C.c_char_p, C.c_char_p, _VP]),
    ("oimgpu_bdev_image_load", _I, [C.c_char_p, C.c_char_p, _VP]),
    ("oimgpu_bdev_image_track", _I, [C.c_char_p, _I]),
    ("oimgpu_bdev_image_save_delta", _I, [C.c_char_p, C.c_char_p, _VP]),
    ("oimgpu_bdev_image_apply_delta", _I, [C.c_char_p, C.c_char_p, _VP]),
    ("oimgpu_bdev_delete", _I, [C.c_char_p]),
    ("oimgpu_bdev_get", _I, [C.c_char_p, C.POINTER(BdevInfo)]),
    ("oimgpu_bdev_list", _I, [C.POINTER(BdevInfo), _I]),
    ("oimgpu_read_strided", _I, [_I, _VP, _VP, C.c_size_t, C.c_size_t, C.c_size_t]),
    ("oimgpu_write_strided", _I, [_I, _VP, _VP, C.c_size_t, C.c_size_t, C.c_size_t]),
    ("oimgpu_bdev_read_raw", _I, [C.c_char_p, _I, _U64, _VP, _U64]),
    ("oimgpu_bdev_write_raw", _I, [C.c_char_p, _I, _U64, _VP, _U64]),
    ("oimgpu_vhost_scsi_ctrlr_create", _I, [C.c_char_p, C.c_char_p]),
    ("oimgpu_vhost_scsi_add_lun", _I, [C.c_char_p, _I, C.c_char_p]),
    ("oimgpu_vhost_scsi_remove_target", _I, [C.c_char_p, _I]),
    ("oimgpu_vhost_ctrlr_remove", _I, [C.c_char_p]),
    ("oimgpu_vhost_ctrlr_set_coalescing", _I, [C.c_char_p, _U32, _U32]),
    ("oimgpu_config_json", C.c_long, [C.c_char_p, C.c_char_p, C.c_size_t]),
    ("oimgpu_vhost_ctrlr_get", _I, [C.c_char_p, C.POINTER(CtrlrInfo)]),
    ("oimgpu_vhost_ctrlr_list", _I, [C.POINTER(CtrlrInfo), _I]),
    ("oimgpu_lun_open", _I, [C.c_char_p, _I, _U32, _U32, C.POINTER(_VP)]),
    ("oimgpu_lun_open_on", _I, [C.c_char_p, _I, _U32, _U32, C.POINTER(_VP)]),
    ("oimgpu_device_ordinal", _I, [_I]),
    ("oimgpu_lun_close", _I, [_VP]),
    ("oimgpu_lun_device", _I, [_VP]),
    ("oimgpu_lun_shared_launches", C.c_longlong, [_VP]),
    ("oimgpu_mem_register", _I, [_VP, C.c_size_t]),
    ("oimgpu_mem_unregister", _I, [_VP]),
    ("oimgpu_mem_device_addr", _I, [_VP, C.POINTER(C.c_uint64)]),
    ("oimgpu_submit", _I, [_VP, _U32, _VP, _U32, _VP, _U32, _I]),
    ("oimgpu_submit_device", _I, [_VP, _U32, _VP, _U32, _VP, _VP]),
    ("oimgpu_kick", _I, [_VP]),
    ("oimgpu_poll", _I, [_VP, _U32, _VP, _U32, _I]),
    ("oimgpu_lun_sync", _I, [_VP]),
    ("oimgpu_submit_batch", _I, [_VP, _U32, _U32, _VP, _VP, _U32, _VP, _I]),
    ("oimgpu_submit_and_wait", _I, [_VP, _U32, _U32, _VP, _VP, _U32, _VP, _I]),
    ("oimgpu_bdev_iostat", _I, [C.c_char_p, C.POINTER(IoStat)]),
    ("oimgpu_bdev_histogram_enable", _I, [C.c_char_p, _I]),
    ("oimgpu_bdev_histogram_get", _I, [C.c_char_p, C.POINTER(C.c_uint64)]),
    ("oimgpu_nbd_serve", _I, [C.c_char_p, _I]),
    ("oimgpu_lun_iostat", _I, [_VP, C.POINTER(IoStat)]),
    ("oimgpu_lun_target_iostat", _I, [_VP, _I, C.POINTER(IoStat)]),
    ("oimgpu_lun_stream", _VP, [_VP]),
    ("oimgpu_lun_set_removed", _I, [_VP, _I, _I]),
    ("oimgpu_lun_start_poller", _I, [_VP, _U32, _U32]),
    ("oimgpu_lun_stop_poller", _I, [_VP]),
    ("oimgpu_lun_poller_running", _I, [_VP]),
    ("oimgpu_lun_set_mem_table", _I, [_VP, _VP, _U32]),
    ("oimgpu_vq_attach", _I, [_VP, _U32, _VP, _VP, _VP, _U32, C.c_uint16, C.c_uint16]),
    ("oimgpu_vq_detach", _I, [_VP, _U32, C.POINTER(C.c_uint16), C.POINTER(C.c_uint16)]),
    ("oimgpu_vq_kick", _I, [_VP]),
    ("oimgpu_timer_create", _I, [C.POINTER(_VP), C.POINTER(_VP)]),
    ("oimgpu_timer_record", _I, [_VP, _VP]),
    ("oimgpu_timer_elapsed_ms", _I, [_VP, _VP, C.POINTER(C.c_float)]),
    ("oimgpu_timer_destroy", None, [_VP, _VP]),
    ("oimgpu_copy_chan_open", _I, [_I, C.POINTER(_VP)]),
    ("oimgpu_copy_chan_close", _I, [_VP]),
    ("oimgpu_copy_chan_copy", _I, [_VP, _VP, _VP, _U64, _VP]),
    ("oimgpu_copy_chan_fill", _I, [_VP, _VP, C.c_uint8, _U64, _VP]),
    ("oimgpu_copy_chan_poll", _I, [_VP, C.POINTER(_VP), _I]),
    ("oimgpu_copy_chan_launches", C.c_ulonglong, [_VP]),
    ("oimgpu_mem_ensure", _I, [_VP, C.c_size_t]),
    ("oimgpu_bio_chan_open", _I, [C.c_char_p, C.POINTER(_VP)]),
    ("oimgpu_bio_chan_submit", _I, [_VP, _VP, _U32, _VP, _U32]),
    ("oimgpu_bio_chan_poll", _I, [_VP, _VP, _I]),
    ("oimgpu_bio_chan_close", _I, [_VP]),
    ("oimgpu_bio_chan_launches", C.c_ulonglong, [_VP]),
    ("oimgpu_copy_submit", _I, [_VP, _VP, _VP, _U64]),
    ("oimgpu_fill_submit", _I, [_VP, _VP, C.c_uint8, _U64]),
]

_lib = None


def load() -> C.CDLL:
    """dlopen liboimgpu.so and type every entry point.  No compute happens here."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise FileNotFoundError(f"{LIB_PATH} not built: run `python -m oim_b200.build` "
                                    "(the CUDA data path has no CPU fallback)")
        lib = C.CDLL(LIB_PATH)
        for name, res, args in SYMBOLS:
            fn = getattr(lib, name)
            fn.restype, fn.argtypes = res, args
        _lib = lib
    return _lib


def _chk(rc: int, what: str) -> int:
    if rc < 0:
        raise OimGpuError(rc, what)
    return rc


def _b(s):
    return None if s is None else s.encode()


def init(devices: list[int] | None = None) -> None:
    lib = load()
    if devices:
        arr = (C.c_int * len(devices))(*devices)
        _chk(lib.oimgpu_init(arr, len(devices)), "oimgpu_init")
    else:
        _chk(lib.oimgpu_init(None, 0), "oimgpu_init")


def fini() -> None:
    load().oimgpu_fini()


# ---- the twelve SPDK RPCs OIM issues, under the names pkg/spdk/spdk.go gives them ---------------

def construct_malloc_bdev(num_blocks: int, block_size: int = 512, name: str | None = None,
                          uuid: str | None = None, device: int = -1) -> str:
    """pkg/spdk/spdk.go:100-111 ConstructMallocBDev -> construct_malloc_bdev."""
    out = C.create_string_buffer(64)
    _chk(load().oimgpu_bdev_create_malloc(_b(name), _b(uuid), num_blocks, block_size, device, out, 64),
         "construct_malloc_bdev")
    return out.value.decode()


def construct_rbd_bdev(pool_name: str, rbd_name: str, block_size: int, size_bytes: int,
                       name: str | None = None, user_id: str | None = None, device: int = -1) -> str:
    """pkg/spdk/spdk.go:113-119 ConstructRBDBDev -> construct_rbd_bdev (HBM-backed)."""
    out = C.create_string_buffer(64)
    _chk(load().oimgpu_bdev_create_rbd(_b(name), _b(pool_name), _b(rbd_name), _b(user_id), block_size,
                                       size_bytes, device, out, 64), "construct_rbd_bdev")
    return out.value.decode()


def construct_mirror_bdev(num_blocks: int, block_size: int, devices: list[int], name: str | None = None) -> str:
    out = C.create_string_buffer(64)
    arr = (C.c_int * len(devices))(*devices)
    _chk(load().oimgpu_bdev_create_mirror(_b(name), num_blocks, block_size, arr, len(devices), out, 64),
         "construct_mirror_bdev")
    return out.value.decode()


IPC_HANDLE_BYTES = 64


def bdev_export_store(name: str, replica: int = 0) -> bytes:
    """CUDA IPC handle of a replica's store: what another process needs to mirror onto this GPU"""
    out = C.create_string_buffer(IPC_HANDLE_BYTES)
    _chk(load().oimgpu_bdev_export_store(_b(name), replica, out), "bdev_export_store")
    return out.raw


def construct_mirror_bdev_remote(num_blocks: int, block_size: int, device: int, peer_handles: list[bytes],
                                 name: str | None = None) -> str:
    """mirror whose replicas 1.. are stores of OTHER processes (one process per GPU), imported by IPC handle"""
    out = C.create_string_buffer(64)
    blob = C.create_string_buffer(b"".join(peer_handles), IPC_HANDLE_BYTES * len(peer_handles))
    _chk(load().oimgpu_bdev_create_mirror_remote(_b(name), num_blocks, block_size, device, blob, len(peer_handles), out, 64),
         "construct_mirror_bdev_remote")
    return out.value.decode()


def mirror_replace_remote(name: str, replica: int, handle: bytes) -> None:
    """move replica `replica` (>= 1) of a mirror built from remote replicas to the store behind `handle`, copying
    replica 0 into it with the sessions held (include/oimgpu.h oimgpu_bdev_mirror_replace_remote)"""
    if len(handle) != IPC_HANDLE_BYTES:
        raise ValueError(f"an IPC handle is {IPC_HANDLE_BYTES} bytes, not {len(handle)}")
    blob = C.create_string_buffer(bytes(handle), IPC_HANDLE_BYTES)
    _chk(load().oimgpu_bdev_mirror_replace_remote(_b(name), replica, blob), "mirror_replace_remote")


def bdev_digest(name: str, replica: int = 0, offset: int = 0, nbytes: int | None = None) -> tuple[int, int]:
    """position-keyed digest of a store range, computed on the GPU (include/oimgpu.h oimgpu_bdev_digest)"""
    if nbytes is None:
        b = get_bdevs(name)[0]
        nbytes = b["num_blocks"] * b["block_size"] - offset
    out = (C.c_uint64 * 2)()
    _chk(load().oimgpu_bdev_digest(_b(name), replica, offset, nbytes, out), "bdev_digest")
    return int(out[0]), int(out[1])


def digest_device(device: int, ptr: int, nbytes: int) -> tuple[int, int]:
    out = (C.c_uint64 * 2)()
    _chk(load().oimgpu_digest_device(device, ptr, nbytes, out), "digest_device")
    return int(out[0]), int(out[1])


def digest_host(data: np.ndarray) -> tuple[int, int]:
    """the same digest over a host array (numpy, wrapping arithmetic): the checker's side"""
    w = np.ascontiguousarray(data).view(np.uint8).view(np.uint64)
    with np.errstate(over="ignore"):
        i = np.arange(len(w), dtype=np.uint64)
        a = int((w * (np.uint64(2) * i + np.uint64(1))).sum(dtype=np.uint64))
        z = w ^ i
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        z = z ^ (z >> np.uint64(31))
        b = int(z.sum(dtype=np.uint64))
    return a, b


def mirror_check(name: str, offset_blocks: int = 0, num_blocks: int | None = None, repair: bool = False,
                 max_ranges: int = 64) -> dict:
    """compare every replica of a mirrored bdev with replica 0 over [offset_blocks, offset_blocks + num_blocks) (default:
    to the end); repair=True copies replica 0 over each block that differs (include/oimgpu.h oimgpu_bdev_mirror_check).
    ranges: the first max_ranges runs of differing blocks, (offset_blocks, num_blocks) in LBA order."""
    if num_blocks is None:
        num_blocks = max(get_bdevs(name)[0]["num_blocks"] - offset_blocks, 0)
    out = np.zeros(1, dtype=abi.mirror_check_dtype)
    ranges = np.zeros(2 * max(max_ranges, 1), dtype=np.uint64)
    _chk(load().oimgpu_bdev_mirror_check(_b(name), offset_blocks, num_blocks, int(repair), ranges.ctypes.data, max_ranges,
                                         out.ctypes.data), "mirror_check")
    o = out[0]
    n = int(o["nranges"])
    return {"blocks_checked": int(o["blocks_checked"]), "mismatched_blocks": int(o["mismatched_blocks"]),
            "repaired_blocks": int(o["repaired_blocks"]),
            "ranges": [(int(ranges[2 * i]), int(ranges[2 * i + 1])) for i in range(n)], "truncated": bool(o["truncated"])}


def _image_call(fn, what: str, name: str, path) -> dict:
    out = np.zeros(1, dtype=abi.image_info_dtype)
    _chk(fn(_b(name), os.fsencode(path), out.ctypes.data), what)
    o = out[0]
    return {"num_blocks": int(o["num_blocks"]), "block_size": int(o["block_size"]), "granule_bytes": int(o["granule_bytes"]),
            "nextents": int(o["nextents"]), "data_bytes": int(o["data_bytes"]), "file_bytes": int(o["file_bytes"]),
            "uuid": bytes(o["uuid"]).split(b"\0", 1)[0].decode()}


def bdev_image_save(name: str, path) -> dict:
    """write bdev `name`'s bytes to the new sparse image file `path` with its sessions held; the image's geometry,
    extent count, sizes and source uuid (include/oimgpu.h oimgpu_bdev_image_save)"""
    return _image_call(load().oimgpu_bdev_image_save, "bdev_image_save", name, path)


def bdev_image_load(name: str, path) -> dict:
    """fill every replica of the unused bdev `name` from the image file `path` (include/oimgpu.h oimgpu_bdev_image_load)"""
    return _image_call(load().oimgpu_bdev_image_load, "bdev_image_load", name, path)


def bdev_image_track(name: str, enable: bool = True) -> None:
    """keep (or stop keeping) the fingerprint tables that let bdev `name`'s next save_delta write only the granules that
    changed since its last save or load (include/oimgpu.h oimgpu_bdev_image_track)"""
    _chk(load().oimgpu_bdev_image_track(_b(name), int(enable)), "bdev_image_track")


def _delta_call(fn, what: str, name: str, path) -> dict:
    out = np.zeros(1, dtype=abi.image_delta_info_dtype)
    _chk(fn(_b(name), os.fsencode(path), out.ctypes.data), what)
    o = out[0]
    return {"num_blocks": int(o["num_blocks"]), "block_size": int(o["block_size"]), "granule_bytes": int(o["granule_bytes"]),
            "nextents": int(o["nextents"]), "data_bytes": int(o["data_bytes"]), "zero_bytes": int(o["zero_bytes"]),
            "file_bytes": int(o["file_bytes"]), "parent_digest": tuple(int(x) for x in o["parent_digest"]),
            "digest": tuple(int(x) for x in o["digest"]), "uuid": bytes(o["uuid"]).split(b"\0", 1)[0].decode()}


def bdev_image_save_delta(name: str, path) -> dict:
    """write the granules of tracked bdev `name` that changed since its baseline to the new delta file `path`
    (include/oimgpu.h oimgpu_bdev_image_save_delta)"""
    return _delta_call(load().oimgpu_bdev_image_save_delta, "bdev_image_save_delta", name, path)


def bdev_image_apply_delta(name: str, path) -> dict:
    """apply the delta file `path` to every replica of the unused bdev `name`, whose content must be the delta's parent
    (include/oimgpu.h oimgpu_bdev_image_apply_delta)"""
    return _delta_call(load().oimgpu_bdev_image_apply_delta, "bdev_image_apply_delta", name, path)


def delete_bdev(name: str) -> None:
    _chk(load().oimgpu_bdev_delete(_b(name)), "delete_bdev")


def _bdev_dict(i: BdevInfo) -> dict:
    return {"name": i.name.decode(), "product_name": i.product_name.decode(), "uuid": i.uuid.decode(),
            "num_blocks": i.num_blocks, "block_size": i.block_size, "claimed": bool(i.claimed),
            "device": i.device, "replicas": i.replicas, "device_ptr": i.device_ptr}


def get_bdevs_iostat(name: str) -> dict:
    """S/lib/bdev/rpc/bdev_rpc.c:50-205 get_bdevs_iostat for one bdev"""
    s = IoStat()
    _chk(load().oimgpu_bdev_iostat(_b(name), C.byref(s)), "get_bdevs_iostat")
    return {n: getattr(s, n) for n, _ in IoStat._fields_}


def enable_bdev_histogram(name: str, enable: bool = True) -> None:
    _chk(load().oimgpu_bdev_histogram_enable(_b(name), int(enable)), "enable_bdev_histogram")


def get_bdev_histogram(name: str) -> np.ndarray:
    """[58, 128] uint64: struct spdk_histogram_data buckets (range, index), datapoints in ns"""
    out = np.zeros(58 * 128, dtype=np.uint64)
    _chk(load().oimgpu_bdev_histogram_get(_b(name), out.ctypes.data_as(C.POINTER(C.c_uint64))), "get_bdev_histogram")
    return out.reshape(58, 128)


def get_bdevs(name: str | None = None) -> list[dict]:
    lib = load()
    if name is not None:
        info = BdevInfo()
        _chk(lib.oimgpu_bdev_get(_b(name), C.byref(info)), "get_bdevs")
        return [_bdev_dict(info)]
    n = lib.oimgpu_bdev_list(None, 0)
    arr = (BdevInfo * max(n, 1))()
    n = lib.oimgpu_bdev_list(arr, n)
    return [_bdev_dict(arr[i]) for i in range(n)]


def construct_vhost_scsi_controller(ctrlr: str, cpumask: str | None = None) -> None:
    _chk(load().oimgpu_vhost_scsi_ctrlr_create(_b(ctrlr), _b(cpumask)), "construct_vhost_scsi_controller")


def add_vhost_scsi_lun(ctrlr: str, scsi_target_num: int, bdev_name: str) -> int:
    return _chk(load().oimgpu_vhost_scsi_add_lun(_b(ctrlr), scsi_target_num, _b(bdev_name)), "add_vhost_scsi_lun")


def remove_vhost_scsi_target(ctrlr: str, scsi_target_num: int) -> None:
    _chk(load().oimgpu_vhost_scsi_remove_target(_b(ctrlr), scsi_target_num), "remove_vhost_scsi_target")


def remove_vhost_controller(ctrlr: str) -> None:
    _chk(load().oimgpu_vhost_ctrlr_remove(_b(ctrlr)), "remove_vhost_controller")


def _ctrlr_dict(c: CtrlrInfo) -> dict:
    return {"ctrlr": c.ctrlr.decode(), "cpumask": c.cpumask.decode(), "delay_base_us": c.delay_base_us,
            "iops_threshold": c.iops_threshold, "socket": c.socket.decode(),
            "backend_specific": {"scsi": [
                {"scsi_dev_num": t.scsi_dev_num, "id": t.id, "target_name": t.target_name.decode(),
                 "luns": [{"id": t.lun_id, "bdev_name": t.bdev_name.decode()}]}
                for t in c.targets[:c.ntargets]]}}


def get_vhost_controllers(name: str | None = None) -> list[dict]:
    lib = load()
    if name is not None:
        info = CtrlrInfo()
        _chk(lib.oimgpu_vhost_ctrlr_get(_b(name), C.byref(info)), "get_vhost_controllers")
        return [_ctrlr_dict(info)]
    n = lib.oimgpu_vhost_ctrlr_list(None, 0)
    arr = (CtrlrInfo * max(n, 1))()
    n = lib.oimgpu_vhost_ctrlr_list(arr, n)
    return [_ctrlr_dict(arr[i]) for i in range(n)]


def bdev_read_raw(name: str, offset: int, nbytes: int, replica: int = 0) -> np.ndarray:
    out = np.empty(nbytes, dtype=np.uint8)
    _chk(load().oimgpu_bdev_read_raw(_b(name), replica, offset, out.ctypes.data, nbytes), "bdev_read_raw")
    return out


def bdev_write_raw(name: str, offset: int, data: np.ndarray, replica: int = 0) -> None:
    data = np.ascontiguousarray(data, dtype=np.uint8)
    _chk(load().oimgpu_bdev_write_raw(_b(name), replica, offset, data.ctypes.data, data.size), "bdev_write_raw")


def read_strided(device: int, src: int, pitch: int, width: int, rows: int) -> np.ndarray:
    """rows x width bytes, pitch apart in device memory -> host, by the copy engine (include/oimgpu.h)"""
    out = np.empty(rows * width, dtype=np.uint8)
    _chk(load().oimgpu_read_strided(device, out.ctypes.data, src, pitch, width, rows), "read_strided")
    return out


def write_strided(device: int, dst: int, data: np.ndarray, pitch: int, width: int) -> None:
    data = np.ascontiguousarray(data).view(np.uint8)
    _chk(load().oimgpu_write_strided(device, dst, data.ctypes.data, pitch, width, data.size // width), "write_strided")


def mem_register(arr: np.ndarray) -> None:
    _chk(load().oimgpu_mem_register(arr.ctypes.data, arr.nbytes), "mem_register")


def mem_unregister(arr: np.ndarray) -> None:
    load().oimgpu_mem_unregister(arr.ctypes.data)


class Timer:
    """CUDA events recorded on a LUN's stream."""

    def __init__(self):
        self.a, self.b = C.c_void_p(), C.c_void_p()
        _chk(load().oimgpu_timer_create(C.byref(self.a), C.byref(self.b)), "timer_create")

    def start(self, lun: "Lun"):
        _chk(load().oimgpu_timer_record(lun.h, self.a), "timer_record")

    def stop(self, lun: "Lun"):
        _chk(load().oimgpu_timer_record(lun.h, self.b), "timer_record")

    def elapsed_ms(self) -> float:
        ms = C.c_float()
        _chk(load().oimgpu_timer_elapsed_ms(self.a, self.b, C.byref(ms)), "timer_elapsed")
        return ms.value

    def close(self):
        load().oimgpu_timer_destroy(self.a, self.b)


class Lun:
    """Data-path session on a vhost controller (oimgpu_lun).  target >= 0: the session's home device;
    target == -1: controller-wide session with no home device.  Either way requests reach every
    target of the controller through lun[1], as in the reference."""

    def __init__(self, ctrlr: str, target: int, num_queues: int = 1, queue_size: int = 1024):
        self.h = C.c_void_p()
        _chk(load().oimgpu_lun_open(_b(ctrlr), target, num_queues, queue_size, C.byref(self.h)), "lun_open")
        self.num_queues, self.queue_size, self.target = num_queues, queue_size, target

    def close(self):
        if self.h:
            load().oimgpu_lun_close(self.h)
            self.h = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    @property
    def device(self) -> int:
        return load().oimgpu_lun_device(self.h)

    @property
    def shared_launches(self) -> int:
        """launches in which the CTAs shared the queues a pass at a time (include/oimgpu.h)"""
        return load().oimgpu_lun_shared_launches(self.h)

    def submit(self, q: int, reqs: np.ndarray, iovs: np.ndarray) -> None:
        """host arrays -> queue q's ring (OIMGPU_MEM_HOST)."""
        assert reqs.dtype == abi.req_dtype and iovs.dtype == abi.iov_dtype
        reqs, iovs = np.ascontiguousarray(reqs), np.ascontiguousarray(iovs)
        _chk(load().oimgpu_submit(self.h, q, reqs.ctypes.data, len(reqs), iovs.ctypes.data, len(iovs),
                                  abi.MEM_HOST), "submit")

    def submit_device(self, q: int, d_reqs: int, nreqs: int, d_iovs: int, d_cpls: int) -> None:
        _chk(load().oimgpu_submit_device(self.h, q, d_reqs, nreqs, d_iovs, d_cpls), "submit_device")

    def submit_batch(self, nq: int, per_q: int, reqs: int, iovs: int, niovs: int, cpls: int, mem: int) -> int:
        """queue i gets reqs[i*per_q:(i+1)*per_q]; submit + kick in one C call (raw addresses)."""
        return _chk(load().oimgpu_submit_batch(self.h, nq, per_q, reqs, iovs, niovs, cpls, mem), "submit_batch")

    def kick(self) -> int:
        return _chk(load().oimgpu_kick(self.h), "kick")

    def sync(self) -> None:
        _chk(load().oimgpu_lun_sync(self.h), "lun_sync")

    def poll(self, q: int, max_n: int, wait: bool = True) -> np.ndarray:
        out = np.zeros(max_n, dtype=abi.cpl_dtype)
        n = _chk(load().oimgpu_poll(self.h, q, out.ctypes.data, max_n, int(wait)), "poll")
        return out[:n]

    def run(self, reqs: np.ndarray, iovs: np.ndarray, q: int = 0) -> np.ndarray:
        """submit + kick + wait + reap on one queue, in chunks that fit the ring; returns completions.
        Assumes the SG table is laid out in request order (as Batch/traces build it)."""
        out = []
        iov_cap = max(1024, self.queue_size * 8)
        starts = reqs["iov_start"].astype(np.int64)
        ends = starts + reqs["iovcnt"]
        lo, n = 0, len(reqs)
        while lo < n:
            hi = lo + 1
            while hi < n and hi - lo < self.queue_size and ends[hi] - starts[lo] <= iov_cap:
                hi += 1
            part = reqs[lo:hi].copy()
            b0, b1 = int(starts[lo]), int(max(ends[lo:hi].max(), starts[lo] + 1))
            part["iov_start"] -= np.uint32(b0)
            self.submit(q, part, iovs[b0:b1])
            self.kick()
            out.append(self.poll(q, len(part), wait=True))
            lo = hi
        return np.concatenate(out) if out else np.zeros(0, dtype=abi.cpl_dtype)

    def iostat(self, target: int | None = None) -> dict:
        """counters of the session's home device, or of any target it reaches"""
        s = IoStat()
        if target is None:
            _chk(load().oimgpu_lun_iostat(self.h, C.byref(s)), "iostat")
        else:
            _chk(load().oimgpu_lun_target_iostat(self.h, target, C.byref(s)), "target_iostat")
        return {n: getattr(s, n) for n, _ in IoStat._fields_}

    def set_removed(self, removed: bool = True, lun_removed: bool = False) -> None:
        _chk(load().oimgpu_lun_set_removed(self.h, int(removed), int(lun_removed)), "set_removed")

    # ---- persistent poller ----
    def start_poller(self, max_ctas: int = 0, idle_timeout_ms: int = 0) -> int:
        return _chk(load().oimgpu_lun_start_poller(self.h, max_ctas, idle_timeout_ms), "start_poller")

    def stop_poller(self) -> None:
        _chk(load().oimgpu_lun_stop_poller(self.h), "stop_poller")

    def poller_running(self) -> bool:
        return bool(_chk(load().oimgpu_lun_poller_running(self.h), "poller_running"))

    # ---- virtqueue mode ----
    def set_mem_table(self, regions: np.ndarray) -> None:
        """regions: flat uint64 array of {guest_phys_addr, size, device address} triples"""
        regions = np.ascontiguousarray(regions, dtype=np.uint64)
        _chk(load().oimgpu_lun_set_mem_table(self.h, regions.ctypes.data, len(regions) // 3), "set_mem_table")

    def vq_attach(self, q: int, desc: int, avail: int, used: int, size: int, last_avail: int = 0, last_used: int = 0):
        _chk(load().oimgpu_vq_attach(self.h, q, desc, avail, used, size, last_avail, last_used), "vq_attach")

    def vq_detach(self, q: int) -> tuple[int, int]:
        la, lu = C.c_uint16(), C.c_uint16()
        _chk(load().oimgpu_vq_detach(self.h, q, C.byref(la), C.byref(lu)), "vq_detach")
        return la.value, lu.value

    def vq_kick(self) -> int:
        return _chk(load().oimgpu_vq_kick(self.h), "vq_kick")

    def copy(self, dst: int, src: int, nbytes: int) -> None:
        _chk(load().oimgpu_copy_submit(self.h, dst, src, nbytes), "copy_submit")

    def fill(self, dst: int, value: int, nbytes: int) -> None:
        _chk(load().oimgpu_fill_submit(self.h, dst, value, nbytes), "fill_submit")


class BioChan:
    """Block-I/O channel on one bdev (oimgpu_bio_chan): batches of abi.bio_dtype with an abi.iov_dtype table,
    completions (abi.bio_cpl_dtype) in submission order."""

    def __init__(self, bdev: str):
        self.h = C.c_void_p()
        _chk(load().oimgpu_bio_chan_open(_b(bdev), C.byref(self.h)), "bio_chan_open")

    def close(self):
        if self.h:
            load().oimgpu_bio_chan_close(self.h)
            self.h = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    @property
    def launches(self) -> int:
        return load().oimgpu_bio_chan_launches(self.h)

    def submit(self, bios: np.ndarray, iovs: np.ndarray) -> None:
        assert bios.dtype == abi.bio_dtype and iovs.dtype == abi.iov_dtype
        bios, iovs = np.ascontiguousarray(bios), np.ascontiguousarray(iovs)
        _chk(load().oimgpu_bio_chan_submit(self.h, bios.ctypes.data, len(bios), iovs.ctypes.data, len(iovs)),
             "bio_chan_submit")

    def poll(self, max_n: int) -> np.ndarray:
        out = np.zeros(max(max_n, 1), dtype=abi.bio_cpl_dtype)
        n = _chk(load().oimgpu_bio_chan_poll(self.h, out.ctypes.data, max_n), "bio_chan_poll")
        return out[:n]

    def wait(self, n: int) -> np.ndarray:
        """reap exactly n completions (blocking: spins on poll)"""
        got = []
        while n > 0:
            c = self.poll(n)
            got.append(c)
            n -= len(c)
        return np.concatenate(got) if got else np.zeros(0, dtype=abi.bio_cpl_dtype)
