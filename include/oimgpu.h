/*
 * oimgpu.h — C ABI of liboimgpu.so, the H100-native block-I/O data path that replaces the
 * SPDK vhost daemon behind intel/oim.
 *
 * Plain C: fixed-width integers, plain pointers and sizes, no callbacks, every function
 * returns 0 / a non-negative count on success or -errno.  That makes it directly bindable
 * from cgo (see INTEGRATION.md), ctypes (oim_b200/_abi.py) and C++ (the JSON-RPC daemon).
 *
 * What each group replaces in the reference (paths relative to /root/reference,
 * S/ = vendor/github.com/spdk/spdk/):
 *
 *   bdev control      construct_malloc_bdev   S/lib/bdev/malloc/bdev_malloc_rpc.c:63-106
 *                                             S/lib/bdev/malloc/bdev_malloc.c:378-443
 *                     construct_rbd_bdev      S/lib/bdev/rbd/bdev_rbd_rpc.c:102-148 (RPC shape only)
 *                     delete_bdev / get_bdevs S/lib/bdev/rpc/bdev_rpc.c:216-300,396-433
 *   vhost-scsi ctrl   construct_vhost_scsi_controller / add_vhost_scsi_lun /
 *                     remove_vhost_scsi_target / remove_vhost_controller / get_vhost_controllers
 *                                             S/lib/vhost/vhost_rpc.c:65-478, vhost_scsi.c:951-1103
 *                     (called by pkg/spdk/spdk.go:47-286 and pkg/oim-controller/controller.go:55-212)
 *   data path         one virtio-scsi request = what task_data_setup() hands to the SCSI layer
 *                                             S/lib/vhost/vhost_scsi.c:490-653 (request build)
 *                                             S/lib/scsi/scsi_bdev.c:1456-1802  (CDB decode, limits)
 *                                             S/lib/bdev/malloc/bdev_malloc.c:153-233 (iovec copy / fill)
 *                                             S/lib/copy/copy_engine.c:114-140 (the memcpy/memset)
 *                                             S/lib/vhost/vhost_scsi.c:311-331 (response fields)
 *   copy engine       struct spdk_copy_engine {copy, fill}   S/include/spdk_internal/copy_engine.h:47-53
 */
#ifndef OIMGPU_H
#define OIMGPU_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define OIMGPU_ABI_VERSION		1

/* ---- limits taken from the reference ---------------------------------------------------- */
#define OIMGPU_CDB_SIZE			32	/* VIRTIO_SCSI_CDB_SIZE */
#define OIMGPU_SENSE_SIZE		18	/* fixed-format sense, S/lib/scsi/task.c:198-236 */
#define OIMGPU_IOVS_MAX			129	/* SPDK_VHOST_IOVS_MAX, S/lib/vhost/vhost_internal.h:68 */
#define OIMGPU_CTRLR_MAX_DEVS		8	/* SPDK_VHOST_SCSI_CTRLR_MAX_DEVS, vhost_internal.h:66 */
#define OIMGPU_MAX_VQ_SIZE		1024	/* SPDK_VHOST_MAX_VQ_SIZE, vhost_internal.h:64 */
#define OIMGPU_REQS_PER_PASS		32	/* reqs[32] in process_requestq, vhost_scsi.c:695 */
#define OIMGPU_MAX_XFER_BYTES		(4u * 1024u * 1024u)	/* SPDK_WORK_BLOCK_SIZE, scsi_bdev.c:50 */
#define OIMGPU_MAX_UNMAP_DESC		256	/* DEFAULT_MAX_UNMAP_BLOCK_DESCRIPTOR_COUNT, scsi_bdev.c:58 */
#define OIMGPU_RESP_SIZE		108	/* sizeof(struct virtio_scsi_cmd_resp) */

/* data direction, numerically equal to enum spdk_scsi_data_dir (S/include/spdk/scsi.h:66-70) */
#define OIMGPU_DIR_NONE			0
#define OIMGPU_DIR_TO_DEV		1	/* guest -> device  (WRITE, UNMAP parameter list) */
#define OIMGPU_DIR_FROM_DEV		2	/* device -> guest  (READ, READ CAPACITY ...)     */

/* virtio-scsi response codes (linux/virtio_scsi.h) */
#define OIMGPU_S_OK			0
#define OIMGPU_S_BAD_TARGET		3

/* SCSI status */
#define OIMGPU_STATUS_GOOD		0x00
#define OIMGPU_STATUS_CHECK_CONDITION	0x02

/* where the addresses in an SG list point */
#define OIMGPU_MEM_DEVICE		0	/* device (HBM) pointers valid on the LUN's GPU */
#define OIMGPU_MEM_HOST			1	/* host pointers; pinned + mapped by oimgpu_mem_register() */

/* ---- wire structures (shared, bit for bit, by host code, the kernels and the oracle) ---- */

/* One scatter-gather element: the iovec spdk_vhost_vring_desc_to_iov() produces
 * (S/lib/vhost/vhost.c:461-509).  16 bytes so 32 of them load as one 512-byte bulk copy. */
struct oimgpu_iov {
	uint64_t addr;		/* byte-granular; no alignment requirement */
	uint32_t len;
	uint32_t flags;		/* reserved, must be 0 */
};

/* One request slot (64 bytes).  Bytes 0..50 are exactly struct virtio_scsi_cmd_req
 * (lun[8], tag, task_attr, prio, crn, cdb[32]; packed) so a vhost front end can copy the guest's
 * request header straight in; the tail carries what task_data_setup() derives from the
 * descriptor chain (direction and the SG list). */
struct oimgpu_req {
	uint8_t  lun[8];	/* lun[0]==1, lun[1]=target, (lun[2]<<8|lun[3])&0x3FFF = LUN id */
	uint64_t tag;
	uint8_t  task_attr;
	uint8_t  prio;
	uint8_t  crn;
	uint8_t  cdb[OIMGPU_CDB_SIZE];
	uint8_t  dir;		/* OIMGPU_DIR_* */
	uint16_t iovcnt;	/* number of SG elements (0..129; more => invalid request) */
	uint16_t flags;		/* reserved, must be 0 */
	uint32_t iov_start;	/* index of the first element in the SG table passed with the batch */
	uint32_t reserved;
};

/* One completion (48 bytes).  Bytes 8..37 are the first 30 bytes of struct virtio_scsi_cmd_resp
 * (sense_len, resid, status_qualifier, status, response, sense[0..17]) as written by
 * spdk_vhost_scsi_task_cpl() (vhost_scsi.c:311-331); used_len is the length published in the
 * used ring (vhost_scsi.c:296, 583, 612). */
struct oimgpu_cpl {
	uint64_t tag;
	uint32_t sense_len;
	uint32_t resid;
	uint16_t status_qualifier;
	uint8_t  status;
	uint8_t  response;
	uint8_t  sense[OIMGPU_SENSE_SIZE];
	uint8_t  resp_valid;	/* 1 = response fields above were written; 0 = invalid_request()
				 * (vhost_scsi.c:347-358): only the used-ring element is produced */
	uint8_t  pad;
	uint32_t used_len;
	uint32_t data_transferred;	/* task->data_transferred, for debugging/iostat */
};

/* get_bdevs entry (S/lib/bdev/rpc/bdev_rpc.c:216-300) */
struct oimgpu_bdev_info {
	char     name[64];
	char     product_name[32];	/* "Malloc disk" | "Ceph Rbd Disk" */
	char     uuid[40];
	uint64_t num_blocks;
	uint32_t block_size;
	int32_t  claimed;
	int32_t  device;	/* CUDA device ordinal holding the backing store */
	uint32_t replicas;	/* 1, or R for a mirrored bdev */
	uint64_t device_ptr;	/* backing store base (device address; tests/digest only) */
};

/* get_vhost_controllers target entry (S/lib/vhost/vhost_scsi.c:1410-1456) */
struct oimgpu_target_info {
	int32_t  scsi_dev_num;
	int32_t  id;
	char     target_name[16];	/* "Target N" */
	int32_t  lun_id;		/* always 0 */
	char     bdev_name[64];
};

struct oimgpu_ctrlr_info {
	char     ctrlr[64];
	char     cpumask[20];		/* "0x1" */
	uint32_t delay_base_us;
	uint32_t iops_threshold;
	char     socket[192];
	uint32_t ntargets;
	struct oimgpu_target_info targets[OIMGPU_CTRLR_MAX_DEVS];
};

/* per-LUN counters (the part of get_bdevs_iostat the path feeds, bdev_rpc.c:213) */
struct oimgpu_iostat {
	uint64_t num_read_ops, num_write_ops, num_unmap_ops, num_other_ops;
	uint64_t bytes_read, bytes_written, bytes_unmapped;
	uint64_t num_errors;
	uint64_t kernel_launches;	/* launches of our kernels on this LUN's stream */
	/* get_bdevs_iostat read/write/unmap_latency_ticks (S/lib/bdev/rpc/bdev_rpc.c:51-105) in nanoseconds of the GPU's
	 * global timer (tick_rate 1e9): per completed request, from the moment its pass was fetched to the moment its
	 * data had moved, summed */
	uint64_t read_latency_ns, write_latency_ns, unmap_latency_ns;
};

/* ---- lifecycle -------------------------------------------------------------------------- */

int  oimgpu_abi_version(void);
/* Initialise on the given CUDA device ordinals (devices==NULL: current device only).
 * Fails with -ENODEV when no CUDA device is usable: there is no CPU fallback. */
int  oimgpu_init(const int *devices, int ndevices);
/* Control plane only (protocol tests without a GPU): no stores are allocated, every data-path call
 * returns -ENODEV.  Not a CPU implementation of the path. */
int  oimgpu_init_control_only(void);
void oimgpu_fini(void);
int  oimgpu_device_count(void);
/* vhost -S <dir> and -m <mask> of S/app/vhost/vhost.c:43-48: socket directory reported by
 * get_vhost_controllers / stripped from controller names, and the application core mask controller
 * cpumasks must be a subset of. */
int  oimgpu_set_socket_dir(const char *dir, const char *app_core_mask);
const char *oimgpu_version_string(void);

/* ---- bdev control ----------------------------------------------------------------------- */

/* construct_malloc_bdev: zero-filled backing store of num_blocks*block_size bytes in HBM.
 * name==NULL -> "Malloc%d"; uuid==NULL -> random.  device<0 -> least-loaded initialised GPU.
 * Returns 0 and the final name in name_out, -EINVAL (num_blocks==0, bad uuid, bad block size),
 * -EEXIST, -ENOMEM. */
int oimgpu_bdev_create_malloc(const char *name, const char *uuid, uint64_t num_blocks,
			      uint32_t block_size, int device, char *name_out, size_t name_cap);
/* construct_rbd_bdev: same HBM store, product "Ceph Rbd Disk"; size comes from size_bytes
 * (the RBD image size the reference would learn from librbd). */
int oimgpu_bdev_create_rbd(const char *name, const char *pool_name, const char *rbd_name,
			   const char *user_id, uint32_t block_size, uint64_t size_bytes,
			   int device, char *name_out, size_t name_cap);
/* R-way mirrored malloc bdev: replica r lives on devices[r]; writes fan out over NVLink. */
int oimgpu_bdev_create_mirror(const char *name, uint64_t num_blocks, uint32_t block_size,
			      const int *devices, int nreplicas, char *name_out, size_t name_cap);
/* Mirrors across PROCESSES (one process per GPU, the way bench.py and a per-GPU daemon run): a replica's
 * store is an ordinary bdev of the process that owns that GPU, exported as a CUDA IPC handle
 * (OIMGPU_IPC_HANDLE_BYTES bytes, any byte transport); the primary's process imports the handles and
 * builds the mirrored bdev on its own GPU.  Writes then fan out exactly as for an in-process mirror
 * (P2P stores over NVLink from the mover warps).  No reference counterpart: S/lib/bdev/raid/bdev_raid.c:848-851
 * is RAID0 only (SURVEY.md 8(c), config 5).  The exporting bdev must outlive every importer. */
#define OIMGPU_IPC_HANDLE_BYTES 64
int oimgpu_bdev_export_store(const char *name, int replica, void *handle_out);
int oimgpu_bdev_create_mirror_remote(const char *name, uint64_t num_blocks, uint32_t block_size, int device,
				     const void *peer_handles, int npeers, char *name_out, size_t name_cap);
/* The two constructors above with the bdev's uuid (NULL: random, as for the functions without it; otherwise as
 * construct_malloc_bdev checks it), so that a restored configuration keeps the volume's identity.  In
 * oimgpu_bdev_create_mirror_uuid, devices == NULL places the replicas by rule: replica 0 on the GPU
 * construct_malloc_bdev would pick (least loaded), replica r on the r-th next initialised GPU, wrapping around.
 * -ENOTSUP: a replica's GPU is not peer-reachable from replica 0's.  The remote form returns -EIO when a handle
 * cannot be opened. */
int oimgpu_bdev_create_mirror_uuid(const char *name, const char *uuid, uint64_t num_blocks, uint32_t block_size,
				   const int *devices, int nreplicas, char *name_out, size_t name_cap);
int oimgpu_bdev_create_mirror_remote_uuid(const char *name, const char *uuid, uint64_t num_blocks, uint32_t block_size,
					  int device, const void *peer_handles, int npeers, char *name_out, size_t name_cap);
/* where replica r of a bdev lives: its CUDA ordinal (an imported replica: the GPU it is reached from) and whether it is
 * another process's store; -ENODEV unknown bdev, -EINVAL no such replica */
int oimgpu_bdev_replica_info(const char *name, int replica, int *device, int *imported);
/* Move replica `replica` (1 .. nreplicas-1) of a mirror built with remote replicas to the store behind `handle`
 * (OIMGPU_IPC_HANDLE_BYTES bytes, as oimgpu_bdev_export_store gives them), as mdadm --replace does: replica 0's bytes
 * are copied into the new store on replica 0's GPU, every session of this process is pointed at it, and the old
 * mapping is closed.  On return every session writes to the new store and none can reach the old one; the replica is
 * still imported, reached from the same GPU, and the counters, histogram, uuid and targets of the bdev are unchanged.
 * -EINVAL NULL argument, replica out of range, or a handle that is already one of the mirror's; -ENODEV no such bdev /
 * control-only; -ENOTSUP not a mirror, a mirror with in-process replicas, or the new store's GPU not peer-reachable
 * from replica 0's; -EIO the handle does not open (the mirror is unchanged and keeps serving on the old replica);
 * -EBUSY an NBD export is serving the bdev.  On every failure the mirror is left as it was.
 * Quiescence: as oimgpu_bdev_mirror_check, every session that reaches the bdev (and every session on replica 0's GPU)
 * is held for the call - resident pollers parked and restarted, launched work waited for - so a guest sees one stall
 * of the call's length.  Writers in ANOTHER process are not paused.  The new store must hold at least the bdev's
 * num_blocks * block_size bytes, which nothing here can check.  The old exporter must keep its bdev until the call
 * returns and may delete it afterwards: this is a planned move, not recovery from a dead peer. */
int oimgpu_bdev_mirror_replace_remote(const char *name, int replica, const void *handle);
/* Position-keyed 128-bit digest of [offset, offset+nbytes) of one replica's store (offset and nbytes multiples of
 * 8): out[0] = sum of w_i * (2i+1), out[1] = sum of mix64(w_i ^ i) over the 64-bit words w_i, i counted from the
 * start of the range, all mod 2^64 (mix64 = the splitmix64 finaliser).  Test/bench infrastructure for the
 * size-independent parity properties (replica == replica == expected content) at sizes a host copy is too slow for. */
int oimgpu_bdev_digest(const char *name, int replica, uint64_t offset, uint64_t nbytes, uint64_t out[2]);
int oimgpu_digest_device(int device, const void *dev_ptr, uint64_t nbytes, uint64_t out[2]);
/* check / repair of a mirrored bdev, as md RAID1's `check` and `repair` (mismatch_cnt): an exact block-by-block compare
 * of every replica with replica 0, on replica 0's GPU. */
struct oimgpu_mirror_check {
	uint64_t blocks_checked, mismatched_blocks, repaired_blocks;
	uint32_t nranges;	/* ranges written to `ranges` */
	uint32_t truncated;	/* more ranges than max_ranges */
};
/* Compare every replica of a mirrored bdev with replica 0 over [offset_blocks, offset_blocks + num_blocks); with
 * repair != 0, copy replica 0 over each block that differs.  ranges: max_ranges pairs {offset_blocks, num_blocks} of
 * differing blocks in LBA order.  -ENODEV no such bdev / control-only, -ENOTSUP not a mirror, -EINVAL range outside
 * the bdev or NULL out, -EBUSY an NBD export is serving it.
 * Quiescence: every session that reaches the bdev (and every session on replica 0's GPU) is held for the call, its
 * resident poller parked and restarted afterwards, and what it launched is waited for.  Writers in ANOTHER process - the
 * exporter of an imported replica writing its own bdev - are not paused: quiesce them first, or the result describes
 * a moment of the race and a repair may undo their writes. */
int oimgpu_bdev_mirror_check(const char *name, uint64_t offset_blocks, uint64_t num_blocks, int repair,
			     uint64_t *ranges, uint32_t max_ranges, struct oimgpu_mirror_check *out);
int oimgpu_bdev_delete(const char *name);			/* -ENODEV if unknown; attached targets are hot-removed
								 * (as spdk_bdev_unregister does); -EBUSY while a
								 * data path (oimgpu_lun) is open on it */
int oimgpu_bdev_get(const char *name, struct oimgpu_bdev_info *out);	/* -ENODEV if unknown */
int oimgpu_bdev_list(struct oimgpu_bdev_info *out, int max);	/* returns count */
/* get_bdevs_iostat (S/lib/bdev/rpc/bdev_rpc.c:50-205): what the bdev has served over its lifetime, through
 * whichever sessions and targets; -ENODEV if there is no such bdev.  kernel_launches is 0 here. */
int oimgpu_bdev_iostat(const char *name, struct oimgpu_iostat *out);
/* enable_bdev_histogram / get_bdev_histogram (S/lib/bdev/rpc/bdev_rpc.c:607-790): the latency histogram of struct
 * spdk_histogram_data at bucket_shift 7 - OIMGPU_HISTOGRAM_BUCKETS = 58 ranges x 128 counters, datapoints in ns of the
 * GPU's global timer - tallied per completed request by the mover warps.  get: -EFAULT while disabled and in use. */
#define OIMGPU_HISTOGRAM_BUCKETS (58 * 128)
int oimgpu_bdev_histogram_enable(const char *name, int enable);
int oimgpu_bdev_histogram_get(const char *name, uint64_t *buckets);

/* NBD export (S/lib/nbd/nbd.c:560-806): serve the kernel's NBD transmission protocol for `bdev_name` on a
 * connected socket - the end of the socketpair that did NOT go to /dev/nbdX - until the peer disconnects.
 * Blocking; run it on a thread of its own.  0 = orderly end, -EINVAL = bad request magic, -ENODEV = no bdev. */
int oimgpu_nbd_serve(const char *bdev_name, int sock_fd);

/* gather `rows` x `width` bytes that lie `pitch` apart in device memory into host memory with the copy engine (works
 * next to a resident poller, which a kernel would not): e.g. the used indices of many rings living in HBM */
int oimgpu_read_strided(int device, void *dst, const void *src, size_t pitch, size_t width, size_t rows);
int oimgpu_write_strided(int device, void *dst, const void *src, size_t pitch, size_t width, size_t rows);	/* host -> device */
/* test/digest helpers: raw access to the backing store of replica r (synchronous) */
int oimgpu_bdev_read_raw(const char *name, int replica, uint64_t offset, void *dst, uint64_t len);
int oimgpu_bdev_write_raw(const char *name, int replica, uint64_t offset, const void *src, uint64_t len);

/* ---- vhost-scsi control ----------------------------------------------------------------- */

int oimgpu_vhost_scsi_ctrlr_create(const char *ctrlr, const char *cpumask);	/* -EEXIST, -EINVAL */
/* returns the target number used (>=0) or -ENODEV (no ctrlr), -EEXIST (occupied),
 * -EINVAL (num >= 8 or no such bdev), -ENOSPC (num == -1 and all 8 used) */
int oimgpu_vhost_scsi_add_lun(const char *ctrlr, int scsi_target_num, const char *bdev_name);
int oimgpu_vhost_scsi_remove_target(const char *ctrlr, int scsi_target_num);	/* -ENODEV */
int oimgpu_vhost_ctrlr_remove(const char *ctrlr);	/* -ENODEV, -EBUSY (has targets) */
/* set_vhost_controller_coalescing (S/lib/vhost/vhost_rpc.c:493-544, vhost.c:358-381): interrupt coalescing of the
 * controller's sessions; -ENODEV unknown controller, -EINVAL threshold below 100 IOPS or delay beyond 32 bits of ticks */
int oimgpu_vhost_ctrlr_set_coalescing(const char *ctrlr, uint32_t delay_base_us, uint32_t iops_threshold);
/* get_subsystem_config for "bdev" / "vhost" (S/lib/event/rpc/subsystem_rpc.c:80-129): JSON array of the calls that
 * rebuild the present state; returns the text length (text written if cap allows), -ENOENT unknown subsystem */
long oimgpu_config_json(const char *subsystem, char *buf, size_t cap);
int oimgpu_vhost_ctrlr_get(const char *ctrlr, struct oimgpu_ctrlr_info *out);
int oimgpu_vhost_ctrlr_list(struct oimgpu_ctrlr_info *out, int max);

/* ---- data path -------------------------------------------------------------------------- */

typedef struct oimgpu_lun oimgpu_lun;	/* a data-path session on a vhost controller: queues + stream */

/* Open a data path on `ctrlr` with `num_queues` request queues of `queue_size` slots (power of two,
 * <= OIMGPU_MAX_VQ_SIZE) each, on its own CUDA stream.
 *
 * As in the reference, the queues belong to the CONTROLLER: every request names its SCSI device in
 * lun[1] and reaches whichever of the eight targets that is (spdk_vhost_scsi_task_init_target,
 * S/lib/vhost/vhost_scsi.c:361-387); targets added to or removed from the controller while the
 * session is open are hot-plugged into it (spdk_vhost_scsi_dev_add_tgt / _remove_tgt, :951-1100).
 *
 * scsi_target_num >= 0 names the session's home device: it must exist, pins its bdev, decides the
 * GPU, and is what oimgpu_lun_iostat / _set_removed refer to.  scsi_target_num == -1 opens a
 * session with no home device (what a vhost-user connection is): it may start with zero targets. */
int oimgpu_lun_open(const char *ctrlr, int scsi_target_num, uint32_t num_queues,
		    uint32_t queue_size, oimgpu_lun **out);
/* the same controller-wide session (as scsi_target_num == -1) placed on GPU `device` instead of the first target's:
 * one per GPU lets a single vhost-user connection use every GPU's PCIe link (see oim_b200/daemon/vhost_user.cpp) */
int oimgpu_lun_open_on(const char *ctrlr, int device, uint32_t num_queues, uint32_t queue_size, oimgpu_lun **out);
int oimgpu_device_ordinal(int index);		/* CUDA ordinal of the index-th initialised GPU (0 <= index < oimgpu_device_count()) */
int oimgpu_lun_close(oimgpu_lun *lun);
int oimgpu_lun_device(const oimgpu_lun *lun);
/* launches so far in which the CTAs SHARED the queues a pass at a time (fewer queues than the GPU holds CTAs)
 * instead of owning one queue each; diagnostics for tests and the bench */
long long oimgpu_lun_shared_launches(const oimgpu_lun *lun);

/* Pin + map a host buffer so SG elements may point into it (OIMGPU_MEM_HOST).  The analogue of
 * spdk_mem_register() on the guest's memory table (S/lib/vhost/vhost.c:1044-1100). */
int oimgpu_mem_register(void *addr, size_t len);
int oimgpu_mem_unregister(void *addr);
/* device-side address of a byte inside a registered range (for oimgpu_lun_set_mem_table / oimgpu_vq_attach) */
int oimgpu_mem_device_addr(const void *addr, uint64_t *dev);

/* Submit `nreqs` requests to queue `q` of the LUN.  reqs[i].iov_start indexes into `iovs`
 * (niovs entries).  `mem` says where SG addresses AND the reqs/iovs/cpls arrays of this call live:
 *   OIMGPU_MEM_HOST   : reqs/iovs are host arrays, copied to the device inside the call
 *   OIMGPU_MEM_DEVICE : reqs/iovs are device arrays already resident in HBM (zero host work)
 * Requests of one queue are executed in order in passes of <= 32 (process_requestq); requests of
 * different queues have no mutual order.  Asynchronous: returns once the work is enqueued on the
 * LUN's stream.  -EAGAIN when the queue has fewer than nreqs free slots. */
int oimgpu_submit(oimgpu_lun *lun, uint32_t q, const struct oimgpu_req *reqs, uint32_t nreqs,
		  const struct oimgpu_iov *iovs, uint32_t niovs, int mem);

/* OIMGPU_MEM_DEVICE submission with the completion array also in HBM (nothing touches the host). */
int oimgpu_submit_device(oimgpu_lun *lun, uint32_t q, const struct oimgpu_req *d_reqs, uint32_t nreqs,
			 const struct oimgpu_iov *d_iovs, struct oimgpu_cpl *d_cpls);

/* Run every queue's outstanding requests to completion on the LUN's stream ("kick").  With
 * OIMGPU_MEM_DEVICE completions stay in HBM at the address returned by oimgpu_queue_cpl_ptr(). */
int oimgpu_kick(oimgpu_lun *lun);
/* Reap up to `max` completions of queue q in submission order into host memory; blocks until the
 * kicked work is finished if wait != 0.  Returns the number reaped. */
int oimgpu_poll(oimgpu_lun *lun, uint32_t q, struct oimgpu_cpl *cpls, uint32_t max, int wait);
int oimgpu_lun_sync(oimgpu_lun *lun);	/* wait for everything kicked so far */

/* Batch forms for callers that own a whole batch: queue i (0..nq-1) gets reqs[i*per_q .. (i+1)*per_q),
 * all indexing the one SG table `iovs`.  oimgpu_submit_batch = submit + kick (asynchronous; with
 * OIMGPU_MEM_DEVICE `cpls` is the device completion array); oimgpu_submit_and_wait adds wait + reap. */
int oimgpu_submit_batch(oimgpu_lun *lun, uint32_t nq, uint32_t per_q,
			const struct oimgpu_req *reqs, const struct oimgpu_iov *iovs,
			uint32_t niovs, struct oimgpu_cpl *cpls, int mem);
int oimgpu_submit_and_wait(oimgpu_lun *lun, uint32_t nq, uint32_t per_q,
			   const struct oimgpu_req *reqs, const struct oimgpu_iov *iovs,
			   uint32_t niovs, struct oimgpu_cpl *cpls, int mem);

int oimgpu_lun_iostat(oimgpu_lun *lun, struct oimgpu_iostat *out);
/* the same counters for any target the session reaches (-ENODEV: none at that number) */
int oimgpu_lun_target_iostat(oimgpu_lun *lun, int scsi_target_num, struct oimgpu_iostat *out);
/* raw CUDA stream handle (cudaStream_t) of the LUN, for callers that time with CUDA events */
void *oimgpu_lun_stream(oimgpu_lun *lun);

/* ---- virtqueue mode: hand the guest's own virtio split rings to the GPU ---------------------
 * Replaces spdk_vhost_vq_avail_ring_get / spdk_vhost_vq_get_desc / spdk_vhost_vring_desc_to_iov /
 * task_data_setup / spdk_vhost_vq_used_ring_enqueue (S/lib/vhost/vhost.c:178-247,397-509,
 * S/lib/vhost/vhost_scsi.c:490-624): the kernel walks descriptor chains (direct and INDIRECT),
 * translates guest-physical addresses through the memory table, and writes the response buffers and
 * the used ring itself. */
struct oimgpu_mem_region {		/* struct rte_vhost_mem_region, S/lib/vhost/rte_vhost/rte_vhost.h:52-60 */
	uint64_t guest_phys_addr;
	uint64_t size;
	uint64_t addr;			/* device-accessible address the range is mapped at */
};
int oimgpu_lun_set_mem_table(oimgpu_lun *lun, const struct oimgpu_mem_region *regions, uint32_t nregions);
int oimgpu_vq_attach(oimgpu_lun *lun, uint32_t q, const void *desc, const void *avail, void *used,
		     uint32_t size, uint16_t last_avail_idx, uint16_t last_used_idx);
int oimgpu_vq_detach(oimgpu_lun *lun, uint32_t q, uint16_t *last_avail_idx, uint16_t *last_used_idx);
int oimgpu_vq_kick(oimgpu_lun *lun);	/* process every attached ring up to its avail->idx; asynchronous */

/* ---- persistent poller: one resident "reactor" kernel per LUN (replaces the vdev_worker poller that
 * spdk_poller_register() keeps running on a reactor core, S/lib/vhost/vhost_scsi.c:758-772,1311-1318).
 * The kernel polls the tail doorbell of every library ring and the avail->idx of every attached
 * virtqueue from mapped host memory; oimgpu_kick() becomes a doorbell write, oimgpu_poll() reads the
 * completion counter.  max_ctas == 0: one CTA per queue up to the GPU's capacity.
 * idle_timeout_ms != 0: watchdog, the kernel leaves after that long without work. */
int oimgpu_lun_start_poller(oimgpu_lun *lun, uint32_t max_ctas, uint32_t idle_timeout_ms);
int oimgpu_lun_stop_poller(oimgpu_lun *lun);
int oimgpu_lun_poller_running(oimgpu_lun *lun);

/* Session-visible hot-remove state of the target (S/lib/vhost/vhost_scsi.c:1093-1100: `removed`;
 * S/lib/scsi/lun.c:171-176: `lun_removed`). */
int oimgpu_lun_set_removed(oimgpu_lun *lun, int removed, int lun_removed);

/* CUDA-event timing on the LUN's stream (torch.cuda.Event only sees torch's streams). */
int  oimgpu_timer_create(void **start, void **stop);
int  oimgpu_timer_record(oimgpu_lun *lun, void *event);
int  oimgpu_timer_elapsed_ms(void *start, void *stop, float *ms);
void oimgpu_timer_destroy(void *start, void *stop);

/* ---- copy-engine level (B2): the operator SPDK's bdev_malloc calls ----------------------- */

/* struct spdk_copy_engine.copy / .fill for device-resident buffers, enqueued on the LUN's
 * stream; completion is observed with oimgpu_lun_sync(). */
int oimgpu_copy_submit(oimgpu_lun *lun, void *dst, const void *src, uint64_t nbytes);
int oimgpu_fill_submit(oimgpu_lun *lun, void *dst, uint8_t fill, uint64_t nbytes);

/* The same operator as an ASYNCHRONOUS engine without a LUN behind it - what a `struct spdk_copy_engine`
 * implementation needs (S/include/spdk_internal/copy_engine.h:47-53; model: the I/OAT engine,
 * S/lib/copy/ioat/copy_engine_ioat.c:159-221: submit returns at once, a poller on the channel's thread reaps
 * completions and calls the callbacks).  integration/spdk/copy_engine_oimgpu.c is that implementation.
 * Pointers may be device memory or host memory; host memory is pinned for the GPU on first use
 * (oimgpu_mem_ensure), the way SPDK's env layer registers its DMA memory with a device's IOMMU. */
typedef struct oimgpu_copy_chan oimgpu_copy_chan;
int oimgpu_copy_chan_open(int device, oimgpu_copy_chan **out);		/* device < 0: the first initialised GPU */
int oimgpu_copy_chan_close(oimgpu_copy_chan *chan);			/* waits for what is in flight */
int oimgpu_copy_chan_copy(oimgpu_copy_chan *chan, void *dst, const void *src, uint64_t nbytes, void *tag);
int oimgpu_copy_chan_fill(oimgpu_copy_chan *chan, void *dst, uint8_t fill, uint64_t nbytes, void *tag);
/* completed operations in submission order: their tags; returns how many (<= max), 0 if none yet */
int oimgpu_copy_chan_poll(oimgpu_copy_chan *chan, void **tags, int max);
unsigned long long oimgpu_copy_chan_launches(const oimgpu_copy_chan *chan);	/* kernels launched so far */
/* make [addr, addr+len) accessible to the GPUs: device memory is taken as it is; host memory is pinned page-granular
 * and idempotently, and pages already registered (by this library or by another owner) are skipped, so a range that
 * straddles another owner's buffer has every page mapped; -EFAULT if the range cannot be pinned */
int oimgpu_mem_ensure(const void *addr, size_t len);

/* ---- block-I/O channel (one level above the copy engine: struct spdk_bdev_fn_table) ---------------------
 * Block I/O with caller iovecs on one HBM-resident oimgpu bdev, for an SPDK bdev module
 * (integration/spdk/bdev_oimgpu.c) whose submit_request hands its bdev_ios over in batches.  No SCSI:
 * no 4 MiB transfer cap, no 129-element SG cap.  One oim_bio_kernel launch serves a whole batch (more when
 * the batch holds overlapping I/Os one of which writes: each launch then ends before the next one starts).
 * Requests of one channel take effect in submission order wherever ranges overlap and one of them writes;
 * different channels are mutually unordered.  iovecs point into device memory or ordinary host memory, which
 * is pinned on first use (oimgpu_mem_ensure).  The buffers of an I/O belong to the channel until it completes.
 * The bdev's own counters (oimgpu_bdev_iostat) do not count these I/Os: the bdev layer above does. */
#define OIMGPU_BIO_READ			0
#define OIMGPU_BIO_WRITE		1
#define OIMGPU_BIO_WRITE_ZEROES		2	/* fills with 0x00 */
#define OIMGPU_BIO_UNMAP		3	/* fills with 0x00, as bdev_malloc_unmap does (bdev_malloc.c:222-233) */

struct oimgpu_bio {
	uint64_t offset_blocks;
	uint64_t num_blocks;
	uint32_t op;		/* OIMGPU_BIO_* */
	uint32_t iov_start;	/* READ / WRITE: first element in the iovec table passed with the batch */
	uint32_t iovcnt;
	uint32_t flags;		/* reserved, must be 0 */
	uint64_t tag;
};

struct oimgpu_bio_cpl {
	uint64_t tag;
	int32_t  status;	/* 0 or -errno: -EINVAL for a bio outside the bdev, a bad op, iovecs out of the table or
				 * READ / WRITE iovecs summing to fewer bytes than the bio; -EFAULT if an iovec could
				 * not be made accessible to the GPU.  A failed bio moves nothing. */
	uint32_t pad;
};

typedef struct oimgpu_bio_chan oimgpu_bio_chan;
/* -ENODEV no GPU or no such bdev, -ENOTSUP mirrored bdev.  The bdev cannot be deleted (-EBUSY) while a channel is open. */
int oimgpu_bio_chan_open(const char *bdev_name, oimgpu_bio_chan **out);
/* Asynchronous: returns once the batch is enqueued.  Exactly num_blocks x block_size bytes move per bio, even where
 * its iovecs hold more.  Returns 0, or -errno when nothing of the batch was taken (-EINVAL: NULL arguments). */
int oimgpu_bio_chan_submit(oimgpu_bio_chan *chan, const struct oimgpu_bio *bios, uint32_t n,
			   const struct oimgpu_iov *iovs, uint32_t niovs);
/* completions in submission order; returns how many (<= max), 0 if none yet */
int oimgpu_bio_chan_poll(oimgpu_bio_chan *chan, struct oimgpu_bio_cpl *out, int max);
int oimgpu_bio_chan_close(oimgpu_bio_chan *chan);		/* waits for what is in flight */
unsigned long long oimgpu_bio_chan_launches(const oimgpu_bio_chan *chan);	/* oim_bio_kernel launches so far */

#ifdef __cplusplus
}
#endif
#endif /* OIMGPU_H */
