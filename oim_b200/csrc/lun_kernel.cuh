/*
 * lun_kernel.cuh — the per-LUN request-queue kernel (sm_90a).
 *
 * This one kernel is the GPU-side replacement of everything SPDK's vhost reactor does per request
 * between "a head appears in the avail ring" and "the used element is published"
 * (SURVEY.md §3.2; S/ = /root/reference/vendor/github.com/spdk/spdk/):
 *
 *   vdev_worker / process_requestq        S/lib/vhost/vhost_scsi.c:758-772, 690-741
 *       one CTA per request queue, <= 32 requests per pass, one parser lane per request
 *   task_data_setup                       vhost_scsi.c:490-624   -> parse_sg()
 *   spdk_vhost_scsi_task_init_target      vhost_scsi.c:361-387   -> parse_request()
 *   spdk_scsi_task_process_null_lun       S/lib/scsi/task.c:258-293
 *   spdk_bdev_scsi_process_block          S/lib/scsi/scsi_bdev.c:1681-1802 (CDB decode)
 *   spdk_bdev_scsi_readwrite/_read/_write scsi_bdev.c:1456-1511, 1318-1411
 *   spdk_bdev_scsi_unmap / __copy_desc    scsi_bdev.c:1545-1679
 *   spdk_bdev_readv/writev, valid_blocks  S/lib/bdev/bdev.c:2474-2509, 2559-2703
 *   bdev_malloc_readv/writev/unmap        S/lib/bdev/malloc/bdev_malloc.c:153-233
 *   mem_copy_submit / mem_copy_fill       S/lib/copy/copy_engine.c:114-140  -> move_unit()
 *   spdk_vhost_scsi_task_cpl              vhost_scsi.c:311-331   -> completion record
 *
 * Data layout in HBM: the backing store is one flat byte array (LBA n at byte n*block_size,
 * bdev_malloc.c:401); request slots (64 B), SG elements (16 B) and completion slots (48 B) are
 * flat arrays per queue (include/oimgpu.h).  Payload moves HBM->HBM (or HBM<->mapped host memory)
 * in 16-byte vectors, 8 outstanding per lane.
 *
 * Ordering: the reference executes a queue's requests one after the other, so within a queue the
 * result is sequentially consistent in ring order.  Here a queue is owned by one CTA; inside a
 * pass, requests whose LBA ranges conflict (RAW/WAW/WAR) are put in successive "waves" separated by
 * a CTA barrier; passes follow each other in order.  Different queues are unordered, as they are
 * for any multi-queue block device.
 */
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "oimgpu.h"

namespace oimgpu {

constexpr int kPass = OIMGPU_REQS_PER_PASS;	/* 32 = one warp of parser lanes */
#ifndef OIM_MOVERS
#define OIM_MOVERS 7
#endif
#ifndef OIM_STAGES
#define OIM_STAGES 3
#endif
constexpr int kMovers = OIM_MOVERS;		/* mover warps per CTA */
constexpr int kThreads = (1 + kMovers) * 32;	/* parser warp + movers */
constexpr int kStages = OIM_STAGES;		/* parser -> mover pipeline depth */
#ifndef OIM_FILL_UNITS
#define OIM_FILL_UNITS 256
#endif
constexpr int kFillUnits = OIM_FILL_UNITS;	/* units per stage fill (a request larger than that has a fill of its own) */
constexpr int kSegCap = 256;			/* SG segments per stage (>= 256 UNMAP descriptors, >= 129 iovecs) */
constexpr uint32_t kUnitBytes = 4096;		/* bytes one warp moves per step: 8 x 16 B per lane */
constexpr int kMaxReplicas = 4;
constexpr int kMaxRegions = 8;			/* VHOST_MEMORY_MAX_NREGIONS */
constexpr int kHistBuckets = 58 * 128;		/* SPDK_HISTOGRAM_NUM_BUCKETS at bucket_shift 7 (S/include/spdk/histogram_data.h:48-55) */
constexpr int kIovRow = OIMGPU_IOVS_MAX + 1;	/* scratch SG row per parser lane in virtqueue mode */

enum : uint8_t { OP_NONE = 0, OP_READ = 1, OP_WRITE = 2, OP_UNMAP = 3, OP_FLUSH = 4 };	/* OP_FLUSH: SYNCHRONIZE CACHE, no data */

enum : uint8_t { SC_GOOD = 0x00, SC_CHECK = 0x02 };
enum : uint8_t { SK_NO_SENSE = 0x0, SK_ILLEGAL_REQUEST = 0x5, SK_ABORTED_COMMAND = 0xb };
enum : uint8_t { ASC_NONE = 0x00, ASC_INVALID_OPCODE = 0x20, ASC_LBA_OOR = 0x21, ASC_INVALID_FIELD = 0x24,
		 ASC_LUN_NOT_SUPPORTED = 0x25 };

/* per-LUN state, resident in HBM: the device-side struct malloc_disk + session target state */
struct LunCtx {
	uint8_t  *store[kMaxReplicas];	/* replica 0 is local; others are peer (NVLink) mappings */
	uint32_t nreplicas;
	uint64_t num_blocks;
	uint32_t block_size;
	uint32_t block_shift;		/* log2(block_size), or 0xffffffff when not a power of two */
	uint8_t  target;		/* SCSI target number of this LUN inside its controller (0xff: none -
					 * a controller-wide session that reaches every device through peer[]) */
	uint8_t  removed;		/* session saw a hot-remove of this target */
	uint8_t  lun_removed;
	/* guest memory table for virtqueue mode: struct rte_vhost_memory (rte_vhost.h:52-66) with
	 * host_user_addr replaced by a device-accessible address */
	uint32_t nregions;
	struct { uint64_t gpa, size, addr; } region[kMaxRegions];
	/* what INQUIRY embeds (S/lib/scsi/scsi_bdev.c:188-805): bdev name / product, SCSI device name and id,
	 * target port name and index, protocol identifier */
	char     bdev_name[64], product_name[32], dev_name[16], port_name[16];
	int32_t  scsi_dev_id;
	uint16_t port_index;
	uint8_t  protocol_id;
	unsigned long long stats[12];	/* read ops, write ops, unmap ops, other, bytes r/w/unmapped, errors,
					 * [8..10] summed latency in ns of reads / writes / unmaps (get_bdevs_iostat *_latency_ticks) */
	/* [0] reads [1] writes + unmaps the session's kernels have served (any target).  Copied to the host behind every
	 * launch: it picks the launch shape from the recent mix - queue sharing pays for read-dominated sessions only */
	unsigned long long mix[2];
	/* enable_bdev_histogram: the bdev's latency histogram in HBM (struct spdk_histogram_data's buckets, 58 ranges x 128;
	 * nullptr while disabled); mover warp 0 tallies every completed request's latency */
	unsigned long long *hist;
	/* the other SCSI devices of the same vhost controller (svdev->scsi_dev[8], vhost_scsi.c:80-94):
	 * one set of virtqueues serves them all */
	LunCtx *peer[OIMGPU_CTRLR_MAX_DEVS];
};

/* per-launch work header: CTAs draw queue indices from `next` so that uneven queue counts and
 * lengths balance across the grid (copied to the device together with the QueueDesc array) */
struct KickHeader {
	uint32_t next;
	uint32_t nqueues;
	/* persistent ("reactor") mode: the kernel stays resident, CTA b polls queues b, b+grid, ... for
	 * new doorbell values until *stop != 0 (or nothing happened for idle_timeout_ms: watchdog) */
	uint32_t persistent;
	uint32_t idle_timeout_ms;
	const volatile uint32_t *stop;		/* mapped host memory, written by the host */
	volatile uint32_t *exited;		/* mapped host memory: CTAs that left the poll loop */
	/* Doorbells live in host memory (the guest's avail->idx, the library's tail counters).  If every idle
	 * CTA polled them itself, the PCIe reads of the idle ones would slow the busy ones down.  With dispatcher != 0 the LAST CTA of the grid is a dispatcher: one warp reads
	 * all doorbells, 32 per sweep step, and mirrors them into VqState::hint in device memory, which is
	 * what the worker CTAs poll; it mirrors the stop flag the same way. */
	uint32_t dispatcher;
	volatile uint32_t stop_mirror;
	/* Queue sharing (fewer queues than CTAs): a queue is no longer owned by one CTA; CTAs claim it a pass at a
	 * time through share[queue] (struct QShare), so one deep queue - or the <= 254 request queues a vhost-user
	 * controller can have (S/lib/vhost/vhost_internal.h:63) - still keeps every SM busy. */
	uint32_t shared;
	uint32_t pad;
	struct QShare *share;			/* [nqueues], device memory, zeroed (launch) / preset (poller) by the host */
	uint32_t workers_exited;		/* persistent + shared: worker CTAs that left; the last one writes the cursors back */
	uint32_t pad2;
};

/* Per-queue coordination block of a shared queue.  All positions count requests from where this launch
 * (or this poller) started on the queue: request x sits at ring position base_avail + x, its completion at
 * base_used + x.
 *   claim   handed out so far (CAS)                       -> which CTA serves which pass
 *   parsed  parse results published, IN RING ORDER        -> a later pass learns whether earlier ones write
 *           (low half of `chain`)
 *   done    completions published, IN RING ORDER          -> used->idx / the host's completion counter stay
 *                                                            monotonic; a writer can wait for "everything before me"
 * Ordering between passes of DIFFERENT CTAs is coarse (a pass that writes waits for every earlier foreign pass,
 * any pass waits for the last foreign pass that wrote); between passes of the SAME CTA the exact wave / drain
 * logic of the exclusive path applies, so a queue served by one CTA at a time loses nothing. */
struct QShare {
	uint64_t chain;			/* low 32 bits: `parsed`; high 32 bits: end of the last parsed pass that contains a
					 * writer (0: none yet).  One word, one store: see the parser */
	uint32_t claim;
	uint32_t done;
	uint32_t latched;		/* launch + virtqueue: 0 unset, 2 being set, 1 count/base_* valid */
	uint32_t count;			/* launch mode: requests this launch serves on the queue */
	uint32_t base_avail, base_used;
	uint32_t pad[8];
};
static_assert(sizeof(QShare) == 64, "QShare is one 64-byte line");

/* ring cursors of an attached virtqueue, device-resident so they survive across launches */
struct VqState {
	uint32_t last_avail;		/* rte_vhost_vring.last_avail_idx (16 significant bits) */
	uint32_t last_used;
	uint32_t hint;			/* persistent mode: doorbell value last seen by the dispatcher CTA */
	uint32_t pad;
};

enum : uint32_t { QMODE_SLOTS = 0, QMODE_VRING = 1 };

/* one request queue as the kernel sees it for one launch */
struct QueueDesc {
	const oimgpu_req *reqs;
	const oimgpu_iov *iovs;		/* SG table (virtqueue mode: this launch's scratch rows) */
	oimgpu_cpl       *cpls;
	uint32_t ring_mask;		/* slot index mask (0xffffffff: linear array) */
	uint32_t iov_mask;
	uint32_t head;			/* first slot to process */
	uint32_t count;			/* number of slots to process */
	uint32_t mode;			/* QMODE_* */
	uint32_t iov_limit;		/* entries in the SG table (0: not checked) */
	uint32_t vq_size;		/* virtqueue mode: a real virtio split ring (linux/virtio_ring.h) */
	/* persistent mode, slot rings: host-written tail doorbell / device-written completion count */
	const volatile uint32_t *doorbell;
	volatile uint32_t *done;
	const uint8_t *vq_desc;		/* struct vring_desc[vq_size] */
	const uint8_t *vq_avail;	/* struct vring_avail */
	uint8_t       *vq_used;		/* struct vring_used */
	VqState       *vq_state;
	uint32_t vq_in_hbm;		/* the ring and the response buffers are device memory: ordering the used
					 * index behind them needs a GPU-scope fence only (host memory: system scope) */
	uint32_t pad;
};

/* one contiguous piece of payload to move (or to zero when src == nullptr) */
enum : uint16_t { kSegWaveMask = 0x7fff, kSegWaitsForDrain = 0x8000 };	/* Segment::wave */

struct Segment {
	const uint8_t *src;
	uint8_t *dst;
	uint64_t len;
	uint32_t first_unit;		/* exclusive prefix sum of units over the round's segments */
	uint16_t wave;
	uint16_t mirror;		/* t+1: dst is in the store of target t, which has replicas to update; 0: plain */
};

/* What a parser lane knows about its request after decode; lives in shared memory so that the
 * parser's state never competes with the movers' data registers */
struct LaneState {
	uint64_t off;			/* byte offset in the backing store */
	uint64_t store_lo, store_hi;	/* device address range touched, for hazard detection */
	uint32_t length;		/* task->length: sum of SG element lengths */
	uint32_t nseg;			/* segments this request emits */
	uint32_t units;
	uint32_t data_transferred;
	uint32_t used_len;
	uint8_t  op;			/* OP_* */
	uint8_t  valid;			/* 0: invalid_request() */
	uint8_t  status, sk, asc;
	uint8_t  response;
	uint8_t  resp_valid;
	uint8_t  hazard;		/* 0 none, 1 reads store, 2 writes store, 3 barrier (multi-range writer) */
	uint8_t  tgt;			/* SCSI target the request addressed (valid once the target check passed) */
	uint64_t unmap_bytes;		/* UNMAP: bytes of the descriptors that were applied */
	uint8_t  scratch[256];		/* control payloads: READ CAPACITY, REQUEST SENSE, INQUIRY pages (<= 125 B),
					 * MODE SENSE (<= 188 B), REPORT LUNS */
};

/* one pipeline stage: what the movers need for (part of) one pass + its completion records */
struct __align__(16) Stage {
	Segment seg[kSegCap];
	oimgpu_cpl cpl[kPass];
	oimgpu_cpl *cpl_ring;		/* where the records go once the movers are done */
	uint32_t cpl_slot0, cpl_mask, ncpl;
	/* virtqueue mode: guest response buffers + used ring instead of completion slots */
	uint64_t resp[kPass];
	uint16_t vq_head[kPass];
	uint8_t  *vq_used;
	VqState  *vq_state;
	volatile uint32_t *done;	/* persistent slot ring: completion counter in host memory */
	uint32_t vq_size, used_base, mode, vq_in_hbm;
	uint32_t nseg, nunits, nwaves;
	uint32_t drain;			/* d != 0: fill c-d must be finished before flagged units of this one move */
	uint32_t drain_upfront;		/* ... before anything of this one moves (later fills of a split pass) */
	uint32_t stop;
	QShare  *share;			/* shared queue: publish in ring order through share->done (nullptr: exclusive) */
	uint32_t share_pos;		/* position of this fill's first request */
	uint32_t share_final;		/* launch + virtqueue: position at which the ring cursors are written back (count) */
	uint32_t persistent;
	uint32_t unit_ctr;		/* shared kernels: movers draw units from here (mover 0 also publishes, so it takes fewer) */
	/* latency accounting (_spdk_bdev_io_complete, bdev.c:3233-3258, per completed bdev_io: the histogram tallies
	 * every one, the latency sums only reads, writes and unmaps): when the pass was taken and how many bdev_ios of
	 * each kind the fill's requests made; mover warp 0 adds (now - t0) x count when the fill's data has moved - the
	 * parser only stamps */
	uint64_t t0;
	uint8_t  lat_ntgt, lat_tgt[OIMGPU_CTRLR_MAX_DEVS];	/* the SCSI targets the fill's bdev_ios went to ... */
	uint16_t lat_n[OIMGPU_CTRLR_MAX_DEVS][4];		/* ... and how many reads / writes / unmap descriptors / flushes each */
};

/* Store ranges of one pass, for hazard detection against the passes after it (parser-private).
 * Exact ranges per request plus two signatures - hashed bitmaps over 4 KiB granules of device address
 * space, one for the granules read, one for the granules written.  A request can only conflict with
 * the pass if one of its granules is set in the signature that matters for it, so the common case (no
 * conflict) costs a handful of shared-memory loads per request instead of a 32-entry range scan. */
constexpr int kSmemIovs = 4;
#ifndef OIM_SIG_LOG2
#define OIM_SIG_LOG2 14		/* 16 384 bits: with 32 writers a pass sets 0.2 % of them.  At 4096 bits (round 1) false positives
				 * were frequent, and the lane that has one scans 32 exact ranges while the others wait */
#endif
constexpr int kSigBits = 1 << OIM_SIG_LOG2, kSigWords = kSigBits / 32, kSigMaxGranules = 32;

struct __align__(16) HazPass {
	uint64_t lo[kPass], hi[kPass];
	uint8_t  haz[kPass];		/* LaneState::hazard of each request */
	uint32_t writers, touching;	/* lane masks: haz >= 2, haz != 0 */
	uint32_t dense;			/* a request too large (or a barrier) for the signatures: always scan */
	uint32_t sig_r[kSigWords], sig_w[kSigWords];
};

struct __align__(16) CtaShared {
	Stage stage[kStages];
	HazPass hist[kStages];		/* ring: the pass being parsed + the kStages-1 before it */
	/* parser-private: the request slots of the pass being parsed and of the next one.  Slot rings are staged here by
	 * the TMA unit (cp.async.bulk, one 2 KiB copy per pass, completion on req_bar): the fetch of pass p+1 is in
	 * flight, outside the register file, while pass p is parsed.  Virtqueue mode builds its slots here itself. */
	oimgpu_req reqbuf[2][kPass];
	uint64_t req_bar[2];
	oimgpu_iov sg[kPass][kSmemIovs];	/* virtqueue mode: the SG list of a request with few elements stays on chip */
	LaneState lane[kPass];
	uint64_t full[kStages];		/* mbarriers */
	uint64_t empty[kStages];
	uint64_t released[kStages];	/* shared kernels: the fill's completions are published, the stage may be refilled */
	uint64_t ubar[kMovers][2];	/* movers: arrival of the two pieces of a byte-granular unit in ustage (move_unit_via_smem) */
	QShare  *pub_q;			/* shared kernels, mover warp 0: queue and end position of its last publication */
	uint32_t pub_end;
	unsigned long long lat_ns[OIMGPU_CTRLR_MAX_DEVS][3];	/* mover warp 0, lane 0: summed latencies of this CTA per target (reads, writes, unmaps) */
	/* one staging buffer per mover warp for units that are not 16-byte aligned on both sides: the aligned bytes
	 * covering a unit (<= kUnitBytes + 16) land here by bulk copy and are realigned on the way out */
	/* LAST member: kernels without the staged path are launched without it (lun_kernel_smem_bytes) */
	__align__(128) uint8_t ustage[kMovers][kUnitBytes + 128];
};

/* the queue kernel's instantiations (lun_kernel.cu); the host picks one per launch */
enum LunKernel : int {
	LUN_KERNEL_QUEUE,		/* one CTA per queue */
	LUN_KERNEL_QUEUE_MIRROR,	/* ... with mirrored bdevs */
	LUN_KERNEL_VRING,		/* ... guest virtqueues only */
	LUN_KERNEL_SHARED_QUEUE,	/* CTAs share the queues a pass at a time (KickHeader::shared) */
	LUN_KERNEL_SHARED_QUEUE_MIRROR,
	LUN_KERNEL_COUNT
};
/* gives every instantiation the shared memory it is launched with; *ctas_per_sm = occupancy of the queue kernels */
cudaError_t lun_kernels_init(int *ctas_per_sm);
void launch_lun_kernel(LunKernel k, uint32_t grid, cudaStream_t stream, LunCtx *ctx, KickHeader *hdr, const QueueDesc *desc);

/* ------------------------------------------------------------------------------------------ */

__device__ __forceinline__ int4 ld_cg16(const void *p)
{
	int4 r;
	asm volatile("ld.global.cg.v4.s32 {%0,%1,%2,%3}, [%4];"
		     : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p) : "memory");
	return r;
}
__device__ __forceinline__ void st_cg16(void *p, const int4 &v)
{
	asm volatile("st.global.cg.v4.s32 [%0], {%1,%2,%3,%4};"
		     :: "l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ uint8_t ld_cg8(const uint8_t *p)
{
	uint32_t r;
	asm volatile("ld.global.cg.u8 %0, [%1];" : "=r"(r) : "l"(p) : "memory");
	return (uint8_t)r;
}
__device__ __forceinline__ uint32_t ld_cg32(const void *p)
{
	uint32_t r;
	asm volatile("ld.global.cg.u32 %0, [%1];" : "=r"(r) : "l"(p) : "memory");
	return r;
}

__device__ __forceinline__ uint16_t be16(const uint8_t *p) { return (uint16_t)(p[0] << 8 | p[1]); }
__device__ __forceinline__ uint32_t be32(const uint8_t *p)
{
	return (uint32_t)p[0] << 24 | (uint32_t)p[1] << 16 | (uint32_t)p[2] << 8 | p[3];
}
__device__ __forceinline__ uint64_t be64(const uint8_t *p) { return (uint64_t)be32(p) << 32 | be32(p + 4); }

/* byte-granular SG element (SURVEY.md §7 "unaligned SG elements"): peel to a 16-byte aligned destination, then
 * aligned 16-byte stores.  A source that is misaligned against the destination by m bytes is read as the two
 * ALIGNED 16-byte vectors that straddle each output vector and realigned in registers with funnel shifts
 * (the second vector is the neighbour lane's first: an L2 hit, DRAM traffic stays 1x).  Aligned vectors never
 * cross a page, and each one read holds at least one byte of the element, so the over-read of up to 15 bytes on
 * either side stays inside mapped memory and is never stored. */
__device__ __forceinline__ int4 realign16(const int4 &a, const int4 &b, uint32_t m)
{
	const uint32_t r = (m & 3) * 8;
	uint32_t w0, w1, w2, w3, w4;
	switch (m >> 2) {
	case 0: w0 = a.x; w1 = a.y; w2 = a.z; w3 = a.w; w4 = b.x; break;
	case 1: w0 = a.y; w1 = a.z; w2 = a.w; w3 = b.x; w4 = b.y; break;
	case 2: w0 = a.z; w1 = a.w; w2 = b.x; w3 = b.y; w4 = b.z; break;
	default: w0 = a.w; w1 = b.x; w2 = b.y; w3 = b.z; w4 = b.w; break;
	}
	return make_int4(__funnelshift_r(w0, w1, r), __funnelshift_r(w1, w2, r), __funnelshift_r(w2, w3, r), __funnelshift_r(w3, w4, r));
}

__device__ __forceinline__ void move_unit_unaligned(uint8_t *dst, const uint8_t *src, uint32_t n, int lane)
{
	/* loads of a half-unit are issued before its first store (a warp issues in order: a store waiting for its data
	 * holds back the loads behind it).  Two halves of 4 vectors per lane, not one of 8 as in the fast path: the
	 * 9 x 4 registers of a whole realigned unit made the mover loop spill, which slows every path. */
	uint32_t head = (uint32_t)((16 - ((uintptr_t)dst & 15)) & 15);
	if (head > n) head = n;
	uint8_t hb = 0, tb = 0;
	if ((uint32_t)lane < head) hb = ld_cg8(src + lane);
	uint8_t *const dst0 = dst;
	dst += head; src += head; n -= head;
	const uint32_t nv = n >> 4;	/* <= 256 output vectors, vector v = lane + 32 k */
	const uint32_t tail = n & 15;
	if ((uint32_t)lane < tail) tb = ld_cg8(src + (size_t)nv * 16 + lane);
	const uint32_t m = (uint32_t)((uintptr_t)src & 15);
	constexpr int H = 4;
	if (m == 0) {
#pragma unroll
		for (int h = 0; h < 2; h++) {
			int4 r[H];
#pragma unroll
			for (int k = 0; k < H; k++) {
				const uint32_t v = lane + 32 * (h * H + k);
				if (v < nv) r[k] = ld_cg16(src + (size_t)v * 16);
			}
			if (h == 0 && (uint32_t)lane < head) dst0[lane] = hb;
#pragma unroll
			for (int k = 0; k < H; k++) {
				const uint32_t v = lane + 32 * (h * H + k);
				if (v < nv) st_cg16(dst + (size_t)v * 16, r[k]);
			}
		}
	} else {
		/* aligned source vector i (at sa + 16 i) is needed for i <= nv; output vector v = realign(i = v, i = v + 1).
		 * Lane l holds i = l + 32 k; its right neighbour is lane l + 1's, and for lane 31 lane 0's next one. */
		const uint8_t *sa = src - m;
#pragma unroll
		for (int h = 0; h < 2; h++) {
			int4 a[H + 1];
#pragma unroll
			for (int k = 0; k <= H; k++) {
				const uint32_t i = lane + 32 * (h * H + k);
				if (i <= nv && (k < H || lane == 0)) a[k] = ld_cg16(sa + (size_t)i * 16);
			}
			if (h == 0 && (uint32_t)lane < head) dst0[lane] = hb;
#pragma unroll
			for (int k = 0; k < H; k++) {
				const uint32_t v = lane + 32 * (h * H + k);
				int4 b;
				b.x = __shfl_down_sync(0xffffffffu, a[k].x, 1); b.y = __shfl_down_sync(0xffffffffu, a[k].y, 1);
				b.z = __shfl_down_sync(0xffffffffu, a[k].z, 1); b.w = __shfl_down_sync(0xffffffffu, a[k].w, 1);
				const int nx = __shfl_sync(0xffffffffu, a[k + 1].x, 0), ny = __shfl_sync(0xffffffffu, a[k + 1].y, 0);
				const int nz = __shfl_sync(0xffffffffu, a[k + 1].z, 0), nw = __shfl_sync(0xffffffffu, a[k + 1].w, 0);
				if (lane == 31) b = make_int4(nx, ny, nz, nw);
				if (v < nv) st_cg16(dst + (size_t)v * 16, realign16(a[k], b, m));
			}
		}
	}
	if ((uint32_t)lane < tail) dst[(size_t)nv * 16 + lane] = tb;
}

/* the compact form of the same (one vector at a time, byte loads when the source disagrees with the destination modulo
 * 4): the mirror kernels use it - they are bound by NVLink at a fraction of the HBM rate, and the batched path above,
 * inlined or called, slows them through spills around it */
__device__ __forceinline__ void move_unit_unaligned_compact(uint8_t *dst, const uint8_t *src, uint32_t n, int lane)
{
	uint32_t head = (uint32_t)((16 - ((uintptr_t)dst & 15)) & 15);
	if (head > n) head = n;
	if ((uint32_t)lane < head) dst[lane] = ld_cg8(src + lane);
	dst += head; src += head; n -= head;
	const uint32_t nv = n >> 4;
	if (((uintptr_t)src & 15) == 0) {
		for (uint32_t v = lane; v < nv; v += 32) st_cg16(dst + (size_t)v * 16, ld_cg16(src + (size_t)v * 16));
	} else {
		for (uint32_t v = lane; v < nv; v += 32) {
			const uint8_t *sp = src + (size_t)v * 16;
			uint32_t w[4];
#pragma unroll
			for (int j = 0; j < 4; j++) {
				w[j] = (uint32_t)ld_cg8(sp + 4 * j) | (uint32_t)ld_cg8(sp + 4 * j + 1) << 8 |
				       (uint32_t)ld_cg8(sp + 4 * j + 2) << 16 | (uint32_t)ld_cg8(sp + 4 * j + 3) << 24;
			}
			st_cg16(dst + (size_t)v * 16, make_int4(w[0], w[1], w[2], w[3]));
		}
	}
	const uint32_t tail = n & 15;
	if ((uint32_t)lane < tail) dst[(size_t)nv * 16 + lane] = ld_cg8(src + (size_t)nv * 16 + lane);
}

/* Move `n` (<= kUnitBytes) bytes with one warp.  Fast path: both sides 16-byte aligned.
 * dst2 != nullptr (mirrored bdev, same alignment as dst): the registers are stored twice, locally
 * and into the peer replica over NVLink - one load, two stores, no second pass. */
template <bool kCompactSlowPath = false>	/* mirror kernels: the compact byte-granular path */
__device__ __forceinline__ void move_unit(uint8_t *dst, const uint8_t *src, uint32_t n, int lane, uint8_t *dst2 = nullptr)
{
	if ((((uintptr_t)dst | (uintptr_t)src | n) & 15) == 0) {
		int4 r[kUnitBytes / 512];
		const uint32_t nv = n >> 4;
#pragma unroll
		for (int k = 0; k < (int)(kUnitBytes / 512); k++) {
			uint32_t v = lane + 32 * k;
			if (v < nv) r[k] = ld_cg16(src + (size_t)v * 16);
		}
#pragma unroll
		for (int k = 0; k < (int)(kUnitBytes / 512); k++) {
			uint32_t v = lane + 32 * k;
			if (v < nv) st_cg16(dst + (size_t)v * 16, r[k]);
		}
		if (dst2) {
#pragma unroll
			for (int k = 0; k < (int)(kUnitBytes / 512); k++) {
				uint32_t v = lane + 32 * k;
				if (v < nv) st_cg16(dst2 + (size_t)v * 16, r[k]);
			}
		}
		return;
	}
	if constexpr (kCompactSlowPath) {
		move_unit_unaligned_compact(dst, src, n, lane);
		if (dst2) move_unit_unaligned_compact(dst2, src, n, lane);
	} else {
		move_unit_unaligned(dst, src, n, lane);
	}
}

/* mem_copy_fill with fill == 0 (copy_engine.c:128-140): zero `n` bytes; block-aligned by construction */
__device__ __forceinline__ void zero_unit(uint8_t *dst, uint32_t n, int lane)
{
	const int4 z = make_int4(0, 0, 0, 0);
	if ((((uintptr_t)dst | n) & 15) == 0) {
		for (uint32_t v = lane; v < (n >> 4); v += 32) st_cg16(dst + (size_t)v * 16, z);
	} else {
		for (uint32_t i = lane; i < n; i += 32) dst[i] = 0;
	}
}


/* spdk_scsi_task_scatter_data (task.c:111-152) of a <=36-byte control payload into the SG list */
__device__ __forceinline__ void set_check(LaneState &s, uint8_t sk, uint8_t asc)
{
	s.status = SC_CHECK; s.sk = sk; s.asc = asc;
}

__device__ inline int scatter_small(const QueueDesc &q, const oimgpu_req &r, uint32_t iovcnt, uint32_t total_len,
				    const uint8_t *buf, uint32_t buf_len, LaneState &st)
{
	if (buf_len == 0) return 0;
	if (total_len < buf_len) {
		set_check(st, SK_ILLEGAL_REQUEST, ASC_INVALID_FIELD);
		return -1;
	}
	uint32_t left = buf_len;
	for (uint32_t j = 0; j < iovcnt && left; j++) {
		const oimgpu_iov v = q.iovs[(r.iov_start + j) & q.iov_mask];
		uint32_t l = v.len < left ? v.len : left;
		uint8_t *d = (uint8_t *)(uintptr_t)v.addr;
		for (uint32_t k = 0; k < l; k++) d[k] = buf[buf_len - left + k];
		left -= l;
	}
	return (int)buf_len;
}

/* byte `pos` of the request's gathered TO_DEV payload (spdk_scsi_task_gather_data, task.c:154-186) */
__device__ inline uint8_t gather_byte(const QueueDesc &q, const oimgpu_req &r, uint32_t iovcnt, uint32_t pos)
{
	for (uint32_t j = 0; j < iovcnt; j++) {
		const oimgpu_iov v = q.iovs[(r.iov_start + j) & q.iov_mask];
		if (pos < v.len) return ld_cg8((const uint8_t *)(uintptr_t)v.addr + pos);
		pos -= v.len;
	}
	return 0;
}

}  // namespace oimgpu
