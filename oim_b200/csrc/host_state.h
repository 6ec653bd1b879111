/*
 * host_state.h - what the host-side files of liboimgpu.so (control.cu, session.cu, nbd.cu, copy_chan.cu, bio_chan.cu,
 * mirror_check.cu) share:
 * the registry, the session, and the helpers more than one of them calls.  Internal, not installed.
 */
#pragma once

#include <cuda_runtime.h>

#include <algorithm>
#include <cerrno>
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "lun_kernel.cuh"

#define CU_OK(expr)                                                                          \
	do {                                                                                 \
		cudaError_t e__ = (expr);                                                    \
		if (e__ != cudaSuccess) {                                                    \
			fprintf(stderr, "oimgpu: %s failed: %s (%s:%d)\n", #expr,             \
				cudaGetErrorString(e__), __FILE__, __LINE__);                 \
			return e__ == cudaErrorMemoryAllocation ? -ENOMEM : -EIO;            \
		}                                                                            \
	} while (0)

namespace oimgpu {

struct Device {
	int ordinal = -1;
	int sm_count = 0;
	uint64_t bytes_allocated = 0;
	/* housekeeping (zero-fill, raw store access) runs here, never on the legacy stream and never behind
	 * a cudaDeviceSynchronize: a resident poller kernel would make either wait for its watchdog */
	cudaStream_t util = nullptr;
};

struct Bdev {
	std::string name, product, uuid;
	std::string pool_name, rbd_name, user_id;	/* construct_rbd_bdev parameters, kept for the config dump */
	uint64_t num_blocks = 0;
	uint32_t block_size = 0;
	int claimed = 0;	/* number of SCSI targets built on it */
	int open_luns = 0;	/* oimgpu_lun handles */
	int nbd_exports = 0;	/* oimgpu_nbd_serve calls serving it (also counted in open_luns) */
	std::vector<int> devices;	/* replica r lives on devices[r] (an imported replica: the device it is reached from) */
	std::vector<uint8_t *> stores;
	std::vector<char> imported;	/* replica r is another process's store, opened from a CUDA IPC handle */
	std::vector<std::string> ipc_handles;	/* the handles the imported replicas were opened from, in replica order (config dump) */
	unsigned long long *hist = nullptr;	/* enable_bdev_histogram: kHistBuckets counters on devices[0] */
	unsigned long long retired[12] = {};	/* counters of sessions that are gone (same layout as LunCtx::stats) */
};

struct Ctrlr {
	std::string name, cpumask;
	uint32_t delay_base_us = 0;			/* interrupt coalescing (vhost.c:270-377) */
	uint32_t iops_threshold = 60000;		/* SPDK_VHOST_VQ_IOPS_COALESCING_THRESHOLD */
	std::string targets[OIMGPU_CTRLR_MAX_DEVS];	/* bdev name or "" */
	int scsi_id[OIMGPU_CTRLR_MAX_DEVS] = {};	/* spdk_scsi_dev.id: slot in the global device table */
};

struct Registry {
	std::mutex mu;
	bool inited = false;
	bool control_only = false;	/* wire-protocol testing without a GPU: no stores, no data path */
	std::vector<Device> devices;
	std::map<std::string, std::unique_ptr<Bdev>> bdevs;
	std::map<std::string, std::unique_ptr<Ctrlr>> ctrlrs;
	std::vector<std::string> bdev_order, ctrlr_order;	/* registration order, as SPDK's TAILQs list them */
	bool scsi_slot_used[1024] = {};	/* g_spdk_scsi.dev[SPDK_SCSI_MAX_DEVS]: ids are the lowest free slot (S/lib/scsi/dev.c:49-66) */
	std::string socket_dir;		/* vhost -S <dir>: prefix of controller socket paths (vhost.c:1185-1205) */
	unsigned long long app_core_mask = 0x1;	/* spdk_app_get_core_mask(): default -m 0x1 */
	int malloc_disk_count = 0;	/* bdev_malloc.c:93 */
	int rbd_count = 0;
	std::map<void *, size_t> registered;
	int open_luns = 0;
	std::vector<oimgpu_lun *> handles;	/* open data-path sessions: told about target hot-plug */
};

extern Registry g;

struct Queue {
	/* library-owned ring in mapped pinned host memory (OIMGPU_MEM_HOST submissions) */
	oimgpu_req *h_reqs = nullptr;
	oimgpu_iov *h_iovs = nullptr;
	oimgpu_cpl *h_cpls = nullptr;
	oimgpu_req *d_reqs = nullptr;	/* device view of the same memory */
	oimgpu_iov *d_iovs = nullptr;
	oimgpu_cpl *d_cpls = nullptr;
	uint32_t tail = 0;		/* next free slot (absolute index) */
	uint32_t kicked = 0;		/* slots [reaped, kicked) handed to the GPU */
	uint32_t reaped = 0;
	uint32_t iov_tail = 0;
	/* pending OIMGPU_MEM_DEVICE submission (caller-owned device arrays), consumed by next kick */
	const oimgpu_req *dev_reqs = nullptr;
	const oimgpu_iov *dev_iovs = nullptr;
	oimgpu_cpl *dev_cpls = nullptr;
	uint32_t dev_count = 0;
	uint32_t dev_iov_limit = 0;	/* entries in dev_iovs (0: caller vouches for the indices) */
	/* attached virtio split ring (virtqueue mode) */
	const uint8_t *vq_desc = nullptr, *vq_avail = nullptr;
	uint8_t *vq_used = nullptr;
	uint32_t vq_size = 0;
	bool vq_pending = false;
	bool vq_in_hbm = false;		/* the used ring is device memory (a guest image in HBM), not pinned host memory */
};

int find_device_slot(int ordinal);
bool device_reachable(int from, int to);
std::string ctrlr_key(const char *ctrlr);
Bdev *find_bdev_locked(const char *name);	/* nullptr: no such bdev */
Ctrlr *find_ctrlr_locked(const char *ctrlr);	/* by ctrlr_key(ctrlr); nullptr: no such controller */
bool read_ctx_stats(int device, const LunCtx *d_ctx, unsigned long long out[12]);
void iostat_from_stats(const unsigned long long stats[12], oimgpu_iostat *out);
void refresh_ctrlr_sessions_locked(const std::string &ctrlr);
int publish_replica_locked(const std::string &bdev, int replica, uint8_t *store);	/* every LunCtx of the bdev */
cudaError_t launch_copy(cudaStream_t st, int sm_count, void *dst, const void *src, uint64_t nbytes);
cudaError_t launch_fill(cudaStream_t st, int sm_count, void *dst, uint8_t fill, uint64_t nbytes);
void unpin_all_host_ranges();	/* oimgpu_mem_ensure's registrations */
bool host_range_pinned(const void *addr, size_t len);	/* inside one range the library pinned or registered (no driver call) */
int pin_host_pages(const void *addr, size_t len);	/* pin what of the pages is not pinned yet; -EFAULT */

}  // namespace oimgpu

using namespace oimgpu;

static_assert(sizeof(oimgpu_req) == 64, "oimgpu_req layout");
static_assert(sizeof(oimgpu_iov) == 16, "oimgpu_iov layout");
static_assert(sizeof(oimgpu_cpl) == 48, "oimgpu_cpl layout");
static_assert(offsetof(oimgpu_req, cdb) == 19 && offsetof(oimgpu_req, dir) == 51, "virtio header prefix");
static_assert(sizeof(Segment) == 32, "Segment layout");

struct oimgpu_lun {
	/* a session is driven by one thread (its owner); the exception is target hot-plug, which reaches
	 * into it from whichever thread runs the control call: the entry points both sides use lock this */
	std::recursive_mutex mu;
	std::string ctrlr, bdev;
	int target = 0;
	int device = 0;
	int sm_count = 0;
	cudaStream_t stream = nullptr;
	cudaEvent_t done = nullptr;
	LunCtx *d_ctx = nullptr;
	LunCtx h_ctx{};
	uint32_t num_queues = 0, queue_size = 0, iov_cap = 0;
	std::vector<Queue> queues;
	/* pinned staging ring for {KickHeader, QueueDesc[]}: a slot is reused only after its upload ran */
	static constexpr int kKickSlots = 4;
	uint8_t *h_kick[kKickSlots] = {};
	cudaEvent_t kick_ev[kKickSlots] = {};
	uint64_t kicks = 0;
	uint8_t *d_kick = nullptr;
	QueueDesc *d_desc = nullptr;
	QShare *d_share = nullptr;		/* [3 x num_queues] coordination blocks of shared queues (lun_kernel.cuh) */
	/* the session's recent read / write mix: LunCtx::mix, copied here (pinned) behind every launch */
	volatile unsigned long long *h_mix = nullptr;
	unsigned long long mix_seen[2] = {0, 0};
	bool write_hot = false;
	uint64_t shared_launches = 0;
	uint64_t launches = 0;
	int grid_cap = 0;
	/* staged batch path (oimgpu_submit_batch with host arrays): metadata is uploaded by the copy
	 * engine and the kernel runs on HBM-resident request/SG/completion arrays, so only payload is
	 * touched over PCIe by the SMs (tools/e2e_probe.py compares the two) */
	oimgpu_req *bs_d_reqs = nullptr;
	oimgpu_iov *bs_d_iovs = nullptr;
	oimgpu_cpl *bs_d_cpls = nullptr;
	uint8_t *bs_h_pin = nullptr;		/* pinned bounce buffer for pageable caller arrays */
	size_t bs_cap_reqs = 0, bs_cap_iovs = 0, bs_h_cap = 0;
	oimgpu_cpl *bs_user_cpls = nullptr;	/* pending copy-out at wait time */
	const oimgpu_cpl *bs_h_cpls = nullptr;
	size_t bs_pending = 0;
	cudaStream_t copy_stream = nullptr;
	/* persistent poller */
	struct Door { volatile uint32_t tail; uint32_t pad0[15]; volatile uint32_t done; uint32_t pad1[15]; };
	Door *h_door = nullptr, *d_door = nullptr;	/* mapped pinned: one doorbell/completion-count pair per queue */
	volatile uint32_t *h_flags = nullptr;	/* mapped pinned: [0] stop, [16] exited */
	uint32_t *d_flags = nullptr;
	bool poller_active = false;
	uint32_t poller_grid = 0;
	uint32_t poller_max_ctas = 0, poller_idle_ms = 0;	/* as given to start_poller: reused when a hot-unplug restarts it */
	/* the other SCSI devices of the controller, reachable through the same queues (LunCtx::peer) */
	LunCtx *d_peer[OIMGPU_CTRLR_MAX_DEVS] = {};
	std::string peer_bdev[OIMGPU_CTRLR_MAX_DEVS];
	bool any_mirror = false;
	VqState *d_vq_state = nullptr;		/* [num_queues] ring cursors */
	oimgpu_iov *d_iov_scratch = nullptr;	/* [grid_cap][32][kIovRow] SG rows built by the parser lanes */
	uint8_t *slab = nullptr;		/* the mapped pinned slab the per-queue rings are carved from */
};

/* cudaFree waits for the whole device, and a resident poller kernel never finishes on its own: park
 * the pollers of that GPU around a free and bring them back afterwards.  Every session of the GPU is
 * held (its mutex taken) for the duration, so that none can start a resident kernel in the window -
 * their owners' calls simply wait.  Caller holds g.mu; sessions never take g.mu while holding their own
 * mutex, so the order g.mu -> session mutex is safe.  The pollers stay parked for the scope's lifetime. */
struct ParkedPollers {
	/* device < 0: every GPU (pinned host memory is mapped into all of them) */
	explicit ParkedPollers(int device, oimgpu_lun *except = nullptr)
	{
		park([&](const oimgpu_lun *L) { return L != except && (device < 0 || L->device == device); });
	}
	/* every session on GPU `device`, and every session that reaches bdev `bdev` (its own device or a peer target) */
	ParkedPollers(int device, const std::string &bdev)
	{
		park([&](const oimgpu_lun *L) {
			if (L->device == device || L->bdev == bdev) return true;
			for (const std::string &p : L->peer_bdev) if (p == bdev) return true;
			return false;
		});
	}
	~ParkedPollers()
	{
		for (const Session &p : parked) {
			if (p.restart) oimgpu_lun_start_poller(p.L, p.L->poller_max_ctas, p.L->poller_idle_ms);
			p.L->mu.unlock();
		}
	}
	ParkedPollers(const ParkedPollers &) = delete;
	ParkedPollers &operator=(const ParkedPollers &) = delete;

	struct Session { oimgpu_lun *L; bool restart; };
	std::vector<Session> parked;

private:
	template <class Want> void park(Want want)
	{
		for (oimgpu_lun *L : g.handles) {
			if (!want(L)) continue;
			L->mu.lock();
			const bool was = L->poller_active;
			if (was) oimgpu_lun_stop_poller(L);
			parked.push_back({L, was});
		}
	}
};

