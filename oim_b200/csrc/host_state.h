/*
 * host_state.h - what the host-side files of liboimgpu.so (control.cu, session.cu, nbd.cu, copy_chan.cu, bio_chan.cu,
 * mirror_check.cu) share: the registry, the session, the helpers more than one of them calls, the Buf that owns device and
 * pinned memory and frees it only under a ParkedPollers scope, and the channels' EventFifo.  Internal, not installed.
 */
#pragma once

#include <cuda_runtime.h>

#include <algorithm>
#include <cerrno>
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <deque>
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

struct ParkedPollers;
constexpr int kAllGpus = -1, kNoGpu = -2;	/* ParkedPollers devices besides one GPU's ordinal */

/* Device memory (cudaMalloc) or pinned host memory (cudaHostAlloc, plain or mapped) of the library: pointer, element count
 * and GPU.  Freeing it waits for that GPU (pinned: every GPU), so it is freed only under a ParkedPollers scope that covers
 * them, which release() checks.  A failed allocation leaves it empty.  It never frees itself: memory still held when it
 * is destroyed stays with the process (the registry's, at exit without oimgpu_fini). */
enum class Mem { Device, Pinned, Mapped };

template <class T, Mem K> class Buf {
public:
	Buf() = default;
	Buf(Buf &&o) noexcept : p_(o.p_), n_(o.n_), device_(o.device_) { o.p_ = nullptr; o.n_ = 0; }
	T *get() const { return p_; }
	T &operator[](size_t i) const { return p_[i]; }
	explicit operator bool() const { return p_ != nullptr; }
	size_t size() const { return n_; }
	/* the GPUs whose pollers a free waits for, as a ParkedPollers device */
	int waits_for() const { return !p_ ? kNoGpu : K == Mem::Device ? device_ : kAllGpus; }
	/* n elements on GPU `device`, into an empty buffer (a live one would have to be freed without a scope) */
	cudaError_t alloc(int device, size_t n)
	{
		release(nullptr);
		cudaError_t e = cudaSetDevice(device);
		if (e == cudaSuccess) e = K == Mem::Device ? cudaMalloc((void **)&p_, n * sizeof(T))
							   : cudaHostAlloc((void **)&p_, n * sizeof(T), K == Mem::Mapped ? cudaHostAllocMapped : cudaHostAllocDefault);
		if (e != cudaSuccess) {
			(void)cudaGetLastError();	/* a refusal must not surface at a later launch check */
			p_ = nullptr;
			return e;
		}
		n_ = n;
		device_ = device;
		return e;
	}
	/* at least n elements: a smaller buffer is freed under `parked` and replaced (contents are not kept) */
	cudaError_t grow(int device, size_t n, const ParkedPollers &parked)
	{
		if (n <= n_) return cudaSuccess;
		release(&parked);
		return alloc(device, n);
	}
	void reset(const ParkedPollers &parked) { release(&parked); }
private:
	void release(const ParkedPollers *parked);
	T *p_ = nullptr;
	size_t n_ = 0;
	int device_ = -1;
};

/* A channel's work in stream order: each piece's payload (a tag, a batch of completions) and the event recorded behind it.
 * Finished entries leave at the front; events are reused, and destroyed with the FIFO once the stream has drained. */
template <class P> struct EventFifo {
	struct Entry { cudaEvent_t ev; P payload; };
	std::deque<Entry> entries;
	std::vector<cudaEvent_t> spare;
	unsigned long long recorded = 0;
	EventFifo() = default;
	EventFifo(const EventFifo &) = delete;
	~EventFifo()
	{
		for (auto &e : entries) cudaEventDestroy(e.ev);
		for (auto ev : spare) cudaEventDestroy(ev);
	}
	int record(cudaStream_t st, P payload)
	{
		cudaEvent_t ev;
		if (!spare.empty()) { ev = spare.back(); spare.pop_back(); }
		else CU_OK(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
		CU_OK(cudaEventRecord(ev, st));
		entries.push_back({ev, std::move(payload)});
		recorded++;
		return 0;
	}
	/* Up to max results from finished entries, oldest first: take(payload, n) adds its results at n, and returns
	 * false to keep an entry it could not finish.  The count, or -EIO when an entry's work failed. */
	template <class Take> int poll(int max, Take take)
	{
		int n = 0;
		while (n < max && !entries.empty()) {
			const cudaError_t e = cudaEventQuery(entries.front().ev);
			if (e == cudaErrorNotReady) { (void)cudaGetLastError(); break; }
			if (e != cudaSuccess) { (void)cudaGetLastError(); return -EIO; }
			if (!take(entries.front().payload, n)) break;
			spare.push_back(entries.front().ev);
			entries.pop_front();
		}
		return n;
	}
};

struct Device {
	int ordinal = -1;
	int sm_count = 0;
	uint64_t bytes_allocated = 0;
	/* housekeeping (zero-fill, raw store access) runs here, never on the legacy stream and never behind
	 * a cudaDeviceSynchronize: a resident poller kernel would make either wait for its watchdog */
	cudaStream_t util = nullptr;
};

struct Replica {
	int device = -1;	/* the GPU the store lives on (an imported store: the GPU it is reached from) */
	uint8_t *store = nullptr;
	bool imported = false;	/* another process's store, opened from a CUDA IPC handle */
	std::string ipc_handle;	/* the handle an imported store was opened from (config dump) */
};

struct Bdev {
	std::string name, product, uuid;
	std::string pool_name, rbd_name, user_id;	/* construct_rbd_bdev parameters, kept for the config dump */
	uint64_t num_blocks = 0;
	uint32_t block_size = 0;
	int opens = 0;		/* open_bdev_locked: session targets (own and peer), NBD exports, bio channels */
	int nbd_exports = 0;	/* oimgpu_nbd_serve calls serving it (also counted in opens) */
	std::vector<Replica> replicas;
	Buf<unsigned long long, Mem::Device> hist;	/* enable_bdev_histogram: kHistBuckets counters on replica 0's GPU */
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
/* A use of a bdev by a session target (its own or a peer), an NBD export or a bio channel begins or ends.  A bdev in
 * use is not deleted, and its disabled histogram reads as -EFAULT.  Caller holds g.mu. */
void open_bdev_locked(Bdev &b);
void close_bdev_locked(const std::string &name);	/* a bdev no longer registered is ignored */
Ctrlr *find_ctrlr_locked(const char *ctrlr);	/* by ctrlr_key(ctrlr); nullptr: no such controller */
bool read_ctx_stats(int device, const LunCtx *d_ctx, unsigned long long out[12]);
void iostat_from_stats(const unsigned long long stats[12], oimgpu_iostat *out);
void refresh_ctrlr_sessions_locked(const std::string &ctrlr);
int publish_ctx_locked(const std::string &bdev, size_t offset, const void *value, size_t len);	/* every LunCtx of the bdev */
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
	Buf<LunCtx, Mem::Device> d_ctx;
	LunCtx h_ctx{};
	uint32_t num_queues = 0, queue_size = 0, iov_cap = 0;
	std::vector<Queue> queues;
	/* pinned staging ring for {KickHeader, QueueDesc[]}: a slot is reused only after its upload ran */
	static constexpr int kKickSlots = 4;
	Buf<uint8_t, Mem::Pinned> h_kick[kKickSlots];
	cudaEvent_t kick_ev[kKickSlots] = {};
	uint64_t kicks = 0;
	Buf<uint8_t, Mem::Device> d_kick;
	QueueDesc *d_desc = nullptr;
	Buf<QShare, Mem::Device> d_share;	/* [3 x num_queues] coordination blocks of shared queues (lun_kernel.cuh) */
	/* the session's recent read / write mix: LunCtx::mix, copied here (pinned) behind every launch */
	Buf<volatile unsigned long long, Mem::Pinned> h_mix;
	unsigned long long mix_seen[2] = {0, 0};
	bool write_hot = false;
	uint64_t shared_launches = 0;
	uint64_t launches = 0;
	int grid_cap = 0;
	/* staged batch path (oimgpu_submit_batch with host arrays): metadata is uploaded by the copy
	 * engine and the kernel runs on HBM-resident request/SG/completion arrays, so only payload is
	 * touched over PCIe by the SMs (tools/e2e_probe.py compares the two) */
	Buf<oimgpu_req, Mem::Device> bs_d_reqs;
	Buf<oimgpu_iov, Mem::Device> bs_d_iovs;
	Buf<oimgpu_cpl, Mem::Device> bs_d_cpls;
	Buf<uint8_t, Mem::Pinned> bs_h_pin;	/* bounce buffer for pageable caller arrays */
	oimgpu_cpl *bs_user_cpls = nullptr;	/* pending copy-out at wait time */
	const oimgpu_cpl *bs_h_cpls = nullptr;
	size_t bs_pending = 0;
	cudaStream_t copy_stream = nullptr;
	/* persistent poller */
	struct Door { volatile uint32_t tail; uint32_t pad0[15]; volatile uint32_t done; uint32_t pad1[15]; };
	Buf<Door, Mem::Mapped> h_door;		/* one doorbell/completion-count pair per queue */
	Door *d_door = nullptr;
	Buf<volatile uint32_t, Mem::Mapped> h_flags;	/* [0] stop, [16] exited */
	uint32_t *d_flags = nullptr;
	bool poller_active = false;
	uint32_t poller_grid = 0;
	uint32_t poller_max_ctas = 0, poller_idle_ms = 0;	/* as given to start_poller: reused when a hot-unplug restarts it */
	/* the other SCSI devices of the controller, reachable through the same queues (LunCtx::peer) */
	Buf<LunCtx, Mem::Device> d_peer[OIMGPU_CTRLR_MAX_DEVS];
	std::string peer_bdev[OIMGPU_CTRLR_MAX_DEVS];
	bool any_mirror = false;
	Buf<VqState, Mem::Device> d_vq_state;	/* [num_queues] ring cursors */
	Buf<oimgpu_iov, Mem::Device> d_iov_scratch;	/* [grid_cap][32][kIovRow] SG rows built by the parser lanes */
	Buf<uint8_t, Mem::Mapped> slab;	/* the slab the per-queue rings are carved from */
};

/* Visit the device-resident LunCtxs of session L with the name of the bdev each serves: its own context (passed with
 * its host copy h_ctx) and then the peer-target contexts of a controller-wide view (passed with nullptr).  Stops at
 * the first visit that returns nonzero and returns that.  Caller holds g.mu, under which the peers change. */
template <class Visit> int for_each_ctx(oimgpu_lun *L, Visit visit)
{
	if (!L->bdev.empty()) {
		if (int rc = visit(L->bdev, L->d_ctx.get(), &L->h_ctx)) return rc;
	}
	for (int t = 0; t < OIMGPU_CTRLR_MAX_DEVS; t++) {
		if (L->peer_bdev[t].empty()) continue;
		if (int rc = visit(L->peer_bdev[t], L->d_peer[t].get(), (LunCtx *)nullptr)) return rc;
	}
	return 0;
}

namespace oimgpu {

/* cudaFree, cudaFreeHost and cudaHostUnregister wait for the GPU, and a resident poller kernel never finishes on its
 * own: park the pollers of that GPU around a free and bring them back afterwards.  Every session of the GPU is
 * held (its mutex taken) for the duration, so that none can start a resident kernel in the window -
 * their owners' calls simply wait.  Caller holds g.mu; sessions never take g.mu while holding their own
 * mutex, so the order g.mu -> session mutex is safe.  The pollers stay parked for the scope's lifetime. */
struct ParkedPollers {
	/* device: one GPU, kAllGpus (pinned host memory is mapped into all of them) or kNoGpu */
	explicit ParkedPollers(int device, oimgpu_lun *except = nullptr) : gpu(device)
	{
		park([&](oimgpu_lun *L) { return L != except && (device == kAllGpus || L->device == device); });
	}
	/* every session on GPU `device`, and every session that reaches bdev `bdev` (its own target or a peer target) */
	ParkedPollers(int device, const std::string &bdev) : gpu(device)
	{
		park([&](oimgpu_lun *L) {
			return L->device == device ||
			       for_each_ctx(L, [&](const std::string &name, LunCtx *, LunCtx *) { return (int)(name == bdev); });
		});
	}
	/* wait for everything the held sessions launched: with their pollers parked, nothing is added behind it */
	int drain()
	{
		for (const Session &p : parked) {
			CU_OK(cudaSetDevice(p.L->device));
			CU_OK(cudaStreamSynchronize(p.L->stream));
		}
		return 0;
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
	const int gpu;	/* as constructed: a Buf checks it before it frees */

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

template <class T, Mem K> void Buf<T, K>::release(const ParkedPollers *parked)
{
	if (!p_) return;
	if (!parked || (parked->gpu != kAllGpus && parked->gpu != waits_for())) {
		fprintf(stderr, "oimgpu: internal error: memory freed outside a ParkedPollers scope that covers its GPUs\n");
		abort();
	}
	cudaSetDevice(device_);
	if (K == Mem::Device) cudaFree((void *)p_);
	else cudaFreeHost((void *)p_);
	(void)cudaGetLastError();
	p_ = nullptr;
	n_ = 0;
}

}  // namespace oimgpu
