/*
 * oimgpu.cu — host side of liboimgpu.so: the C ABI declared in include/oimgpu.h.
 *
 * Control plane state mirrors what the SPDK daemon keeps for OIM's twelve RPCs
 * (bdev list: S/lib/bdev/bdev.c + bdev_malloc.c:378-443; vhost controllers and their 8 target
 * slots: S/lib/vhost/vhost_scsi.c:951-1103), the data plane launches oim_lun_queue_kernel on the
 * LUN's own CUDA stream.  There is deliberately no CPU implementation of the data path in this
 * library: without a usable CUDA device oimgpu_init() fails and every other call returns -ENODEV.
 */
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <cerrno>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <map>
#include <memory>
#include <mutex>
#include <random>
#include <string>
#include <vector>

#include <sys/socket.h>
#include <unistd.h>

#include "lun_kernel.cuh"

namespace oimgpu {
__global__ void oim_copy_kernel(uint8_t *dst, const uint8_t *src, uint64_t nbytes);
__global__ void oim_fill_kernel(uint8_t *dst, uint8_t fill, uint64_t nbytes);
}  // namespace oimgpu

using namespace oimgpu;

static_assert(sizeof(oimgpu_req) == 64, "oimgpu_req layout");
static_assert(sizeof(oimgpu_iov) == 16, "oimgpu_iov layout");
static_assert(sizeof(oimgpu_cpl) == 48, "oimgpu_cpl layout");
static_assert(offsetof(oimgpu_req, cdb) == 19 && offsetof(oimgpu_req, dir) == 51, "virtio header prefix");
static_assert(sizeof(Segment) == 32, "Segment layout");

#define CU_OK(expr)                                                                          \
	do {                                                                                 \
		cudaError_t e__ = (expr);                                                    \
		if (e__ != cudaSuccess) {                                                    \
			fprintf(stderr, "oimgpu: %s failed: %s (%s:%d)\n", #expr,             \
				cudaGetErrorString(e__), __FILE__, __LINE__);                 \
			return e__ == cudaErrorMemoryAllocation ? -ENOMEM : -EIO;            \
		}                                                                            \
	} while (0)

struct oimgpu_lun;

namespace {

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
	std::vector<int> devices;	/* replica r lives on devices[r] (an imported replica: the device it is reached from) */
	std::vector<uint8_t *> stores;
	std::vector<char> imported;	/* replica r is another process's store, opened from a CUDA IPC handle */
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

Registry g;

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

}  // namespace

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
	cudaEvent_t bs_uploaded = nullptr;
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

/* ---------------------------------------------------------------------------------------------- */

/* Small host->device updates of a session's state.  A plain cudaMemcpy from pageable memory may return
 * before the DMA has landed, and it runs on the legacy stream, which the sessions' non-blocking streams do
 * not wait for: a kernel launched right afterwards could still read the old bytes.  Going through the
 * session's own stream and waiting for it closes both gaps.  (Never called with a resident poller on
 * that stream: those paths stop it first.) */
static cudaError_t h2d_sync(oimgpu_lun *L, void *dst, const void *src, size_t n)
{
	cudaError_t e = cudaMemcpyAsync(dst, src, n, cudaMemcpyHostToDevice, L->stream);
	if (e != cudaSuccess) return e;
	return cudaStreamSynchronize(L->stream);
}

static int find_device_slot(int ordinal)
{
	for (size_t i = 0; i < g.devices.size(); i++) {
		if (g.devices[i].ordinal == ordinal) return (int)i;
	}
	return -1;
}

/* what the kernel needs to know about one SCSI device: geometry, stores, and the identity strings
 * INQUIRY reports: spdk_scsi_dev_construct("Target N", ...) + port 0 "vhost", SAS
 * (vhost_scsi.c:1004-1013); the device id is the slot add_vhost_scsi_lun took in the global table */
static void fill_lun_ctx(LunCtx &c, const Bdev &b, const Ctrlr &ctrlr, int target)
{
	for (size_t r = 0; r < b.stores.size(); r++) c.store[r] = b.stores[r];
	c.nreplicas = (uint32_t)b.stores.size();
	c.num_blocks = b.num_blocks;
	c.block_size = b.block_size;
	c.hist = b.hist;
	c.block_shift = (b.block_size & (b.block_size - 1)) ? 0xffffffffu : (uint32_t)__builtin_ctz(b.block_size);
	c.target = (uint8_t)target;
	snprintf(c.bdev_name, sizeof(c.bdev_name), "%s", b.name.c_str());
	snprintf(c.product_name, sizeof(c.product_name), "%s", b.product.c_str());
	snprintf(c.dev_name, sizeof(c.dev_name), "Target %d", target);
	snprintf(c.port_name, sizeof(c.port_name), "vhost");
	c.scsi_dev_id = ctrlr.scsi_id[target];
	c.port_index = 0;
	c.protocol_id = 0x06;
}

/* counters of one device-resident context, read on the housekeeping stream (works next to a resident poller) */
static bool read_ctx_stats(int device, const LunCtx *d_ctx, unsigned long long out[12])
{
	const int slot = find_device_slot(device);
	if (slot < 0 || !d_ctx) return false;
	cudaSetDevice(device);
	cudaStream_t st = g.devices[slot].util;
	if (cudaMemcpyAsync(out, (const uint8_t *)d_ctx + offsetof(LunCtx, stats), sizeof(unsigned long long) * 12,
			    cudaMemcpyDeviceToHost, st) != cudaSuccess) return false;
	return cudaStreamSynchronize(st) == cudaSuccess;
}

/* a session lets go of a bdev: keep what it counted (get_bdevs_iostat is per bdev, for its lifetime) */
static void retire_stats_locked(const std::string &bdev, int device, const LunCtx *d_ctx)
{
	auto bi = g.bdevs.find(bdev);
	unsigned long long v[12];
	if (bi == g.bdevs.end() || !read_ctx_stats(device, d_ctx, v)) return;
	for (int k = 0; k < 12; k++) bi->second->retired[k] += v[k];
}

static bool device_reachable(int from, int to)
{
	if (from == to) return true;
	int can = 0;
	if (cudaDeviceCanAccessPeer(&can, from, to) != cudaSuccess || !can) return false;
	cudaSetDevice(from);
	cudaError_t e = cudaDeviceEnablePeerAccess(to, 0);
	if (e == cudaErrorPeerAccessAlreadyEnabled) { cudaGetLastError(); e = cudaSuccess; }
	return e == cudaSuccess;
}

/* Bring the session's view of its controller up to date: every target other than the session's
 * own gets a device-resident LunCtx reachable through peer[] (the reference keeps all eight in
 * svdev->scsi_dev[], vhost_scsi.c:80-94, and hot-plugs them while a session runs,
 * spdk_vhost_scsi_dev_add_tgt / _remove_tgt).  Caller holds g.mu. */
static int refresh_peers_locked(oimgpu_lun *L)
{
	std::lock_guard<std::recursive_mutex> hl(L->mu);
	auto it = g.ctrlrs.find(L->ctrlr);
	CU_OK(cudaSetDevice(L->device));
	bool changed = false, restart = false;
	std::string wants[OIMGPU_CTRLR_MAX_DEVS];
	for (int t = 0; t < OIMGPU_CTRLR_MAX_DEVS; t++) {
		std::string &want = wants[t];
		if (it != g.ctrlrs.end() && t != L->target) want = it->second->targets[t];
		if (!want.empty()) {
			auto bi = g.bdevs.find(want);
			if (bi == g.bdevs.end() || !device_reachable(L->device, bi->second->devices[0])) want.clear();
		}
		if (want != L->peer_bdev[t] && !L->peer_bdev[t].empty()) restart = true;	/* a device goes away */
		if (!want.empty() && g.bdevs[want]->stores.size() > 1 && !L->any_mirror) restart = true;	/* other kernel variant */
	}
	/* a resident poller may be in the middle of a pass on a device that is being unplugged: park it,
	 * like the reference waits for the session's outstanding tasks (process_removed_devs,
	 * vhost_scsi.c:236-289), and bring it back afterwards */
	const bool was_polling = L->poller_active;
	if (restart && was_polling) {
		int rc = oimgpu_lun_stop_poller(L);
		if (rc) return rc;
	}
	for (int t = 0; t < OIMGPU_CTRLR_MAX_DEVS; t++) {
		const std::string &want = wants[t];
		if (want == L->peer_bdev[t]) continue;
		changed = true;
		if (!L->peer_bdev[t].empty()) {
			auto bi = g.bdevs.find(L->peer_bdev[t]);
			if (bi != g.bdevs.end() && bi->second->open_luns > 0) bi->second->open_luns--;
			if (!L->poller_active) cudaStreamSynchronize(L->stream);
			retire_stats_locked(L->peer_bdev[t], L->device, L->d_peer[t]);
		}
		L->peer_bdev[t] = want;
		if (want.empty()) {
			L->h_ctx.peer[t] = nullptr;	/* the context itself is freed at close: a resident kernel may still hold it */
			continue;
		}
		Bdev &b = *g.bdevs[want];
		b.open_luns++;
		LunCtx c;
		memset(&c, 0, sizeof(c));
		fill_lun_ctx(c, b, *it->second, t);
		if (!L->d_peer[t]) CU_OK(cudaMalloc((void **)&L->d_peer[t], sizeof(LunCtx)));
		CU_OK(cudaMemcpyAsync(L->d_peer[t], &c, sizeof(c), cudaMemcpyHostToDevice, L->copy_stream));
		CU_OK(cudaStreamSynchronize(L->copy_stream));	/* `c` is pageable stack memory */
		L->h_ctx.peer[t] = L->d_peer[t];
	}
	if (!changed) {
		if (restart && was_polling) return oimgpu_lun_start_poller(L, L->poller_max_ctas, L->poller_idle_ms) < 0 ? -EIO : 0;
		return 0;
	}
	L->any_mirror = L->h_ctx.nreplicas > 1;
	for (int t = 0; t < OIMGPU_CTRLR_MAX_DEVS; t++) {
		if (!L->peer_bdev[t].empty() && g.bdevs[L->peer_bdev[t]]->stores.size() > 1) L->any_mirror = true;
	}
	/* publish the pointers after the contexts they point at (same stream); a separate stream so that a
	 * resident poller kernel on L->stream does not block the update */
	CU_OK(cudaMemcpyAsync((uint8_t *)L->d_ctx + offsetof(LunCtx, peer), L->h_ctx.peer, sizeof(L->h_ctx.peer),
			      cudaMemcpyHostToDevice, L->copy_stream));
	CU_OK(cudaStreamSynchronize(L->copy_stream));
	if (!L->poller_active) CU_OK(cudaStreamSynchronize(L->stream));
	if (restart && was_polling) {
		int rc = oimgpu_lun_start_poller(L, L->poller_max_ctas, L->poller_idle_ms);
		if (rc < 0) return rc;
	}
	return 0;
}

/* cudaFree waits for the whole device, and a resident poller kernel never finishes on its own: park
 * the pollers of that GPU around a free and bring them back afterwards.  Every session of the GPU is
 * held (its mutex taken) for the duration, so that none can start a resident kernel in the window -
 * their owners' calls simply wait.  Caller holds g.mu; sessions never take g.mu while holding their own
 * mutex, so the order g.mu -> session mutex is safe. */
struct ParkedSession { oimgpu_lun *L; bool restart; };

static std::vector<ParkedSession> park_pollers_locked(int device, oimgpu_lun *except = nullptr)
{
	/* device < 0: every GPU (pinned host memory is mapped into all of them) */
	std::vector<ParkedSession> parked;
	for (oimgpu_lun *L : g.handles) {
		if (L == except || (device >= 0 && L->device != device)) continue;
		L->mu.lock();
		const bool was = L->poller_active;
		if (was) oimgpu_lun_stop_poller(L);
		parked.push_back({L, was});
	}
	return parked;
}

static void unpark_pollers_locked(const std::vector<ParkedSession> &parked)
{
	for (const ParkedSession &p : parked) {
		if (p.restart) oimgpu_lun_start_poller(p.L, p.L->poller_max_ctas, p.L->poller_idle_ms);
		p.L->mu.unlock();
	}
}

static void refresh_ctrlr_sessions_locked(const std::string &ctrlr)
{
	for (oimgpu_lun *L : g.handles) {
		if (L->ctrlr == ctrlr) refresh_peers_locked(L);
	}
}

static std::string random_uuid()
{
	std::random_device rd;
	uint8_t u[16];
	for (int i = 0; i < 16; i++) u[i] = (uint8_t)rd();
	u[6] = (u[6] & 0x0f) | 0x40;
	u[8] = (u[8] & 0x3f) | 0x80;
	char out[40];
	snprintf(out, sizeof(out), "%02x%02x%02x%02x-%02x%02x-%02x%02x-%02x%02x-%02x%02x%02x%02x%02x%02x",
		 u[0], u[1], u[2], u[3], u[4], u[5], u[6], u[7], u[8], u[9], u[10], u[11], u[12], u[13], u[14], u[15]);
	return out;
}

/* spdk_uuid_parse -> uuid_parse: exactly 36 chars, hex with dashes at 8/13/18/23 */
static bool uuid_valid(const char *s)
{
	if (strlen(s) != 36) return false;
	for (int i = 0; i < 36; i++) {
		if (i == 8 || i == 13 || i == 18 || i == 23) {
			if (s[i] != '-') return false;
		} else if (!isxdigit((unsigned char)s[i])) {
			return false;
		}
	}
	return true;
}

static void copy_str(char *dst, size_t cap, const std::string &s)
{
	if (!dst || !cap) return;
	snprintf(dst, cap, "%s", s.c_str());
}

/* ---- lifecycle ------------------------------------------------------------------------------- */

static void release_store(Bdev &b, size_t r)
{
	cudaSetDevice(b.devices[r]);
	if (b.imported[r]) cudaIpcCloseMemHandle(b.stores[r]);
	else cudaFree(b.stores[r]);
	(void)cudaGetLastError();
}


extern "C" int oimgpu_abi_version(void) { return OIMGPU_ABI_VERSION; }

extern "C" const char *oimgpu_version_string(void)
{
	return "oimgpu 0.1 (sm_90a; replaces SPDK v19.04-pre vhost-scsi/Malloc data path behind intel/oim)";
}

extern "C" int oimgpu_init(const int *devices, int ndevices)
{
	std::lock_guard<std::mutex> lk(g.mu);
	if (g.inited) return 0;
	int count = 0;
	if (cudaGetDeviceCount(&count) != cudaSuccess || count == 0) {
		fprintf(stderr, "oimgpu: no CUDA device; the data path has no CPU fallback\n");
		return -ENODEV;
	}
	std::vector<int> ords;
	if (devices && ndevices > 0) {
		ords.assign(devices, devices + ndevices);
	} else {
		int cur = 0;
		CU_OK(cudaGetDevice(&cur));
		ords.push_back(cur);
	}
	for (int o : ords) {
		if (o < 0 || o >= count) return -EINVAL;
		cudaDeviceProp prop;
		CU_OK(cudaGetDeviceProperties(&prop, o));
		Device d;
		d.ordinal = o;
		d.sm_count = prop.multiProcessorCount;
		CU_OK(cudaSetDevice(o));
		CU_OK(cudaStreamCreateWithFlags(&d.util, cudaStreamNonBlocking));
		g.devices.push_back(d);
	}
	/* mirrored bdevs store to peer HBM directly: enable P2P between every pair we manage */
	for (size_t i = 0; i < g.devices.size(); i++) {
		for (size_t j = 0; j < g.devices.size(); j++) {
			if (i == j) continue;
			int can = 0;
			cudaDeviceCanAccessPeer(&can, g.devices[i].ordinal, g.devices[j].ordinal);
			if (can) {
				cudaSetDevice(g.devices[i].ordinal);
				cudaError_t e = cudaDeviceEnablePeerAccess(g.devices[j].ordinal, 0);
				if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) (void)cudaGetLastError();
				(void)cudaGetLastError();
			}
		}
	}
	cudaSetDevice(g.devices[0].ordinal);
	g.inited = true;
	return 0;
}

/* Control plane only: bdev/controller bookkeeping for protocol tests on a machine without a GPU.
 * No backing store is allocated and every data-path entry point fails with -ENODEV; this is NOT a
 * CPU implementation of the path. */
extern "C" int oimgpu_init_control_only(void)
{
	std::lock_guard<std::mutex> lk(g.mu);
	if (g.inited) return g.control_only ? 0 : -EBUSY;
	Device d;
	d.ordinal = 0;
	d.sm_count = 0;
	g.devices.push_back(d);
	g.control_only = true;
	g.inited = true;
	return 0;
}

static void unpin_all_host_ranges();	/* oimgpu_mem_ensure's registrations (end of this file) */

extern "C" void oimgpu_fini(void)
{
	std::lock_guard<std::mutex> lk(g.mu);
	if (!g.inited) return;
	if (!g.control_only) unpin_all_host_ranges();
	for (auto &kv : g.bdevs) {
		for (size_t r = 0; r < kv.second->stores.size() && !g.control_only; r++) release_store(*kv.second, r);
		if (kv.second->hist && !g.control_only) { cudaSetDevice(kv.second->devices[0]); cudaFree(kv.second->hist); }
	}
	g.control_only = false;
	g.bdevs.clear();
	g.ctrlrs.clear();
	g.bdev_order.clear();
	g.ctrlr_order.clear();
	memset(g.scsi_slot_used, 0, sizeof(g.scsi_slot_used));
	for (auto &d : g.devices) {
		if (d.util) { cudaSetDevice(d.ordinal); cudaStreamDestroy(d.util); }
	}
	g.devices.clear();
	g.malloc_disk_count = g.rbd_count = 0;
	g.inited = false;
}

extern "C" int oimgpu_device_count(void) { return (int)g.devices.size(); }

/* ---- bdev control ---------------------------------------------------------------------------- */

static int pick_device(int device)
{
	if (device >= 0) return find_device_slot(device) >= 0 ? device : -1;
	size_t best = 0;
	for (size_t i = 1; i < g.devices.size(); i++) {
		if (g.devices[i].bytes_allocated < g.devices[best].bytes_allocated) best = i;
	}
	return g.devices[best].ordinal;
}

static int alloc_store(int ordinal, uint64_t bytes, uint8_t **out)
{
	if (g.control_only) {
		*out = nullptr;
		return 0;
	}
	CU_OK(cudaSetDevice(ordinal));
	cudaError_t e = cudaMalloc((void **)out, bytes);
	if (e != cudaSuccess) {
		(void)cudaGetLastError();
		return -ENOMEM;
	}
	/* spdk_dma_zmalloc: the disk starts zero-filled (bdev_malloc.c:401) */
	Device &dev = g.devices[find_device_slot(ordinal)];
	CU_OK(cudaMemsetAsync(*out, 0, bytes, dev.util));
	CU_OK(cudaStreamSynchronize(dev.util));
	dev.bytes_allocated += bytes;
	return 0;
}

static int create_bdev_locked(const char *name, const char *uuid, uint64_t num_blocks, uint32_t block_size,
			      const std::vector<int> &devs, const char *product, const std::string &auto_name,
			      char *name_out, size_t name_cap)
{
	if (!g.inited) return -ENODEV;
	/* create_malloc_disk: "Disk must be more than 0 blocks" (bdev_malloc.c:384-387); block size must
	 * be a positive multiple the SCSI layer can divide 4 MiB by */
	if (num_blocks == 0 || block_size == 0 || block_size > OIMGPU_MAX_XFER_BYTES) return -EINVAL;
	if (uuid && !uuid_valid(uuid)) return -EINVAL;
	std::string nm = name && name[0] ? name : auto_name;
	if (g.bdevs.count(nm)) return -EEXIST;	/* spdk_bdev_register: name already in use */
	auto b = std::make_unique<Bdev>();
	b->name = nm;
	b->product = product;
	b->uuid = uuid ? uuid : random_uuid();
	b->num_blocks = num_blocks;
	b->block_size = block_size;
	for (int d : devs) {
		uint8_t *p = nullptr;
		int rc = alloc_store(d, num_blocks * (uint64_t)block_size, &p);
		if (rc != 0) {
			for (size_t r = 0; r < b->stores.size(); r++) {
				cudaSetDevice(b->devices[r]);
				cudaFree(b->stores[r]);
			}
			return rc;
		}
		b->devices.push_back(d);
		b->stores.push_back(p);
		b->imported.push_back(0);
	}
	copy_str(name_out, name_cap, nm);
	g.bdevs[nm] = std::move(b);
	g.bdev_order.push_back(nm);
	return 0;
}

extern "C" int oimgpu_bdev_create_malloc(const char *name, const char *uuid, uint64_t num_blocks,
					 uint32_t block_size, int device, char *name_out, size_t name_cap)
{
	std::lock_guard<std::mutex> lk(g.mu);
	if (!g.inited) return -ENODEV;
	int d = pick_device(device);
	if (d < 0) return -EINVAL;
	std::string auto_name;
	if (!(name && name[0])) auto_name = "Malloc" + std::to_string(g.malloc_disk_count);
	int rc = create_bdev_locked(name, uuid, num_blocks, block_size, {d}, "Malloc disk", auto_name, name_out, name_cap);
	if (rc == 0 && !(name && name[0])) g.malloc_disk_count++;
	return rc;
}

extern "C" int oimgpu_bdev_create_rbd(const char *name, const char *pool_name, const char *rbd_name,
				      const char *user_id, uint32_t block_size, uint64_t size_bytes,
				      int device, char *name_out, size_t name_cap)
{
	(void)user_id;
	std::lock_guard<std::mutex> lk(g.mu);
	if (!g.inited) return -ENODEV;
	/* spdk_rpc_construct_rbd_bdev requires pool_name, rbd_name and block_size (bdev_rbd_rpc.c:81-96) */
	if (!pool_name || !pool_name[0] || !rbd_name || !rbd_name[0] || block_size == 0) return -EINVAL;
	if (size_bytes == 0 || size_bytes % block_size) return -EINVAL;
	int d = pick_device(device);
	if (d < 0) return -EINVAL;
	std::string auto_name;
	if (!(name && name[0])) auto_name = "Ceph" + std::to_string(g.rbd_count);	/* bdev_rbd.c:732 */
	int rc = create_bdev_locked(name, nullptr, size_bytes / block_size, block_size, {d}, "Ceph Rbd Disk",
				    auto_name, name_out, name_cap);
	if (rc == 0 && !(name && name[0])) g.rbd_count++;
	if (rc == 0) {
		Bdev &b = *g.bdevs[name && name[0] ? std::string(name) : auto_name];
		b.pool_name = pool_name;
		b.rbd_name = rbd_name;
		b.user_id = user_id ? user_id : "";
	}
	return rc;
}

extern "C" int oimgpu_bdev_create_mirror(const char *name, uint64_t num_blocks, uint32_t block_size,
					 const int *devices, int nreplicas, char *name_out, size_t name_cap)
{
	std::lock_guard<std::mutex> lk(g.mu);
	if (!g.inited) return -ENODEV;
	if (!devices || nreplicas < 1 || nreplicas > kMaxReplicas) return -EINVAL;
	std::vector<int> devs(devices, devices + nreplicas);
	for (int d : devs) {
		if (find_device_slot(d) < 0) return -EINVAL;
	}
	for (int r = 1; r < nreplicas; r++) {
		int can = 0;
		cudaDeviceCanAccessPeer(&can, devs[0], devs[r]);
		if (!can && devs[0] != devs[r]) return -ENOTSUP;
	}
	std::string auto_name;
	if (!(name && name[0])) auto_name = "Mirror" + std::to_string(g.malloc_disk_count);
	int rc = create_bdev_locked(name, nullptr, num_blocks, block_size, devs, "Malloc disk", auto_name, name_out, name_cap);
	if (rc == 0 && !(name && name[0])) g.malloc_disk_count++;
	return rc;
}

extern "C" int oimgpu_bdev_export_store(const char *name, int replica, void *handle_out)
{
	static_assert(sizeof(cudaIpcMemHandle_t) == OIMGPU_IPC_HANDLE_BYTES, "IPC handle size");
	std::lock_guard<std::mutex> lk(g.mu);
	if (!g.inited || g.control_only) return -ENODEV;
	if (!handle_out) return -EINVAL;
	auto it = g.bdevs.find(name ? name : "");
	if (it == g.bdevs.end()) return -ENODEV;
	Bdev &b = *it->second;
	if (replica < 0 || replica >= (int)b.stores.size() || b.imported[replica]) return -EINVAL;
	CU_OK(cudaSetDevice(b.devices[replica]));
	cudaIpcMemHandle_t h;
	CU_OK(cudaIpcGetMemHandle(&h, b.stores[replica]));
	memcpy(handle_out, &h, sizeof(h));
	return 0;
}

extern "C" int oimgpu_bdev_create_mirror_remote(const char *name, uint64_t num_blocks, uint32_t block_size, int device,
						 const void *peer_handles, int npeers, char *name_out, size_t name_cap)
{
	std::lock_guard<std::mutex> lk(g.mu);
	if (!g.inited || g.control_only) return -ENODEV;
	if (!peer_handles || npeers < 1 || npeers >= kMaxReplicas) return -EINVAL;
	int d = pick_device(device);
	if (d < 0) return -EINVAL;
	std::string auto_name;
	if (!(name && name[0])) auto_name = "Mirror" + std::to_string(g.malloc_disk_count);
	char nm[64];
	int rc = create_bdev_locked(name, nullptr, num_blocks, block_size, {d}, "Malloc disk", auto_name, nm, sizeof(nm));
	if (rc) return rc;
	if (!(name && name[0])) g.malloc_disk_count++;
	Bdev &b = *g.bdevs[nm];
	CU_OK(cudaSetDevice(d));
	for (int r = 0; r < npeers; r++) {
		cudaIpcMemHandle_t h;
		memcpy(&h, (const uint8_t *)peer_handles + (size_t)r * sizeof(h), sizeof(h));
		void *p = nullptr;
		cudaError_t e = cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess);
		if (e != cudaSuccess) {
			fprintf(stderr, "oimgpu: cudaIpcOpenMemHandle failed: %s\n", cudaGetErrorString(e));
			(void)cudaGetLastError();
			for (size_t k = 0; k < b.stores.size(); k++) release_store(b, k);
			g.bdev_order.erase(std::remove(g.bdev_order.begin(), g.bdev_order.end(), std::string(nm)), g.bdev_order.end());
			g.bdevs.erase(nm);
			return -EIO;
		}
		b.devices.push_back(d);
		b.stores.push_back((uint8_t *)p);
		b.imported.push_back(1);
	}
	copy_str(name_out, name_cap, nm);
	return 0;
}

namespace oimgpu { __global__ void oim_digest_kernel(const uint64_t *p, uint64_t nwords, unsigned long long *out); }

static int digest_locked(int device, const void *dptr, uint64_t nbytes, uint64_t out[2])
{
	if (!dptr || !out || (nbytes & 7) || ((uintptr_t)dptr & 7)) return -EINVAL;
	const int slot = find_device_slot(device);
	if (slot < 0) return -EINVAL;
	CU_OK(cudaSetDevice(device));
	cudaStream_t st = g.devices[slot].util;
	unsigned long long *d = nullptr;
	CU_OK(cudaMalloc((void **)&d, 16));
	CU_OK(cudaMemsetAsync(d, 0, 16, st));
	oim_digest_kernel<<<g.devices[slot].sm_count * 4, 256, 0, st>>>((const uint64_t *)dptr, nbytes / 8, d);
	unsigned long long h[2] = {0, 0};
	cudaError_t e = cudaMemcpyAsync(h, d, 16, cudaMemcpyDeviceToHost, st);
	if (e == cudaSuccess) e = cudaStreamSynchronize(st);
	cudaFree(d);
	if (e != cudaSuccess) { (void)cudaGetLastError(); return -EIO; }
	out[0] = h[0]; out[1] = h[1];
	return 0;
}

extern "C" int oimgpu_digest_device(int device, const void *dev_ptr, uint64_t nbytes, uint64_t out[2])
{
	std::lock_guard<std::mutex> lk(g.mu);
	if (!g.inited || g.control_only) return -ENODEV;
	return digest_locked(device, dev_ptr, nbytes, out);
}

extern "C" int oimgpu_bdev_digest(const char *name, int replica, uint64_t offset, uint64_t nbytes, uint64_t out[2])
{
	std::lock_guard<std::mutex> lk(g.mu);
	if (!g.inited || g.control_only) return -ENODEV;
	auto it = g.bdevs.find(name ? name : "");
	if (it == g.bdevs.end()) return -ENODEV;
	Bdev &b = *it->second;
	if (replica < 0 || replica >= (int)b.stores.size()) return -EINVAL;
	const uint64_t size = b.num_blocks * (uint64_t)b.block_size;
	if (offset > size || nbytes > size - offset || (offset & 7)) return -EINVAL;
	/* everything already launched on the sessions' streams comes first */
	for (oimgpu_lun *L : g.handles) {
		if (!L->poller_active) { CU_OK(cudaSetDevice(L->device)); CU_OK(cudaStreamSynchronize(L->stream)); }
	}
	return digest_locked(b.devices[replica], b.stores[replica] + offset, nbytes, out);
}

extern "C" int oimgpu_bdev_delete(const char *name)
{
	std::lock_guard<std::mutex> lk(g.mu);
	if (!g.inited) return -ENODEV;
	auto it = g.bdevs.find(name ? name : "");
	if (it == g.bdevs.end()) return -ENODEV;
	/* a session opened on exactly this device pins it; controller-wide sessions let go of it below */
	int peer_refs = 0;
	for (oimgpu_lun *L : g.handles) {
		if (L->bdev == it->first) return -EBUSY;
		for (int t = 0; t < OIMGPU_CTRLR_MAX_DEVS; t++) peer_refs += L->peer_bdev[t] == it->first;
	}
	/* every other pin (an NBD export, oimgpu_nbd_serve) is checked BEFORE anything is taken apart: a failed
	 * delete must leave the targets where they were */
	if (it->second->open_luns > peer_refs) return -EBUSY;
	/* spdk_bdev_unregister hot-removes the SCSI LUNs built on the bdev (lun.c:213-260): the targets go */
	for (auto &kv : g.ctrlrs) {
		bool touched = false;
		for (int t = 0; t < OIMGPU_CTRLR_MAX_DEVS; t++) {
			if (kv.second->targets[t] == it->first) {
				g.scsi_slot_used[kv.second->scsi_id[t]] = false;
				kv.second->targets[t].clear();
				touched = true;
			}
		}
		if (touched && !g.control_only) refresh_ctrlr_sessions_locked(kv.first);
	}
	if (it->second->open_luns) return -EBUSY;
	g.bdev_order.erase(std::remove(g.bdev_order.begin(), g.bdev_order.end(), it->first), g.bdev_order.end());
	for (size_t r = 0; r < it->second->stores.size() && !g.control_only; r++) {
		auto parked = park_pollers_locked(it->second->devices[r]);
		const bool own = !it->second->imported[r];
		release_store(*it->second, r);
		unpark_pollers_locked(parked);
		if (own) g.devices[find_device_slot(it->second->devices[r])].bytes_allocated -=
			it->second->num_blocks * (uint64_t)it->second->block_size;
	}
	if (it->second->hist) { cudaSetDevice(it->second->devices[0]); cudaFree(it->second->hist); }
	g.bdevs.erase(it);
	return 0;
}

/* every open session's device-resident view of the bdev learns where its histogram is (or that it is gone) */
static int publish_hist_locked(const std::string &name, unsigned long long *hist)
{
	for (oimgpu_lun *L : g.handles) {
		std::lock_guard<std::recursive_mutex> hl(L->mu);
		CU_OK(cudaSetDevice(L->device));
		if (L->bdev == name) {
			L->h_ctx.hist = hist;
			CU_OK(cudaMemcpyAsync((uint8_t *)L->d_ctx + offsetof(LunCtx, hist), &L->h_ctx.hist, sizeof(hist), cudaMemcpyHostToDevice, L->copy_stream));
			CU_OK(cudaStreamSynchronize(L->copy_stream));
		}
		for (int t = 0; t < OIMGPU_CTRLR_MAX_DEVS; t++) {
			if (L->peer_bdev[t] != name || !L->d_peer[t]) continue;
			CU_OK(cudaMemcpyAsync((uint8_t *)L->d_peer[t] + offsetof(LunCtx, hist), &hist, sizeof(hist), cudaMemcpyHostToDevice, L->copy_stream));
			CU_OK(cudaStreamSynchronize(L->copy_stream));
		}
	}
	return 0;
}

/* enable_bdev_histogram (S/lib/bdev/rpc/bdev_rpc.c:607-671, spdk_bdev_histogram_enable bdev.c:4367-4400): enabling starts
 * from an empty histogram, disabling drops it */
extern "C" int oimgpu_bdev_histogram_enable(const char *name, int enable)
{
	std::lock_guard<std::mutex> lk(g.mu);
	if (!g.inited) return -ENODEV;
	auto it = g.bdevs.find(name ? name : "");
	if (it == g.bdevs.end()) return -ENODEV;
	Bdev &b = *it->second;
	if (g.control_only) { b.hist = enable ? (unsigned long long *)1 : nullptr; return 0; }
	CU_OK(cudaSetDevice(b.devices[0]));
	cudaStream_t st = g.devices[find_device_slot(b.devices[0])].util;
	if (enable) {
		if (!b.hist) {
			unsigned long long *h = nullptr;
			CU_OK(cudaMalloc((void **)&h, sizeof(unsigned long long) * kHistBuckets));
			b.hist = h;
		}
		CU_OK(cudaMemsetAsync(b.hist, 0, sizeof(unsigned long long) * kHistBuckets, st));
		CU_OK(cudaStreamSynchronize(st));
		return publish_hist_locked(it->first, b.hist);
	}
	if (b.hist) {
		int rc = publish_hist_locked(it->first, nullptr);
		if (rc) return rc;
		/* kernels already launched may still tally: everything in flight first, resident pollers parked */
		auto parked = park_pollers_locked(-1);
		for (oimgpu_lun *L : g.handles) { cudaSetDevice(L->device); cudaStreamSynchronize(L->stream); }
		cudaSetDevice(b.devices[0]);
		cudaFree(b.hist);
		unpark_pollers_locked(parked);
		b.hist = nullptr;
	}
	return 0;
}

/* get_bdev_histogram (bdev_rpc.c:675-790): the kHistBuckets bucket counters.  Disabled: -EFAULT while anything has the
 * bdev open (the reference's per-channel histogram is NULL then), an empty histogram otherwise (no channel to ask) */
extern "C" int oimgpu_bdev_histogram_get(const char *name, uint64_t *buckets)
{
	std::lock_guard<std::mutex> lk(g.mu);
	if (!g.inited) return -ENODEV;
	auto it = g.bdevs.find(name ? name : "");
	if (it == g.bdevs.end()) return -ENODEV;
	if (!buckets) return -EINVAL;
	Bdev &b = *it->second;
	memset(buckets, 0, sizeof(uint64_t) * kHistBuckets);
	if (!b.hist) return b.open_luns > 0 ? -EFAULT : 0;	/* I/O channels exist while a session runs (spdk_scsi_dev_allocate_io_channels) */
	if (g.control_only) return 0;
	CU_OK(cudaSetDevice(b.devices[0]));
	cudaStream_t st = g.devices[find_device_slot(b.devices[0])].util;
	CU_OK(cudaMemcpyAsync(buckets, b.hist, sizeof(uint64_t) * kHistBuckets, cudaMemcpyDeviceToHost, st));
	CU_OK(cudaStreamSynchronize(st));
	return 0;
}

static void fill_bdev_info(const Bdev &b, oimgpu_bdev_info *o)
{
	memset(o, 0, sizeof(*o));
	copy_str(o->name, sizeof(o->name), b.name);
	copy_str(o->product_name, sizeof(o->product_name), b.product);
	copy_str(o->uuid, sizeof(o->uuid), b.uuid);
	o->num_blocks = b.num_blocks;
	o->block_size = b.block_size;
	o->claimed = 0;	/* SCSI LUNs open the bdev without claiming it (lun.c:342): get_bdevs says false */
	o->device = b.devices[0];
	o->replicas = (uint32_t)b.stores.size();
	o->device_ptr = (uint64_t)(uintptr_t)b.stores[0];
}

extern "C" int oimgpu_bdev_get(const char *name, oimgpu_bdev_info *out)
{
	std::lock_guard<std::mutex> lk(g.mu);
	if (!g.inited) return -ENODEV;
	auto it = g.bdevs.find(name ? name : "");
	if (it == g.bdevs.end()) return -ENODEV;
	if (out) fill_bdev_info(*it->second, out);
	return 0;
}

extern "C" int oimgpu_bdev_list(oimgpu_bdev_info *out, int max)
{
	std::lock_guard<std::mutex> lk(g.mu);
	int n = 0;
	for (auto &nm : g.bdev_order) {
		if (out && n < max) fill_bdev_info(*g.bdevs[nm], &out[n]);
		n++;
	}
	return n;
}

static int raw_access(const char *name, int replica, uint64_t offset, void *host, uint64_t len, bool write)
{
	std::lock_guard<std::mutex> lk(g.mu);
	if (!g.inited || g.control_only) return -ENODEV;
	auto it = g.bdevs.find(name ? name : "");
	if (it == g.bdevs.end()) return -ENODEV;
	Bdev &b = *it->second;
	if (replica < 0 || replica >= (int)b.stores.size()) return -EINVAL;
	uint64_t size = b.num_blocks * (uint64_t)b.block_size;
	if (offset > size || len > size - offset) return -EINVAL;
	CU_OK(cudaSetDevice(b.devices[replica]));
	/* everything already launched on the sessions' streams comes first (a resident poller cannot be
	 * waited for: with one running, quiescing the I/O is the caller's business) */
	for (oimgpu_lun *L : g.handles) {
		if (!L->poller_active) {
			CU_OK(cudaSetDevice(L->device));
			CU_OK(cudaStreamSynchronize(L->stream));
		}
	}
	CU_OK(cudaSetDevice(b.devices[replica]));
	cudaStream_t st = g.devices[find_device_slot(b.devices[replica])].util;
	if (write) CU_OK(cudaMemcpyAsync(b.stores[replica] + offset, host, len, cudaMemcpyHostToDevice, st));
	else CU_OK(cudaMemcpyAsync(host, b.stores[replica] + offset, len, cudaMemcpyDeviceToHost, st));
	CU_OK(cudaStreamSynchronize(st));
	return 0;
}

/* `rows` pieces of `width` bytes, `pitch` apart in device memory, gathered into host memory by the COPY ENGINE on the
 * device's housekeeping stream: how a host thread looks at ring indices in HBM while a resident poller holds every SM
 * slot (a kernel launched for the same purpose would wait for the poller to leave) */
extern "C" int oimgpu_read_strided(int device, void *dst, const void *src, size_t pitch, size_t width, size_t rows)
{
	if (!dst || !src || !width || !rows) return -EINVAL;
	std::lock_guard<std::mutex> lk(g.mu);
	if (!g.inited || g.control_only) return -ENODEV;
	const int slot = find_device_slot(device);
	if (slot < 0) return -EINVAL;
	CU_OK(cudaSetDevice(device));
	cudaStream_t st = g.devices[slot].util;
	CU_OK(cudaMemcpy2DAsync(dst, width, src, pitch, width, rows, cudaMemcpyDeviceToHost, st));
	CU_OK(cudaStreamSynchronize(st));
	return 0;
}

/* the scatter counterpart (host -> device), e.g. a test guest publishing avail->idx on many rings in HBM */
extern "C" int oimgpu_write_strided(int device, void *dst, const void *src, size_t pitch, size_t width, size_t rows)
{
	if (!dst || !src || !width || !rows) return -EINVAL;
	std::lock_guard<std::mutex> lk(g.mu);
	if (!g.inited || g.control_only) return -ENODEV;
	const int slot = find_device_slot(device);
	if (slot < 0) return -EINVAL;
	CU_OK(cudaSetDevice(device));
	cudaStream_t st = g.devices[slot].util;
	CU_OK(cudaMemcpy2DAsync(dst, pitch, src, width, width, rows, cudaMemcpyHostToDevice, st));
	CU_OK(cudaStreamSynchronize(st));
	return 0;
}

extern "C" int oimgpu_bdev_read_raw(const char *name, int replica, uint64_t offset, void *dst, uint64_t len)
{
	return raw_access(name, replica, offset, dst, len, false);
}

extern "C" int oimgpu_bdev_write_raw(const char *name, int replica, uint64_t offset, const void *src, uint64_t len)
{
	return raw_access(name, replica, offset, const_cast<void *>(src), len, true);
}

/* ---- vhost-scsi control ------------------------------------------------------------------------ */

/* spdk_vhost_dev_register strips the socket directory prefix from the name (vhost.c:611-628);
 * callers may pass a path, we keep the last component */
static std::string ctrlr_key(const char *ctrlr)
{
	std::string s = ctrlr ? ctrlr : "";
	if (!g.socket_dir.empty() && s.compare(0, g.socket_dir.size(), g.socket_dir) == 0) return s.substr(g.socket_dir.size());
	if (g.socket_dir.empty()) {
		/* no -S directory configured: accept a path and keep its last component */
		size_t p = s.find_last_of('/');
		if (p != std::string::npos) return s.substr(p + 1);
	}
	return s;
}

/* vhost -S <dir> (S/lib/vhost/vhost.c:1185-1205): controller sockets live at <dir>/<name> */
extern "C" int oimgpu_set_socket_dir(const char *dir, const char *app_core_mask)
{
	std::lock_guard<std::mutex> lk(g.mu);
	g.socket_dir = dir ? dir : "";
	if (!g.socket_dir.empty() && g.socket_dir.back() != '/') g.socket_dir += '/';
	if (app_core_mask && app_core_mask[0]) {
		char *end = nullptr;
		unsigned long long v = strtoull(app_core_mask, &end, 16);
		if (end == app_core_mask || *end || v == 0) return -EINVAL;
		g.app_core_mask = v;
	}
	return 0;
}

extern "C" int oimgpu_vhost_scsi_ctrlr_create(const char *ctrlr, const char *cpumask)
{
	std::lock_guard<std::mutex> lk(g.mu);
	if (!g.inited) return -ENODEV;
	/* spdk_vhost_dev_register takes the name verbatim (only lookups strip the socket directory,
	 * spdk_vhost_dev_find, vhost.c:611-628) */
	std::string key = ctrlr ? ctrlr : "";
	if (key.empty()) return -EINVAL;
	if (g.ctrlrs.count(ctrlr_key(ctrlr)) || g.ctrlrs.count(key)) return -EEXIST;
	std::string mask = "0x1";
	if (cpumask && cpumask[0]) {
		/* spdk_vhost_parse_core_mask: a hex mask that must select at least one core (vhost.c:560-590) */
		char *end = nullptr;
		unsigned long long v = strtoull(cpumask, &end, 16);
		if (end == cpumask || *end != 0) return -EINVAL;
		v &= g.app_core_mask;		/* spdk_app_parse_core_mask keeps only the application's cores ... */
		if (v == 0) return -EINVAL;	/* ... "no cpu is selected among reactor mask" (vhost.c:560-590) */
		char buf[24];
		snprintf(buf, sizeof(buf), "0x%llx", v);
		mask = buf;
	}
	auto c = std::make_unique<Ctrlr>();
	c->name = key;
	c->cpumask = mask;
	g.ctrlrs[key] = std::move(c);
	g.ctrlr_order.push_back(key);
	return 0;
}

extern "C" int oimgpu_vhost_scsi_add_lun(const char *ctrlr, int scsi_target_num, const char *bdev_name)
{
	std::lock_guard<std::mutex> lk(g.mu);
	if (!g.inited) return -ENODEV;
	auto it = g.ctrlrs.find(ctrlr_key(ctrlr));
	if (it == g.ctrlrs.end()) return -ENODEV;
	Ctrlr &c = *it->second;
	/* spdk_vhost_scsi_dev_add_tgt (vhost_scsi.c:951-1021) */
	if (scsi_target_num < 0) {
		for (scsi_target_num = 0; scsi_target_num < OIMGPU_CTRLR_MAX_DEVS; scsi_target_num++) {
			if (c.targets[scsi_target_num].empty()) break;
		}
		if (scsi_target_num == OIMGPU_CTRLR_MAX_DEVS) return -ENOSPC;
	} else {
		if (scsi_target_num >= OIMGPU_CTRLR_MAX_DEVS) return -EINVAL;
	}
	if (!bdev_name) return -EINVAL;
	if (!c.targets[scsi_target_num].empty()) return -EEXIST;
	auto b = g.bdevs.find(bdev_name);
	if (b == g.bdevs.end()) return -EINVAL;	/* spdk_scsi_dev_construct failed */
	int slot = 0;
	while (slot < 1024 && g.scsi_slot_used[slot]) slot++;
	if (slot == 1024) return -EINVAL;	/* spdk_scsi_dev_construct: no free device slot */
	g.scsi_slot_used[slot] = true;
	c.scsi_id[scsi_target_num] = slot;
	c.targets[scsi_target_num] = bdev_name;
	b->second->claimed++;
	if (!g.control_only) refresh_ctrlr_sessions_locked(it->first);	/* hot-plug into running sessions */
	return scsi_target_num;
}

extern "C" int oimgpu_vhost_scsi_remove_target(const char *ctrlr, int scsi_target_num)
{
	std::lock_guard<std::mutex> lk(g.mu);
	if (!g.inited) return -ENODEV;
	auto it = g.ctrlrs.find(ctrlr_key(ctrlr));
	if (it == g.ctrlrs.end()) return -ENODEV;
	if (scsi_target_num < 0 || scsi_target_num >= OIMGPU_CTRLR_MAX_DEVS) return -EINVAL;
	Ctrlr &c = *it->second;
	if (c.targets[scsi_target_num].empty()) return -ENODEV;
	auto b = g.bdevs.find(c.targets[scsi_target_num]);
	if (b != g.bdevs.end() && b->second->claimed > 0) b->second->claimed--;
	/* a session opened on exactly this target keeps serving it until it is closed (the reference
	 * defers the removal until the session has no task in flight, vhost_scsi.c:236-289); for every
	 * other session of the controller the target disappears now */
	g.scsi_slot_used[c.scsi_id[scsi_target_num]] = false;
	c.targets[scsi_target_num].clear();
	if (!g.control_only) refresh_ctrlr_sessions_locked(it->first);
	return 0;
}

extern "C" int oimgpu_vhost_ctrlr_remove(const char *ctrlr)
{
	std::lock_guard<std::mutex> lk(g.mu);
	if (!g.inited) return -ENODEV;
	auto it = g.ctrlrs.find(ctrlr_key(ctrlr));
	if (it == g.ctrlrs.end()) return -ENODEV;
	for (auto &t : it->second->targets) {
		if (!t.empty()) return -EBUSY;	/* vhost_scsi.c:837-842 */
	}
	g.ctrlr_order.erase(std::remove(g.ctrlr_order.begin(), g.ctrlr_order.end(), it->first), g.ctrlr_order.end());
	g.ctrlrs.erase(it);
	return 0;
}

/* spdk_vhost_set_coalescing (S/lib/vhost/vhost.c:358-381): the threshold is kept as requests per statistics
 * interval of 10 ms (SPDK_VHOST_STATS_CHECK_INTERVAL_MS), so fewer than 100 IOPS rounds to nothing and is refused;
 * the delay must fit 32 bits of timer ticks (ours: nanoseconds) */
extern "C" int oimgpu_vhost_ctrlr_set_coalescing(const char *ctrlr, uint32_t delay_base_us, uint32_t iops_threshold)
{
	std::lock_guard<std::mutex> lk(g.mu);
	if (!g.inited) return -ENODEV;
	auto it = g.ctrlrs.find(ctrlr_key(ctrlr));
	if (it == g.ctrlrs.end()) return -ENODEV;
	if ((uint64_t)delay_base_us * 1000ull >= UINT32_MAX) return -EINVAL;
	if (iops_threshold * 10u / 1000u == 0) return -EINVAL;
	it->second->delay_base_us = delay_base_us;
	it->second->iops_threshold = iops_threshold;
	return 0;
}

static std::string json_escape(const std::string &in)
{
	std::string o = "\"";
	for (unsigned char c : in) {
		if (c == '"' || c == '\\') { o += '\\'; o += (char)c; }
		else if (c < 0x20) { char b[8]; snprintf(b, sizeof(b), "\\u%04x", c); o += b; }
		else o += (char)c;
	}
	return o + "\"";
}

/* get_subsystem_config (S/lib/event/rpc/subsystem_rpc.c:80-129): the RPC calls that would rebuild the subsystem's
 * present state, as a JSON array of {"method", "params"} - spdk_bdev_subsystem_config_json (S/lib/bdev/bdev.c:676-708)
 * with bdev_malloc_write_json_config (bdev_malloc.c:350-368) / bdev_rbd_write_config_json (bdev_rbd.c:635-666), and
 * spdk_vhost_config_json (vhost.c:1460-1494) with spdk_vhost_scsi_write_config_json (vhost_scsi.c:1459-1499).
 * Returns the length of the text (written if it fits, NUL-terminated), -ENOENT for an unknown subsystem. */
extern "C" long oimgpu_config_json(const char *subsystem, char *buf, size_t cap)
{
	std::lock_guard<std::mutex> lk(g.mu);
	if (!g.inited) return -ENODEV;
	std::string sub = subsystem ? subsystem : "", out = "[";
	if (sub == "bdev") {
		out += "{\"method\":\"set_bdev_options\",\"params\":{\"bdev_io_pool_size\":65536,\"bdev_io_cache_size\":256}}";
		for (auto &nm : g.bdev_order) {
			const Bdev &b = *g.bdevs[nm];
			if (b.product == "Ceph Rbd Disk") {
				out += ",{\"method\":\"construct_rbd_bdev\",\"params\":{\"name\":" + json_escape(b.name) + ",\"pool_name\":" +
				       json_escape(b.pool_name) + ",\"rbd_name\":" + json_escape(b.rbd_name) + ",\"block_size\":" + std::to_string(b.block_size);
				if (!b.user_id.empty()) out += ",\"user_id\":" + json_escape(b.user_id);
				out += "}}";
			} else {
				out += ",{\"method\":\"construct_malloc_bdev\",\"params\":{\"name\":" + json_escape(b.name) + ",\"num_blocks\":" +
				       std::to_string(b.num_blocks) + ",\"block_size\":" + std::to_string(b.block_size) + ",\"uuid\":" + json_escape(b.uuid) + "}}";
			}
		}
	} else if (sub == "vhost") {
		bool first = true;
		for (auto &nm : g.ctrlr_order) {
			const Ctrlr &c = *g.ctrlrs[nm];
			out += std::string(first ? "" : ",") + "{\"method\":\"construct_vhost_scsi_controller\",\"params\":{\"ctrlr\":" +
			       json_escape(c.name) + ",\"cpumask\":" + json_escape(c.cpumask) + "}}";
			first = false;
			for (int t = 0; t < OIMGPU_CTRLR_MAX_DEVS; t++) {
				if (c.targets[t].empty()) continue;
				out += ",{\"method\":\"add_vhost_scsi_lun\",\"params\":{\"ctrlr\":" + json_escape(c.name) + ",\"scsi_target_num\":" +
				       std::to_string(t) + ",\"bdev_name\":" + json_escape(c.targets[t]) + "}}";
			}
			if (c.delay_base_us) {
				out += ",{\"method\":\"set_vhost_controller_coalescing\",\"params\":{\"ctrlr\":" + json_escape(c.name) +
				       ",\"delay_base_us\":" + std::to_string(c.delay_base_us) + ",\"iops_threshold\":" + std::to_string(c.iops_threshold) + "}}";
			}
		}
	} else {
		return -ENOENT;
	}
	out += "]";
	if (buf && cap > out.size()) memcpy(buf, out.c_str(), out.size() + 1);
	return (long)out.size();
}

static void fill_ctrlr_info(const Ctrlr &c, oimgpu_ctrlr_info *o)
{
	memset(o, 0, sizeof(*o));
	copy_str(o->ctrlr, sizeof(o->ctrlr), c.name);
	copy_str(o->cpumask, sizeof(o->cpumask), c.cpumask);
	copy_str(o->socket, sizeof(o->socket), g.socket_dir + c.name);
	o->delay_base_us = c.delay_base_us;
	o->iops_threshold = c.iops_threshold;
	for (int t = 0; t < OIMGPU_CTRLR_MAX_DEVS; t++) {
		if (c.targets[t].empty()) continue;
		oimgpu_target_info &ti = o->targets[o->ntargets++];
		ti.scsi_dev_num = t;
		ti.id = c.scsi_id[t];
		snprintf(ti.target_name, sizeof(ti.target_name), "Target %d", t);
		ti.lun_id = 0;
		copy_str(ti.bdev_name, sizeof(ti.bdev_name), c.targets[t]);
	}
}

extern "C" int oimgpu_vhost_ctrlr_get(const char *ctrlr, oimgpu_ctrlr_info *out)
{
	std::lock_guard<std::mutex> lk(g.mu);
	if (!g.inited) return -ENODEV;
	auto it = g.ctrlrs.find(ctrlr_key(ctrlr));
	if (it == g.ctrlrs.end()) return -ENODEV;
	if (out) fill_ctrlr_info(*it->second, out);
	return 0;
}

extern "C" int oimgpu_vhost_ctrlr_list(oimgpu_ctrlr_info *out, int max)
{
	std::lock_guard<std::mutex> lk(g.mu);
	int n = 0;
	for (auto &nm : g.ctrlr_order) {
		if (out && n < max) fill_ctrlr_info(*g.ctrlrs[nm], &out[n]);
		n++;
	}
	return n;
}

/* ---- data path ----------------------------------------------------------------------------------- */

/* everything a session allocated, whether oimgpu_lun_open got through or not (every member starts null).
 * Caller holds g.mu and has parked the other sessions' pollers (the frees wait for the device). */
static void free_lun_resources(oimgpu_lun *L)
{
	cudaSetDevice(L->device);
	if (L->h_door) cudaFreeHost((void *)L->h_door);
	if (L->h_mix) cudaFreeHost((void *)L->h_mix);
	if (L->h_flags) cudaFreeHost((void *)L->h_flags);
	if (L->slab) cudaFreeHost(L->slab);
	for (int k = 0; k < oimgpu_lun::kKickSlots; k++) {
		if (L->h_kick[k]) cudaFreeHost(L->h_kick[k]);
		if (L->kick_ev[k]) cudaEventDestroy(L->kick_ev[k]);
	}
	cudaFree(L->d_kick);
	cudaFree(L->d_share);
	cudaFree(L->d_vq_state);
	cudaFree(L->d_iov_scratch);
	cudaFree(L->bs_d_reqs);
	cudaFree(L->bs_d_iovs);
	cudaFree(L->bs_d_cpls);
	if (L->bs_h_pin) cudaFreeHost(L->bs_h_pin);
	if (L->bs_uploaded) cudaEventDestroy(L->bs_uploaded);
	if (L->copy_stream) cudaStreamDestroy(L->copy_stream);
	cudaFree(L->d_ctx);
	for (int t = 0; t < OIMGPU_CTRLR_MAX_DEVS; t++) {
		cudaFree(L->d_peer[t]);
		if (!L->peer_bdev[t].empty()) {
			auto bi = g.bdevs.find(L->peer_bdev[t]);
			if (bi != g.bdevs.end() && bi->second->open_luns > 0) bi->second->open_luns--;
		}
	}
	if (L->done) cudaEventDestroy(L->done);
	if (L->stream) cudaStreamDestroy(L->stream);
	(void)cudaGetLastError();
}

static int lun_open_on(const char *ctrlr, int scsi_target_num, int on_device, uint32_t num_queues, uint32_t queue_size, oimgpu_lun **out);

extern "C" int oimgpu_lun_open(const char *ctrlr, int scsi_target_num, uint32_t num_queues,
			       uint32_t queue_size, oimgpu_lun **out)
{
	return lun_open_on(ctrlr, scsi_target_num, -1, num_queues, queue_size, out);
}

/* a controller-wide session (scsi_target_num == -1) on a GPU of the caller's choice: every target of the controller
 * is reached from there, local ones in its own HBM, the others over NVLink (peer mappings).  A daemon that owns
 * several GPUs opens one such session per GPU for ONE vhost-user connection and deals the guest's request queues
 * out among them, so that payload crosses every GPU's PCIe link, wherever the volumes live. */
extern "C" int oimgpu_lun_open_on(const char *ctrlr, int device, uint32_t num_queues, uint32_t queue_size, oimgpu_lun **out)
{
	if (device < 0) return -EINVAL;
	return lun_open_on(ctrlr, -1, device, num_queues, queue_size, out);
}

extern "C" int oimgpu_device_ordinal(int index)
{
	std::lock_guard<std::mutex> lk(g.mu);
	if (index < 0 || index >= (int)g.devices.size()) return -EINVAL;
	return g.devices[index].ordinal;
}

static int lun_open_on(const char *ctrlr, int scsi_target_num, int on_device, uint32_t num_queues, uint32_t queue_size, oimgpu_lun **out)
{
	std::lock_guard<std::mutex> lk(g.mu);
	if (!g.inited || g.control_only) return -ENODEV;
	if (!out || num_queues == 0 || queue_size == 0 || (queue_size & (queue_size - 1)) ||
	    queue_size > OIMGPU_MAX_VQ_SIZE) return -EINVAL;
	auto it = g.ctrlrs.find(ctrlr_key(ctrlr));
	if (it == g.ctrlrs.end()) return -ENODEV;
	/* target -1: a controller-wide session (what a vhost-user connection is): no device of its own,
	 * every target is reached through peer[]; it lives on the GPU of the first target present */
	const bool session = scsi_target_num == -1;
	if (!session && (scsi_target_num < 0 || scsi_target_num >= OIMGPU_CTRLR_MAX_DEVS)) return -EINVAL;
	std::string bn;
	if (!session) {
		bn = it->second->targets[scsi_target_num];
		if (bn.empty()) return -ENODEV;
	}
	Bdev *bp = session ? nullptr : g.bdevs[bn].get();
	int session_device = g.devices[0].ordinal;
	for (int t = 0; session && t < OIMGPU_CTRLR_MAX_DEVS; t++) {
		if (!it->second->targets[t].empty()) { session_device = g.bdevs[it->second->targets[t]]->devices[0]; break; }
	}
	if (on_device >= 0) {
		if (!session || find_device_slot(on_device) < 0) return -EINVAL;
		session_device = on_device;
	}

	/* whatever a failed step leaves behind (streams, events, pinned and device allocations) is released here */
	struct Guard {
		oimgpu_lun *L;
		~Guard() { if (L) { free_lun_resources(L); delete L; } }
		oimgpu_lun *operator->() { return L; }
		oimgpu_lun *get() { return L; }
		oimgpu_lun *release() { oimgpu_lun *r = L; L = nullptr; return r; }
	} L{new oimgpu_lun()};
	L->ctrlr = it->first;
	L->bdev = bn;
	L->target = session ? 0xff : scsi_target_num;
	L->device = session ? session_device : bp->devices[0];
	L->sm_count = g.devices[find_device_slot(L->device)].sm_count;
	L->num_queues = num_queues;
	L->queue_size = queue_size;
	L->iov_cap = queue_size * 8 < 1024 ? 1024 : queue_size * 8;	/* power of two >= 7 x 129 */
	CU_OK(cudaSetDevice(L->device));
	CU_OK(cudaStreamCreateWithFlags(&L->stream, cudaStreamNonBlocking));
	CU_OK(cudaStreamCreateWithFlags(&L->copy_stream, cudaStreamNonBlocking));
	CU_OK(cudaEventCreateWithFlags(&L->done, cudaEventDisableTiming));
	CU_OK(cudaEventCreateWithFlags(&L->bs_uploaded, cudaEventDisableTiming));

	memset(&L->h_ctx, 0, sizeof(L->h_ctx));
	if (session) L->h_ctx.target = 0xff;
	else fill_lun_ctx(L->h_ctx, *bp, *it->second, scsi_target_num);
	CU_OK(cudaHostAlloc((void **)&L->h_mix, 64, cudaHostAllocDefault));
	memset((void *)L->h_mix, 0, 64);
	L->any_mirror = L->h_ctx.nreplicas > 1;
	CU_OK(cudaMalloc((void **)&L->d_ctx, sizeof(LunCtx)));
	CU_OK(h2d_sync(L.get(), L->d_ctx, &L->h_ctx, sizeof(LunCtx)));

	for (int k = 0; k < oimgpu_lun::kKickSlots; k++) {
		CU_OK(cudaHostAlloc((void **)&L->h_kick[k], sizeof(KickHeader) + sizeof(QueueDesc) * num_queues * 3, cudaHostAllocDefault));
		memset(L->h_kick[k], 0, sizeof(KickHeader));
		CU_OK(cudaEventCreateWithFlags(&L->kick_ev[k], cudaEventDisableTiming));
	}
	CU_OK(cudaMalloc((void **)&L->d_kick, sizeof(KickHeader) + sizeof(QueueDesc) * num_queues * 3));	/* ring + device-array + virtqueue per queue */
	L->d_desc = (QueueDesc *)(L->d_kick + sizeof(KickHeader));
	CU_OK(cudaMalloc((void **)&L->d_share, sizeof(QShare) * num_queues * 3));
	L->queues.resize(num_queues);
	/* one mapped pinned slab per LUN, carved into per-queue rings: the "virtqueues" */
	const size_t per_q = sizeof(oimgpu_req) * queue_size + sizeof(oimgpu_iov) * L->iov_cap + sizeof(oimgpu_cpl) * queue_size;
	uint8_t *slab = nullptr, *dslab = nullptr;
	CU_OK(cudaHostAlloc((void **)&slab, per_q * num_queues, cudaHostAllocMapped));
	L->slab = slab;
	CU_OK(cudaHostGetDevicePointer((void **)&dslab, slab, 0));
	memset(slab, 0, per_q * num_queues);
	for (uint32_t q = 0; q < num_queues; q++) {
		Queue &Q = L->queues[q];
		uint8_t *h = slab + per_q * q, *d = dslab + per_q * q;
		Q.h_reqs = (oimgpu_req *)h;
		Q.d_reqs = (oimgpu_req *)d;
		h += sizeof(oimgpu_req) * queue_size; d += sizeof(oimgpu_req) * queue_size;
		Q.h_iovs = (oimgpu_iov *)h;
		Q.d_iovs = (oimgpu_iov *)d;
		h += sizeof(oimgpu_iov) * L->iov_cap; d += sizeof(oimgpu_iov) * L->iov_cap;
		Q.h_cpls = (oimgpu_cpl *)h;
		Q.d_cpls = (oimgpu_cpl *)d;
	}
	CU_OK(cudaHostAlloc((void **)&L->h_door, sizeof(oimgpu_lun::Door) * num_queues, cudaHostAllocMapped));
	CU_OK(cudaHostGetDevicePointer((void **)&L->d_door, L->h_door, 0));
	memset((void *)L->h_door, 0, sizeof(oimgpu_lun::Door) * num_queues);
	CU_OK(cudaHostAlloc((void **)&L->h_flags, 256, cudaHostAllocMapped));
	CU_OK(cudaHostGetDevicePointer((void **)&L->d_flags, (void *)L->h_flags, 0));
	memset((void *)L->h_flags, 0, 256);
	CU_OK(cudaMalloc((void **)&L->d_vq_state, sizeof(VqState) * num_queues));
	CU_OK(cudaMemsetAsync(L->d_vq_state, 0, sizeof(VqState) * num_queues, L->stream));
	CU_OK(cudaStreamSynchronize(L->stream));
	int per_sm = 0;
	CU_OK(lun_kernels_init(&per_sm));
	if (per_sm < 1) per_sm = 1;
	L->grid_cap = L->sm_count * per_sm;
	int rc = refresh_peers_locked(L.get());
	if (rc) return rc;
	g.open_luns++;
	if (bp) bp->open_luns++;
	g.handles.push_back(L.get());
	*out = L.release();
	return 0;
}

extern "C" int oimgpu_lun_close(oimgpu_lun *L)
{
	if (!L) return -EINVAL;
	std::lock_guard<std::mutex> lk(g.mu);
	cudaSetDevice(L->device);
	if (L->poller_active) {
		L->h_flags[0] = 1;
		L->poller_active = false;
	}
	cudaStreamSynchronize(L->stream);
	if (!L->bdev.empty()) retire_stats_locked(L->bdev, L->device, L->d_ctx);
	for (int t = 0; t < OIMGPU_CTRLR_MAX_DEVS; t++) {
		if (!L->peer_bdev[t].empty()) retire_stats_locked(L->peer_bdev[t], L->device, L->d_peer[t]);
	}
	auto parked = park_pollers_locked(L->device, L);	/* other sessions' resident kernels: see park_pollers_locked */
	free_lun_resources(L);
	g.handles.erase(std::remove(g.handles.begin(), g.handles.end(), L), g.handles.end());
	unpark_pollers_locked(parked);
	g.open_luns--;
	{
		auto bi = g.bdevs.find(L->bdev);
		if (bi != g.bdevs.end() && bi->second->open_luns > 0) bi->second->open_luns--;
	}
	delete L;
	return 0;
}

extern "C" int oimgpu_lun_device(const oimgpu_lun *L) { return L ? L->device : -EINVAL; }
extern "C" long long oimgpu_lun_shared_launches(const oimgpu_lun *L) { return L ? (long long)L->shared_launches : -EINVAL; }
extern "C" void *oimgpu_lun_stream(oimgpu_lun *L) { return L ? (void *)L->stream : nullptr; }

extern "C" int oimgpu_mem_register(void *addr, size_t len)
{
	std::lock_guard<std::mutex> lk(g.mu);
	if (!g.inited) return -ENODEV;
	if (!addr || !len) return -EINVAL;
	cudaError_t e = cudaHostRegister(addr, len, cudaHostRegisterMapped | cudaHostRegisterPortable);
	if (e != cudaSuccess) {
		(void)cudaGetLastError();
		return e == cudaErrorHostMemoryAlreadyRegistered ? -EEXIST : -EFAULT;
	}
	g.registered[addr] = len;
	return 0;
}

/* the address the GPU uses for a byte of registered host memory (identical to the host address on
 * systems with a unified address space for registered memory, but that is the driver's call) */
extern "C" int oimgpu_mem_device_addr(const void *addr, uint64_t *dev)
{
	if (!addr || !dev) return -EINVAL;
	if (!g.inited || g.control_only) return -ENODEV;
	void *d = nullptr;
	cudaError_t e = cudaHostGetDevicePointer(&d, const_cast<void *>(addr), 0);
	if (e != cudaSuccess) {
		(void)cudaGetLastError();
		return -EFAULT;
	}
	*dev = (uint64_t)(uintptr_t)d;
	return 0;
}

extern "C" int oimgpu_mem_unregister(void *addr)
{
	std::lock_guard<std::mutex> lk(g.mu);
	auto it = g.registered.find(addr);
	if (it == g.registered.end()) return -ENOENT;
	/* cuMemHostUnregister waits for the GPUs to go idle while holding a driver lock that every launch
	 * needs: with a resident poller anywhere that is a deadlock, not a delay (seen: one VM's teardown
	 * against another VM's poller restart).  Same remedy as for cudaFree. */
	auto parked = park_pollers_locked(-1);
	cudaHostUnregister(addr);
	unpark_pollers_locked(parked);
	g.registered.erase(it);
	return 0;
}

extern "C" int oimgpu_submit(oimgpu_lun *L, uint32_t q, const oimgpu_req *reqs, uint32_t nreqs,
			     const oimgpu_iov *iovs, uint32_t niovs, int mem)
{
	if (!L || q >= L->num_queues || (!reqs && nreqs)) return -EINVAL;
	Queue &Q = L->queues[q];
	if (nreqs == 0) return 0;
	if (mem == OIMGPU_MEM_DEVICE) {
		/* caller-owned device arrays, used in place; completions go to the array given through
		 * oimgpu_submit_device() or to the ring's device view */
		if (Q.dev_count) return -EAGAIN;
		Q.dev_reqs = reqs;
		Q.dev_iovs = iovs;
		Q.dev_cpls = nullptr;
		Q.dev_count = nreqs;
		return 0;
	}
	if (mem != OIMGPU_MEM_HOST) return -EINVAL;
	if (nreqs > L->queue_size - (Q.tail - Q.reaped)) return -EAGAIN;
	if (niovs > L->iov_cap) return -E2BIG;
	/* copy into the ring, rebasing iov_start onto the ring's SG table */
	const uint32_t qmask = L->queue_size - 1, imask = L->iov_cap - 1;
	for (uint32_t i = 0; i < niovs; i++) Q.h_iovs[(Q.iov_tail + i) & imask] = iovs[i];
	for (uint32_t i = 0; i < nreqs; i++) {
		oimgpu_req r = reqs[i];
		r.iov_start += Q.iov_tail;
		Q.h_reqs[(Q.tail + i) & qmask] = r;
	}
	Q.tail += nreqs;
	Q.iov_tail += niovs;
	return 0;
}

/* OIMGPU_MEM_DEVICE submission with an explicit completion array in HBM */
extern "C" int oimgpu_submit_device(oimgpu_lun *L, uint32_t q, const oimgpu_req *d_reqs, uint32_t nreqs,
				    const oimgpu_iov *d_iovs, oimgpu_cpl *d_cpls)
{
	if (!L || q >= L->num_queues || !d_reqs || !d_cpls) return -EINVAL;
	Queue &Q = L->queues[q];
	if (Q.dev_count) return -EAGAIN;
	Q.dev_reqs = d_reqs;
	Q.dev_iovs = d_iovs;
	Q.dev_cpls = d_cpls;
	Q.dev_count = nreqs;
	Q.dev_iov_limit = 0;
	return 0;
}

/* most queues for which the CTAs share queues instead of owning one each (see oimgpu_kick) */
static uint32_t share_max_queues(const oimgpu_lun *L)
{
	const char *e = getenv("OIMGPU_SHARE_MAX_QUEUES");
	if (e && *e) return (uint32_t)strtoul(e, nullptr, 0);
	return (uint32_t)L->grid_cap * 160 / 296;
}

static void launch_queue_kernel(oimgpu_lun *L, uint32_t grid, bool shared, bool vrings_only)
{
	LunKernel k;
	if (!shared && !L->any_mirror && vrings_only && !getenv("OIMGPU_NO_VRING_KERNEL")) k = LUN_KERNEL_VRING;
	else if (shared) k = L->any_mirror ? LUN_KERNEL_SHARED_QUEUE_MIRROR : LUN_KERNEL_SHARED_QUEUE;
	else k = L->any_mirror ? LUN_KERNEL_QUEUE_MIRROR : LUN_KERNEL_QUEUE;
	launch_lun_kernel(k, grid, L->stream, L->d_ctx, (KickHeader *)L->d_kick, L->d_desc);
}

/* ---- the QueueDesc records of a launch, one builder per kind of queue ---- */

/* caller-owned device arrays, served once from slot 0 */
static QueueDesc desc_device_arrays(oimgpu_lun *L, uint32_t q)
{
	const Queue &Q = L->queues[q];
	QueueDesc D;
	memset(&D, 0, sizeof(D));
	D.vq_state = L->d_vq_state + q;
	D.reqs = Q.dev_reqs;
	D.iovs = Q.dev_iovs;
	D.cpls = Q.dev_cpls ? Q.dev_cpls : Q.d_cpls;
	D.ring_mask = 0xffffffffu;
	D.iov_mask = 0xffffffffu;
	D.iov_limit = Q.dev_iov_limit;
	D.head = 0;
	D.count = Q.dev_count;
	return D;
}

/* the library's slot ring (the caller sets head / count, or the poller's doorbells) */
static QueueDesc desc_slot_ring(oimgpu_lun *L, uint32_t q)
{
	const Queue &Q = L->queues[q];
	QueueDesc D;
	memset(&D, 0, sizeof(D));
	D.vq_state = L->d_vq_state + q;
	D.reqs = Q.d_reqs;
	D.iovs = Q.d_iovs;
	D.cpls = Q.d_cpls;
	D.ring_mask = L->queue_size - 1;
	D.iov_mask = L->iov_cap - 1;
	return D;
}

/* an attached guest virtqueue; the parser lanes build their SG rows in d_iov_scratch */
static QueueDesc desc_virtqueue(oimgpu_lun *L, uint32_t q)
{
	const Queue &Q = L->queues[q];
	QueueDesc D;
	memset(&D, 0, sizeof(D));
	D.mode = QMODE_VRING;
	D.iovs = L->d_iov_scratch;
	D.vq_size = Q.vq_size;
	D.vq_desc = Q.vq_desc;
	D.vq_avail = Q.vq_avail;
	D.vq_used = Q.vq_used;
	D.vq_in_hbm = Q.vq_in_hbm ? 1 : 0;
	D.vq_state = L->d_vq_state + q;
	return D;
}

/* [grid_cap][32][kIovRow] SG rows for the parser lanes of virtqueue mode */
static cudaError_t ensure_iov_scratch(oimgpu_lun *L)
{
	if (L->d_iov_scratch) return cudaSuccess;
	return cudaMalloc((void **)&L->d_iov_scratch, sizeof(oimgpu_iov) * (size_t)L->grid_cap * kPass * kIovRow);
}

extern "C" int oimgpu_kick(oimgpu_lun *L)
{
	if (!L) return -EINVAL;
	std::lock_guard<std::recursive_mutex> hl(L->mu);
	if (L->poller_active) {
		/* the resident kernel is polling: a kick is a doorbell write (after the slot contents) */
		int n = 0;
		std::atomic_thread_fence(std::memory_order_release);
		for (uint32_t q = 0; q < L->num_queues; q++) {
			Queue &Q = L->queues[q];
			if (Q.dev_count) return -EBUSY;		/* caller-owned device arrays need a launch */
			if (Q.tail != Q.kicked) {
				L->h_door[q].tail = Q.tail;
				Q.kicked = Q.tail;
				n++;
			}
		}
		return n;
	}
	CU_OK(cudaSetDevice(L->device));
	const int slot = (int)(L->kicks % oimgpu_lun::kKickSlots);
	if (L->kicks >= (uint64_t)oimgpu_lun::kKickSlots) CU_OK(cudaEventSynchronize(L->kick_ev[slot]));
	QueueDesc *h_desc = (QueueDesc *)(L->h_kick[slot] + sizeof(KickHeader));
	uint32_t nd = 0, nvring = 0;
	uint64_t passes = 0;	/* passes of <= 32 requests this kick will take (virtqueues: at most a ring full) */
	for (uint32_t q = 0; q < L->num_queues; q++) {
		Queue &Q = L->queues[q];
		if (Q.dev_count) {
			passes += (Q.dev_count + kPass - 1) / kPass;
			h_desc[nd++] = desc_device_arrays(L, q);
			Q.dev_count = 0;
		}
		if (Q.vq_pending) {
			passes += (Q.vq_size + kPass - 1) / kPass;
			nvring++;
			h_desc[nd++] = desc_virtqueue(L, q);
			Q.vq_pending = false;
		}
		if (Q.tail != Q.kicked) {
			passes += (Q.tail - Q.kicked + kPass - 1) / kPass;
			QueueDesc &D = h_desc[nd++];
			D = desc_slot_ring(L, q);
			D.head = Q.kicked;
			D.count = Q.tail - Q.kicked;
			Q.kicked = Q.tail;
		}
	}
	if (nd == 0) return 0;
	/* One CTA per queue while there are at least as many queues as the GPU holds CTAs; with fewer queues the
	 * CTAs SHARE them, a pass at a time (KickHeader::shared), so that a single deep queue - or the <= 254
	 * request queues of a vhost controller - still fills the machine. */
	uint32_t grid = (uint32_t)std::min<uint64_t>(std::max<uint64_t>(nd, passes), (uint64_t)L->grid_cap);
	/* Sharing pays while the queues alone cannot fill HBM with one CTA each; above share_max_queues ownership is cheaper
	 * (tools/queue_sweep.py measures both sides, 4 KiB random read, 2^21 requests). */
	/* ... and only for read-dominated sessions: passes of different CTAs are ordered coarsely, a write-hot queue is
	 * served by its home CTA alone and slower than the one-CTA-per-queue kernel would.  The kernels count what they served (LunCtx::mix, copied back behind every launch); once 1024 requests have
	 * been seen since the last look, more than one write in eight switches sharing off (and back on when they stop). */
	{
		const unsigned long long r = L->h_mix[0] - L->mix_seen[0], w = L->h_mix[1] - L->mix_seen[1];
		if (r + w >= 1024) {
			L->write_hot = w * 8 > r + w;
			L->mix_seen[0] += r;
			L->mix_seen[1] += w;
		}
	}
	const bool shared = nd < grid && nd <= share_max_queues(L) && !L->write_hot && !getenv("OIMGPU_NO_SHARED_QUEUES");
	if (!shared) grid = std::min(grid, nd);
	KickHeader *kh = (KickHeader *)L->h_kick[slot];
	memset(kh, 0, sizeof(*kh));	/* run-to-completion: persistent = 0 (the staging buffer is recycled pinned memory) */
	kh->next = grid;	/* queues 0..grid-1 are taken statically by CTA index */
	kh->nqueues = nd;
	if (shared) {
		kh->shared = 1;
		kh->share = L->d_share;
		CU_OK(cudaMemsetAsync(L->d_share, 0, sizeof(QShare) * nd, L->stream));
		L->shared_launches++;
	}
	CU_OK(cudaMemcpyAsync(L->d_kick, L->h_kick[slot], sizeof(KickHeader) + sizeof(QueueDesc) * nd, cudaMemcpyHostToDevice, L->stream));
	CU_OK(cudaEventRecord(L->kick_ev[slot], L->stream));
	L->kicks++;
	launch_queue_kernel(L, grid, shared, nvring == nd);
	CU_OK(cudaGetLastError());
	CU_OK(cudaMemcpyAsync((void *)L->h_mix, (const uint8_t *)L->d_ctx + offsetof(LunCtx, mix), sizeof(unsigned long long) * 2,
			      cudaMemcpyDeviceToHost, L->stream));
	CU_OK(cudaEventRecord(L->done, L->stream));
	L->launches++;
	return (int)nd;
}

static int batch_finish(oimgpu_lun *L);

extern "C" int oimgpu_lun_sync(oimgpu_lun *L)
{
	if (!L) return -EINVAL;
	std::lock_guard<std::recursive_mutex> hl(L->mu);
	return batch_finish(L);		/* stream sync + hand over the completions of a host-array batch */
}

extern "C" int oimgpu_poll(oimgpu_lun *L, uint32_t q, oimgpu_cpl *cpls, uint32_t max, int wait)
{
	if (!L || q >= L->num_queues) return -EINVAL;
	Queue &Q = L->queues[q];
	if (Q.kicked == Q.reaped) return 0;
	if (L->poller_active) {
		uint32_t done = L->h_door[q].done;
		if (wait) {
			while ((int32_t)(done - Q.kicked) < 0) {
				if (L->h_flags[16] >= L->poller_grid) return -ESHUTDOWN;	/* the poller left (watchdog) */
				done = L->h_door[q].done;
			}
		}
		std::atomic_thread_fence(std::memory_order_acquire);
		uint32_t n = std::min(max, done - Q.reaped);
		const uint32_t qmask = L->queue_size - 1;
		for (uint32_t i = 0; i < n; i++) cpls[i] = Q.h_cpls[(Q.reaped + i) & qmask];
		Q.reaped += n;
		return (int)n;
	}
	if (wait) {
		int rc = oimgpu_lun_sync(L);
		if (rc) return rc;
	} else if (cudaEventQuery(L->done) != cudaSuccess) {
		(void)cudaGetLastError();
		return 0;
	}
	uint32_t n = std::min(max, Q.kicked - Q.reaped);
	const uint32_t qmask = L->queue_size - 1;
	for (uint32_t i = 0; i < n; i++) cpls[i] = Q.h_cpls[(Q.reaped + i) & qmask];
	Q.reaped += n;
	return (int)n;
}

/* submit to queues 0..nq-1 (queue i gets reqs[i*per_q .. (i+1)*per_q)) and kick; asynchronous */
extern "C" int oimgpu_submit_batch(oimgpu_lun *L, uint32_t nq, uint32_t per_q, const oimgpu_req *reqs,
				   const oimgpu_iov *iovs, uint32_t niovs, oimgpu_cpl *cpls, int mem)
{
	if (!L || nq == 0 || nq > L->num_queues || !reqs) return -EINVAL;
	if (mem == OIMGPU_MEM_DEVICE) {
		if (!cpls) return -EINVAL;
		for (uint32_t q = 0; q < nq; q++) {
			int rc = oimgpu_submit_device(L, q, reqs + (size_t)q * per_q, per_q, iovs, cpls + (size_t)q * per_q);
			if (rc) return rc;
		}
		return oimgpu_kick(L);
	}
	if (mem != OIMGPU_MEM_HOST) return -EINVAL;
	if (!cpls) return -EINVAL;
	/* Host arrays.  The SG *addresses* stay host pointers (payload is loaded/stored by the movers
	 * straight from/to pinned client memory); the request, SG and completion *arrays* are moved by the
	 * copy engine so that the parser never waits on a PCIe read. */
	if (L->poller_active) {
		/* resident kernel: requests go through the host-visible rings, the kick is a doorbell write.
		 * Every queue's requests index the one SG table of the call. */
		for (uint32_t q = 0; q < nq; q++) {
			const oimgpu_req *r = reqs + (size_t)q * per_q;
			uint32_t lo = 0xffffffffu, hi = 0;
			for (uint32_t i = 0; i < per_q; i++) {
				if (r[i].iovcnt == 0) continue;
				lo = std::min(lo, r[i].iov_start);
				hi = std::max(hi, r[i].iov_start + r[i].iovcnt);
			}
			if (lo == 0xffffffffu) lo = hi = 0;
			if (hi > niovs) return -EINVAL;
			Queue &Q = L->queues[q];
			if (per_q > L->queue_size - (Q.tail - Q.reaped)) return -EAGAIN;
			if (hi - lo > L->iov_cap) return -E2BIG;
			const uint32_t qmask = L->queue_size - 1, imask = L->iov_cap - 1;
			for (uint32_t i = lo; i < hi; i++) Q.h_iovs[(Q.iov_tail + (i - lo)) & imask] = iovs[i];
			for (uint32_t i = 0; i < per_q; i++) {
				oimgpu_req t = r[i];
				t.iov_start = t.iov_start - lo + Q.iov_tail;
				Q.h_reqs[(Q.tail + i) & qmask] = t;
			}
			Q.tail += per_q;
			Q.iov_tail += hi - lo;
		}
		return oimgpu_kick(L);
	}
	CU_OK(cudaSetDevice(L->device));
	if (L->bs_pending) return -EAGAIN;
	const size_t n = (size_t)nq * per_q;
	if (n > L->bs_cap_reqs || niovs > L->bs_cap_iovs) {
		CU_OK(cudaStreamSynchronize(L->stream));
		/* growing the staging arrays frees the old ones: see park_pollers_locked */
		std::lock_guard<std::mutex> lk(g.mu);
		auto parked = park_pollers_locked(L->device, L);
		struct Unpark { std::vector<ParkedSession> &p; ~Unpark() { unpark_pollers_locked(p); } } unpark{parked};
		if (n > L->bs_cap_reqs) {
			cudaFree(L->bs_d_reqs); cudaFree(L->bs_d_cpls);
			CU_OK(cudaMalloc((void **)&L->bs_d_reqs, n * sizeof(oimgpu_req)));
			CU_OK(cudaMalloc((void **)&L->bs_d_cpls, n * sizeof(oimgpu_cpl)));
			L->bs_cap_reqs = n;
		}
		if (niovs > L->bs_cap_iovs) {
			cudaFree(L->bs_d_iovs);
			CU_OK(cudaMalloc((void **)&L->bs_d_iovs, (size_t)std::max<uint32_t>(niovs, 1) * sizeof(oimgpu_iov)));
			L->bs_cap_iovs = niovs;
		}
	}
	auto pinned = [](const void *p) {
		cudaPointerAttributes a;
		if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { (void)cudaGetLastError(); return false; }
		return a.type == cudaMemoryTypeHost;
	};
	const bool pin_in = pinned(reqs) && (niovs == 0 || pinned(iovs));
	const bool pin_out = pinned(cpls);
	const size_t need = (pin_in ? 0 : n * sizeof(oimgpu_req) + (size_t)niovs * sizeof(oimgpu_iov)) +
			    (pin_out ? 0 : n * sizeof(oimgpu_cpl));
	if (need > L->bs_h_cap) {
		CU_OK(cudaStreamSynchronize(L->stream));
		if (L->bs_h_pin) {
			/* cudaFreeHost waits for every GPU the memory is mapped into: see park_pollers_locked */
			std::lock_guard<std::mutex> lk(g.mu);
			auto parked = park_pollers_locked(-1, L);
			cudaFreeHost(L->bs_h_pin);
			unpark_pollers_locked(parked);
		}
		L->bs_h_pin = nullptr;
		CU_OK(cudaHostAlloc((void **)&L->bs_h_pin, need, cudaHostAllocDefault));
		L->bs_h_cap = need;
	}
	uint8_t *bounce = L->bs_h_pin;
	const oimgpu_iov *src_iovs = iovs;
	const oimgpu_req *src_reqs = reqs;
	if (!pin_in) {
		/* SG table first (small), then requests group by group so the GPU starts early */
		memcpy(bounce, iovs, (size_t)niovs * sizeof(oimgpu_iov));
		src_iovs = (const oimgpu_iov *)bounce;
		bounce += (size_t)niovs * sizeof(oimgpu_iov);
		src_reqs = (const oimgpu_req *)bounce;
		bounce += n * sizeof(oimgpu_req);
	}
	oimgpu_cpl *h_cpls = pin_out ? cpls : (oimgpu_cpl *)bounce;
	if (niovs) CU_OK(cudaMemcpyAsync(L->bs_d_iovs, src_iovs, (size_t)niovs * sizeof(oimgpu_iov), cudaMemcpyHostToDevice, L->stream));
	const uint32_t groups = pin_in ? 1 : std::min<uint32_t>(8, nq);
	int kicked = 0;
	for (uint32_t g = 0; g < groups; g++) {
		const uint32_t q0 = (uint32_t)((uint64_t)nq * g / groups), q1 = (uint32_t)((uint64_t)nq * (g + 1) / groups);
		const size_t r0 = (size_t)q0 * per_q, rn = (size_t)(q1 - q0) * per_q;
		if (!pin_in) memcpy(const_cast<oimgpu_req *>(src_reqs) + r0, reqs + r0, rn * sizeof(oimgpu_req));
		CU_OK(cudaMemcpyAsync(L->bs_d_reqs + r0, src_reqs + r0, rn * sizeof(oimgpu_req), cudaMemcpyHostToDevice, L->stream));
		for (uint32_t q = q0; q < q1; q++) {
			Queue &Q = L->queues[q];
			if (Q.dev_count) return -EAGAIN;
			Q.dev_reqs = L->bs_d_reqs + (size_t)q * per_q;
			Q.dev_iovs = L->bs_d_iovs;
			Q.dev_cpls = L->bs_d_cpls + (size_t)q * per_q;
			Q.dev_count = per_q;
			Q.dev_iov_limit = niovs;
		}
		int rc = oimgpu_kick(L);
		if (rc < 0) return rc;
		kicked += rc;
		CU_OK(cudaMemcpyAsync(h_cpls + r0, L->bs_d_cpls + r0, rn * sizeof(oimgpu_cpl), cudaMemcpyDeviceToHost, L->stream));
	}
	L->bs_user_cpls = pin_out ? nullptr : cpls;
	L->bs_h_cpls = h_cpls;
	L->bs_pending = n;
	return kicked;
}

/* completes a host-array batch: wait, then hand the completions to the caller's array */
static int batch_finish(oimgpu_lun *L)
{
	if (L->poller_active) return -EBUSY;	/* the stream never drains while the poller is resident */
	CU_OK(cudaSetDevice(L->device));
	CU_OK(cudaStreamSynchronize(L->stream));
	if (L->bs_pending && L->bs_user_cpls) memcpy(L->bs_user_cpls, L->bs_h_cpls, L->bs_pending * sizeof(oimgpu_cpl));
	L->bs_pending = 0;
	L->bs_user_cpls = nullptr;
	return 0;
}

extern "C" int oimgpu_submit_and_wait(oimgpu_lun *L, uint32_t nq, uint32_t per_q, const oimgpu_req *reqs,
				      const oimgpu_iov *iovs, uint32_t niovs, oimgpu_cpl *cpls, int mem)
{
	int rc = oimgpu_submit_batch(L, nq, per_q, reqs, iovs, niovs, cpls, mem);
	if (rc < 0) return rc;
	if (L->poller_active && mem == OIMGPU_MEM_HOST) {
		for (uint32_t q = 0; q < nq; q++) {
			uint32_t got = 0;
			while (got < per_q) {
				int n = oimgpu_poll(L, q, cpls + (size_t)q * per_q + got, per_q - got, 1);
				if (n < 0) return n;
				got += (uint32_t)n;
			}
		}
		return 0;
	}
	return oimgpu_lun_sync(L);
}

static int read_iostat(oimgpu_lun *L, const LunCtx *d_ctx, oimgpu_iostat *out)
{
	if (L->poller_active) return -EBUSY;
	CU_OK(cudaSetDevice(L->device));
	CU_OK(cudaStreamSynchronize(L->stream));
	LunCtx c;
	CU_OK(cudaMemcpy(&c, d_ctx, sizeof(c), cudaMemcpyDeviceToHost));
	memset(out, 0, sizeof(*out));
	out->num_read_ops = c.stats[0];
	out->num_write_ops = c.stats[1];
	out->num_unmap_ops = c.stats[2];
	out->num_other_ops = c.stats[3];
	out->bytes_read = c.stats[4];
	out->bytes_written = c.stats[5];
	out->bytes_unmapped = c.stats[6];
	out->num_errors = c.stats[7];
	out->read_latency_ns = c.stats[8];
	out->write_latency_ns = c.stats[9];
	out->unmap_latency_ns = c.stats[10];
	out->kernel_launches = L->launches;
	return 0;
}

extern "C" int oimgpu_lun_iostat(oimgpu_lun *L, oimgpu_iostat *out)
{
	if (!L || !out) return -EINVAL;
	return read_iostat(L, L->d_ctx, out);
}

extern "C" int oimgpu_lun_target_iostat(oimgpu_lun *L, int scsi_target_num, oimgpu_iostat *out)
{
	if (!L || !out || scsi_target_num < 0 || scsi_target_num >= OIMGPU_CTRLR_MAX_DEVS) return -EINVAL;
	if (scsi_target_num == L->target) return read_iostat(L, L->d_ctx, out);
	std::lock_guard<std::mutex> lk(g.mu);
	if (L->peer_bdev[scsi_target_num].empty()) return -ENODEV;
	return read_iostat(L, L->d_peer[scsi_target_num], out);
}

/* spdk_bdev_get_device_stat as get_bdevs_iostat reports it (S/lib/bdev/rpc/bdev_rpc.c:50-110): the counters of
 * a bdev over its lifetime, whichever sessions and targets the I/O came through */
extern "C" int oimgpu_bdev_iostat(const char *name, oimgpu_iostat *out)
{
	if (!out) return -EINVAL;
	std::lock_guard<std::mutex> lk(g.mu);
	if (!g.inited) return -ENODEV;
	auto it = g.bdevs.find(name ? name : "");
	if (it == g.bdevs.end()) return -ENODEV;
	unsigned long long sum[12], v[12];
	memcpy(sum, it->second->retired, sizeof(sum));
	for (oimgpu_lun *L : g.handles) {
		if (L->bdev == it->first && read_ctx_stats(L->device, L->d_ctx, v)) {
			for (int k = 0; k < 8; k++) sum[k] += v[k];
		}
		for (int t = 0; t < OIMGPU_CTRLR_MAX_DEVS; t++) {
			if (L->peer_bdev[t] == it->first && read_ctx_stats(L->device, L->d_peer[t], v)) {
				for (int k = 0; k < 8; k++) sum[k] += v[k];
			}
		}
	}
	memset(out, 0, sizeof(*out));
	out->num_read_ops = sum[0];
	out->num_write_ops = sum[1];
	out->num_unmap_ops = sum[2];
	out->num_other_ops = sum[3];
	out->bytes_read = sum[4];
	out->bytes_written = sum[5];
	out->bytes_unmapped = sum[6];
	out->num_errors = sum[7];
	out->read_latency_ns = sum[8];
	out->write_latency_ns = sum[9];
	out->unmap_latency_ns = sum[10];
	return 0;
}

/* ---- NBD export (S/lib/nbd/nbd.c): OIM's local mode without a VM ------------------------------------ */

static bool read_full(int fd, void *buf, size_t n)
{
	size_t got = 0;
	while (got < n) {
		ssize_t r = read(fd, (char *)buf + got, n - got);
		if (r < 0 && errno == EINTR) continue;
		if (r <= 0) return false;
		got += (size_t)r;
	}
	return true;
}

static bool write_full(int fd, const void *buf, size_t n)
{
	size_t put = 0;
	while (put < n) {
		ssize_t r = send(fd, (const char *)buf + put, n - put, MSG_NOSIGNAL);
		if (r < 0 && errno == EINTR) continue;
		if (r <= 0) return false;
		put += (size_t)r;
	}
	return true;
}

/* Serve the kernel's NBD transmission protocol on `sock_fd` (the daemon's end of the socketpair whose
 * other end went to /dev/nbdX with NBD_SET_SOCK) until the peer disconnects: struct nbd_request in,
 * struct nbd_reply (+ payload for reads) out, as spdk_nbd_poll does (nbd.c:560-806).  The store stays
 * in HBM; payload crosses a pinned bounce buffer with the copy engine - this is a CPU-socket path by
 * nature (the reference moves every byte through the same socket), not a hot path.
 * Returns 0 on an orderly end (NBD_CMD_DISC or EOF), -EINVAL on a bad request magic, -errno otherwise. */
extern "C" int oimgpu_nbd_serve(const char *bdev_name, int sock_fd)
{
	uint8_t *stores[kMaxReplicas] = {};
	int devices[kMaxReplicas] = {};
	int nrep = 0;
	uint64_t size = 0;
	uint32_t bs = 0;
	std::string name = bdev_name ? bdev_name : "";
	{
		std::lock_guard<std::mutex> lk(g.mu);
		if (!g.inited || g.control_only) return -ENODEV;
		auto it = g.bdevs.find(name);
		if (it == g.bdevs.end()) return -ENODEV;
		Bdev &b = *it->second;
		nrep = (int)b.stores.size();
		for (int r = 0; r < nrep; r++) { stores[r] = b.stores[r]; devices[r] = b.devices[r]; }
		size = b.num_blocks * (uint64_t)b.block_size;
		bs = b.block_size;
		b.open_luns++;		/* pins the bdev like a session does */
	}
	int rc = 0;
	cudaStream_t st = nullptr;
	uint8_t *bounce = nullptr;
	size_t cap = 0;
	cudaSetDevice(devices[0]);
	if (cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking) != cudaSuccess) rc = -EIO;
	auto book = [&](int op, uint64_t bytes) {	/* get_bdevs_iostat counts these like any other bdev I/O */
		std::lock_guard<std::mutex> lk(g.mu);
		auto it = g.bdevs.find(name);
		if (it == g.bdevs.end()) return;
		it->second->retired[op] += 1;
		it->second->retired[4 + op] += bytes;
	};
	while (rc == 0) {
		uint8_t req[28];	/* struct nbd_request: magic, type, handle[8], from, len - big endian */
		if (!read_full(sock_fd, req, sizeof(req))) break;
		auto be32 = [](const uint8_t *p) { return (uint32_t)p[0] << 24 | (uint32_t)p[1] << 16 | (uint32_t)p[2] << 8 | p[3]; };
		if (be32(req) != 0x25609513u) { rc = -EINVAL; break; }
		const uint32_t type = be32(req + 4), len = be32(req + 24);
		uint64_t from = 0;
		for (int k = 0; k < 8; k++) from = from << 8 | req[16 + k];
		const uint32_t payload = (type == 0 || type == 1) ? len : 0;	/* only READ / WRITE carry one */
		if (payload > cap) {
			if (bounce) {
				std::lock_guard<std::mutex> lk(g.mu);
				auto parked = park_pollers_locked(-1);
				cudaFreeHost(bounce);
				unpark_pollers_locked(parked);
			}
			cap = ((size_t)payload + (1u << 20) - 1) & ~(size_t)((1u << 20) - 1);
			if (cudaHostAlloc((void **)&bounce, cap, cudaHostAllocDefault) != cudaSuccess) { bounce = nullptr; cap = 0; rc = -ENOMEM; break; }
		}
		if (type == 1 && payload && !read_full(sock_fd, bounce, payload)) break;
		if (type == 2) break;	/* NBD_CMD_DISC: nothing outstanding here, close */
		/* spdk_bdev_bytes_to_blocks + spdk_bdev_io_valid_blocks (bdev.c:2474-2509): whole blocks, inside the device */
		const bool range_ok = from % bs == 0 && len % bs == 0 && from <= size && len <= size - from;
		bool ok = false;
		cudaError_t e = cudaSuccess;
		switch (type) {
		case 0:		/* NBD_CMD_READ */
			ok = range_ok;
			if (ok && payload) e = cudaMemcpyAsync(bounce, stores[0] + from, payload, cudaMemcpyDeviceToHost, st);
			break;
		case 1:		/* NBD_CMD_WRITE */
			ok = range_ok;
			for (int r = 0; ok && payload && r < nrep && e == cudaSuccess; r++)
				e = cudaMemcpyAsync(stores[r] + from, bounce, payload, cudaMemcpyHostToDevice, st);
			break;
		case 3:		/* NBD_CMD_FLUSH: the whole device, a no-op for RAM */
			ok = true;
			break;
		case 4:		/* NBD_CMD_TRIM -> spdk_bdev_unmap: zero fill; "Can't unmap 0 bytes" (bdev.c:2796-2799) */
			ok = range_ok && len != 0;
			for (int r = 0; ok && len && r < nrep && e == cudaSuccess; r++) e = cudaMemsetAsync(stores[r] + from, 0, len, st);
			break;
		default:	/* unknown command: EIO (nbd.c:527-540) */
			break;
		}
		if (e == cudaSuccess) e = cudaStreamSynchronize(st);
		if (e != cudaSuccess) { (void)cudaGetLastError(); ok = false; }
		if (ok && (type == 0 || type == 1 || type == 4)) book(type == 0 ? 0 : type == 1 ? 1 : 2, len);
		uint8_t resp[16] = {0x67, 0x44, 0x66, 0x98, 0, 0, 0, (uint8_t)(ok ? 0 : EIO)};	/* struct nbd_reply */
		memcpy(resp + 8, req + 8, 8);
		if (!write_full(sock_fd, resp, sizeof(resp))) break;
		if (type == 0 && ok && payload && !write_full(sock_fd, bounce, payload)) break;
	}
	{
		std::lock_guard<std::mutex> lk(g.mu);
		if (bounce) {
			auto parked = park_pollers_locked(-1);
			cudaFreeHost(bounce);
			unpark_pollers_locked(parked);
		}
		auto it = g.bdevs.find(name);
		if (it != g.bdevs.end() && it->second->open_luns > 0) it->second->open_luns--;
	}
	if (st) cudaStreamDestroy(st);
	return rc;
}

/* session-visible target state: hot-remove flags (vhost_scsi.c:1093-1100, lun.c:171-176) */
extern "C" int oimgpu_lun_set_removed(oimgpu_lun *L, int removed, int lun_removed)
{
	if (!L) return -EINVAL;
	if (L->poller_active) return -EBUSY;
	CU_OK(cudaSetDevice(L->device));
	CU_OK(cudaStreamSynchronize(L->stream));
	L->h_ctx.removed = removed != 0;
	L->h_ctx.lun_removed = lun_removed != 0;
	CU_OK(h2d_sync(L, L->d_ctx, &L->h_ctx, offsetof(LunCtx, stats)));
	return 0;
}

/* ---- virtqueue mode --------------------------------------------------------------------------------- */

/* rte_vhost_memory table of the session (S/lib/vhost/rte_vhost/rte_vhost.h:52-66): guest-physical
 * ranges and the device-accessible address each one is mapped at */
extern "C" int oimgpu_lun_set_mem_table(oimgpu_lun *L, const oimgpu_mem_region *regions, uint32_t nregions)
{
	if (!L || (!regions && nregions) || nregions > (uint32_t)kMaxRegions) return -EINVAL;
	std::lock_guard<std::recursive_mutex> hl(L->mu);
	if (L->poller_active) return -EBUSY;
	CU_OK(cudaSetDevice(L->device));
	CU_OK(cudaStreamSynchronize(L->stream));
	L->h_ctx.nregions = nregions;
	for (uint32_t i = 0; i < nregions; i++) {
		L->h_ctx.region[i].gpa = regions[i].guest_phys_addr;
		L->h_ctx.region[i].size = regions[i].size;
		L->h_ctx.region[i].addr = regions[i].addr;
	}
	CU_OK(h2d_sync(L, L->d_ctx, &L->h_ctx, offsetof(LunCtx, stats)));
	return 0;
}

/* Attach a virtio split ring to queue q: the three areas rte_vhost_get_vhost_vring reports
 * (S/lib/vhost/vhost.c:1120-1134), as device-accessible addresses, plus the ring cursors. */
extern "C" int oimgpu_vq_attach(oimgpu_lun *L, uint32_t q, const void *desc, const void *avail, void *used,
				uint32_t size, uint16_t last_avail_idx, uint16_t last_used_idx)
{
	if (!L || q >= L->num_queues || !desc || !avail || !used) return -EINVAL;
	std::lock_guard<std::recursive_mutex> hl(L->mu);
	if (size == 0 || size > OIMGPU_MAX_VQ_SIZE || (size & (size - 1))) return -EINVAL;
	if (L->poller_active) return -EBUSY;
	CU_OK(cudaSetDevice(L->device));
	CU_OK(cudaStreamSynchronize(L->stream));
	CU_OK(ensure_iov_scratch(L));
	VqState st ={ last_avail_idx, last_used_idx, last_avail_idx, 0 };
	CU_OK(h2d_sync(L, L->d_vq_state + q, &st, sizeof(st)));
	Queue &Q = L->queues[q];
	Q.vq_desc = (const uint8_t *)desc;
	Q.vq_avail = (const uint8_t *)avail;
	Q.vq_used = (uint8_t *)used;
	Q.vq_size = size;
	Q.vq_pending = false;
	cudaPointerAttributes attr{};
	Q.vq_in_hbm = cudaPointerGetAttributes(&attr, used) == cudaSuccess && attr.type == cudaMemoryTypeDevice;
	(void)cudaGetLastError();
	return 0;
}

extern "C" int oimgpu_vq_detach(oimgpu_lun *L, uint32_t q, uint16_t *last_avail_idx, uint16_t *last_used_idx)
{
	if (!L || q >= L->num_queues || !L->queues[q].vq_size) return -EINVAL;
	std::lock_guard<std::recursive_mutex> hl(L->mu);
	if (L->poller_active) return -EBUSY;
	CU_OK(cudaSetDevice(L->device));
	CU_OK(cudaStreamSynchronize(L->stream));
	VqState st;
	CU_OK(cudaMemcpy(&st, L->d_vq_state + q, sizeof(st), cudaMemcpyDeviceToHost));
	if (last_avail_idx) *last_avail_idx = (uint16_t)st.last_avail;
	if (last_used_idx) *last_used_idx = (uint16_t)st.last_used;
	Queue &Q = L->queues[q];
	Q.vq_desc = Q.vq_avail = nullptr;
	Q.vq_used = nullptr;
	Q.vq_size = 0;
	Q.vq_pending = false;
	return 0;
}

/* The guest's "kick": process every attached ring up to its avail->idx (one launch, asynchronous). */
extern "C" int oimgpu_vq_kick(oimgpu_lun *L)
{
	if (!L) return -EINVAL;
	std::lock_guard<std::recursive_mutex> hl(L->mu);
	if (L->poller_active) return 0;	/* the resident kernel sees avail->idx by itself */
	int n = 0;
	for (auto &Q : L->queues) {
		if (Q.vq_size) { Q.vq_pending = true; n++; }
	}
	if (!n) return 0;
	return oimgpu_kick(L);
}

/* ---- persistent poller ("one reactor kernel per LUN") ------------------------------------------------ */

/* Launch oim_lun_queue_kernel in persistent mode on the LUN's stream: it stays resident and serves the
 * library rings of every queue (doorbell = tail index in mapped host memory) and every attached
 * virtqueue (doorbell = the guest's avail->idx) until oimgpu_lun_stop_poller().  While it runs,
 * oimgpu_kick() is a doorbell write and oimgpu_poll() reads the completion counter the kernel
 * publishes; nothing is launched per request.  idle_timeout_ms != 0 arms a watchdog that lets the
 * kernel leave after that long without work (tests use it so a lost host cannot wedge the GPU). */
extern "C" int oimgpu_lun_start_poller(oimgpu_lun *L, uint32_t max_ctas, uint32_t idle_timeout_ms)
{
	if (!L) return -EINVAL;
	std::lock_guard<std::recursive_mutex> hl(L->mu);
	if (L->poller_active) return -EALREADY;
	CU_OK(cudaSetDevice(L->device));
	CU_OK(cudaStreamSynchronize(L->stream));
	CU_OK(ensure_iov_scratch(L));
	const int slot = (int)(L->kicks % oimgpu_lun::kKickSlots);
	QueueDesc *h_desc = (QueueDesc *)(L->h_kick[slot] + sizeof(KickHeader));
	uint32_t nd = 0;
	std::vector<VqState> cursors(L->num_queues);
	CU_OK(cudaMemcpy(cursors.data(), L->d_vq_state, sizeof(VqState) * L->num_queues, cudaMemcpyDeviceToHost));
	std::vector<std::pair<uint32_t, VqState>> ring_cursor;
	for (uint32_t q = 0; q < L->num_queues; q++) {
		Queue &Q = L->queues[q];
		if (Q.dev_count || Q.tail != Q.kicked) return -EBUSY;	/* drain pending launches first */
		if (Q.vq_size) {
			h_desc[nd++] = desc_virtqueue(L, q);
		} else {
			QueueDesc &D = h_desc[nd++];
			D = desc_slot_ring(L, q);
			D.doorbell = &L->d_door[q].tail;
			D.done = &L->d_door[q].done;
			/* everything kicked so far was served by launches: the poller starts from there */
			L->h_door[q].tail = Q.kicked;
			L->h_door[q].done = Q.kicked;
			cursors[q].last_avail = Q.kicked;
		}
	}
	/* slot-ring cursors live in the same VqState array (virtqueues keep theirs); the dispatcher's view of
	 * every doorbell starts at "nothing new" */
	for (uint32_t q = 0; q < L->num_queues; q++) cursors[q].hint = cursors[q].last_avail;
	CU_OK(h2d_sync(L, L->d_vq_state, cursors.data(), sizeof(VqState) * L->num_queues));
	/* worker CTAs + one dispatcher CTA (KickHeader::dispatcher).  With fewer queues than that, the workers share
	 * the queues a pass at a time: up to a ring's worth of passes per queue can be in flight at once. */
	uint64_t want = 0;
	for (uint32_t q = 0; q < L->num_queues; q++) {
		const uint32_t depth = L->queues[q].vq_size ? L->queues[q].vq_size : L->queue_size;
		want += std::max<uint32_t>(1, std::min<uint32_t>(8, (depth + kPass - 1) / kPass));
	}
	uint32_t grid = (uint32_t)std::min<uint64_t>(std::max<uint64_t>(nd, want), (uint64_t)L->grid_cap - 1);
	if (max_ctas) grid = std::min(grid, max_ctas);
	if (grid == 0) grid = 1;
	/* (rings of 64 or fewer slots hold at most two passes: nothing to share, and the closed-loop round trip of a
	 * single small ring is shorter on the one-CTA-per-queue kernel) */
	const bool shared = nd < grid && grid >= 4 * nd && nd <= share_max_queues(L) && !getenv("OIMGPU_NO_SHARED_QUEUES");
	if (!shared) grid = std::min(grid, nd);
	if (shared) {
		std::vector<QShare> sh(nd);
		memset(sh.data(), 0, sizeof(QShare) * nd);
		for (uint32_t k = 0; k < nd; k++) {	/* descriptor k = queue k here: one descriptor per queue */
			sh[k].base_avail = cursors[k].last_avail;
			sh[k].base_used = cursors[k].last_used;
			sh[k].latched = 1;
		}
		CU_OK(h2d_sync(L, L->d_share, sh.data(), sizeof(QShare) * nd));
	}
	L->h_flags[0] = 0;
	L->h_flags[16] = 0;
	KickHeader *kh = (KickHeader *)L->h_kick[slot];
	memset(kh, 0, sizeof(*kh));
	kh->next = grid;
	kh->nqueues = nd;
	kh->persistent = 1;
	kh->idle_timeout_ms = idle_timeout_ms;
	kh->stop = L->d_flags;
	kh->exited = L->d_flags + 16;
	kh->dispatcher = 1;
	kh->shared = shared ? 1 : 0;
	kh->share = shared ? L->d_share : nullptr;
	CU_OK(cudaMemcpyAsync(L->d_kick, L->h_kick[slot], sizeof(KickHeader) + sizeof(QueueDesc) * nd, cudaMemcpyHostToDevice, L->stream));
	{
		uint32_t nv = 0;
		for (uint32_t q = 0; q < L->num_queues; q++) nv += L->queues[q].vq_size != 0;
		launch_queue_kernel(L, grid + 1, shared, nv == nd);
	}
	if (shared) L->shared_launches++;
	CU_OK(cudaGetLastError());
	CU_OK(cudaEventRecord(L->kick_ev[slot], L->stream));
	L->kicks++;
	L->launches++;
	L->poller_grid = grid + 1;	/* CTAs that report in `exited` when the poller winds down */
	L->poller_max_ctas = max_ctas;
	L->poller_idle_ms = idle_timeout_ms;
	L->poller_active = true;
	return (int)grid;
}

extern "C" int oimgpu_lun_stop_poller(oimgpu_lun *L)
{
	if (!L) return -EINVAL;
	std::lock_guard<std::recursive_mutex> hl(L->mu);
	if (!L->poller_active) return 0;
	CU_OK(cudaSetDevice(L->device));
	std::atomic_thread_fence(std::memory_order_seq_cst);
	L->h_flags[0] = 1;
	L->poller_active = false;
	CU_OK(cudaStreamSynchronize(L->stream));
	return 0;
}

/* 1 while the resident kernel is polling, 0 after it left (stop or watchdog) */
extern "C" int oimgpu_lun_poller_running(oimgpu_lun *L)
{
	if (!L) return -EINVAL;
	return L->poller_active && L->h_flags[16] < L->poller_grid;
}

/* ---- device-timed region helpers (bench.py times on the LUN's own stream) ------------------------- */

extern "C" int oimgpu_timer_create(void **start, void **stop)
{
	cudaEvent_t a, b;
	CU_OK(cudaEventCreate(&a));
	CU_OK(cudaEventCreate(&b));
	*start = a;
	*stop = b;
	return 0;
}

extern "C" int oimgpu_timer_record(oimgpu_lun *L, void *ev)
{
	if (!L || !ev) return -EINVAL;
	CU_OK(cudaSetDevice(L->device));
	CU_OK(cudaEventRecord((cudaEvent_t)ev, L->stream));
	return 0;
}

extern "C" int oimgpu_timer_elapsed_ms(void *start, void *stop, float *ms)
{
	CU_OK(cudaEventSynchronize((cudaEvent_t)stop));
	CU_OK(cudaEventElapsedTime(ms, (cudaEvent_t)start, (cudaEvent_t)stop));
	return 0;
}

extern "C" void oimgpu_timer_destroy(void *start, void *stop)
{
	if (start) cudaEventDestroy((cudaEvent_t)start);
	if (stop) cudaEventDestroy((cudaEvent_t)stop);
}

/* ---- copy-engine level ----------------------------------------------------------------------------- */

extern "C" int oimgpu_copy_submit(oimgpu_lun *L, void *dst, const void *src, uint64_t nbytes)
{
	if (!L || !dst || !src) return -EINVAL;
	if (nbytes == 0) return 0;
	CU_OK(cudaSetDevice(L->device));
	const uint64_t units = (nbytes + kUnitBytes - 1) / kUnitBytes;
	const uint32_t grid = (uint32_t)std::min<uint64_t>((units + 7) / 8, (uint64_t)L->sm_count * 8);
	oim_copy_kernel<<<grid, 256, 0, L->stream>>>((uint8_t *)dst, (const uint8_t *)src, nbytes);
	CU_OK(cudaGetLastError());
	L->launches++;
	return 0;
}

extern "C" int oimgpu_fill_submit(oimgpu_lun *L, void *dst, uint8_t fill, uint64_t nbytes)
{
	if (!L || !dst) return -EINVAL;
	if (nbytes == 0) return 0;
	CU_OK(cudaSetDevice(L->device));
	const uint32_t grid = (uint32_t)std::min<uint64_t>((nbytes / 16 + 255) / 256 + 1, (uint64_t)L->sm_count * 8);
	oim_fill_kernel<<<grid, 256, 0, L->stream>>>((uint8_t *)dst, fill, nbytes);
	CU_OK(cudaGetLastError());
	L->launches++;
	return 0;
}


/* ---- asynchronous copy channel (the engine behind integration/spdk/copy_engine_oimgpu.c) ------------- */

namespace {
std::mutex g_pin_mu;
std::map<uintptr_t, uintptr_t> g_pinned;	/* [start, end) of host ranges pinned by oimgpu_mem_ensure, disjoint */
}

static void unpin_all_host_ranges()
{
	std::lock_guard<std::mutex> lk(g_pin_mu);
	for (auto &kv : g_pinned) {
		if (cudaHostUnregister((void *)kv.first) != cudaSuccess) (void)cudaGetLastError();
	}
	g_pinned.clear();
}

static bool pin_range(uintptr_t a, uintptr_t b)
{
	cudaError_t e = cudaHostRegister((void *)a, b - a, cudaHostRegisterMapped | cudaHostRegisterPortable);
	if (e == cudaSuccess) return true;
	(void)cudaGetLastError();
	return e == cudaErrorHostMemoryAlreadyRegistered;	/* by someone else (cudaHostAlloc, oimgpu_mem_register): fine */
}

extern "C" int oimgpu_mem_ensure(const void *addr, size_t len)
{
	if (!g.inited || g.control_only) return -ENODEV;
	if (!addr || !len) return 0;
	cudaPointerAttributes attr{};
	if (cudaPointerGetAttributes(&attr, addr) == cudaSuccess && attr.type != cudaMemoryTypeUnregistered) {
		/* device memory, or host memory CUDA already knows: check the far end too (a range may straddle) */
		cudaPointerAttributes last{};
		if (cudaPointerGetAttributes(&last, (const uint8_t *)addr + len - 1) == cudaSuccess && last.type != cudaMemoryTypeUnregistered) return 0;
	}
	(void)cudaGetLastError();
	const uintptr_t page = 4096, big = 2u << 20;
	uintptr_t a = (uintptr_t)addr & ~(page - 1), b = ((uintptr_t)addr + len + page - 1) & ~(page - 1);
	std::lock_guard<std::mutex> lk(g_pin_mu);
	/* walk the gaps between what is already pinned */
	while (a < b) {
		auto it = g_pinned.upper_bound(a);
		if (it != g_pinned.begin()) {
			auto pv = std::prev(it);
			if (pv->second > a) { a = pv->second; continue; }	/* inside a pinned range: skip it */
		}
		uintptr_t gap_end = (it != g_pinned.end() && it->first < b) ? it->first : b;
		/* try the whole 2 MiB-aligned surroundings first (a big buffer then takes few registrations), clipped to
		 * the neighbours; fall back to exactly the pages asked for (the surroundings may not be mapped) */
		uintptr_t lo = a & ~(big - 1), hi = (gap_end + big - 1) & ~(big - 1);
		if (it != g_pinned.begin() && std::prev(it)->second > lo) lo = std::prev(it)->second;
		if (it != g_pinned.end() && it->first < hi) hi = it->first;
		if (!(lo == a && hi == gap_end) && pin_range(lo, hi)) {
			g_pinned[lo] = hi;
		} else if (pin_range(a, gap_end)) {
			g_pinned[a] = gap_end;
			lo = a; hi = gap_end;
		} else {
			return -EFAULT;
		}
		a = hi;
	}
	return 0;
}

struct oimgpu_copy_chan {
	int device = 0;
	int sm_count = 0;
	cudaStream_t stream = nullptr;
	struct Op { cudaEvent_t ev; void *tag; };
	std::deque<Op> inflight;
	std::vector<cudaEvent_t> spare;
	unsigned long long launches = 0;
};

extern "C" int oimgpu_copy_chan_open(int device, oimgpu_copy_chan **out)
{
	std::lock_guard<std::mutex> lk(g.mu);
	if (!g.inited || g.control_only) return -ENODEV;
	if (!out) return -EINVAL;
	int d = device < 0 ? g.devices[0].ordinal : device;
	const int slot = find_device_slot(d);
	if (slot < 0) return -EINVAL;
	auto c = std::make_unique<oimgpu_copy_chan>();
	c->device = d;
	c->sm_count = g.devices[slot].sm_count;
	CU_OK(cudaSetDevice(d));
	CU_OK(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
	*out = c.release();
	return 0;
}

extern "C" int oimgpu_copy_chan_close(oimgpu_copy_chan *c)
{
	if (!c) return -EINVAL;
	cudaSetDevice(c->device);
	cudaStreamSynchronize(c->stream);
	for (auto &op : c->inflight) cudaEventDestroy(op.ev);
	for (auto ev : c->spare) cudaEventDestroy(ev);
	cudaStreamDestroy(c->stream);
	delete c;
	return 0;
}

static int chan_record(oimgpu_copy_chan *c, void *tag)
{
	cudaEvent_t ev;
	if (!c->spare.empty()) { ev = c->spare.back(); c->spare.pop_back(); }
	else CU_OK(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
	CU_OK(cudaEventRecord(ev, c->stream));
	c->inflight.push_back({ev, tag});
	c->launches++;
	return 0;
}

extern "C" int oimgpu_copy_chan_copy(oimgpu_copy_chan *c, void *dst, const void *src, uint64_t nbytes, void *tag)
{
	if (!c || !dst || !src) return -EINVAL;
	int rc = oimgpu_mem_ensure(dst, nbytes);
	if (rc == 0) rc = oimgpu_mem_ensure(src, nbytes);
	if (rc) return rc;
	CU_OK(cudaSetDevice(c->device));
	if (nbytes) {
		const uint64_t units = (nbytes + kUnitBytes - 1) / kUnitBytes;
		const uint32_t grid = (uint32_t)std::min<uint64_t>((units + 7) / 8, (uint64_t)c->sm_count * 8);
		oim_copy_kernel<<<grid, 256, 0, c->stream>>>((uint8_t *)dst, (const uint8_t *)src, nbytes);
		CU_OK(cudaGetLastError());
	}
	return chan_record(c, tag);
}

extern "C" int oimgpu_copy_chan_fill(oimgpu_copy_chan *c, void *dst, uint8_t fill, uint64_t nbytes, void *tag)
{
	if (!c || !dst) return -EINVAL;
	int rc = oimgpu_mem_ensure(dst, nbytes);
	if (rc) return rc;
	CU_OK(cudaSetDevice(c->device));
	if (nbytes) {
		const uint32_t grid = (uint32_t)std::min<uint64_t>((nbytes / 16 + 255) / 256 + 1, (uint64_t)c->sm_count * 8);
		oim_fill_kernel<<<grid, 256, 0, c->stream>>>((uint8_t *)dst, fill, nbytes);
		CU_OK(cudaGetLastError());
	}
	return chan_record(c, tag);
}

extern "C" int oimgpu_copy_chan_poll(oimgpu_copy_chan *c, void **tags, int max)
{
	if (!c || (!tags && max > 0)) return -EINVAL;
	int n = 0;
	while (n < max && !c->inflight.empty()) {
		cudaError_t e = cudaEventQuery(c->inflight.front().ev);
		if (e == cudaErrorNotReady) { (void)cudaGetLastError(); break; }
		if (e != cudaSuccess) { (void)cudaGetLastError(); return -EIO; }
		tags[n++] = c->inflight.front().tag;
		c->spare.push_back(c->inflight.front().ev);
		c->inflight.pop_front();
	}
	return n;
}

extern "C" unsigned long long oimgpu_copy_chan_launches(const oimgpu_copy_chan *c) { return c ? c->launches : 0; }
