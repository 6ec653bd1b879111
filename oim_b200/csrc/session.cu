/*
 * session.cu - the data path of liboimgpu.so: sessions, submission, kicks, the resident poller.
 */
#include <atomic>

#include "host_state.h"

namespace oimgpu {
__global__ void oim_copy_kernel(uint8_t *dst, const uint8_t *src, uint64_t nbytes);
__global__ void oim_fill_kernel(uint8_t *dst, uint8_t fill, uint64_t nbytes);
}  // namespace oimgpu

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

/* what the kernel needs to know about one SCSI device: geometry, stores, and the identity strings
 * INQUIRY reports: spdk_scsi_dev_construct("Target N", ...) + port 0 "vhost", SAS
 * (vhost_scsi.c:1004-1013); the device id is the slot add_vhost_scsi_lun took in the global table */
static void fill_lun_ctx(LunCtx &c, const Bdev &b, const Ctrlr &ctrlr, int target)
{
	for (size_t r = 0; r < b.replicas.size(); r++) c.store[r] = b.replicas[r].store;
	c.nreplicas = (uint32_t)b.replicas.size();
	c.num_blocks = b.num_blocks;
	c.block_size = b.block_size;
	c.hist = b.hist.get();
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
bool oimgpu::read_ctx_stats(int device, const LunCtx *d_ctx, unsigned long long out[12])
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
	Bdev *b = find_bdev_locked(bdev.c_str());
	unsigned long long v[12];
	if (!b || !read_ctx_stats(device, d_ctx, v)) return;
	for (int k = 0; k < 12; k++) b->retired[k] += v[k];
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
		const Bdev *b = want.empty() ? nullptr : find_bdev_locked(want.c_str());
		if (b && !device_reachable(L->device, b->replicas[0].device)) b = nullptr;
		if (!b) want.clear();
		if (want != L->peer_bdev[t] && !L->peer_bdev[t].empty()) restart = true;	/* a device goes away */
		if (b && b->replicas.size() > 1 && !L->any_mirror) restart = true;	/* other kernel variant */
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
		/* before anything changes: a peer target that is named has its context (for_each_ctx visits it) */
		if (!want.empty() && !L->d_peer[t]) CU_OK(L->d_peer[t].alloc(L->device, 1));
		if (!L->peer_bdev[t].empty()) {
			close_bdev_locked(L->peer_bdev[t]);
			if (!L->poller_active) cudaStreamSynchronize(L->stream);
			retire_stats_locked(L->peer_bdev[t], L->device, L->d_peer[t].get());
		}
		L->peer_bdev[t] = want;
		if (want.empty()) {
			L->h_ctx.peer[t] = nullptr;	/* the context itself is freed at close: a resident kernel may still hold it */
			continue;
		}
		Bdev &b = *find_bdev_locked(want.c_str());
		open_bdev_locked(b);
		LunCtx c;
		memset(&c, 0, sizeof(c));
		fill_lun_ctx(c, b, *it->second, t);
		CU_OK(cudaMemcpyAsync(L->d_peer[t].get(), &c, sizeof(c), cudaMemcpyHostToDevice, L->copy_stream));
		CU_OK(cudaStreamSynchronize(L->copy_stream));	/* `c` is pageable stack memory */
		L->h_ctx.peer[t] = L->d_peer[t].get();
	}
	if (!changed) {
		if (restart && was_polling) return oimgpu_lun_start_poller(L, L->poller_max_ctas, L->poller_idle_ms) < 0 ? -EIO : 0;
		return 0;
	}
	L->any_mirror = L->h_ctx.nreplicas > 1;
	for (int t = 0; t < OIMGPU_CTRLR_MAX_DEVS; t++) {
		if (!L->peer_bdev[t].empty() && find_bdev_locked(L->peer_bdev[t].c_str())->replicas.size() > 1) L->any_mirror = true;
	}
	/* a launch still in flight finishes with the peers it started with: published under it, a mirror attached
	 * while the plain kernel runs would be served by a kernel that ignores Segment::mirror (GOOD, replica 0 only) */
	if (!L->poller_active) CU_OK(cudaStreamSynchronize(L->stream));
	/* publish the pointers after the contexts they point at (same stream); a separate stream so that a
	 * resident poller kernel on L->stream does not block the update */
	CU_OK(cudaMemcpyAsync((uint8_t *)L->d_ctx.get() + offsetof(LunCtx, peer), L->h_ctx.peer, sizeof(L->h_ctx.peer),
			      cudaMemcpyHostToDevice, L->copy_stream));
	CU_OK(cudaStreamSynchronize(L->copy_stream));
	if (restart && was_polling) {
		int rc = oimgpu_lun_start_poller(L, L->poller_max_ctas, L->poller_idle_ms);
		if (rc < 0) return rc;
	}
	return 0;
}

void oimgpu::refresh_ctrlr_sessions_locked(const std::string &ctrlr)
{
	for (oimgpu_lun *L : g.handles) {
		if (L->ctrlr == ctrlr) refresh_peers_locked(L);
	}
}

/* Write the `len` bytes at `value` at `offset` of every device-resident context of bdev `bdev` - a session's own and
 * the peer-target contexts of controller-wide sessions.  refresh_peers_locked rebuilds a context only when a target's
 * bdev name changes, so a field that changes under the same name (a histogram, a replica's store) needs this.  The
 * caller holds g.mu and makes sure that no kernel reads the field while it changes.  The host copy of a session's own
 * context changes too, since oimgpu_lun_set_removed and oimgpu_lun_set_mem_table upload it whole. */
int oimgpu::publish_ctx_locked(const std::string &bdev, size_t offset, const void *value, size_t len)
{
	for (oimgpu_lun *L : g.handles) {
		std::lock_guard<std::recursive_mutex> hl(L->mu);
		CU_OK(cudaSetDevice(L->device));
		int rc = for_each_ctx(L, [&](const std::string &name, LunCtx *d, LunCtx *h) {
			if (name != bdev) return 0;
			if (h) memcpy((uint8_t *)h + offset, value, len);
			CU_OK(cudaMemcpyAsync((uint8_t *)d + offset, value, len, cudaMemcpyHostToDevice, L->copy_stream));
			return 0;
		});
		if (rc) return rc;
		CU_OK(cudaStreamSynchronize(L->copy_stream));	/* `value` is pageable */
	}
	return 0;
}

/* ---- data path ----------------------------------------------------------------------------------- */

/* Take session L apart, whether lun_open_on got through or not (every member starts empty).  Caller holds g.mu and has
 * stopped L's poller.  L's pinned memory is mapped into every GPU: the other sessions' pollers are parked on all of them. */
static void destroy_session_locked(oimgpu_lun *L)
{
	ParkedPollers parked(kAllGpus, L);
	auto reset = [&](auto &...buf) { (buf.reset(parked), ...); };
	reset(L->h_door, L->h_mix, L->h_flags, L->slab, L->bs_h_pin, L->d_kick, L->d_share, L->d_vq_state,
	      L->d_iov_scratch, L->bs_d_reqs, L->bs_d_iovs, L->bs_d_cpls, L->d_ctx);
	for (auto &h : L->h_kick) h.reset(parked);
	for (auto &d : L->d_peer) d.reset(parked);
	cudaSetDevice(L->device);
	for (cudaEvent_t ev : L->kick_ev) if (ev) cudaEventDestroy(ev);
	if (L->copy_stream) cudaStreamDestroy(L->copy_stream);
	if (L->done) cudaEventDestroy(L->done);
	if (L->stream) cudaStreamDestroy(L->stream);
	(void)cudaGetLastError();
	g.handles.erase(std::remove(g.handles.begin(), g.handles.end(), L), g.handles.end());
	close_bdev_locked(L->bdev);
	for (const std::string &p : L->peer_bdev) close_bdev_locked(p);
	delete L;
}

static int lun_open_on(const char *ctrlr, int scsi_target_num, int on_device, uint32_t num_queues, uint32_t queue_size, oimgpu_lun **out)
{
	std::lock_guard<std::mutex> lk(g.mu);
	if (!g.inited || g.control_only) return -ENODEV;
	if (!out || num_queues == 0 || queue_size == 0 || (queue_size & (queue_size - 1)) ||
	    queue_size > OIMGPU_MAX_VQ_SIZE) return -EINVAL;
	Ctrlr *c = find_ctrlr_locked(ctrlr);
	if (!c) return -ENODEV;
	/* target -1: a controller-wide session (what a vhost-user connection is): no device of its own,
	 * every target is reached through peer[]; it lives on the GPU of the first target present */
	const bool session = scsi_target_num == -1;
	if (!session && (scsi_target_num < 0 || scsi_target_num >= OIMGPU_CTRLR_MAX_DEVS)) return -EINVAL;
	std::string bn;
	if (!session) {
		bn = c->targets[scsi_target_num];
		if (bn.empty()) return -ENODEV;
	}
	Bdev *bp = session ? nullptr : find_bdev_locked(bn.c_str());
	int session_device = g.devices[0].ordinal;
	for (int t = 0; session && t < OIMGPU_CTRLR_MAX_DEVS; t++) {
		if (!c->targets[t].empty()) { session_device = find_bdev_locked(c->targets[t].c_str())->replicas[0].device; break; }
	}
	if (on_device >= 0) {
		if (!session || find_device_slot(on_device) < 0) return -EINVAL;
		session_device = on_device;
	}

	/* whatever a failed step leaves behind (streams, events, buffers, bdev uses) is released here */
	std::unique_ptr<oimgpu_lun, void (*)(oimgpu_lun *)> L(new oimgpu_lun(), destroy_session_locked);
	L->ctrlr = c->name;
	L->bdev = bn;
	L->target = session ? 0xff : scsi_target_num;
	L->device = session ? session_device : bp->replicas[0].device;
	L->sm_count = g.devices[find_device_slot(L->device)].sm_count;
	L->num_queues = num_queues;
	L->queue_size = queue_size;
	L->iov_cap = queue_size * 8 < 1024 ? 1024 : queue_size * 8;	/* power of two >= 7 x 129 */
	if (bp) open_bdev_locked(*bp);
	CU_OK(cudaSetDevice(L->device));
	CU_OK(cudaStreamCreateWithFlags(&L->stream, cudaStreamNonBlocking));
	CU_OK(cudaStreamCreateWithFlags(&L->copy_stream, cudaStreamNonBlocking));
	CU_OK(cudaEventCreateWithFlags(&L->done, cudaEventDisableTiming));

	memset(&L->h_ctx, 0, sizeof(L->h_ctx));
	if (session) L->h_ctx.target = 0xff;
	else fill_lun_ctx(L->h_ctx, *bp, *c, scsi_target_num);
	CU_OK(L->h_mix.alloc(L->device, 8));
	memset((void *)L->h_mix.get(), 0, 64);
	L->any_mirror = L->h_ctx.nreplicas > 1;
	CU_OK(L->d_ctx.alloc(L->device, 1));
	CU_OK(h2d_sync(L.get(), L->d_ctx.get(), &L->h_ctx, sizeof(LunCtx)));

	for (int k = 0; k < oimgpu_lun::kKickSlots; k++) {
		CU_OK(L->h_kick[k].alloc(L->device, sizeof(KickHeader) + sizeof(QueueDesc) * num_queues * 3));
		memset(L->h_kick[k].get(), 0, sizeof(KickHeader));
		CU_OK(cudaEventCreateWithFlags(&L->kick_ev[k], cudaEventDisableTiming));
	}
	CU_OK(L->d_kick.alloc(L->device, sizeof(KickHeader) + sizeof(QueueDesc) * num_queues * 3));	/* ring + device-array + virtqueue per queue */
	L->d_desc = (QueueDesc *)(L->d_kick.get() + sizeof(KickHeader));
	CU_OK(L->d_share.alloc(L->device, (size_t)num_queues * 3));
	L->queues.resize(num_queues);
	/* one mapped pinned slab per LUN, carved into per-queue rings: the "virtqueues" */
	const size_t per_q = sizeof(oimgpu_req) * queue_size + sizeof(oimgpu_iov) * L->iov_cap + sizeof(oimgpu_cpl) * queue_size;
	CU_OK(L->slab.alloc(L->device, per_q * num_queues));
	uint8_t *slab = L->slab.get(), *dslab = nullptr;
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
	CU_OK(L->h_door.alloc(L->device, num_queues));
	CU_OK(cudaHostGetDevicePointer((void **)&L->d_door, L->h_door.get(), 0));
	memset((void *)L->h_door.get(), 0, sizeof(oimgpu_lun::Door) * num_queues);
	CU_OK(L->h_flags.alloc(L->device, 64));
	CU_OK(cudaHostGetDevicePointer((void **)&L->d_flags, (void *)L->h_flags.get(), 0));
	memset((void *)L->h_flags.get(), 0, 256);
	CU_OK(L->d_vq_state.alloc(L->device, num_queues));
	CU_OK(cudaMemsetAsync(L->d_vq_state.get(), 0, sizeof(VqState) * num_queues, L->stream));
	CU_OK(cudaStreamSynchronize(L->stream));
	int per_sm = 0;
	CU_OK(lun_kernels_init(&per_sm));
	if (per_sm < 1) per_sm = 1;
	L->grid_cap = L->sm_count * per_sm;
	int rc = refresh_peers_locked(L.get());
	if (rc) return rc;
	g.handles.push_back(L.get());
	*out = L.release();
	return 0;
}

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

extern "C" int oimgpu_lun_close(oimgpu_lun *L)
{
	if (!L) return -EINVAL;
	std::lock_guard<std::mutex> lk(g.mu);
	oimgpu_lun_stop_poller(L);
	cudaSetDevice(L->device);
	cudaStreamSynchronize(L->stream);
	for_each_ctx(L, [&](const std::string &bn, LunCtx *d, LunCtx *) {
		retire_stats_locked(bn, L->device, d);
		return 0;
	});
	destroy_session_locked(L);
	return 0;
}

extern "C" int oimgpu_lun_device(const oimgpu_lun *L) { return L ? L->device : -EINVAL; }
extern "C" long long oimgpu_lun_shared_launches(const oimgpu_lun *L) { return L ? (long long)L->shared_launches : -EINVAL; }
extern "C" void *oimgpu_lun_stream(oimgpu_lun *L) { return L ? (void *)L->stream : nullptr; }

/* Append n requests to queue Q's slot ring together with the SG entries iovs[lo, hi) they index, rebasing iov_start
 * from lo onto the ring's SG table.  -EAGAIN: the ring has no room; -E2BIG: the SG entries do not fit it. */
static int ring_append(oimgpu_lun *L, Queue &Q, const oimgpu_req *reqs, uint32_t n, const oimgpu_iov *iovs, uint32_t lo, uint32_t hi)
{
	if (n > L->queue_size - (Q.tail - Q.reaped)) return -EAGAIN;
	if (hi - lo > L->iov_cap) return -E2BIG;
	const uint32_t qmask = L->queue_size - 1, imask = L->iov_cap - 1;
	for (uint32_t i = lo; i < hi; i++) Q.h_iovs[(Q.iov_tail + (i - lo)) & imask] = iovs[i];
	for (uint32_t i = 0; i < n; i++) {
		oimgpu_req r = reqs[i];
		r.iov_start = r.iov_start - lo + Q.iov_tail;
		Q.h_reqs[(Q.tail + i) & qmask] = r;
	}
	Q.tail += n;
	Q.iov_tail += hi - lo;
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
	return ring_append(L, Q, reqs, nreqs, iovs, 0, niovs);
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
	launch_lun_kernel(k, grid, L->stream, L->d_ctx.get(), (KickHeader *)L->d_kick.get(), L->d_desc);
}

/* CTAs share the queues a pass at a time (KickHeader::shared) only while the queues alone cannot fill HBM with one CTA
 * each; above share_max_queues ownership is cheaper (tools/queue_sweep.py measures both sides, 4 KiB random read). */
static bool may_share_queues(const oimgpu_lun *L, uint32_t nd, uint32_t grid)
{
	return nd < grid && nd <= share_max_queues(L) && !getenv("OIMGPU_NO_SHARED_QUEUES");
}

/* where the next launch's QueueDesc records go, once the upload that last read that staging slot has run */
static int staged_descs(oimgpu_lun *L, QueueDesc **desc)
{
	const int slot = (int)(L->kicks % oimgpu_lun::kKickSlots);
	if (L->kicks >= (uint64_t)oimgpu_lun::kKickSlots) CU_OK(cudaEventSynchronize(L->kick_ev[slot]));
	*desc = (QueueDesc *)(L->h_kick[slot].get() + sizeof(KickHeader));
	return 0;
}

/* Upload header kh and the nd records staged_descs() handed out, and launch `grid` CTAs (+ kh.dispatcher) on them.
 * kh brings the persistent-mode fields, all zero for a run-to-completion launch. */
static int launch_staged(oimgpu_lun *L, KickHeader kh, uint32_t nd, uint32_t grid, bool shared)
{
	const int slot = (int)(L->kicks % oimgpu_lun::kKickSlots);
	const QueueDesc *desc = (const QueueDesc *)(L->h_kick[slot].get() + sizeof(KickHeader));
	bool vrings_only = true;
	for (uint32_t k = 0; k < nd; k++) vrings_only &= desc[k].mode == QMODE_VRING;
	kh.next = grid;		/* queues 0..grid-1 are taken statically by CTA index */
	kh.nqueues = nd;
	kh.shared = shared ? 1 : 0;
	kh.share = shared ? L->d_share.get() : nullptr;
	memcpy(L->h_kick[slot].get(), &kh, sizeof(kh));
	CU_OK(cudaMemcpyAsync(L->d_kick.get(), L->h_kick[slot].get(), sizeof(KickHeader) + sizeof(QueueDesc) * nd, cudaMemcpyHostToDevice, L->stream));
	CU_OK(cudaEventRecord(L->kick_ev[slot], L->stream));
	L->kicks++;
	launch_queue_kernel(L, grid + (kh.dispatcher ? 1 : 0), shared, vrings_only);
	CU_OK(cudaGetLastError());
	L->launches++;
	if (shared) L->shared_launches++;
	return 0;
}

/* ---- the QueueDesc records of a launch, one builder per kind of queue ---- */

/* caller-owned device arrays, served once from slot 0 */
static QueueDesc desc_device_arrays(oimgpu_lun *L, uint32_t q)
{
	const Queue &Q = L->queues[q];
	QueueDesc D;
	memset(&D, 0, sizeof(D));
	D.vq_state = L->d_vq_state.get() + q;
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
	D.vq_state = L->d_vq_state.get() + q;
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
	D.iovs = L->d_iov_scratch.get();
	D.vq_size = Q.vq_size;
	D.vq_desc = Q.vq_desc;
	D.vq_avail = Q.vq_avail;
	D.vq_used = Q.vq_used;
	D.vq_in_hbm = Q.vq_in_hbm ? 1 : 0;
	D.vq_state = L->d_vq_state.get() + q;
	return D;
}

/* [grid_cap][32][kIovRow] SG rows for the parser lanes of virtqueue mode */
static cudaError_t ensure_iov_scratch(oimgpu_lun *L)
{
	return L->d_iov_scratch ? cudaSuccess : L->d_iov_scratch.alloc(L->device, (size_t)L->grid_cap * kPass * kIovRow);
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
	QueueDesc *h_desc;
	int rc = staged_descs(L, &h_desc);
	if (rc) return rc;
	uint32_t nd = 0;
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
	/* Sharing pays only for read-dominated sessions: passes of different CTAs are ordered coarsely, a write-hot queue is
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
	const bool shared = !L->write_hot && may_share_queues(L, nd, grid);
	if (!shared) grid = std::min(grid, nd);
	if (shared) CU_OK(cudaMemsetAsync(L->d_share.get(), 0, sizeof(QShare) * nd, L->stream));
	KickHeader kh;
	memset(&kh, 0, sizeof(kh));	/* run-to-completion: persistent = 0 */
	rc = launch_staged(L, kh, nd, grid, shared);
	if (rc) return rc;
	CU_OK(cudaMemcpyAsync((void *)L->h_mix.get(), (const uint8_t *)L->d_ctx.get() + offsetof(LunCtx, mix), sizeof(unsigned long long) * 2,
			      cudaMemcpyDeviceToHost, L->stream));
	CU_OK(cudaEventRecord(L->done, L->stream));
	return (int)nd;
}

extern "C" int oimgpu_poll(oimgpu_lun *L, uint32_t q, oimgpu_cpl *cpls, uint32_t max, int wait)
{
	if (!L || q >= L->num_queues) return -EINVAL;
	Queue &Q = L->queues[q];
	if (Q.kicked == Q.reaped) return 0;
	uint32_t done = Q.kicked;	/* completions [reaped, done) are in the ring */
	if (L->poller_active) {
		done = L->h_door[q].done;
		if (wait) {
			while ((int32_t)(done - Q.kicked) < 0) {
				if (L->h_flags[16] >= L->poller_grid) return -ESHUTDOWN;	/* the poller left (watchdog) */
				done = L->h_door[q].done;
			}
		}
		std::atomic_thread_fence(std::memory_order_acquire);
	} else if (wait) {
		int rc = oimgpu_lun_sync(L);
		if (rc) return rc;
	} else if (cudaEventQuery(L->done) != cudaSuccess) {
		(void)cudaGetLastError();
		return 0;
	}
	uint32_t n = std::min(max, done - Q.reaped);
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
			int rc = ring_append(L, L->queues[q], r, per_q, iovs, lo, hi);
			if (rc) return rc;
		}
		return oimgpu_kick(L);
	}
	CU_OK(cudaSetDevice(L->device));
	if (L->bs_pending) return -EAGAIN;
	const size_t n = (size_t)nq * per_q;
	if (n > L->bs_d_reqs.size() || n > L->bs_d_cpls.size() || niovs > L->bs_d_iovs.size()) {
		CU_OK(cudaStreamSynchronize(L->stream));
		std::lock_guard<std::mutex> lk(g.mu);
		ParkedPollers parked(L->device, L);
		CU_OK(L->bs_d_reqs.grow(L->device, n, parked));
		CU_OK(L->bs_d_cpls.grow(L->device, n, parked));
		CU_OK(L->bs_d_iovs.grow(L->device, niovs, parked));
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
	if (need > L->bs_h_pin.size()) {
		CU_OK(cudaStreamSynchronize(L->stream));
		std::lock_guard<std::mutex> lk(g.mu);
		CU_OK(L->bs_h_pin.grow(L->device, need, ParkedPollers(L->bs_h_pin.waits_for(), L)));
	}
	uint8_t *bounce = L->bs_h_pin.get();
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
	if (niovs) CU_OK(cudaMemcpyAsync(L->bs_d_iovs.get(), src_iovs, (size_t)niovs * sizeof(oimgpu_iov), cudaMemcpyHostToDevice, L->stream));
	const uint32_t groups = pin_in ? 1 : std::min<uint32_t>(8, nq);
	int kicked = 0;
	for (uint32_t g = 0; g < groups; g++) {
		const uint32_t q0 = (uint32_t)((uint64_t)nq * g / groups), q1 = (uint32_t)((uint64_t)nq * (g + 1) / groups);
		const size_t r0 = (size_t)q0 * per_q, rn = (size_t)(q1 - q0) * per_q;
		if (!pin_in) memcpy(const_cast<oimgpu_req *>(src_reqs) + r0, reqs + r0, rn * sizeof(oimgpu_req));
		CU_OK(cudaMemcpyAsync(L->bs_d_reqs.get() + r0, src_reqs + r0, rn * sizeof(oimgpu_req), cudaMemcpyHostToDevice, L->stream));
		for (uint32_t q = q0; q < q1; q++) {
			Queue &Q = L->queues[q];
			if (Q.dev_count) return -EAGAIN;
			Q.dev_reqs = L->bs_d_reqs.get() + (size_t)q * per_q;
			Q.dev_iovs = L->bs_d_iovs.get();
			Q.dev_cpls = L->bs_d_cpls.get() + (size_t)q * per_q;
			Q.dev_count = per_q;
			Q.dev_iov_limit = niovs;
		}
		int rc = oimgpu_kick(L);
		if (rc < 0) return rc;
		kicked += rc;
		CU_OK(cudaMemcpyAsync(h_cpls + r0, L->bs_d_cpls.get() + r0, rn * sizeof(oimgpu_cpl), cudaMemcpyDeviceToHost, L->stream));
	}
	L->bs_user_cpls = pin_out ? nullptr : cpls;
	L->bs_h_cpls = h_cpls;
	L->bs_pending = n;
	return kicked;
}

/* wait for everything launched on the session's stream: -EBUSY under a resident poller, which never lets it drain */
static int drain_stream(oimgpu_lun *L)
{
	if (L->poller_active) return -EBUSY;
	CU_OK(cudaSetDevice(L->device));
	CU_OK(cudaStreamSynchronize(L->stream));
	return 0;
}

/* completes a host-array batch: wait, then hand the completions to the caller's array */
static int batch_finish(oimgpu_lun *L)
{
	if (int rc = drain_stream(L)) return rc;
	if (L->bs_pending && L->bs_user_cpls) memcpy(L->bs_user_cpls, L->bs_h_cpls, L->bs_pending * sizeof(oimgpu_cpl));
	L->bs_pending = 0;
	L->bs_user_cpls = nullptr;
	return 0;
}

extern "C" int oimgpu_lun_sync(oimgpu_lun *L)
{
	if (!L) return -EINVAL;
	std::lock_guard<std::recursive_mutex> hl(L->mu);
	return batch_finish(L);		/* stream sync + hand over the completions of a host-array batch */
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

/* the counters of LunCtx::stats as oimgpu_iostat reports them (kernel_launches left 0) */
void oimgpu::iostat_from_stats(const unsigned long long stats[12], oimgpu_iostat *out)
{
	memset(out, 0, sizeof(*out));
	out->num_read_ops = stats[0];
	out->num_write_ops = stats[1];
	out->num_unmap_ops = stats[2];
	out->num_other_ops = stats[3];
	out->bytes_read = stats[4];
	out->bytes_written = stats[5];
	out->bytes_unmapped = stats[6];
	out->num_errors = stats[7];
	out->read_latency_ns = stats[8];
	out->write_latency_ns = stats[9];
	out->unmap_latency_ns = stats[10];
}

static int read_iostat(oimgpu_lun *L, const LunCtx *d_ctx, oimgpu_iostat *out)
{
	if (int rc = drain_stream(L)) return rc;
	LunCtx c;
	CU_OK(cudaMemcpy(&c, d_ctx, sizeof(c), cudaMemcpyDeviceToHost));
	iostat_from_stats(c.stats, out);
	out->kernel_launches = L->launches;
	return 0;
}

extern "C" int oimgpu_lun_iostat(oimgpu_lun *L, oimgpu_iostat *out)
{
	if (!L || !out) return -EINVAL;
	return read_iostat(L, L->d_ctx.get(), out);
}

extern "C" int oimgpu_lun_target_iostat(oimgpu_lun *L, int scsi_target_num, oimgpu_iostat *out)
{
	if (!L || !out || scsi_target_num < 0 || scsi_target_num >= OIMGPU_CTRLR_MAX_DEVS) return -EINVAL;
	if (scsi_target_num == L->target) return read_iostat(L, L->d_ctx.get(), out);
	std::lock_guard<std::mutex> lk(g.mu);
	if (L->peer_bdev[scsi_target_num].empty()) return -ENODEV;
	return read_iostat(L, L->d_peer[scsi_target_num].get(), out);
}

/* session-visible target state: hot-remove flags (vhost_scsi.c:1093-1100, lun.c:171-176) */
extern "C" int oimgpu_lun_set_removed(oimgpu_lun *L, int removed, int lun_removed)
{
	if (!L) return -EINVAL;
	if (int rc = drain_stream(L)) return rc;
	L->h_ctx.removed = removed != 0;
	L->h_ctx.lun_removed = lun_removed != 0;
	CU_OK(h2d_sync(L, L->d_ctx.get(), &L->h_ctx, offsetof(LunCtx, stats)));
	return 0;
}

/* ---- virtqueue mode --------------------------------------------------------------------------------- */

/* rte_vhost_memory table of the session (S/lib/vhost/rte_vhost/rte_vhost.h:52-66): guest-physical
 * ranges and the device-accessible address each one is mapped at */
extern "C" int oimgpu_lun_set_mem_table(oimgpu_lun *L, const oimgpu_mem_region *regions, uint32_t nregions)
{
	if (!L || (!regions && nregions) || nregions > (uint32_t)kMaxRegions) return -EINVAL;
	std::lock_guard<std::recursive_mutex> hl(L->mu);
	if (int rc = drain_stream(L)) return rc;
	L->h_ctx.nregions = nregions;
	for (uint32_t i = 0; i < nregions; i++) {
		L->h_ctx.region[i].gpa = regions[i].guest_phys_addr;
		L->h_ctx.region[i].size = regions[i].size;
		L->h_ctx.region[i].addr = regions[i].addr;
	}
	CU_OK(h2d_sync(L, L->d_ctx.get(), &L->h_ctx, offsetof(LunCtx, stats)));
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
	if (int rc = drain_stream(L)) return rc;
	CU_OK(ensure_iov_scratch(L));
	VqState st ={ last_avail_idx, last_used_idx, last_avail_idx, 0 };
	CU_OK(h2d_sync(L, L->d_vq_state.get() + q, &st, sizeof(st)));
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
	if (int rc = drain_stream(L)) return rc;
	VqState st;
	CU_OK(cudaMemcpy(&st, L->d_vq_state.get() + q, sizeof(st), cudaMemcpyDeviceToHost));
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
	QueueDesc *h_desc;
	int rc = staged_descs(L, &h_desc);
	if (rc) return rc;
	uint32_t nd = 0;
	std::vector<VqState> cursors(L->num_queues);
	CU_OK(cudaMemcpy(cursors.data(), L->d_vq_state.get(), sizeof(VqState) * L->num_queues, cudaMemcpyDeviceToHost));
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
	CU_OK(h2d_sync(L, L->d_vq_state.get(), cursors.data(), sizeof(VqState) * L->num_queues));
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
	const bool shared = grid >= 4 * nd && may_share_queues(L, nd, grid);
	if (!shared) grid = std::min(grid, nd);
	if (shared) {
		std::vector<QShare> sh(nd);
		memset(sh.data(), 0, sizeof(QShare) * nd);
		for (uint32_t k = 0; k < nd; k++) {	/* descriptor k = queue k here: one descriptor per queue */
			sh[k].base_avail = cursors[k].last_avail;
			sh[k].base_used = cursors[k].last_used;
			sh[k].latched = 1;
		}
		CU_OK(h2d_sync(L, L->d_share.get(), sh.data(), sizeof(QShare) * nd));
	}
	L->h_flags[0] = 0;
	L->h_flags[16] = 0;
	KickHeader kh;
	memset(&kh, 0, sizeof(kh));
	kh.persistent = 1;
	kh.idle_timeout_ms = idle_timeout_ms;
	kh.stop = L->d_flags;
	kh.exited = L->d_flags + 16;
	kh.dispatcher = 1;
	rc = launch_staged(L, kh, nd, grid, shared);
	if (rc) return rc;
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

/* oim_copy_kernel / oim_fill_kernel over nbytes > 0 on `st`, sized for a GPU of sm_count SMs; the launch's error */
cudaError_t oimgpu::launch_copy(cudaStream_t st, int sm_count, void *dst, const void *src, uint64_t nbytes)
{
	const uint64_t units = (nbytes + kUnitBytes - 1) / kUnitBytes;
	const uint32_t grid = (uint32_t)std::min<uint64_t>((units + 7) / 8, (uint64_t)sm_count * 8);
	oim_copy_kernel<<<grid, 256, 0, st>>>((uint8_t *)dst, (const uint8_t *)src, nbytes);
	return cudaGetLastError();
}

cudaError_t oimgpu::launch_fill(cudaStream_t st, int sm_count, void *dst, uint8_t fill, uint64_t nbytes)
{
	const uint32_t grid = (uint32_t)std::min<uint64_t>((nbytes / 16 + 255) / 256 + 1, (uint64_t)sm_count * 8);
	oim_fill_kernel<<<grid, 256, 0, st>>>((uint8_t *)dst, fill, nbytes);
	return cudaGetLastError();
}

extern "C" int oimgpu_copy_submit(oimgpu_lun *L, void *dst, const void *src, uint64_t nbytes)
{
	if (!L || !dst || !src) return -EINVAL;
	if (nbytes == 0) return 0;
	CU_OK(cudaSetDevice(L->device));
	CU_OK(launch_copy(L->stream, L->sm_count, dst, src, nbytes));
	L->launches++;
	return 0;
}

extern "C" int oimgpu_fill_submit(oimgpu_lun *L, void *dst, uint8_t fill, uint64_t nbytes)
{
	if (!L || !dst) return -EINVAL;
	if (nbytes == 0) return 0;
	CU_OK(cudaSetDevice(L->device));
	CU_OK(launch_fill(L->stream, L->sm_count, dst, fill, nbytes));
	L->launches++;
	return 0;
}


