/*
 * control.cu - the control plane of liboimgpu.so: devices, bdevs, vhost-scsi controllers, config JSON.
 *
 * Control plane state mirrors what the SPDK daemon keeps for OIM's twelve RPCs
 * (bdev list: S/lib/bdev/bdev.c + bdev_malloc.c:378-443; vhost controllers and their 8 target
 * slots: S/lib/vhost/vhost_scsi.c:951-1103), the data plane launches oim_lun_queue_kernel on the
 * LUN's own CUDA stream.  There is deliberately no CPU implementation of the data path in this
 * library: without a usable CUDA device oimgpu_init() fails and every other call returns -ENODEV.
 */
#include <random>

#include "host_state.h"

Registry oimgpu::g;

int oimgpu::find_device_slot(int ordinal)
{
	for (size_t i = 0; i < g.devices.size(); i++) {
		if (g.devices[i].ordinal == ordinal) return (int)i;
	}
	return -1;
}

/* peer access from one GPU to another's memory, enabled on first use */
bool oimgpu::device_reachable(int from, int to)
{
	if (from == to) return true;
	int can = 0;
	if (cudaDeviceCanAccessPeer(&can, from, to) != cudaSuccess || !can) return false;
	cudaSetDevice(from);
	cudaError_t e = cudaDeviceEnablePeerAccess(to, 0);
	(void)cudaGetLastError();	/* "already enabled" or a refusal: neither may surface at a later launch check */
	return e == cudaSuccess || e == cudaErrorPeerAccessAlreadyEnabled;
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

static void release_store(const Replica &r)
{
	cudaSetDevice(r.device);
	if (r.imported) cudaIpcCloseMemHandle(r.store);
	else cudaFree(r.store);
	(void)cudaGetLastError();
}

/* Take a bdev apart once nothing uses it: own stores are freed (their bytes given back to their GPU's count, which
 * places later bdevs), imported ones closed, the histogram freed and the name unregistered.  The pollers of each
 * replica's GPU are parked around its release; the histogram goes with replica 0, on whose GPU it lives. */
static void drop_bdev_locked(Bdev *b)
{
	if (!g.control_only) {
		for (const Replica &r : b->replicas) {
			{
				ParkedPollers parked(r.device);
				release_store(r);
				b->hist.reset(parked);
			}
			if (!r.imported) g.devices[find_device_slot(r.device)].bytes_allocated -= b->num_blocks * (uint64_t)b->block_size;
		}
	}
	g.bdev_order.erase(std::remove(g.bdev_order.begin(), g.bdev_order.end(), b->name), g.bdev_order.end());
	g.bdevs.erase(g.bdevs.find(b->name));
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
	for (const Device &a : g.devices) {
		for (const Device &b : g.devices) device_reachable(a.ordinal, b.ordinal);
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


extern "C" void oimgpu_fini(void)
{
	std::lock_guard<std::mutex> lk(g.mu);
	if (!g.inited) return;
	if (!g.control_only) unpin_all_host_ranges();
	while (!g.bdevs.empty()) drop_bdev_locked(g.bdevs.begin()->second.get());
	g.control_only = false;
	g.ctrlrs.clear();
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

extern "C" int oimgpu_device_ordinal(int index)
{
	std::lock_guard<std::mutex> lk(g.mu);
	if (index < 0 || index >= (int)g.devices.size()) return -EINVAL;
	return g.devices[index].ordinal;
}

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

/* A bdev with an own store on each of `devs`, named `name` or, without one, `prefix` + `counter` (the counter advances
 * only when such a bdev is made).  *out: the registered bdev. */
static int create_bdev_locked(const char *name, const char *uuid, uint64_t num_blocks, uint32_t block_size,
			      const std::vector<int> &devs, const char *product, const char *prefix, int &counter, Bdev **out)
{
	if (!g.inited) return -ENODEV;
	/* create_malloc_disk: "Disk must be more than 0 blocks" (bdev_malloc.c:384-387); block size must
	 * be a positive multiple the SCSI layer can divide 4 MiB by */
	if (num_blocks == 0 || block_size == 0 || block_size > OIMGPU_MAX_XFER_BYTES) return -EINVAL;
	if (uuid && !uuid_valid(uuid)) return -EINVAL;
	const bool auto_named = !(name && name[0]);
	const std::string nm = auto_named ? prefix + std::to_string(counter) : name;
	if (g.bdevs.count(nm)) return -EEXIST;	/* spdk_bdev_register: name already in use */
	Bdev *b = (g.bdevs[nm] = std::make_unique<Bdev>()).get();
	g.bdev_order.push_back(nm);
	b->name = nm;
	b->product = product;
	b->uuid = uuid ? uuid : random_uuid();
	b->num_blocks = num_blocks;
	b->block_size = block_size;
	for (int d : devs) {
		Replica r;
		r.device = d;
		if (int rc = alloc_store(d, num_blocks * (uint64_t)block_size, &r.store)) {
			drop_bdev_locked(b);
			return rc;
		}
		b->replicas.push_back(r);
	}
	if (auto_named) counter++;
	*out = b;
	return 0;
}

extern "C" int oimgpu_bdev_create_malloc(const char *name, const char *uuid, uint64_t num_blocks,
					 uint32_t block_size, int device, char *name_out, size_t name_cap)
{
	std::lock_guard<std::mutex> lk(g.mu);
	if (!g.inited) return -ENODEV;
	int d = pick_device(device);
	if (d < 0) return -EINVAL;
	Bdev *b = nullptr;
	int rc = create_bdev_locked(name, uuid, num_blocks, block_size, {d}, "Malloc disk", "Malloc", g.malloc_disk_count, &b);
	if (rc == 0) copy_str(name_out, name_cap, b->name);
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
	Bdev *b = nullptr;
	int rc = create_bdev_locked(name, nullptr, size_bytes / block_size, block_size, {d}, "Ceph Rbd Disk",
				    "Ceph", g.rbd_count, &b);	/* bdev_rbd.c:732 */
	if (rc) return rc;
	b->pool_name = pool_name;
	b->rbd_name = rbd_name;
	b->user_id = user_id ? user_id : "";
	copy_str(name_out, name_cap, b->name);
	return 0;
}

extern "C" int oimgpu_bdev_create_mirror(const char *name, uint64_t num_blocks, uint32_t block_size,
					 const int *devices, int nreplicas, char *name_out, size_t name_cap)
{
	if (!devices) return -EINVAL;	/* placement by rule is the uuid entry point's */
	return oimgpu_bdev_create_mirror_uuid(name, nullptr, num_blocks, block_size, devices, nreplicas, name_out, name_cap);
}

extern "C" int oimgpu_bdev_create_mirror_uuid(const char *name, const char *uuid, uint64_t num_blocks, uint32_t block_size,
					      const int *devices, int nreplicas, char *name_out, size_t name_cap)
{
	std::lock_guard<std::mutex> lk(g.mu);
	if (!g.inited) return -ENODEV;
	if (nreplicas < 1 || nreplicas > kMaxReplicas) return -EINVAL;
	std::vector<int> devs;
	if (devices) {
		devs.assign(devices, devices + nreplicas);
	} else {
		/* replica 0 where construct_malloc_bdev would put it, replica r on the r-th next initialised GPU */
		const int first = find_device_slot(pick_device(-1));
		for (int r = 0; r < nreplicas; r++) devs.push_back(g.devices[(first + r) % g.devices.size()].ordinal);
	}
	for (int d : devs) {
		if (find_device_slot(d) < 0) return -EINVAL;
	}
	for (int r = 1; r < nreplicas; r++) {
		int can = 0;
		if (devs[0] != devs[r] && (cudaDeviceCanAccessPeer(&can, devs[0], devs[r]) != cudaSuccess || !can)) return -ENOTSUP;
	}
	Bdev *b = nullptr;
	int rc = create_bdev_locked(name, uuid, num_blocks, block_size, devs, "Malloc disk", "Mirror", g.malloc_disk_count, &b);
	if (rc == 0) copy_str(name_out, name_cap, b->name);
	return rc;
}

extern "C" int oimgpu_bdev_export_store(const char *name, int replica, void *handle_out)
{
	static_assert(sizeof(cudaIpcMemHandle_t) == OIMGPU_IPC_HANDLE_BYTES, "IPC handle size");
	std::lock_guard<std::mutex> lk(g.mu);
	if (!g.inited || g.control_only) return -ENODEV;
	if (!handle_out) return -EINVAL;
	Bdev *b = find_bdev_locked(name);
	if (!b) return -ENODEV;
	if (replica < 0 || replica >= (int)b->replicas.size() || b->replicas[replica].imported) return -EINVAL;
	CU_OK(cudaSetDevice(b->replicas[replica].device));
	cudaIpcMemHandle_t h;
	CU_OK(cudaIpcGetMemHandle(&h, b->replicas[replica].store));
	memcpy(handle_out, &h, sizeof(h));
	return 0;
}

extern "C" int oimgpu_bdev_create_mirror_remote(const char *name, uint64_t num_blocks, uint32_t block_size, int device,
						 const void *peer_handles, int npeers, char *name_out, size_t name_cap)
{
	return oimgpu_bdev_create_mirror_remote_uuid(name, nullptr, num_blocks, block_size, device, peer_handles, npeers,
						     name_out, name_cap);
}

extern "C" int oimgpu_bdev_create_mirror_remote_uuid(const char *name, const char *uuid, uint64_t num_blocks,
						     uint32_t block_size, int device, const void *peer_handles, int npeers,
						     char *name_out, size_t name_cap)
{
	std::lock_guard<std::mutex> lk(g.mu);
	if (!g.inited || g.control_only) return -ENODEV;
	if (!peer_handles || npeers < 1 || npeers >= kMaxReplicas) return -EINVAL;
	int d = pick_device(device);
	if (d < 0) return -EINVAL;
	Bdev *b = nullptr;
	int rc = create_bdev_locked(name, uuid, num_blocks, block_size, {d}, "Malloc disk", "Mirror", g.malloc_disk_count, &b);
	if (rc) return rc;
	CU_OK(cudaSetDevice(d));
	for (int r = 0; r < npeers; r++) {
		cudaIpcMemHandle_t h;
		memcpy(&h, (const uint8_t *)peer_handles + (size_t)r * sizeof(h), sizeof(h));
		void *p = nullptr;
		cudaError_t e = cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess);
		if (e != cudaSuccess) {
			fprintf(stderr, "oimgpu: cudaIpcOpenMemHandle failed: %s\n", cudaGetErrorString(e));
			(void)cudaGetLastError();
			drop_bdev_locked(b);
			return -EIO;
		}
		b->replicas.push_back({d, (uint8_t *)p, true, std::string((const char *)&h, sizeof(h))});
	}
	copy_str(name_out, name_cap, b->name);
	return 0;
}

extern "C" int oimgpu_bdev_replica_info(const char *name, int replica, int *device, int *imported)
{
	std::lock_guard<std::mutex> lk(g.mu);
	if (!g.inited) return -ENODEV;
	Bdev *b = find_bdev_locked(name);
	if (!b) return -ENODEV;
	if (replica < 0 || replica >= (int)b->replicas.size()) return -EINVAL;
	if (device) *device = b->replicas[replica].device;
	if (imported) *imported = b->replicas[replica].imported;
	return 0;
}

/* A planned move of an imported replica (mdadm --replace): the new store is filled from replica 0 and swapped in with
 * every session that reaches the mirror held, so no request ever sees a replica that is missing or behind. */
extern "C" int oimgpu_bdev_mirror_replace_remote(const char *name, int replica, const void *handle)
{
	if (!name || !handle) return -EINVAL;
	std::lock_guard<std::mutex> lk(g.mu);
	if (!g.inited || g.control_only) return -ENODEV;
	Bdev *b = find_bdev_locked(name);
	if (!b) return -ENODEV;
	/* only a mirror built from handles: the configuration dump can then name the new store */
	if (b->replicas.size() < 2) return -ENOTSUP;
	for (size_t r = 1; r < b->replicas.size(); r++) {
		if (!b->replicas[r].imported) return -ENOTSUP;
	}
	if (replica < 1 || replica >= (int)b->replicas.size()) return -EINVAL;
	/* by its bytes, before it is opened: what the driver does with a handle this process holds open is not ours to rely on */
	const std::string h((const char *)handle, OIMGPU_IPC_HANDLE_BYTES);
	for (const Replica &r : b->replicas) {
		if (r.ipc_handle == h) return -EINVAL;
	}
	if (b->nbd_exports) return -EBUSY;	/* an NBD export moves payload with no point at which it could be paused */

	/* as oimgpu_bdev_mirror_check: every session that reaches the bdev, and every session on replica 0's GPU, held
	 * and drained for the whole call */
	const int dev0 = b->replicas[0].device;
	ParkedPollers held(dev0, b->name);
	if (int rc = held.drain()) return rc;
	CU_OK(cudaSetDevice(dev0));
	cudaIpcMemHandle_t ih;
	memcpy(&ih, handle, sizeof(ih));
	void *p = nullptr;
	cudaError_t e = cudaIpcOpenMemHandle(&p, ih, cudaIpcMemLazyEnablePeerAccess);
	if (e != cudaSuccess) {
		fprintf(stderr, "oimgpu: cudaIpcOpenMemHandle failed: %s\n", cudaGetErrorString(e));
		(void)cudaGetLastError();
		return e == cudaErrorPeerAccessUnsupported ? -ENOTSUP : -EIO;
	}
	Replica &rep = b->replicas[replica];
	uint8_t *fresh = (uint8_t *)p, *old = rep.store;
	auto drop = [&](int rc) {
		cudaSetDevice(dev0);
		cudaIpcCloseMemHandle(fresh);
		(void)cudaGetLastError();
		return rc;
	};
	cudaPointerAttributes at;
	if (cudaPointerGetAttributes(&at, fresh) != cudaSuccess) return drop(-EIO);
	if (!device_reachable(dev0, at.device)) return drop(-ENOTSUP);
	const Device &dev = g.devices[find_device_slot(dev0)];
	e = cudaSetDevice(dev0);
	if (e == cudaSuccess) e = launch_copy(dev.util, dev.sm_count, fresh, b->replicas[0].store, b->num_blocks * (uint64_t)b->block_size);
	if (e == cudaSuccess) e = cudaStreamSynchronize(dev.util);
	if (e != cudaSuccess) {
		fprintf(stderr, "oimgpu: copy of %s replica 0 to its new replica %d failed: %s\n", b->name.c_str(), replica,
			cudaGetErrorString(e));
		return drop(-EIO);
	}
	const size_t field = offsetof(LunCtx, store) + sizeof(uint8_t *) * replica;
	int rc = publish_ctx_locked(b->name, field, &fresh, sizeof(fresh));
	if (rc) {
		publish_ctx_locked(b->name, field, &old, sizeof(old));
		return drop(rc);
	}
	release_store(rep);
	rep.store = fresh;
	rep.ipc_handle = h;
	return 0;
}

/* Everything already launched on the sessions' streams comes first.  A resident poller cannot be waited for: with one
 * running, quiescing its I/O is the caller's business. */
static int sync_session_streams_locked()
{
	for (oimgpu_lun *L : g.handles) {
		if (!L->poller_active) {
			CU_OK(cudaSetDevice(L->device));
			CU_OK(cudaStreamSynchronize(L->stream));
		}
	}
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
	CU_OK(cudaMallocAsync((void **)&d, 16, st));	/* stream-ordered: the free does not wait for a resident poller */
	CU_OK(cudaMemsetAsync(d, 0, 16, st));
	oim_digest_kernel<<<g.devices[slot].sm_count * 4, 256, 0, st>>>((const uint64_t *)dptr, nbytes / 8, d);
	unsigned long long h[2] = {0, 0};
	cudaError_t e = cudaMemcpyAsync(h, d, 16, cudaMemcpyDeviceToHost, st);
	if (e == cudaSuccess) e = cudaStreamSynchronize(st);
	cudaFreeAsync(d, st);
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
	Bdev *b = find_bdev_locked(name);
	if (!b) return -ENODEV;
	if (replica < 0 || replica >= (int)b->replicas.size()) return -EINVAL;
	const uint64_t size = b->num_blocks * (uint64_t)b->block_size;
	if (offset > size || nbytes > size - offset || (offset & 7)) return -EINVAL;
	int rc = sync_session_streams_locked();
	if (rc) return rc;
	return digest_locked(b->replicas[replica].device, b->replicas[replica].store + offset, nbytes, out);
}

extern "C" int oimgpu_bdev_delete(const char *name)
{
	std::lock_guard<std::mutex> lk(g.mu);
	if (!g.inited) return -ENODEV;
	Bdev *b = find_bdev_locked(name);
	if (!b) return -ENODEV;
	/* the peer-target contexts of controller-wide sessions let go of it below, as its targets go; every other use (a
	 * session opened on exactly this device, an NBD export, a bio channel) is checked BEFORE anything is taken apart: a
	 * failed delete must leave the targets where they were */
	int peer_refs = 0;
	for (oimgpu_lun *L : g.handles) {
		for_each_ctx(L, [&](const std::string &name, LunCtx *, LunCtx *h) { peer_refs += !h && name == b->name; return 0; });
	}
	if (b->opens > peer_refs) return -EBUSY;
	/* spdk_bdev_unregister hot-removes the SCSI LUNs built on the bdev (lun.c:213-260): the targets go */
	for (auto &kv : g.ctrlrs) {
		bool touched = false;
		for (int t = 0; t < OIMGPU_CTRLR_MAX_DEVS; t++) {
			if (kv.second->targets[t] == b->name) {
				g.scsi_slot_used[kv.second->scsi_id[t]] = false;
				kv.second->targets[t].clear();
				touched = true;
			}
		}
		if (touched && !g.control_only) refresh_ctrlr_sessions_locked(kv.first);
	}
	if (b->opens) return -EBUSY;
	drop_bdev_locked(b);
	return 0;
}

/* enable_bdev_histogram (S/lib/bdev/rpc/bdev_rpc.c:607-671, spdk_bdev_histogram_enable bdev.c:4367-4400): enabling starts
 * from an empty histogram, disabling drops it */
extern "C" int oimgpu_bdev_histogram_enable(const char *name, int enable)
{
	std::lock_guard<std::mutex> lk(g.mu);
	if (!g.inited) return -ENODEV;
	Bdev *b = find_bdev_locked(name);
	if (!b) return -ENODEV;
	if (g.control_only) return 0;	/* no data path: the histogram reads as empty either way */
	const int dev0 = b->replicas[0].device;
	CU_OK(cudaSetDevice(dev0));
	cudaStream_t st = g.devices[find_device_slot(dev0)].util;
	/* every open session's device-resident view of the bdev learns where its histogram is (or that it is gone) */
	if (enable) {
		if (!b->hist) CU_OK(b->hist.alloc(dev0, kHistBuckets));
		CU_OK(cudaMemsetAsync(b->hist.get(), 0, sizeof(unsigned long long) * kHistBuckets, st));
		CU_OK(cudaStreamSynchronize(st));
	} else if (!b->hist) {
		return 0;
	}
	unsigned long long *h = enable ? b->hist.get() : nullptr;
	int rc = publish_ctx_locked(b->name, offsetof(LunCtx, hist), &h, sizeof(h));
	if (rc || enable) return rc;
	/* kernels already launched may still tally: everything in flight first, resident pollers parked */
	ParkedPollers parked(kAllGpus);
	(void)sync_session_streams_locked();
	b->hist.reset(parked);
	return 0;
}

/* get_bdev_histogram (bdev_rpc.c:675-790): the kHistBuckets bucket counters.  Disabled: -EFAULT while anything has the
 * bdev open (the reference's per-channel histogram is NULL then), an empty histogram otherwise (no channel to ask) */
extern "C" int oimgpu_bdev_histogram_get(const char *name, uint64_t *buckets)
{
	std::lock_guard<std::mutex> lk(g.mu);
	if (!g.inited) return -ENODEV;
	Bdev *b = find_bdev_locked(name);
	if (!b) return -ENODEV;
	if (!buckets) return -EINVAL;
	memset(buckets, 0, sizeof(uint64_t) * kHistBuckets);
	if (!b->hist) return b->opens > 0 ? -EFAULT : 0;	/* I/O channels exist while a session runs (spdk_scsi_dev_allocate_io_channels) */
	if (g.control_only) return 0;
	CU_OK(cudaSetDevice(b->replicas[0].device));
	cudaStream_t st = g.devices[find_device_slot(b->replicas[0].device)].util;
	CU_OK(cudaMemcpyAsync(buckets, b->hist.get(), sizeof(uint64_t) * kHistBuckets, cudaMemcpyDeviceToHost, st));
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
	o->device = b.replicas[0].device;
	o->replicas = (uint32_t)b.replicas.size();
	o->device_ptr = (uint64_t)(uintptr_t)b.replicas[0].store;
}

extern "C" int oimgpu_bdev_get(const char *name, oimgpu_bdev_info *out)
{
	std::lock_guard<std::mutex> lk(g.mu);
	if (!g.inited) return -ENODEV;
	Bdev *b = find_bdev_locked(name);
	if (!b) return -ENODEV;
	if (out) fill_bdev_info(*b, out);
	return 0;
}

extern "C" int oimgpu_bdev_list(oimgpu_bdev_info *out, int max)
{
	std::lock_guard<std::mutex> lk(g.mu);
	int n = 0;
	for (auto &nm : g.bdev_order) {
		if (out && n < max) fill_bdev_info(*find_bdev_locked(nm.c_str()), &out[n]);
		n++;
	}
	return n;
}

static int raw_access(const char *name, int replica, uint64_t offset, void *host, uint64_t len, bool write)
{
	std::lock_guard<std::mutex> lk(g.mu);
	if (!g.inited || g.control_only) return -ENODEV;
	Bdev *b = find_bdev_locked(name);
	if (!b) return -ENODEV;
	if (replica < 0 || replica >= (int)b->replicas.size()) return -EINVAL;
	const Replica &r = b->replicas[replica];
	uint64_t size = b->num_blocks * (uint64_t)b->block_size;
	if (offset > size || len > size - offset) return -EINVAL;
	CU_OK(cudaSetDevice(r.device));
	int rc = sync_session_streams_locked();
	if (rc) return rc;
	CU_OK(cudaSetDevice(r.device));
	cudaStream_t st = g.devices[find_device_slot(r.device)].util;
	if (write) CU_OK(cudaMemcpyAsync(r.store + offset, host, len, cudaMemcpyHostToDevice, st));
	else CU_OK(cudaMemcpyAsync(host, r.store + offset, len, cudaMemcpyDeviceToHost, st));
	CU_OK(cudaStreamSynchronize(st));
	return 0;
}

static int copy_strided(int device, void *dst, size_t dpitch, const void *src, size_t spitch, size_t width, size_t rows,
			cudaMemcpyKind kind)
{
	if (!dst || !src || !width || !rows) return -EINVAL;
	std::lock_guard<std::mutex> lk(g.mu);
	if (!g.inited || g.control_only) return -ENODEV;
	const int slot = find_device_slot(device);
	if (slot < 0) return -EINVAL;
	CU_OK(cudaSetDevice(device));
	cudaStream_t st = g.devices[slot].util;
	CU_OK(cudaMemcpy2DAsync(dst, dpitch, src, spitch, width, rows, kind, st));
	CU_OK(cudaStreamSynchronize(st));
	return 0;
}

/* `rows` pieces of `width` bytes, `pitch` apart in device memory, gathered into host memory by the COPY ENGINE on the
 * device's housekeeping stream: how a host thread looks at ring indices in HBM while a resident poller holds every SM
 * slot (a kernel launched for the same purpose would wait for the poller to leave) */
extern "C" int oimgpu_read_strided(int device, void *dst, const void *src, size_t pitch, size_t width, size_t rows)
{
	return copy_strided(device, dst, width, src, pitch, width, rows, cudaMemcpyDeviceToHost);
}

/* the scatter counterpart (host -> device), e.g. a test guest publishing avail->idx on many rings in HBM */
extern "C" int oimgpu_write_strided(int device, void *dst, const void *src, size_t pitch, size_t width, size_t rows)
{
	return copy_strided(device, dst, pitch, src, width, width, rows, cudaMemcpyHostToDevice);
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
std::string oimgpu::ctrlr_key(const char *ctrlr)
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

Ctrlr *oimgpu::find_ctrlr_locked(const char *ctrlr)
{
	auto it = g.ctrlrs.find(ctrlr_key(ctrlr));
	return it == g.ctrlrs.end() ? nullptr : it->second.get();
}

Bdev *oimgpu::find_bdev_locked(const char *name)
{
	auto it = g.bdevs.find(name ? name : "");
	return it == g.bdevs.end() ? nullptr : it->second.get();
}

void oimgpu::open_bdev_locked(Bdev &b) { b.opens++; }

void oimgpu::close_bdev_locked(const std::string &name)
{
	Bdev *b = find_bdev_locked(name.c_str());
	if (b && b->opens > 0) b->opens--;
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
	Ctrlr *c = find_ctrlr_locked(ctrlr);
	if (!c) return -ENODEV;
	/* spdk_vhost_scsi_dev_add_tgt (vhost_scsi.c:951-1021) */
	if (scsi_target_num < 0) {
		for (scsi_target_num = 0; scsi_target_num < OIMGPU_CTRLR_MAX_DEVS; scsi_target_num++) {
			if (c->targets[scsi_target_num].empty()) break;
		}
		if (scsi_target_num == OIMGPU_CTRLR_MAX_DEVS) return -ENOSPC;
	} else {
		if (scsi_target_num >= OIMGPU_CTRLR_MAX_DEVS) return -EINVAL;
	}
	if (!bdev_name) return -EINVAL;
	if (!c->targets[scsi_target_num].empty()) return -EEXIST;
	if (!find_bdev_locked(bdev_name)) return -EINVAL;	/* spdk_scsi_dev_construct failed */
	int slot = 0;
	while (slot < 1024 && g.scsi_slot_used[slot]) slot++;
	if (slot == 1024) return -EINVAL;	/* spdk_scsi_dev_construct: no free device slot */
	g.scsi_slot_used[slot] = true;
	c->scsi_id[scsi_target_num] = slot;
	c->targets[scsi_target_num] = bdev_name;
	if (!g.control_only) refresh_ctrlr_sessions_locked(c->name);	/* hot-plug into running sessions */
	return scsi_target_num;
}

extern "C" int oimgpu_vhost_scsi_remove_target(const char *ctrlr, int scsi_target_num)
{
	std::lock_guard<std::mutex> lk(g.mu);
	if (!g.inited) return -ENODEV;
	Ctrlr *c = find_ctrlr_locked(ctrlr);
	if (!c) return -ENODEV;
	if (scsi_target_num < 0 || scsi_target_num >= OIMGPU_CTRLR_MAX_DEVS) return -EINVAL;
	if (c->targets[scsi_target_num].empty()) return -ENODEV;
	/* a session opened on exactly this target keeps serving it until it is closed (the reference
	 * defers the removal until the session has no task in flight, vhost_scsi.c:236-289); for every
	 * other session of the controller the target disappears now */
	g.scsi_slot_used[c->scsi_id[scsi_target_num]] = false;
	c->targets[scsi_target_num].clear();
	if (!g.control_only) refresh_ctrlr_sessions_locked(c->name);
	return 0;
}

extern "C" int oimgpu_vhost_ctrlr_remove(const char *ctrlr)
{
	std::lock_guard<std::mutex> lk(g.mu);
	if (!g.inited) return -ENODEV;
	Ctrlr *c = find_ctrlr_locked(ctrlr);
	if (!c) return -ENODEV;
	for (auto &t : c->targets) {
		if (!t.empty()) return -EBUSY;	/* vhost_scsi.c:837-842 */
	}
	g.ctrlr_order.erase(std::remove(g.ctrlr_order.begin(), g.ctrlr_order.end(), c->name), g.ctrlr_order.end());
	g.ctrlrs.erase(g.ctrlrs.find(c->name));
	return 0;
}

/* spdk_vhost_set_coalescing (S/lib/vhost/vhost.c:358-381): the threshold is kept as requests per statistics
 * interval of 10 ms (SPDK_VHOST_STATS_CHECK_INTERVAL_MS), so fewer than 100 IOPS rounds to nothing and is refused;
 * the delay must fit 32 bits of timer ticks (ours: nanoseconds) */
extern "C" int oimgpu_vhost_ctrlr_set_coalescing(const char *ctrlr, uint32_t delay_base_us, uint32_t iops_threshold)
{
	std::lock_guard<std::mutex> lk(g.mu);
	if (!g.inited) return -ENODEV;
	Ctrlr *c = find_ctrlr_locked(ctrlr);
	if (!c) return -ENODEV;
	if ((uint64_t)delay_base_us * 1000ull >= UINT32_MAX) return -EINVAL;
	if (iops_threshold * 10u / 1000u == 0) return -EINVAL;
	c->delay_base_us = delay_base_us;
	c->iops_threshold = iops_threshold;
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

static std::string base64(const std::string &in)
{
	static const char tbl[] = "ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789+/";
	const uint8_t *p = (const uint8_t *)in.data();
	const size_t n = in.size();
	std::string o;
	for (size_t i = 0; i < n; i += 3) {
		const uint32_t v = (uint32_t)p[i] << 16 | (i + 1 < n ? (uint32_t)p[i + 1] << 8 : 0) | (i + 2 < n ? p[i + 2] : 0);
		o += tbl[v >> 18];
		o += tbl[(v >> 12) & 63];
		o += i + 1 < n ? tbl[(v >> 6) & 63] : '=';
		o += i + 2 < n ? tbl[v & 63] : '=';
	}
	return o;
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
			const Bdev &b = *find_bdev_locked(nm.c_str());
			if (b.product == "Ceph Rbd Disk") {
				out += ",{\"method\":\"construct_rbd_bdev\",\"params\":{\"name\":" + json_escape(b.name) + ",\"pool_name\":" +
				       json_escape(b.pool_name) + ",\"rbd_name\":" + json_escape(b.rbd_name) + ",\"block_size\":" + std::to_string(b.block_size);
				if (!b.user_id.empty()) out += ",\"user_id\":" + json_escape(b.user_id);
				out += "}}";
			} else if (b.replicas.size() > 1) {
				/* a mirror: in-process replicas are placed again by the rule, imported ones opened again from their
				 * handles (which stay valid while the exporting process keeps its bdev) */
				out += ",{\"method\":\"construct_mirror_bdev\",\"params\":{\"name\":" + json_escape(b.name) + ",\"num_blocks\":" +
				       std::to_string(b.num_blocks) + ",\"block_size\":" + std::to_string(b.block_size) + ",\"uuid\":" + json_escape(b.uuid);
				std::string remote;
				for (const Replica &r : b.replicas) {
					if (r.imported) remote += (remote.empty() ? "\"" : ",\"") + base64(r.ipc_handle) + "\"";
				}
				if (remote.empty()) out += ",\"replicas\":" + std::to_string(b.replicas.size()) + "}}";
				else out += ",\"remote_replicas\":[" + remote + "]}}";
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
	Ctrlr *c = find_ctrlr_locked(ctrlr);
	if (!c) return -ENODEV;
	if (out) fill_ctrlr_info(*c, out);
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

/* spdk_bdev_get_device_stat as get_bdevs_iostat reports it (S/lib/bdev/rpc/bdev_rpc.c:50-110): the counters of
 * a bdev over its lifetime, whichever sessions and targets the I/O came through */
extern "C" int oimgpu_bdev_iostat(const char *name, oimgpu_iostat *out)
{
	if (!out) return -EINVAL;
	std::lock_guard<std::mutex> lk(g.mu);
	if (!g.inited) return -ENODEV;
	Bdev *b = find_bdev_locked(name);
	if (!b) return -ENODEV;
	unsigned long long sum[12], v[12];
	memcpy(sum, b->retired, sizeof(sum));
	for (oimgpu_lun *L : g.handles) {
		for_each_ctx(L, [&](const std::string &bn, LunCtx *d, LunCtx *) {
			if (bn == b->name && read_ctx_stats(L->device, d, v)) {
				for (int k = 0; k < 12; k++) sum[k] += v[k];
			}
			return 0;
		});
	}
	iostat_from_stats(sum, out);
	return 0;
}

