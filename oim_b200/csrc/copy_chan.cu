/*
 * copy_chan.cu - host memory for the GPU (registration, on-demand pinning) and the asynchronous copy channel.
 */
#include "host_state.h"

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
	{
		ParkedPollers parked(kAllGpus);
		cudaHostUnregister(addr);
	}
	g.registered.erase(it);
	return 0;
}

/* ---- asynchronous copy channel (the engine behind integration/spdk/copy_engine_oimgpu.c) ------------- */

namespace {
std::mutex g_pin_mu;
std::map<uintptr_t, uintptr_t> g_pinned;	/* [start, end) of host ranges pinned by oimgpu_mem_ensure, disjoint */
}

void oimgpu::unpin_all_host_ranges()
{
	std::lock_guard<std::mutex> lk(g_pin_mu);
	for (auto &kv : g_pinned) {
		if (cudaHostUnregister((void *)kv.first) != cudaSuccess) (void)cudaGetLastError();
	}
	g_pinned.clear();
}

bool oimgpu::host_range_pinned(const void *addr, size_t len)
{
	const uintptr_t a = (uintptr_t)addr;
	{
		std::lock_guard<std::mutex> lk(g_pin_mu);
		auto it = g_pinned.upper_bound(a);
		if (it != g_pinned.begin() && std::prev(it)->first <= a && a + len <= std::prev(it)->second) return true;
	}
	std::lock_guard<std::mutex> lk(g.mu);
	auto it = g.registered.upper_bound((void *)addr);
	return it != g.registered.begin() && (uintptr_t)std::prev(it)->first + std::prev(it)->second >= a + len;
}

static bool pin_range(uintptr_t a, uintptr_t b)
{
	if (cudaHostRegister((void *)a, b - a, cudaHostRegisterMapped | cudaHostRegisterPortable) == cudaSuccess) return true;
	(void)cudaGetLastError();
	return false;
}

/* a page CUDA already knows at its first or its last byte: registered or allocated pinned by another owner
 * (oimgpu_mem_register, cudaHostRegister, cudaHostAlloc) - theirs to keep or let go */
static bool foreign_page(uintptr_t p)
{
	for (uintptr_t q : {p, p + 4095}) {
		cudaPointerAttributes attr{};
		if (cudaPointerGetAttributes(&attr, (const void *)q) == cudaSuccess && attr.type != cudaMemoryTypeUnregistered) return true;
		(void)cudaGetLastError();
	}
	return false;
}

/* [a, b) could not be registered as a whole: pin each maximal run of its pages that no other owner holds.  Rare (a
 * range in, or straddling the edge of, another owner's buffer), so two driver queries per page are fine.  A run
 * that still fails - unmapped, or sharing a page with a registration that touches neither end of it - is refused,
 * never taken as pinned. */
static int pin_around_foreign(uintptr_t a, uintptr_t b)
{
	const uintptr_t page = 4096;
	while (a < b) {
		while (a < b && foreign_page(a)) a += page;
		uintptr_t e = a;
		while (e < b && !foreign_page(e)) e += page;
		if (e == a) break;
		if (!pin_range(a, e)) return -EFAULT;
		g_pinned[a] = e;
		a = e;
	}
	return 0;
}

int oimgpu::pin_host_pages(const void *addr, size_t len)
{
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
		 * the neighbours; fall back to exactly the pages asked for (the surroundings may not be mapped, or may
		 * overlap someone else's registration, which would leave part of them unpinned).  Where the exact pages
		 * cannot be registered either, they are taken page by page. */
		uintptr_t lo = a & ~(big - 1), hi = (gap_end + big - 1) & ~(big - 1);
		if (it != g_pinned.begin() && std::prev(it)->second > lo) lo = std::prev(it)->second;
		if (it != g_pinned.end() && it->first < hi) hi = it->first;
		if (!(lo == a && hi == gap_end) && pin_range(lo, hi)) {
			g_pinned[lo] = hi;
		} else {
			if (pin_range(a, gap_end)) g_pinned[a] = gap_end;
			else if (pin_around_foreign(a, gap_end) != 0) return -EFAULT;
			hi = gap_end;
		}
		a = hi;
	}
	return 0;
}

extern "C" int oimgpu_mem_ensure(const void *addr, size_t len)
{
	if (!g.inited || g.control_only) return -ENODEV;
	if (!addr || !len) return 0;
	/* host ranges the library pinned or registered are found without asking the driver.  Otherwise device memory
	 * is taken as it is, and host memory is pinned page by page: a range whose two ends CUDA knows may still have
	 * pages in between that nobody pinned. */
	if (host_range_pinned(addr, len)) return 0;
	cudaPointerAttributes attr{};
	if (cudaPointerGetAttributes(&attr, addr) == cudaSuccess &&
	    (attr.type == cudaMemoryTypeDevice || attr.type == cudaMemoryTypeManaged)) return 0;
	(void)cudaGetLastError();
	return pin_host_pages(addr, len);
}

struct oimgpu_copy_chan {
	int device = 0;
	int sm_count = 0;
	cudaStream_t stream = nullptr;
	EventFifo<void *> inflight;	/* the tag of each copy or fill */
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
	cudaStreamDestroy(c->stream);
	delete c;
	return 0;
}

extern "C" int oimgpu_copy_chan_copy(oimgpu_copy_chan *c, void *dst, const void *src, uint64_t nbytes, void *tag)
{
	if (!c || !dst || !src) return -EINVAL;
	int rc = oimgpu_mem_ensure(dst, nbytes);
	if (rc == 0) rc = oimgpu_mem_ensure(src, nbytes);
	if (rc) return rc;
	CU_OK(cudaSetDevice(c->device));
	if (nbytes) CU_OK(launch_copy(c->stream, c->sm_count, dst, src, nbytes));
	return c->inflight.record(c->stream, tag);
}

extern "C" int oimgpu_copy_chan_fill(oimgpu_copy_chan *c, void *dst, uint8_t fill, uint64_t nbytes, void *tag)
{
	if (!c || !dst) return -EINVAL;
	int rc = oimgpu_mem_ensure(dst, nbytes);
	if (rc) return rc;
	CU_OK(cudaSetDevice(c->device));
	if (nbytes) CU_OK(launch_fill(c->stream, c->sm_count, dst, fill, nbytes));
	return c->inflight.record(c->stream, tag);
}

extern "C" int oimgpu_copy_chan_poll(oimgpu_copy_chan *c, void **tags, int max)
{
	if (!c || (!tags && max > 0)) return -EINVAL;
	return c->inflight.poll(max, [&](void *tag, int &n) { tags[n++] = tag; return true; });
}

extern "C" unsigned long long oimgpu_copy_chan_launches(const oimgpu_copy_chan *c) { return c ? c->inflight.recorded : 0; }
