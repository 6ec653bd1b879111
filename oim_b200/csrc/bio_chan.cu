/*
 * bio_chan.cu - the block-I/O channel: batches of READ / WRITE / WRITE_ZEROES / UNMAP with caller iovecs on one
 * HBM store, moved by oim_bio_kernel.  The engine behind integration/spdk/bdev_oimgpu.c (include/oimgpu.h).
 *
 * The kernel lives here and not in lun_kernel.cu so that nothing it needs can shift the register allocation of
 * the queue kernels; it reuses their unit movers (move_unit, zero_unit in lun_kernel.cuh).
 */
#include "host_state.h"

namespace {

/* one contiguous piece of one bio: store range <-> client range (client == nullptr: zero fill) */
struct BioSeg {
	uint8_t *store;
	uint8_t *client;
	uint64_t len;
	uint32_t first_unit;		/* exclusive prefix sum of 4 KiB units over the launch's segments */
	uint32_t op;			/* OIMGPU_BIO_* */
};
static_assert(sizeof(BioSeg) == 32, "BioSeg layout");

constexpr int kBioThreads = 256;
constexpr uint32_t kMaxUnitsPerLaunch = 1u << 30;

}  // namespace

/* Warps take 4 KiB units grid-stride and find their segment by binary search on first_unit, as the queue kernels'
 * movers do; a unit keeps its segment's alignment on both sides, so move_unit picks the aligned or the
 * byte-granular path per unit. */
__global__ void __launch_bounds__(kBioThreads)
oim_bio_kernel(const BioSeg *__restrict__ seg, uint32_t nseg, uint32_t nunits)
{
	const int lane = threadIdx.x & 31;
	const uint32_t nwarps = gridDim.x * (kBioThreads / 32);
	for (uint32_t u = blockIdx.x * (kBioThreads / 32) + (threadIdx.x >> 5); u < nunits; u += nwarps) {
		uint32_t lo = 0, hi = nseg;
		while (hi - lo > 1) {
			const uint32_t mid = (lo + hi) >> 1;
			if (seg[mid].first_unit <= u) lo = mid; else hi = mid;
		}
		const BioSeg g = seg[lo];
		const uint64_t off = (uint64_t)(u - g.first_unit) * kUnitBytes;
		const uint32_t n = (uint32_t)min((uint64_t)kUnitBytes, g.len - off);
		if (g.op == OIMGPU_BIO_READ) move_unit(g.client + off, g.store + off, n, lane);
		else if (g.op == OIMGPU_BIO_WRITE) move_unit(g.store + off, g.client + off, n, lane);
		else zero_unit(g.store + off, n, lane);
	}
}

struct oimgpu_bio_chan {
	std::string bdev;
	int device = 0;
	int sm_count = 0;
	uint8_t *store = nullptr;
	uint64_t num_blocks = 0;
	uint32_t block_size = 0;
	cudaStream_t stream = nullptr;
	/* the segments of one batch: built here, staged in pinned memory, uploaded in one copy.  One device array is
	 * enough - the upload of batch k+1 is behind batch k's launches on the stream.  Two staging buffers: batch k+1
	 * is built while batch k's upload may still be pending.  (Not a pageable copy: this process may have pinned
	 * pages next to any heap buffer, and the driver refuses a copy that straddles a registration.) */
	std::vector<BioSeg> segs;
	struct Staging { Buf<BioSeg, Mem::Pinned> h; uint64_t batch = 0; };
	Staging staging[2];
	std::vector<Buf<BioSeg, Mem::Pinned>> retired_staging;	/* outgrown, freed at close: a submit never parks pollers */
	uint64_t batches = 0, reaped = 0;
	std::vector<uint32_t> launch_end;	/* segments [launch_end[i-1], launch_end[i]) form launch i */
	std::vector<uint32_t> launch_units;
	BioSeg *d_segs = nullptr;
	size_t d_cap = 0;
	struct Range { uint64_t lo, hi; bool writes; };
	std::vector<Range> group;		/* store ranges of the launch being built */
	struct Batch { std::vector<oimgpu_bio_cpl> cpls; size_t next; };
	EventFifo<Batch> inflight;
	unsigned long long launches = 0;
};

extern "C" int oimgpu_bio_chan_open(const char *bdev_name, oimgpu_bio_chan **out)
{
	if (!bdev_name || !out) return -EINVAL;
	std::lock_guard<std::mutex> lk(g.mu);
	if (!g.inited || g.control_only) return -ENODEV;
	Bdev *b = find_bdev_locked(bdev_name);
	if (!b) return -ENODEV;
	if (b->replicas.size() != 1) return -ENOTSUP;	/* mirrored: the fan-out to replicas is not done here */
	auto c = std::make_unique<oimgpu_bio_chan>();
	c->bdev = b->name;
	c->device = b->replicas[0].device;
	c->sm_count = g.devices[find_device_slot(c->device)].sm_count;
	c->store = b->replicas[0].store;
	c->num_blocks = b->num_blocks;
	c->block_size = b->block_size;
	CU_OK(cudaSetDevice(c->device));
	CU_OK(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
	open_bdev_locked(*b);	/* oimgpu_bdev_delete returns -EBUSY while the channel is open */
	b->bio_chans++;	/* and an image save: a channel's submissions cannot be paused */
	*out = c.release();
	return 0;
}

extern "C" int oimgpu_bio_chan_close(oimgpu_bio_chan *c)
{
	if (!c) return -EINVAL;
	cudaSetDevice(c->device);
	cudaStreamSynchronize(c->stream);
	if (c->d_segs) cudaFreeAsync(c->d_segs, c->stream);	/* stream-ordered: does not wait for the whole device */
	cudaStreamSynchronize(c->stream);
	cudaStreamDestroy(c->stream);
	{
		std::lock_guard<std::mutex> lk(g.mu);
		ParkedPollers parked(kAllGpus);
		for (auto &st : c->staging) st.h.reset(parked);
		for (auto &h : c->retired_staging) h.reset(parked);
		close_bdev_locked(c->bdev);
		Bdev *b = find_bdev_locked(c->bdev.c_str());
		if (b && b->bio_chans > 0) b->bio_chans--;
	}
	delete c;
	return 0;
}

/* validate one bio (bdev_malloc_check_iov_len, bdev.c's range check) and emit its segments; 0 or -errno */
static int emit_bio(oimgpu_bio_chan *c, const oimgpu_bio &b, const oimgpu_iov *iovs, uint32_t niovs)
{
	if (b.op > OIMGPU_BIO_UNMAP || b.flags != 0) return -EINVAL;
	if (b.offset_blocks > c->num_blocks || b.num_blocks > c->num_blocks - b.offset_blocks) return -EINVAL;
	const uint64_t bytes = b.num_blocks * c->block_size;
	uint8_t *store = c->store + b.offset_blocks * c->block_size;
	if (b.op == OIMGPU_BIO_WRITE_ZEROES || b.op == OIMGPU_BIO_UNMAP) {
		if (bytes) c->segs.push_back({store, nullptr, bytes, 0, b.op});
		return 0;
	}
	if (b.iovcnt > niovs || b.iov_start > niovs - b.iovcnt) return -EINVAL;
	const oimgpu_iov *v = iovs + b.iov_start;
	uint64_t have = 0;
	for (uint32_t i = 0; i < b.iovcnt && have < bytes; i++) {
		if (v[i].flags != 0 || (v[i].len && !v[i].addr)) return -EINVAL;
		have += v[i].len;
	}
	if (have < bytes) return -EINVAL;
	/* exactly `bytes` move: an iovec list that holds more is cut where the bio ends */
	uint64_t left = bytes;
	for (uint32_t i = 0; i < b.iovcnt && left; i++) {
		const uint32_t take = (uint32_t)std::min<uint64_t>(v[i].len, left);
		if (take && oimgpu_mem_ensure((const void *)(uintptr_t)v[i].addr, take) != 0) return -EFAULT;
		left -= take;
	}
	left = bytes;
	for (uint32_t i = 0; i < b.iovcnt && left; i++) {
		const uint32_t take = (uint32_t)std::min<uint64_t>(v[i].len, left);
		if (!take) continue;
		c->segs.push_back({store, (uint8_t *)(uintptr_t)v[i].addr, take, 0, b.op});
		store += take;
		left -= take;
	}
	return 0;
}

extern "C" int oimgpu_bio_chan_submit(oimgpu_bio_chan *c, const oimgpu_bio *bios, uint32_t n, const oimgpu_iov *iovs, uint32_t niovs)
{
	if (!c || (!bios && n) || (!iovs && niovs)) return -EINVAL;
	if (n == 0) return 0;
	oimgpu_bio_chan::Batch batch{std::vector<oimgpu_bio_cpl>(n), 0};
	c->segs.clear();
	c->launch_end.clear();
	c->launch_units.clear();
	c->group.clear();
	uint32_t units = 0;
	for (uint32_t i = 0; i < n; i++) {
		const oimgpu_bio &b = bios[i];
		batch.cpls[i] = {b.tag, 0, 0};
		const size_t seg0 = c->segs.size();
		const int rc = emit_bio(c, b, iovs, niovs);
		if (rc) {
			c->segs.resize(seg0);
			batch.cpls[i].status = rc;
			continue;
		}
		if (c->segs.size() == seg0) continue;
		uint64_t bio_units = 0;
		for (size_t s = seg0; s < c->segs.size(); s++) bio_units += (c->segs[s].len + kUnitBytes - 1) / kUnitBytes;
		/* a launch ends before a bio whose store range overlaps one of the launch's where one of the two writes:
		 * inside a launch the units have no order */
		const uint64_t lo = b.offset_blocks * c->block_size, hi = lo + b.num_blocks * c->block_size;
		const bool writes = b.op != OIMGPU_BIO_READ;
		bool conflict = false;
		for (const auto &r : c->group) conflict |= lo < r.hi && r.lo < hi && (writes || r.writes);
		if (conflict || units + bio_units > kMaxUnitsPerLaunch) {
			if (units) { c->launch_end.push_back((uint32_t)seg0); c->launch_units.push_back(units); }
			units = 0;
			c->group.clear();
		}
		c->group.push_back({lo, hi, writes});
		for (size_t s = seg0; s < c->segs.size(); s++) {
			c->segs[s].first_unit = units;
			units += (uint32_t)((c->segs[s].len + kUnitBytes - 1) / kUnitBytes);
		}
	}
	if (units) { c->launch_end.push_back((uint32_t)c->segs.size()); c->launch_units.push_back(units); }
	CU_OK(cudaSetDevice(c->device));
	const uint64_t seq = ++c->batches;
	if (!c->segs.empty()) {
		const size_t bytes = c->segs.size() * sizeof(BioSeg);
		if (c->segs.size() > c->d_cap) {
			if (c->d_segs) CU_OK(cudaFreeAsync(c->d_segs, c->stream));
			c->d_segs = nullptr;
			c->d_cap = 0;
			const size_t cap = std::max<size_t>(c->segs.size() * 2, 1024);
			CU_OK(cudaMallocAsync((void **)&c->d_segs, cap * sizeof(BioSeg), c->stream));
			c->d_cap = cap;
		}
		auto &st = c->staging[seq & 1];
		if (st.batch > c->reaped) CU_OK(cudaEventSynchronize(c->inflight.entries[st.batch - c->reaped - 1].ev));	/* its upload is queued */
		if (c->segs.size() > st.h.size()) {
			if (st.h) c->retired_staging.push_back(std::move(st.h));
			CU_OK(st.h.alloc(c->device, std::max<size_t>(c->segs.size() * 2, 1024)));
		}
		memcpy(st.h.get(), c->segs.data(), bytes);
		st.batch = seq;
		CU_OK(cudaMemcpyAsync(c->d_segs, st.h.get(), bytes, cudaMemcpyHostToDevice, c->stream));
		uint32_t s0 = 0;
		for (size_t l = 0; l < c->launch_end.size(); l++) {
			const uint32_t s1 = c->launch_end[l], nu = c->launch_units[l];
			const uint32_t grid = std::max<uint32_t>(1, std::min<uint32_t>((nu + 7) / 8, (uint32_t)c->sm_count * 8));
			oim_bio_kernel<<<grid, kBioThreads, 0, c->stream>>>(c->d_segs + s0, s1 - s0, nu);
			CU_OK(cudaGetLastError());
			c->launches++;
			s0 = s1;
		}
	}
	return c->inflight.record(c->stream, std::move(batch));
}

extern "C" int oimgpu_bio_chan_poll(oimgpu_bio_chan *c, oimgpu_bio_cpl *out, int max)
{
	if (!c || (!out && max > 0)) return -EINVAL;
	return c->inflight.poll(max, [&](oimgpu_bio_chan::Batch &b, int &n) {
		while (n < max && b.next < b.cpls.size()) out[n++] = b.cpls[b.next++];
		if (b.next < b.cpls.size()) return false;
		c->reaped++;
		return true;
	});
}

extern "C" unsigned long long oimgpu_bio_chan_launches(const oimgpu_bio_chan *c) { return c ? c->launches : 0; }
