/*
 * mirror_check.cu - check and repair of a mirrored bdev (oimgpu_bdev_mirror_check): an exact block-by-block compare of
 * every replica with replica 0, and a copy of replica 0 over the blocks that differ, in HBM on replica 0's GPU.
 *
 * The kernels live here and not in lun_kernel.cu so that nothing they need can shift the register allocation of the
 * queue kernels; they reuse the queue kernels' vector loads and unit mover (ld_cg16, move_unit in lun_kernel.cuh).
 */
#include <cstdlib>

#include "host_state.h"

namespace {

constexpr int kCheckThreads = 256;
constexpr int kVecsPerLane = kUnitBytes / (32 * 16);	/* a warp's 4 KiB unit: 8 vectors of 16 B per lane */

/* the range [begin, end) in bytes of every store; bit b of `bitmap` is block first_block + b */
struct MirrorRange {
	uint8_t *store[kMaxReplicas];	/* replica 0 local; the others peer or imported mappings, as the write fan-out's */
	uint32_t nreplicas, block_size;
	uint64_t first_block, num_blocks;
	uint64_t begin, end;
	uint32_t *bitmap;
};

/* the bytes of a 16-byte vector in which x and y differ, as a 16-bit mask */
__device__ __forceinline__ uint32_t diff_bytes(const int4 &x, const int4 &y)
{
	const uint32_t w[4] = {(uint32_t)(x.x ^ y.x), (uint32_t)(x.y ^ y.y), (uint32_t)(x.z ^ y.z), (uint32_t)(x.w ^ y.w)};
	uint32_t m = 0;
#pragma unroll
	for (int j = 0; j < 16; j++) m |= ((w[j >> 2] >> (8 * (j & 3))) & 0xffu) ? 1u << j : 0u;
	return m;
}

/* mark the blocks that own the differing bytes of the vector at byte `pos`; bytes outside the range are ignored */
__device__ __noinline__ void mark_blocks(const MirrorRange &a, uint64_t pos, uint32_t diff)
{
	uint64_t blk = pos / a.block_size, bound = (blk + 1) * a.block_size, last = ~0ull;
	while (diff) {
		const uint64_t p = pos + (uint64_t)(__ffs(diff) - 1);
		diff &= diff - 1;
		if (p < a.begin || p >= a.end) continue;
		while (p >= bound) { blk++; bound += a.block_size; }
		if (blk == last) continue;
		last = blk;
		const uint64_t bit = blk - a.first_block;
		atomicOr(&a.bitmap[bit >> 5], 1u << (bit & 31));
	}
}

}  // namespace

/* Warps take 4 KiB units grid-stride.  Units are cut from the range widened to 16-byte boundaries: every store is an
 * allocation of its own (256-byte aligned), so a vector is aligned in all of them at once.  An aligned vector never
 * crosses a page and holds at least one byte of the range, so the widening reads only mapped memory; its bytes outside
 * the range are never marked. */
__global__ void __launch_bounds__(kCheckThreads)
oim_mirror_check_kernel(const __grid_constant__ MirrorRange a)
{
	const int lane = threadIdx.x & 31;
	const uint64_t lo = a.begin & ~15ull, hi = (a.end + 15) & ~15ull;
	const uint64_t nunits = (hi - lo + kUnitBytes - 1) / kUnitBytes;
	const uint64_t nwarps = (uint64_t)gridDim.x * (kCheckThreads / 32);
	for (uint64_t u = (uint64_t)blockIdx.x * (kCheckThreads / 32) + (threadIdx.x >> 5); u < nunits; u += nwarps) {
		const uint64_t base = lo + u * kUnitBytes;
		const uint32_t nv = (uint32_t)(min((uint64_t)kUnitBytes, hi - base) >> 4);
		int4 ref[kVecsPerLane];
		uint32_t diff[kVecsPerLane];
#pragma unroll
		for (int k = 0; k < kVecsPerLane; k++) {
			const uint32_t v = lane + 32 * k;
			diff[k] = 0;
			if (v < nv) ref[k] = ld_cg16(a.store[0] + base + (size_t)v * 16);
		}
#pragma unroll 1
		for (uint32_t r = 1; r < a.nreplicas; r++) {
			int4 x[kVecsPerLane];
#pragma unroll
			for (int k = 0; k < kVecsPerLane; k++) {
				const uint32_t v = lane + 32 * k;
				if (v < nv) x[k] = ld_cg16(a.store[r] + base + (size_t)v * 16);
			}
#pragma unroll
			for (int k = 0; k < kVecsPerLane; k++) {
				if (lane + 32 * k < nv) diff[k] |= diff_bytes(ref[k], x[k]);
			}
		}
#pragma unroll
		for (int k = 0; k < kVecsPerLane; k++) {
			if (diff[k]) mark_blocks(a, base + (size_t)(lane + 32 * k) * 16, diff[k]);
		}
	}
}

/* Warps take (block, 4 KiB piece of the block) items grid-stride, so that large blocks spread over the grid; an item
 * of a marked block copies replica 0's piece over every other replica's.  Blocks that matched are not written. */
__global__ void __launch_bounds__(kCheckThreads)
oim_mirror_repair_kernel(const __grid_constant__ MirrorRange a)
{
	const int lane = threadIdx.x & 31;
	const uint32_t pieces = (a.block_size + kUnitBytes - 1) / kUnitBytes;
	const uint64_t nitems = a.num_blocks * pieces;
	const uint64_t nwarps = (uint64_t)gridDim.x * (kCheckThreads / 32);
	for (uint64_t t = (uint64_t)blockIdx.x * (kCheckThreads / 32) + (threadIdx.x >> 5); t < nitems; t += nwarps) {
		const uint64_t bit = pieces == 1 ? t : t / pieces;
		if (!(a.bitmap[bit >> 5] >> (bit & 31) & 1)) continue;
		const uint32_t done = (uint32_t)(t - bit * pieces) * kUnitBytes;
		const uint32_t n = min(kUnitBytes, a.block_size - done);
		const uint64_t off = (a.first_block + bit) * a.block_size + done;
#pragma unroll 1
		for (uint32_t r = 1; r < a.nreplicas; r++) move_unit<true>(a.store[r] + off, a.store[0] + off, n, lane);
	}
}

/* runs of set bits of the host bitmap -> ranges (LBA order), and the number of set bits */
static void collect_ranges(const uint32_t *bits, uint64_t first_block, uint64_t num_blocks, uint64_t *ranges,
			   uint32_t max_ranges, oimgpu_mirror_check *out)
{
	uint64_t nruns = 0, start = 0;
	bool in_run = false;
	auto emit = [&](uint64_t end) {
		if (nruns < max_ranges) {
			ranges[2 * nruns] = first_block + start;
			ranges[2 * nruns + 1] = end - start;
		}
		nruns++;
	};
	const uint64_t nwords = (num_blocks + 31) / 32;
	for (uint64_t w = 0; w < nwords; w++) {
		const uint32_t x = bits[w];
		if (x == (in_run ? 0xffffffffu : 0u)) {
			out->mismatched_blocks += in_run ? 32 : 0;
			continue;
		}
		out->mismatched_blocks += (uint64_t)__builtin_popcount(x);
		for (int i = 0; i < 32; i++) {
			const bool set = x >> i & 1;
			if (set == in_run) continue;
			if (set) start = w * 32 + i;
			else emit(w * 32 + i);
			in_run = set;
		}
	}
	if (in_run) emit(num_blocks);	/* bits past num_blocks are never set */
	out->nranges = (uint32_t)std::min<uint64_t>(nruns, max_ranges);
	out->truncated = nruns > max_ranges;
}

extern "C" int oimgpu_bdev_mirror_check(const char *name, uint64_t offset_blocks, uint64_t num_blocks, int repair,
					uint64_t *ranges, uint32_t max_ranges, oimgpu_mirror_check *out)
{
	if (!out || (!ranges && max_ranges)) return -EINVAL;
	std::lock_guard<std::mutex> lk(g.mu);
	if (!g.inited || g.control_only) return -ENODEV;
	Bdev *b = find_bdev_locked(name);
	if (!b) return -ENODEV;
	if (b->replicas.size() < 2) return -ENOTSUP;
	if (offset_blocks > b->num_blocks || num_blocks > b->num_blocks - offset_blocks) return -EINVAL;
	/* an NBD export moves payload with no point at which it could be paused */
	if (b->nbd_exports) return -EBUSY;
	memset(out, 0, sizeof(*out));
	out->blocks_checked = num_blocks;
	if (num_blocks == 0) return 0;

	/* Writers in this process are held for the whole call: their resident pollers are parked (and restarted when
	 * `held` goes), and what they launched is waited for.  The sessions on replica 0's GPU are held too: a resident
	 * poller there could keep the check's CTAs from being scheduled. */
	const int dev0 = b->replicas[0].device;
	ParkedPollers held(dev0, b->name);
	if (int rc = held.drain()) return rc;
	const Device &dev = g.devices[find_device_slot(dev0)];
	CU_OK(cudaSetDevice(dev0));
	MirrorRange a;
	memset(&a, 0, sizeof(a));
	for (size_t r = 0; r < b->replicas.size(); r++) a.store[r] = b->replicas[r].store;
	a.nreplicas = (uint32_t)b->replicas.size();
	a.block_size = b->block_size;
	a.first_block = offset_blocks;
	a.num_blocks = num_blocks;
	a.begin = offset_blocks * b->block_size;
	a.end = a.begin + num_blocks * b->block_size;
	const size_t bitmap_bytes = (num_blocks + 31) / 32 * sizeof(uint32_t);
	/* the host copy is page-aligned and page-rounded: a pageable copy that shared a page with a range this process
	 * registered would be refused by the driver */
	const size_t host_bytes = (bitmap_bytes + 4095) & ~(size_t)4095;
	std::unique_ptr<uint32_t, decltype(&free)> h_bits((uint32_t *)aligned_alloc(4096, host_bytes), &free);
	if (!h_bits) return -ENOMEM;
	CU_OK(cudaMallocAsync((void **)&a.bitmap, bitmap_bytes, dev.util));
	auto run = [&]() -> cudaError_t {
		cudaError_t e = cudaMemsetAsync(a.bitmap, 0, bitmap_bytes, dev.util);
		if (e != cudaSuccess) return e;
		const uint64_t units = (((a.end + 15) & ~15ull) - (a.begin & ~15ull) + kUnitBytes - 1) / kUnitBytes;
		const uint64_t warps = kCheckThreads / 32;
		uint32_t grid = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>((units + warps - 1) / warps, (uint64_t)dev.sm_count * 8));
		oim_mirror_check_kernel<<<grid, kCheckThreads, 0, dev.util>>>(a);
		if ((e = cudaGetLastError()) != cudaSuccess) return e;
		if ((e = cudaMemcpyAsync(h_bits.get(), a.bitmap, bitmap_bytes, cudaMemcpyDeviceToHost, dev.util)) != cudaSuccess) return e;
		if ((e = cudaStreamSynchronize(dev.util)) != cudaSuccess) return e;
		collect_ranges(h_bits.get(), offset_blocks, num_blocks, ranges, max_ranges, out);
		if (!repair || !out->mismatched_blocks) return cudaSuccess;
		const uint64_t items = num_blocks * ((b->block_size + kUnitBytes - 1) / kUnitBytes);
		grid = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>((items + warps - 1) / warps, (uint64_t)dev.sm_count * 8));
		oim_mirror_repair_kernel<<<grid, kCheckThreads, 0, dev.util>>>(a);
		if ((e = cudaGetLastError()) != cudaSuccess) return e;
		if ((e = cudaStreamSynchronize(dev.util)) != cudaSuccess) return e;
		out->repaired_blocks = out->mismatched_blocks;
		return cudaSuccess;
	};
	const cudaError_t e = run();
	cudaFreeAsync(a.bitmap, dev.util);
	if (e != cudaSuccess) {
		fprintf(stderr, "oimgpu: mirror check of %s failed: %s\n", b->name.c_str(), cudaGetErrorString(e));
		(void)cudaGetLastError();
		return -EIO;
	}
	return 0;
}
