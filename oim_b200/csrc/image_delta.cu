/*
 * image_delta.cu - incremental volume images (oimgpu_bdev_image_track / _save_delta / _apply_delta): the 4 KiB granules
 * of a bdev that changed since its last save or load, written to a canonical delta file and applied back to every
 * replica (include/oimgpu.h gives the format).
 *
 * A tracked bdev keeps a 128-bit fingerprint per granule of the content at its baseline.  A delta save runs one pass over
 * replica 0 at HBM rate (oim_image_delta_scan_kernel) that fingerprints every granule into the spare table, marks the
 * granules whose fingerprint moved and those that hold a non-zero byte, and sums the whole-store digest on the way; only
 * the changed non-zero granules then cross PCIe, through bdev_image.cu's staging pipeline.  Nothing is added to the
 * queue kernels: a change is found by comparing content, so writes this process never saw (the exporter of an imported
 * replica writing its own bdev) are found too.
 *
 * The fingerprint of a granule is keyed and independent of oimgpu_bdev_digest: over its 64-bit words w_i (i counted
 * from the start of the store), the sums of fmix64(w_i ^ (k0 + i * phi)) and mix64(w_i ^ k1 ^ (i * psi)), with fmix64 the
 * murmur3 finaliser, mix64 the splitmix64 one and {k0, k1} a random key drawn when the bdev's tables are allocated.  The
 * same pass sums the unkeyed whole-store digest separately.  The format is defined by true byte difference, not by the
 * fingerprint: two contents of a granule with equal fingerprints would leave a changed granule out of the delta.  Since
 * the digest is a different function, such a delta then reaches apply with the digest of the real content, which the
 * store it leaves behind does not match, and oimgpu_bdev_image_apply_delta refuses it with -EIO; only a collision of the
 * fingerprint and of the digest at once would pass.  The key is not known outside the process, so a guest cannot aim
 * its writes at a fingerprint collision.
 */
#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>

#include <random>

#include "bdev_image.h"

namespace {

constexpr uint32_t kDeltaVersion = 1;
constexpr char kDeltaMagic[8] = {'O', 'I', 'M', 'G', 'P', 'U', 'D', 'L'};
constexpr uint64_t kZeroRun = 1ull << 63;	/* in a table entry's len: the run is now all zero */

/* the first 128 bytes of the 4096-byte header, little-endian: the image header's first 100, then the delta's own */
struct DeltaHeader {
	char magic[8];
	uint32_t version, block_size;
	uint64_t num_blocks;
	uint32_t granule_bytes, reserved;
	uint64_t nextents, data_bytes;
	uint64_t digest[2];
	char uuid[36];
	uint32_t reserved2;
	uint64_t parent_digest[2];
	uint64_t zero_bytes;
};
static_assert(offsetof(DeltaHeader, nextents) == 32 && offsetof(DeltaHeader, digest) == 48 && offsetof(DeltaHeader, uuid) == 64 &&
	      offsetof(DeltaHeader, reserved2) == 100 && offsetof(DeltaHeader, parent_digest) == 104 &&
	      offsetof(DeltaHeader, zero_bytes) == 120 && sizeof(DeltaHeader) == 128, "delta header layout");

struct DeltaScan {
	const uint8_t *store;
	uint64_t nbytes;
	const ulonglong2 *base;		/* the baseline's fingerprints, or nullptr: no changed bits */
	ulonglong2 *out;		/* this content's fingerprints */
	uint32_t *changed;		/* bit g: granule g's fingerprint differs from the baseline's */
	uint32_t *nonzero;		/* bit g: granule g holds a non-zero byte */
	unsigned long long *digest;	/* [2]: oimgpu_bdev_digest of the whole store, its last word zero-padded */
	uint64_t key[2];		/* the fingerprint's key (Bdev::track_key) */
};

/* the zero runs of a delta: run k covers store bytes [store_off, store_off + len), and data_off counts the zero bytes of
 * the runs before it, so the runs laid end to end are [0, total) */
struct DeltaZero {
	uint8_t *store[kMaxReplicas];	/* as ImageMove's: replica 0 local, the others peer or imported mappings */
	uint32_t nreplicas;
	const ImageSeg *segs;
	uint64_t nsegs, total;
};

__device__ __forceinline__ uint64_t mix64(uint64_t z)
{
	z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
	z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
	return z ^ (z >> 31);
}

__device__ __forceinline__ uint64_t fmix64(uint64_t z)
{
	z = (z ^ (z >> 33)) * 0xFF51AFD7ED558CCDull;
	z = (z ^ (z >> 33)) * 0xC4CEB9FE1A85EC53ull;
	return z ^ (z >> 33);
}

/* one word's terms: its fingerprint pair into f, its digest pair into d */
__device__ __forceinline__ void fold_word(uint64_t w, uint64_t i, const uint64_t key[2], uint64_t f[2], uint64_t d[2])
{
	f[0] += fmix64(w ^ (key[0] + i * 0x9E3779B97F4A7C15ull));
	f[1] += mix64(w ^ key[1] ^ (i * 0xD6E8FEB86659FD93ull));
	d[0] += w * (2 * i + 1);
	d[1] += mix64(w ^ i);
}

}  // namespace

/* Warps take granules grid-stride, as oim_image_scan_kernel: 8 vectors per lane in flight, the store read up to its end
 * widened to a 16-byte boundary (the store is an allocation of its own, 256-byte aligned, so an aligned vector that
 * holds one byte of it never leaves the allocation) and the bytes past the end masked.  A word counts in the
 * fingerprint and the digest when it starts inside the store, so the last partial word counts zero-padded, as the
 * digest rule of the images has it.  Each lane keeps its words' share of the digest across granules, and each CTA adds
 * one pair into it. */
__global__ void __launch_bounds__(kImageThreads)
oim_image_delta_scan_kernel(const __grid_constant__ DeltaScan a)
{
	__shared__ unsigned long long part[kImageThreads / 32][2];
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const uint64_t hi = (a.nbytes + 15) & ~15ull;
	const uint64_t nwords = (a.nbytes + 7) / 8;
	const uint64_t ngran = (a.nbytes + kGranule - 1) / kGranule;
	const uint64_t nwarps = (uint64_t)gridDim.x * (kImageThreads / 32);
	uint64_t dg[2] = {0, 0};
	for (uint64_t gi = (uint64_t)blockIdx.x * (kImageThreads / 32) + warp; gi < ngran; gi += nwarps) {
		const uint64_t base = gi * kGranule;
		const uint32_t nv = (uint32_t)(min((uint64_t)kGranule, hi - base) >> 4);
		int4 x[kGranule / 512];
#pragma unroll
		for (int k = 0; k < (int)(kGranule / 512); k++) {
			const uint32_t v = lane + 32 * k;
			x[k] = v < nv ? ld_cg16(a.store + base + (size_t)v * 16) : make_int4(0, 0, 0, 0);
		}
		ulonglong2 old = make_ulonglong2(0, 0);
		if (lane == 0 && a.base) old = a.base[gi];
		uint64_t f[2] = {0, 0};
		int acc = 0;
#pragma unroll
		for (int k = 0; k < (int)(kGranule / 512); k++) {
			const uint64_t pos = base + (uint64_t)(lane + 32 * k) * 16;
			if (pos < a.nbytes && pos + 16 > a.nbytes) keep_low_bytes(x[k], (uint32_t)(a.nbytes - pos));
			acc |= x[k].x | x[k].y | x[k].z | x[k].w;
			const uint64_t i = pos >> 3;
			const uint64_t w0 = (uint64_t)(uint32_t)x[k].x | (uint64_t)(uint32_t)x[k].y << 32;
			const uint64_t w1 = (uint64_t)(uint32_t)x[k].z | (uint64_t)(uint32_t)x[k].w << 32;
			if (i < nwords) fold_word(w0, i, a.key, f, dg);
			if (i + 1 < nwords) fold_word(w1, i + 1, a.key, f, dg);
		}
#pragma unroll
		for (int o = 16; o; o >>= 1) {
			f[0] += __shfl_xor_sync(0xffffffffu, f[0], o);
			f[1] += __shfl_xor_sync(0xffffffffu, f[1], o);
		}
		const bool nonzero = __any_sync(0xffffffffu, acc != 0);
		if (lane == 0) {
			if (a.base && (old.x != f[0] || old.y != f[1])) atomicOr(&a.changed[gi >> 5], 1u << (gi & 31));
			if (nonzero) atomicOr(&a.nonzero[gi >> 5], 1u << (gi & 31));
			a.out[gi] = make_ulonglong2(f[0], f[1]);
		}
	}
#pragma unroll
	for (int o = 16; o; o >>= 1) {
		dg[0] += __shfl_xor_sync(0xffffffffu, dg[0], o);
		dg[1] += __shfl_xor_sync(0xffffffffu, dg[1], o);
	}
	if (lane == 0) { part[warp][0] = dg[0]; part[warp][1] = dg[1]; }
	__syncthreads();
	if (threadIdx.x == 0) {
		unsigned long long s0 = 0, s1 = 0;
		for (int w = 0; w < kImageThreads / 32; w++) { s0 += part[w][0]; s1 += part[w][1]; }
		atomicAdd(&a.digest[0], s0);
		atomicAdd(&a.digest[1], s1);
	}
}

/* Warps take the 4 KiB units of the zero runs laid end to end grid-stride and find each unit's run by binary search, as
 * oim_image_move_kernel finds an extent.  Runs start on granule boundaries in the store and in the concatenation alike,
 * and only the last run of the store can end elsewhere, so a unit never spans two runs. */
__global__ void __launch_bounds__(kImageThreads)
oim_image_delta_zero_kernel(const __grid_constant__ DeltaZero a)
{
	const int lane = threadIdx.x & 31;
	const uint64_t nunits = (a.total + kUnitBytes - 1) / kUnitBytes;
	const uint64_t nwarps = (uint64_t)gridDim.x * (kImageThreads / 32);
	for (uint64_t u = (uint64_t)blockIdx.x * (kImageThreads / 32) + (threadIdx.x >> 5); u < nunits; u += nwarps) {
		const uint64_t pos = u * kUnitBytes;
		uint64_t lo = 0, hi = a.nsegs;	/* the last run that starts at or before pos */
		while (hi - lo > 1) {
			const uint64_t mid = (lo + hi) >> 1;
			if (a.segs[mid].data_off <= pos) lo = mid;
			else hi = mid;
		}
		const ImageSeg s = a.segs[lo];
		const uint32_t n = (uint32_t)min((uint64_t)kUnitBytes, s.data_off + s.len - pos);
		const uint64_t off = s.store_off + (pos - s.data_off);
#pragma unroll 1
		for (uint32_t r = 0; r < a.nreplicas; r++) zero_unit(a.store[r] + off, n, lane);
	}
}

int oimgpu::track_scan_locked(const Bdev &b, bool compare, TrackScan *out)
{
	const Replica &r0 = b.replicas[0];
	const Device &dev = g.devices[find_device_slot(r0.device)];
	const uint64_t size = b.num_blocks * (uint64_t)b.block_size, ngran = granules_of(b);
	const uint64_t words = (ngran + 31) / 32;
	/* one scratch: the digest, then the changed bitmap, then the non-zero bitmap */
	const size_t bytes = 16 + 2 * words * sizeof(uint32_t);
	out->bits = host_pages(bytes);
	if (!out->bits) return -ENOMEM;
	DeltaScan a{r0.store, size, compare ? b.track[b.track_base].get() : nullptr, b.track[b.track_base ^ 1].get(),
		    nullptr, nullptr, nullptr, {b.track_key[0], b.track_key[1]}};
	uint8_t *d = nullptr;
	CU_OK(cudaSetDevice(r0.device));
	CU_OK(cudaMallocAsync((void **)&d, bytes, dev.util));
	a.digest = (unsigned long long *)d;
	a.changed = (uint32_t *)(d + 16);
	a.nonzero = a.changed + words;
	/* one wave of as many CTAs as fit on the GPU: a grid of several waves would end in a partial one */
	static int per_sm = 0;
	cudaError_t e = per_sm ? cudaSuccess
			       : cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, oim_image_delta_scan_kernel, kImageThreads, 0);
	if (e == cudaSuccess) e = cudaMemsetAsync(d, 0, bytes, dev.util);
	if (e == cudaSuccess) {
		const uint32_t grid = std::min<uint32_t>(grid_for(dev, ngran), (uint32_t)std::max(1, dev.sm_count * per_sm));
		oim_image_delta_scan_kernel<<<grid, kImageThreads, 0, dev.util>>>(a);
		e = cudaGetLastError();
	}
	if (e == cudaSuccess) e = cudaMemcpyAsync(out->bits.get(), d, bytes, cudaMemcpyDeviceToHost, dev.util);
	if (e == cudaSuccess) e = cudaStreamSynchronize(dev.util);
	cudaFreeAsync(d, dev.util);
	if (e != cudaSuccess) {
		fprintf(stderr, "oimgpu: delta scan of %s failed: %s\n", b.name.c_str(), cudaGetErrorString(e));
		(void)cudaGetLastError();
		return -EIO;
	}
	memcpy(out->digest, out->bits.get(), 16);
	out->changed = (const uint32_t *)(out->bits.get() + 16);
	out->nonzero = out->changed + words;
	return 0;
}

void oimgpu::track_commit_locked(Bdev &b, const uint64_t digest[2])
{
	b.track_base ^= 1;
	b.has_base = true;
	b.base_digest[0] = digest[0];
	b.base_digest[1] = digest[1];
}

int oimgpu::finish_load_locked(Bdev &b, int rc, const uint64_t want[2])
{
	uint64_t d[2] = {0, 0};
	TrackScan ts;
	if (!rc && tracked(b)) {
		rc = track_scan_locked(b, false, &ts);
		memcpy(d, ts.digest, sizeof(d));
	} else if (!rc) {
		rc = store_digest(b, 0, d);
	}
	if (!rc && (d[0] != want[0] || d[1] != want[1])) {
		fprintf(stderr, "oimgpu: content written into %s does not match its digest\n", b.name.c_str());
		rc = -EIO;
	}
	if (rc) b.has_base = false;
	else if (tracked(b)) track_commit_locked(b, d);
	return rc;
}

namespace {

void fill_info(const DeltaHeader &h, oimgpu_image_delta_info *out)
{
	memset(out, 0, sizeof(*out));
	out->num_blocks = h.num_blocks;
	out->block_size = h.block_size;
	out->granule_bytes = h.granule_bytes;
	out->nextents = h.nextents;
	out->data_bytes = h.data_bytes;
	out->zero_bytes = h.zero_bytes;
	out->file_bytes = kHeaderBytes + table_bytes(h.nextents) + h.data_bytes;
	memcpy(out->parent_digest, h.parent_digest, sizeof(h.parent_digest));
	memcpy(out->digest, h.digest, sizeof(h.digest));
	memcpy(out->uuid, h.uuid, sizeof(h.uuid));
}

/* The runs of changed granules, split by kind, from a scan's two bitmaps: table entries in store order, the data runs
 * as segments of the data section, and the byte counts of both kinds. */
void cut_runs(const TrackScan &s, uint64_t size, std::vector<uint64_t> &table, std::vector<ImageSeg> &data_segs,
	      uint64_t *data_bytes, uint64_t *zero_bytes)
{
	const uint64_t ngran = (size + kGranule - 1) / kGranule;
	uint64_t start = 0, data = 0, zero = 0;
	bool in_run = false, run_data = false;
	auto emit = [&](uint64_t end_gran) {
		const uint64_t off = start * kGranule, len = std::min(end_gran * kGranule, size) - off;
		table.push_back(off);
		table.push_back(run_data ? len : len | kZeroRun);
		if (run_data) {
			data_segs.push_back({off, data, len});
			data += len;
		} else {
			zero += len;
		}
		in_run = false;
	};
	for (uint64_t w = 0; w < (ngran + 31) / 32; w++) {
		const uint32_t c = s.changed[w], nz = s.nonzero[w];
		if (!c && !in_run) continue;
		for (int i = 0; i < 32; i++) {
			const uint64_t gi = w * 32 + i;
			if (!(c >> i & 1)) {
				if (in_run) emit(gi);
				continue;
			}
			const bool k = nz >> i & 1;
			if (in_run && k == run_data) continue;
			if (in_run) emit(gi);
			start = gi;
			run_data = k;
			in_run = true;
		}
	}
	if (in_run) emit(ngran);	/* bits past ngran are never set */
	*data_bytes = data;
	*zero_bytes = zero;
}

int save_delta_locked(const Bdev &b, int fd, oimgpu_image_delta_info *out, TrackScan *ts)
{
	if (int rc = track_scan_locked(b, true, ts)) return rc;
	std::vector<uint64_t> table;
	std::vector<ImageSeg> segs;
	DeltaHeader h;
	memset(&h, 0, sizeof(h));
	cut_runs(*ts, b.num_blocks * (uint64_t)b.block_size, table, segs, &h.data_bytes, &h.zero_bytes);
	memcpy(h.magic, kDeltaMagic, sizeof(h.magic));
	h.version = kDeltaVersion;
	h.block_size = b.block_size;
	h.num_blocks = b.num_blocks;
	h.granule_bytes = kGranule;
	h.nextents = table.size() / 2;
	memcpy(h.digest, ts->digest, sizeof(h.digest));
	memcpy(h.parent_digest, b.base_digest, sizeof(h.parent_digest));
	memcpy(h.uuid, b.uuid.data(), std::min(b.uuid.size(), sizeof(h.uuid)));
	const uint64_t meta = kHeaderBytes + table_bytes(h.nextents);
	std::vector<uint8_t> head(meta, 0);
	memcpy(head.data(), &h, sizeof(h));
	if (!table.empty()) memcpy(&head[kHeaderBytes], table.data(), 8 * table.size());
	if (int rc = write_all(fd, head.data(), meta, 0)) return rc;
	if (int rc = move_data(b, segs, h.data_bytes, fd, meta, false)) return rc;
	fill_info(h, out);
	return 0;
}

/* the header and table of a delta for bdev b, checked against b and the file's size before anything is touched:
 * -EINVAL for anything that is not a well-formed delta of b's geometry */
int read_delta_meta(const Bdev &b, int fd, DeltaHeader *h, std::vector<ImageSeg> &data_segs, std::vector<ImageSeg> &zero_segs)
{
	struct stat st;
	if (fstat(fd, &st)) return -errno;
	if (!S_ISREG(st.st_mode) || (uint64_t)st.st_size < kHeaderBytes) return -EINVAL;
	std::vector<uint8_t> head(kHeaderBytes);
	if (int rc = read_all(fd, head.data(), kHeaderBytes, 0)) return rc;
	memcpy(h, head.data(), sizeof(*h));
	/* canonical: everything past the fields is zero, the uuid's tail included */
	const char *uend = (const char *)memchr(h->uuid, 0, sizeof(h->uuid));
	if (uend && std::any_of(uend, (const char *)h->uuid + sizeof(h->uuid), [](char c) { return c != 0; })) return -EINVAL;
	if (std::any_of(head.begin() + sizeof(*h), head.end(), [](uint8_t c) { return c != 0; })) return -EINVAL;
	const uint64_t size = b.num_blocks * (uint64_t)b.block_size;
	if (memcmp(h->magic, kDeltaMagic, sizeof(h->magic)) || h->version != kDeltaVersion || h->granule_bytes != kGranule ||
	    h->reserved != 0 || h->reserved2 != 0)
		return -EINVAL;
	if (h->block_size != b.block_size || h->num_blocks != b.num_blocks) return -EINVAL;
	/* runs never overlap: at most one per granule */
	if (h->nextents > granules_of(b) || h->data_bytes > size || h->zero_bytes > size - h->data_bytes) return -EINVAL;
	const uint64_t meta = kHeaderBytes + table_bytes(h->nextents);
	if ((uint64_t)st.st_size != meta + h->data_bytes) return -EINVAL;
	std::vector<uint64_t> table(table_bytes(h->nextents) / 8);
	if (h->nextents) {
		if (int rc = read_all(fd, (uint8_t *)table.data(), 8 * table.size(), kHeaderBytes)) return rc;
	}
	if (std::any_of(table.begin() + 2 * h->nextents, table.end(), [](uint64_t x) { return x != 0; })) return -EINVAL;
	uint64_t data = 0, zero = 0, prev_end = 0;
	bool prev_zero = false;
	for (uint64_t i = 0; i < h->nextents; i++) {
		const uint64_t off = table[2 * i], len = table[2 * i + 1] & ~kZeroRun;
		const bool is_zero = table[2 * i + 1] & kZeroRun;
		if (off % kGranule || off >= size || len == 0 || len > size - off) return -EINVAL;
		if ((off + len) % kGranule && off + len != size) return -EINVAL;
		/* sorted, not overlapping, and touching only a run of the other kind */
		if (i && (off < prev_end || (off == prev_end && is_zero == prev_zero))) return -EINVAL;
		if (is_zero) {
			zero_segs.push_back({off, zero, len});
			zero += len;
		} else {
			data_segs.push_back({off, data, len});
			data += len;
		}
		prev_end = off + len;
		prev_zero = is_zero;
	}
	return data == h->data_bytes && zero == h->zero_bytes ? 0 : -EINVAL;
}

/* the zero runs cleared in every replica: one launch over the whole table */
int zero_runs(const Bdev &b, const std::vector<ImageSeg> &segs, uint64_t total)
{
	if (!total) return 0;
	const int dev0 = b.replicas[0].device;
	const Device &dev = g.devices[find_device_slot(dev0)];
	const size_t bytes = segs.size() * sizeof(ImageSeg);
	HostPages h_segs = host_pages(bytes);
	if (!h_segs) return -ENOMEM;
	memcpy(h_segs.get(), segs.data(), bytes);
	DeltaZero z;
	memset(&z, 0, sizeof(z));
	for (size_t r = 0; r < b.replicas.size(); r++) z.store[r] = b.replicas[r].store;
	z.nreplicas = (uint32_t)b.replicas.size();
	z.nsegs = segs.size();
	z.total = total;
	ImageSeg *d_segs = nullptr;
	CU_OK(cudaSetDevice(dev0));
	CU_OK(cudaMallocAsync((void **)&d_segs, bytes, dev.util));
	z.segs = d_segs;
	cudaError_t e = cudaMemcpyAsync(d_segs, h_segs.get(), bytes, cudaMemcpyHostToDevice, dev.util);
	if (e == cudaSuccess) {
		oim_image_delta_zero_kernel<<<grid_for(dev, (total + kUnitBytes - 1) / kUnitBytes), kImageThreads, 0, dev.util>>>(z);
		e = cudaGetLastError();
	}
	if (e == cudaSuccess) e = cudaStreamSynchronize(dev.util);
	cudaFreeAsync(d_segs, dev.util);
	if (e != cudaSuccess) {
		fprintf(stderr, "oimgpu: zero runs of %s failed: %s\n", b.name.c_str(), cudaGetErrorString(e));
		(void)cudaGetLastError();
		return -EIO;
	}
	return 0;
}

int apply_delta_locked(Bdev &b, int fd, oimgpu_image_delta_info *out)
{
	DeltaHeader h;
	std::vector<ImageSeg> data_segs, zero_segs;
	if (int rc = read_delta_meta(b, fd, &h, data_segs, zero_segs)) return rc;
	/* a resident poller on replica 0's GPU could keep the kernels' CTAs from being scheduled (as for an image load) */
	ParkedPollers held(b.replicas[0].device);
	for (size_t r = 0; r < b.replicas.size(); r++) {
		uint64_t d[2];
		if (int rc = store_digest(b, r, d)) return rc;
		if (d[0] != h.parent_digest[0] || d[1] != h.parent_digest[1]) return -ESTALE;
	}
	int rc = zero_runs(b, zero_segs, h.zero_bytes);
	if (!rc) rc = move_data(b, data_segs, h.data_bytes, fd, kHeaderBytes + table_bytes(h.nextents), true);
	if ((rc = finish_load_locked(b, rc, h.digest))) return rc;
	fill_info(h, out);
	return 0;
}

}  // namespace

extern "C" int oimgpu_bdev_image_track(const char *name, int enable)
{
	if (!name) return -EINVAL;
	std::lock_guard<std::mutex> lk(g.mu);
	if (!g.inited || g.control_only) return -ENODEV;
	Bdev *b = find_bdev_locked(name);
	if (!b) return -ENODEV;
	const int dev0 = b->replicas[0].device;
	if (enable) {
		if (!tracked(*b)) {
			std::random_device rd;
			for (uint64_t &k : b->track_key) k = (uint64_t)rd() << 32 | rd();
		}
		for (auto &t : b->track) {
			if (t) continue;
			if (t.alloc(dev0, granules_of(*b)) == cudaSuccess) continue;
			ParkedPollers parked(dev0);
			for (auto &u : b->track) u.reset(parked);
			return -ENOMEM;
		}
		return 0;
	}
	if (tracked(*b)) {
		ParkedPollers parked(dev0);
		for (auto &t : b->track) t.reset(parked);
	}
	b->has_base = false;
	return 0;
}

extern "C" int oimgpu_bdev_image_save_delta(const char *name, const char *path, oimgpu_image_delta_info *out)
{
	if (!name || !path || !out) return -EINVAL;
	std::lock_guard<std::mutex> lk(g.mu);
	if (!g.inited || g.control_only) return -ENODEV;
	Bdev *b = find_bdev_locked(name);
	if (!b) return -ENODEV;
	if (!tracked(*b) || !b->has_base) return -ENODATA;
	/* as oimgpu_bdev_image_save: neither an NBD export nor a block-I/O channel can be paused */
	if (b->nbd_exports || b->bio_chans) return -EBUSY;
	const int fd = open(path, O_WRONLY | O_CREAT | O_EXCL | O_CLOEXEC, 0644);
	if (fd < 0) return -errno;
	int rc;
	TrackScan ts;
	{
		ParkedPollers held(b->replicas[0].device, b->name);
		rc = held.drain();
		if (!rc) rc = save_delta_locked(*b, fd, out, &ts);
	}
	if (!rc && fsync(fd)) rc = -errno;
	if (close(fd) && !rc) rc = -errno;
	if (rc) unlink(path);
	else track_commit_locked(*b, ts.digest);
	return rc;
}

extern "C" int oimgpu_bdev_image_apply_delta(const char *name, const char *path, oimgpu_image_delta_info *out)
{
	if (!name || !path || !out) return -EINVAL;
	std::lock_guard<std::mutex> lk(g.mu);
	if (!g.inited || g.control_only) return -ENODEV;
	Bdev *b = find_bdev_locked(name);
	if (!b) return -ENODEV;
	if (b->opens > 0) return -EBUSY;
	const int fd = open(path, O_RDONLY | O_CLOEXEC);
	if (fd < 0) return -errno;
	const int rc = apply_delta_locked(*b, fd, out);
	close(fd);
	return rc;
}
