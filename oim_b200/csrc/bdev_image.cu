/*
 * bdev_image.cu - volume images (oimgpu_bdev_image_save / oimgpu_bdev_image_load): a bdev's bytes written to a sparse,
 * canonical image file and read back into every replica (include/oimgpu.h gives the format).
 *
 * The GPU finds the 4 KiB granules that hold a non-zero byte at HBM rate and gathers them into contiguous staging
 * chunks (save), or scatters chunks back into every replica (load); only the granules that are really there cross PCIe.
 * The copy engine moves each chunk between a device staging buffer and pinned host memory, and two chunks are in
 * flight so that it overlaps the pwrite / pread of the other.  The kernels live here and not in lun_kernel.cu so that
 * nothing they need can shift the register allocation of the queue kernels; they reuse its vector loads and unit mover
 * (ld_cg16, move_unit in lun_kernel.cuh).
 */
#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>

#include "bdev_image.h"

namespace {

constexpr uint64_t kChunkBytes = 64ull << 20;		/* payload per staging chunk (two in flight) */
constexpr uint32_t kImageVersion = 1;
constexpr char kImageMagic[8] = {'O', 'I', 'M', 'G', 'P', 'U', 'I', 'M'};

/* the first 100 bytes of the 4096-byte header, little-endian; the rest (the struct's tail padding included) is zero */
struct ImageHeader {
	char magic[8];
	uint32_t version, block_size;
	uint64_t num_blocks;
	uint32_t granule_bytes, reserved;
	uint64_t nextents, data_bytes;
	uint64_t digest[2];
	char uuid[36];
};
static_assert(offsetof(ImageHeader, num_blocks) == 16 && offsetof(ImageHeader, nextents) == 32 &&
	      offsetof(ImageHeader, digest) == 48 && offsetof(ImageHeader, uuid) == 64,
	      "image header layout");

struct ImageScan {
	const uint8_t *store;
	uint64_t nbytes;
	uint32_t *bitmap;	/* bit g: granule g holds a non-zero byte */
};

/* data bytes [begin, end) of the image, held at `stage`, and the stores they belong to */
struct ImageMove {
	uint8_t *store[kMaxReplicas];	/* replica 0 local; the others peer or imported mappings, as the write fan-out's */
	uint32_t nreplicas;
	uint32_t to_store;		/* 1: stage -> every replica (load); 0: replica 0 -> stage (save) */
	uint8_t *stage;
	const ImageSeg *segs;
	uint64_t nsegs, begin, end;
};

}  // namespace

/* Warps take granules grid-stride.  The store is read up to its end widened to a 16-byte boundary: the store is an
 * allocation of its own (256-byte aligned), so an aligned vector that holds one byte of it never leaves the
 * allocation (mirror_check.cu makes the same argument); the bytes past the end are masked before they count. */
__global__ void __launch_bounds__(kImageThreads)
oim_image_scan_kernel(const __grid_constant__ ImageScan a)
{
	const int lane = threadIdx.x & 31;
	const uint64_t hi = (a.nbytes + 15) & ~15ull;
	const uint64_t ngran = (a.nbytes + kGranule - 1) / kGranule;
	const uint64_t nwarps = (uint64_t)gridDim.x * (kImageThreads / 32);
	for (uint64_t gi = (uint64_t)blockIdx.x * (kImageThreads / 32) + (threadIdx.x >> 5); gi < ngran; gi += nwarps) {
		const uint64_t base = gi * kGranule;
		const uint32_t nv = (uint32_t)(min((uint64_t)kGranule, hi - base) >> 4);
		int4 x[kGranule / 512];
#pragma unroll
		for (int k = 0; k < (int)(kGranule / 512); k++) {
			const uint32_t v = lane + 32 * k;
			x[k] = v < nv ? ld_cg16(a.store + base + (size_t)v * 16) : make_int4(0, 0, 0, 0);
		}
		int acc = 0;
#pragma unroll
		for (int k = 0; k < (int)(kGranule / 512); k++) {
			const uint64_t pos = base + (uint64_t)(lane + 32 * k) * 16;
			if (pos < a.nbytes && pos + 16 > a.nbytes) keep_low_bytes(x[k], (uint32_t)(a.nbytes - pos));
			acc |= x[k].x | x[k].y | x[k].z | x[k].w;
		}
		if (__any_sync(0xffffffffu, acc != 0) && lane == 0) atomicOr(&a.bitmap[gi >> 5], 1u << (gi & 31));
	}
}

/* Warps take the chunk's 4 KiB units grid-stride and find the extent of each by binary search, as oim_bio_kernel
 * finds a segment.  Extents start on granule boundaries in the store and in the data section alike, and only the
 * last one can end elsewhere (at the end of the store), so a unit never spans two extents. */
__global__ void __launch_bounds__(kImageThreads)
oim_image_move_kernel(const __grid_constant__ ImageMove a)
{
	const int lane = threadIdx.x & 31;
	const uint64_t nunits = (a.end - a.begin + kUnitBytes - 1) / kUnitBytes;
	const uint64_t nwarps = (uint64_t)gridDim.x * (kImageThreads / 32);
	for (uint64_t u = (uint64_t)blockIdx.x * (kImageThreads / 32) + (threadIdx.x >> 5); u < nunits; u += nwarps) {
		const uint64_t pos = a.begin + u * kUnitBytes;
		uint64_t lo = 0, hi = a.nsegs;	/* the last extent whose data starts at or before pos */
		while (hi - lo > 1) {
			const uint64_t mid = (lo + hi) >> 1;
			if (a.segs[mid].data_off <= pos) lo = mid;
			else hi = mid;
		}
		const ImageSeg s = a.segs[lo];
		const uint32_t n = (uint32_t)min((uint64_t)kUnitBytes, min(s.data_off + s.len, a.end) - pos);
		const uint64_t off = s.store_off + (pos - s.data_off);
		uint8_t *stage = a.stage + (pos - a.begin);
		if (a.to_store) {
#pragma unroll 1
			for (uint32_t r = 0; r < a.nreplicas; r++) move_unit<true>(a.store[r] + off, stage, n, lane);
		} else {
			move_unit<true>(stage, a.store[0] + off, n, lane);
		}
	}
}

HostPages oimgpu::host_pages(size_t n)
{
	return HostPages((uint8_t *)aligned_alloc(4096, std::max<size_t>(4096, (n + 4095) & ~(size_t)4095)), &free);
}

uint32_t oimgpu::grid_for(const Device &dev, uint64_t warps_of_work)
{
	const uint64_t per_cta = kImageThreads / 32;
	return (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>((warps_of_work + per_cta - 1) / per_cta, (uint64_t)dev.sm_count * 8));
}

int oimgpu::write_all(int fd, const uint8_t *p, uint64_t n, uint64_t off)
{
	while (n) {
		const ssize_t w = pwrite(fd, p, std::min<uint64_t>(n, 1ull << 30), (off_t)off);
		if (w < 0 && errno == EINTR) continue;
		if (w < 0) return -errno;
		if (w == 0) return -EIO;
		p += w; n -= (uint64_t)w; off += (uint64_t)w;
	}
	return 0;
}

int oimgpu::read_all(int fd, uint8_t *p, uint64_t n, uint64_t off)
{
	while (n) {
		const ssize_t r = pread(fd, p, std::min<uint64_t>(n, 1ull << 30), (off_t)off);
		if (r < 0 && errno == EINTR) continue;
		if (r < 0) return -errno;
		if (r == 0) return -EIO;	/* short read: the file shrank under us */
		p += r; n -= (uint64_t)r; off += (uint64_t)r;
	}
	return 0;
}

/* the words the GPU can read whole, then the last bytes zero-padded to a word */
int oimgpu::store_digest(const Bdev &b, size_t r, uint64_t out[2])
{
	const Replica &rep = b.replicas[r];
	const uint64_t size = b.num_blocks * (uint64_t)b.block_size, whole = size & ~7ull;
	if (int rc = digest_locked(rep.device, rep.store, whole, out)) return rc;
	if (size == whole) return 0;
	HostPages tail = host_pages(8);
	if (!tail) return -ENOMEM;
	memset(tail.get(), 0, 8);
	cudaStream_t st = g.devices[find_device_slot(rep.device)].util;
	CU_OK(cudaMemcpyAsync(tail.get(), rep.store + whole, size - whole, cudaMemcpyDeviceToHost, st));
	CU_OK(cudaStreamSynchronize(st));
	uint64_t w, i = whole / 8;
	memcpy(&w, tail.get(), 8);
	out[0] += w * (2 * i + 1);
	uint64_t z = w ^ i;
	z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
	z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
	out[1] += z ^ (z >> 31);
	return 0;
}

namespace {

void fill_info(const ImageHeader &h, oimgpu_image_info *out)
{
	memset(out, 0, sizeof(*out));
	out->num_blocks = h.num_blocks;
	out->block_size = h.block_size;
	out->granule_bytes = h.granule_bytes;
	out->nextents = h.nextents;
	out->data_bytes = h.data_bytes;
	out->file_bytes = kHeaderBytes + table_bytes(h.nextents) + h.data_bytes;
	memcpy(out->uuid, h.uuid, sizeof(h.uuid));
}

}  // namespace

int oimgpu::move_data(const Bdev &b, const std::vector<ImageSeg> &segs, uint64_t data_bytes, int fd, uint64_t data_pos, bool load)
{
	if (!data_bytes) return 0;
	const int dev0 = b.replicas[0].device;
	const Device &dev = g.devices[find_device_slot(dev0)];
	const uint64_t chunk = std::min(kChunkBytes, data_bytes);
	const uint64_t nchunks = (data_bytes + chunk - 1) / chunk;
	HostPages h_segs = host_pages(segs.size() * sizeof(ImageSeg));
	if (!h_segs) return -ENOMEM;
	memcpy(h_segs.get(), segs.data(), segs.size() * sizeof(ImageSeg));
	Buf<uint8_t, Mem::Pinned> h_stage[2];
	uint8_t *d_stage[2] = {nullptr, nullptr};
	ImageSeg *d_segs = nullptr;
	cudaEvent_t ev[2] = {nullptr, nullptr};
	int rc = 0;
	auto cu = [&](cudaError_t e) {
		if (e != cudaSuccess && !rc) {
			fprintf(stderr, "oimgpu: image %s of %s failed: %s\n", load ? "load" : "save", b.name.c_str(), cudaGetErrorString(e));
			(void)cudaGetLastError();
			rc = e == cudaErrorMemoryAllocation ? -ENOMEM : -EIO;
		}
		return rc == 0;
	};
	for (int k = 0; k < 2 && !rc; k++) {
		cu(h_stage[k].alloc(dev0, chunk));
		if (!rc) cu(cudaSetDevice(dev0));
		if (!rc) cu(cudaMallocAsync((void **)&d_stage[k], chunk, dev.util));
		if (!rc) cu(cudaEventCreateWithFlags(&ev[k], cudaEventDisableTiming));
	}
	if (!rc) cu(cudaMallocAsync((void **)&d_segs, segs.size() * sizeof(ImageSeg), dev.util));
	if (!rc) cu(cudaMemcpyAsync(d_segs, h_segs.get(), segs.size() * sizeof(ImageSeg), cudaMemcpyHostToDevice, dev.util));
	ImageMove m;
	memset(&m, 0, sizeof(m));
	for (size_t r = 0; r < b.replicas.size(); r++) m.store[r] = b.replicas[r].store;
	m.nreplicas = (uint32_t)b.replicas.size();
	m.to_store = load;
	m.segs = d_segs;
	m.nsegs = segs.size();
	/* chunk i: its move kernel and its copy, then event ev[i & 1] */
	auto enqueue = [&](uint64_t i) {
		const int k = (int)(i & 1);
		m.stage = d_stage[k];
		m.begin = i * chunk;
		m.end = std::min(data_bytes, m.begin + chunk);
		const uint64_t len = m.end - m.begin;
		if (load && !cu(cudaMemcpyAsync(d_stage[k], h_stage[k].get(), len, cudaMemcpyHostToDevice, dev.util))) return false;
		oim_image_move_kernel<<<grid_for(dev, (len + kUnitBytes - 1) / kUnitBytes), kImageThreads, 0, dev.util>>>(m);
		if (!cu(cudaGetLastError())) return false;
		if (!load && !cu(cudaMemcpyAsync(h_stage[k].get(), d_stage[k], len, cudaMemcpyDeviceToHost, dev.util))) return false;
		return cu(cudaEventRecord(ev[k], dev.util));
	};
	if (!load && !rc) enqueue(0);
	for (uint64_t i = 0; i < nchunks && !rc; i++) {
		const int k = (int)(i & 1);
		const uint64_t begin = i * chunk, len = std::min(chunk, data_bytes - begin);
		if (load) {
			/* h_stage[k] is free once chunk i - 2's copy has run */
			if (i >= 2 && !cu(cudaEventSynchronize(ev[k]))) break;
			if ((rc = read_all(fd, h_stage[k].get(), len, data_pos + begin))) break;
			enqueue(i);
		} else {
			/* chunk i + 1 reuses the buffers of chunk i - 1, whose bytes are in the file */
			if (i + 1 < nchunks && !enqueue(i + 1)) break;
			if (!cu(cudaEventSynchronize(ev[k]))) break;
			rc = write_all(fd, h_stage[k].get(), len, data_pos + begin);
		}
	}
	cudaError_t e = cudaStreamSynchronize(dev.util);
	if (e != cudaSuccess) cu(e);
	for (int k = 0; k < 2; k++) {
		if (d_stage[k]) cudaFreeAsync(d_stage[k], dev.util);
		if (ev[k]) cudaEventDestroy(ev[k]);
	}
	if (d_segs) cudaFreeAsync(d_segs, dev.util);
	{
		/* pinned memory is mapped into every GPU: its free waits for all of them */
		ParkedPollers all(kAllGpus);
		for (auto &h : h_stage) h.reset(all);
	}
	return rc;
}

namespace {

/* the runs of set bits of a granule bitmap, as extents in store order (collect_ranges' walk over a bitmap) */
void extents_of(const uint32_t *bits, uint64_t size, std::vector<ImageSeg> &segs, uint64_t *data_bytes)
{
	const uint64_t ngran = (size + kGranule - 1) / kGranule;
	uint64_t start = 0, data = 0;
	bool in_run = false;
	auto emit = [&](uint64_t end_gran) {
		const uint64_t off = start * kGranule, len = std::min(end_gran * kGranule, size) - off;
		segs.push_back({off, data, len});
		data += len;
	};
	for (uint64_t w = 0; w < (ngran + 31) / 32; w++) {
		const uint32_t x = bits[w];
		if (x == (in_run ? 0xffffffffu : 0u)) continue;
		for (int i = 0; i < 32; i++) {
			const bool set = x >> i & 1;
			if (set == in_run) continue;
			if (set) start = w * 32 + i;
			else emit(w * 32 + i);
			in_run = set;
		}
	}
	if (in_run) emit(ngran);	/* bits past ngran are never set */
	*data_bytes = data;
}

/* the granules of replica 0 that hold a non-zero byte, as extents in store order */
int scan_extents(const Bdev &b, std::vector<ImageSeg> &segs, uint64_t *data_bytes)
{
	const Replica &r0 = b.replicas[0];
	const Device &dev = g.devices[find_device_slot(r0.device)];
	const uint64_t size = b.num_blocks * (uint64_t)b.block_size;
	const uint64_t ngran = (size + kGranule - 1) / kGranule;
	const size_t bitmap_bytes = (ngran + 31) / 32 * sizeof(uint32_t);
	HostPages h_bits = host_pages(bitmap_bytes);
	if (!h_bits) return -ENOMEM;
	ImageScan a{r0.store, size, nullptr};
	CU_OK(cudaSetDevice(r0.device));
	CU_OK(cudaMallocAsync((void **)&a.bitmap, bitmap_bytes, dev.util));
	cudaError_t e = cudaMemsetAsync(a.bitmap, 0, bitmap_bytes, dev.util);
	if (e == cudaSuccess) {
		oim_image_scan_kernel<<<grid_for(dev, ngran), kImageThreads, 0, dev.util>>>(a);
		e = cudaGetLastError();
	}
	if (e == cudaSuccess) e = cudaMemcpyAsync(h_bits.get(), a.bitmap, bitmap_bytes, cudaMemcpyDeviceToHost, dev.util);
	if (e == cudaSuccess) e = cudaStreamSynchronize(dev.util);
	cudaFreeAsync(a.bitmap, dev.util);
	if (e != cudaSuccess) {
		fprintf(stderr, "oimgpu: image scan of %s failed: %s\n", b.name.c_str(), cudaGetErrorString(e));
		(void)cudaGetLastError();
		return -EIO;
	}
	extents_of((const uint32_t *)h_bits.get(), size, segs, data_bytes);
	return 0;
}

/* ts: a tracked bdev's scan, whose table becomes the baseline once the file is on disk */
int save_locked(const Bdev &b, int fd, oimgpu_image_info *out, TrackScan *ts)
{
	std::vector<ImageSeg> segs;
	ImageHeader h;
	memset(&h, 0, sizeof(h));
	if (tracked(b)) {
		/* the tracking scan finds the non-zero granules and the digest in the one pass it makes anyway */
		if (int rc = track_scan_locked(b, false, ts)) return rc;
		extents_of(ts->nonzero, b.num_blocks * (uint64_t)b.block_size, segs, &h.data_bytes);
		memcpy(h.digest, ts->digest, sizeof(h.digest));
	} else {
		if (int rc = scan_extents(b, segs, &h.data_bytes)) return rc;
		if (int rc = store_digest(b, 0, h.digest)) return rc;
	}
	memcpy(h.magic, kImageMagic, sizeof(h.magic));
	h.version = kImageVersion;
	h.block_size = b.block_size;
	h.num_blocks = b.num_blocks;
	h.granule_bytes = kGranule;
	h.nextents = segs.size();
	memcpy(h.uuid, b.uuid.data(), std::min(b.uuid.size(), sizeof(h.uuid)));
	const uint64_t meta = kHeaderBytes + table_bytes(h.nextents);
	std::vector<uint8_t> head(meta, 0);
	memcpy(head.data(), &h, sizeof(h));
	for (size_t i = 0; i < segs.size(); i++) {
		memcpy(&head[kHeaderBytes + 16 * i], &segs[i].store_off, 8);
		memcpy(&head[kHeaderBytes + 16 * i + 8], &segs[i].len, 8);
	}
	if (int rc = write_all(fd, head.data(), meta, 0)) return rc;
	if (int rc = move_data(b, segs, h.data_bytes, fd, meta, false)) return rc;
	fill_info(h, out);
	return 0;
}

/* the header and extent table of an image for bdev b, checked against b and the file's size before anything is
 * touched: -EINVAL for anything that is not a well-formed image of b's geometry */
int read_image_meta(const Bdev &b, int fd, ImageHeader *h, std::vector<ImageSeg> &segs)
{
	struct stat st;
	if (fstat(fd, &st)) return -errno;
	if (!S_ISREG(st.st_mode) || (uint64_t)st.st_size < kHeaderBytes) return -EINVAL;
	if (int rc = read_all(fd, (uint8_t *)h, sizeof(*h), 0)) return rc;
	const uint64_t size = b.num_blocks * (uint64_t)b.block_size;
	const uint64_t ngran = (size + kGranule - 1) / kGranule;
	if (memcmp(h->magic, kImageMagic, sizeof(h->magic)) || h->version != kImageVersion || h->granule_bytes != kGranule ||
	    h->reserved != 0)
		return -EINVAL;
	if (h->block_size != b.block_size || h->num_blocks != b.num_blocks) return -EINVAL;
	/* runs are neither overlapping nor adjacent: at most one per two granules, rounded up */
	if (h->nextents > (ngran + 1) / 2 || h->data_bytes > size) return -EINVAL;
	const uint64_t meta = kHeaderBytes + table_bytes(h->nextents);
	if ((uint64_t)st.st_size != meta + h->data_bytes) return -EINVAL;
	std::vector<uint64_t> table(2 * h->nextents);
	if (h->nextents) {
		if (int rc = read_all(fd, (uint8_t *)table.data(), 16 * h->nextents, kHeaderBytes)) return rc;
	}
	uint64_t data = 0, prev_end = 0;
	for (uint64_t i = 0; i < h->nextents; i++) {
		const uint64_t off = table[2 * i], len = table[2 * i + 1];
		if (off % kGranule || off >= size || len == 0 || len > size - off) return -EINVAL;
		if ((off + len) % kGranule && off + len != size) return -EINVAL;
		if (i && off <= prev_end) return -EINVAL;	/* sorted, not overlapping, not adjacent */
		segs.push_back({off, data, len});
		data += len;
		prev_end = off + len;
	}
	return data == h->data_bytes ? 0 : -EINVAL;
}

int load_locked(Bdev &b, int fd, oimgpu_image_info *out)
{
	ImageHeader h;
	std::vector<ImageSeg> segs;
	if (int rc = read_image_meta(b, fd, &h, segs)) return rc;
	const int dev0 = b.replicas[0].device;
	/* a resident poller on replica 0's GPU could keep the kernels' CTAs from being scheduled (as for a mirror check) */
	ParkedPollers held(dev0);
	const Device &dev = g.devices[find_device_slot(dev0)];
	const uint64_t size = b.num_blocks * (uint64_t)b.block_size;
	cudaError_t e = cudaSetDevice(dev0);
	for (const Replica &r : b.replicas) {
		if (e == cudaSuccess) e = launch_fill(dev.util, dev.sm_count, r.store, 0, size);
	}
	int rc = 0;
	if (e != cudaSuccess) {
		fprintf(stderr, "oimgpu: image load into %s failed: %s\n", b.name.c_str(), cudaGetErrorString(e));
		(void)cudaGetLastError();
		rc = -EIO;
	}
	if (!rc) rc = move_data(b, segs, h.data_bytes, fd, kHeaderBytes + table_bytes(h.nextents), true);
	if ((rc = finish_load_locked(b, rc, h.digest))) return rc;
	fill_info(h, out);
	return 0;
}

}  // namespace

extern "C" int oimgpu_bdev_image_save(const char *name, const char *path, oimgpu_image_info *out)
{
	if (!name || !path || !out) return -EINVAL;
	std::lock_guard<std::mutex> lk(g.mu);
	if (!g.inited || g.control_only) return -ENODEV;
	Bdev *b = find_bdev_locked(name);
	if (!b) return -ENODEV;
	/* an NBD export or a block-I/O channel moves payload with no point at which it could be paused */
	if (b->nbd_exports || b->bio_chans) return -EBUSY;
	const int fd = open(path, O_WRONLY | O_CREAT | O_EXCL | O_CLOEXEC, 0644);
	if (fd < 0) return -errno;
	int rc;
	TrackScan ts;
	{
		/* as oimgpu_bdev_mirror_check: every session that reaches the bdev, and every session on replica 0's GPU,
		 * held and drained for the whole call, so the image is the volume between two writes of this process */
		ParkedPollers held(b->replicas[0].device, b->name);
		rc = held.drain();
		if (!rc) rc = save_locked(*b, fd, out, &ts);
	}
	if (!rc && fsync(fd)) rc = -errno;
	if (close(fd) && !rc) rc = -errno;
	if (rc) unlink(path);
	else if (tracked(*b)) track_commit_locked(*b, ts.digest);
	return rc;
}

extern "C" int oimgpu_bdev_image_load(const char *name, const char *path, oimgpu_image_info *out)
{
	if (!name || !path || !out) return -EINVAL;
	std::lock_guard<std::mutex> lk(g.mu);
	if (!g.inited || g.control_only) return -ENODEV;
	Bdev *b = find_bdev_locked(name);
	if (!b) return -ENODEV;
	if (b->opens > 0) return -EBUSY;
	const int fd = open(path, O_RDONLY | O_CLOEXEC);
	if (fd < 0) return -errno;
	const int rc = load_locked(*b, fd, out);
	close(fd);
	return rc;
}
