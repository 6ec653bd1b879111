/*
 * bdev_image.h - what volume images (bdev_image.cu) and incremental images (image_delta.cu) share: the granule, the
 * staging pipeline that moves runs of a store through a file, the file and digest helpers, and the fingerprint
 * tables of tracked bdevs (oimgpu_bdev_image_track).  Internal, not installed.
 */
#pragma once

#include "host_state.h"

namespace oimgpu {

constexpr int kImageThreads = 256;
constexpr uint32_t kGranule = 4096;		/* the images' unit of sparseness and change, independent of the block size */
constexpr uint64_t kHeaderBytes = 4096;

/* the bytes of v at and after byte `keep` (1..15) cleared */
__device__ __forceinline__ void keep_low_bytes(int4 &v, uint32_t keep)
{
	int *w = &v.x;
#pragma unroll
	for (int j = 0; j < 4; j++) {
		const uint32_t lo = 4 * j;
		if (keep <= lo) w[j] = 0;
		else if (keep < lo + 4) w[j] &= (int)((1u << (8 * (keep - lo))) - 1);
	}
}

/* a run of the store and where its bytes sit in a file's data section */
struct ImageSeg { uint64_t store_off, data_off, len; };

/* page-aligned, page-rounded host memory: a pageable copy that shared a page with a range this process registered
 * would be refused by the driver (mirror_check.cu) */
using HostPages = std::unique_ptr<uint8_t, decltype(&free)>;
HostPages host_pages(size_t n);

inline uint64_t table_bytes(uint64_t nextents) { return (16 * nextents + 4095) & ~4095ull; }
inline uint64_t granules_of(const Bdev &b) { return (b.num_blocks * (uint64_t)b.block_size + kGranule - 1) / kGranule; }
uint32_t grid_for(const Device &dev, uint64_t warps_of_work);
int write_all(int fd, const uint8_t *p, uint64_t n, uint64_t off);
int read_all(int fd, uint8_t *p, uint64_t n, uint64_t off);
/* oimgpu_bdev_digest of replica r's whole store, its last word zero-padded */
int store_digest(const Bdev &b, size_t r, uint64_t out[2]);
/* The data section of a file through two staging chunks in flight: save gathers replica 0's runs `segs` into a chunk and
 * writes it at file offset data_pos; load reads a chunk and scatters it into every replica.  Caller holds g.mu and
 * the sessions. */
int move_data(const Bdev &b, const std::vector<ImageSeg> &segs, uint64_t data_bytes, int fd, uint64_t data_pos, bool load);

/* A scan of replica 0 of a tracked bdev (image_delta.cu): every granule's fingerprint written into the spare table, and
 * two bitmaps copied back - granules whose fingerprint differs from the baseline's (with compare) and granules that
 * hold a non-zero byte - with the whole-store digest.  Caller holds g.mu and the sessions. */
struct TrackScan {
	HostPages bits{nullptr, &free};
	const uint32_t *changed = nullptr, *nonzero = nullptr;
	uint64_t digest[2] = {0, 0};
};
inline bool tracked(const Bdev &b) { return (bool)b.track[0]; }
int track_scan_locked(const Bdev &b, bool compare, TrackScan *out);
void track_commit_locked(Bdev &b, const uint64_t digest[2]);	/* the spare table becomes the baseline */
/* After a load or a delta was written into every replica (rc: how that went): the digest of replica 0 checked against
 * `want`.  On a tracked bdev the check is a scan, whose table becomes the baseline on success; on failure the baseline
 * is dropped, since the store no longer holds it.  -EIO on a mismatch. */
int finish_load_locked(Bdev &b, int rc, const uint64_t want[2]);

}  // namespace oimgpu
