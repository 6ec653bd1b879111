/*
 * bdev_oimgpu.h — the oimgpu bdev module for SPDK applications: a bdev whose store is an oimgpu bdev in HBM,
 * served in batches by oim_bio_kernel (include/oimgpu.h, oimgpu_bio_chan).
 */
#ifndef BDEV_OIMGPU_H
#define BDEV_OIMGPU_H

#include "spdk/stdinc.h"

#include "spdk/bdev.h"
#include "spdk/uuid.h"

typedef void (*spdk_delete_oimgpu_complete)(void *cb_arg, int bdeverrno);

/* name NULL: "OimGpu%d"; uuid NULL: random.  NULL on failure (num_blocks 0, a name in use, no GPU, no memory). */
struct spdk_bdev *create_oimgpu_disk(const char *name, const struct spdk_uuid *uuid, uint64_t num_blocks,
				     uint32_t block_size);
/* cb_fn(cb_arg, -ENODEV) if bdev is not one of this module's */
void delete_oimgpu_disk(struct spdk_bdev *bdev, spdk_delete_oimgpu_complete cb_fn, void *cb_arg);

#endif /* BDEV_OIMGPU_H */
