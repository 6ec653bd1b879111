/*
 * bdev_oimgpu.c — an SPDK bdev module whose store is an oimgpu bdev in HBM (SURVEY.md 8(b) row B2, the level
 * above the copy engine: struct spdk_bdev_fn_table + spdk_bdev_register, S/include/spdk/bdev_module.h:53,173,1017).
 *
 * What an SPDK application gets by linking this file (and liboimgpu): a bdev that every front end SPDK has -
 * vhost-scsi, vhost-blk, NBD, iSCSI, NVMe-oF, bdevperf - serves unchanged, with its blocks in GPU memory.
 *   - submit_request appends READ / WRITE / WRITE_ZEROES / UNMAP to the calling thread's channel; a poller on that
 *     thread hands everything collected since its last run to the GPU in one oimgpu_bio_chan_submit (one
 *     oim_bio_kernel launch for the batch), reaps completions and calls spdk_bdev_io_complete.  Payload crosses
 *     PCIe once, between the I/O's buffers and HBM.
 *   - A READ without a buffer gets one from the bdev layer (spdk_bdev_io_get_buf): the Malloc bdev's zero-copy read
 *     hands out a pointer into its store, which here is HBM.
 *   - FLUSH completes at once (the store is memory); RESET completes once everything the channel took before it
 *     has completed.
 *   - Requests of one channel take effect in submission order wherever they overlap and one writes, as on the
 *     synchronous Malloc bdev; channels of different threads are unordered, as in SPDK.
 * Written against SPDK's public headers as vendored by intel/oim; nothing here is copied from the Malloc bdev.
 */
#include "spdk/stdinc.h"

#include "spdk/bdev.h"
#include "spdk/bdev_module.h"
#include "spdk/json.h"
#include "spdk/log.h"
#include "spdk/string.h"
#include "spdk/thread.h"
#include "spdk/uuid.h"

#include "bdev_oimgpu.h"
#include "oimgpu.h"

#define OIMGPU_REAP_BATCH 64

struct oimgpu_disk {
	struct spdk_bdev		disk;
	TAILQ_ENTRY(oimgpu_disk)	link;
};

/* bdev_io->driver_ctx: only a RESET waits in the channel */
struct oimgpu_task {
	uint64_t			wait_for;	/* RESET: completions the channel must have delivered */
	TAILQ_ENTRY(oimgpu_task)	link;
};

struct oimgpu_channel {
	oimgpu_bio_chan			*chan;
	struct spdk_poller		*poller;
	/* the batch being collected */
	struct oimgpu_bio		*bios;
	struct oimgpu_iov		*iovs;
	uint32_t			nbios, bio_cap, niovs, iov_cap;
	uint64_t			taken, delivered;	/* bios handed to the channel / completed by it */
	unsigned long long		launches_seen;
	TAILQ_HEAD(, oimgpu_task)	resets;
};

static TAILQ_HEAD(, oimgpu_disk) g_oimgpu_disks = TAILQ_HEAD_INITIALIZER(g_oimgpu_disks);
static int g_oimgpu_disk_count;
static bool g_oimgpu_ready;
static unsigned long long g_oimgpu_launches;

static int bdev_oimgpu_initialize(void);

static int
bdev_oimgpu_get_ctx_size(void)
{
	return sizeof(struct oimgpu_task);
}

static struct spdk_bdev_module oimgpu_if = {
	.name = "oimgpu",
	.module_init = bdev_oimgpu_initialize,
	.get_ctx_size = bdev_oimgpu_get_ctx_size,
};

SPDK_BDEV_MODULE_REGISTER(oimgpu, &oimgpu_if)

/* oim_bio_kernel launches of every channel so far (diagnostics for the test driver) */
unsigned long long bdev_oimgpu_launches(void) { return __atomic_load_n(&g_oimgpu_launches, __ATOMIC_RELAXED); }

static void
oimgpu_io_done(struct oimgpu_channel *ch, struct spdk_bdev_io *bdev_io, int status)
{
	ch->delivered++;
	spdk_bdev_io_complete(bdev_io, status == 0 ? SPDK_BDEV_IO_STATUS_SUCCESS :
			      status == -ENOMEM ? SPDK_BDEV_IO_STATUS_NOMEM : SPDK_BDEV_IO_STATUS_FAILED);
}

static int
oimgpu_channel_poll(void *arg)
{
	struct oimgpu_channel *ch = arg;
	struct oimgpu_bio_cpl cpl[OIMGPU_REAP_BATCH];
	struct oimgpu_task *task;
	unsigned long long launches;
	int i, n, work = 0;
	uint32_t k;

	if (ch->nbios) {
		int rc = oimgpu_bio_chan_submit(ch->chan, ch->bios, ch->nbios, ch->iovs, ch->niovs);

		if (rc != 0) {
			for (k = 0; k < ch->nbios; k++) {
				oimgpu_io_done(ch, (struct spdk_bdev_io *)(uintptr_t)ch->bios[k].tag, rc);
			}
		}
		work += ch->nbios;
		ch->nbios = ch->niovs = 0;
		launches = oimgpu_bio_chan_launches(ch->chan);
		__atomic_add_fetch(&g_oimgpu_launches, launches - ch->launches_seen, __ATOMIC_RELAXED);
		ch->launches_seen = launches;
	}
	do {
		n = oimgpu_bio_chan_poll(ch->chan, cpl, OIMGPU_REAP_BATCH);
		if (n < 0) {
			SPDK_ERRLOG("oimgpu: channel failed: %s\n", spdk_strerror(-n));
		}
		for (i = 0; i < n; i++) {
			oimgpu_io_done(ch, (struct spdk_bdev_io *)(uintptr_t)cpl[i].tag, cpl[i].status);
		}
		work += n > 0 ? n : 0;
	} while (n == OIMGPU_REAP_BATCH);
	while ((task = TAILQ_FIRST(&ch->resets)) != NULL && task->wait_for <= ch->delivered) {
		TAILQ_REMOVE(&ch->resets, task, link);
		spdk_bdev_io_complete(spdk_bdev_io_from_ctx(task), SPDK_BDEV_IO_STATUS_SUCCESS);
		work++;
	}
	return work > 0 ? work : -1;
}

static int
oimgpu_grow(void **p, uint32_t *cap, uint32_t need, size_t elem)
{
	uint32_t c = *cap ? *cap : 64;
	void *q;

	if (need <= *cap) {
		return 0;
	}
	while (c < need) {
		c *= 2;
	}
	q = realloc(*p, (size_t)c * elem);
	if (!q) {
		return -ENOMEM;
	}
	*p = q;
	*cap = c;
	return 0;
}

/* add one bdev_io to the batch the poller sends next; a bdev_io that cannot be added completes at once */
static void
oimgpu_append(struct oimgpu_channel *ch, struct spdk_bdev_io *bdev_io, uint32_t op)
{
	const bool data = op == OIMGPU_BIO_READ || op == OIMGPU_BIO_WRITE;
	const int iovcnt = data ? bdev_io->u.bdev.iovcnt : 0;
	struct oimgpu_bio *b;
	int i;

	if (oimgpu_grow((void **)&ch->bios, &ch->bio_cap, ch->nbios + 1, sizeof(*ch->bios)) != 0 ||
	    oimgpu_grow((void **)&ch->iovs, &ch->iov_cap, ch->niovs + iovcnt, sizeof(*ch->iovs)) != 0) {
		spdk_bdev_io_complete(bdev_io, SPDK_BDEV_IO_STATUS_NOMEM);
		return;
	}
	for (i = 0; i < iovcnt; i++) {
		if (bdev_io->u.bdev.iovs[i].iov_len > UINT32_MAX) {
			spdk_bdev_io_complete(bdev_io, SPDK_BDEV_IO_STATUS_FAILED);
			return;
		}
	}
	b = &ch->bios[ch->nbios++];
	b->offset_blocks = bdev_io->u.bdev.offset_blocks;
	b->num_blocks = bdev_io->u.bdev.num_blocks;
	b->op = op;
	b->iov_start = ch->niovs;
	b->iovcnt = iovcnt;
	b->flags = 0;
	b->tag = (uint64_t)(uintptr_t)bdev_io;
	for (i = 0; i < iovcnt; i++) {
		ch->iovs[ch->niovs].addr = (uint64_t)(uintptr_t)bdev_io->u.bdev.iovs[i].iov_base;
		ch->iovs[ch->niovs].len = (uint32_t)bdev_io->u.bdev.iovs[i].iov_len;
		ch->iovs[ch->niovs].flags = 0;
		ch->niovs++;
	}
	ch->taken++;
}

static void
oimgpu_read_get_buf_cb(struct spdk_io_channel *_ch, struct spdk_bdev_io *bdev_io)
{
	oimgpu_append(spdk_io_channel_get_ctx(_ch), bdev_io, OIMGPU_BIO_READ);
}

static void
bdev_oimgpu_submit_request(struct spdk_io_channel *_ch, struct spdk_bdev_io *bdev_io)
{
	struct oimgpu_channel *ch = spdk_io_channel_get_ctx(_ch);
	struct oimgpu_task *task = (struct oimgpu_task *)bdev_io->driver_ctx;

	switch (bdev_io->type) {
	case SPDK_BDEV_IO_TYPE_READ:
		if (bdev_io->u.bdev.iovs[0].iov_base == NULL) {
			spdk_bdev_io_get_buf(bdev_io, oimgpu_read_get_buf_cb,
					     bdev_io->u.bdev.num_blocks * bdev_io->bdev->blocklen);
			return;
		}
		oimgpu_append(ch, bdev_io, OIMGPU_BIO_READ);
		return;
	case SPDK_BDEV_IO_TYPE_WRITE:
		oimgpu_append(ch, bdev_io, OIMGPU_BIO_WRITE);
		return;
	case SPDK_BDEV_IO_TYPE_WRITE_ZEROES:
		oimgpu_append(ch, bdev_io, OIMGPU_BIO_WRITE_ZEROES);
		return;
	case SPDK_BDEV_IO_TYPE_UNMAP:
		oimgpu_append(ch, bdev_io, OIMGPU_BIO_UNMAP);
		return;
	case SPDK_BDEV_IO_TYPE_FLUSH:
		spdk_bdev_io_complete(bdev_io, SPDK_BDEV_IO_STATUS_SUCCESS);
		return;
	case SPDK_BDEV_IO_TYPE_RESET:
		task->wait_for = ch->taken;
		TAILQ_INSERT_TAIL(&ch->resets, task, link);
		return;
	default:
		spdk_bdev_io_complete(bdev_io, SPDK_BDEV_IO_STATUS_FAILED);
		return;
	}
}

static bool
bdev_oimgpu_io_type_supported(void *ctx, enum spdk_bdev_io_type io_type)
{
	switch (io_type) {
	case SPDK_BDEV_IO_TYPE_READ:
	case SPDK_BDEV_IO_TYPE_WRITE:
	case SPDK_BDEV_IO_TYPE_FLUSH:
	case SPDK_BDEV_IO_TYPE_RESET:
	case SPDK_BDEV_IO_TYPE_UNMAP:
	case SPDK_BDEV_IO_TYPE_WRITE_ZEROES:
		return true;
	default:
		return false;
	}
}

static struct spdk_io_channel *
bdev_oimgpu_get_io_channel(void *ctx)
{
	return spdk_get_io_channel(ctx);	/* the io_device is the oimgpu_disk: one bio channel per bdev per thread */
}

static void
bdev_oimgpu_write_json_config(struct spdk_bdev *bdev, struct spdk_json_write_ctx *w)
{
	char uuid[SPDK_UUID_STRING_LEN];

	spdk_uuid_fmt_lower(uuid, sizeof(uuid), &bdev->uuid);
	spdk_json_write_object_begin(w);
	spdk_json_write_named_string(w, "method", "construct_oimgpu_bdev");
	spdk_json_write_named_object_begin(w, "params");
	spdk_json_write_named_string(w, "name", bdev->name);
	spdk_json_write_named_uint64(w, "num_blocks", bdev->blockcnt);
	spdk_json_write_named_uint32(w, "block_size", bdev->blocklen);
	spdk_json_write_named_string(w, "uuid", uuid);
	spdk_json_write_object_end(w);
	spdk_json_write_object_end(w);
}

static void
oimgpu_disk_free(struct oimgpu_disk *d)
{
	free(d->disk.name);
	free(d);
}

/* every channel of the disk is gone: the store can go */
static void
oimgpu_disk_unregistered(void *io_device)
{
	struct oimgpu_disk *d = io_device;
	int rc = oimgpu_bdev_delete(d->disk.name);

	spdk_bdev_destruct_done(&d->disk, rc);
	oimgpu_disk_free(d);
}

static int
bdev_oimgpu_destruct(void *ctx)
{
	struct oimgpu_disk *d = ctx;

	TAILQ_REMOVE(&g_oimgpu_disks, d, link);
	spdk_io_device_unregister(d, oimgpu_disk_unregistered);
	return 1;	/* finished by spdk_bdev_destruct_done */
}

static const struct spdk_bdev_fn_table oimgpu_fn_table = {
	.destruct		= bdev_oimgpu_destruct,
	.submit_request		= bdev_oimgpu_submit_request,
	.io_type_supported	= bdev_oimgpu_io_type_supported,
	.get_io_channel		= bdev_oimgpu_get_io_channel,
	.write_config_json	= bdev_oimgpu_write_json_config,
};

static int
oimgpu_channel_create(void *io_device, void *ctx_buf)
{
	struct oimgpu_disk *d = io_device;
	struct oimgpu_channel *ch = ctx_buf;
	int rc;

	memset(ch, 0, sizeof(*ch));
	TAILQ_INIT(&ch->resets);
	rc = oimgpu_bio_chan_open(d->disk.name, &ch->chan);
	if (rc != 0) {
		SPDK_ERRLOG("oimgpu: no channel on %s: %s\n", d->disk.name, spdk_strerror(-rc));
		return rc;
	}
	ch->poller = spdk_poller_register(oimgpu_channel_poll, ch, 0);
	return 0;
}

static void
oimgpu_channel_destroy(void *io_device, void *ctx_buf)
{
	struct oimgpu_channel *ch = ctx_buf;

	spdk_poller_unregister(&ch->poller);
	oimgpu_bio_chan_close(ch->chan);
	free(ch->bios);
	free(ch->iovs);
}

static void
oimgpu_disk_free_unregistered(void *io_device)
{
	oimgpu_disk_free(io_device);
}

struct spdk_bdev *
create_oimgpu_disk(const char *name, const struct spdk_uuid *uuid, uint64_t num_blocks, uint32_t block_size)
{
	struct oimgpu_disk *d;
	char uuid_str[SPDK_UUID_STRING_LEN], store_name[64];
	int rc;

	if (num_blocks == 0) {
		SPDK_ERRLOG("Disk must be more than 0 blocks\n");
		return NULL;
	}
	if (!g_oimgpu_ready) {
		SPDK_ERRLOG("oimgpu: no usable GPU\n");
		return NULL;
	}
	d = calloc(1, sizeof(*d));
	if (!d) {
		return NULL;
	}
	d->disk.name = name ? strdup(name) : spdk_sprintf_alloc("OimGpu%d", g_oimgpu_disk_count++);
	if (!d->disk.name) {
		free(d);
		return NULL;
	}
	if (uuid) {
		d->disk.uuid = *uuid;
	} else {
		spdk_uuid_generate(&d->disk.uuid);
	}
	spdk_uuid_fmt_lower(uuid_str, sizeof(uuid_str), &d->disk.uuid);
	rc = oimgpu_bdev_create_malloc(d->disk.name, uuid_str, num_blocks, block_size, -1, store_name, sizeof(store_name));
	if (rc != 0) {
		SPDK_ERRLOG("oimgpu: could not create the store of %s: %s\n", d->disk.name, spdk_strerror(-rc));
		oimgpu_disk_free(d);
		return NULL;
	}
	d->disk.product_name = "OimGpu disk";
	d->disk.write_cache = 1;
	d->disk.blocklen = block_size;
	d->disk.blockcnt = num_blocks;
	d->disk.ctxt = d;
	d->disk.fn_table = &oimgpu_fn_table;
	d->disk.module = &oimgpu_if;
	spdk_io_device_register(d, oimgpu_channel_create, oimgpu_channel_destroy, sizeof(struct oimgpu_channel),
				"oimgpu_disk");
	rc = spdk_bdev_register(&d->disk);
	if (rc != 0) {
		oimgpu_bdev_delete(d->disk.name);
		spdk_io_device_unregister(d, oimgpu_disk_free_unregistered);
		return NULL;
	}
	TAILQ_INSERT_TAIL(&g_oimgpu_disks, d, link);
	return &d->disk;
}

void
delete_oimgpu_disk(struct spdk_bdev *bdev, spdk_delete_oimgpu_complete cb_fn, void *cb_arg)
{
	if (!bdev || bdev->module != &oimgpu_if) {
		cb_fn(cb_arg, -ENODEV);
		return;
	}
	spdk_bdev_unregister(bdev, cb_fn, cb_arg);
}

/* the library as the application left it (already initialised, control-only included), else the current GPU;
 * without one the module registers no bdevs and the application carries on */
static int
bdev_oimgpu_initialize(void)
{
	int rc = oimgpu_init(NULL, 0);

	g_oimgpu_ready = rc == 0;
	if (rc != 0) {
		SPDK_NOTICELOG("oimgpu bdev module: no usable GPU (%s), no oimgpu bdevs\n", spdk_strerror(-rc));
	}
	return 0;
}
