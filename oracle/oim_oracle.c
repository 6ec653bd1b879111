/*
 * oim_oracle.c — TEST INFRASTRUCTURE: plain-C restatement of the reference's block-I/O hot path.
 *
 * Parity status: PINNED.  This file is checked (tests/test_oracle.py) against
 * oracle/_ref/liboim_ref.so, which is the reference's own SPDK sources compiled from
 * /root/reference and driven through process_requestq() (oracle/ref_driver.c), on the golden
 * cases of SPDK's unit tests (scsi_bdev_ut.c:639-897, vhost_ut.c:153-235), the bdevio data-integrity
 * suite (S/test/bdev/bdevio/bdevio.c:388-800) and seeded random request traces; the resulting
 * vectors are committed under tests/golden/ so the check also runs where /root/reference is absent.
 *
 * One function per reference function, each citing the file:line it follows
 * (S/ = /root/reference/vendor/github.com/spdk/spdk/).  Requests are executed strictly in
 * submission order, as the single reactor thread does.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's CPU legs may load this library; the product
 * (oim_b200/, liboimgpu.so) never does.
 */
#include <errno.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <stdbool.h>

#include "oimgpu.h"

_Static_assert(sizeof(struct oimgpu_req) == 64, "oimgpu_req must be 64 bytes");
_Static_assert(sizeof(struct oimgpu_iov) == 16, "oimgpu_iov must be 16 bytes");
_Static_assert(sizeof(struct oimgpu_cpl) == 48, "oimgpu_cpl must be 48 bytes");
_Static_assert(offsetof(struct oimgpu_req, cdb) == 19, "cdb offset = virtio_scsi_cmd_req.cdb");
_Static_assert(offsetof(struct oimgpu_req, dir) == 51, "tail starts after the 51-byte virtio header");
_Static_assert(offsetof(struct oimgpu_cpl, sense) == 20, "sense offset");

/* SCSI constants (S/include/spdk/scsi_spec.h) */
enum {
	SC_GOOD = 0x00, SC_CHECK_CONDITION = 0x02,
	SK_NO_SENSE = 0x0, SK_ILLEGAL_REQUEST = 0x5, SK_ABORTED_COMMAND = 0xb,
	ASC_NONE = 0x00, ASC_INVALID_OPCODE = 0x20, ASC_LBA_OOR = 0x21, ASC_INVALID_FIELD = 0x24,
	ASC_LUN_NOT_SUPPORTED = 0x25,
	ASCQ_NONE = 0x00,
};
enum { TASK_COMPLETE = 0, TASK_PENDING = 1, TASK_UNKNOWN = 2 };

/* struct malloc_disk (S/lib/bdev/malloc/bdev_malloc.c:50-54) + the bits of struct spdk_bdev used */
struct orc_bdev {
	uint8_t  *buf;		/* malloc_buf: num_blocks*block_size zero-filled bytes */
	uint64_t blockcnt;
	uint32_t blocklen;
	/* what INQUIRY embeds: spdk_bdev name/product_name, spdk_scsi_dev name/id, port name/index,
	 * protocol identifier (vhost-scsi: SAS, vhost_scsi.c:1004-1013) */
	char name[64], product_name[32], dev_name[16], port_name[16];
	int  dev_id, port_index, protocol_id;
	/* spdk_bdev_get_device_stat + the latency histogram's total (oimorc_iostat): num_read_ops, bytes_read,
	 * num_write_ops, bytes_written, num_unmap_ops, bytes_unmapped, bdev_ios */
	uint64_t stat[7];
};

/* per-session target state (struct spdk_scsi_dev_vhost_state, vhost_scsi.c:66-71) */
struct orc_tgt {
	struct orc_bdev *bdev;	/* LUN 0's bdev, NULL = no device in this slot */
	bool removed;		/* session saw a hot-remove (vhost_scsi.c:1093-1100) */
	bool lun_removed;	/* spdk_scsi_lun.removed: LUN being torn down (lun.c:171-176) */
};

struct oimorc {
	struct orc_bdev bdev;		/* the device oimorc_create made */
	struct orc_tgt  tgt[OIMGPU_CTRLR_MAX_DEVS];
	struct orc_bdev *extra[OIMGPU_CTRLR_MAX_DEVS];	/* devices added later (oimorc_add_target), owned */
};

/* struct spdk_scsi_task, the fields the path touches (S/include/spdk/scsi.h:97-146) */
struct orc_task {
	uint8_t  status;
	uint32_t transfer_len, length, dxfer_dir, data_transferred;
	const uint8_t *cdb;
	struct { uint8_t *base; uint32_t len; } iovs[OIMGPU_IOVS_MAX];
	uint16_t iovcnt;
	uint8_t  sense_data[32];
	uint32_t sense_data_len;
};

static inline uint16_t be16(const uint8_t *p) { return (uint16_t)(p[0] << 8 | p[1]); }
static inline uint32_t be32(const uint8_t *p) { return (uint32_t)p[0] << 24 | (uint32_t)p[1] << 16 | (uint32_t)p[2] << 8 | p[3]; }
static inline uint64_t be64(const uint8_t *p) { return (uint64_t)be32(p) << 32 | be32(p + 4); }
static inline void to_be32(uint8_t *p, uint32_t v) { p[0] = v >> 24; p[1] = v >> 16; p[2] = v >> 8; p[3] = v; }
static inline void to_be64(uint8_t *p, uint64_t v) { to_be32(p, v >> 32); to_be32(p + 4, (uint32_t)v); }

int oimorc_desc_to_iov(const uint64_t *regions, uint32_t nregions, uint64_t addr, uint32_t len,
		       struct oimgpu_iov *out, uint32_t start_index);

/* spdk_scsi_task_build_sense_data + spdk_scsi_task_set_status (S/lib/scsi/task.c:198-247) */
static void task_set_status(struct orc_task *t, int sc, int sk, int asc, int ascq)
{
	if (sc == SC_CHECK_CONDITION) {
		uint8_t *cp = t->sense_data;
		memset(cp, 0, 18);
		cp[0] = 0x80 | 0x70;	/* VALID | current, fixed format */
		cp[2] = sk & 0xf;
		cp[7] = 10;		/* additional sense length */
		cp[12] = asc;
		cp[13] = ascq;
		t->sense_data_len = 18;
	}
	t->status = sc;
}

/* spdk_scsi_task_scatter_data (S/lib/scsi/task.c:111-152); the internal-buffer branch
 * (iovcnt==1 && iov_base==NULL) cannot be reached with mapped SG elements and is left out */
static int task_scatter_data(struct orc_task *t, const uint8_t *src, size_t buf_len)
{
	size_t len = 0, buf_left = buf_len;
	int i;

	if (buf_len == 0) return 0;
	for (i = 0; i < t->iovcnt; i++) len += t->iovs[i].len;
	if (len < buf_len) {
		task_set_status(t, SC_CHECK_CONDITION, SK_ILLEGAL_REQUEST, ASC_INVALID_FIELD, ASCQ_NONE);
		return -1;
	}
	for (i = 0; i < t->iovcnt; i++) {
		len = t->iovs[i].len < buf_left ? t->iovs[i].len : buf_left;
		buf_left -= len;
		if (len) memcpy(t->iovs[i].base, src, len);
		src += len;
	}
	return (int)buf_len;
}

/* spdk_bdev_bytes_to_blocks + spdk_bdev_io_valid_blocks (S/lib/bdev/bdev.c:2474-2509) */
static int bdev_bytes_to_blocks(const struct orc_bdev *b, uint64_t off, uint64_t *off_blk,
				uint64_t n, uint64_t *n_blk)
{
	*off_blk = off / b->blocklen;
	*n_blk = n / b->blocklen;
	return (off % b->blocklen) | (n % b->blocklen) ? -1 : 0;
}
static bool bdev_valid_blocks(const struct orc_bdev *b, uint64_t off_blk, uint64_t n_blk)
{
	if (off_blk + n_blk < off_blk) return false;
	if (off_blk + n_blk > b->blockcnt) return false;
	return true;
}

/* What _spdk_bdev_io_complete books for one completed bdev_io (S/lib/bdev/bdev.c:3236-3258): the histogram
 * tallies every bdev_io whatever its type and status, the counters only successful reads, writes and unmaps.
 * A request refused before a bdev_io exists (spdk_bdev_readv & co. returning -EINVAL) books nothing. */
enum { IO_READ, IO_WRITE, IO_UNMAP, IO_FLUSH };
static void bdev_io_complete(struct orc_bdev *b, int type, uint64_t nb, bool success)
{
	b->stat[6]++;
	if (!success || type == IO_FLUSH) return;
	b->stat[2 * type]++;
	b->stat[2 * type + 1] += nb * b->blocklen;
}

/* bdev_malloc_check_iov_len (S/lib/bdev/malloc/bdev_malloc.c:137-150): fails only when the
 * iovecs are SHORTER than nbytes */
static int malloc_check_iov_len(const struct orc_task *t, size_t nbytes)
{
	int i;
	for (i = 0; i < t->iovcnt; i++) {
		if (nbytes < t->iovs[i].len) return 0;
		nbytes -= t->iovs[i].len;
	}
	return nbytes != 0;
}

/* spdk_bdev_readv -> bdev_malloc_readv -> mem_copy_submit
 * (bdev.c:2559-2602, bdev_malloc.c:153-185, S/lib/copy/copy_engine.c:114-126).
 * Returns 0, -EINVAL, or 1 when the bdev_io itself completes FAILED. */
static int bdev_readv(struct orc_bdev *b, struct orc_task *t, uint64_t offset, uint64_t nbytes)
{
	uint64_t ob, nb;
	const uint8_t *src;
	int i;

	if (bdev_bytes_to_blocks(b, offset, &ob, nbytes, &nb) != 0) return -EINVAL;
	if (!bdev_valid_blocks(b, ob, nb)) return -EINVAL;
	if (malloc_check_iov_len(t, nb * b->blocklen)) {
		bdev_io_complete(b, IO_READ, nb, false);
		return 1;
	}
	src = b->buf + ob * b->blocklen;
	for (i = 0; i < t->iovcnt; i++) {
		if (t->iovs[i].len) memcpy(t->iovs[i].base, src, t->iovs[i].len);
		src += t->iovs[i].len;
	}
	bdev_io_complete(b, IO_READ, nb, true);
	return 0;
}

/* spdk_bdev_writev -> bdev_malloc_writev -> mem_copy_submit (bdev.c:2656-2703, bdev_malloc.c:188-219) */
static int bdev_writev(struct orc_bdev *b, struct orc_task *t, uint64_t offset, uint64_t nbytes)
{
	uint64_t ob, nb;
	uint8_t *dst;
	int i;

	if (bdev_bytes_to_blocks(b, offset, &ob, nbytes, &nb) != 0) return -EINVAL;
	if (!bdev_valid_blocks(b, ob, nb)) return -EINVAL;
	if (malloc_check_iov_len(t, nb * b->blocklen)) {
		bdev_io_complete(b, IO_WRITE, nb, false);
		return 1;
	}
	dst = b->buf + ob * b->blocklen;
	for (i = 0; i < t->iovcnt; i++) {
		if (t->iovs[i].len) memcpy(dst, t->iovs[i].base, t->iovs[i].len);
		dst += t->iovs[i].len;
	}
	bdev_io_complete(b, IO_WRITE, nb, true);
	return 0;
}

/* spdk_bdev_unmap_blocks -> bdev_malloc_unmap -> mem_copy_fill
 * (bdev.c:2780-2821, bdev_malloc.c:222-233, copy_engine.c:128-140) */
static int bdev_unmap_blocks(struct orc_bdev *b, uint64_t ob, uint64_t nb)
{
	if (!bdev_valid_blocks(b, ob, nb)) return -EINVAL;
	if (nb == 0) return -EINVAL;
	memset(b->buf + ob * b->blocklen, 0, nb * b->blocklen);
	bdev_io_complete(b, IO_UNMAP, nb, true);
	return 0;
}

/* bdev_io FAILED -> spdk_bdev_io_get_scsi_status default branch (bdev.c:3391-3423) */
static void task_set_bdev_failed(struct orc_task *t)
{
	task_set_status(t, SC_CHECK_CONDITION, SK_ABORTED_COMMAND, ASC_NONE, ASCQ_NONE);
}

/* spdk_bdev_scsi_read (S/lib/scsi/scsi_bdev.c:1318-1357) */
static int scsi_read(struct orc_bdev *b, struct orc_task *t, uint64_t lba)
{
	uint64_t nbytes = t->length;	/* NOT xfer_len*blocklen: the payload length rules */
	int rc = bdev_readv(b, t, lba * b->blocklen, nbytes);

	if (rc < 0) {
		task_set_status(t, SC_CHECK_CONDITION, SK_NO_SENSE, ASC_NONE, ASCQ_NONE);
		return TASK_COMPLETE;
	}
	t->data_transferred = (uint32_t)nbytes;
	if (rc > 0) task_set_bdev_failed(t);
	return TASK_PENDING;
}

/* spdk_bdev_scsi_write (scsi_bdev.c:1360-1411) */
static int scsi_write(struct orc_bdev *b, struct orc_task *t, uint64_t lba, uint32_t len)
{
	uint64_t nbytes = (uint64_t)len * b->blocklen;
	int rc;

	if (nbytes > t->transfer_len) {
		task_set_status(t, SC_CHECK_CONDITION, SK_NO_SENSE, ASC_NONE, ASCQ_NONE);
		return TASK_COMPLETE;
	}
	rc = bdev_writev(b, t, lba * b->blocklen, t->length);
	if (rc < 0) {
		task_set_status(t, SC_CHECK_CONDITION, SK_NO_SENSE, ASC_NONE, ASCQ_NONE);
		return TASK_COMPLETE;
	}
	t->data_transferred = t->length;
	if (rc > 0) task_set_bdev_failed(t);
	return TASK_PENDING;
}

/* spdk_bdev_scsi_readwrite (scsi_bdev.c:1456-1511) */
static int scsi_readwrite(struct orc_bdev *b, struct orc_task *t, uint64_t lba, uint32_t xfer_len,
			  bool is_read)
{
	uint32_t max_xfer_len;

	t->data_transferred = 0;
	if (t->dxfer_dir != OIMGPU_DIR_NONE &&
	    t->dxfer_dir != (is_read ? OIMGPU_DIR_FROM_DEV : OIMGPU_DIR_TO_DEV)) {
		task_set_status(t, SC_CHECK_CONDITION, SK_NO_SENSE, ASC_NONE, ASCQ_NONE);
		return TASK_COMPLETE;
	}
	if (b->blockcnt <= lba || b->blockcnt - lba < xfer_len) {
		task_set_status(t, SC_CHECK_CONDITION, SK_ILLEGAL_REQUEST, ASC_LBA_OOR, ASCQ_NONE);
		return TASK_COMPLETE;
	}
	if (xfer_len == 0) {
		t->status = SC_GOOD;
		return TASK_COMPLETE;
	}
	max_xfer_len = OIMGPU_MAX_XFER_BYTES / b->blocklen;
	if (xfer_len > max_xfer_len) {
		task_set_status(t, SC_CHECK_CONDITION, SK_ILLEGAL_REQUEST, ASC_INVALID_FIELD, ASCQ_NONE);
		return TASK_COMPLETE;
	}
	return is_read ? scsi_read(b, t, lba) : scsi_write(b, t, lba, xfer_len);
}

/* spdk_bdev_scsi_sync (scsi_bdev.c:1414-1454); Malloc FLUSH is a no-op success (bdev_malloc.c:235-241), but its
 * bdev_io is tallied like any other */
static int scsi_sync(struct orc_bdev *b, struct orc_task *t, uint64_t lba, uint32_t num_blocks)
{
	if (num_blocks == 0) return TASK_COMPLETE;
	if (lba >= b->blockcnt || num_blocks > b->blockcnt || lba > b->blockcnt - num_blocks) {
		task_set_status(t, SC_CHECK_CONDITION, SK_NO_SENSE, ASC_NONE, ASCQ_NONE);
		return TASK_COMPLETE;
	}
	bdev_io_complete(b, IO_FLUSH, num_blocks, true);
	t->data_transferred = 0;
	return TASK_PENDING;
}

/* __copy_desc + spdk_bdev_scsi_unmap (scsi_bdev.c:1545-1679) */
static int scsi_unmap(struct orc_bdev *b, struct orc_task *t)
{
	uint8_t *data = NULL, *gathered = NULL;
	size_t data_len = 0;
	int desc_count = -1, i, submitted = 0;

	if (t->iovcnt == 1) {
		data = t->iovs[0].base;
		data_len = t->iovs[0].len;
	} else {
		/* spdk_scsi_task_gather_data (task.c:154-186) */
		for (i = 0; i < t->iovcnt; i++) data_len += t->iovs[i].len;
		if (data_len != 0) {
			uint8_t *pos = gathered = malloc(data_len);
			for (i = 0; i < t->iovcnt; i++) {
				memcpy(pos, t->iovs[i].base, t->iovs[i].len);
				pos += t->iovs[i].len;
			}
			data = gathered;
		}
	}
	if (data && data_len >= 8) {
		uint16_t desc_data_len = be16(&data[2]);
		if (desc_data_len <= data_len - 8 && desc_data_len / 16 <= OIMGPU_MAX_UNMAP_DESC) {
			desc_count = desc_data_len / 16;
		}
	}
	if (desc_count < 0) {
		free(gathered);
		task_set_status(t, SC_CHECK_CONDITION, SK_ILLEGAL_REQUEST, ASC_INVALID_FIELD, ASCQ_NONE);
		return TASK_COMPLETE;
	}
	for (i = 0; i < desc_count; i++) {
		const uint8_t *d = &data[8 + 16 * i];
		uint64_t ob = be64(d);
		uint32_t nb = be32(d + 8);

		if (nb == 0) continue;
		if (bdev_unmap_blocks(b, ob, nb) != 0) {
			/* descriptors before this one stay applied; the rest are skipped */
			task_set_status(t, SC_CHECK_CONDITION, SK_NO_SENSE, ASC_NONE, ASCQ_NONE);
			break;
		}
		submitted++;
	}
	free(gathered);
	return submitted == 0 ? TASK_COMPLETE : TASK_PENDING;
}

/* spdk_bdev_scsi_process_block (scsi_bdev.c:1681-1802) */
static int scsi_process_block(struct orc_bdev *b, struct orc_task *t)
{
	const uint8_t *cdb = t->cdb;
	uint64_t lba;
	uint32_t xfer_len, len;

	switch (cdb[0]) {
	case 0x08: case 0x0a:	/* READ_6 / WRITE_6 */
		lba = (uint64_t)cdb[1] << 16 | (uint64_t)cdb[2] << 8 | cdb[3];
		xfer_len = cdb[4];
		if (xfer_len == 0) xfer_len = 256;
		return scsi_readwrite(b, t, lba, xfer_len, cdb[0] == 0x08);
	case 0x28: case 0x2a:	/* READ_10 / WRITE_10 */
		return scsi_readwrite(b, t, be32(&cdb[2]), be16(&cdb[7]), cdb[0] == 0x28);
	case 0xa8: case 0xaa:	/* READ_12 / WRITE_12 */
		return scsi_readwrite(b, t, be32(&cdb[2]), be32(&cdb[6]), cdb[0] == 0xa8);
	case 0x88: case 0x8a:	/* READ_16 / WRITE_16 */
		return scsi_readwrite(b, t, be64(&cdb[2]), be32(&cdb[10]), cdb[0] == 0x88);

	case 0x25: {		/* READ CAPACITY (10) */
		uint8_t buffer[8];
		if (b->blockcnt - 1 > 0xffffffffULL) memset(buffer, 0xff, 4);
		else to_be32(buffer, (uint32_t)(b->blockcnt - 1));
		to_be32(&buffer[4], b->blocklen);
		len = t->length < sizeof(buffer) ? t->length : sizeof(buffer);
		if (task_scatter_data(t, buffer, len) < 0) break;
		t->data_transferred = len;
		t->status = SC_GOOD;
		break;
	}
	case 0x9e:		/* SERVICE ACTION IN (16) */
		if ((cdb[1] & 0x1f) != 0x10) return TASK_UNKNOWN;
		{		/* READ CAPACITY (16) */
			uint8_t buffer[32] = {0};
			to_be64(&buffer[0], b->blockcnt - 1);
			to_be32(&buffer[8], b->blocklen);
			buffer[14] |= 1 << 7;	/* TPE: Malloc supports UNMAP (bdev_malloc.c:326-340) */
			len = be32(&cdb[10]) < sizeof(buffer) ? be32(&cdb[10]) : sizeof(buffer);
			if (task_scatter_data(t, buffer, len) < 0) break;
			t->data_transferred = len;
			t->status = SC_GOOD;
		}
		break;

	case 0x35: case 0x91:	/* SYNCHRONIZE CACHE (10) / (16) */
		if (cdb[0] == 0x35) { lba = be32(&cdb[2]); len = be16(&cdb[7]); }
		else { lba = be64(&cdb[2]); len = be32(&cdb[10]); }
		if (len == 0) len = (uint32_t)(b->blockcnt - lba);	/* u64 -> u32 truncation as in the reference */
		return scsi_sync(b, t, lba, len);

	case 0x42:		/* UNMAP */
		return scsi_unmap(b, t);

	default:
		return TASK_UNKNOWN;
	}
	return TASK_COMPLETE;
}

static inline void to_be16(uint8_t *p, uint16_t v) { p[0] = v >> 8; p[1] = (uint8_t)v; }

/* spdk_strcpy_pad (S/lib/util/string.c:220-231) */
static void strcpy_pad(uint8_t *dst, const char *src, size_t size, int pad)
{
	size_t len = strlen(src);
	if (len < size) { memcpy(dst, src, len); memset(dst + len, pad, size - len); }
	else memcpy(dst, src, size);
}

/* spdk_bdev_scsi_set_naa_ieee_extended (scsi_bdev.c:78-103): nibbles of the first 16 name characters,
 * non-hex characters taken at face value and truncated to a byte */
static void set_naa_ieee_extended(const char *name, uint8_t *buf)
{
	int i, count = 0;
	uint64_t v = 0;
	for (i = 0; i < 16 && name[i] != '\0'; i++) {
		int ch = name[i], value;
		if (ch >= '0' && ch <= '9') value = ch - '0';
		else {
			ch = (ch >= 'A' && ch <= 'Z') ? ch + 32 : ch;
			value = (ch >= 'a' && ch <= 'f') ? ch - 'a' + 10 : ch;
		}
		if (i % 2) buf[count++] |= (uint8_t)(value << 4);
		else buf[count] = (uint8_t)value;
	}
	memcpy(&v, buf, 8);		/* host (little-endian) load, as *(uint64_t *)buf */
	v &= 0x0fff000000ffffffull;
	v |= 0x2000000347000000ull;	/* NAA 2, IEEE company id 00 03 47 (Intel) */
	to_be64(buf, v);
}

/* spdk_bdev_scsi_inquiry (scsi_bdev.c:188-805).  data: zeroed buffer of max(4096, alloc_len).
 * Returns the response length or -1 with the task status set. */
static int scsi_inquiry(const struct orc_bdev *b, struct orc_task *t, const uint8_t *cdb, uint8_t *data, uint16_t alloc_len)
{
	const int pc = cdb[2], evpd = cdb[1] & 1;
	int hlen = 0, len = 0, i;

	if (alloc_len < 0x24) goto inq_error;
	if (!evpd && pc) {
		task_set_status(t, SC_CHECK_CONDITION, SK_ILLEGAL_REQUEST, ASC_INVALID_FIELD, ASCQ_NONE);
		return -1;
	}
	if (evpd) {
		uint8_t *params = data + 4;
		data[0] = 0;		/* peripheral qualifier 0 (connected) | device type 0 (disk) */
		data[1] = pc;
		switch (pc) {
		case 0x00: {		/* supported VPD pages */
			static const uint8_t pages[] = { 0x00, 0x80, 0x83, 0x85, 0x86, 0x87, 0x88, 0xb0, 0xb1, 0xb2 };
			hlen = 4;
			memcpy(params, pages, sizeof(pages));
			len = sizeof(pages);	/* Malloc supports UNMAP: page 0xb2 is listed */
			to_be16(&data[2], len);
			break;
		}
		case 0x80:		/* unit serial number = bdev name, at most 31 characters + NUL */
			hlen = 4;
			len = (int)strlen(b->name) + 1;
			if (len > 32) len = 32;
			memcpy(params, b->name, len - 1);
			params[len - 1] = 0;
			to_be16(&data[2], len);
			break;
		case 0x83: {		/* device identification */
			uint8_t *buf = params;
			int dl;
			hlen = 4;
			/* worst-case size check made before anything is built (scsi_bdev.c:284-299) */
			len = (4 + 8) + (4 + 8 + 16 + 32) + (4 + 255 + 1) + (4 + 255) + (4 + 4) * 3;
			if (4 + len > alloc_len) {
				task_set_status(t, SC_CHECK_CONDITION, SK_ILLEGAL_REQUEST, ASC_INVALID_FIELD, ASCQ_NONE);
				return -1;
			}
#define DESIG(code_set, type, assoc, dlen) do { buf[0] = (code_set) | b->protocol_id << 4; \
		buf[1] = (type) | (assoc) << 4 | 1 << 7; buf[2] = 0; buf[3] = (dlen); } while (0)
			DESIG(1, 3, 0, 8);				/* NAA, logical unit */
			set_naa_ieee_extended(b->name, buf + 4);
			len = 4 + 8; buf += 4 + 8;
			DESIG(2, 1, 0, 8 + 16 + 32);			/* T10 vendor id, logical unit */
			strcpy_pad(buf + 4, "INTEL", 8, ' ');
			strcpy_pad(buf + 12, b->product_name, 16, ' ');
			strcpy_pad(buf + 28, b->name, 32, ' ');
			len += 4 + 56; buf += 4 + 56;
			dl = (int)strlen(b->dev_name);			/* spdk_bdev_scsi_pad_scsi_name: NUL-pad to x4 */
			memcpy(buf + 4, b->dev_name, dl);
			do { buf[4 + dl++] = 0; } while (dl & 3);
			DESIG(3, 8, 2, dl);				/* SCSI name, target device */
			len += 4 + dl; buf += 4 + dl;
			dl = (int)strlen(b->port_name);
			memcpy(buf + 4, b->port_name, dl);
			DESIG(3, 8, 1, dl);				/* SCSI name, target port */
			len += 4 + dl; buf += 4 + dl;
			DESIG(1, 4, 1, 4);				/* relative target port */
			to_be16(buf + 6, b->port_index);
			len += 8; buf += 8;
			DESIG(1, 5, 1, 4);				/* target port group */
			len += 8; buf += 8;
			DESIG(1, 6, 0, 4);				/* logical unit group = device id */
			to_be16(buf + 6, b->dev_id);
			len += 8;
#undef DESIG
			to_be16(&data[2], len);
			break;
		}
		case 0x86:		/* extended inquiry: the memset wipes the page code too (scsi_bdev.c:420) */
			memset(data, 0, 64);
			hlen = 4;
			data[5] = 0x04 | 0x01;	/* HEADSUP | SIMPSUP */
			len = 64 - hlen;
			to_be16(&data[2], len);
			break;
		case 0x85:		/* management network addresses: empty */
			hlen = 4;
			to_be16(&data[2], len);
			break;
		case 0x87:		/* mode page policy: all pages / subpages shared */
			hlen = 4;
			params[0] = 0x3f; params[1] = 0xff; params[2] = 0; params[3] = 0;
			len += 4;
			to_be16(&data[2], len);
			break;
		case 0x88: {		/* SCSI ports: one used port.  struct spdk_scsi_port_desc is 14 bytes but only
					 * 12 are counted, so the reported length cuts the name short by 2 (scsi_bdev.c:503-540) */
			uint8_t *sd = params;
			int plen = (int)strlen(b->port_name);
			hlen = 4;
			to_be16(sd + 2, b->port_index);
			len += 12;
			sd[14] = 0x05 << 4 | 0x03;	/* iSCSI | UTF-8 */
			sd[15] = 0x80 | 1 << 4 | 8;	/* PIV | target port | SCSI name */
			sd[16] = 0;
			sd[17] = plen;
			memcpy(sd + 18, b->port_name, plen);
			to_be16(sd + 12, 4 + plen);
			len += 4 + plen;
			to_be16(&data[2], len);
			break;
		}
		case 0xb0: {		/* block limits */
			uint32_t blocks = (1024u * 1024u) / b->blocklen;
			memset(&data[4], 0, 60);
			hlen = 4;
			data[5] = blocks > 0xff ? 0xff : blocks;
			to_be16(&data[6], b->blocklen < 4096 ? 4096 / b->blocklen : 1);
			blocks = OIMGPU_MAX_XFER_BYTES / b->blocklen;
			to_be32(&data[8], blocks);
			to_be32(&data[12], blocks);
			to_be32(&data[20], 4194304);	/* maximum unmap LBA count */
			to_be32(&data[24], OIMGPU_MAX_UNMAP_DESC);
			to_be64(&data[36], 512);	/* maximum write same length */
			len = 64 - hlen;
			to_be16(&data[2], len);
			break;
		}
		case 0xb1:		/* block device characteristics: non-rotating, 3.5" */
			hlen = 4;
			len = 64 - hlen;
			to_be16(&data[4], 1);
			data[6] = 0;
			data[7] = 0x02 << 4;
			memset(&data[8], 0, 64 - 8);
			to_be16(&data[2], len);
			break;
		case 0xb2:		/* logical block provisioning: LBPU, thin */
			hlen = 4;
			len = 7;
			data[4] = 0;
			data[5] |= 1 << 7;
			data[6] = 0x02;
			to_be16(&data[2], len);
			break;
		default:
			goto inq_error;
		}
	} else {
		/* standard INQUIRY data (struct spdk_scsi_cdb_inquiry_data) */
		data[0] = 0;
		data[1] = 0;
		data[2] = 0x05;		/* SPC-3 */
		data[3] = 2 | 1 << 4;	/* response format 2, HISUP */
		hlen = 5;
		data[5] = 0;
		data[6] = 0x10;		/* MULTIP */
		data[7] = 0x2;		/* CMDQUE */
		strcpy_pad(&data[8], "INTEL", 8, ' ');
		strcpy_pad(&data[16], b->product_name, 16, ' ');
		strcpy_pad(&data[32], "0001", 4, ' ');
		len = 36 - 5;
		if (alloc_len >= 56) { memset(&data[36], 0x20, 20); len += 20; }
		if (alloc_len >= 57) { data[56] = 0; len += 1; }
		if (alloc_len >= 58) { data[57] = 0; len += 1; }
		if (alloc_len >= 58 + 2) { to_be16(&data[58], 0x0960); len += 2; }
		if (alloc_len >= 58 + 4) { to_be16(&data[60], 0x0300); len += 2; }
		if (alloc_len >= 58 + 6) { to_be16(&data[62], 0x0320); len += 2; }
		if (alloc_len >= 58 + 8) { to_be16(&data[64], 0x0040); len += 2; }
		if (alloc_len > 58 + 8) {
			i = alloc_len - (58 + 8);
			if (i > 30) i = 30;
			memset(&data[66], 0, i);
			len += i;
		}
		data[4] = len;		/* additional length */
	}
	return hlen + len;

inq_error:
	t->data_transferred = 0;
	task_set_status(t, SC_CHECK_CONDITION, SK_NO_SENSE, ASC_NONE, ASCQ_NONE);
	return -1;
}

/* mode_sense_page_init + spdk_bdev_scsi_mode_sense_page (scsi_bdev.c:807-1100); cp may be NULL */
static void mode_page_init(uint8_t *buf, int len, int page, int subpage)
{
	if (!buf) return;
	memset(buf, 0, len);
	if (subpage != 0) { buf[0] = page | 0x40; buf[1] = subpage; to_be16(&buf[2], len - 4); }
	else { buf[0] = page; buf[1] = len - 2; }
}

static int scsi_mode_sense_page(struct orc_task *t, int pc, int page, int subpage, uint8_t *cp)
{
	int len = 0, plen = 0, i;

	if (pc == 3) {
		task_set_status(t, SC_CHECK_CONDITION, SK_ILLEGAL_REQUEST, 0x39 /* SAVING PARAMETERS NOT SUPPORTED */, ASCQ_NONE);
		return -1;
	}
	switch (page) {
	case 0x01: case 0x07: case 0x1a: case 0x1c: plen = 0x0a + 2; break;	/* error recovery, verify, power, IEC */
	case 0x02: plen = 0x0e + 2; break;					/* disconnect-reconnect */
	case 0x08: plen = 0x12 + 2; break;					/* caching */
	case 0x10: plen = 0x16 + 2; break;					/* XOR control */
	case 0x0a:
		if (subpage == 0x00) { plen = 0x0a + 2; break; }
		if (subpage == 0x01) { mode_page_init(cp, 0x1c + 4, page, subpage); return 0x1c + 4; }
		if (subpage == 0xff) {
			len += scsi_mode_sense_page(t, pc, page, 0x00, cp ? &cp[len] : NULL);
			len += scsi_mode_sense_page(t, pc, page, 0x01, cp ? &cp[len] : NULL);
		}
		return len;
	case 0x3f:
		if (subpage == 0x00 || subpage == 0xff) {
			for (i = 0x00; i < 0x3e; i++) len += scsi_mode_sense_page(t, pc, i, 0x00, cp ? &cp[len] : NULL);
		}
		if (subpage == 0xff) {
			for (i = 0x00; i < 0x3e; i++) len += scsi_mode_sense_page(t, pc, i, 0xff, cp ? &cp[len] : NULL);
		}
		return len;
	default:
		return 0;
	}
	if (subpage != 0x00) return 0;
	mode_page_init(cp, plen, page, subpage);
	if (page == 0x08 && cp && pc != 0x01) cp[2] |= 0x4 | 0x1;	/* WCE (Malloc has a write cache) | RCD */
	return plen;
}

/* spdk_bdev_scsi_mode_sense (scsi_bdev.c:1102-1174) */
static int scsi_mode_sense(const struct orc_bdev *b, struct orc_task *t, int md, int dbd, int llbaa, int pc,
			   int page, int subpage, uint8_t *data)
{
	int hlen = md == 6 ? 4 : 8, blen = md == 6 ? 8 : (llbaa ? 16 : 8), plen, total;

	if (dbd) blen = 0;
	plen = scsi_mode_sense_page(t, pc, page, subpage, data ? &data[hlen + blen] : NULL);
	if (plen < 0) return -1;
	total = hlen + blen + plen;
	if (!data) return total;
	if (hlen == 4) {
		data[0] = total - 1; data[1] = 0; data[2] = 0; data[3] = blen;
	} else {
		to_be16(&data[0], total - 2);
		data[2] = 0; data[3] = 0; data[4] = llbaa ? 1 : 0; data[5] = 0;
		to_be16(&data[6], blen);
	}
	if (blen == 16) {
		to_be64(&data[hlen], b->blockcnt);
		memset(&data[hlen + 8], 0, 4);
		to_be32(&data[hlen + 12], b->blocklen);
	} else if (blen == 8) {
		if (b->blockcnt > 0xffffffffULL) memset(&data[hlen], 0xff, 4);
		else to_be32(&data[hlen], (uint32_t)b->blockcnt);
		to_be32(&data[hlen + 4], b->blocklen);
	}
	return total;
}

/* spdk_bdev_scsi_check_len (scsi_bdev.c:1812-1825) */
static int scsi_check_len(struct orc_task *t, int len, int min_len)
{
	if (len >= min_len) return 0;
	task_set_status(t, SC_CHECK_CONDITION, SK_ILLEGAL_REQUEST, ASC_INVALID_FIELD, ASCQ_NONE);
	return -1;
}

/* spdk_bdev_scsi_process_primary (scsi_bdev.c:1827-2077) */
static int scsi_process_primary(struct orc_bdev *b, struct orc_task *t)
{
	const uint8_t *cdb = t->cdb;
	int rc = 0, data_len = -1, alloc_len = -1, md = 0, pllen, bdlen = 0;
	uint8_t *data = NULL;

	switch (cdb[0]) {
	case 0x12:		/* INQUIRY */
		alloc_len = be16(&cdb[3]);
		data_len = alloc_len > 4096 ? alloc_len : 4096;
		data = calloc(1, data_len);
		rc = scsi_inquiry(b, t, cdb, data, (uint16_t)data_len);	/* the BUFFER size, not the CDB's allocation length (scsi_bdev.c:1850) */
		data_len = rc < data_len ? rc : data_len;
		break;
	case 0xa0:		/* REPORT LUNS: one LUN (id 0), flat addressing (scsi_bdev.c:105-172) */
		alloc_len = (int)be32(&cdb[6]);
		rc = scsi_check_len(t, alloc_len, 16);
		if (rc < 0) break;
		data_len = alloc_len > 4096 ? alloc_len : 4096;
		data = calloc(1, data_len);
		if (cdb[2] > 0x02) {
			rc = -1;
			task_set_status(t, SC_CHECK_CONDITION, SK_NO_SENSE, ASC_NONE, ASCQ_NONE);
			data_len = rc;
			break;
		}
		to_be32(data, 8);
		rc = data_len = 16;
		break;
	case 0x15: case 0x55:	/* MODE SELECT (6) / (10): lengths are validated, pages are accepted and ignored */
		md = cdb[0] == 0x15 ? 4 : 8;
		pllen = cdb[0] == 0x15 ? cdb[4] : be16(&cdb[7]);
		if (pllen == 0) break;
		rc = scsi_check_len(t, pllen, md);
		if (rc < 0) break;
		{
			size_t total = 0;
			int i;
			for (i = 0; i < t->iovcnt; i++) total += t->iovs[i].len;
			data_len = (int)total;
			if (total) {
				uint8_t *pos = data = malloc(total);
				for (i = 0; i < t->iovcnt; i++) { if (t->iovs[i].len) memcpy(pos, t->iovs[i].base, t->iovs[i].len); pos += t->iovs[i].len; }
			}
		}
		rc = scsi_check_len(t, data_len, md);
		if (rc >= 0) bdlen = md == 4 ? data[3] : be16(&data[6]);
		if (rc < 0) break;
		(void)bdlen;	/* spdk_bdev_scsi_mode_select_page only walks the pages; nothing is applied */
		rc = pllen;
		data_len = 0;
		break;
	case 0x1a: case 0x5a: {	/* MODE SENSE (6) / (10) */
		int llba = 0, dbd, pc, page, subpage;
		if (cdb[0] == 0x1a) { alloc_len = cdb[4]; md = 6; }
		else { alloc_len = be16(&cdb[7]); llba = !!(cdb[1] & 0x10); md = 10; }
		dbd = !!(cdb[1] & 0x8);
		pc = (cdb[2] & 0xc0) >> 6;
		page = cdb[2] & 0x3f;
		subpage = cdb[3];
		rc = scsi_mode_sense(b, t, md, dbd, llba, pc, page, subpage, NULL);
		if (rc < 0) break;
		data_len = rc;
		data = calloc(1, data_len);
		rc = scsi_mode_sense(b, t, md, dbd, llba, pc, page, subpage, data);
		break;
	}
	case 0x03:		/* REQUEST SENSE */
		if (cdb[1] & 0x1) {
			task_set_status(t, SC_CHECK_CONDITION, SK_ILLEGAL_REQUEST, ASC_INVALID_FIELD, ASCQ_NONE);
			break;
		}
		alloc_len = cdb[4];
		task_set_status(t, SC_CHECK_CONDITION, SK_NO_SENSE, 0, 0);	/* build_sense_data only... */
		t->status = SC_GOOD;						/* ...status is set below */
		data_len = (int)t->sense_data_len;
		data = malloc(data_len);
		memcpy(data, t->sense_data, data_len);
		break;
	case 0x4c: case 0x4d:	/* LOG SELECT / LOG SENSE */
		task_set_status(t, SC_CHECK_CONDITION, SK_ILLEGAL_REQUEST, ASC_INVALID_OPCODE, ASCQ_NONE);
		rc = -1;
		break;
	case 0x00: case 0x1b:	/* TEST UNIT READY / START STOP UNIT */
		rc = 0;
		break;
	default:
		return TASK_UNKNOWN;
	}
	if (rc >= 0 && data_len > 0) {
		task_scatter_data(t, data, alloc_len < data_len ? alloc_len : data_len);
		rc = data_len < alloc_len ? data_len : alloc_len;
	}
	if (rc >= 0) {
		t->data_transferred = rc;
		t->status = SC_GOOD;
	}
	free(data);
	return TASK_COMPLETE;
}

/* spdk_bdev_scsi_execute (scsi_bdev.c:2079-2097) */
static void scsi_execute(struct orc_bdev *b, struct orc_task *t)
{
	int rc = scsi_process_block(b, t);
	if (rc == TASK_UNKNOWN) rc = scsi_process_primary(b, t);
	if (rc == TASK_UNKNOWN) {
		task_set_status(t, SC_CHECK_CONDITION, SK_ILLEGAL_REQUEST, ASC_INVALID_OPCODE, ASCQ_NONE);
	}
}

/* spdk_scsi_task_process_null_lun (S/lib/scsi/task.c:258-293) */
static void task_process_null_lun(struct orc_task *t)
{
	t->length = t->transfer_len;
	if (t->cdb[0] == 0x12) {	/* INQUIRY */
		uint8_t buffer[36];
		uint32_t alloc_len = be16(&t->cdb[3]);
		memset(buffer, 0, sizeof(buffer));
		buffer[0] = 0x03 << 5 | 0x1f;
		buffer[4] = sizeof(buffer) - 5;
		if (task_scatter_data(t, buffer, alloc_len < sizeof(buffer) ? alloc_len : sizeof(buffer)) >= 0) {
			t->data_transferred = sizeof(buffer);
			t->status = SC_GOOD;
		}
	} else {
		task_set_status(t, SC_CHECK_CONDITION, SK_ILLEGAL_REQUEST, ASC_LUN_NOT_SUPPORTED, ASCQ_NONE);
		t->data_transferred = 0;
	}
}

/* process_request after task_data_setup (vhost_scsi.c:633-653) -> task_submit / null-LUN early
 * completion / BAD_TARGET, then spdk_vhost_scsi_task_cpl (311-331).  `t` carries the SG list. */
static void execute_task(struct oimorc *o, struct orc_task *t, const uint8_t *lun, struct oimgpu_cpl *c)
{
	struct orc_tgt *tgt;
	struct orc_bdev *lun_bdev = NULL;
	uint16_t lun_id;

	/* ---- spdk_vhost_scsi_task_init_target ---- */
	lun_id = (((uint16_t)lun[2] << 8) | lun[3]) & 0x3FFF;
	if (lun[0] != 1 || lun[1] >= OIMGPU_CTRLR_MAX_DEVS) {
		c->response = OIMGPU_S_BAD_TARGET;
		return;
	}
	tgt = &o->tgt[lun[1]];
	if (tgt->bdev == NULL || tgt->removed) {
		if (!tgt->removed) {
			c->response = OIMGPU_S_BAD_TARGET;
			return;
		}
		/* hot-detached: LUN stays NULL so the guest gets a sense code */
	} else if (lun_id == 0) {
		lun_bdev = tgt->bdev;	/* spdk_scsi_dev_get_lun(dev, 0) */
	}

	c->response = OIMGPU_S_OK;
	if (lun_bdev == NULL) {
		task_process_null_lun(t);
	} else {
		/* _spdk_scsi_lun_execute_task (S/lib/scsi/lun.c:163-189) */
		t->status = SC_GOOD;
		if (tgt->lun_removed) {
			/* spdk_scsi_task_process_abort (task.c:295-302) */
			task_set_status(t, SC_CHECK_CONDITION, SK_ABORTED_COMMAND, ASC_NONE, ASCQ_NONE);
		} else {
			scsi_execute(lun_bdev, t);
		}
	}

	/* ---- spdk_vhost_scsi_task_cpl ---- */
	c->status = t->status;
	if (t->status != SC_GOOD) {
		memcpy(c->sense, t->sense_data, t->sense_data_len);
		c->sense_len = t->sense_data_len;
	}
	c->resid = t->length - t->data_transferred;
	c->data_transferred = t->data_transferred;
}

/* One request through process_requestq's loop body (vhost_scsi.c:702-739):
 * task_data_setup (490-624) -> spdk_vhost_scsi_task_init_target (361-387) -> process_request
 * (626-653) -> task_submit / early completion / invalid_request -> spdk_vhost_scsi_task_cpl (311-331) */
static void process_one(struct oimorc *o, const struct oimgpu_req *q, const struct oimgpu_iov *iovs,
			struct oimgpu_cpl *c)
{
	struct orc_task t;
	uint32_t cnt = q->iovcnt, len = 0, i, used_len;
	bool from_dev = (q->dir == OIMGPU_DIR_FROM_DEV) || cnt == 0;

	memset(&t, 0, sizeof(t));
	memset(c, 0, sizeof(*c));
	c->tag = q->tag;
	t.cdb = q->cdb;
	t.dxfer_dir = from_dev ? OIMGPU_DIR_FROM_DEV : OIMGPU_DIR_TO_DEV;

	/* ---- task_data_setup ---- */
	if (cnt == 0) {
		/* "TEST UNIT READY command and some others might not contain any payload" (548-560) */
		used_len = OIMGPU_RESP_SIZE;
		t.iovcnt = 1;
		t.iovs[0].base = NULL;
		t.iovs[0].len = 0;
	} else {
		for (i = 0; i < cnt; i++) {
			const struct oimgpu_iov *v = &iovs[q->iov_start + i];
			/* spdk_vhost_vring_desc_to_iov (vhost.c:461-509) with GPA == VA: one iovec per
			 * descriptor; fails at the 130th element or on an untranslatable (0) address */
			if (i >= OIMGPU_IOVS_MAX || v->addr == 0) {
				c->used_len = 0;	/* invalid_request(): used elem only */
				c->resp_valid = 0;
				return;
			}
			t.iovs[i].base = (uint8_t *)(uintptr_t)v->addr;
			t.iovs[i].len = v->len;
			len += v->len;
		}
		t.iovcnt = cnt;
		used_len = from_dev ? OIMGPU_RESP_SIZE + len : OIMGPU_RESP_SIZE;
	}
	t.length = t.transfer_len = len;
	c->used_len = used_len;
	c->resp_valid = 1;
	execute_task(o, &t, q->lun, c);
}

/* ------------------------------------------------------------------------------------------ */

void *oimorc_create(uint64_t num_blocks, uint32_t block_size, int target_num)
{
	struct oimorc *o;

	/* create_malloc_disk (bdev_malloc.c:378-443): zero blocks refused, 2 MiB-aligned zeroed buffer */
	if (num_blocks == 0 || block_size == 0 || target_num < 0 || target_num >= OIMGPU_CTRLR_MAX_DEVS) return NULL;
	o = calloc(1, sizeof(*o));
	if (!o) return NULL;
	if (posix_memalign((void **)&o->bdev.buf, 2 * 1024 * 1024, num_blocks * block_size) != 0) {
		free(o);
		return NULL;
	}
	memset(o->bdev.buf, 0, num_blocks * block_size);
	o->bdev.blockcnt = num_blocks;
	o->bdev.blocklen = block_size;
	snprintf(o->bdev.name, sizeof(o->bdev.name), "Malloc0");
	snprintf(o->bdev.product_name, sizeof(o->bdev.product_name), "Malloc disk");
	snprintf(o->bdev.dev_name, sizeof(o->bdev.dev_name), "Target %d", target_num);
	snprintf(o->bdev.port_name, sizeof(o->bdev.port_name), "vhost");
	o->bdev.protocol_id = 0x06;	/* SAS */
	o->tgt[target_num].bdev = &o->bdev;
	return o;
}

void oimorc_destroy(void *h)
{
	struct oimorc *o = h;
	int t;
	if (!o) return;
	for (t = 0; t < OIMGPU_CTRLR_MAX_DEVS; t++) {
		if (o->extra[t]) { free(o->extra[t]->buf); free(o->extra[t]); }
	}
	free(o->bdev.buf);
	free(o);
}

/* add_vhost_scsi_lun on the same controller (spdk_vhost_scsi_dev_add_tgt, vhost_scsi.c:951-1021):
 * one more SCSI device, with its own Malloc bdev, behind the same request queues */
int oimorc_add_target(void *h, const char *bdev_name, int scsi_dev_id, uint64_t num_blocks, uint32_t block_size, int target_num)
{
	struct oimorc *o = h;
	struct orc_bdev *b;
	if (num_blocks == 0 || block_size == 0 || target_num < 0 || target_num >= OIMGPU_CTRLR_MAX_DEVS) return -22;
	if (o->tgt[target_num].bdev) return -17;
	b = calloc(1, sizeof(*b));
	if (!b || posix_memalign((void **)&b->buf, 2 * 1024 * 1024, num_blocks * block_size) != 0) { free(b); return -12; }
	memset(b->buf, 0, num_blocks * block_size);
	b->blockcnt = num_blocks;
	b->blocklen = block_size;
	snprintf(b->name, sizeof(b->name), "%s", bdev_name ? bdev_name : "Malloc1");
	snprintf(b->product_name, sizeof(b->product_name), "Malloc disk");
	snprintf(b->dev_name, sizeof(b->dev_name), "Target %d", target_num);
	snprintf(b->port_name, sizeof(b->port_name), "vhost");
	b->protocol_id = 0x06;
	b->dev_id = scsi_dev_id;
	o->extra[target_num] = b;
	o->tgt[target_num].bdev = b;
	return 0;
}

uint8_t *oimorc_target_store(void *h, int target_num)
{
	struct oimorc *o = h;
	if (target_num < 0 || target_num >= OIMGPU_CTRLR_MAX_DEVS || !o->tgt[target_num].bdev) return NULL;
	return o->tgt[target_num].bdev->buf;
}

/* the strings / ids INQUIRY reports: bdev name and the global SCSI device id */
void oimorc_set_identity(void *h, const char *bdev_name, int scsi_dev_id)
{
	struct oimorc *o = h;
	snprintf(o->bdev.name, sizeof(o->bdev.name), "%s", bdev_name);
	o->bdev.dev_id = scsi_dev_id;
}

void *oimorc_create_named(const char *bdev_name, uint64_t num_blocks, uint32_t block_size, int target_num)
{
	void *h = oimorc_create(num_blocks, block_size, target_num);
	if (h) oimorc_set_identity(h, bdev_name, 0);
	return h;
}

int oimorc_scsi_dev_id(void *h, int target_num)
{
	struct oimorc *o = h;
	return o->tgt[target_num].bdev ? o->tgt[target_num].bdev->dev_id : -1;
}

uint8_t *oimorc_store(void *h) { return ((struct oimorc *)h)->bdev.buf; }

/* the target's bdev counters, in oimref_iostat's order; -ENODEV: no device in that slot */
int oimorc_iostat(void *h, int target_num, uint64_t out[7])
{
	struct oimorc *o = h;
	if (target_num < 0 || target_num >= OIMGPU_CTRLR_MAX_DEVS || !o->tgt[target_num].bdev) return -ENODEV;
	memcpy(out, o->tgt[target_num].bdev->stat, sizeof(o->tgt[target_num].bdev->stat));
	return 0;
}
uint64_t oimorc_num_blocks(void *h) { return ((struct oimorc *)h)->bdev.blockcnt; }

void oimorc_set_removed(void *h, int target_num, int removed)
{
	((struct oimorc *)h)->tgt[target_num].removed = removed != 0;
}

int oimorc_submit(void *h, const struct oimgpu_req *reqs, uint32_t nreqs,
		  const struct oimgpu_iov *iovs, uint32_t niovs, struct oimgpu_cpl *cpls)
{
	uint32_t i;
	(void)niovs;
	for (i = 0; i < nreqs; i++) process_one(h, &reqs[i], iovs, &cpls[i]);
	return 0;
}

/* spdk_vhost_vring_desc_to_iov (S/lib/vhost/vhost.c:461-509) over a region table
 * {gpa, size, hva} x nregions (rte_vhost_gpa_to_vva, rte_vhost.h:133-150). */
static uint64_t gpa_to_vva(const uint64_t *reg, uint32_t n, uint64_t gpa)
{
	uint32_t i;
	for (i = 0; i < n; i++) {
		if (gpa >= reg[3 * i] && gpa < reg[3 * i] + reg[3 * i + 1]) return gpa - reg[3 * i] + reg[3 * i + 2];
	}
	return 0;
}

int oimorc_desc_to_iov(const uint64_t *regions, uint32_t nregions, uint64_t addr, uint32_t len,
		       struct oimgpu_iov *out, uint32_t start_index)
{
	const uint64_t MB2 = 2ull * 1024 * 1024;
	uint32_t remaining = len, idx = start_index;
	uint64_t payload = addr;

	do {
		uint64_t vva;
		uint32_t to_boundary, l;
		if (idx >= OIMGPU_IOVS_MAX) return -1;
		vva = gpa_to_vva(regions, nregions, payload);
		if (vva == 0) return -1;
		to_boundary = (uint32_t)(MB2 - (payload & (MB2 - 1)));
		if (remaining <= to_boundary) {
			l = remaining;
		} else {
			/* split only where the two sides of a 2 MiB boundary are not VA-contiguous */
			l = to_boundary;
			while (l < remaining) {
				if (vva + l != gpa_to_vva(regions, nregions, payload + l)) break;
				l += (remaining - l) < MB2 ? (remaining - l) : (uint32_t)MB2;
			}
		}
		out[idx - start_index].addr = vva;
		out[idx - start_index].len = l;
		out[idx - start_index].flags = 0;
		remaining -= l;
		payload += l;
		idx++;
	} while (remaining);
	return (int)(idx - start_index);
}

/* ---------------------------------------------------------------------------------------------
 * Virtqueue level: the split-ring walk of the reference's poller, restated.
 * ------------------------------------------------------------------------------------------- */

struct vq_desc { uint64_t addr; uint32_t len; uint16_t flags; uint16_t next; };	/* struct vring_desc */
#define VQ_F_NEXT	1
#define VQ_F_WRITE	2
#define VQ_F_INDIRECT	4

struct vq_ctx {
	const uint64_t *regions;
	uint32_t nregions;
};

/* spdk_vhost_gpa_to_vva (vhost.c:93-106) over rte_vhost_va_from_guest_pa (rte_vhost.h:167-190):
 * the whole [gpa, gpa+len) must sit inside the region that contains gpa */
static void *vq_gpa_to_vva(const struct vq_ctx *m, uint64_t gpa, uint64_t len)
{
	uint32_t i;
	for (i = 0; i < m->nregions; i++) {
		uint64_t g = m->regions[3 * i], sz = m->regions[3 * i + 1], hva = m->regions[3 * i + 2];
		if (gpa >= g && gpa < g + sz) {
			if (len > g + sz - gpa) return NULL;
			return (void *)(uintptr_t)(gpa - g + hva);
		}
	}
	return NULL;
}

/* spdk_vhost_vring_desc_get_next (vhost.c:433-453): 0 ok (possibly *desc == NULL), -1 bad index */
static int vq_desc_get_next(const struct vq_desc **desc, const struct vq_desc *table, uint32_t table_size)
{
	const struct vq_desc *old = *desc;
	if ((old->flags & VQ_F_NEXT) == 0) { *desc = NULL; return 0; }
	if (old->next >= table_size) { *desc = NULL; return -1; }
	*desc = &table[old->next];
	return 0;
}

/* spdk_vhost_vring_desc_to_iov (vhost.c:461-509) appending to the task's SG list */
static int vq_desc_to_iov(const struct vq_ctx *m, struct orc_task *t, uint16_t *iov_index, const struct vq_desc *d)
{
	struct oimgpu_iov out[OIMGPU_IOVS_MAX];
	int n = oimorc_desc_to_iov(m->regions, m->nregions, d->addr, d->len, out, *iov_index), i;
	if (n < 0) return -1;
	for (i = 0; i < n; i++) {
		t->iovs[*iov_index + i].base = (uint8_t *)(uintptr_t)out[i].addr;
		t->iovs[*iov_index + i].len = out[i].len;
	}
	*iov_index += n;
	return 0;
}

/* task_data_setup (vhost_scsi.c:490-624).  Returns 0 and fills t/req/resp/used_len, or -1 (invalid) */
static int vq_task_data_setup(const struct vq_ctx *m, const struct vq_desc *ring, uint32_t ring_size, uint16_t req_idx,
			      struct orc_task *t, const uint8_t **req, uint8_t **resp, uint32_t *used_len)
{
	const struct vq_desc *desc, *table;
	uint32_t table_size, len = 0;
	uint16_t iovcnt = 0;
	int rc;

	/* spdk_vhost_vq_get_desc (vhost.c:219-247) */
	if (req_idx >= ring_size) return -1;
	desc = &ring[req_idx];
	if (desc->flags & VQ_F_INDIRECT) {
		table_size = desc->len / sizeof(*desc);
		table = vq_gpa_to_vva(m, desc->addr, sizeof(*desc) * (uint64_t)table_size);
		desc = table;
		if (desc == NULL) return -1;
	} else {
		table = ring;
		table_size = ring_size;
	}
	/* "First descriptor must be readable" and hold a whole virtio_scsi_cmd_req (51 bytes) */
	if ((desc->flags & VQ_F_WRITE) || desc->len < 51) return -1;
	*req = vq_gpa_to_vva(m, desc->addr, 51);
	if (*req == NULL) return -1;
	vq_desc_get_next(&desc, table, table_size);
	if (desc == NULL) return -1;	/* "contains neither payload nor response buffer" */
	t->dxfer_dir = (desc->flags & VQ_F_WRITE) ? OIMGPU_DIR_FROM_DEV : OIMGPU_DIR_TO_DEV;

	if (t->dxfer_dir == OIMGPU_DIR_FROM_DEV) {
		/* FROM_DEV (READ): [RD_req][WR_resp][WR_buf0]...[WR_bufN] */
		*resp = vq_gpa_to_vva(m, desc->addr, OIMGPU_RESP_SIZE);
		if (desc->len < OIMGPU_RESP_SIZE || *resp == NULL) return -1;
		rc = vq_desc_get_next(&desc, table, table_size);
		if (rc != 0) return -1;
		if (desc == NULL) {
			*used_len = OIMGPU_RESP_SIZE;
			t->iovcnt = 1;
			t->iovs[0].base = NULL;
			t->iovs[0].len = 0;
			t->length = t->transfer_len = 0;
			return 0;
		}
		while (desc) {
			if (!(desc->flags & VQ_F_WRITE)) return -1;
			if (vq_desc_to_iov(m, t, &iovcnt, desc)) return -1;
			len += desc->len;
			rc = vq_desc_get_next(&desc, table, table_size);
			if (rc != 0) return -1;
		}
		*used_len = OIMGPU_RESP_SIZE + len;
	} else {
		/* TO_DEV (WRITE): [RD_req][RD_buf0]...[RD_bufN][WR_resp] */
		while (!(desc->flags & VQ_F_WRITE)) {
			if (vq_desc_to_iov(m, t, &iovcnt, desc)) return -1;
			len += desc->len;
			vq_desc_get_next(&desc, table, table_size);
			if (desc == NULL) return -1;	/* "no response descriptor" */
		}
		*resp = vq_gpa_to_vva(m, desc->addr, OIMGPU_RESP_SIZE);
		if (desc->len < OIMGPU_RESP_SIZE || *resp == NULL) return -1;
		*used_len = OIMGPU_RESP_SIZE;
	}
	t->iovcnt = iovcnt;
	t->length = t->transfer_len = len;
	return 0;
}

/* process_requestq + spdk_vhost_vq_avail_ring_get + spdk_vhost_vq_used_ring_enqueue
 * (vhost_scsi.c:690-741, vhost.c:178-211, 397-431).  Used elements are produced in ring order (the
 * reference's order depends on when its thread polls deferred completions, see ref_driver.c). */
int oimorc_vq_process(void *h, uint64_t desc, uint64_t avail, uint64_t used, uint32_t size,
		      const uint64_t *regions, uint32_t nregions, uint16_t *last_avail_idx, uint16_t *last_used_idx)
{
	struct oimorc *o = h;
	const struct vq_desc *ring = (const struct vq_desc *)(uintptr_t)desc;
	const volatile uint16_t *av = (const volatile uint16_t *)(uintptr_t)avail;	/* flags, idx, ring[] */
	uint8_t *us = (uint8_t *)(uintptr_t)used;					/* flags, idx, {id,len}[] */
	struct vq_ctx m = { regions, nregions };
	uint16_t count = (uint16_t)(av[1] - *last_avail_idx), i;
	int produced = 0;

	if (size == 0 || size > OIMGPU_MAX_VQ_SIZE || (size & (size - 1))) return -EINVAL;
	if (count > size) return 0;	/* broken queue: report nothing (vhost.c:193-198) */
	for (i = 0; i < count; i++) {
		uint16_t head = av[2 + ((*last_avail_idx + i) & (size - 1))];
		struct orc_task t;
		struct oimgpu_cpl c;
		const uint8_t *req = NULL;
		uint8_t *resp = NULL;
		uint32_t used_len = 0, slot;

		memset(&t, 0, sizeof(t));
		memset(&c, 0, sizeof(c));
		if (vq_task_data_setup(&m, ring, size, head, &t, &req, &resp, &used_len) == 0) {
			t.cdb = req + 19;	/* virtio_scsi_cmd_req.cdb */
			c.used_len = used_len;
			execute_task(o, &t, req, &c);
			/* what spdk_vhost_scsi_task_cpl / process_request write into the guest's response */
			resp[11] = c.response;
			if (c.response == OIMGPU_S_OK) {
				resp[10] = c.status;
				if (c.status != SC_GOOD) {
					memcpy(resp + 12, c.sense, c.sense_len);
					memcpy(resp + 0, &c.sense_len, 4);
				}
				memcpy(resp + 4, &c.resid, 4);
			}
		} else {
			used_len = 0;	/* invalid_request(): used element with length 0, nothing else */
		}
		slot = (uint16_t)(*last_used_idx) & (size - 1);
		memcpy(us + 4 + 8 * slot, &(uint32_t){ head }, 4);
		memcpy(us + 4 + 8 * slot + 4, &used_len, 4);
		(*last_used_idx)++;
		__sync_synchronize();
		memcpy(us + 2, last_used_idx, 2);
		produced++;
	}
	*last_avail_idx += count;
	return produced;
}

uint64_t oimorc_busy_ns(void *h, int reset) { (void)h; (void)reset; return 0; }	/* caller times the call */

const char *oimorc_describe(void)
{
	return "port: plain-C restatement of SPDK v19.04-pre vhost-scsi/scsi/bdev/malloc path (oracle/oim_oracle.c)";
}

/* ------------------------------------------------------------------------------------------
 * NBD export: the server side of the kernel's transmission protocol, restating spdk_nbd_poll
 * (S/lib/nbd/nbd.c:560-806: spdk_nbd_io_recv_internal, nbd_submit_bdev_io, nbd_io_done,
 * spdk_nbd_io_xmit_internal) on the restated bdev.  Blocking; one request at a time, which is
 * also the order the reference answers in for a Malloc bdev (completions are immediate).
 * Returns 0 when the peer disconnects (EOF or NBD_CMD_DISC), -EINVAL on a bad request magic.
 * ---------------------------------------------------------------------------------------- */
#include <unistd.h>
#include <sys/socket.h>

static int nbd_read_full(int fd, void *buf, size_t n)
{
	size_t got = 0;
	while (got < n) {
		ssize_t r = read(fd, (char *)buf + got, n - got);
		if (r < 0 && errno == EINTR) continue;
		if (r <= 0) return -1;
		got += (size_t)r;
	}
	return 0;
}

static int nbd_write_full(int fd, const void *buf, size_t n)
{
	size_t put = 0;
	while (put < n) {
		ssize_t r = send(fd, (const char *)buf + put, n - put, MSG_NOSIGNAL);
		if (r < 0 && errno == EINTR) continue;
		if (r <= 0) return -1;
		put += (size_t)r;
	}
	return 0;
}

int oimorc_nbd_serve(void *h, int fd)
{
	struct oimorc *o = h;
	struct orc_bdev *b = &o->bdev;
	uint8_t *payload = NULL;
	size_t cap = 0;
	int rc = 0;

	for (;;) {
		uint8_t req[28], resp[16];	/* struct nbd_request / struct nbd_reply (linux/nbd.h), big endian */
		uint32_t type, len, psize;
		uint64_t from, ob, nb;
		bool ok = false;

		if (nbd_read_full(fd, req, sizeof(req)) != 0) break;
		if (be32(req) != 0x25609513u) { rc = -EINVAL; break; }	/* NBD_REQUEST_MAGIC */
		type = be32(req + 4);
		from = be64(req + 16);
		len = be32(req + 24);
		/* "io except read/write should ignore payload" (nbd.c:607-613) */
		psize = (type == 0 || type == 1) ? len : 0;
		if (psize > cap) {
			free(payload);
			payload = malloc(psize);
			cap = psize;
		}
		if (type == 1 && psize && nbd_read_full(fd, payload, psize) != 0) break;
		if (type == 2) break;	/* NBD_CMD_DISC: soft disconnect, nothing outstanding */
		switch (type) {
		case 0:	/* NBD_CMD_READ -> spdk_bdev_read */
			ok = bdev_bytes_to_blocks(b, from, &ob, len, &nb) == 0 && bdev_valid_blocks(b, ob, nb);
			if (ok && len) memcpy(payload, b->buf + from, len);
			break;
		case 1:	/* NBD_CMD_WRITE -> spdk_bdev_write */
			ok = bdev_bytes_to_blocks(b, from, &ob, len, &nb) == 0 && bdev_valid_blocks(b, ob, nb);
			if (ok && len) memcpy(b->buf + from, payload, len);
			break;
		case 3:	/* NBD_CMD_FLUSH -> spdk_bdev_flush over the whole device */
			ok = true;
			break;
		case 4:	/* NBD_CMD_TRIM -> spdk_bdev_unmap */
			ok = bdev_bytes_to_blocks(b, from, &ob, len, &nb) == 0 && bdev_unmap_blocks(b, ob, nb) == 0;
			break;
		default:	/* rc = -1 -> nbd_io_done(NULL, false, io) */
			break;
		}
		memset(resp, 0, sizeof(resp));
		to_be32(resp, 0x67446698u);		/* NBD_REPLY_MAGIC */
		to_be32(resp + 4, ok ? 0 : EIO);
		memcpy(resp + 8, req + 8, 8);
		if (nbd_write_full(fd, resp, sizeof(resp)) != 0) break;
		if (type == 0 && ok && len && nbd_write_full(fd, payload, len) != 0) break;
	}
	free(payload);
	return rc;
}
