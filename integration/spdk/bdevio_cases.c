/*
 * bdevio_cases.c — the data-integrity cases of S/test/bdev/bdevio/bdevio.c:388-800 (sizes, offsets, patterns, iovec
 * shapes, the out-of-range cases) through SPDK's public bdev API: spdk_bdev_writev/readv/write_zeroes/unmap on the
 * bdev the caller opened.  Our glue, written against SPDK's public API; it holds no code of the reference.
 */
#include "bdevio_cases.h"

#include "spdk/env.h"

struct spdk_thread *g_thread;
struct spdk_bdev_desc *g_desc;
struct spdk_io_channel *g_ch;
uint64_t g_size;

struct io_wait { int done; bool ok; };

static void io_done(struct spdk_bdev_io *bdev_io, bool success, void *cb_arg)
{
	struct io_wait *w = cb_arg;

	w->ok = success;
	w->done = 1;
	spdk_bdev_free_io(bdev_io);
}

static int wait_io(int rc, struct io_wait *w)
{
	if (rc != 0) return rc;		/* rejected at submit (bdev layer: -EINVAL and friends) */
	while (!w->done) spdk_thread_poll(g_thread, 0, 0);
	return w->ok ? 0 : -EIO;
}

enum { OP_WRITE, OP_READ, OP_ZEROES, OP_UNMAP };

static int do_io(int op, struct iovec *iov, int iovcnt, uint64_t offset, uint64_t len)
{
	struct io_wait w = {0, false};

	switch (op) {
	case OP_WRITE: return wait_io(spdk_bdev_writev(g_desc, g_ch, iov, iovcnt, offset, len, io_done, &w), &w);
	case OP_READ: return wait_io(spdk_bdev_readv(g_desc, g_ch, iov, iovcnt, offset, len, io_done, &w), &w);
	case OP_ZEROES: return wait_io(spdk_bdev_write_zeroes(g_desc, g_ch, offset, len, io_done, &w), &w);
	default: return wait_io(spdk_bdev_unmap(g_desc, g_ch, offset, len, io_done, &w), &w);
	}
}

/* split `len` bytes at `base` into iovecs of `piece` bytes (0: one iovec) */
static int make_iov(struct iovec *iov, uint8_t *base, uint64_t len, uint64_t piece)
{
	int n = 0;
	uint64_t off = 0;

	if (piece == 0) piece = len;
	while (off < len) {
		iov[n].iov_base = base + off;
		iov[n].iov_len = len - off < piece ? len - off : piece;
		off += iov[n].iov_len;
		n++;
	}
	return n;
}

int g_fail, g_cases;

static void check(const char *what, bool ok)
{
	g_cases++;
	if (!ok) {
		g_fail++;
		fprintf(stderr, "bdevio_oimgpu: FAILED %s\n", what);
	}
}

/* I/O buffers come from one arena that stays mapped for the life of the process, as SPDK's DMA memory does (hugepages
 * handed out by spdk_dma_malloc are never returned to the kernel): the engine pins host memory for the GPU on first
 * use, and a buffer that free() unmaps and a later malloc() maps again at the same address would leave that pinning
 * pointing at the old pages.  (The DPDK-free test env under this driver is plain posix_memalign/free.) */
static uint8_t *g_arena;
static size_t g_arena_used;
#define ARENA_BYTES (32u << 20)

static uint8_t *arena_get(size_t n)
{
	uint8_t *p;

	if (!g_arena) g_arena = spdk_dma_zmalloc(ARENA_BYTES, 0x200000, NULL);
	g_arena_used = (g_arena_used + 0xfff) & ~(size_t)0xfff;
	if (g_arena_used + n > ARENA_BYTES) abort();
	p = g_arena + g_arena_used;
	g_arena_used += n;
	return p;
}

static void arena_reset(void) { g_arena_used = 0; }

/* blockdev_write_read (bdevio.c:320-386): write the pattern (or write zeroes), read back, compare */
static void write_read(const char *name, uint64_t len, uint64_t piece, int pattern, uint64_t offset, int expected_rc, int zeroes,
		       unsigned misalign)
{
	struct iovec iov[160];
	uint8_t *tx, *rx;
	int rc, n;
	bool same = true;

	arena_reset();
	tx = arena_get(len + 64);
	rx = arena_get(len + 64);
	memset(tx + misalign, pattern, len);
	memset(rx, 0x5a, len + 64);
	if (zeroes) {
		rc = do_io(OP_ZEROES, NULL, 0, offset, len);
		memset(tx + misalign, 0, len);
	} else {
		n = make_iov(iov, tx + misalign, len, piece);
		rc = do_io(OP_WRITE, iov, n, offset, len);
	}
	if (expected_rc == 0) {
		check(name, rc == 0);
		n = make_iov(iov, rx + misalign, len, piece);
		rc = do_io(OP_READ, iov, n, offset, len);
		check(name, rc == 0);
		same = memcmp(tx + misalign, rx + misalign, len) == 0 && rx[misalign + len] == 0x5a && (misalign == 0 || rx[misalign - 1] == 0x5a);
		check(name, same);
	} else {
		check(name, rc != 0);
	}
}

void bdevio_run_cases(void)
{
	uint8_t *buf;
	struct iovec iov[4];

	write_read("write_read_4k", 4096, 0, 0xA3, 0, 0, 0, 0);
	write_read("write_zeroes_read_4k", 4096, 0, 0xA3, 0, 0, 1, 0);
	write_read("write_zeroes_read_1m", 1048576, 0, 0xA3, 0, 0, 1, 0);
	write_read("write_zeroes_read_3m", 3145728, 0, 0xA3, 0, 0, 1, 0);
	write_read("write_zeroes_read_3m_500k", 3670016, 0, 0xA3, 0, 0, 1, 0);
	write_read("writev_readv_4k", 4096, 4096, 0xA3, 0, 0, 0, 0);
	write_read("writev_readv_30x4k", 4096 * 30, 4096, 0xA3, 0, 0, 0, 0);
	write_read("write_read_512Bytes", 512, 0, 0xA3, 8192, 0, 0, 0);
	write_read("writev_readv_512Bytes", 512, 512, 0xA3, 8192, 0, 0, 0);
	write_read("write_read_size_gt_128k", 135168, 0, 0xA3, 8192, 0, 0, 0);
	write_read("writev_readv_size_gt_128k", 135168, 0, 0xA3, 8192, 0, 0, 0);
	write_read("writev_readv_size_gt_128k_two_iov", 135168, 131072, 0xA3, 8192, 0, 0, 0);
	write_read("write_read_invalid_size", 0x1234, 0, 0xA3, 8192, -1, 0, 0);		/* not a multiple of the block size */
	write_read("write_read_offset_plus_nbytes_equals_bdev_size", 1024, 0, 0xA3, g_size - 1024, 0, 0, 0);
	write_read("write_read_offset_plus_nbytes_gt_bdev_size", 4096, 0, 0xA3, g_size - 1024, -1, 0, 0);
	write_read("write_read_max_offset", 4096, 0, 0xA3, UINT64_MAX - 4095, -1, 0, 0);
	write_read("overlapped_write_read_8k_a", 8192, 0, 0xA3, 0, 0, 0, 0);
	write_read("overlapped_write_read_8k_b", 8192, 0, 0xBB, 4096, 0, 0, 0);
	/* SURVEY 8(d) C3: byte-granular iovecs (the engine sees src/dst that are not 16-byte aligned) */
	write_read("writev_readv_ragged_iovecs", 131072, 4097, 0x6C, 65536, 0, 0, 0);
	write_read("writev_readv_misaligned_buffers", 131072, 0, 0x3D, 1048576, 0, 0, 3);

	/* unmap = fill 0x00 over the range (bdev_malloc_unmap, bdev_malloc.c:222-233), neighbours untouched */
	arena_reset();
	buf = arena_get(3 * 65536);
	memset(buf, 0x77, 3 * 65536);
	iov[0].iov_base = buf; iov[0].iov_len = 3 * 65536;
	check("unmap: prefill", do_io(OP_WRITE, iov, 1, 2097152, 3 * 65536) == 0);
	check("unmap", do_io(OP_UNMAP, NULL, 0, 2097152 + 65536, 65536) == 0);
	memset(buf, 0x11, 3 * 65536);
	check("unmap: read back", do_io(OP_READ, iov, 1, 2097152, 3 * 65536) == 0);
	{
		bool ok = true;
		uint64_t i;

		for (i = 0; i < 3 * 65536; i++) ok &= buf[i] == ((i >= 65536 && i < 2 * 65536) ? 0x00 : 0x77);
		check("unmap: contents", ok);
	}
}
