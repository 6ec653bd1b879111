/*
 * bdev_oimgpu_driver.c — the oimgpu bdev module (bdev_oimgpu.c) in the reference's own bdev layer, next to the
 * reference's Malloc bdev, so that every byte and status of the module can be checked against Malloc.
 *
 *   bdev_oimgpu_driver --bdev oimgpu|malloc MODE ...
 *     bdevio                 the bdevio cases (bdevio_cases.c) on a 64 MiB bdev
 *     fuzz SEED [BS] [NT]    a seeded I/O sequence at block size BS on NT SPDK threads (1 or 2), many I/Os outstanding
 *                            per poller tick; prints per-I/O status, a digest per read buffer and one of the whole
 *                            bdev, read back through the bdev API
 *     rpc SOCK               the reference's JSON-RPC server with its bdev RPCs and ours, until SIGTERM/SIGINT
 *     config N:NB:BS:UUID..  creates the bdevs and prints spdk_bdev_subsystem_config_json
 *     perf RW BS QD SECS     bdevperf-style closed loop (RW: randread | randwrite | write) timed with the host clock
 *   OIMGPU_COPY_ENGINE=off gives Malloc the memcpy engine; OIMGPU_CONTROL_ONLY=1 starts the library control-only.
 * Prints one JSON line (config: the JSON array).  Our glue, written against SPDK's public API.
 */
#include "spdk/stdinc.h"

#include <malloc.h>

#include "spdk/bdev.h"
#include "spdk/copy_engine.h"
#include "spdk/env.h"
#include "spdk/json.h"
#include "spdk/log.h"
#include "spdk/rpc.h"
#include "spdk/thread.h"
#include "spdk/uuid.h"
#include "spdk_internal/thread.h"

#include "bdev_malloc.h"
#include "bdev_oimgpu.h"
#include "bdevio_cases.h"
#include "oimgpu.h"

uint32_t spdk_env_get_current_core(void) { return 0; }

int copy_engine_oimgpu_active(void);
void copy_engine_oimgpu_counters(unsigned long long *ops, unsigned long long *bytes);
unsigned long long bdev_oimgpu_launches(void);

static bool g_oimgpu;

static void init_done(void *arg, int rc) { *(int *)arg = rc ? -1 : 1; }

static struct spdk_bdev *create_disk(const char *name, const struct spdk_uuid *uuid, uint64_t nb, uint32_t bs)
{
	return g_oimgpu ? create_oimgpu_disk(name, uuid, nb, bs) : create_malloc_disk(name, uuid, nb, bs);
}

/* host memory for I/O buffers that stays mapped for the life of the process, as SPDK's DMA memory does: the GPU
 * side pins host memory on first use */
static uint8_t *arena_alloc(size_t n)
{
	uint8_t *p = spdk_dma_zmalloc(n, 0x200000, NULL);

	if (!p) abort();
	return p;
}

static uint64_t splitmix(uint64_t *s)
{
	uint64_t z = (*s += 0x9E3779B97F4A7C15ull);

	z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
	z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
	return z ^ (z >> 31);
}

static uint64_t fnv(uint64_t h, const uint8_t *p, size_t n)
{
	size_t i;

	for (i = 0; i < n; i++) h = (h ^ p[i]) * 0x100000001b3ull;
	return h;
}
#define FNV0 0xcbf29ce484222325ull

/* ---- fuzz ---------------------------------------------------------------------------------------------- */

#define FZ_MAX_IOS 64
#define FZ_MAX_IOV 256
#define FZ_ARENA (96u << 20)

struct fz_io {
	int		op;		/* 0 write, 1 read, 2 read without buffer, 3 write zeroes, 4 unmap */
	int		thread;
	uint64_t	off, nb;
	struct iovec	iov[FZ_MAX_IOV];
	int		iovcnt;
	uint64_t	digest;
	char		status;		/* S success, F failed, R rejected at submit */
	bool		done;
};

static struct spdk_thread *g_thr[2];
static struct spdk_io_channel *g_chs[2];
static int g_outstanding;
static uint32_t g_bs;

static void fz_done(struct spdk_bdev_io *bdev_io, bool success, void *arg)
{
	struct fz_io *io = arg;
	struct iovec *iov;
	int iovcnt, i;

	io->status = success ? 'S' : 'F';
	if (success && io->op == 2) {
		spdk_bdev_io_get_iovec(bdev_io, &iov, &iovcnt);
		io->digest = FNV0;
		for (i = 0; i < iovcnt; i++) io->digest = fnv(io->digest, iov[i].iov_base, iov[i].iov_len);
	}
	io->done = true;
	g_outstanding--;
	spdk_bdev_free_io(bdev_io);
}

static void fz_submit(struct fz_io *io)
{
	struct spdk_io_channel *ch = g_chs[io->thread];
	int rc;

	spdk_set_thread(g_thr[io->thread]);
	switch (io->op) {
	case 0: rc = spdk_bdev_writev_blocks(g_desc, ch, io->iov, io->iovcnt, io->off, io->nb, fz_done, io); break;
	case 1: rc = spdk_bdev_readv_blocks(g_desc, ch, io->iov, io->iovcnt, io->off, io->nb, fz_done, io); break;
	case 2: rc = spdk_bdev_read_blocks(g_desc, ch, NULL, io->off, io->nb, fz_done, io); break;
	case 3: rc = spdk_bdev_write_zeroes_blocks(g_desc, ch, io->off, io->nb, fz_done, io); break;
	default: rc = spdk_bdev_unmap_blocks(g_desc, ch, io->off, io->nb, fz_done, io); break;
	}
	if (rc == 0) {
		g_outstanding++;
	} else {
		io->status = 'R';
		io->done = true;
	}
}

static void poll_all(int nthreads)
{
	int t;

	while (g_outstanding > 0) {
		for (t = 0; t < nthreads; t++) spdk_thread_poll(g_thr[t], 0, 0);
	}
}

/* byte-granular iovecs over [p, p + len): up to `pieces` cuts at random byte positions */
static int fz_iovs(struct iovec *iov, uint8_t *p, uint64_t len, int pieces, uint64_t *rng)
{
	uint64_t cut[FZ_MAX_IOV + 1];
	int n = 1, i, j;

	cut[0] = 0;
	for (i = 1; i < pieces && len > 1; i++) cut[n++] = 1 + splitmix(rng) % (len - 1);
	cut[n] = len;
	for (i = 1; i < n; i++) {	/* insertion sort; duplicates give empty elements, which are fine */
		uint64_t v = cut[i];

		for (j = i; j > 0 && cut[j - 1] > v; j--) cut[j] = cut[j - 1];
		cut[j] = v;
	}
	for (i = 0; i < n; i++) {
		iov[i].iov_base = p + cut[i];
		iov[i].iov_len = cut[i + 1] - cut[i];
	}
	return n;
}

static int run_fuzz(uint64_t seed, uint32_t bs, int nthreads)
{
	const uint64_t dev_bytes = 48ull << 20, nb = dev_bytes / bs;
	/* windows: thread t writes only in [win[t], win[t] + wlen); with two threads, [win[2], nb) is read-only shared */
	const uint64_t wlen = nthreads == 1 ? nb : nb / 3;
	uint64_t win[3] = {0, wlen, 2 * wlen};
	uint64_t rng = seed * 0x2545F4914F6CDD1Dull + 1;
	static struct fz_io ios[FZ_MAX_IOS];
	uint8_t *arena = arena_alloc(FZ_ARENA), *p;
	struct spdk_bdev *bdev;
	char *status;
	uint64_t *reads, dev;
	int nstatus = 0, nreads = 0, round, i, t, nrounds = 40;
	uint64_t arena_used;

	status = calloc(FZ_MAX_IOS * (nrounds + 2), 1);
	reads = calloc(FZ_MAX_IOS * (nrounds + 2), sizeof(*reads));
	g_bs = bs;
	bdev = create_disk("Fuzz0", NULL, nb, bs);
	if (!bdev || spdk_bdev_open(bdev, true, NULL, NULL, &g_desc) != 0) return 2;
	for (t = 0; t < nthreads; t++) {
		spdk_set_thread(g_thr[t]);
		g_chs[t] = spdk_bdev_get_io_channel(g_desc);
		if (!g_chs[t]) return 2;
	}
	for (round = 0; round <= nrounds; round++) {
		/* round 0 fills the device (and the shared window) with data; the last round is the 8 MiB pair */
		const bool big = round == nrounds;
		const int n = round == 0 ? 1 : big ? 2 : 16 + (int)(splitmix(&rng) % 33);

		arena_used = 0;
		for (i = 0; i < n; i++) {
			struct fz_io *io = &ios[i];
			uint64_t len, misalign, k;
			int pick, pieces;

			memset(io, 0, sizeof(*io));
			io->thread = nthreads == 1 ? 0 : (int)(splitmix(&rng) % nthreads);
			pick = (int)(splitmix(&rng) % 100);
			if (round == 0) {
				io->op = 0; io->thread = 0; io->off = 0; io->nb = nb;
			} else if (big) {
				io->op = i == 0 ? 0 : 1;
				io->nb = (8u << 20) / bs;
				io->off = win[io->thread] + (i == 0 ? 0 : io->nb / 3);
			} else {
				io->op = pick < 36 ? 0 : pick < 72 ? 1 : pick < 82 ? 2 : pick < 91 ? 3 : 4;
				io->nb = 1 + splitmix(&rng) % (pick & 1 ? 8 : 64);
				if (io->op == 2 && io->nb * bs > 32768) io->nb = 32768 / bs;	/* a buffer from the bdev layer's pool */
				/* a small hot window half of the time: overlapping writes, reads after writes in one batch */
				if (nthreads == 2 && (io->op == 1 || io->op == 2) && splitmix(&rng) % 3 == 0) {
					const uint64_t span = nb - win[2] - io->nb;

					io->off = win[2] + (splitmix(&rng) & 1 ? splitmix(&rng) % 32 : splitmix(&rng) % span);
				} else {
					const uint64_t span = wlen - io->nb;

					io->off = win[io->thread] + (splitmix(&rng) & 1 ? splitmix(&rng) % 32 : splitmix(&rng) % span);
				}
				if (splitmix(&rng) % 25 == 0) io->off = nb - io->nb / 2;	/* out of range */
				/* Malloc's read without a buffer hands out a pointer into its store, which later writes of the
				 * round would change under the reader: such a range is only read for the rest of the round */
				for (k = 0; k < (uint64_t)i && io->op != 1 && io->op != 2; k++) {
					if (ios[k].op == 2 && io->off < ios[k].off + ios[k].nb && ios[k].off < io->off + io->nb) io->op = 1;
				}
			}
			len = io->nb * bs;
			if (io->op <= 1) {
				misalign = splitmix(&rng) % 16;
				arena_used = (arena_used + 63) & ~63ull;
				p = arena + arena_used + misalign;
				arena_used += misalign + len + 64;
				if (arena_used > FZ_ARENA) abort();
				if (io->op == 0) {
					for (k = 0; k < len; k++) p[k] = (uint8_t)splitmix(&rng);
				} else {
					memset(p, 0xEE, len);
				}
				pieces = big ? (i == 0 ? 200 : 150) : 1 + (int)(splitmix(&rng) % 8);
				io->iovcnt = fz_iovs(io->iov, p, len, pieces, &rng);
				/* now and then an iovec list that holds fewer bytes than the I/O */
				if (!big && round > 0 && io->iov[io->iovcnt - 1].iov_len && splitmix(&rng) % 20 == 0)
					io->iov[io->iovcnt - 1].iov_len -= 1 + splitmix(&rng) % io->iov[io->iovcnt - 1].iov_len;
			}
		}
		for (i = 0; i < n; i++) fz_submit(&ios[i]);
		poll_all(nthreads);
		for (i = 0; i < n; i++) {
			struct fz_io *io = &ios[i];

			status[nstatus++] = io->status;
			if (io->op == 1 && io->status == 'S') {
				io->digest = FNV0;
				for (t = 0; t < io->iovcnt; t++) io->digest = fnv(io->digest, io->iov[t].iov_base, io->iov[t].iov_len);
			}
			if ((io->op == 1 || io->op == 2) && io->status == 'S') reads[nreads++] = io->digest;
		}
	}
	/* the whole device, read back through the bdev API */
	{
		struct fz_io *io = &ios[0];
		uint64_t chunk = (4u << 20) / bs, off;

		dev = FNV0;
		for (off = 0; off < nb; off += chunk) {
			memset(io, 0, sizeof(*io));
			io->op = 1;
			io->off = off;
			io->nb = nb - off < chunk ? nb - off : chunk;
			io->iov[0].iov_base = arena;
			io->iov[0].iov_len = io->nb * bs;
			io->iovcnt = 1;
			fz_submit(io);
			poll_all(nthreads);
			if (io->status != 'S') return 3;
			dev = fnv(dev, arena, io->nb * bs);
		}
	}
	printf("{\"bdev\": \"%s\", \"seed\": %llu, \"block_size\": %u, \"threads\": %d, \"status\": \"%.*s\", \"reads\": [",
	       g_oimgpu ? "oimgpu" : "malloc", (unsigned long long)seed, bs, nthreads, nstatus, status);
	for (i = 0; i < nreads; i++) printf("%s\"%016llx\"", i ? ", " : "", (unsigned long long)reads[i]);
	{
		unsigned long long ops = 0, bytes = 0;

		copy_engine_oimgpu_counters(&ops, &bytes);
		printf("], \"device\": \"%016llx\", \"launches\": %llu, \"engine_ops\": %llu}\n", (unsigned long long)dev,
		       bdev_oimgpu_launches(), ops);
	}
	for (t = 0; t < nthreads; t++) {
		spdk_set_thread(g_thr[t]);
		spdk_put_io_channel(g_chs[t]);
		spdk_thread_poll(g_thr[t], 0, 0);
	}
	spdk_set_thread(g_thr[0]);
	spdk_bdev_close(g_desc);
	return 0;
}

/* ---- perf ---------------------------------------------------------------------------------------------- */

struct pf_slot { uint8_t *buf; };
static uint64_t g_pf_done, g_pf_next, g_pf_nb, g_pf_ioblocks, g_pf_rng;
static int g_pf_write, g_pf_random, g_pf_stop, g_pf_inflight;

static void pf_submit(struct pf_slot *s);

static void pf_done(struct spdk_bdev_io *bdev_io, bool success, void *arg)
{
	spdk_bdev_free_io(bdev_io);
	g_pf_inflight--;
	if (!success) abort();
	g_pf_done++;
	if (!g_pf_stop) pf_submit(arg);
}

static void pf_submit(struct pf_slot *s)
{
	const uint64_t slots = g_pf_nb / g_pf_ioblocks;
	uint64_t off;
	int rc;

	if (g_pf_random) {
		off = (splitmix(&g_pf_rng) % slots) * g_pf_ioblocks;
	} else {
		off = (g_pf_next++ % slots) * g_pf_ioblocks;
	}
	rc = g_pf_write ? spdk_bdev_write_blocks(g_desc, g_ch, s->buf, off, g_pf_ioblocks, pf_done, s)
			: spdk_bdev_read_blocks(g_desc, g_ch, s->buf, off, g_pf_ioblocks, pf_done, s);
	if (rc) abort();
	g_pf_inflight++;
}

static double now_s(void)
{
	struct timespec ts;

	clock_gettime(CLOCK_MONOTONIC, &ts);
	return ts.tv_sec + ts.tv_nsec * 1e-9;
}

static int run_perf(const char *rw, uint32_t io_bytes, int qd, double secs)
{
	const uint32_t bs = 512;
	const uint64_t nb = (1ull << 30) / bs;
	struct pf_slot *slots = calloc(qd, sizeof(*slots));
	uint8_t *arena = arena_alloc((size_t)qd * io_bytes);
	struct spdk_bdev *bdev;
	double t0, t1;
	uint64_t done0;
	int i;

	g_pf_write = strcmp(rw, "randread") != 0;
	g_pf_random = strcmp(rw, "write") != 0;
	g_pf_nb = nb;
	g_pf_ioblocks = io_bytes / bs;
	g_pf_rng = 42;
	bdev = create_disk("Perf0", NULL, nb, bs);
	if (!bdev || spdk_bdev_open(bdev, true, NULL, NULL, &g_desc) != 0) return 2;
	g_ch = spdk_bdev_get_io_channel(g_desc);
	if (!g_ch) return 2;
	for (i = 0; i < qd; i++) {
		slots[i].buf = arena + (size_t)i * io_bytes;
		memset(slots[i].buf, i, io_bytes);
	}
	/* warm-up: one second, so pinning and first launches are outside the timed window */
	for (i = 0; i < qd; i++) pf_submit(&slots[i]);
	t0 = now_s();
	while (now_s() - t0 < 1.0) spdk_thread_poll(g_thread, 0, 0);
	done0 = g_pf_done;
	t0 = now_s();
	do {
		spdk_thread_poll(g_thread, 0, 0);
		t1 = now_s();
	} while (t1 - t0 < secs);
	{
		const uint64_t n = g_pf_done - done0;

		g_pf_stop = 1;
		while (g_pf_inflight) spdk_thread_poll(g_thread, 0, 0);
		printf("{\"bdev\": \"%s\", \"engine\": \"%s\", \"rw\": \"%s\", \"io_bytes\": %u, \"qd\": %d, \"seconds\": %.3f, "
		       "\"ios\": %llu, \"iops\": %.1f, \"gbps\": %.4f, \"launches\": %llu}\n",
		       g_oimgpu ? "oimgpu" : "malloc", copy_engine_oimgpu_active() ? "oimgpu" : "memcpy", rw, io_bytes, qd,
		       t1 - t0, (unsigned long long)n, n / (t1 - t0), n * (double)io_bytes / (t1 - t0) / 1e9,
		       bdev_oimgpu_launches());
	}
	spdk_put_io_channel(g_ch);
	spdk_bdev_close(g_desc);
	return 0;
}

/* ---- rpc / config ------------------------------------------------------------------------------------------ */

static volatile sig_atomic_t g_stop;
static void on_signal(int sig) { g_stop = 1; }

static int run_rpc(const char *sock)
{
	signal(SIGTERM, on_signal);
	signal(SIGINT, on_signal);
	if (spdk_rpc_listen(sock) != 0) return 3;
	spdk_rpc_set_state(SPDK_RPC_RUNTIME);
	printf("{\"listening\": \"%s\"}\n", sock);
	fflush(stdout);
	while (!g_stop) {
		spdk_rpc_accept();
		spdk_thread_poll(g_thread, 0, 0);
		usleep(200);
	}
	spdk_rpc_close();
	return 0;
}

static int write_stdout(void *ctx, const void *data, size_t size)
{
	return fwrite(data, 1, size, stdout) == size ? 0 : -1;
}

static int run_config(int argc, char **argv)
{
	struct spdk_json_write_ctx *w;
	int i;

	for (i = 0; i < argc; i++) {
		char name[64], uuid_s[64] = "";
		unsigned long long nb;
		unsigned bs;
		struct spdk_uuid uuid;

		if (sscanf(argv[i], "%63[^:]:%llu:%u:%63s", name, &nb, &bs, uuid_s) < 3) return 2;
		if (uuid_s[0] && spdk_uuid_parse(&uuid, uuid_s) != 0) return 2;
		if (!create_disk(name, uuid_s[0] ? &uuid : NULL, nb, bs)) return 2;
	}
	w = spdk_json_write_begin(write_stdout, NULL, 0);
	spdk_bdev_subsystem_config_json(w);
	spdk_json_write_end(w);
	printf("\n");
	return 0;
}

int main(int argc, char **argv)
{
	const char *mode;
	int done = 0, rc = 2, nthreads = 1, t;

	if (argc < 4 || strcmp(argv[1], "--bdev") != 0) {
		fprintf(stderr, "usage: %s --bdev oimgpu|malloc bdevio|fuzz|rpc|config|perf ...\n", argv[0]);
		return 2;
	}
	g_oimgpu = strcmp(argv[2], "oimgpu") == 0;
	mode = argv[3];
	/* SPDK's DMA memory (hugepages) stays mapped for the life of the process, and the GPU side relies on that: host
	 * memory is pinned on first use.  The DPDK-free test env under this driver hands out the bdev layer's buffers
	 * with malloc/free; keep freed memory mapped too (no mmap'ed chunks, no heap trimming) */
	mallopt(M_MMAP_MAX, 0);
	mallopt(M_TRIM_THRESHOLD, INT_MAX);
	if (strcmp(mode, "fuzz") == 0 && argc > 6) nthreads = atoi(argv[6]) == 2 ? 2 : 1;
	if (!getenv("OIMREF_VERBOSE")) spdk_log_set_print_level(SPDK_LOG_ERROR);
	if (getenv("OIMGPU_CONTROL_ONLY") && oimgpu_init_control_only() != 0) return 2;
	spdk_thread_lib_init(NULL, 0);
	for (t = 0; t < nthreads; t++) g_thr[t] = spdk_thread_create(t ? "fuzz1" : "main");
	g_thread = g_thr[0];
	spdk_set_thread(g_thread);
	spdk_copy_engine_initialize();
	spdk_bdev_initialize(init_done, &done);
	while (!done) spdk_thread_poll(g_thread, 0, 0);
	if (done < 0) return 2;

	if (strcmp(mode, "bdevio") == 0) {
		const uint64_t num_blocks = 131072, block_size = 512;
		struct spdk_bdev *bdev = create_disk("Bdevio0", NULL, num_blocks, block_size);
		unsigned long long ops = 0, bytes = 0;

		if (!bdev || spdk_bdev_open(bdev, true, NULL, NULL, &g_desc) != 0) return 2;
		g_ch = spdk_bdev_get_io_channel(g_desc);
		if (!g_ch) return 2;
		g_size = num_blocks * block_size;
		bdevio_run_cases();
		copy_engine_oimgpu_counters(&ops, &bytes);
		printf("{\"bdev\": \"%s\", \"cases\": %d, \"failed\": %d, \"launches\": %llu, \"engine_ops\": %llu}\n",
		       g_oimgpu ? "oimgpu" : "malloc", g_cases, g_fail, bdev_oimgpu_launches(), ops);
		spdk_put_io_channel(g_ch);
		spdk_bdev_close(g_desc);
		rc = g_fail ? 1 : 0;
	} else if (strcmp(mode, "fuzz") == 0 && argc > 4) {
		rc = run_fuzz(strtoull(argv[4], NULL, 0), argc > 5 ? (uint32_t)atoi(argv[5]) : 512, nthreads);
	} else if (strcmp(mode, "rpc") == 0 && argc > 4) {
		rc = run_rpc(argv[4]);
	} else if (strcmp(mode, "config") == 0) {
		rc = run_config(argc - 4, argv + 4);
	} else if (strcmp(mode, "perf") == 0 && argc > 7) {
		rc = run_perf(argv[4], (uint32_t)atoi(argv[5]), atoi(argv[6]), atof(argv[7]));
	}
	fflush(stdout);
	for (t = 0; t < nthreads; t++) {
		while (spdk_thread_poll(g_thr[t], 0, 0) > 0) {}
	}
	return rc;
}
