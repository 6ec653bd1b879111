/*
 * bdevio_oimgpu.c — the reference's Malloc bdev, UNMODIFIED, with the oimgpu copy engine underneath.
 *
 * Drives the data-integrity cases of S/test/bdev/bdevio/bdevio.c:388-800 (sizes, offsets, patterns, iovec
 * shapes, the out-of-range cases) through SPDK's public bdev API against a bdev made by the reference's own
 * create_malloc_disk(): spdk_bdev_writev/readv/write_zeroes/unmap -> bdev_malloc_* -> spdk_copy_submit ->
 * [the registered engine].  With copy_engine_oimgpu.c linked in, that engine is ours; with
 * OIMGPU_COPY_ENGINE=off it is SPDK's memcpy engine - the same binary then serves as the CPU control run.
 * Prints one JSON line.  Our glue, written against SPDK's public API; it holds no code of the reference.
 */
#include "spdk/stdinc.h"

#include "spdk/bdev.h"
#include "spdk/copy_engine.h"
#include "spdk/env.h"
#include "spdk/log.h"
#include "spdk/thread.h"
#include "spdk_internal/thread.h"

#include "bdev_malloc.h"
#include "bdevio_cases.h"

/* the one env hook SPDK's DPDK-free test env (S/test/common/lib/test_env.c) leaves to the application */
uint32_t spdk_env_get_current_core(void) { return 0; }

int copy_engine_oimgpu_active(void);
void copy_engine_oimgpu_counters(unsigned long long *ops, unsigned long long *bytes);

static void init_done(void *arg, int rc) { *(int *)arg = rc ? -1 : 1; }

int main(int argc, char **argv)
{
	const uint64_t num_blocks = 131072, block_size = 512;	/* 64 MiB: BASELINE config 1 */
	struct spdk_bdev *bdev;
	unsigned long long ops = 0, bytes = 0;
	int done = 0;

	if (!getenv("OIMREF_VERBOSE")) spdk_log_set_print_level(SPDK_LOG_ERROR);
	spdk_thread_lib_init(NULL, 0);
	g_thread = spdk_thread_create("bdevio");
	spdk_set_thread(g_thread);
	spdk_copy_engine_initialize();		/* module_init of every registered engine, ours included */
	spdk_bdev_initialize(init_done, &done);
	while (!done) spdk_thread_poll(g_thread, 0, 0);
	if (done < 0) return 2;
	bdev = create_malloc_disk("Malloc0", NULL, num_blocks, block_size);
	if (!bdev || spdk_bdev_open(bdev, true, NULL, NULL, &g_desc) != 0) return 2;
	g_ch = spdk_bdev_get_io_channel(g_desc);
	g_size = num_blocks * block_size;

	/* the cases of bdevio.c:388-800 */
	bdevio_run_cases();
	copy_engine_oimgpu_counters(&ops, &bytes);
	printf("{\"engine\": \"%s\", \"cases\": %d, \"failed\": %d, \"engine_ops\": %llu, \"engine_bytes\": %llu}\n",
	       copy_engine_oimgpu_active() ? "oimgpu" : "memcpy", g_cases, g_fail, ops, bytes);

	spdk_put_io_channel(g_ch);
	spdk_bdev_close(g_desc);
	while (spdk_thread_poll(g_thread, 0, 0) > 0) {}
	return g_fail ? 1 : 0;
}
