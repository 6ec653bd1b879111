/*
 * bdevio_cases.h — the data-integrity cases of S/test/bdev/bdevio/bdevio.c:388-800, run through SPDK's public bdev
 * API on one open bdev.  Shared by bdevio_oimgpu.c (Malloc on the copy engine) and bdev_oimgpu_driver.c (any bdev).
 */
#ifndef BDEVIO_CASES_H
#define BDEVIO_CASES_H

#include "spdk/stdinc.h"

#include "spdk/bdev.h"
#include "spdk/thread.h"

/* set by the caller before bdevio_run_cases */
extern struct spdk_thread *g_thread;
extern struct spdk_bdev_desc *g_desc;
extern struct spdk_io_channel *g_ch;
extern uint64_t g_size;

/* cases run / failed so far */
extern int g_fail, g_cases;

void bdevio_run_cases(void);

#endif /* BDEVIO_CASES_H */
