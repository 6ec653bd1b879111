/*
 * ref_driver.c — TEST INFRASTRUCTURE.  Glue that drives the REFERENCE's own C implementation of
 * the hot path (compiled from /root/reference by oracle/Makefile into oracle/_ref/liboim_ref.so)
 * with the same request/completion structures the product's C ABI uses (include/oimgpu.h).
 *
 * Nothing here re-implements the path: every request is turned into a real virtio split-ring
 * descriptor chain in (identity-mapped) "guest memory" and handed to the reference's
 * process_requestq() (S/lib/vhost/vhost_scsi.c:690-741), which runs task_data_setup ->
 * spdk_scsi_dev_queue_task -> spdk_bdev_scsi_execute -> spdk_bdev_readv/writev ->
 * bdev_malloc_readv/writev -> mem_copy_submit (memcpy) -> spdk_vhost_scsi_task_cpl ->
 * spdk_vhost_vq_used_ring_enqueue, exactly as the vhost poller would.  We then read the used ring
 * and the response buffers back.  vhost_scsi.c is #included (as SPDK's own unit tests include
 * the .c under test) because process_requestq() is static.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's CPU legs may load this library.
 */
#include "vhost/vhost_scsi.c"

#include "spdk/bdev.h"
#include "spdk/bdev_module.h"
#include "spdk/copy_engine.h"
#include "bdev_malloc.h"
#include "spdk/rpc.h"
#include "oimgpu.h"

/* ------------------------------------------------------------------------------------------
 * Stubs for the vhost-user transport and the event framework, which the data path never calls
 * once a session is running (same set SPDK's vhost_ut.c stubs out).
 * ---------------------------------------------------------------------------------------- */
#ifndef OIMREF_REAL_VHOST
int rte_vhost_driver_callback_register(const char *p, struct vhost_device_ops const *const o) { return 0; }
int rte_vhost_driver_disable_features(const char *p, uint64_t f) { return 0; }
int rte_vhost_driver_set_features(const char *p, uint64_t f) { return 0; }
int rte_vhost_driver_register(const char *p, uint64_t f) { return 0; }
int rte_vhost_driver_unregister(const char *p) { return 0; }
int rte_vhost_driver_start(const char *p) { return 0; }
int rte_vhost_enable_guest_notification(int vid, uint16_t q, int e) { return 0; }
int rte_vhost_get_ifname(int vid, char *buf, size_t len) { if (len) buf[0] = 0; return 0; }
int rte_vhost_get_mem_table(int vid, struct rte_vhost_memory **mem) { return -1; }
int rte_vhost_get_negotiated_features(int vid, uint64_t *f) { *f = 0; return 0; }
int rte_vhost_get_vhost_vring(int vid, uint16_t idx, struct rte_vhost_vring *v) { return -1; }
void rte_vhost_log_used_vring(int vid, uint16_t idx, uint64_t off, uint64_t len) {}
void rte_vhost_log_write(int vid, uint64_t addr, uint64_t len) {}
int rte_vhost_set_vhost_vring_last_idx(int vid, uint16_t i, uint16_t a, uint16_t u) { return 0; }
#else
/* liboim_ref_vhost.so: the reference's own vhost-user transport (S/lib/vhost/rte_vhost/{socket,vhost_user,
 * vhost,fd_man}.c) is linked instead of the stubs above; what it needs from DPDK is a logger, an
 * allocator and an address translation, provided here. */
#include <stdarg.h>
int rte_log(uint32_t level, uint32_t logtype, const char *fmt, ...)
{
	va_list ap;
	if (!getenv("OIMREF_VERBOSE")) return 0;
	va_start(ap, fmt);
	vfprintf(stderr, fmt, ap);
	va_end(ap);
	return 0;
}
static void *ref_alloc(size_t size, unsigned align, int zero)
{
	void *p = NULL;
	if (posix_memalign(&p, align < 64 ? 64 : align, size ? size : 1) != 0) return NULL;
	if (zero) memset(p, 0, size);
	return p;
}
void *rte_malloc(const char *type, size_t size, unsigned align) { return ref_alloc(size, align, 0); }
void *rte_zmalloc(const char *type, size_t size, unsigned align) { return ref_alloc(size, align, 1); }
void *rte_malloc_socket(const char *type, size_t size, unsigned align, int socket) { return ref_alloc(size, align, 0); }
void *rte_zmalloc_socket(const char *type, size_t size, unsigned align, int socket) { return ref_alloc(size, align, 1); }
void rte_free(void *p) { free(p); }
uint64_t rte_mem_virt2phy(const void *virt) { return (uint64_t)(uintptr_t)virt; }
void rte_pktmbuf_free(void *m) {}
#endif
int spdk_vhost_nvme_admin_passthrough(int vid, void *cmd, void *cqe, void *buf) { return 0; }
int spdk_vhost_nvme_set_cq_call(int vid, uint16_t qid, int fd) { return 0; }
int spdk_vhost_nvme_set_bar_mr(int vid, void *bar, uint64_t sz) { return 0; }
int spdk_vhost_nvme_get_cap(int vid, uint64_t *cap) { return 0; }
int spdk_vhost_nvme_controller_construct(void) { return 0; }
int spdk_vhost_blk_controller_construct(void) { return 0; }
/* vhost-blk / vhost-nvme are never configured by OIM (SURVEY.md 2b): their RPC handlers link but refuse */
int spdk_vhost_blk_construct(const char *n, const char *m, const char *d, bool ro) { return -ENOTSUP; }
int spdk_vhost_nvme_dev_construct(const char *n, const char *m, uint32_t q) { return -ENOTSUP; }
int spdk_vhost_nvme_dev_add_ns(struct spdk_vhost_dev *v, const char *b) { return -ENOTSUP; }
#ifndef OIMREF_REAL_VHOST
struct spdk_event *spdk_event_allocate(uint32_t lcore, spdk_event_fn fn, void *a1, void *a2) { return NULL; }
void spdk_event_call(struct spdk_event *e) {}
static void ref_run_events(void) {}
#else
/* the reactor's event ring, reduced to what the transport needs: the vhost-user thread posts
 * start/stop-session events (spdk_vhost_event_send, vhost.c:927-968), the one polling thread runs them */
struct spdk_event { spdk_event_fn fn; void *a1, *a2; struct spdk_event *next; };
static pthread_mutex_t g_ev_mu = PTHREAD_MUTEX_INITIALIZER;
static struct spdk_event *g_ev_head, **g_ev_tail = &g_ev_head;
struct spdk_event *spdk_event_allocate(uint32_t lcore, spdk_event_fn fn, void *a1, void *a2)
{
	struct spdk_event *e = calloc(1, sizeof(*e));
	e->fn = fn; e->a1 = a1; e->a2 = a2;
	return e;
}
void spdk_event_call(struct spdk_event *e)
{
	pthread_mutex_lock(&g_ev_mu);
	*g_ev_tail = e;
	g_ev_tail = &e->next;
	pthread_mutex_unlock(&g_ev_mu);
}
static void ref_run_events(void)
{
	for (;;) {
		struct spdk_event *e;
		pthread_mutex_lock(&g_ev_mu);
		e = g_ev_head;
		if (e) {
			g_ev_head = e->next;
			if (!g_ev_head) g_ev_tail = &g_ev_head;
		}
		pthread_mutex_unlock(&g_ev_mu);
		if (!e) return;
		e->fn(e->a1, e->a2);
		free(e);
	}
}
#endif
int spdk_mem_register(void *vaddr, size_t len) { return 0; }
int spdk_mem_unregister(void *vaddr, size_t len) { return 0; }
void *spdk_call_unaffinitized(void *cb(void *arg), void *arg) { return cb(arg); }
uint32_t spdk_env_get_current_core(void) { return 0; }
uint32_t spdk_env_get_first_core(void) { return 0; }
uint32_t spdk_env_get_last_core(void) { return 0; }
uint32_t spdk_env_get_next_core(uint32_t c) { return UINT32_MAX; }

static struct spdk_cpuset *g_core_mask;
struct spdk_cpuset *spdk_app_get_core_mask(void)
{
	if (!g_core_mask) {
		g_core_mask = spdk_cpuset_alloc();
		spdk_cpuset_set_cpu(g_core_mask, 0, true);
	}
	return g_core_mask;
}
int spdk_app_parse_core_mask(const char *mask, struct spdk_cpuset *cpumask)
{
	/* as S/lib/event/app.c and S/test/unit/lib/vhost/vhost.c/vhost_ut.c:58-72: parse, then keep only
	 * the cores of the application mask */
	int ret = spdk_cpuset_parse(cpumask, mask);
	if (ret < 0) return ret;
	spdk_cpuset_and(cpumask, spdk_app_get_core_mask());
	return 0;
}

/* ------------------------------------------------------------------------------------------ */

#define REF_VQ_SIZE	1024

struct oimref {
	struct spdk_bdev		*bdev;
	char				bdev_name[32];
	struct spdk_bdev		*extra[SPDK_VHOST_SCSI_CTRLR_MAX_DEVS];	/* oimref_add_target */
	struct spdk_vhost_scsi_dev	*svdev;
	struct spdk_vhost_scsi_session	*svsession;
	struct spdk_vhost_virtqueue	*vq;		/* request queue (index VIRTIO_SCSI_REQUESTQ) */
	struct rte_vhost_memory		*mem;
	struct vring_desc		*desc;
	struct vring_avail		*avail;
	struct vring_used		*used;
	struct virtio_scsi_cmd_req	*req_bufs;	/* [OIMGPU_REQS_PER_PASS] */
	struct virtio_scsi_cmd_resp	*resp_bufs;	/* [OIMGPU_REQS_PER_PASS] */
	struct vring_desc		*indirect;	/* [OIMGPU_REQS_PER_PASS][REF_INDIRECT_MAX] */
	uint16_t			used_seen;
	uint64_t			poller_ns;	/* time spent inside the reference's poller only */
	int				eventfd;
	struct oimref			*next_on_thread;
};

#define REF_INDIRECT_MAX	(OIMGPU_IOVS_MAX + 8)

static __thread struct spdk_thread *g_thread;
static int g_lib_inited;
static int g_subsys_inited;
static int g_name_seq;

static void init_done(void *arg, int rc) { *(int *)arg = rc ? -1 : 1; }

/* the unit-test environment's tick counter (test_env.c:412-435).  It only moves when we move it: the driver
 * advances it before it polls for completions, so every bdev_io takes at least one tick, as the histogram's
 * tally requires (histogram_data.h:120-135 asserts a non-zero datapoint) */
extern uint64_t ut_spdk_get_ticks;

/* latency histogram on, as enable_bdev_histogram does it (bdev_rpc.c): every bdev_io of the bdev is tallied */
static int ref_histogram_on(struct spdk_bdev *b)
{
	int done = 0;
	spdk_bdev_histogram_enable(b, init_done, &done, true);
	while (!done) spdk_thread_poll(g_thread, 0, 0);
	return done < 0 ? -1 : 0;
}

static int ref_global_init(void)
{
	if (!g_lib_inited) {
		/* malformed requests are part of the tests: keep the reference's ERRLOG lines quiet */
		if (!getenv("OIMREF_VERBOSE")) spdk_log_set_print_level(SPDK_LOG_DISABLED);
		spdk_thread_lib_init(NULL, 0);
		g_lib_inited = 1;
	}
	if (!g_thread) {
		g_thread = spdk_thread_create("oimref");
		if (!g_thread) return -1;
	}
	spdk_set_thread(g_thread);
	if (!g_subsys_inited) {
		int done = 0;
		spdk_copy_engine_initialize();
		spdk_bdev_initialize(init_done, &done);
		while (!done) spdk_thread_poll(g_thread, 0, 0);
		if (done < 0) return -1;
		if (spdk_scsi_init() != 0) return -1;
		g_subsys_inited = 1;
	}
	return 0;
}

static void ref_hotremove_cb(struct spdk_scsi_lun *lun, void *arg) {}

/* Create one Malloc bdev and expose it as "Target <target_num>" LUN 0 of a vhost-scsi session,
 * the state add_vhost_scsi_lun + a connected guest produce (vhost_scsi.c:951-1021, 1236-1292). */
static void *ref_create(const char *bdev_name, uint64_t num_blocks, uint32_t block_size, int target_num);

void *oimref_create(uint64_t num_blocks, uint32_t block_size, int target_num)
{
	return ref_create(NULL, num_blocks, block_size, target_num);
}

/* same with an explicit bdev name (INQUIRY reports it: serial number, NAA and T10 designators) */
void *oimref_create_named(const char *bdev_name, uint64_t num_blocks, uint32_t block_size, int target_num)
{
	return ref_create(bdev_name, num_blocks, block_size, target_num);
}

/* spdk_scsi_dev.id of the target: slot in the process-wide SCSI device table (S/lib/scsi/dev.c:49-66) */
int oimref_scsi_dev_id(void *h, int target_num)
{
	struct oimref *r = h;
	return spdk_scsi_dev_get_id(r->svsession->scsi_dev_state[target_num].dev);
}

static void *ref_create(const char *bdev_name, uint64_t num_blocks, uint32_t block_size, int target_num)
{
	struct oimref *r;
	const char *names[1];
	int lun_ids[1] = { 0 };
	char tname[32];
	struct spdk_scsi_dev *sdev;
	uint16_t i;

	if (target_num < 0 || target_num >= SPDK_VHOST_SCSI_CTRLR_MAX_DEVS) return NULL;
	if (ref_global_init() != 0) return NULL;

	r = calloc(1, sizeof(*r));
	if (bdev_name) snprintf(r->bdev_name, sizeof(r->bdev_name), "%s", bdev_name);
	else snprintf(r->bdev_name, sizeof(r->bdev_name), "RefMalloc%d", __sync_fetch_and_add(&g_name_seq, 1));
	r->bdev = create_malloc_disk(r->bdev_name, NULL, num_blocks, block_size);
	if (!r->bdev) { free(r); return NULL; }
	if (ref_histogram_on(r->bdev) != 0) return NULL;

	posix_memalign((void **)&r->svdev, 64, sizeof(*r->svdev));
	memset(r->svdev, 0, sizeof(*r->svdev));
	r->svdev->vdev.name = strdup("oimref.ctrlr");
	posix_memalign((void **)&r->svsession, 64, sizeof(*r->svsession));
	memset(r->svsession, 0, sizeof(*r->svsession));
	r->svsession->svdev = r->svdev;
	r->svsession->vsession.vdev = &r->svdev->vdev;
	r->svsession->vsession.max_queues = VIRTIO_SCSI_REQUESTQ + 1;
	r->svsession->vsession.negotiated_features = 1ULL << VIRTIO_RING_F_INDIRECT_DESC;

	names[0] = r->bdev_name;
	snprintf(tname, sizeof(tname), "Target %d", target_num);
	sdev = spdk_scsi_dev_construct(tname, names, lun_ids, 1, SPDK_SPC_PROTOCOL_IDENTIFIER_SAS,
				       ref_hotremove_cb, r);
	if (!sdev) return NULL;
	spdk_scsi_dev_add_port(sdev, 0, "vhost");
	if (spdk_scsi_dev_allocate_io_channels(sdev) != 0) return NULL;
	r->svdev->scsi_dev_state[target_num].dev = sdev;
	r->svsession->scsi_dev_state[target_num].dev = sdev;

	/* identity-mapped guest memory: GPA == host VA, one region covering the address space */
	r->mem = calloc(1, sizeof(*r->mem) + sizeof(struct rte_vhost_mem_region));
	r->mem->nregions = 1;
	r->mem->regions[0].guest_phys_addr = 0;
	r->mem->regions[0].host_user_addr = 0;
	r->mem->regions[0].size = UINT64_MAX;
	r->svsession->vsession.mem = r->mem;

	r->desc = calloc(REF_VQ_SIZE, sizeof(struct vring_desc));
	r->avail = calloc(1, sizeof(struct vring_avail) + REF_VQ_SIZE * sizeof(uint16_t) + 8);
	r->used = calloc(1, sizeof(struct vring_used) + REF_VQ_SIZE * sizeof(struct vring_used_elem) + 8);
	r->req_bufs = calloc(OIMGPU_REQS_PER_PASS, sizeof(*r->req_bufs));
	r->resp_bufs = calloc(OIMGPU_REQS_PER_PASS, sizeof(*r->resp_bufs));
	r->indirect = calloc((size_t)OIMGPU_REQS_PER_PASS * REF_INDIRECT_MAX, sizeof(struct vring_desc));
	r->eventfd = eventfd(0, EFD_NONBLOCK);

	r->vq = &r->svsession->vsession.virtqueue[VIRTIO_SCSI_REQUESTQ];
	r->vq->vring.desc = r->desc;
	r->vq->vring.avail = r->avail;
	r->vq->vring.used = r->used;
	r->vq->vring.size = REF_VQ_SIZE;
	r->vq->vring.callfd = r->eventfd;
	r->vq->vring.kickfd = -1;
	/* task pool, as alloc_task_pool() builds it (vhost_scsi.c:1180-1225) */
	r->vq->tasks = calloc(REF_VQ_SIZE, sizeof(struct spdk_vhost_scsi_task));
	for (i = 0; i < REF_VQ_SIZE; i++) {
		struct spdk_vhost_scsi_task *t = &((struct spdk_vhost_scsi_task *)r->vq->tasks)[i];
		t->svsession = r->svsession;
		t->vq = r->vq;
		t->req_idx = i;
	}
	return r;
}

/* add_vhost_scsi_lun on the same controller: one more Malloc bdev + SCSI device in another target
 * slot of the same session (spdk_vhost_scsi_dev_add_tgt, vhost_scsi.c:951-1021, minus the RPC) */
int oimref_add_target(void *h, const char *bdev_name, uint64_t num_blocks, uint32_t block_size, int target_num)
{
	struct oimref *r = h;
	const char *names[1];
	int lun_ids[1] = { 0 };
	char tname[32], auto_name[32];
	struct spdk_scsi_dev *sdev;
	struct spdk_bdev *b;

	if (target_num < 0 || target_num >= SPDK_VHOST_SCSI_CTRLR_MAX_DEVS) return -22;
	if (r->svdev->scsi_dev_state[target_num].dev) return -17;
	spdk_set_thread(g_thread);
	if (!bdev_name) {
		snprintf(auto_name, sizeof(auto_name), "RefMalloc%d", __sync_fetch_and_add(&g_name_seq, 1));
		bdev_name = auto_name;
	}
	b = create_malloc_disk(bdev_name, NULL, num_blocks, block_size);
	if (!b) return -12;
	if (ref_histogram_on(b) != 0) return -12;
	names[0] = spdk_bdev_get_name(b);
	snprintf(tname, sizeof(tname), "Target %d", target_num);
	sdev = spdk_scsi_dev_construct(tname, names, lun_ids, 1, SPDK_SPC_PROTOCOL_IDENTIFIER_SAS, ref_hotremove_cb, r);
	if (!sdev) return -22;
	spdk_scsi_dev_add_port(sdev, 0, "vhost");
	if (spdk_scsi_dev_allocate_io_channels(sdev) != 0) return -12;
	r->svdev->scsi_dev_state[target_num].dev = sdev;
	r->svsession->scsi_dev_state[target_num].dev = sdev;
	r->extra[target_num] = b;
	return 0;
}

uint8_t *oimref_target_store(void *h, int target_num)
{
	struct oimref *r = h;
	struct spdk_bdev *b = r->extra[target_num];
	if (!b) {
		struct spdk_scsi_dev *d = r->svdev->scsi_dev_state[target_num].dev;
		if (!d) return NULL;
		b = r->bdev;
	}
	return *(uint8_t **)((char *)b->ctxt + sizeof(struct spdk_bdev));
}

uint8_t *oimref_store(void *h)
{
	struct oimref *r = h;
	/* struct malloc_disk { struct spdk_bdev disk; void *malloc_buf; ... } (bdev_malloc.c:50-54):
	 * the bdev's ctxt is the malloc_disk, whose first member is the bdev itself. */
	return *(uint8_t **)((char *)r->bdev->ctxt + sizeof(struct spdk_bdev));
}

static struct spdk_bdev *ref_target_bdev(struct oimref *r, int target_num)
{
	if (target_num < 0 || target_num >= SPDK_VHOST_SCSI_CTRLR_MAX_DEVS) return NULL;
	if (r->extra[target_num]) return r->extra[target_num];
	return r->svdev->scsi_dev_state[target_num].dev ? r->bdev : NULL;
}

static void stat_done(struct spdk_bdev *b, struct spdk_bdev_io_stat *stat, void *arg, int rc) { *(int *)arg = rc ? -1 : 1; }
static void hist_done(void *arg, int rc, struct spdk_histogram_data *h) { *(int *)arg = rc ? -1 : 1; }
static void hist_sum(void *ctx, uint64_t start, uint64_t end, uint64_t count, uint64_t total, uint64_t so_far)
{
	*(uint64_t *)ctx += count;
}

/* The target bdev's counters as get_bdevs_iostat reads them (spdk_bdev_get_device_stat, bdev_rpc.c:186) and the
 * total of its latency histogram (spdk_bdev_histogram_get, as get_bdev_histogram): out = num_read_ops, bytes_read,
 * num_write_ops, bytes_written, num_unmap_ops, bytes_unmapped, bdev_ios.  -ENODEV: no device in that slot. */
int oimref_iostat(void *h, int target_num, uint64_t out[7])
{
	struct oimref *r = h;
	struct spdk_bdev *b = ref_target_bdev(r, target_num);
	struct spdk_bdev_io_stat stat;
	struct spdk_histogram_data *hist;
	int done = 0;

	if (!b) return -ENODEV;
	spdk_set_thread(g_thread);
	memset(&stat, 0, sizeof(stat));
	spdk_bdev_get_device_stat(b, &stat, stat_done, &done);
	while (!done) spdk_thread_poll(g_thread, 0, 0);
	if (done < 0) return -EIO;
	out[0] = stat.num_read_ops;
	out[1] = stat.bytes_read;
	out[2] = stat.num_write_ops;
	out[3] = stat.bytes_written;
	out[4] = stat.num_unmap_ops;
	out[5] = stat.bytes_unmapped;
	hist = spdk_histogram_data_alloc();
	if (!hist) return -ENOMEM;
	done = 0;
	spdk_bdev_histogram_get(b, hist, hist_done, &done);
	while (!done) spdk_thread_poll(g_thread, 0, 0);
	out[6] = 0;
	if (done > 0) spdk_histogram_data_iterate(hist, hist_sum, &out[6]);
	spdk_histogram_data_free(hist);
	return done < 0 ? -EIO : 0;
}

uint64_t oimref_num_blocks(void *h) { return spdk_bdev_get_num_blocks(((struct oimref *)h)->bdev); }

/* Mark the target hot-removed for this session (what remove_vhost_scsi_target does first,
 * vhost_scsi.c:1093-1100) without draining, so the "removed" branches can be exercised. */
void oimref_set_removed(void *h, int target_num, int removed)
{
	struct oimref *r = h;
	r->svsession->scsi_dev_state[target_num].removed = removed;
}

static void dummy_unregister_cb(void *arg, int rc) {}

void oimref_destroy(void *h)
{
	struct oimref *r = h;
	int t;
	if (!r) return;
	spdk_set_thread(g_thread);
	for (t = 0; t < SPDK_VHOST_SCSI_CTRLR_MAX_DEVS; t++) {
		struct spdk_scsi_dev *d = r->svdev->scsi_dev_state[t].dev;
		if (d) {
			spdk_scsi_dev_free_io_channels(d);
			spdk_scsi_dev_destruct(d);
		}
	}
	for (t = 0; t < 8; t++) spdk_thread_poll(g_thread, 0, 0);
	delete_malloc_disk(r->bdev, dummy_unregister_cb, NULL);
	for (t = 0; t < SPDK_VHOST_SCSI_CTRLR_MAX_DEVS; t++) {
		if (r->extra[t]) delete_malloc_disk(r->extra[t], dummy_unregister_cb, NULL);
	}
	for (t = 0; t < 8; t++) spdk_thread_poll(g_thread, 0, 0);
	close(r->eventfd);
	free(r->vq->tasks); free(r->indirect); free(r->resp_bufs); free(r->req_bufs);
	free(r->used); free(r->avail); free(r->desc); free(r->mem);
	free(r->svdev->vdev.name); free(r->svdev); free(r->svsession); free(r);
}

/* Build the descriptor chain of one request.  Layouts (vhost_scsi.c:531-613):
 *   FROM_DEV: [RO req 51 B][WR resp 108 B][WR data ...]      TO_DEV: [RO req][RO data ...][WR resp]
 * Returns the number of ring descriptors consumed (1 when an indirect table is used). */
static int build_chain(struct oimref *r, int slot, uint16_t head, uint16_t *next_free,
		       const struct oimgpu_req *q, const struct oimgpu_iov *iovs)
{
	struct vring_desc *tbl;
	uint32_t n = 0, i, cnt = q->iovcnt;
	int use_indirect;
	struct virtio_scsi_cmd_req *rq = &r->req_bufs[slot];
	struct virtio_scsi_cmd_resp *rs = &r->resp_bufs[slot];
	int from_dev = (q->dir == OIMGPU_DIR_FROM_DEV) || cnt == 0;

	memcpy(rq, q, sizeof(*rq));		/* bytes 0..50 of oimgpu_req ARE virtio_scsi_cmd_req */
	memset(rs, 0, sizeof(*rs));

	if (cnt > REF_INDIRECT_MAX - 2) cnt = REF_INDIRECT_MAX - 2;	/* still > 129: stays invalid */
	use_indirect = (cnt + 2 > 16);
	tbl = use_indirect ? &r->indirect[(size_t)slot * REF_INDIRECT_MAX] : r->desc;

#define DIDX(k) (use_indirect ? (uint16_t)(k) : (uint16_t)((head + (k)) % REF_VQ_SIZE))
#define PUT(_addr, _len, _wr, _last) do {						\
		struct vring_desc *d = &tbl[DIDX(n)];					\
		d->addr = (uint64_t)(_addr); d->len = (_len);				\
		d->flags = ((_wr) ? VRING_DESC_F_WRITE : 0) | ((_last) ? 0 : VRING_DESC_F_NEXT); \
		d->next = (_last) ? 0 : DIDX(n + 1);					\
		n++;									\
	} while (0)

	PUT(rq, sizeof(*rq), 0, 0);
	if (from_dev) {
		PUT(rs, sizeof(*rs), 1, cnt == 0);
		for (i = 0; i < cnt; i++) {
			const struct oimgpu_iov *v = &iovs[q->iov_start + i];
			PUT(v->addr, v->len, 1, i + 1 == cnt);
		}
	} else {
		for (i = 0; i < cnt; i++) {
			const struct oimgpu_iov *v = &iovs[q->iov_start + i];
			PUT(v->addr, v->len, 0, 0);
		}
		PUT(rs, sizeof(*rs), 1, 1);
	}
#undef PUT
#undef DIDX
	if (use_indirect) {
		struct vring_desc *d = &r->desc[head];
		d->addr = (uint64_t)(uintptr_t)tbl;
		d->len = n * sizeof(struct vring_desc);
		d->flags = VRING_DESC_F_INDIRECT;
		d->next = 0;
		*next_free = (head + 1) % REF_VQ_SIZE;
		return 1;
	}
	*next_free = (head + n) % REF_VQ_SIZE;
	return n;
}

/* Execute nreqs requests in order, <= 32 per process_requestq() pass, and report what the guest
 * would observe: used-ring length and the response fields.  SG addresses are host pointers. */
int oimref_submit(void *h, const struct oimgpu_req *reqs, uint32_t nreqs,
		  const struct oimgpu_iov *iovs, uint32_t niovs, struct oimgpu_cpl *cpls)
{
	struct oimref *r = h;
	uint32_t done = 0;
	struct timespec t0, t1;

	(void)niovs;
	spdk_set_thread(g_thread);
	while (done < nreqs) {
		uint32_t batch = nreqs - done, i;
		uint16_t head = 0, heads[OIMGPU_REQS_PER_PASS];
		uint16_t avail_idx = r->avail->idx;

		if (batch > OIMGPU_REQS_PER_PASS) batch = OIMGPU_REQS_PER_PASS;
		for (i = 0; i < batch; i++) {
			uint16_t nf;
			heads[i] = head;
			build_chain(r, i, head, &nf, &reqs[done + i], iovs);
			head = nf;
			r->avail->ring[(avail_idx + i) & (REF_VQ_SIZE - 1)] = heads[i];
		}
		__sync_synchronize();
		r->avail->idx = avail_idx + batch;

		clock_gettime(CLOCK_MONOTONIC, &t0);
		process_requestq(r->svsession, r->vq);
		ut_spdk_get_ticks++;
		/* The Malloc module copies inline, but bdev.c defers the completion callback of an I/O
		 * that finished inside submit_request to the next thread poll (bdev.c:3213-3229), so
		 * successful I/Os reach the used ring after the pass, behind any request that failed
		 * validation.  Data effects are in submission order; used-ring order is not. */
		for (i = 0; i < 64 && (uint16_t)(r->used->idx - r->used_seen) != batch; i++) {
			spdk_thread_poll(g_thread, 0, 0);
		}
		spdk_vhost_vq_used_signal(&r->svsession->vsession, r->vq);
		clock_gettime(CLOCK_MONOTONIC, &t1);
		r->poller_ns += (uint64_t)(t1.tv_sec - t0.tv_sec) * 1000000000ull + (uint64_t)(t1.tv_nsec - t0.tv_nsec);

		if ((uint16_t)(r->used->idx - r->used_seen) != batch) return -EIO;
		for (i = 0; i < batch; i++) {
			struct vring_used_elem *ue = &r->used->ring[(r->used_seen + i) & (REF_VQ_SIZE - 1)];
			struct virtio_scsi_cmd_resp *rs;
			struct oimgpu_cpl *c;
			uint32_t k;
			for (k = 0; k < batch && heads[k] != ue->id; k++) {}
			if (k == batch) return -EPROTO;		/* used id that was never made available */
			rs = &r->resp_bufs[k];
			c = &cpls[done + k];
			memset(c, 0, sizeof(*c));
			c->tag = reqs[done + k].tag;
			c->used_len = ue->len;
			c->resp_valid = ue->len != 0;
			c->sense_len = rs->sense_len;
			c->resid = rs->resid;
			c->status_qualifier = rs->status_qualifier;
			c->status = rs->status;
			c->response = rs->response;
			memcpy(c->sense, rs->sense, OIMGPU_SENSE_SIZE);
		}
		r->used_seen += batch;
		done += batch;
	}
	return 0;
}

/* The reference's SG translation on its own (golden vectors of vhost_ut.c:153-235):
 * regions = {gpa, size, hva} triples. Returns iov count or -1. */
int oimref_desc_to_iov(const uint64_t *regions, uint32_t nregions, uint64_t addr, uint32_t len,
		       struct oimgpu_iov *out, uint32_t start_index)
{
	struct spdk_vhost_session vs;
	struct rte_vhost_memory *mem = calloc(1, sizeof(*mem) + nregions * sizeof(struct rte_vhost_mem_region));
	struct iovec iov[SPDK_VHOST_IOVS_MAX];
	struct vring_desc d = { .addr = addr, .len = len };
	uint16_t idx = start_index, i;
	int rc;

	mem->nregions = nregions;
	for (i = 0; i < nregions; i++) {
		mem->regions[i].guest_phys_addr = regions[3 * i];
		mem->regions[i].size = regions[3 * i + 1];
		mem->regions[i].host_user_addr = regions[3 * i + 2];
	}
	memset(&vs, 0, offsetof(struct spdk_vhost_session, virtqueue));
	vs.mem = mem;
	rc = spdk_vhost_vring_desc_to_iov(&vs, iov, &idx, &d);
	free(mem);
	if (rc != 0) return -1;
	for (i = start_index; i < idx; i++) {
		out[i - start_index].addr = (uint64_t)(uintptr_t)iov[i].iov_base;
		out[i - start_index].len = iov[i].iov_len;
		out[i - start_index].flags = 0;
	}
	return idx - start_index;
}

/* Virtqueue level: run the reference's poller over a caller-built split ring living in caller
 * memory.  desc/avail/used are host addresses of the three ring areas (what rte_vhost_get_vhost_vring
 * reports), regions = {guest_phys_addr, size, host_user_addr} triples (the rte_vhost_memory table).
 * Processes everything up to avail->idx in passes of <= 32 and returns the number of used elements
 * produced; *last_avail_idx / *last_used_idx are the ring cursors, updated in place. */
int oimref_vq_process(void *h, uint64_t desc, uint64_t avail, uint64_t used, uint32_t size,
		      const uint64_t *regions, uint32_t nregions, uint16_t *last_avail_idx, uint16_t *last_used_idx)
{
	struct oimref *r = h;
	struct spdk_vhost_session *vs = &r->svsession->vsession;
	struct spdk_vhost_virtqueue *vq = &vs->virtqueue[VIRTIO_SCSI_REQUESTQ + 1];
	struct rte_vhost_memory *mem, *saved_mem = vs->mem;
	struct vring_avail *av = (struct vring_avail *)(uintptr_t)avail;
	struct vring_used *us = (struct vring_used *)(uintptr_t)used;
	struct timespec t0, t1;
	uint16_t start_used = *last_used_idx, want, i;
	int spins = 0;

	if (size == 0 || size > SPDK_VHOST_MAX_VQ_SIZE || (size & (size - 1))) return -EINVAL;
	spdk_set_thread(g_thread);
	mem = calloc(1, sizeof(*mem) + nregions * sizeof(struct rte_vhost_mem_region));
	mem->nregions = nregions;
	for (i = 0; i < nregions; i++) {
		mem->regions[i].guest_phys_addr = regions[3 * i];
		mem->regions[i].size = regions[3 * i + 1];
		mem->regions[i].host_user_addr = regions[3 * i + 2];
	}
	vs->mem = mem;
	memset(vq, 0, sizeof(*vq));
	vq->vring.desc = (struct vring_desc *)(uintptr_t)desc;
	vq->vring.avail = av;
	vq->vring.used = us;
	vq->vring.size = size;
	vq->vring.callfd = r->eventfd;
	vq->vring.kickfd = -1;
	vq->vring.last_avail_idx = *last_avail_idx;
	vq->vring.last_used_idx = *last_used_idx;
	vq->tasks = calloc(size, sizeof(struct spdk_vhost_scsi_task));
	for (i = 0; i < size; i++) {
		struct spdk_vhost_scsi_task *t = &((struct spdk_vhost_scsi_task *)vq->tasks)[i];
		t->svsession = r->svsession;
		t->vq = vq;
		t->req_idx = i;
	}
	want = (uint16_t)(av->idx - *last_avail_idx);
	if (want > size) want = 0;	/* "the queue is unrecoverably broken" (vhost.c:193-198) */

	clock_gettime(CLOCK_MONOTONIC, &t0);
	while ((uint16_t)(us->idx - start_used) != want && spins++ < 100000) {
		process_requestq(r->svsession, vq);
		ut_spdk_get_ticks++;
		spdk_thread_poll(g_thread, 0, 0);
		spdk_vhost_vq_used_signal(vs, vq);
	}
	clock_gettime(CLOCK_MONOTONIC, &t1);
	r->poller_ns += (uint64_t)(t1.tv_sec - t0.tv_sec) * 1000000000ull + (uint64_t)(t1.tv_nsec - t0.tv_nsec);

	*last_avail_idx = vq->vring.last_avail_idx;
	*last_used_idx = vq->vring.last_used_idx;
	free(vq->tasks);
	vq->tasks = NULL;
	vs->mem = saved_mem;
	free(mem);
	return (uint16_t)(us->idx - start_used) == want ? (int)want : -EIO;
}

/* ---- the reference's own JSON-RPC server (S/lib/rpc, S/lib/jsonrpc) with its registered handlers:
 * get_bdevs / construct_malloc_bdev / delete_bdev (bdev_rpc.c, bdev_malloc_rpc.c) and the vhost-scsi
 * methods (vhost_rpc.c).  Used to pin the wire behaviour of our daemon (tests/test_rpc_daemon.py). */
#include <execinfo.h>
#include <signal.h>
static void ref_segv(int sig)
{
	void *bt[48];
	int n = backtrace(bt, 48);
	backtrace_symbols_fd(bt, n, 2);
	_exit(139);
}

void oimref_enter(void)
{
	ref_global_init();
	spdk_set_thread(g_thread);
}

/* run the SPDK thread's pollers and messages (what a reactor iteration does); a tick passes before each */
void oimref_thread_poll(int iterations)
{
	int i;
	spdk_set_thread(g_thread);
	for (i = 0; i < iterations; i++) {
		ut_spdk_get_ticks++;
		spdk_thread_poll(g_thread, 0, 0);
	}
}

const char *oimref_bdev_name(void *h) { return ((struct oimref *)h)->bdev_name; }

int oimref_rpc_start(const char *sock_path, const char *vhost_socket_dir)
{
	if (getenv("OIMREF_VERBOSE")) signal(SIGSEGV, ref_segv);
	if (ref_global_init() != 0) return -1;
	if (vhost_socket_dir && spdk_vhost_set_socket_path(vhost_socket_dir) != 0) return -2;
	if (spdk_vhost_init() != 0) return -4;	/* per-core controller counters used when a session starts */
	if (spdk_rpc_listen(sock_path) != 0) return -3;
	spdk_rpc_set_state(SPDK_RPC_RUNTIME);
	return 0;
}

void oimref_rpc_poll(int iterations)
{
	int i;
	spdk_set_thread(g_thread);
	for (i = 0; i < iterations; i++) {
		struct timespec ts;
		/* the unit-test env's clock (1 tick = 1 us, test_env.c:412-435) follows real time here, so that
		 * timed pollers - the 5 ms management poller, the session-stop poller - run as in the daemon */
		clock_gettime(CLOCK_MONOTONIC, &ts);
		ut_spdk_get_ticks = (uint64_t)ts.tv_sec * 1000000 + ts.tv_nsec / 1000;
		/* SPDK polls its RPC socket from a timed poller (4 ms), not on every reactor iteration: do not charge
		 * the data path an accept() syscall per loop */
		if ((i & 63) == 0) spdk_rpc_accept();
		ref_run_events();
		spdk_thread_poll(g_thread, 0, 0);
	}
}

void oimref_rpc_stop(void)
{
	spdk_set_thread(g_thread);
	spdk_rpc_close();
}

/* nanoseconds spent in process_requestq() + completion polling + used_signal since the last reset:
 * the reference's own work, without this driver's descriptor-chain building (which a guest does) */
uint64_t oimref_busy_ns(void *h, int reset)
{
	struct oimref *r = h;
	uint64_t v = r->poller_ns;
	if (reset) r->poller_ns = 0;
	return v;
}

const char *oimref_describe(void)
{
	return "reference: intel/oim vendored SPDK v19.04-pre (rev 8bbf0391), lib/{vhost,scsi,bdev,bdev/malloc,copy}, -O2";
}
