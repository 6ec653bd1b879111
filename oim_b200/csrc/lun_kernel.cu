/*
 * lun_kernel.cu — oim_lun_queue_kernel: see lun_kernel.cuh for the map onto the reference.
 *
 * Warp-specialised: every CTA is a small "reactor" with
 *   warp 0            the PARSER   = vdev_worker/process_requestq (vhost_scsi.c:690-772): pulls <= 32
 *                     request slots per pass, lane i parses request i (SG walk, LUN check, CDB
 *                     decode, limits), the warp orders LBA hazards, emits SG segments into a stage
 *                     and later publishes the pass's completion records;
 *   warps 1..kMovers  the MOVERS   = bdev_malloc_readv/writev/unmap + mem_copy_submit
 *                     (bdev_malloc.c:153-233, copy_engine.c:114-140): stream the payload of the
 *                     stage, one 4 KiB unit per warp-step, 8 x 16-byte loads in flight per lane.
 * Parser and movers are decoupled by a ring of kStages stages guarded by mbarriers
 * (full[s]: parser -> movers, empty[s]: movers -> parser), so request fetch, SG walk and CDB decode
 * of pass p+1/p+2 overlap the data movement of pass p.  Request slots of the next pass are
 * prefetched into registers while the current one is parsed.
 *
 * Launch shape: grid = min(#queues, SMs x CTAs/SM) CTAs of (1 + kMovers) x 32 threads; CTA b starts on
 * queue b, then draws further queues from a shared counter (KickHeader.next, preset to the grid size),
 * and keeps the pipeline running across queue boundaries.
 */
#include "lun_kernel.cuh"

namespace oimgpu {

/* ---- mbarrier helpers (shared::cta) ------------------------------------------------------------ */

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count)
{
	asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar)
{
	asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0];\n\t}" :: "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity)
{
	asm volatile(
		"{\n\t.reg .pred p;\n\t"
		"WAIT_%=:\n\t"
		"mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
		"@p bra DONE_%=;\n\t"
		"bra WAIT_%=;\n\t"
		"DONE_%=:\n\t}"
		:: "r"(smem_u32(bar)), "r"(parity) : "memory");
}
/* non-blocking: has the phase with this parity completed? */
__device__ __forceinline__ bool mbar_test(uint64_t *bar, uint32_t parity)
{
	uint32_t ok;
	asm volatile(
		"{\n\t.reg .pred p;\n\t"
		"mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
		"selp.u32 %0, 1, 0, p;\n\t}"
		: "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
	return ok != 0;
}

/* ---- TMA: request slots global -> shared memory in one bulk copy per pass ---------------------------- */

/* one thread: expect `bytes` on the barrier (and arrive on it: the barrier's only arrival) */
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes)
{
	asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
}
/* one thread: dst (shared), src (global), bytes: 16-byte aligned; completion = `bytes` arriving on the barrier */
__device__ __forceinline__ void tma_load_bulk(void *dst_smem, const void *src_gmem, uint32_t bytes, uint64_t *bar)
{
	asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
		     :: "r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

/* ---- byte-granular SG elements: the unit goes through shared memory ---------------------------------
 *
 * A unit whose source, destination or length is not a multiple of 16 (SURVEY.md §7 "unaligned SG elements",
 * the 100 B + 31 x 4096 B + 3996 B list of SURVEY §8(d) C3 when its elements do not continue each other) cannot
 * take the register path at full depth: realigning in registers needs the neighbour lane's vector (shuffles) and
 * a ninth vector per lane, which spills at 128 registers, and with half-units in flight the movers are latency
 * bound.  Here the TMA unit fetches the aligned bytes
 * that cover the unit (<= 4112) in ONE bulk copy - no registers held while it flies - and the lanes realign
 * from shared memory: two aligned 16-byte LDS per output vector, funnel shifts, aligned 16-byte stores.
 * Over-read: up to 15 bytes on either side, inside aligned vectors that hold a byte of the element (never across
 * a page), read into shared memory and never stored. */
__device__ __forceinline__ int4 lds16(const uint8_t *p)
{
	int4 r;
	asm volatile("ld.shared.v4.s32 {%0,%1,%2,%3}, [%4];"
		     : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "r"(smem_u32(p)) : "memory");
	return r;
}

/* output vector = bytes m .. m+15 of the 32 bytes (a, b); Q = m / 4 picks the words at compile time, the byte shift
 * r = 8 (m % 4) is a funnel-shift operand */
template <int Q>
__device__ __forceinline__ void realign_rows(uint8_t *d, const uint8_t *base, uint32_t nv, uint32_t r, int lane)
{
#pragma unroll 4
	for (uint32_t v = lane; v < nv; v += 32) {
		const int4 a = lds16(base + v * 16), b = lds16(base + v * 16 + 16);
		const uint32_t w[8] = {(uint32_t)a.x, (uint32_t)a.y, (uint32_t)a.z, (uint32_t)a.w, (uint32_t)b.x, (uint32_t)b.y, (uint32_t)b.z, (uint32_t)b.w};
		st_cg16(d + (size_t)v * 16, make_int4(__funnelshift_r(w[Q], w[Q + 1], r), __funnelshift_r(w[Q + 1], w[Q + 2], r),
						      __funnelshift_r(w[Q + 2], w[Q + 3], r), __funnelshift_r(w[Q + 3], w[Q + 4], r)));
	}
}

/* One unit = two pieces, each with its own half of the warp's staging buffer and its own barrier: the first ends
 * where the destination is 16-byte aligned (head + 127 vectors), the second takes the rest.  While a piece is realigned
 * out of shared memory the other one is still flying, and when the mover knows its NEXT unit (same fill, no barrier in
 * between) that unit's pieces are requested as soon as the buffers are free: loads and realignment overlap, which is
 * what the register path could not do (there the movers stalled on the arrival of the unit they were about to
 * realign). */
constexpr uint32_t kPieceBody = 2032;			/* 127 vectors */
constexpr uint32_t kPieceBuf = (kUnitBytes + 128) / 2;	/* 2112 >= 15 + (kUnitBytes - kPieceBody) + 15 rounded to 16 */

struct UStage {			/* per mover warp, in registers */
	const uint8_t *pf_src;	/* source of the unit whose pieces are already requested (nullptr: none) */
	uint32_t phase;		/* bit s: parity of the barrier of piece s */
};

__device__ __forceinline__ uint32_t piece0_bytes(const uint8_t *dst, uint32_t n)
{
	const uint32_t head = (uint32_t)((16 - ((uintptr_t)dst & 15)) & 15);
	return min(n, head + kPieceBody);
}

/* lane 0: request the aligned bytes that cover [src, src + n) */
__device__ __forceinline__ void ustage_issue(const uint8_t *src, uint32_t n, uint8_t *buf, uint64_t *bar)
{
	const uint32_t so = (uint32_t)((uintptr_t)src & 15);
	const uint32_t span = (so + n + 15) & ~15u;
	mbar_expect_tx(bar, span);
	tma_load_bulk(buf, src - so, span, bar);
}

/* the warp: wait for the piece, move it out */
__device__ __forceinline__ void ustage_consume(uint8_t *dst, const uint8_t *src, uint32_t n, int lane,
					       const uint8_t *buf, uint64_t *bar, uint32_t parity)
{
	const uint32_t so = (uint32_t)((uintptr_t)src & 15);
	uint32_t head = (uint32_t)((16 - ((uintptr_t)dst & 15)) & 15);
	if (head > n) head = n;
	const uint32_t body = n - head, nv = body >> 4, tail = body & 15;
	const uint32_t o = so + head;			/* where the body starts in the staged bytes */
	const uint32_t m = o & 15, r = (m & 3) * 8;
	const uint8_t *base = buf + (o & ~15u);
	uint8_t *d = dst + head;
	mbar_wait(bar, parity);
	if ((uint32_t)lane < head) dst[lane] = buf[so + lane];
	if (m == 0) {
#pragma unroll 4
		for (uint32_t v = lane; v < nv; v += 32) st_cg16(d + (size_t)v * 16, lds16(base + v * 16));
	} else {
		switch (m >> 2) {
		case 0: realign_rows<0>(d, base, nv, r, lane); break;
		case 1: realign_rows<1>(d, base, nv, r, lane); break;
		case 2: realign_rows<2>(d, base, nv, r, lane); break;
		default: realign_rows<3>(d, base, nv, r, lane); break;
		}
	}
	if ((uint32_t)lane < tail) d[(size_t)nv * 16 + lane] = buf[o + nv * 16 + lane];
	__syncwarp();		/* every lane has read its bytes: the buffer may be refilled */
}

/* pfence: a mover of this or another CTA may have written the source bytes earlier in this launch (a read behind
 * a write, ordered by the stage / drain / wave barriers - generic-proxy events) and the bulk copy reads through the
 * async proxy: the first staged unit after such a barrier crosses proxies with a fence.  Prefetched units never
 * follow a barrier (the mover asks for the next unit only when nothing has to be waited for in between).
 * nsrc != nullptr: the unit this warp moves next, (ndst, nsrc, nn), also takes this path - request it. */
__device__ __forceinline__ void move_unit_via_smem(uint8_t *dst, const uint8_t *src, uint32_t n, int lane,
							  uint8_t *ust, uint64_t *bar, UStage &us, bool &pfence,
							  uint8_t *ndst, const uint8_t *nsrc, uint32_t nn)
{
	const uint32_t n0 = piece0_bytes(dst, n), n1 = n - n0;
	if (us.pf_src != src) {
		if (lane == 0) {
			if (pfence) asm volatile("fence.proxy.async.global;" ::: "memory");
			ustage_issue(src, n0, ust, &bar[0]);
			if (n1) ustage_issue(src + n0, n1, ust + kPieceBuf, &bar[1]);
		}
		pfence = false;
	}
	ustage_consume(dst, src, n0, lane, ust, &bar[0], us.phase & 1);
	us.phase ^= 1;
	uint32_t m0 = 0;
	if (nsrc) {
		m0 = piece0_bytes(ndst, nn);
		if (lane == 0) ustage_issue(nsrc, m0, ust, &bar[0]);
	}
	if (n1) {
		ustage_consume(dst + n0, src + n0, n1, lane, ust + kPieceBuf, &bar[1], (us.phase >> 1) & 1);
		us.phase ^= 2;
	}
	if (nsrc && nn > m0 && lane == 0) ustage_issue(nsrc + m0, nn - m0, ust + kPieceBuf, &bar[1]);
	us.pf_src = nsrc;
}

/* ---- shared queues: position counters in device memory, handed from CTA to CTA ------------------- */

__device__ __forceinline__ uint32_t ld_acquire32(const uint32_t *p)
{
	uint32_t r;
	asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(r) : "l"(p) : "memory");
	return r;
}
__device__ __forceinline__ void st_release32(uint32_t *p, uint32_t v)
{
	asm volatile("st.release.gpu.global.u32 [%0], %1;" :: "l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint64_t ld_vol64(const uint64_t *p)
{
	uint64_t r;
	asm volatile("ld.volatile.global.u64 %0, [%1];" : "=l"(r) : "l"(p) : "memory");
	return r;
}
__device__ __forceinline__ void st_vol64(uint64_t *p, uint64_t v)
{
	asm volatile("st.volatile.global.u64 [%0], %1;" :: "l"(p), "l"(v) : "memory");
}
/* wait until the in-order counter reaches exactly `pos` (its predecessor has published) */
__device__ __forceinline__ void chain_wait(const uint32_t *ctr, uint32_t pos)
{
	while (ld_acquire32(ctr) != pos) __nanosleep(20);
}

__device__ __forceinline__ void movers_barrier()
{
	asm volatile("bar.sync 1, %0;" :: "n"(kMovers * 32) : "memory");
}

/* ---- parser: one lane, one request ------------------------------------------------------- */

__device__ __forceinline__ uint32_t units_of(uint64_t len) { return (uint32_t)((len + kUnitBytes - 1) / kUnitBytes); }

/* spdk_bdev_bytes_to_blocks + spdk_bdev_io_valid_blocks (bdev.c:2474-2509) on (offset, nbytes) */
__device__ __forceinline__ bool bdev_range_ok(const LunCtx &L, uint64_t lba, uint64_t nbytes, uint64_t *nblk)
{
	uint64_t nb;
	if (L.block_shift != 0xffffffffu) {
		nb = nbytes >> L.block_shift;
		if ((nb << L.block_shift) != nbytes) return false;
	} else {
		nb = nbytes / L.block_size;
		if (nb * L.block_size != nbytes) return false;
	}
	if (lba + nb < lba) return false;
	if (lba + nb > L.num_blocks) return false;
	*nblk = nb;
	return true;
}

/* spdk_bdev_scsi_readwrite + _read/_write (scsi_bdev.c:1456-1511, 1318-1411) */
__device__ __forceinline__ void scsi_readwrite(const LunCtx &L, LaneState &s, uint32_t dxfer_dir, uint32_t transfer_len,
					       uint64_t lba, uint32_t xfer_len, bool is_read)
{
	s.data_transferred = 0;
	if (dxfer_dir != OIMGPU_DIR_NONE && dxfer_dir != (is_read ? OIMGPU_DIR_FROM_DEV : OIMGPU_DIR_TO_DEV)) {
		set_check(s, SK_NO_SENSE, ASC_NONE);
		return;
	}
	if (L.num_blocks <= lba || L.num_blocks - lba < xfer_len) {
		set_check(s, SK_ILLEGAL_REQUEST, ASC_LBA_OOR);
		return;
	}
	if (xfer_len == 0) {
		s.status = SC_GOOD;
		return;
	}
	if (xfer_len > OIMGPU_MAX_XFER_BYTES / L.block_size) {
		set_check(s, SK_ILLEGAL_REQUEST, ASC_INVALID_FIELD);
		return;
	}
	uint64_t nblk;
	if (!is_read) {
		if ((uint64_t)xfer_len * L.block_size > transfer_len) {
			set_check(s, SK_NO_SENSE, ASC_NONE);
			return;
		}
	}
	/* both directions move task->length bytes, not xfer_len blocks (scsi_bdev.c:1333, 1387) */
	if (!bdev_range_ok(L, lba, s.length, &nblk)) {
		set_check(s, SK_NO_SENSE, ASC_NONE);
		return;
	}
	s.data_transferred = s.length;
	s.off = lba * L.block_size;
	s.store_lo = (uint64_t)(uintptr_t)L.store[0] + s.off;	/* absolute: two targets conflict only on a shared bdev */
	s.store_hi = s.store_lo + nblk * L.block_size;
	s.op = is_read ? OP_READ : OP_WRITE;
	s.hazard = nblk ? (is_read ? 1 : 2) : 0;
}

/* UNMAP parameter list walk (scsi_bdev.c:1545-1679).  emit == nullptr: validate and count;
 * otherwise also write one zero-fill segment per accepted descriptor. */
__device__ __noinline__ void scsi_unmap(const LunCtx &L, const QueueDesc &q, const oimgpu_req &r, uint32_t iovcnt,
					LaneState &s, Segment *emit, uint32_t first_unit, uint16_t wave)
{
	const uint32_t data_len = s.length;
	int desc_count = -1;
	if (data_len >= 8) {
		uint16_t ddl = (uint16_t)(gather_byte(q, r, iovcnt, 2) << 8 | gather_byte(q, r, iovcnt, 3));
		if (ddl <= data_len - 8 && ddl / 16 <= OIMGPU_MAX_UNMAP_DESC) desc_count = ddl / 16;
	}
	if (desc_count < 0) {
		if (!emit) set_check(s, SK_ILLEGAL_REQUEST, ASC_INVALID_FIELD);
		return;
	}
	uint32_t nseg = 0, units = 0;
	uint64_t total = 0;
	for (int i = 0; i < desc_count; i++) {
		uint64_t ob = 0;
		uint32_t nb = 0;
		for (int k = 0; k < 8; k++) ob = ob << 8 | gather_byte(q, r, iovcnt, 8 + 16 * i + k);
		for (int k = 8; k < 12; k++) nb = nb << 8 | gather_byte(q, r, iovcnt, 8 + 16 * i + k);
		if (nb == 0) continue;
		if (ob + nb < ob || ob + nb > L.num_blocks) {
			/* spdk_bdev_unmap_blocks -> -EINVAL: earlier descriptors stay applied, the rest are skipped */
			if (!emit) set_check(s, SK_NO_SENSE, ASC_NONE);
			break;
		}
		uint64_t bytes = (uint64_t)nb * L.block_size;
		if (emit) {
			Segment &g = emit[nseg];
			g.src = nullptr;
			g.dst = L.store[0] + ob * L.block_size;
			g.len = bytes;
			g.first_unit = first_unit + units;
			g.wave = wave;
			g.mirror = L.nreplicas > 1 ? (uint8_t)(L.target + 1) : 0;
		}
		nseg++;
		units += units_of(bytes);
		total += bytes;
	}
	if (!emit) {
		s.nseg = nseg;
		s.units = units;
		s.unmap_bytes = total;
		s.op = OP_UNMAP;
		s.hazard = nseg ? 3 : 0;
	}
}

/* control payloads: READ CAPACITY 10/16, REQUEST SENSE, null-LUN INQUIRY (kept out of line: rare) */
__device__ __noinline__ void scsi_control(const LunCtx &L, const QueueDesc &q, const oimgpu_req &r, uint32_t cnt,
					  uint32_t len, LaneState &s, int which)
{
	uint8_t *buf = s.scratch;
	for (int k = 0; k < 36; k++) buf[k] = 0;
	const uint8_t *cdb = r.cdb;
	if (which == 0) {		/* spdk_scsi_task_process_null_lun INQUIRY (task.c:263-281) */
		buf[0] = 0x03 << 5 | 0x1f;
		buf[4] = 36 - 5;
		uint32_t alloc_len = be16(&cdb[3]);
		if (scatter_small(q, r, cnt, len, buf, alloc_len < 36 ? alloc_len : 36, s) >= 0) {
			s.data_transferred = 36;
			s.status = SC_GOOD;
		}
	} else if (which == 1) {	/* READ CAPACITY (10) (scsi_bdev.c:1729-1749) */
		uint64_t last = L.num_blocks - 1;
		uint32_t v = last > 0xffffffffULL ? 0xffffffffu : (uint32_t)last;
		buf[0] = v >> 24; buf[1] = v >> 16; buf[2] = v >> 8; buf[3] = v;
		buf[4] = L.block_size >> 24; buf[5] = L.block_size >> 16; buf[6] = L.block_size >> 8; buf[7] = L.block_size;
		uint32_t l = len < 8 ? len : 8;
		if (scatter_small(q, r, cnt, len, buf, l, s) >= 0) {
			s.data_transferred = l;
			s.status = SC_GOOD;
		}
	} else if (which == 2) {	/* READ CAPACITY (16) (scsi_bdev.c:1751-1777) */
		uint64_t last = L.num_blocks - 1;
		for (int k = 0; k < 8; k++) buf[k] = (uint8_t)(last >> (56 - 8 * k));
		buf[8] = L.block_size >> 24; buf[9] = L.block_size >> 16; buf[10] = L.block_size >> 8; buf[11] = L.block_size;
		buf[14] |= 1 << 7;	/* TPE: UNMAP supported */
		uint32_t al = be32(&cdb[10]);
		uint32_t l = al < 32 ? al : 32;
		if (scatter_small(q, r, cnt, len, buf, l, s) >= 0) {
			s.data_transferred = l;
			s.status = SC_GOOD;
		}
	} else {			/* REQUEST SENSE (scsi_bdev.c:1997-2026) */
		if (!(cdb[1] & 0x1)) {
			buf[0] = 0xf0; buf[7] = 10;
			uint32_t al = cdb[4];
			scatter_small(q, r, cnt, len, buf, al < 18 ? al : 18, s);
			s.data_transferred = al < 18 ? al : 18;
		}
		s.status = SC_GOOD;	/* rc >= 0 path overrides whatever status was set (scsi_bdev.c:2066-2069) */
	}
}

__device__ void scsi_primary(const LunCtx &L, const QueueDesc &q, const oimgpu_req &r, uint32_t cnt, uint32_t len, LaneState &s);

/* spdk_vhost_scsi_task_init_target (vhost_scsi.c:361-387): all targets of a controller share its
 * virtqueues; lun[1] selects the SCSI device.  nullptr = no such device (VIRTIO_SCSI_S_BAD_TARGET). */
__device__ __forceinline__ const LunCtx *target_ctx(const LunCtx &L, const uint8_t *lun)
{
	if (lun[0] != 1 || lun[1] >= OIMGPU_CTRLR_MAX_DEVS) return nullptr;
	if (lun[1] == L.target) return &L;
	return L.peer[lun[1]];
}

__device__ __forceinline__ void parse_request(const LunCtx &L, const QueueDesc &q, const oimgpu_req &r, LaneState &s)
{
	const uint32_t cnt = r.iovcnt;
	const bool from_dev = (r.dir == OIMGPU_DIR_FROM_DEV) || cnt == 0;
	const uint32_t dxfer_dir = from_dev ? OIMGPU_DIR_FROM_DEV : OIMGPU_DIR_TO_DEV;
	uint32_t nonzero = 0, units = 0;
	uint64_t len64 = 0, run_len = 0, run_end = 0;	/* the run of contiguous elements being summed */

	s.op = OP_NONE; s.nseg = 0; s.valid = 1; s.length = 0; s.off = 0; s.tgt = L.target;
	s.store_lo = s.store_hi = 0;
	s.status = SC_GOOD; s.sk = 0; s.asc = 0;
	s.data_transferred = 0; s.units = 0; s.hazard = 0; s.response = OIMGPU_S_OK; s.resp_valid = 1;

	/* ---- task_data_setup (vhost_scsi.c:490-624): walk the SG list ---- */
	bool valid = true;
	for (uint32_t j = 0; j < cnt; j++) {
		if (j >= OIMGPU_IOVS_MAX) { valid = false; break; }
		if (q.iov_limit && r.iov_start + j >= q.iov_limit) { valid = false; break; }	/* index outside the SG table */
		const oimgpu_iov v = q.iovs[(r.iov_start + j) & q.iov_mask];
		if (v.addr == 0) { valid = false; break; }
		len64 += v.len;
		if (v.len) {
			/* elements that continue each other in client memory (a buffer that starts inside a page, split at
			 * page boundaries, as guests hand them over) move as ONE segment: the store side is contiguous by
			 * construction, so the per-element memcpys of bdev_malloc.c:180-189 add up to one copy of the run -
			 * with unit boundaries on the run, not on every element's odd head and tail.  A run that ends on
			 * a unit boundary is closed: joining the next element would give the same units, and separate
			 * segments keep the movers' loads spread (bench.py seq128k_sg: pages vs single) */
			if ((run_len & (kUnitBytes - 1)) && v.addr == run_end) {
				run_len += v.len;
			} else {
				units += units_of(run_len);
				run_len = v.len;
				nonzero++;
			}
			run_end = v.addr + v.len;
		}
	}
	units += units_of(run_len);
	/* The reference sums the element lengths in 32 bits (vhost_scsi.c:573, 596 `len += desc->len`): two
	 * elements of 2 GiB + 4 KiB wrap to 4 KiB, every length check passes on the wrapped value, and the copy
	 * then runs over the full elements.  There that overruns the target's own process; here it would cross
	 * into other tenants' LUNs in the same HBM.  A payload that does not fit task->length is an invalid request. */
	if (len64 > 0xffffffffull) valid = false;
	const uint32_t len = (uint32_t)len64;
	if (!valid) {
		s.valid = 0;
		s.used_len = 0;		/* invalid_request(): used element only (vhost_scsi.c:347-358) */
		s.resp_valid = 0;
		s.response = 0;
		return;
	}
	s.length = len;
	s.used_len = from_dev ? OIMGPU_RESP_SIZE + len : OIMGPU_RESP_SIZE;

	/* ---- spdk_vhost_scsi_task_init_target (vhost_scsi.c:361-387) ---- */
	const uint16_t lun_id = (uint16_t)((((uint16_t)r.lun[2] << 8) | r.lun[3]) & 0x3FFF);
	const LunCtx *tp = target_ctx(L, r.lun);
	if (tp == nullptr) {
		s.response = OIMGPU_S_BAD_TARGET;	/* resp->response only; nothing else is written */
		return;
	}
	s.tgt = r.lun[1];
	const LunCtx &T = *tp;	/* the SCSI device the request addresses: everything below is per target */
	const uint8_t *cdb = r.cdb;
	if (T.removed || lun_id != 0) {
		/* spdk_scsi_task_process_null_lun (task.c:258-293) */
		if (cdb[0] == 0x12) {
			scsi_control(T, q, r, cnt, len, s, 0);
		} else {
			set_check(s, SK_ILLEGAL_REQUEST, ASC_LUN_NOT_SUPPORTED);
			s.data_transferred = 0;
		}
		return;
	}
	if (T.lun_removed) {
		set_check(s, SK_ABORTED_COMMAND, ASC_NONE);	/* spdk_scsi_task_process_abort */
		return;
	}

	/* ---- spdk_bdev_scsi_process_block (scsi_bdev.c:1681-1802) ---- */
	switch (cdb[0]) {
	case 0x08: case 0x0a: {
		uint64_t lba = (uint64_t)cdb[1] << 16 | (uint64_t)cdb[2] << 8 | cdb[3];
		uint32_t xl = cdb[4] ? cdb[4] : 256;
		scsi_readwrite(T, s, dxfer_dir, len, lba, xl, cdb[0] == 0x08);
		break;
	}
	case 0x28: case 0x2a:
		scsi_readwrite(T, s, dxfer_dir, len, be32(&cdb[2]), be16(&cdb[7]), cdb[0] == 0x28);
		break;
	case 0xa8: case 0xaa:
		scsi_readwrite(T, s, dxfer_dir, len, be32(&cdb[2]), be32(&cdb[6]), cdb[0] == 0xa8);
		break;
	case 0x88: case 0x8a:
		scsi_readwrite(T, s, dxfer_dir, len, be64(&cdb[2]), be32(&cdb[10]), cdb[0] == 0x88);
		break;
	case 0x25:
		scsi_control(T, q, r, cnt, len, s, 1);
		break;
	case 0x9e:
		if ((cdb[1] & 0x1f) == 0x10) scsi_control(T, q, r, cnt, len, s, 2);
		else set_check(s, SK_ILLEGAL_REQUEST, ASC_INVALID_OPCODE);
		break;
	case 0x35: case 0x91: {	/* SYNCHRONIZE CACHE: bounds check; the FLUSH is a no-op on a RAM disk, but a bdev_io all the same */
		uint64_t lba; uint32_t n;
		if (cdb[0] == 0x35) { lba = be32(&cdb[2]); n = be16(&cdb[7]); }
		else { lba = be64(&cdb[2]); n = be32(&cdb[10]); }
		if (n == 0) n = (uint32_t)(T.num_blocks - lba);
		if (n != 0 && (lba >= T.num_blocks || n > T.num_blocks || lba > T.num_blocks - n)) {
			set_check(s, SK_NO_SENSE, ASC_NONE);
		} else if (n != 0) {
			s.op = OP_FLUSH;	/* spdk_bdev_flush_blocks (scsi_bdev.c:1437) */
		}
		break;
	}
	case 0x42:
		scsi_unmap(T, q, r, cnt, s, nullptr, 0, 0);
		break;
	/* ---- spdk_bdev_scsi_process_primary (scsi_bdev.c:1827-2077), table-free commands ---- */
	case 0x03:
		scsi_control(T, q, r, cnt, len, s, 3);
		break;
	case 0x4c: case 0x4d:	/* LOG SELECT / LOG SENSE */
		set_check(s, SK_ILLEGAL_REQUEST, ASC_INVALID_OPCODE);
		break;
	case 0x00: case 0x1b:	/* TEST UNIT READY / START STOP UNIT */
		break;
	case 0x12: case 0xa0: case 0x15: case 0x55: case 0x1a: case 0x5a:
		scsi_primary(T, q, r, cnt, len, s);
		break;
	default:
		set_check(s, SK_ILLEGAL_REQUEST, ASC_INVALID_OPCODE);
		break;
	}
	if (s.op == OP_READ || s.op == OP_WRITE) {
		s.nseg = nonzero;
		s.units = units;
	}
}

/* emit the payload segments of one parsed request into a stage */
__device__ __forceinline__ void emit_segments(const LunCtx &L, const QueueDesc &q, const oimgpu_req &r, LaneState &s,
					      Segment *out, uint32_t first_unit, uint16_t wave)
{
	const LunCtx &T = (s.tgt == L.target) ? L : *L.peer[s.tgt];
	const uint8_t mirror_tag = T.nreplicas > 1 ? (uint8_t)(s.tgt + 1) : 0;	/* writes fan out to the replicas */
	if (s.op == OP_UNMAP) {
		scsi_unmap(T, q, r, r.iovcnt, s, out, first_unit, wave);
		return;
	}
	uint8_t *pos = T.store[0] + s.off;
	const bool rd = s.op == OP_READ;
	uint32_t k = 0, u = first_unit;
	uint64_t run_end = 0;
	Segment *g = nullptr;		/* the open run of contiguous elements (see parse_request: same rule, same counts) */
	for (uint32_t j = 0; j < r.iovcnt; j++) {
		const oimgpu_iov v = q.iovs[(r.iov_start + j) & q.iov_mask];
		if (v.len == 0) continue;
		if (g && (g->len & (kUnitBytes - 1)) && v.addr == run_end) {
			g->len += v.len;
		} else {
			if (g) u += units_of(g->len);
			g = &out[k++];
			uint8_t *client = (uint8_t *)(uintptr_t)v.addr;
			g->src = rd ? pos : client;
			g->dst = rd ? client : pos;
			g->mirror = rd ? 0 : mirror_tag;
			g->len = v.len;
			g->first_unit = u;
			g->wave = wave;
		}
		run_end = v.addr + v.len;
		pos += v.len;
	}
}

/* completion record of one request (spdk_vhost_scsi_task_cpl, vhost_scsi.c:311-331) into the stage */
__device__ __forceinline__ void build_cpl(const oimgpu_req &r, const LaneState &s, oimgpu_cpl *out)
{
	__align__(16) oimgpu_cpl c;
	int4 *cz = reinterpret_cast<int4 *>(&c);
	cz[0] = cz[1] = cz[2] = make_int4(0, 0, 0, 0);
	c.tag = r.tag;
	c.used_len = s.used_len;
	c.resp_valid = s.resp_valid;
	c.response = s.response;
	if (s.resp_valid && s.response == OIMGPU_S_OK) {
		c.status = s.status;
		if (s.status != SC_GOOD) {
			c.sense[0] = 0xf0; c.sense[2] = s.sk & 0xf; c.sense[7] = 10;
			c.sense[12] = s.asc; c.sense[13] = 0;
			c.sense_len = OIMGPU_SENSE_SIZE;
		}
		c.resid = s.length - s.data_transferred;
		c.data_transferred = s.data_transferred;
	}
	int4 *o = reinterpret_cast<int4 *>(out);
	o[0] = cz[0]; o[1] = cz[1]; o[2] = cz[2];
}

/* ---- SPC primary commands a guest needs to attach the disk (scsi_bdev.c:188-1265, 1827-2077):
 *      INQUIRY (standard + VPD pages), REPORT LUNS, MODE SENSE 6/10, MODE SELECT 6/10.
 *      Responses are built in the lane's shared-memory scratch and scattered into the SG list. ------ */

__device__ __forceinline__ void d_be16(uint8_t *p, uint32_t v) { p[0] = (uint8_t)(v >> 8); p[1] = (uint8_t)v; }
__device__ __forceinline__ void d_be32(uint8_t *p, uint32_t v) { p[0] = (uint8_t)(v >> 24); p[1] = (uint8_t)(v >> 16); p[2] = (uint8_t)(v >> 8); p[3] = (uint8_t)v; }
__device__ __forceinline__ void d_be64(uint8_t *p, uint64_t v) { d_be32(p, (uint32_t)(v >> 32)); d_be32(p + 4, (uint32_t)v); }
__device__ __forceinline__ int d_strlen(const char *s) { int n = 0; while (s[n]) n++; return n; }

/* spdk_strcpy_pad (S/lib/util/string.c:220-231) */
__device__ __forceinline__ void d_strcpy_pad(uint8_t *dst, const char *src, int size, uint8_t pad)
{
	int i = 0;
	for (; i < size && src[i]; i++) dst[i] = (uint8_t)src[i];
	for (; i < size; i++) dst[i] = pad;
}

/* spdk_bdev_scsi_inquiry (scsi_bdev.c:188-805).  Its alloc_len argument is the size of the staging
 * buffer (>= 4096, scsi_bdev.c:1847-1850), so the short-allocation branches never trigger.
 * Returns the response length in `data` or -1 with the status set. */
__device__ __noinline__ int scsi_inquiry(const LunCtx &L, const uint8_t *cdb, uint8_t *data, LaneState &s)
{
	const int pc = cdb[2], evpd = cdb[1] & 1;
	int hlen = 0, len = 0;
	for (int k = 0; k < 256; k++) data[k] = 0;
	if (!evpd && pc) {
		set_check(s, SK_ILLEGAL_REQUEST, ASC_INVALID_FIELD);
		return -1;
	}
	if (!evpd) {
		/* standard INQUIRY data: all 96 bytes */
		data[2] = 0x05;			/* SPC-3 */
		data[3] = 2 | 1 << 4;		/* response format 2, HISUP */
		data[6] = 0x10;			/* MULTIP */
		data[7] = 0x2;			/* CMDQUE */
		d_strcpy_pad(&data[8], "INTEL", 8, ' ');
		d_strcpy_pad(&data[16], L.product_name, 16, ' ');
		d_strcpy_pad(&data[32], "0001", 4, ' ');
		for (int k = 36; k < 56; k++) data[k] = 0x20;
		d_be16(&data[58], 0x0960); d_be16(&data[60], 0x0300); d_be16(&data[62], 0x0320); d_be16(&data[64], 0x0040);
		data[4] = 96 - 5;		/* additional length */
		return 96;
	}
	uint8_t *params = data + 4;
	data[1] = (uint8_t)pc;
	hlen = 4;
	switch (pc) {
	case 0x00: {
		const uint8_t pages[10] = { 0x00, 0x80, 0x83, 0x85, 0x86, 0x87, 0x88, 0xb0, 0xb1, 0xb2 };
		for (int k = 0; k < 10; k++) params[k] = pages[k];
		len = 10;
		break;
	}
	case 0x80:
		len = d_strlen(L.bdev_name) + 1;
		if (len > 32) len = 32;
		for (int k = 0; k < len - 1; k++) params[k] = (uint8_t)L.bdev_name[k];
		params[len - 1] = 0;
		break;
	case 0x83: {
		uint8_t *buf = params;
		int dl;
#define DESIG(code_set, type, assoc, dlen) do { buf[0] = (uint8_t)((code_set) | L.protocol_id << 4); \
		buf[1] = (uint8_t)((type) | (assoc) << 4 | 1 << 7); buf[2] = 0; buf[3] = (uint8_t)(dlen); } while (0)
		DESIG(1, 3, 0, 8);
		{	/* spdk_bdev_scsi_set_naa_ieee_extended (scsi_bdev.c:78-103) */
			uint8_t *nb = buf + 4;
			int count = 0;
			for (int i = 0; i < 16 && L.bdev_name[i]; i++) {
				int ch = L.bdev_name[i], value;
				if (ch >= '0' && ch <= '9') value = ch - '0';
				else {
					if (ch >= 'A' && ch <= 'Z') ch += 32;
					value = (ch >= 'a' && ch <= 'f') ? ch - 'a' + 10 : ch;
				}
				if (i % 2) nb[count++] |= (uint8_t)(value << 4);
				else nb[count] = (uint8_t)value;
			}
			uint64_t v = 0;
			for (int k = 7; k >= 0; k--) v = v << 8 | nb[k];	/* little-endian load */
			v &= 0x0fff000000ffffffull;
			v |= 0x2000000347000000ull;
			d_be64(nb, v);
		}
		len = 12; buf += 12;
		DESIG(2, 1, 0, 56);
		d_strcpy_pad(buf + 4, "INTEL", 8, ' ');
		d_strcpy_pad(buf + 12, L.product_name, 16, ' ');
		d_strcpy_pad(buf + 28, L.bdev_name, 32, ' ');
		len += 60; buf += 60;
		dl = d_strlen(L.dev_name);
		for (int k = 0; k < dl; k++) buf[4 + k] = (uint8_t)L.dev_name[k];
		do { buf[4 + dl++] = 0; } while (dl & 3);
		DESIG(3, 8, 2, dl);
		len += 4 + dl; buf += 4 + dl;
		dl = d_strlen(L.port_name);
		for (int k = 0; k < dl; k++) buf[4 + k] = (uint8_t)L.port_name[k];
		DESIG(3, 8, 1, dl);
		len += 4 + dl; buf += 4 + dl;
		DESIG(1, 4, 1, 4);
		d_be16(buf + 6, L.port_index);
		len += 8; buf += 8;
		DESIG(1, 5, 1, 4);
		len += 8; buf += 8;
		DESIG(1, 6, 0, 4);
		d_be16(buf + 6, (uint32_t)L.scsi_dev_id);
		len += 8;
#undef DESIG
		break;
	}
	case 0x86:
		data[1] = 0;			/* the reference's memset wipes the page code (scsi_bdev.c:420) */
		data[5] = 0x04 | 0x01;
		len = 60;
		break;
	case 0x85:
		len = 0;
		break;
	case 0x87:
		params[0] = 0x3f; params[1] = 0xff;
		len = 4;
		break;
	case 0x88: {
		const int plen = d_strlen(L.port_name);
		d_be16(params + 2, L.port_index);
		params[14] = 0x05 << 4 | 0x03;
		params[15] = 0x80 | 1 << 4 | 8;
		params[17] = (uint8_t)plen;
		for (int k = 0; k < plen; k++) params[18 + k] = (uint8_t)L.port_name[k];
		d_be16(params + 12, 4 + plen);
		len = 12 + 4 + plen;		/* 14-byte descriptor counted as 12: name cut by 2 (scsi_bdev.c:503-540) */
		break;
	}
	case 0xb0: {
		uint32_t blocks = (1024u * 1024u) / L.block_size;
		data[5] = (uint8_t)(blocks > 0xff ? 0xff : blocks);
		d_be16(&data[6], L.block_size < 4096 ? 4096 / L.block_size : 1);
		blocks = OIMGPU_MAX_XFER_BYTES / L.block_size;
		d_be32(&data[8], blocks);
		d_be32(&data[12], blocks);
		d_be32(&data[20], 4194304);
		d_be32(&data[24], OIMGPU_MAX_UNMAP_DESC);
		d_be64(&data[36], 512);
		len = 60;
		break;
	}
	case 0xb1:
		d_be16(&data[4], 1);
		data[7] = 0x02 << 4;
		len = 60;
		break;
	case 0xb2:
		data[5] = 1 << 7;
		data[6] = 0x02;
		len = 7;
		break;
	default:
		s.data_transferred = 0;
		set_check(s, SK_NO_SENSE, ASC_NONE);
		return -1;
	}
	d_be16(&data[2], (uint32_t)len);
	return hlen + len;
}

/* mode_sense_page_init + spdk_bdev_scsi_mode_sense_page for one (page, subpage) without recursion
 * (scsi_bdev.c:807-1100); cp == nullptr only sizes */
__device__ __forceinline__ int mode_page_one(int pc, int page, int subpage, uint8_t *cp)
{
	int plen;
	switch (page) {
	case 0x01: case 0x07: case 0x1a: case 0x1c: plen = 0x0a + 2; break;
	case 0x02: plen = 0x0e + 2; break;
	case 0x08: plen = 0x12 + 2; break;
	case 0x10: plen = 0x16 + 2; break;
	case 0x0a:
		if (subpage == 0x01) {
			plen = 0x1c + 4;
			if (cp) { for (int k = 0; k < plen; k++) cp[k] = 0; cp[0] = (uint8_t)(page | 0x40); cp[1] = 1; d_be16(&cp[2], plen - 4); }
			return plen;
		}
		plen = 0x0a + 2;
		break;
	default:
		return 0;
	}
	if (subpage != 0) return 0;
	if (cp) {
		for (int k = 0; k < plen; k++) cp[k] = 0;
		cp[0] = (uint8_t)page; cp[1] = (uint8_t)(plen - 2);
		if (page == 0x08 && pc != 0x01) cp[2] |= 0x4 | 0x1;	/* WCE | RCD */
	}
	return plen;
}

__device__ __forceinline__ int mode_pages(int pc, int page, int subpage, uint8_t *cp)
{
	int len = 0;
	if (page == 0x0a && subpage == 0xff) {
		len += mode_page_one(pc, 0x0a, 0x00, cp ? cp + len : nullptr);
		len += mode_page_one(pc, 0x0a, 0x01, cp ? cp + len : nullptr);
		return len;
	}
	if (page == 0x3f) {
		if (subpage == 0x00 || subpage == 0xff) {
			for (int i = 0; i < 0x3e; i++) len += mode_page_one(pc, i, 0x00, cp ? cp + len : nullptr);
		}
		if (subpage == 0xff) {
			/* the second round asks every page for subpage 0xff: only page 0x0a answers (00h + 01h) */
			len += mode_page_one(pc, 0x0a, 0x00, cp ? cp + len : nullptr);
			len += mode_page_one(pc, 0x0a, 0x01, cp ? cp + len : nullptr);
		}
		return len;
	}
	return mode_page_one(pc, page, subpage, cp);
}

/* spdk_bdev_scsi_process_primary (scsi_bdev.c:1827-2077) for INQUIRY / REPORT LUNS / MODE SENSE / MODE SELECT */
__device__ __noinline__ void scsi_primary(const LunCtx &L, const QueueDesc &q, const oimgpu_req &r, uint32_t cnt,
					  uint32_t len, LaneState &s)
{
	const uint8_t *cdb = r.cdb;
	uint8_t *data = s.scratch;
	int rc = 0, data_len = -1, alloc_len = -1;

	switch (cdb[0]) {
	case 0x12:
		alloc_len = be16(&cdb[3]);
		rc = scsi_inquiry(L, cdb, data, s);
		data_len = rc;
		break;
	case 0xa0:
		alloc_len = (int)be32(&cdb[6]);
		if (alloc_len < 16) { set_check(s, SK_ILLEGAL_REQUEST, ASC_INVALID_FIELD); rc = -1; break; }
		if (cdb[2] > 0x02) { set_check(s, SK_NO_SENSE, ASC_NONE); rc = -1; break; }
		for (int k = 0; k < 16; k++) data[k] = 0;
		d_be32(data, 8);		/* one LUN, id 0, flat addressing (scsi_bdev.c:105-172) */
		rc = data_len = 16;
		break;
	case 0x15: case 0x55: {
		const int md = cdb[0] == 0x15 ? 4 : 8;
		const int pllen = cdb[0] == 0x15 ? cdb[4] : be16(&cdb[7]);
		if (pllen == 0) break;
		if (pllen < md || (int)len < md) { set_check(s, SK_ILLEGAL_REQUEST, ASC_INVALID_FIELD); rc = -1; break; }
		/* spdk_bdev_scsi_mode_select_page walks the pages and applies nothing (scsi_bdev.c:1176-1265) */
		rc = pllen;
		data_len = 0;
		break;
	}
	case 0x1a: case 0x5a: {
		int md, llba = 0;
		if (cdb[0] == 0x1a) { alloc_len = cdb[4]; md = 6; }
		else { alloc_len = be16(&cdb[7]); llba = !!(cdb[1] & 0x10); md = 10; }
		const int dbd = !!(cdb[1] & 0x8), pc = (cdb[2] & 0xc0) >> 6, page = cdb[2] & 0x3f, subpage = cdb[3];
		if (pc == 3) { set_check(s, SK_ILLEGAL_REQUEST, 0x39); rc = -1; break; }	/* SAVING PARAMETERS NOT SUPPORTED */
		const int hlen = md == 6 ? 4 : 8;
		const int blen = dbd ? 0 : (md == 6 ? 8 : (llba ? 16 : 8));
		for (int k = 0; k < 256; k++) data[k] = 0;
		const int plen = mode_pages(pc, page, subpage, data + hlen + blen);
		const int total = hlen + blen + plen;
		if (hlen == 4) { data[0] = (uint8_t)(total - 1); data[3] = (uint8_t)blen; }
		else { d_be16(&data[0], total - 2); data[4] = llba ? 1 : 0; d_be16(&data[6], blen); }
		if (blen == 16) { d_be64(&data[hlen], L.num_blocks); d_be32(&data[hlen + 12], L.block_size); }
		else if (blen == 8) {
			d_be32(&data[hlen], L.num_blocks > 0xffffffffULL ? 0xffffffffu : (uint32_t)L.num_blocks);
			d_be32(&data[hlen + 4], L.block_size);
		}
		rc = data_len = total;
		break;
	}
	default:
		return;
	}
	if (rc >= 0 && data_len > 0) {
		/* the scatter may fail (SG list shorter than the data) without changing the outcome (scsi_bdev.c:2060-2069) */
		scatter_small(q, r, cnt, len, data, alloc_len < data_len ? alloc_len : data_len, s);
		rc = data_len < alloc_len ? data_len : alloc_len;
	}
	if (rc >= 0) {
		s.data_transferred = rc;
		s.status = SC_GOOD;
	}
}

/* ---- virtqueue mode: the split-ring walk of the reference's poller on one parser lane ---------- */

__device__ __forceinline__ uint32_t ld_vol32(const volatile void *p)
{
	uint32_t r;
	asm volatile("ld.volatile.global.u32 %0, [%1];" : "=r"(r) : "l"(p) : "memory");
	return r;
}
__device__ __forceinline__ uint64_t globaltimer_ns()
{
	uint64_t t;
	asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
	return t;
}

__device__ __forceinline__ void st_vol32(volatile void *p, uint32_t v)
{
	asm volatile("st.volatile.global.u32 [%0], %1;" :: "l"(p), "r"(v) : "memory");
}

__device__ __forceinline__ uint16_t ld_vol16(const void *p)
{
	uint16_t r;
	asm volatile("ld.volatile.global.u16 %0, [%1];" : "=h"(r) : "l"(p) : "memory");
	return r;
}

/* rte_vhost_gpa_to_vva (rte_vhost.h:133-150): first region containing gpa, no length check */
__device__ __forceinline__ uint64_t gpa_to_dev(const LunCtx &L, uint64_t gpa)
{
	for (uint32_t i = 0; i < L.nregions; i++) {
		if (gpa >= L.region[i].gpa && gpa < L.region[i].gpa + L.region[i].size) return gpa - L.region[i].gpa + L.region[i].addr;
	}
	return 0;
}

/* spdk_vhost_gpa_to_vva (vhost.c:93-106): the whole [gpa, gpa+len) must lie inside one region */
__device__ __forceinline__ uint64_t gpa_to_dev_len(const LunCtx &L, uint64_t gpa, uint64_t len)
{
	for (uint32_t i = 0; i < L.nregions; i++) {
		if (gpa >= L.region[i].gpa && gpa < L.region[i].gpa + L.region[i].size) {
			if (len > L.region[i].gpa + L.region[i].size - gpa) return 0;
			return gpa - L.region[i].gpa + L.region[i].addr;
		}
	}
	return 0;
}

struct VDesc { uint64_t addr; uint32_t len; uint16_t flags, next; };	/* struct vring_desc */
enum : uint16_t { VD_NEXT = 1, VD_WRITE = 2, VD_INDIRECT = 4 };

__device__ __forceinline__ VDesc decode_desc(const int4 v)
{
	VDesc d;
	d.addr = (uint64_t)(uint32_t)v.x | (uint64_t)(uint32_t)v.y << 32;
	d.len = (uint32_t)v.z;
	d.flags = (uint16_t)((uint32_t)v.w & 0xffff);
	d.next = (uint16_t)((uint32_t)v.w >> 16);
	return d;
}

__device__ __forceinline__ VDesc load_desc(const uint8_t *p)
{
	VDesc d;
	if (((uintptr_t)p & 15) == 0) {
		d = decode_desc(ld_cg16(p));
	} else {
		uint64_t a = 0; uint32_t l = 0, w = 0;
		for (int k = 7; k >= 0; k--) a = a << 8 | ld_cg8(p + k);
		for (int k = 11; k >= 8; k--) l = l << 8 | ld_cg8(p + k);
		for (int k = 15; k >= 12; k--) w = w << 8 | ld_cg8(p + k);
		d.addr = a; d.len = l; d.flags = (uint16_t)(w & 0xffff); d.next = (uint16_t)(w >> 16);
	}
	return d;
}

/* spdk_vhost_vring_desc_get_next (vhost.c:433-453): 0 = ok (have == false: end of chain), -1 = bad index */
__device__ __forceinline__ int desc_get_next(VDesc &d, bool &have, const uint8_t *table, uint32_t table_size)
{
	if ((d.flags & VD_NEXT) == 0) { have = false; return 0; }
	if (d.next >= table_size) { have = false; return -1; }
	d = load_desc(table + (size_t)d.next * 16);
	return 0;
}

/* spdk_vhost_vring_desc_to_iov (vhost.c:461-509): append the iovecs of one descriptor to the lane's
 * scratch SG row; split only where two sides of a 2 MiB boundary are not contiguous in device VA */
__device__ __forceinline__ int desc_to_iov(const LunCtx &L, oimgpu_iov *row, oimgpu_iov *srow, uint32_t &iov_index, const VDesc &d)
{
	const uint64_t MB2 = 2ull << 20;
	uint32_t remaining = d.len;
	uint64_t payload = d.addr;
	do {
		if (iov_index >= OIMGPU_IOVS_MAX) return -1;
		const uint64_t vva = gpa_to_dev(L, payload);
		if (vva == 0) return -1;
		const uint32_t to_boundary = (uint32_t)(MB2 - (payload & (MB2 - 1)));
		uint32_t len;
		if (remaining <= to_boundary) {
			len = remaining;
		} else {
			len = to_boundary;
			while (len < remaining) {
				if (vva + len != gpa_to_dev(L, payload + len)) break;
				len += (remaining - len) < MB2 ? (remaining - len) : (uint32_t)MB2;
			}
		}
		oimgpu_iov v;
		v.addr = vva; v.len = len; v.flags = 0;
		row[iov_index] = v;
		if (iov_index < (uint32_t)kSmemIovs) srow[iov_index] = v;	/* short lists are read back from shared memory */
		remaining -= len;
		payload += len;
		iov_index++;
	} while (remaining);
	return 0;
}

/* task_data_setup (vhost_scsi.c:490-624) for the chain starting at ring index `head`.  Fills the
 * request slot `r` (virtio header + direction + SG row reference) and *resp (device address of the
 * guest's response buffer).  Returns false for every `goto invalid_task`. */
__device__ __noinline__ bool vq_task_data_setup(const LunCtx &L, const QueueDesc &q, uint32_t head, VDesc d, oimgpu_req &r,
						oimgpu_iov *row, oimgpu_iov *srow, uint32_t row_index, uint64_t *resp)
{
	*resp = 0;
	/* spdk_vhost_vq_get_desc (vhost.c:219-247); `d` = desc[head], loaded one pass ahead by the caller */
	if (head >= q.vq_size) return false;
	const uint8_t *table = q.vq_desc;
	uint32_t table_size = q.vq_size;
	if (d.flags & VD_INDIRECT) {
		table_size = d.len / 16;
		/* a table shorter than one descriptor: the reference reads 16 bytes it never checked; out of
		 * bounds for us means a fault that takes the whole session down, so the chain is invalid */
		if (table_size == 0) return false;
		table = (const uint8_t *)(uintptr_t)gpa_to_dev_len(L, d.addr, 16ull * table_size);
		if (table == nullptr) return false;
		d = load_desc(table);
	}
	/* first descriptor: readable, holds a whole virtio_scsi_cmd_req */
	if ((d.flags & VD_WRITE) || d.len < 51) return false;
	const uint8_t *req = (const uint8_t *)(uintptr_t)gpa_to_dev_len(L, d.addr, 51);
	if (req == nullptr) return false;
	uint8_t *rb = reinterpret_cast<uint8_t *>(&r);
	if (((uintptr_t)req & 3) == 0) {
		for (int k = 0; k < 12; k++) reinterpret_cast<uint32_t *>(rb)[k] = ld_cg32(req + 4 * k);
		for (int k = 48; k < 51; k++) rb[k] = ld_cg8(req + k);
	} else {
		for (int k = 0; k < 51; k++) rb[k] = ld_cg8(req + k);
	}
	bool have = true;
	desc_get_next(d, have, table, table_size);
	if (!have) return false;	/* neither payload nor response buffer */
	const bool from_dev = (d.flags & VD_WRITE) != 0;
	uint32_t iovcnt = 0;
	if (from_dev) {
		/* FROM_DEV: [RD_req][WR_resp][WR_buf0]...[WR_bufN] */
		*resp = gpa_to_dev_len(L, d.addr, OIMGPU_RESP_SIZE);
		if (d.len < OIMGPU_RESP_SIZE || *resp == 0) return false;
		if (desc_get_next(d, have, table, table_size) != 0) return false;
		while (have) {
			if (!(d.flags & VD_WRITE)) return false;
			if (desc_to_iov(L, row, srow, iovcnt, d)) return false;
			if (desc_get_next(d, have, table, table_size) != 0) return false;
		}
	} else {
		/* TO_DEV: [RD_req][RD_buf0]...[RD_bufN][WR_resp] */
		while (!(d.flags & VD_WRITE)) {
			if (desc_to_iov(L, row, srow, iovcnt, d)) return false;
			desc_get_next(d, have, table, table_size);
			if (!have) return false;	/* no response descriptor */
		}
		*resp = gpa_to_dev_len(L, d.addr, OIMGPU_RESP_SIZE);
		if (d.len < OIMGPU_RESP_SIZE || *resp == 0) return false;
	}
	r.dir = from_dev ? OIMGPU_DIR_FROM_DEV : OIMGPU_DIR_TO_DEV;
	r.iovcnt = (uint16_t)iovcnt;	/* 0 with from_dev == the reference's "no payload" task (iovcnt 1, len 0) */
	r.flags = 0;
	r.iov_start = row_index;
	r.reserved = 0;
	return true;
}

#ifndef OIM_IDLE_NS
#define OIM_IDLE_NS 500
#endif

/* hazard signature: which bit a 4 KiB granule of device address space maps to */
__device__ __forceinline__ uint32_t sig_index(uint64_t granule)
{
	return (uint32_t)(((uint32_t)granule ^ (uint32_t)(granule >> 20)) * 0x9E3779B1u) >> (32 - OIM_SIG_LOG2);
}
static_assert(kSigBits == 1 << OIM_SIG_LOG2, "sig_index produces OIM_SIG_LOG2 bits");

/* ---- the kernel ----------------------------------------------------------------------------- */

/* one lane: the ring cursors back into VqState - a virtqueue's avail and used index (16 significant bits), a slot
 * ring's consumed position */
__device__ __forceinline__ void store_cursors(VqState *vs, bool vring, uint32_t last_avail, uint32_t last_used)
{
	if (vring) {
		vs->last_avail = last_avail & 0xffff;
		vs->last_used = last_used & 0xffff;
	} else {
		vs->last_avail = last_avail;
	}
}

/* parser side: publish the completions of the fill that occupied `st` (all movers are done with it) */
/* pub_q / pub_end (shared kernels): the queue and end position this CTA published last - a fill that starts right
 * there has nothing of anybody else's to wait for */
__device__ __forceinline__ void reap_stage(Stage &st, int lane, QShare **pub_q = nullptr, uint32_t *pub_end = nullptr)
{
	const bool follows_own = pub_q && st.share && *pub_q == st.share && *pub_end == st.share_pos;
	const uint32_t n = st.ncpl;
	if (st.mode == QMODE_SLOTS) {
		for (uint32_t v = lane; v < n * 3; v += 32) {
			const uint32_t slot = (st.cpl_slot0 + v / 3) & st.cpl_mask;
			st_cg16(reinterpret_cast<int4 *>(&st.cpl_ring[slot]) + v % 3,
				reinterpret_cast<const int4 *>(&st.cpl[v / 3])[v % 3]);
		}
		if (st.share) {
			/* shared queue: the completion counter the host polls must stay monotonic, and `done` is what a
			 * writer of another CTA waits on, so fills publish in ring order */
			if (lane == 0 && !follows_own) chain_wait(&st.share->done, st.share_pos);
			__syncwarp();
		}
		if (st.done) {
			/* persistent mode: make payload + records visible to the host, then bump the counter it polls */
			__threadfence_system();
			__syncwarp();
			if (lane == 0 && n) *st.done = st.cpl_slot0 + n;
		}
		if (st.share) {
			__syncwarp();
			if (lane == 0) {
				st_release32(&st.share->done, st.share_pos + n);	/* releases the records written by the whole warp */
				if (pub_q) { *pub_q = st.share; *pub_end = st.share_pos + n; }
			}
		}
		return;
	}
	/* virtqueue mode: spdk_vhost_scsi_task_cpl writes into the guest's response buffer
	 * (vhost_scsi.c:311-331), then spdk_vhost_vq_used_ring_enqueue publishes {id, len} (vhost.c:397-431) */
	if ((uint32_t)lane < n) {
		const oimgpu_cpl &c = st.cpl[lane];
		uint8_t *resp = (uint8_t *)(uintptr_t)st.resp[lane];
		if (c.resp_valid && resp) {
			resp[11] = c.response;
			if (c.response == OIMGPU_S_OK) {
				resp[10] = c.status;
				if (c.status != SC_GOOD) {
					for (int k = 0; k < OIMGPU_SENSE_SIZE; k++) resp[12 + k] = c.sense[k];
					resp[0] = (uint8_t)c.sense_len; resp[1] = 0; resp[2] = 0; resp[3] = 0;
				}
				resp[4] = (uint8_t)c.resid; resp[5] = (uint8_t)(c.resid >> 8);
				resp[6] = (uint8_t)(c.resid >> 16); resp[7] = (uint8_t)(c.resid >> 24);
			}
		}
		const uint32_t slot = (st.used_base + lane) & (st.vq_size - 1);
		uint32_t *ue = reinterpret_cast<uint32_t *>(st.vq_used + 4 + 8 * (size_t)slot);
		ue[0] = st.vq_head[lane];
		ue[1] = c.used_len;
	}
	/* "Ensure the used ring is updated before we ... increment used->idx" (vhost.c:416-417).  Guest memory in
	 * host RAM needs that at system scope (the guest's CPUs are watching); when the guest image lives in HBM
	 * the observers are on this GPU and the cheaper scope does */
	if (st.share) {
		/* used->idx moves in ring order: wait for the fills before this one (other CTAs') to publish theirs */
		if (lane == 0 && !follows_own) chain_wait(&st.share->done, st.share_pos);
		__syncwarp();
	}
	if (st.vq_in_hbm) __threadfence();
	else __threadfence_system();
	__syncwarp();
	if (lane == 0 && n) *reinterpret_cast<volatile uint16_t *>(st.vq_used + 2) = (uint16_t)(st.used_base + n);
	if (st.share && lane == 0) {
		if (!st.persistent && st.share_pos + n == st.share_final) {
			/* last fill of this launch on the queue: everything before it is published - write the cursors back */
			store_cursors(st.vq_state, true, st.share->base_avail + st.share_final, st.used_base + n);
		}
		st_release32(&st.share->done, st.share_pos + n);
		if (pub_q) { *pub_q = st.share; *pub_end = st.share_pos + n; }
	}
}

/* mirrored bdev (config 5): the same bytes go to every replica in one step - local HBM and, by P2P
 * stores over NVLink, the peers.  Replica 1 shares the loaded registers with the local store (one load,
 * two stores).  Out of line so that it does not weigh on the plain mover loop's registers. */
static __device__ __forceinline__ void mirror_unit(const LunCtx &L, uint8_t *dst, const uint8_t *src, uint64_t off,
						uint32_t nbytes, int lane, uint32_t nrep)
{
	const uint64_t soff = (uint64_t)(dst - L.store[0]) + off;
	if (src) move_unit<true>(dst + off, src + off, nbytes, lane, L.store[1] + soff);
	else { zero_unit(dst + off, nbytes, lane); zero_unit(L.store[1] + soff, nbytes, lane); }
	for (uint32_t rep = 2; rep < nrep; rep++) {
		if (src) move_unit<true>(L.store[rep] + soff, src + off, nbytes, lane);
		else zero_unit(L.store[rep] + soff, nbytes, lane);
	}
}

/* ---- queue positions ----------------------------------------------------------------------------------- */

/* a queue's producer index: the host's tail doorbell (slot ring), the guest's avail->idx (virtqueue), or the
 * dispatcher's mirror of either (hinted) */
__device__ __forceinline__ uint32_t producer_index(const QueueDesc &q, bool hinted)
{
	if (hinted) return ld_vol32(&q.vq_state->hint);
	return q.mode == QMODE_VRING ? (uint32_t)ld_vol16(q.vq_avail + 2) : ld_vol32(q.doorbell);
}

/* new entries on a virtqueue from ring position `from` up to avail index `idx` (16-bit arithmetic); 0 when there are
 * more than the ring holds: "the queue is unrecoverably broken" */
__device__ __forceinline__ uint32_t vq_new_entries(uint32_t idx, uint32_t from, uint32_t vq_size)
{
	const uint32_t k = (uint16_t)(idx - from);
	return k > vq_size ? 0 : k;
}

/* one lane: the avail entry at ring position pos, i.e. the head of a request's chain.  Volatile, as every avail entry
 * read: a resident CTA has this line in its L1 from the batch before, when the guest had not written it yet */
__device__ __forceinline__ uint32_t vq_avail_entry(const QueueDesc &q, uint32_t pos)
{
	return reinterpret_cast<const volatile uint16_t *>(q.vq_avail + 4)[pos & (q.vq_size - 1)];
}

/* a lane whose request moves nothing: no request in this pass, or an invalid one */
__device__ __forceinline__ void lane_reset(LaneState &s)
{
	s.op = OP_NONE; s.nseg = 0; s.units = 0; s.hazard = 0; s.valid = 0; s.store_lo = s.store_hi = 0;
}

/* ---- shared queues: who takes which pass --------------------------------------------------------------- */

/* lane 0: take the next pass (<= 32 requests) of a shared queue.  Returns its length (0: nothing unclaimed right
 * now) and its position in *pos.  q.head = ring position of position 0; q.count = the launch's limit. */
__device__ __forceinline__ uint32_t claim_pass(const QueueDesc &q, QShare *qs, bool persistent, bool hinted, uint32_t *pos,
					       uint32_t want = kPass)
{
	for (;;) {
		const uint32_t c = ld_vol32(&qs->claim);
		uint32_t avail;
		if (!persistent) avail = q.count - c;
		else if (q.mode == QMODE_VRING) avail = vq_new_entries(producer_index(q, hinted), q.head + c, q.vq_size);
		else avail = producer_index(q, hinted) - (q.head + c);
		if (avail == 0) return 0;
		const uint32_t n = avail < want ? avail : want;
		if (atomicCAS(&qs->claim, c, c + n) == c) {
			*pos = c;
			return n;
		}
	}
}

/* one lane, one queue: is there something to claim?  A CTA that is not at home on the queue stays away while the
 * queue is being written: passes of different CTAs are ordered coarsely (see QShare), two CTAs alternating on a
 * write-heavy queue would mostly wait for each other, and its home CTA serves it at the exclusive path's speed. */
__device__ __forceinline__ bool shared_queue_has_work(const QueueDesc &q, QShare &qs, bool persistent, bool hinted, bool home)
{
	const uint32_t c = ld_vol32(&qs.claim);
	if (!home) {
		const uint32_t we = (uint32_t)(ld_vol64(&qs.chain) >> 32);	/* end of the last pass that wrote */
		if (we != 0 && c - we < 8192u) return false;
	}
	if (!persistent) {
		if (q.mode == QMODE_VRING) {
			if (ld_vol32(&qs.latched) != 1u) return true;	/* nobody has looked at avail->idx yet */
			return c < ld_vol32(&qs.count);
		}
		return c < q.count;
	}
	const uint32_t ring = ld_vol32(&qs.base_avail) + c;
	if (q.mode == QMODE_VRING) return vq_new_entries(producer_index(q, hinted), ring, q.vq_size) != 0;
	return producer_index(q, hinted) != ring;
}

/* warp-wide: first queue with unclaimed work in cyclic order from `from` (0xffffffff: none), 32 queues per step */
__device__ __forceinline__ uint32_t find_shared_work(const KickHeader *hdr, const QueueDesc *queues, QShare *shares, uint32_t nq,
						      uint32_t nworkers, uint32_t from, bool persistent, bool hinted, int lane)
{
	for (uint32_t base = 0; base < nq; base += 32) {
		const uint32_t k = base + lane;
		bool has = false;
		uint32_t qi = 0;
		if (k < nq) {
			qi = from + k;
			if (qi >= nq) qi -= nq;
			has = shared_queue_has_work(queues[qi], shares[qi], persistent, hinted, qi % nworkers == blockIdx.x);
		}
		const uint32_t m = __ballot_sync(0xffffffffu, has);
		if (m) return __shfl_sync(0xffffffffu, qi, __ffs(m) - 1);
	}
	return 0xffffffffu;
}

#ifndef OIM_MIN_BLOCKS
#define OIM_MIN_BLOCKS 2	/* 128 registers: the mover loop must stay spill-free (a lower register cap spills it) */
#endif

/* every mover has finished fill f (a mover arrives on `empty` only after finishing its share of all earlier fills too) */
__device__ __forceinline__ void wait_fill_moved(CtaShared &sh, uint32_t f)
{
	mbar_wait(&sh.empty[f % kStages], (f / kStages) & 1);
}

/* ---- the dispatcher CTA (see KickHeader) --------------------------------------------------------------- */

/* one warp: mirror every queue's doorbell into VqState::hint, and the stop flag into stop_mirror */
__device__ __forceinline__ void dispatcher_cta(KickHeader *hdr, const QueueDesc *queues, int lane)
{
	const uint32_t nq = hdr->nqueues;
	uint64_t last_change = globaltimer_ns();
	for (;;) {
		bool changed = false;
		for (uint32_t base = 0; base < nq; base += 32) {
			const uint32_t qi = base + lane;
			if (qi < nq) {
				const QueueDesc &q = queues[qi];
				const uint32_t v = q.mode == QMODE_VRING ? (uint32_t)ld_vol16(q.vq_avail + 2) : ld_vol32(q.doorbell);
				if (v != ld_vol32(&q.vq_state->hint)) {
					st_vol32(&q.vq_state->hint, v);
					changed = true;
				}
			}
		}
		changed = __any_sync(0xffffffffu, changed);
		uint32_t quit = 0;
		if (lane == 0) {
			const uint64_t now = globaltimer_ns();
			if (changed) last_change = now;
			quit = ld_vol32(hdr->stop) != 0;
			if (!quit && hdr->idle_timeout_ms && now - last_change > (uint64_t)hdr->idle_timeout_ms * 1000000ull) quit = 1;
			if (quit) st_vol32(&hdr->stop_mirror, 1u);
		}
		if (__shfl_sync(0xffffffffu, quit, 0)) break;
	}
	if (lane == 0) {
		__threadfence_system();
		atomicAdd_system(const_cast<uint32_t *>(hdr->exited), 1u);
	}
}

/* ---- parser: one pass ---------------------------------------------------------------------------------- */

struct PassHazards {
	uint32_t writers, touching;	/* lane masks of the pass: haz >= 2, haz != 0 */
	uint32_t drain;			/* 0 = none, d = fill c-d must be finished before flagged units move */
	bool cross;			/* this lane's request is one of the conflicting ones */
	bool mydense;			/* its range is too large (or a barrier) for the signatures */
	bool wcollide;			/* a writer found one of its granules already written in this pass */
	uint64_t g0, g1;		/* its first and last 4 KiB granule */
};

/* Hazards against the passes whose movers may still be running.  The history ring hist[] keeps the store ranges of
 * the previous kStages-1 passes per lane: movers are not in lock-step, one may already work on pass p+2 while another
 * is still in pass p (the stage ring only stops the parser from refilling pass p's stage).  The segments of a request
 * that conflicts with one of them are flagged; a mover that reaches a flagged unit first waits until the conflicting
 * fill is finished, everything else in the pass proceeds at once.  (Waiting for fill c-d's `empty` barrier covers all
 * older ones too.)  Records this pass in hist[pass_no % kStages]. */
__device__ __forceinline__ PassHazards cross_pass_hazards(HazPass *hist, uint32_t pass_no, uint32_t haz, uint64_t lo, uint64_t hi, int lane)
{
	constexpr int kHist = kStages - 1;
	PassHazards r;
	r.drain = 0;
	r.cross = false;
	r.writers = __ballot_sync(0xffffffffu, haz >= 2);
	r.touching = __ballot_sync(0xffffffffu, haz != 0);
	HazPass &cur = hist[pass_no % kStages];
	/* a read-only stream never needs signatures: while neither this pass nor the ones it could be compared with
	 * contain a writer, the pass is left unsigned (= "dense": whoever meets it later falls back to the exact ranges) */
	bool sign = r.writers != 0;
#pragma unroll
	for (int h = 1; h <= kHist; h++) {
		if ((uint32_t)h <= pass_no) sign |= hist[(pass_no - h) % kStages].writers != 0;
	}
	if (sign) {
		for (int k = lane; k < kSigWords; k += 32) { cur.sig_r[k] = 0; cur.sig_w[k] = 0; }
	}
	cur.lo[lane] = lo;
	cur.hi[lane] = hi;
	cur.haz[lane] = (uint8_t)haz;
	if (lane == 0) { cur.writers = r.writers; cur.touching = r.touching; cur.dense = sign ? 0 : 1; }
	__syncwarp();
	r.g0 = lo >> 12;
	r.g1 = haz ? (hi - 1) >> 12 : r.g0;
	r.mydense = haz == 3 || (haz && r.g1 - r.g0 >= (uint64_t)kSigMaxGranules);
	r.wcollide = false;
	if (!sign) { /* nothing to publish */ }
	else if (r.mydense) cur.dense = 1;
	else if (haz) {
		for (uint64_t g = r.g0; g <= r.g1; g++) {
			const uint32_t idx = sig_index(g);
			if (haz >= 2) r.wcollide |= (atomicOr(&cur.sig_w[idx >> 5], 1u << (idx & 31)) >> (idx & 31)) & 1u;
			else atomicOr(&cur.sig_r[idx >> 5], 1u << (idx & 31));
		}
	}
	__syncwarp();
	/* against the kStages-1 passes before this one: signature first, exact ranges only for the requests the signature
	 * cannot clear */
#pragma unroll
	for (int h = kHist; h >= 1; h--) {
		if ((uint32_t)h > pass_no) continue;
		const HazPass &pp = hist[(pass_no - h) % kStages];
		const uint32_t candidates = haz >= 2 ? pp.touching : haz ? pp.writers : 0u;
		bool maybe = false;
		if (candidates) {
			if (r.mydense || pp.dense) maybe = true;
			else {
				for (uint64_t g = r.g0; g <= r.g1; g++) {
					const uint32_t idx = sig_index(g);
					uint32_t word = pp.sig_w[idx >> 5];
					if (haz >= 2) word |= pp.sig_r[idx >> 5];
					maybe |= (word >> (idx & 31)) & 1u;
				}
			}
		}
		bool hit = false;
		if (maybe) {
			uint32_t scan = candidates;
			while (scan) {
				const int j = __ffs(scan) - 1;
				scan &= scan - 1;
				if (haz == 3 || pp.haz[j] == 3 || (lo < pp.hi[j] && pp.lo[j] < hi)) hit = true;
			}
		}
		r.cross |= hit;
		if (__any_sync(0xffffffffu, hit)) r.drain = (uint32_t)h;	/* nearest pass wins */
	}
	return r;
}

/* Hazards inside the pass -> waves.  Writers are visited in ring order; a writer is pushed behind every earlier
 * request it overlaps, every later overlapping request behind the writer.  Most passes have no overlap at all: the
 * signatures say so.  Returns this lane's wave and the pass's number of waves in nwaves. */
__device__ __forceinline__ uint16_t assign_waves(const HazPass &cur, const PassHazards &hz, uint32_t haz, uint64_t lo, uint64_t hi,
						 int lane, uint32_t &nwaves)
{
	uint16_t wave = 0;
	nwaves = 1;
	bool inpass = false;
	if (hz.writers && (hz.touching & (hz.touching - 1)) && haz) {
		if (hz.mydense || cur.dense) inpass = true;
		else if (haz >= 2) {
			inpass = hz.wcollide;
			for (uint64_t g = hz.g0; g <= hz.g1; g++) {
				const uint32_t idx = sig_index(g);
				inpass |= (cur.sig_r[idx >> 5] >> (idx & 31)) & 1u;
			}
		} else {
			for (uint64_t g = hz.g0; g <= hz.g1; g++) {
				const uint32_t idx = sig_index(g);
				inpass |= (cur.sig_w[idx >> 5] >> (idx & 31)) & 1u;
			}
		}
	}
	if (!__any_sync(0xffffffffu, inpass)) return wave;
	uint32_t w = hz.writers;
	while (w) {
		const int j = __ffs(w) - 1;
		w &= w - 1;
		const uint64_t jlo = __shfl_sync(0xffffffffu, lo, j);
		const uint64_t jhi = __shfl_sync(0xffffffffu, hi, j);
		const uint32_t jhaz = __shfl_sync(0xffffffffu, haz, j);
		const bool overlap = haz != 0 && lane != j &&
			(jhaz == 3 || haz == 3 || (lo < jhi && jlo < hi));
		uint32_t need = (overlap && lane < j) ? (uint32_t)wave + 1 : 0;
		need = __reduce_max_sync(0xffffffffu, need);
		if (lane == j && need > wave) wave = (uint16_t)need;
		const uint32_t jw = __shfl_sync(0xffffffffu, (uint32_t)wave, j);
		if (overlap && lane > j && jw + 1 > wave) wave = (uint16_t)(jw + 1);
	}
	nwaves = __reduce_max_sync(0xffffffffu, (uint32_t)wave) + 1;
	return wave;
}

/* counters for get_bdevs_iostat, per parser lane; one atomic per counter per CTA when the parser leaves */
struct IoStats {
	uint32_t rd = 0, wr = 0, um = 0, er = 0;
	uint32_t mix_r = 0, mix_w = 0;		/* good reads / writes + unmaps of ANY target: the session's mix */
	unsigned long long rb = 0, wb = 0, ub = 0;

	/* good: the request completed with GOOD status */
	__device__ __forceinline__ void count(const LunCtx &L, const LaneState &s, bool active, bool good)
	{
		const bool own = !good || s.tgt == L.target;	/* failures are booked on the session's device */
		const bool ok = good && own;
		rd += __popc(__ballot_sync(0xffffffffu, ok && s.op == OP_READ));
		wr += __popc(__ballot_sync(0xffffffffu, ok && s.op == OP_WRITE));
		/* UNMAP reaches the bdev once per applied descriptor, whatever the command's final status */
		const bool unmapped = active && s.resp_valid && s.response == OIMGPU_S_OK && s.op == OP_UNMAP && s.tgt == L.target;
		um += __reduce_add_sync(0xffffffffu, unmapped ? s.nseg : 0u);
		if (unmapped) ub += s.unmap_bytes;
		er += __popc(__ballot_sync(0xffffffffu, active && !good));
		mix_r += __popc(__ballot_sync(0xffffffffu, good && s.op == OP_READ));
		mix_w += __popc(__ballot_sync(0xffffffffu, good && (s.op == OP_WRITE || s.op == OP_UNMAP)));
		if (ok && s.op == OP_READ) rb += s.length;
		if (ok && s.op == OP_WRITE) wb += s.length;
		if (active && s.resp_valid && s.response == OIMGPU_S_OK && s.tgt != L.target &&
		    ((good && (s.op == OP_READ || s.op == OP_WRITE)) || s.op == OP_UNMAP)) {
			/* another device of the controller: book it there (rare path, plain atomics) */
			LunCtx *P = L.peer[s.tgt];
			if (s.op == OP_UNMAP) {
				if (s.nseg) { atomicAdd(&P->stats[2], (unsigned long long)s.nseg); atomicAdd(&P->stats[6], (unsigned long long)s.unmap_bytes); }
			} else {
				const int k = s.op == OP_READ ? 0 : 1;
				atomicAdd(&P->stats[k], 1ull);
				atomicAdd(&P->stats[4 + k], (unsigned long long)s.length);
			}
		}
	}

	/* every fill is retired: mover warp 0 is done adding to sh.lat_ns */
	__device__ __forceinline__ void flush(LunCtx *lun, const CtaShared &sh, int lane)
	{
		for (int o = 16; o; o >>= 1) {
			rb += __shfl_xor_sync(0xffffffffu, rb, o);
			wb += __shfl_xor_sync(0xffffffffu, wb, o);
			ub += __shfl_xor_sync(0xffffffffu, ub, o);
		}
		if (lane != 0) return;
		if (ub) atomicAdd(&lun->stats[6], ub);
		if (rd) { atomicAdd(&lun->stats[0], (unsigned long long)rd); atomicAdd(&lun->stats[4], rb); }
		if (wr) { atomicAdd(&lun->stats[1], (unsigned long long)wr); atomicAdd(&lun->stats[5], wb); }
		if (um) atomicAdd(&lun->stats[2], (unsigned long long)um);
		if (er) atomicAdd(&lun->stats[7], (unsigned long long)er);
		if (mix_r) atomicAdd(&lun->mix[0], (unsigned long long)mix_r);
		if (mix_w) atomicAdd(&lun->mix[1], (unsigned long long)mix_w);
		for (int t = 0; t < OIMGPU_CTRLR_MAX_DEVS; t++) {
			LunCtx *T = (t == lun->target) ? lun : lun->peer[t];
			for (int k = 0; k < 3 && T; k++) {
				if (sh.lat_ns[t][k]) atomicAdd(&T->stats[8 + k], sh.lat_ns[t][k]);
			}
		}
	}
};

/* ---- movers -------------------------------------------------------------------------------------------- */

/* the fill a mover warp works through */
struct MoverFill {
	const Stage &st;
	uint32_t nseg, nunits, nw;

	/* the segment that holds unit u: the last one with first_unit <= u */
	__device__ __forceinline__ const Segment &seg_of(uint32_t u) const
	{
		uint32_t lo = u, hi = nseg;
		/* as many units as segments: segment u IS unit u.  Taken for passes of small requests (the 4 KiB case); long
		 * SG lists of single pages keep the search - the lookup's latency spreads the movers' loads there */
		if (nunits != nseg || nseg > (uint32_t)kPass) {
			lo = 0;
			while (hi - lo > 1) {
				const uint32_t mid = (lo + hi) >> 1;
				if (st.seg[mid].first_unit <= u) lo = mid; else hi = mid;
			}
		}
		return st.seg[lo];
	}
};

/* the unit a mover warp takes after u: every kMovers-th, or (dyn) the next one from the fill's counter */
__device__ __forceinline__ uint32_t next_unit(Stage &st, bool dyn, uint32_t u, int lane)
{
	if (!dyn) return u + kMovers;
	uint32_t v = 0;
	if (lane == 0) v = atomicAdd(&st.unit_ctr, 1u);
	return __shfl_sync(0xffffffffu, v, 0);
}

/* Unit u of segment g: mirror fan-out, zero fill, aligned copy, or a byte-granular copy - in registers (mirror and
 * vring kernels) or, in the staged kernels, through this warp's staging buffer with the next unit requested early */
template <bool kMirrored, bool kStaged>
__device__ __forceinline__ void move_seg_unit(const LunCtx *lun, const MoverFill &f, const Segment &g, uint32_t u, uint32_t u_next,
					      uint32_t w, bool drained, int lane, uint8_t *ust, uint64_t *ubar, UStage &us, bool &upfence)
{
	const uint64_t off = (uint64_t)(u - g.first_unit) * kUnitBytes;
	const uint32_t nbytes = (uint32_t)min((uint64_t)kUnitBytes, g.len - off);
	const uint8_t *src = g.src;
	uint8_t *dst = g.dst;
	if (kMirrored && g.mirror) {
		const LunCtx &T = (g.mirror - 1 == lun->target) ? *lun : *lun->peer[g.mirror - 1];
		mirror_unit(T, dst, src, off, nbytes, lane, T.nreplicas);
	} else if (!src) {
		zero_unit(dst + off, nbytes, lane);
	} else if constexpr (kMirrored) {
		move_unit<true>(dst + off, src + off, nbytes, lane);
	} else if ((((uintptr_t)(dst + off) | (uintptr_t)(src + off) | nbytes) & 15) == 0) {
		move_unit(dst + off, src + off, nbytes, lane);
	} else if constexpr (!kStaged) {
		move_unit(dst + off, src + off, nbytes, lane);
	} else {
		/* the unit this warp moves next, when it is known and nothing has to be waited for before it may be read:
		 * its bytes are requested while this one is realigned */
		uint8_t *ndst = nullptr; const uint8_t *nsrc = nullptr; uint32_t nn = 0;
		if (u_next < f.nunits) {
			const Segment &g2 = f.seg_of(u_next);
			if (g2.src && (f.nw == 1 || (g2.wave & kSegWaveMask) == w) && (!(g2.wave & kSegWaitsForDrain) || drained)) {
				const uint64_t off2 = (uint64_t)(u_next - g2.first_unit) * kUnitBytes;
				nn = (uint32_t)min((uint64_t)kUnitBytes, g2.len - off2);
				if ((((uintptr_t)(g2.dst + off2) | (uintptr_t)(g2.src + off2) | nn) & 15) != 0) { ndst = g2.dst + off2; nsrc = g2.src + off2; }
			}
		}
		move_unit_via_smem(dst + off, src + off, nbytes, lane, ust, ubar, us, upfence, ndst, nsrc, nn);
	}
}

/* mover warp 0, lane 0: the fill's data has moved - add its latency to the sums and histograms of its targets */
__device__ __forceinline__ void tally_fill_latency(CtaShared &sh, const Stage &st, const LunCtx *lun)
{
	const unsigned long long dt = globaltimer_ns() - st.t0;
	for (uint32_t i = 0; i < st.lat_ntgt; i++) {
		const uint32_t t = st.lat_tgt[i] & (OIMGPU_CTRLR_MAX_DEVS - 1);
		unsigned long long *acc = sh.lat_ns[t];
		acc[0] += dt * st.lat_n[i][0]; acc[1] += dt * st.lat_n[i][1]; acc[2] += dt * st.lat_n[i][2];
		/* spdk_histogram_data_tally (histogram_data.h:120-160) of the fill's latency, once per bdev_io.  A latency
		 * below the timer's resolution (dt == 0: __clzll gives 64) lands in bucket 0, so that no bdev_io goes untallied */
		const LunCtx *T = (t == lun->target) ? lun : lun->peer[t];
		unsigned long long *hist = T ? *reinterpret_cast<unsigned long long *const volatile *>(&T->hist) : nullptr;
		if (hist) {
			const uint32_t clz = (uint32_t)__clzll((long long)dt);
			const uint32_t range = clz <= 57u ? 57u - clz : 0u;
			const uint32_t index = (uint32_t)(dt >> (range ? range - 1 : 0)) & 127u;
			atomicAdd(&hist[(range << 7) + index], (unsigned long long)(st.lat_n[i][0] + st.lat_n[i][1] + st.lat_n[i][2] + st.lat_n[i][3]));
		}
	}
}

/* ======================= MOVERS (warps 1..kMovers) ======================= */
template <bool kMirrored, bool kMoverReap, bool kStaged>
__device__ __forceinline__ void mover_warp(CtaShared &sh, const LunCtx *lun, int mw, int lane)
{
	UStage us = {nullptr, 0};	/* this warp's staging buffer (move_unit_via_smem) */
	bool upfence = true;		/* the next staged unit follows a barrier another mover's stores may hide behind */
	for (uint32_t c = 0;; c++) {
		const uint32_t sidx = c % kStages;
		Stage &st = sh.stage[sidx];
		mbar_wait(&sh.full[sidx], (c / kStages) & 1);
		if (st.stop) break;
		upfence = true;
		const MoverFill f = {st, st.nseg, st.nunits, st.nwaves};
		/* RAW/WAW/WAR against fill c-drain: before touching a flagged unit, wait until every mover has left that fill */
		const uint32_t drain = st.drain;
		bool drained = !(drain && c >= drain);
		if (!drained && st.drain_upfront) {
			wait_fill_moved(sh, c - drain);
			drained = true;
		}
		/* shared kernels: units are drawn from a counter (mover 0 spends part of its time publishing) unless the fill
		 * has waves, whose barrier wants every mover to walk the same list */
		const bool dyn = kMoverReap && f.nw == 1;
		for (uint32_t w = 0; w < f.nw; w++) {
			for (uint32_t u = dyn ? next_unit(st, true, 0, lane) : (uint32_t)mw, u_next = 0; u < f.nunits; u = u_next) {
				u_next = next_unit(st, dyn, u, lane);	/* drawn before this unit moves: the counter's latency hides behind the loads */
				const Segment &g = f.seg_of(u);
				if (f.nw > 1 && (g.wave & kSegWaveMask) != w) continue;
				if ((g.wave & kSegWaitsForDrain) && !drained) {
					wait_fill_moved(sh, c - drain);
					drained = true;
					upfence = true;
				}
				move_seg_unit<kMirrored, kStaged>(lun, f, g, u, u_next, w, drained, lane, sh.ustage[mw], sh.ubar[mw], us, upfence);
			}
			if (f.nw > 1) { movers_barrier(); upfence = true; }
		}
		if (mw == 0 && lane == 0 && st.lat_ntgt) tally_fill_latency(sh, st, lun);
		__syncwarp();
		if (lane == 0) mbar_arrive(&sh.empty[sidx]);
		if constexpr (kMoverReap) {
			if (mw == 0) {
				/* every mover is done with the fill: publish its completions (in ring order across CTAs, reap_stage
				 * waits for the fills before it) and hand the stage back to the parser */
				wait_fill_moved(sh, c);
				reap_stage(st, lane, &sh.pub_q, &sh.pub_end);
				__syncwarp();
				if (lane == 0) mbar_arrive(&sh.released[sidx]);
			}
		}
	}
}

__device__ __forceinline__ void init_cta_shared(CtaShared &sh)
{
	for (int s = 0; s < kStages; s++) {
		mbar_init(&sh.full[s], 1);
		mbar_init(&sh.empty[s], kMovers);
		mbar_init(&sh.released[s], 1);
	}
	mbar_init(&sh.req_bar[0], 1);
	mbar_init(&sh.req_bar[1], 1);
	for (int w = 0; w < kMovers; w++) { mbar_init(&sh.ubar[w][0], 1); mbar_init(&sh.ubar[w][1], 1); }
	sh.pub_q = nullptr;
	sh.pub_end = 0;
	for (int t = 0; t < OIMGPU_CTRLR_MAX_DEVS; t++) sh.lat_ns[t][0] = sh.lat_ns[t][1] = sh.lat_ns[t][2] = 0;
	asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}

/* kMoverReap: mover warp 0 publishes the completions of a fill instead of the parser.  Always so with shared queues
 * (§ QShare); also for launches that serve guest virtqueues only, where publishing means byte stores into 32 response
 * buffers, 32 used elements and a fence that waits for every load the parser has in flight - time taken from the
 * warp the virtqueue mode is bound by.  The slot-ring kernels keep the parser publishing: they
 * are bound by the movers, and their publication is three coalesced vectors per request without a fence. */
/* kStaged: byte-granular units go through this warp's staging buffer (move_unit_via_smem) - the kernel is launched
 * with the 29 KB the buffers take.  The mirror kernels (NVLink-bound, compact path) and the vring kernel do without:
 * the virtqueue parser lives on the L1 (descriptor tables, rings, the memory table), and two CTAs with staging
 * buffers leave it a third of the L1 they would have without (measured: shared memory that nothing used costs the
 * same), while guests' buffers are sector-aligned as a rule */
template <bool kMirrored, bool kShared, bool kMoverReap = kShared, bool kStaged = !kMirrored>
__device__ __forceinline__ void lun_queue_body(LunCtx *lun, KickHeader *hdr, const QueueDesc *queues)
{
	extern __shared__ __align__(16) unsigned char smem_raw[];
	CtaShared &sh = *reinterpret_cast<CtaShared *>(smem_raw);
	const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	if (hdr->persistent && hdr->dispatcher && blockIdx.x == gridDim.x - 1) {
		if (warp == 0) dispatcher_cta(hdr, queues, lane);
		return;
	}
	if (tid == 0) init_cta_shared(sh);
	__syncthreads();
	if (warp == 0) {
		/* ======================= PARSER ======================= */
		const LunCtx &L = *lun;
		LaneState &s = sh.lane[lane];
		uint32_t fills = 0;			/* stage fills so far */
		uint32_t reaped = 0;			/* fills whose completions are published */
		uint32_t pass_no = 0;			/* passes parsed by this CTA: index into the hazard history ring */
		if (lane < kStages) { sh.hist[lane].writers = 0; sh.hist[lane].touching = 0; }
		__syncwarp();
		IoStats stats;
		bool first = true;
		/* Who publishes a fill's completions.  One CTA per queue: the parser, when it needs the stage again.
		 * Shared queues: completions are published in ring order ACROSS CTAs, so a fill that waits for the
		 * parser's convenience holds up every later pass of the queue - there mover warp 0 publishes as soon as
		 * the movers are done with the fill, and the parser only waits for the stage to be released. */
		auto retire = [&](uint32_t f) {
			const uint32_t sidx_ = f % kStages;
			if constexpr (kMoverReap) {
				mbar_wait(&sh.released[sidx_], (f / kStages) & 1);
			} else {
				mbar_wait(&sh.empty[sidx_], (f / kStages) & 1);
				reap_stage(sh.stage[sidx_], lane);
			}
		};

		/* request slots of slot rings: staged by the TMA unit into reqbuf[fetch_no & 1]; fetches are consumed in the
		 * order they were issued, one per pass, so buffer and barrier phase follow from the two counters */
		uint32_t fetch_no = 0, consume_no = 0;
		auto issue_fetch = [&](const QueueDesc &qd, uint32_t first_slot, uint32_t nslots) {
			const uint32_t b_ = fetch_no & 1;
			if (lane == 0) {
				mbar_expect_tx(&sh.req_bar[b_], nslots * (uint32_t)sizeof(oimgpu_req));
				const uint32_t s0 = first_slot & qd.ring_mask;
				uint32_t n1 = nslots;
				if (qd.ring_mask != 0xffffffffu && s0 + nslots > qd.ring_mask + 1) n1 = qd.ring_mask + 1 - s0;	/* the ring wraps */
				tma_load_bulk(&sh.reqbuf[b_][0], &qd.reqs[s0], n1 * (uint32_t)sizeof(oimgpu_req), &sh.req_bar[b_]);
				if (n1 < nslots) tma_load_bulk(&sh.reqbuf[b_][n1], &qd.reqs[0], (nslots - n1) * (uint32_t)sizeof(oimgpu_req), &sh.req_bar[b_]);
			}
			fetch_no++;
		};
		auto consume_fetch = [&]() -> oimgpu_req * {
			const uint32_t b_ = consume_no & 1;
			mbar_wait(&sh.req_bar[b_], (consume_no >> 1) & 1);
			consume_no++;
			return sh.reqbuf[b_];
		};

		const uint32_t nqueues = hdr->nqueues;
		const bool persistent = hdr->persistent != 0;
		const bool hinted = persistent && hdr->dispatcher != 0;
		const uint32_t nworkers = hinted ? gridDim.x - 1 : gridDim.x;
		constexpr bool shared = kShared;	/* compiled out of the one-CTA-per-queue kernels */
		QShare *const shares = hdr->share;
		uint32_t scan_from = blockIdx.x % nqueues;	/* shared: where the search for unclaimed work resumes */
		uint32_t run_q = 0xffffffffu, run_start = 0, run_end = 0, run_wr = 0, run_we = 0, run_ok = 0;	/* shared, lane 0: this CTA's current run */
		bool run_ok_valid = false;
		uint32_t sweep_qi = blockIdx.x;
		bool progress = false;
		uint64_t last_progress = persistent ? globaltimer_ns() : 0;
		for (;;) {
			uint32_t qi = 0;
			if (shared) {
				/* any queue with unclaimed requests, this CTA's home queue(s) first */
				qi = find_shared_work(hdr, queues, shares, nqueues, nworkers, scan_from, persistent, hinted, lane);
				if (qi == 0xffffffffu) {
					if (!persistent) break;
					if (progress) {
						progress = false;
						last_progress = globaltimer_ns();
						continue;
					}
					/* idle: as below, publish what the pipeline still holds, then stop flag / watchdog */
					while (reaped < fills) retire(reaped++);
					uint32_t quit = 0;
					if (lane == 0) {
						quit = (hinted ? ld_vol32(&hdr->stop_mirror) : ld_vol32(hdr->stop)) != 0;
						if (!quit && hdr->idle_timeout_ms &&
						    globaltimer_ns() - last_progress > (uint64_t)hdr->idle_timeout_ms * 1000000ull) quit = 1;
					}
					if (__shfl_sync(0xffffffffu, quit, 0)) break;
					__nanosleep(OIM_IDLE_NS);
					continue;
				}
				scan_from = qi;		/* stay on it while it has work */
			} else if (!persistent) {
				/* next queue: first one static (no atomic on the critical path), then work-stealing */
				if (lane == 0) qi = first ? blockIdx.x : atomicAdd(&hdr->next, 1u);
				qi = __shfl_sync(0xffffffffu, qi, 0);
				first = false;
				if (qi >= nqueues) break;
			} else {
				if (sweep_qi >= nqueues) {
					/* end of one sweep over this CTA's queues (spdk_thread_poll returning) */
					sweep_qi = blockIdx.x;
					if (progress) {
						progress = false;
						last_progress = globaltimer_ns();
						continue;
					}
					/* idle: publish every completion still held back by the pipeline, then look at the
					 * stop flag / watchdog */
					while (reaped < fills) retire(reaped++);
					uint32_t quit = 0;
					if (lane == 0) {
						quit = (hinted ? ld_vol32(&hdr->stop_mirror) : ld_vol32(hdr->stop)) != 0;
						if (!quit && hdr->idle_timeout_ms &&
						    globaltimer_ns() - last_progress > (uint64_t)hdr->idle_timeout_ms * 1000000ull) quit = 1;
					}
					if (__shfl_sync(0xffffffffu, quit, 0)) break;
					__nanosleep(OIM_IDLE_NS);
					continue;
				}
				qi = sweep_qi;
				sweep_qi += nworkers;
			}
			QueueDesc q = queues[qi];
			QShare *const qs = shared ? &shares[qi] : nullptr;
			uint32_t vq_last_avail = 0, vq_last_used = 0;
			if (shared) {
				/* positions on a shared queue count from where this launch (this poller) started on it: request x
				 * sits at ring position base_avail + x, its completion at base_used + x */
				uint32_t ba = 0, bu = 0, cnt = 0xffffffffu;	/* poller: no fixed count, claims follow the doorbell */
				if (lane == 0) {
					if (!persistent && q.mode == QMODE_SLOTS) {
						ba = q.head;
						cnt = q.count;
					} else {
						if (!persistent) {
							/* the first CTA on the queue fixes what this launch serves: everything up to avail->idx
							 * (spdk_vhost_vq_avail_ring_get, vhost.c:178-211); the others wait for its word */
							if (atomicCAS(&qs->latched, 0u, 2u) == 0u) {
								const uint32_t la = q.vq_state->last_avail, lu = q.vq_state->last_used;
								const uint32_t c = vq_new_entries(producer_index(q, false), la, q.vq_size);
								qs->base_avail = la; qs->base_used = lu; qs->count = c;
								st_release32(&qs->latched, 1u);
							} else {
								while (ld_acquire32(&qs->latched) != 1u) __nanosleep(20);
							}
							cnt = ld_vol32(&qs->count);
						}
						ba = ld_vol32(&qs->base_avail);
						bu = ld_vol32(&qs->base_used);
					}
				}
				q.head = __shfl_sync(0xffffffffu, ba, 0);
				q.count = __shfl_sync(0xffffffffu, cnt, 0);
				vq_last_avail = q.head;
				vq_last_used = __shfl_sync(0xffffffffu, bu, 0);
				if (q.mode == QMODE_VRING) {
					q.iov_mask = 0xffffffffu;
					q.iovs += (size_t)blockIdx.x * kPass * kIovRow;	/* this CTA's scratch SG rows */
				}
			} else if (persistent && q.mode == QMODE_SLOTS) {
				/* new slots = host doorbell (tail) - consumed cursor */
				uint32_t cnt = 0, consumed = 0;
				if (lane == 0) {
					consumed = q.vq_state->last_avail;
					cnt = producer_index(q, hinted) - consumed;
				}
				q.count = __shfl_sync(0xffffffffu, cnt, 0);
				q.head = __shfl_sync(0xffffffffu, consumed, 0);
			} else if (q.mode == QMODE_VRING) {
				/* spdk_vhost_vq_avail_ring_get (vhost.c:178-211): everything up to avail->idx */
				uint32_t cnt = 0;
				if (lane == 0) {
					vq_last_avail = q.vq_state->last_avail;
					vq_last_used = q.vq_state->last_used;
					cnt = vq_new_entries(producer_index(q, hinted), vq_last_avail, q.vq_size);
				}
				q.count = __shfl_sync(0xffffffffu, cnt, 0);
				vq_last_avail = __shfl_sync(0xffffffffu, vq_last_avail, 0);
				vq_last_used = __shfl_sync(0xffffffffu, vq_last_used, 0);
				q.head = vq_last_avail;
				q.iov_mask = 0xffffffffu;
				q.iovs += (size_t)blockIdx.x * kPass * kIovRow;	/* this CTA's scratch SG rows */
			}
			const oimgpu_iov *const iov_base = q.iovs;
			if (persistent && !shared) {
				if (q.count == 0) continue;
				progress = true;
			}
			/* request slots are fetched one pass ahead by the TMA unit (issue_fetch).  On a shared queue the next pass
			 * is not known before it is claimed: there the fetch is issued right after the claim. */
			if (!shared && q.count && q.mode == QMODE_SLOTS) issue_fetch(q, q.head, min((uint32_t)kPass, q.count));
			/* virtqueue mode walks guest memory: avail entry -> head descriptor -> chain -> request
			 * header, each a dependent DRAM access under a saturated memory system.  The first two
			 * are loaded one pass ahead into registers (an L2 prefetch of the rest does not survive:
			 * the payload stream turns the 50 MB L2 over within one pass). */
			uint32_t vq_head_cur = 0, vq_head_nxt = 0;
			int4 vq_raw = make_int4(0, 0, 0, 0);	/* desc[head] of the coming pass, still in flight */
			const bool vq_tbl_aligned = ((uintptr_t)q.vq_desc & 15) == 0;
			if (!shared && q.count && q.mode == QMODE_VRING && (uint32_t)lane < min((uint32_t)kPass, q.count)) {
				vq_head_cur = vq_avail_entry(q, q.head + lane);
				if (vq_tbl_aligned && vq_head_cur < q.vq_size) vq_raw = ld_cg16(q.vq_desc + (size_t)vq_head_cur * 16);
			}
			uint32_t done = 0;	/* position of the current pass on the queue */
			/* shared: the NEXT pass is claimed, and its slots / ring entries fetched, as soon as this pass's parse
			 * results are published - before the emission, which may wait for a free stage - so that claim and
			 * fetch latency stay off the parser's critical path */
			uint32_t next_n = 0, next_done = 0;
			uint32_t chunk_left = 0;	/* requests behind next_done + next_n that this CTA already owns */
			uint32_t streak = 0;		/* consecutive claims that continued this CTA's own run */
			for (uint32_t it = 0;; it++) {
				uint32_t n;
				if (!shared) {
					if (it) done += kPass;
					if (done >= q.count) break;
					n = min((uint32_t)kPass, q.count - done);
				} else {
					if (next_n == 0) {
						uint32_t pos = 0, got = 0;
						if (lane == 0) got = claim_pass(q, qs, persistent, hinted, &pos);
						next_n = __shfl_sync(0xffffffffu, got, 0);
						if (next_n == 0) break;
						next_done = __shfl_sync(0xffffffffu, pos, 0);
						chunk_left = 0;
						streak = 0;
						if (q.mode == QMODE_SLOTS) {
							issue_fetch(q, q.head + next_done, next_n);
						} else if ((uint32_t)lane < next_n) {
							vq_head_cur = vq_avail_entry(q, q.head + next_done + lane);
							if (vq_tbl_aligned && vq_head_cur < q.vq_size) vq_raw = ld_cg16(q.vq_desc + (size_t)vq_head_cur * 16);
						}
					}
					n = next_n;
					done = next_done;
					next_n = 0;
					progress = true;
				}
				const uint32_t slot0 = q.head + done;
				const uint64_t pass_t0 = globaltimer_ns();	/* the requests are in hand: their latency clock starts */
				__syncwarp();
				/* this pass's slots: wait for their bulk copy; virtqueue mode builds its slots in a buffer of its own */
				oimgpu_req *const rq = q.mode == QMODE_SLOTS ? consume_fetch() : sh.reqbuf[consume_no & 1];
				const uint32_t ahead = shared ? 0u : (done + kPass < q.count ? q.count - done - kPass : 0u);
				if (q.mode == QMODE_SLOTS && ahead) issue_fetch(q, slot0 + n, min((uint32_t)kPass, ahead));

				const bool active = (uint32_t)lane < n;
				uint64_t my_resp = 0;
				uint32_t my_head = 0;
				bool chain_ok = true;
				const bool vq_more = q.mode == QMODE_VRING && (uint32_t)lane < min((uint32_t)kPass, ahead);
				if (vq_more)	/* next pass's avail entries: in flight while this pass is walked */
					vq_head_nxt = vq_avail_entry(q, slot0 + n + lane);
				if (q.mode == QMODE_VRING && active) {
					my_head = vq_head_cur;
					VDesc d0 = {0, 0, 0, 0};
					if (my_head < q.vq_size) d0 = vq_tbl_aligned ? decode_desc(vq_raw) : load_desc(q.vq_desc + (size_t)my_head * 16);
					chain_ok = vq_task_data_setup(L, q, my_head, d0, rq[lane], const_cast<oimgpu_iov *>(iov_base) + (size_t)lane * kIovRow,
								      sh.sg[lane], lane * kIovRow, &my_resp);
					/* from here on this lane's `q.iovs` is its own SG list: on chip when it is short (the
					 * usual case: one data buffer), else its row of the scratch table in HBM */
					if (chain_ok && rq[lane].iovcnt <= kSmemIovs) {
						q.iovs = sh.sg[lane];
						rq[lane].iov_start = 0;
					} else {
						q.iovs = iov_base;
					}
				}
				/* next pass's head descriptors: issued now, consumed after the hazard analysis, the
				 * reap and the segment emission of this pass */
				if (vq_more && vq_tbl_aligned && vq_head_nxt < q.vq_size) vq_raw = ld_cg16(q.vq_desc + (size_t)vq_head_nxt * 16);
				if (active && chain_ok) parse_request(L, q, rq[lane], s);
				else if (active) {
					/* invalid_request(): used element of length 0, response untouched (vhost_scsi.c:347-358) */
					lane_reset(s);
					s.length = 0; s.data_transferred = 0; s.used_len = 0; s.resp_valid = 0; s.response = 0;
					s.status = SC_GOOD; s.sk = 0; s.asc = 0;
					rq[lane].tag = 0; rq[lane].iovcnt = 0;
				}
				else lane_reset(s);
				const uint32_t haz = active ? s.hazard : 0;
				const uint64_t lo = s.store_lo, hi = s.store_hi;

				const PassHazards hz = cross_pass_hazards(sh.hist, pass_no, haz, lo, hi, lane);
				const HazPass &cur = sh.hist[pass_no % kStages];
				pass_no++;
				const uint32_t writers = hz.writers; const uint32_t drain = hz.drain; const bool cross = hz.cross;

				if (shared) {
					/* Passes of other CTAs on this queue.  Parse results are published in ring order; with them
					 * a pass learns where the current run of passes parsed by ONE CTA began (inside a run the exact
					 * logic above applies: same parser, same history) and where the last writer before that run
					 * ended.  A pass that writes waits until everything before its run is complete, a pass that only
					 * reads until the last foreign writer is.  (spdk_scsi_lun_execute_tasks runs a LUN's tasks one
					 * after the other, lun.c:163-211: any interleaving that keeps every RAW/WAW/WAR pair in ring
					 * order gives the same bytes.) */
					uint32_t need = 0;
					if (lane == 0) {
						/* {parsed, wr_end} travel in ONE 64-bit word: nothing else is published with it, so the
						 * hand-over needs no fence (which would wait for the parser's read-ahead loads) */
						/* a run = passes this CTA took back to back (nobody else claimed in between): known locally.
						 * Inside a run the chain word is still the one this lane stored last - no need to read it */
						uint32_t we;
						if (run_q == qi && run_end == done) {
							we = run_we;
						} else {
							uint64_t w;
							while ((uint32_t)(w = ld_vol64(&qs->chain)) != done) __nanosleep(20);
							we = (uint32_t)(w >> 32);
							run_q = qi; run_start = done; run_wr = we; run_ok_valid = false;
						}
						run_end = done + n;
						run_we = writers ? done + n : we;
						st_vol64(&qs->chain, (uint64_t)run_we << 32 | (uint64_t)(done + n));
						need = writers ? run_start : run_wr;
						/* run_ok: the largest position of this run's foreign past already seen complete */
						if (need && run_ok_valid && (int32_t)(run_ok - need) >= 0) need = 0;
						else if (need && (int32_t)(ld_acquire32(&qs->done) - need) >= 0) { run_ok = need; run_ok_valid = true; need = 0; }
					}
					need = __shfl_sync(0xffffffffu, need, 0);
					if (need) {
						/* (our own earlier fills are published by mover warp 0 as they finish: nothing here may depend
						 * on this parser, which holds a claimed pass while it waits) */
						if (lane == 0) {
							while ((int32_t)(ld_acquire32(&qs->done) - need) < 0) __nanosleep(40);
							run_ok = need;
							run_ok_valid = true;
						}
						__syncwarp();
					}
					/* the next pass: claim it and start its fetch now (the other slot buffer / vq_raw / vq_head_nxt are free) */
					{
						/* A CTA that has had the queue to itself for a few passes takes four passes' worth per claim
						 * (one atomic round trip per 128 requests instead of per 32); the moment somebody else's claim
						 * lands in between it is back to single passes, so that sharers interleave finely. */
						if (chunk_left) {
							next_done = done + n;
							next_n = min((uint32_t)kPass, chunk_left);
							chunk_left -= next_n;
						} else {
							uint32_t pos = 0, got = 0;
							if (lane == 0) got = claim_pass(q, qs, persistent, hinted, &pos, streak >= 2 ? 4u * kPass : (uint32_t)kPass);
							got = __shfl_sync(0xffffffffu, got, 0);
							next_done = __shfl_sync(0xffffffffu, pos, 0);
							streak = (got && next_done == done + n) ? streak + 1 : 0;
							next_n = min((uint32_t)kPass, got);
							chunk_left = got - next_n;
						}
						if (next_n && q.mode == QMODE_SLOTS) {
							issue_fetch(q, q.head + next_done, next_n);
						} else if (next_n && (uint32_t)lane < next_n) {
							vq_head_nxt = vq_avail_entry(q, q.head + next_done + lane);
							if (vq_tbl_aligned && vq_head_nxt < q.vq_size) vq_raw = ld_cg16(q.vq_desc + (size_t)vq_head_nxt * 16);
						}
					}
				}

				uint32_t nwaves;
				const uint16_t wave = assign_waves(cur, hz, haz, lo, hi, lane, nwaves);

				const bool good = active && s.resp_valid && s.response == OIMGPU_S_OK && s.status == SC_GOOD;
				stats.count(L, s, active, good);

				/* rounds: as many whole requests as fit in one stage's segment table */
				uint32_t r0 = 0;
				while (r0 < n) {
					const bool in = (uint32_t)lane >= r0 && (uint32_t)lane < n;
					const uint32_t segs = in ? s.nseg : 0, units = in ? s.units : 0;
					uint32_t seg_incl = segs, unit_incl = units;
#pragma unroll
					for (int o = 1; o < 32; o <<= 1) {
						const uint32_t a = __shfl_up_sync(0xffffffffu, seg_incl, o);
						const uint32_t b = __shfl_up_sync(0xffffffffu, unit_incl, o);
						if (lane >= o) { seg_incl += a; unit_incl += b; }
					}
					/* ... and a bounded number of units (the first request of a round always fits): a pass of 32 x
					 * 128 KiB in ONE fill of 1024 units ran at 0.958 of the HBM peak, in fills of <= 256 units at
					 * 0.984 (bench.py seq128k_sg "single"; 4 KiB passes are 32 units and never split) */
					const uint32_t fits = __ballot_sync(0xffffffffu, in && seg_incl <= (uint32_t)kSegCap &&
									    (unit_incl <= (uint32_t)kFillUnits || (uint32_t)lane == r0));
					const uint32_t r1 = r0 + __popc(fits);	/* prefix property: seg_incl is monotonic */
					const bool mine = in && (uint32_t)lane < r1;

					/* claim the next stage: wait until its previous fill is consumed, publish that
					 * fill's completions, then refill */
					const uint32_t sidx = fills % kStages;
					Stage &st = sh.stage[sidx];
					if (fills >= kStages && reaped + kStages <= fills) {
						retire(reaped++);
						__syncwarp();
					}
					if (mine) {
						if (segs) emit_segments(L, q, rq[lane], s, &st.seg[seg_incl - segs], unit_incl - units,
									(uint16_t)(wave | (cross ? kSegWaitsForDrain : 0)));
						build_cpl(rq[lane], s, &st.cpl[lane - r0]);
						if (q.mode == QMODE_VRING) {
							st.resp[lane - r0] = my_resp;
							st.vq_head[lane - r0] = (uint16_t)my_head;
						}
					}
					/* latency accounting: the fill's bdev_ios per target and kind (usually one target).  A good READ, WRITE
					 * or SYNCHRONIZE CACHE is one; an UNMAP is one per applied descriptor, whatever its final status */
					{
						const bool bios = mine && (s.op == OP_UNMAP ? s.resp_valid && s.response == OIMGPU_S_OK && s.nseg != 0
											   : good && s.op != OP_NONE);
						uint32_t left = __ballot_sync(0xffffffffu, bios);
						uint32_t nt = 0;
						while (left && nt < OIMGPU_CTRLR_MAX_DEVS) {
							const uint32_t t = __shfl_sync(0xffffffffu, (uint32_t)s.tgt, __ffs(left) - 1);
							const bool me = bios && s.tgt == t;
							const uint32_t all = __ballot_sync(0xffffffffu, me);
							const uint32_t rd = __ballot_sync(0xffffffffu, me && s.op == OP_READ);
							const uint32_t wr = __ballot_sync(0xffffffffu, me && s.op == OP_WRITE);
							const uint32_t fl = __ballot_sync(0xffffffffu, me && s.op == OP_FLUSH);
							const uint32_t um = __reduce_add_sync(0xffffffffu, me && s.op == OP_UNMAP ? s.nseg : 0u);
							if (lane == 0) {
								st.lat_tgt[nt] = (uint8_t)t;
								st.lat_n[nt][0] = (uint16_t)__popc(rd); st.lat_n[nt][1] = (uint16_t)__popc(wr);
								st.lat_n[nt][2] = (uint16_t)um; st.lat_n[nt][3] = (uint16_t)__popc(fl);
							}
							left &= ~all;
							nt++;
						}
						if (lane == 0) st.lat_ntgt = (uint8_t)nt;
					}
					const uint32_t tot_seg = __shfl_sync(0xffffffffu, seg_incl, r1 - 1);
					const uint32_t tot_unit = __shfl_sync(0xffffffffu, unit_incl, r1 - 1);
					if (lane == 0) {
						st.nseg = tot_seg;
						st.nunits = tot_unit;
						st.nwaves = nwaves;
						/* later fills of a split pass simply wait for the fill before them, up front */
						st.drain = (r0 > 0) ? 1 : drain;
						st.drain_upfront = r0 > 0;
						st.stop = 0;
						st.ncpl = r1 - r0;
						st.cpl_ring = q.cpls;
						st.cpl_slot0 = slot0 + r0;
						st.cpl_mask = q.ring_mask;
						st.mode = q.mode;
						st.vq_used = q.vq_used;
						st.vq_state = q.vq_state;
						st.vq_size = q.vq_size;
						st.vq_in_hbm = q.vq_in_hbm;
						st.used_base = vq_last_used + done + r0;
						st.done = persistent ? q.done : nullptr;
						st.unit_ctr = 0;
						st.t0 = pass_t0;
						st.share = qs;
						st.share_pos = done + r0;
						st.share_final = q.count;
						st.persistent = persistent;
					}
					__syncwarp();
					if (lane == 0) mbar_arrive(&sh.full[sidx]);
					fills++;
					r0 = r1;
				}
				vq_head_cur = vq_head_nxt;
			}
			if (!shared && q.mode == QMODE_VRING && lane == 0) {
				/* the parser owns both cursors: every consumed avail entry has its used element at vq_last_used + its
				 * position, published or not.  A resident CTA that comes straight back to this ring while the movers
				 * still hold the batch must place the next one behind it, not where publication has got to */
				store_cursors(q.vq_state, true, vq_last_avail + q.count, vq_last_used + q.count);
			}
			if (!shared && persistent && q.mode == QMODE_SLOTS && lane == 0) store_cursors(q.vq_state, false, q.head + q.count, 0);
		}
		/* tell the movers to stop, then publish the completions still in flight */
		{
			const uint32_t sidx = fills % kStages;
			Stage &st = sh.stage[sidx];
			if (fills >= kStages && reaped + kStages <= fills) {
				retire(reaped++);
				__syncwarp();
			}
			if (lane == 0) { st.stop = 1; st.nunits = 0; st.nseg = 0; st.nwaves = 1; st.drain = 0; st.ncpl = 0; st.mode = QMODE_SLOTS; st.done = nullptr; st.share = nullptr; }
			__syncwarp();
			if (lane == 0) mbar_arrive(&sh.full[sidx]);
		}
		while (reaped < fills) retire(reaped++);
		if (persistent && shared) {
			/* the last worker to leave writes the ring cursors back: by then every claimed pass is published */
			uint32_t last = 0;
			if (lane == 0) last = atomicAdd(&hdr->workers_exited, 1u) == nworkers - 1;
			if (__shfl_sync(0xffffffffu, last, 0)) {
				__threadfence();
				for (uint32_t k = lane; k < nqueues; k += 32) {
					const bool vring = queues[k].mode == QMODE_VRING;
					const uint32_t c = ld_vol32(&shares[k].claim);
					const uint32_t la = ld_vol32(&shares[k].base_avail) + c;
					store_cursors(queues[k].vq_state, vring, la, vring ? ld_vol32(&shares[k].base_used) + c : 0);
				}
				__threadfence();
			}
		}
		if (persistent && lane == 0) {
			__threadfence_system();
			atomicAdd_system(const_cast<uint32_t *>(hdr->exited), 1u);
		}
		stats.flush(lun, sh, lane);
	} else mover_warp<kMirrored, kMoverReap, kStaged>(sh, lun, warp - 1, lane);
}

/* the plain kernel carries no mirror code at all (a call in the mover loop would spill the
 * caller-saved data registers); mirrored bdevs use the second instantiation.  Likewise queue
 * sharing (KickHeader::shared) has its own pair, so the one-CTA-per-queue kernels carry none of its code. */
__global__ void __launch_bounds__(kThreads, OIM_MIN_BLOCKS)
oim_lun_queue_kernel(LunCtx *lun, KickHeader *hdr, const QueueDesc *queues)
{
	lun_queue_body<false, false>(lun, hdr, queues);
}

__global__ void __launch_bounds__(kThreads, OIM_MIN_BLOCKS)
oim_lun_queue_mirror_kernel(LunCtx *lun, KickHeader *hdr, const QueueDesc *queues)
{
	lun_queue_body<true, false>(lun, hdr, queues);
}

/* one CTA per queue, guest virtqueues only: mover warp 0 publishes (see kMoverReap) */
__global__ void __launch_bounds__(kThreads, OIM_MIN_BLOCKS)
oim_lun_vring_kernel(LunCtx *lun, KickHeader *hdr, const QueueDesc *queues)
{
	lun_queue_body<false, false, true, false>(lun, hdr, queues);
}

__global__ void __launch_bounds__(kThreads, OIM_MIN_BLOCKS)
oim_lun_shared_queue_kernel(LunCtx *lun, KickHeader *hdr, const QueueDesc *queues)
{
	lun_queue_body<false, true>(lun, hdr, queues);
}

__global__ void __launch_bounds__(kThreads, OIM_MIN_BLOCKS)
oim_lun_shared_queue_mirror_kernel(LunCtx *lun, KickHeader *hdr, const QueueDesc *queues)
{
	lun_queue_body<true, true>(lun, hdr, queues);
}

/* struct spdk_copy_engine.copy / .fill (S/include/spdk_internal/copy_engine.h:47-53) for
 * device-resident buffers: a plain grid-stride mover built from the same unit routines */
__global__ void __launch_bounds__(256)
oim_copy_kernel(uint8_t *dst, const uint8_t *src, uint64_t nbytes)
{
	const int lane = threadIdx.x & 31;
	const uint64_t warp = (uint64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
	const uint64_t nwarps = (uint64_t)gridDim.x * 8;
	const uint64_t nunits = (nbytes + kUnitBytes - 1) / kUnitBytes;
	for (uint64_t u = warp; u < nunits; u += nwarps) {
		const uint64_t off = u * kUnitBytes;
		const uint32_t n = (uint32_t)min((uint64_t)kUnitBytes, nbytes - off);
		move_unit(dst + off, src + off, n, lane);
	}
}

__global__ void __launch_bounds__(256)
oim_fill_kernel(uint8_t *dst, uint8_t fill, uint64_t nbytes)
{
	const uint64_t i0 = ((uint64_t)blockIdx.x * 256 + threadIdx.x) * 16;
	const uint64_t stride = (uint64_t)gridDim.x * 256 * 16;
	const uint32_t w = fill * 0x01010101u;
	const int4 v = make_int4(w, w, w, w);
	if (((uintptr_t)dst & 15) == 0) {
		for (uint64_t i = i0; i + 16 <= nbytes; i += stride) st_cg16(dst + i, v);
		const uint64_t tail = nbytes & ~15ull;
		if (blockIdx.x == 0 && threadIdx.x < (nbytes & 15)) dst[tail + threadIdx.x] = fill;
	} else {
		for (uint64_t i = (uint64_t)blockIdx.x * 256 + threadIdx.x; i < nbytes; i += (uint64_t)gridDim.x * 256) dst[i] = fill;
	}
}

/* oimgpu_bdev_digest: position-keyed sums over 64-bit words (include/oimgpu.h) */
__global__ void __launch_bounds__(256)
oim_digest_kernel(const uint64_t *p, uint64_t nwords, unsigned long long *out)
{
	unsigned long long a = 0, b = 0;
	for (uint64_t i = (uint64_t)blockIdx.x * 256 + threadIdx.x; i < nwords; i += (uint64_t)gridDim.x * 256) {
		const uint64_t w = p[i];
		a += w * (2 * i + 1);
		uint64_t z = w ^ i;
		z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
		z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
		b += z ^ (z >> 31);
	}
	for (int o = 16; o; o >>= 1) {
		a += __shfl_xor_sync(0xffffffffu, a, o);
		b += __shfl_xor_sync(0xffffffffu, b, o);
	}
	if ((threadIdx.x & 31) == 0) { atomicAdd(&out[0], a); atomicAdd(&out[1], b); }
}

/* ---- host side: the five instantiations and what each is launched with ------------------------------------- */

/* the kStaged instantiations carry the movers' staging buffers (the last member of CtaShared); the others keep the L1 */
static size_t lun_kernel_smem_bytes(LunKernel k)
{
	const bool staged = k == LUN_KERNEL_QUEUE || k == LUN_KERNEL_SHARED_QUEUE;
	return staged ? sizeof(CtaShared) : offsetof(CtaShared, ustage);
}

cudaError_t lun_kernels_init(int *ctas_per_sm)
{
	/* more than the 48 KB a kernel gets without asking */
	cudaError_t e = cudaSuccess;
	auto set_smem = [&](auto kernel, LunKernel k) {
		if (e == cudaSuccess) e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)lun_kernel_smem_bytes(k));
	};
	set_smem(oim_lun_queue_kernel, LUN_KERNEL_QUEUE);
	set_smem(oim_lun_queue_mirror_kernel, LUN_KERNEL_QUEUE_MIRROR);
	set_smem(oim_lun_vring_kernel, LUN_KERNEL_VRING);
	set_smem(oim_lun_shared_queue_kernel, LUN_KERNEL_SHARED_QUEUE);
	set_smem(oim_lun_shared_queue_mirror_kernel, LUN_KERNEL_SHARED_QUEUE_MIRROR);
	if (e != cudaSuccess) return e;
	return cudaOccupancyMaxActiveBlocksPerMultiprocessor(ctas_per_sm, oim_lun_queue_kernel, kThreads,
							     lun_kernel_smem_bytes(LUN_KERNEL_QUEUE));
}

void launch_lun_kernel(LunKernel k, uint32_t grid, cudaStream_t stream, LunCtx *ctx, KickHeader *hdr, const QueueDesc *desc)
{
	const size_t smem = lun_kernel_smem_bytes(k);
	switch (k) {
	case LUN_KERNEL_QUEUE: oim_lun_queue_kernel<<<grid, kThreads, smem, stream>>>(ctx, hdr, desc); break;
	case LUN_KERNEL_QUEUE_MIRROR: oim_lun_queue_mirror_kernel<<<grid, kThreads, smem, stream>>>(ctx, hdr, desc); break;
	case LUN_KERNEL_VRING: oim_lun_vring_kernel<<<grid, kThreads, smem, stream>>>(ctx, hdr, desc); break;
	case LUN_KERNEL_SHARED_QUEUE: oim_lun_shared_queue_kernel<<<grid, kThreads, smem, stream>>>(ctx, hdr, desc); break;
	case LUN_KERNEL_SHARED_QUEUE_MIRROR: oim_lun_shared_queue_mirror_kernel<<<grid, kThreads, smem, stream>>>(ctx, hdr, desc); break;
	default: break;
	}
}

}  // namespace oimgpu
