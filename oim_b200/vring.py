"""virtio split rings in a guest-memory image, for the virtqueue-level path.

Builds what a guest's virtio-scsi driver would put in memory — descriptor table, avail ring, used
ring (linux/virtio_ring.h), `virtio_scsi_cmd_req` headers, response buffers, data buffers, INDIRECT
tables — inside one numpy arena addressed through a guest-physical → arena-offset region table
(the `rte_vhost_memory` of S/lib/vhost/rte_vhost/rte_vhost.h:52-66).  The same image is handed to
the compiled reference, to the C restatement (host addresses) and to the CUDA path (device
addresses), then compared byte for byte.

Layouts (S/lib/vhost/vhost_scsi.c:531-613):
    FROM_DEV:  [RO req 51 B] [WR resp 108 B] [WR data ...]
    TO_DEV:    [RO req 51 B] [RO data ...]   [WR resp 108 B]
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

from . import abi, traces

F_NEXT, F_WRITE, F_INDIRECT = 1, 2, 4
desc_dtype = np.dtype([("addr", "<u8"), ("len", "<u4"), ("flags", "<u2"), ("next", "<u2")])
used_elem_dtype = np.dtype([("id", "<u4"), ("len", "<u4")])
MB2 = 2 << 20
USED_SENTINEL = 0xA5C3_5A3C      # both words of every used element nobody has written yet

# guest-physical layout: two 4 MiB regions that are adjacent in GPA but swapped in the arena (so a
# buffer crossing 0x600000 is NOT contiguous in VA and must be split, vhost.c:481-500), then one big
# region for rings, headers and most data.
R0_GPA, R1_GPA, R2_GPA = 0x0020_0000, 0x0060_0000, 0x1_0000_0000   # region edges on 2 MiB (hugepage) boundaries
R01_SIZE = 4 << 20


@dataclass
class GuestImage:
    arena: np.ndarray                       # the guest's RAM (uint8)
    ring_size: int
    desc_off: int
    avail_off: int
    used_off: int
    regions: list[tuple[int, int, int]]     # (guest_phys_addr, size, arena offset)
    heads: list[int] = field(default_factory=list)
    meta: dict = field(default_factory=dict)

    def region_table(self, base: int) -> np.ndarray:
        """{gpa, size, address} triples with address = base + arena offset"""
        return np.array([[g, s, base + o] for g, s, o in self.regions], dtype=np.uint64).reshape(-1)

    def gpa_to_off(self, gpa: int) -> int:
        for g, s, o in self.regions:
            if g <= gpa < g + s:
                return gpa - g + o
        raise KeyError(hex(gpa))

    @property
    def desc(self) -> np.ndarray:
        return self.arena[self.desc_off:self.desc_off + 16 * self.ring_size].view(desc_dtype)

    @property
    def avail_idx(self) -> int:
        return int(self.arena[self.avail_off + 2:self.avail_off + 4].view("<u2")[0])

    def used_entries(self, arena: np.ndarray | None = None) -> tuple[int, np.ndarray]:
        a = self.arena if arena is None else arena
        idx = int(a[self.used_off + 2:self.used_off + 4].view("<u2")[0])
        ring = a[self.used_off + 4:self.used_off + 4 + 8 * self.ring_size].view(used_elem_dtype)
        return idx, ring

    def used_in_order(self, arena: np.ndarray | None, start_used: int, n: int) -> np.ndarray:
        """the n used elements from ring position start_used on, in ring order (they wrap at the ring's end)"""
        ring = self.used_entries(arena)[1]
        return ring[(start_used + np.arange(n)) & (self.ring_size - 1)]

    def used_untouched(self, arena: np.ndarray, start_used: int, n: int) -> bool:
        """every used element outside the n from start_used on still holds USED_SENTINEL"""
        ring = self.used_entries(arena)[1].view("<u4").reshape(-1, 2)
        keep = np.ones(self.ring_size, dtype=bool)
        keep[(start_used + np.arange(n)) & (self.ring_size - 1)] = False
        return bool((ring[keep] == USED_SENTINEL).all())

    def masked(self, arena: np.ndarray) -> np.ndarray:
        """copy of an arena with the used ring's element area zeroed (its order is timing-dependent
        in the reference); the used idx stays"""
        c = arena.copy()
        c[self.used_off + 4:self.used_off + 4 + 8 * self.ring_size] = 0
        return c


class _Alloc:
    def __init__(self, lo: int, hi: int):
        self.lo, self.hi, self.cur = lo, hi, lo

    def take(self, n: int, align: int = 1) -> int:
        o = -(-self.cur // align) * align
        if o + n > self.hi:
            raise MemoryError("guest image region exhausted")
        self.cur = o + n
        return o


def build_image(requests: list[dict], *, ring_size: int = 256, data_bytes: int = 24 << 20, seed: int = 0,
                mutate: bool = True, pattern_seed: int = 0x5EED, contiguous: bool = False, start_avail: int = 0,
                start_used: int = 0, all_indirect: bool = False) -> GuestImage:
    """requests: [{'cdb','dir','lun','tag','sg': [len,...], 'payload': optional bytes for TO_DEV}]
    One kick's worth: at most ring_size requests.
    contiguous: a request's data elements are cuts of one guest buffer (each continues its predecessor, with an
    occasional gap) instead of separate buffers.
    start_avail / start_used: the ring cursors the device resumes from.  The requests sit at avail positions
    (start_avail + i) mod ring_size, avail->idx = start_avail + n and used->idx = start_used (both mod 2^16).  The
    avail entries outside that window hold random descriptor indices below ring_size, so a device that reads the
    wrong entry serves a wrong but plausible chain; every used element holds USED_SENTINEL until it is written.
    all_indirect: every chain is one INDIRECT ring slot, so the ring holds ring_size requests."""
    rng = np.random.default_rng(seed)
    r2_size = (4 << 20) + data_bytes
    arena = np.zeros(2 * R01_SIZE + r2_size, dtype=np.uint8)
    arena[:] = traces.pattern_bytes(pattern_seed, 0, arena.size)
    regions = [(R0_GPA, R01_SIZE, R01_SIZE), (R1_GPA, R01_SIZE, 0), (R2_GPA, r2_size, 2 * R01_SIZE)]
    # metadata at the start of R2
    meta = _Alloc(2 * R01_SIZE, 2 * R01_SIZE + (4 << 20))
    desc_off = meta.take(16 * ring_size, 16)
    avail_off = meta.take(4 + 2 * ring_size + 2, 2)
    used_off = meta.take(4 + 8 * ring_size + 2, 4)
    arena[desc_off:desc_off + 16 * ring_size] = 0
    arena[avail_off:avail_off + 6 + 2 * ring_size] = 0
    arena[used_off:used_off + 6 + 8 * ring_size] = 0
    img = GuestImage(arena, ring_size, desc_off, avail_off, used_off, regions)
    data = _Alloc(2 * R01_SIZE + (4 << 20), arena.size)
    crossed = [False]          # at most one buffer per image straddles the R0/R1 boundary (no aliasing)

    def off_to_gpa(off: int) -> int:
        for g, s, o in regions:
            if o <= off < o + s:
                return off - o + g
        raise KeyError(off)

    desc = img.desc
    free = list(rng.permutation(ring_size))
    avail_ring = arena[avail_off + 4:avail_off + 4 + 2 * ring_size].view("<u2")
    n_avail = 0
    notes = []

    placed = 0
    for rq in requests[:ring_size]:
        if len(free) < (1 if all_indirect else 4):
            break                                      # ring full: the rest goes into the next kick
        placed += 1
        sg_lens = list(rq["sg"])
        from_dev = rq["dir"] == abi.DIR_FROM_DEV or not sg_lens
        # request header and response buffer (ragged alignment on purpose)
        hdr_off = meta.take(51, int(rng.choice([1, 4, 16])))
        hdr = np.zeros(51, dtype=np.uint8)
        hdr[0:8] = rq["lun"]
        hdr[8:16] = np.frombuffer(int(rq["tag"]).to_bytes(8, "little"), dtype=np.uint8)
        hdr[19:51] = rq["cdb"]
        arena[hdr_off:hdr_off + 51] = hdr
        resp_off = meta.take(108, int(rng.choice([1, 4, 16])))
        arena[resp_off:resp_off + 108] = 0xEE          # so untouched response bytes are recognisable
        # data buffers
        bufs = []
        pos = 0
        run_next = None                                # contiguous: where the next element goes
        for ln in sg_lens:
            cross = mutate and ln >= 8192 and not crossed[0] and rng.integers(0, 6) == 0
            if cross:
                crossed[0] = True
                # buffer that straddles the R0/R1 boundary: GPA-contiguous, VA-discontiguous
                try:
                    before = int(rng.integers(1, min(ln, 128 << 10)))
                    g = R1_GPA - before
                    o_lo = img.gpa_to_off(g)
                    # fill both halves (they are not contiguous in the arena)
                    bufs.append(("gpa", g, ln))
                    if not from_dev and rq.get("payload") is not None:
                        p = rq["payload"][pos:pos + ln]
                        arena[o_lo:o_lo + before] = p[:before]
                        arena[0:ln - before] = p[before:]
                    pos += ln
                    continue
                except (KeyError, ValueError):
                    pass
            if contiguous and ln:
                if run_next is None or rng.integers(0, 5) == 0:
                    run_next = data.take(sum(sg_lens) - pos + 16, 1) + int(rng.integers(0, 16))
                o, run_next = run_next, run_next + ln
            else:
                o = data.take(ln + 16, 1) + int(rng.integers(0, 16)) if ln else data.take(16, 1)
            if not from_dev and rq.get("payload") is not None and ln:
                arena[o:o + ln] = rq["payload"][pos:pos + ln]
            pos += ln
            bufs.append(("off", o, ln))
        chain = [(off_to_gpa(hdr_off), 51, 0)]
        data_descs = [((b[1] if b[0] == "gpa" else off_to_gpa(b[1])), b[2], F_WRITE if from_dev else 0) for b in bufs]
        resp_desc = (off_to_gpa(resp_off), 108, F_WRITE)
        chain += ([resp_desc] + data_descs) if from_dev else (data_descs + [resp_desc])

        # ---- malformed chains (each maps to one `goto invalid_task` of task_data_setup) ----
        kind = int(rng.integers(0, 80)) if mutate else 99
        bad_next = False
        if kind == 0:
            chain[0] = (chain[0][0], 51, F_WRITE)                     # first descriptor writable
        elif kind == 1:
            chain[0] = (chain[0][0], 50, 0)                           # request header too short
        elif kind == 2:
            chain[0] = (0x9_0000_0000, 51, 0)                         # request header unmapped
        elif kind == 3:
            chain = chain[:1]                                         # neither payload nor response
        elif kind == 4:
            i = chain.index(resp_desc)
            chain[i] = (resp_desc[0], 107, F_WRITE)                   # response buffer too short
        elif kind == 5:
            i = chain.index(resp_desc)
            chain[i] = (0x9_0000_0000, 108, F_WRITE)                  # response buffer unmapped
        elif kind == 6 and from_dev and data_descs:
            j = 2 + int(rng.integers(0, len(data_descs)))
            chain[j] = (chain[j][0], chain[j][1], 0)                  # read-only descriptor in a FROM_DEV payload
        elif kind == 7 and not from_dev:
            chain = chain[:-1]                                        # TO_DEV without a response descriptor
        elif kind == 8:
            bad_next = True                                           # next index beyond the table
        elif kind == 9 and data_descs:
            j = (2 if from_dev else 1) + int(rng.integers(0, len(data_descs)))
            chain[j] = (R0_GPA - 4096, chain[j][1], chain[j][2])      # payload starts in unmapped space
        elif kind == 10 and data_descs:
            j = (2 if from_dev else 1) + int(rng.integers(0, len(data_descs)))
            chain[j] = (R2_GPA + r2_size - 100, max(chain[j][1], 4096), chain[j][2])   # runs off the end of a region

        use_indirect = all_indirect or len(chain) > len(free) - 3 or (mutate and rng.integers(0, 3) == 0) or len(chain) > 40
        if use_indirect:
            tbl_off = meta.take(16 * len(chain), 16)
            tbl = arena[tbl_off:tbl_off + 16 * len(chain)].view(desc_dtype)
            for k, (a, ln, fl) in enumerate(chain):
                last = k + 1 == len(chain)
                tbl[k] = (a, ln, fl | (0 if last else F_NEXT), 0 if last else k + 1)
            if bad_next:
                tbl[0]["next"] = len(chain) + 7
            head = int(free.pop())
            tbl_gpa = off_to_gpa(tbl_off)
            if kind == 11:
                tbl_gpa = 0x9_0000_0000                               # indirect table unmapped
            desc[head] = (tbl_gpa, 16 * len(chain), F_INDIRECT, 0)
        else:
            idxs = [int(free.pop()) for _ in chain]
            for k, (a, ln, fl) in enumerate(chain):
                last = k + 1 == len(chain)
                desc[idxs[k]] = (a, ln, fl | (0 if last else F_NEXT), 0 if last else idxs[k + 1])
            if bad_next:
                desc[idxs[0]]["next"] = ring_size + 3
            if kind == 12 and len(chain) > 2:
                desc[idxs[-1]]["flags"] |= F_NEXT                     # chain loops back: stops at 129 iovecs
                desc[idxs[-1]]["next"] = idxs[-1] if from_dev else idxs[1]
            head = idxs[0]
        if kind == 13:
            head = ring_size + int(rng.integers(0, 100))              # avail entry beyond the ring
        avail_ring[(start_avail + n_avail) & (ring_size - 1)] = head
        n_avail += 1
        img.heads.append(head)
        notes.append(kind)
    # what lies outside the published window comes from a generator of its own: at cursor 0 an image keeps the
    # draws it always had
    rest = np.random.default_rng([seed, 0xA7A1])
    outside = np.ones(ring_size, dtype=bool)
    outside[(start_avail + np.arange(n_avail)) & (ring_size - 1)] = False
    avail_ring[outside] = rest.integers(0, ring_size, int(outside.sum()))
    img.used_entries()[1].view("<u4")[:] = USED_SENTINEL
    arena[avail_off + 2:avail_off + 4] = np.frombuffer(np.uint16((start_avail + n_avail) & 0xFFFF).tobytes(), dtype=np.uint8)
    arena[used_off + 2:used_off + 4] = np.frombuffer(np.uint16(start_used & 0xFFFF).tobytes(), dtype=np.uint8)
    img.meta["kinds"] = notes
    img.meta["placed"] = placed
    img.meta["start"] = (start_avail & 0xFFFF, start_used & 0xFFFF)
    return img


def requests_from_trace(t: traces.Trace, arena_init: np.ndarray) -> list[dict]:
    """turn a Layer-1 trace (oimgpu_req + SG table) into chain specs; TO_DEV payloads are taken from
    the trace's arena so that e.g. UNMAP parameter lists survive the relocation"""
    out = []
    for r in t.reqs:
        s, c = int(r["iov_start"]), int(r["iovcnt"])
        iov = t.iovs[s:s + c]
        null = (iov["addr"] & traces.NULL_ADDR_FLAG) != 0
        sg = [int(x) for x in iov["len"]]
        payload = None
        if r["dir"] != abi.DIR_FROM_DEV and c:
            parts = [arena_init[int(a):int(a) + int(l)] if not n else np.zeros(int(l), np.uint8)
                     for a, l, n in zip(iov["addr"] & ~traces.NULL_ADDR_FLAG, iov["len"], null)]
            payload = np.concatenate(parts) if parts else np.zeros(0, np.uint8)
        out.append({"cdb": r["cdb"].copy(), "dir": int(r["dir"]), "lun": r["lun"].copy(), "tag": int(r["tag"]),
                    "sg": sg[:130], "payload": payload})
    return out


# ------------------------------------------------------------------------------------------------
# Uniform multi-queue guest image for throughput measurements (bench.py `virtqueue` leg)
# ------------------------------------------------------------------------------------------------

@dataclass
class UniformGuest:
    arena: np.ndarray            # metadata part of guest memory (rings, headers, responses); payload follows it
    nq: int
    per_q: int
    ring_size: int
    q_stride: int                # bytes of metadata per queue
    desc_off: int                # offsets inside one queue's metadata block
    avail_off: int
    used_off: int
    data_off: int                # arena offset where the payload area starts (not materialised on the host)
    data_bytes: int
    gpa_base: int

    def total_bytes(self) -> int:
        return self.data_off + self.data_bytes


def build_uniform_queues(nq: int, per_q: int, num_blocks: int, *, io_blocks: int = 8, ring_size: int = 1024,
                         seed: int = 1, target: int = 0, gpa_base: int = R2_GPA, ntargets: int = 1,
                         indirect: bool = False) -> UniformGuest:
    """nq virtqueues, each holding per_q READ(10) requests of io_blocks as 3-descriptor direct chains
    [RO req 51 B][WR resp 108 B][WR data], random LBAs over the whole device (reads only: no ordering
    question).  The avail ring is pre-filled with the heads repeated ring_size/per_q times, so bumping
    avail->idx by per_q re-publishes the same chains (what a guest re-using its buffers does)."""
    # indirect: one ring slot per request (VRING_DESC_F_INDIRECT) pointing at its 3-descriptor table in guest memory - how
    # a Linux guest submits (virtio_ring uses indirect descriptors whenever the device offers them), and what lets a
    # 1024-entry ring hold 1024 requests instead of 341
    assert (per_q if indirect else 3 * per_q) <= ring_size and ring_size % per_q == 0
    io_bytes = io_blocks * 512
    desc_off = 0
    avail_off = 16 * ring_size
    used_off = -(-(avail_off + 6 + 2 * ring_size) // 8) * 8
    hdr_off = -(-(used_off + 6 + 8 * ring_size) // 64) * 64
    resp_off = hdr_off + 64 * per_q
    ind_off = resp_off + 128 * per_q                     # indirect tables: 3 x 16 B per request
    q_stride = -(-(ind_off + (48 * per_q if indirect else 0)) // 4096) * 4096
    data_off = nq * q_stride
    data_bytes = nq * per_q * io_bytes
    arena = np.zeros(data_off, dtype=np.uint8)
    meta = arena.reshape(nq, q_stride)
    qbase = (np.arange(nq, dtype=np.uint64) * np.uint64(q_stride))[:, None] + np.uint64(gpa_base)      # [nq,1] GPA of a queue block
    k = np.arange(per_q, dtype=np.uint64)[None, :]
    # descriptors: chain i uses ring slots 3i, 3i+1, 3i+2
    d = np.zeros((nq, max(ring_size, 3 * per_q)), dtype=desc_dtype)
    d["addr"][:, 0:3 * per_q:3] = qbase + np.uint64(hdr_off) + k * np.uint64(64)
    d["len"][:, 0:3 * per_q:3] = 51
    d["flags"][:, 0:3 * per_q:3] = F_NEXT
    d["next"][:, 0:3 * per_q:3] = (3 * k + 1).astype(np.uint16)
    d["addr"][:, 1:3 * per_q:3] = qbase + np.uint64(resp_off) + k * np.uint64(128)
    d["len"][:, 1:3 * per_q:3] = 108
    d["flags"][:, 1:3 * per_q:3] = F_NEXT | F_WRITE
    d["next"][:, 1:3 * per_q:3] = (3 * k + 2).astype(np.uint16)
    qi = np.arange(nq, dtype=np.uint64)[:, None]
    d["addr"][:, 2:3 * per_q:3] = np.uint64(gpa_base + data_off) + (qi * np.uint64(per_q) + k) * np.uint64(io_bytes)
    d["len"][:, 2:3 * per_q:3] = io_bytes
    d["flags"][:, 2:3 * per_q:3] = F_WRITE
    if indirect:
        # the three descriptors move into the request's table (next = 1, 2 inside the table) ...
        tbl = np.zeros((nq, per_q, 3), dtype=desc_dtype)
        for j in range(3):
            for f in ("addr", "len", "flags"):
                tbl[f][:, :, j] = d[f][:, j:3 * per_q:3]
        tbl["next"][:, :, 0] = 1
        tbl["next"][:, :, 1] = 2
        meta[:, ind_off:ind_off + 48 * per_q] = tbl.view(np.uint8).reshape(nq, -1)
        # ... and ring slot i is one INDIRECT descriptor covering it
        d = np.zeros((nq, ring_size), dtype=desc_dtype)
        d["addr"][:, :per_q] = qbase + np.uint64(ind_off) + k * np.uint64(48)
        d["len"][:, :per_q] = 48
        d["flags"][:, :per_q] = F_INDIRECT
    meta[:, desc_off:desc_off + 16 * ring_size] = np.ascontiguousarray(d[:, :ring_size]).view(np.uint8).reshape(nq, -1)
    # avail ring: heads 0,3,6,... (indirect: 0,1,2,...) repeated
    heads = np.tile(((1 if indirect else 3) * np.arange(per_q)).astype("<u2"), ring_size // per_q)
    meta[:, avail_off + 4:avail_off + 4 + 2 * ring_size] = heads.view(np.uint8)[None, :]
    # request headers: virtio_scsi_cmd_req with a READ(10) at a random LBA
    rnd = traces.splitmix64_stream(seed, nq * per_q).reshape(nq, per_q)
    lba = (rnd % np.uint64(num_blocks // io_blocks)) * np.uint64(io_blocks)
    hdr = np.zeros((nq, per_q, 64), dtype=np.uint8)
    hdr[:, :, 0:8] = abi.virtio_lun(target)
    if ntargets > 1:                                     # requests dealt out over targets target .. target+ntargets-1 (lun[1])
        hdr[:, :, 1] = (target + (np.arange(nq)[:, None] * per_q + np.arange(per_q)[None, :]) % ntargets).astype(np.uint8)
    hdr[:, :, 19] = abi.READ_10
    hdr[:, :, 21:25] = lba.astype(">u4").view(np.uint8).reshape(nq, per_q, 4)
    hdr[:, :, 26:28] = np.array([io_blocks >> 8, io_blocks & 0xFF], dtype=np.uint8)
    meta[:, hdr_off:hdr_off + 64 * per_q] = hdr.reshape(nq, -1)
    g = UniformGuest(arena, nq, per_q, ring_size, q_stride, desc_off, avail_off, used_off, data_off, data_bytes, gpa_base)
    g.lba = lba
    return g
