"""Synthetic request traces for the block-I/O path (SURVEY.md §8(d)).

A trace is a request array + SG table whose addresses are *offsets* into a data arena until
``Trace.bind(base)`` turns them into pointers (host or device).  The same trace object therefore
feeds the CUDA path (arena in HBM or pinned host memory), the C restatement and the compiled
reference (arena in host memory), which is what makes bit-exact comparison possible.

Workload shapes follow SPDK's bdevperf (S/test/bdev/bdevperf/bdevperf.c:454-493): random offsets
``rand % size_in_ios`` (:460-462), sequential ``offset_in_ios++`` with wrap (:463-466), and
``is_read = rand % 100 < rw_percentage`` (:484-485).  PRNG = splitmix64.
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

from . import abi

GAMMA = np.uint64(0x9E3779B97F4A7C15)
_M1 = np.uint64(0xBF58476D1CE4E5B9)
_M2 = np.uint64(0x94D049BB133111EB)
NULL_ADDR_FLAG = np.uint64(1) << np.uint64(63)   # marks an SG element that must stay address 0


def mix64(x: np.ndarray) -> np.ndarray:
    """splitmix64 finaliser on a uint64 array (wrapping arithmetic)."""
    z = x.astype(np.uint64, copy=True)
    z ^= z >> np.uint64(30)
    z *= _M1
    z ^= z >> np.uint64(27)
    z *= _M2
    z ^= z >> np.uint64(31)
    return z


def splitmix64_stream(seed: int, n: int, start: int = 0) -> np.ndarray:
    """First n outputs (from index `start`) of splitmix64 seeded with `seed`."""
    with np.errstate(over="ignore"):
        idx = np.arange(start + 1, start + n + 1, dtype=np.uint64)
        return mix64(np.uint64(seed) + idx * GAMMA)


def pattern_words(seed: int, first_word: int, nwords: int) -> np.ndarray:
    """Fill pattern: the 64-bit word at byte offset o is mix64(seed ^ (o/8) * GAMMA-ish)
    (SURVEY.md §8(d) C2 prefill).  Position-keyed so any sub-range can be regenerated."""
    with np.errstate(over="ignore"):
        idx = np.arange(first_word, first_word + nwords, dtype=np.uint64)
        return mix64((np.uint64(seed) ^ idx) * GAMMA + GAMMA)


def pattern_bytes(seed: int, offset: int, nbytes: int) -> np.ndarray:
    """Byte view of the fill pattern for [offset, offset+nbytes) (any alignment)."""
    w0 = offset // 8
    w1 = (offset + nbytes + 7) // 8
    b = pattern_words(seed, w0, w1 - w0).view(np.uint8)
    s = offset - w0 * 8
    return b[s:s + nbytes]


@dataclass
class Trace:
    reqs: np.ndarray                 # abi.req_dtype
    iovs: np.ndarray                 # abi.iov_dtype, addr = arena offset (| NULL_ADDR_FLAG)
    arena_bytes: int                 # size of the data arena the offsets index
    name: str = ""
    meta: dict = field(default_factory=dict)

    def bind(self, base: int) -> np.ndarray:
        """SG table with real addresses: base + offset (flagged elements become address 0)."""
        out = self.iovs.copy()
        null = (out["addr"] & NULL_ADDR_FLAG) != 0
        out["addr"] = out["addr"] + np.uint64(base)
        out["addr"][null] = 0
        return out

    def __len__(self) -> int:
        return len(self.reqs)

    def split_queues(self, nq: int) -> list["Trace"]:
        """Contiguous split into nq per-queue traces (queue i = requests [i*per, (i+1)*per))."""
        per = len(self.reqs) // nq
        assert per * nq == len(self.reqs)
        out = []
        for i in range(nq):
            r = self.reqs[i * per:(i + 1) * per].copy()
            lo = int(r["iov_start"][0])
            hi = int(r["iov_start"][-1]) + int(r["iovcnt"][-1])
            r["iov_start"] -= np.uint32(lo)
            out.append(Trace(r, self.iovs[lo:hi].copy(), self.arena_bytes, f"{self.name}.q{i}"))
        return out


def _rw_cdbs(opcode10: int, opcode16: int, lba: np.ndarray, nblk: np.ndarray) -> np.ndarray:
    """Vectorised READ/WRITE(10) CDBs, falling back to the 16-byte form where the fields overflow."""
    n = len(lba)
    cdb = np.zeros((n, abi.CDB_SIZE), dtype=np.uint8)
    small = (lba < (1 << 32)) & (nblk < (1 << 16))
    lba64 = lba.astype(np.uint64)
    nb32 = nblk.astype(np.uint32)
    s = np.nonzero(small)[0]
    cdb[s, 0] = opcode10
    cdb[s, 2:6] = lba64[s].astype(">u4").view(np.uint8).reshape(-1, 4)
    cdb[s, 7:9] = nb32[s].astype(">u2").view(np.uint8).reshape(-1, 2)
    b = np.nonzero(~small)[0]
    cdb[b, 0] = opcode16
    cdb[b, 2:10] = lba64[b].astype(">u8").view(np.uint8).reshape(-1, 8)
    cdb[b, 10:14] = nb32[b].astype(">u4").view(np.uint8).reshape(-1, 4)
    return cdb


def _finish(n: int, cdb: np.ndarray, direction: np.ndarray, iovcnt: np.ndarray, target: int) -> np.ndarray:
    reqs = np.zeros(n, dtype=abi.req_dtype)
    reqs["lun"] = abi.virtio_lun(target)
    reqs["tag"] = np.arange(n, dtype=np.uint64)
    reqs["cdb"] = cdb
    reqs["dir"] = direction
    reqs["iovcnt"] = iovcnt
    starts = np.zeros(n, dtype=np.uint64)
    np.cumsum(iovcnt[:-1], out=starts[1:])
    reqs["iov_start"] = starts.astype(np.uint32)
    return reqs


def _sg_layout(n: int, io_bytes: int, sg: str) -> list[int]:
    """Element lengths of one request's SG list (SURVEY.md §8(d) C3 variants)."""
    if sg == "single":
        return [io_bytes]
    if sg == "pages":                       # guest pages
        assert io_bytes % 4096 == 0
        return [4096] * (io_bytes // 4096)
    if sg == "unaligned":                   # byte-granular head and tail, e.g. 100 + k*4096 + rest
        assert io_bytes > 8192
        head = 100
        mid = (io_bytes - head) // 4096
        tail = io_bytes - head - mid * 4096
        return [head] + [4096] * mid + ([tail] if tail else [])
    raise ValueError(sg)


def uniform_trace(n: int, num_blocks: int, *, io_blocks: int = 8, block_size: int = 512,
                  pattern: str = "randread", read_pct: int = 70, sg: str = "single",
                  seed: int = 0xB2000000, target: int = 0, lba_lo: int = 0,
                  lba_span: int | None = None, buf_align: int = 4096) -> Trace:
    """Fixed-size I/O trace.

    pattern: "randread" | "randwrite" | "randrw" (read_pct) | "seqread" | "seqwrite"
    Each request gets its own data buffer in the arena (request i at i*stride), so within one
    trace no two requests share client memory and every byte moved is distinct.
    lba_lo/lba_span restrict the LBA window (used to give each queue its own region).
    """
    io_bytes = io_blocks * block_size
    span = (num_blocks - lba_lo) if lba_span is None else lba_span
    size_in_ios = span // io_blocks
    assert size_in_ios > 0
    rnd = splitmix64_stream(seed, 2 * n)
    if pattern.startswith("rand"):
        off_in_ios = rnd[:n] % np.uint64(size_in_ios)
    else:
        off_in_ios = np.arange(n, dtype=np.uint64) % np.uint64(size_in_ios)
    lba = off_in_ios * np.uint64(io_blocks) + np.uint64(lba_lo)
    if pattern in ("randread", "seqread"):
        is_read = np.ones(n, dtype=bool)
    elif pattern in ("randwrite", "seqwrite"):
        is_read = np.zeros(n, dtype=bool)
    else:
        is_read = (rnd[n:] % np.uint64(100)) < np.uint64(read_pct)
    nblk = np.full(n, io_blocks, dtype=np.uint64)
    cdb = np.where(is_read[:, None], _rw_cdbs(abi.READ_10, abi.READ_16, lba, nblk),
                   _rw_cdbs(abi.WRITE_10, abi.WRITE_16, lba, nblk))
    shift = 0
    if sg.endswith("+3"):                    # client buffers 3 bytes off the store's alignment: the realign path
        sg, shift = sg[:-2], 3
    scattered = sg == "scattered"            # the unaligned elements, but none continues its predecessor in client memory
    lens = _sg_layout(n, io_bytes, "unaligned" if scattered else sg)
    k = len(lens)
    stride = -(-(io_bytes + shift) // buf_align) * buf_align
    reqs = _finish(n, cdb, np.where(is_read, abi.DIR_FROM_DEV, abi.DIR_TO_DEV).astype(np.uint8),
                   np.full(n, k, dtype=np.uint16), target)
    iovs = np.zeros(n * k, dtype=abi.iov_dtype)
    within = np.concatenate([[0], np.cumsum(lens[:-1])]).astype(np.uint64)
    if scattered:                            # element j sits where the reversed list would put it
        within = (io_bytes - np.cumsum(lens)).astype(np.uint64)
    base = (np.arange(n, dtype=np.uint64) * np.uint64(stride) + np.uint64(shift))[:, None]
    iovs["addr"] = (base + within[None, :]).reshape(-1)
    iovs["len"] = np.tile(np.asarray(lens, dtype=np.uint32), n)
    return Trace(reqs, iovs, n * stride, f"{pattern}-{io_bytes}B-{sg}",
                 {"io_bytes": io_bytes, "n": n, "reads": int(is_read.sum()), "stride": stride,
                  "payload_bytes": n * io_bytes})


def partitioned_queues(nq: int, per_q: int, num_blocks: int, **kw) -> Trace:
    """nq queues x per_q requests, queue q confined to LBA window q (fio `offset_increment`
    style) so cross-queue order — undefined for any multi-queue block device — cannot change the
    result.  Requests are laid out queue-major: queue q = [q*per_q, (q+1)*per_q)."""
    io_blocks = kw.get("io_blocks", 8)
    span = (num_blocks // nq) // io_blocks * io_blocks
    seed = kw.pop("seed", 0xB2000000)
    parts = [uniform_trace(per_q, num_blocks, lba_lo=q * span, lba_span=span, seed=seed + q, **kw)
             for q in range(nq)]
    stride = parts[0].meta["stride"]
    reqs = np.concatenate([p.reqs for p in parts])
    iovs = np.concatenate([p.iovs for p in parts])
    k = len(parts[0].iovs) // per_q
    for q in range(nq):
        sl = slice(q * per_q, (q + 1) * per_q)
        reqs["iov_start"][sl] += np.uint32(q * per_q * k)
        reqs["tag"][sl] += np.uint64(q * per_q)
        iovs["addr"][q * per_q * k:(q + 1) * per_q * k] += np.uint64(q * per_q * stride)
    t = Trace(reqs, iovs, nq * per_q * stride, f"{parts[0].name}-q{nq}x{per_q}", dict(parts[0].meta))
    t.meta.update(n=nq * per_q, nq=nq, per_q=per_q, reads=sum(p.meta["reads"] for p in parts),
                  payload_bytes=nq * per_q * parts[0].meta["io_bytes"])
    return t


# ------------------------------------------------------------------------------------------------
# Adversarial trace: every opcode the path decodes, ragged / unaligned / empty SG lists, limits,
# out-of-range and malformed requests.  Drives the parity tests (oracle vs reference, CUDA vs oracle).
# ------------------------------------------------------------------------------------------------

def fuzz_trace(n: int, num_blocks: int, *, block_size: int = 512, seed: int = 1, target: int = 0,
               max_io_blocks: int = 64, arena_bytes: int = 8 << 20, allow_overlap: bool = True,
               include_malformed: bool = True, contiguous: bool = False) -> Trace:
    """contiguous: multi-element SG lists are cuts of ONE client buffer (a guest buffer split at arbitrary
    places: elements continue each other, with zero-length elements and an occasional gap in between) instead
    of separate allocations."""
    rng = np.random.default_rng(seed)
    b = abi.Batch(target)
    cursor = [0]

    def alloc(nbytes: int, align: int = 1) -> int:
        """arena offset for a client buffer.  Never reused: two requests never share client memory, as
        no initiator hands one buffer to two commands in flight (the device tracks LBA hazards, not
        aliasing of guest memory).  The arena grows to whatever the trace needs."""
        o = -(-(cursor[0] + 64) // align) * align
        cursor[0] = o + nbytes
        return o

    def split(nbytes: int) -> list[tuple[int, int]]:
        """random SG list covering nbytes: aligned pages, ragged cuts, zero-length elements"""
        style = rng.integers(0, 6)
        if nbytes == 0:
            return [(alloc(0), 0)] if style < 3 else []
        if style == 0:
            return [(alloc(nbytes, 4096), nbytes)]
        if style == 1:
            return [(alloc(nbytes, 16), nbytes)]
        if style == 2:                                   # byte-granular everything
            return [(alloc(nbytes + 16, 1) + int(rng.integers(0, 16)), nbytes)]
        cuts = sorted(set(int(x) for x in rng.integers(0, nbytes + 1, size=int(rng.integers(1, 9)))))
        if style == 3:                                   # cuts on 512-byte boundaries
            cuts = sorted(set((c // 512) * 512 for c in cuts))
        edges = [0] + [c for c in cuts if 0 < c < nbytes] + [nbytes]
        out = []
        if contiguous:
            base = alloc(nbytes + 16, 1) + (int(rng.integers(0, 16)) if style == 5 else 0)
            for a, z in zip(edges[:-1], edges[1:]):
                if rng.integers(0, 5) == 0:              # a gap: the rest lives in another buffer
                    base = alloc(nbytes + 16, 1) + int(rng.integers(0, 16))
                out.append((base + a, z - a))
                if rng.integers(0, 4) == 0:
                    out.append((alloc(0), 0))            # a zero-length element does not break a run
            return out
        for a, z in zip(edges[:-1], edges[1:]):
            out.append((alloc(z - a + 16, 1) + int(rng.integers(0, 16)) if style == 5
                        else alloc(z - a, 1), z - a))
            if style == 5 and rng.integers(0, 4) == 0:
                out.append((alloc(0), 0))                # zero-length element in the middle
        return out

    hot = int(rng.integers(0, max(1, num_blocks - 4 * max_io_blocks)))   # collision hot-spot

    def pick_lba(nblk: int) -> int:
        if allow_overlap and rng.integers(0, 3) == 0:
            return hot + int(rng.integers(0, 2 * max_io_blocks))
        return int(rng.integers(0, max(1, num_blocks - nblk + 1)))

    rd = {6: abi.READ_6, 10: abi.READ_10, 12: abi.READ_12, 16: abi.READ_16}
    wr = {6: abi.WRITE_6, 10: abi.WRITE_10, 12: abi.WRITE_12, 16: abi.WRITE_16}

    for _ in range(n):
        kind = int(rng.integers(0, 100))
        width = int(rng.choice([6, 10, 12, 16]))
        nblk = int(rng.integers(1, max_io_blocks + 1))
        if width == 6:
            nblk = min(nblk, 255)
        lba = pick_lba(nblk)
        if width == 6:
            lba &= 0x1FFFFF
            if lba + nblk > num_blocks:
                lba = max(0, num_blocks - nblk)
        nbytes = nblk * block_size
        if kind < 38:                                    # well-formed READ
            b.add(abi.cdb_rw(rd[width], lba, nblk), abi.DIR_FROM_DEV, split(nbytes))
        elif kind < 70:                                  # well-formed WRITE
            b.add(abi.cdb_rw(wr[width], lba, nblk), abi.DIR_TO_DEV, split(nbytes))
        elif kind < 74:                                  # UNMAP, 0..4 descriptors, some empty
            nd = int(rng.integers(0, 5))
            descs = [(pick_lba(32), int(rng.integers(0, 33))) for _ in range(nd)]
            pl = abi.unmap_param_list(descs)
            b.add(abi.cdb_unmap(len(pl)), abi.DIR_TO_DEV, _param_iovs(alloc, pl, rng))
            _stash_payload(b, pl)
        elif kind < 77:                                  # SYNCHRONIZE CACHE 10/16 incl. len 0
            op = abi.SYNCHRONIZE_CACHE_10 if rng.integers(0, 2) else abi.SYNCHRONIZE_CACHE_16
            b.add(abi.cdb_sync(op, lba, int(rng.integers(0, 3)) * nblk), abi.DIR_FROM_DEV, [])
        elif kind < 80:                                  # READ CAPACITY 10 / 16
            six = bool(rng.integers(0, 2))
            want = int(rng.choice([8, 12, 32, 64]))
            b.add(abi.cdb_read_capacity(six, alloc_len=int(rng.choice([0, 8, 12, 32, 40]))),
                  abi.DIR_FROM_DEV, split(want))
        elif kind < 82:                                  # TEST UNIT READY / START STOP / REQUEST SENSE
            c = np.zeros(abi.CDB_SIZE, dtype=np.uint8)
            c[0] = int(rng.choice([0x00, 0x1B, 0x03]))
            if c[0] == 0x03:
                c[4] = int(rng.choice([0, 8, 18, 252]))
                b.add(c, abi.DIR_FROM_DEV, split(int(rng.choice([18, 32, 252]))))
            else:
                b.add(c, abi.DIR_FROM_DEV, [])
        elif not include_malformed:
            b.add(abi.cdb_rw(rd[10], lba, nblk), abi.DIR_FROM_DEV, split(nbytes))
        elif kind < 85:                                  # LBA / length out of range
            far = num_blocks - int(rng.integers(0, nblk)) if rng.integers(0, 2) else num_blocks + int(rng.integers(0, 1000))
            op = rd[16] if rng.integers(0, 2) else wr[16]
            b.add(abi.cdb_rw(op, far, nblk), abi.DIR_FROM_DEV if op == rd[16] else abi.DIR_TO_DEV,
                  split(nbytes))
        elif kind < 87:                                  # zero transfer length (valid / past the end)
            at = lba if rng.integers(0, 2) else num_blocks
            b.add(abi.cdb_rw(rd[16], at, 0), abi.DIR_FROM_DEV, [])
        elif kind < 89:                                  # payload shorter / longer than the CDB says
            delta = int(rng.choice([-1, 1, 2])) * block_size
            plen = max(0, nbytes + delta)
            if rng.integers(0, 2):
                b.add(abi.cdb_rw(rd[10], min(lba, num_blocks - nblk - 4), nblk), abi.DIR_FROM_DEV, split(plen))
            else:
                b.add(abi.cdb_rw(wr[10], min(lba, num_blocks - nblk - 4), nblk), abi.DIR_TO_DEV, split(plen))
        elif kind < 91:                                  # payload not a multiple of the block size
            plen = nbytes + int(rng.integers(1, block_size))
            op, d = (rd[10], abi.DIR_FROM_DEV) if rng.integers(0, 2) else (wr[10], abi.DIR_TO_DEV)
            b.add(abi.cdb_rw(op, lba, nblk), d, split(plen))
        elif kind < 93:                                  # wrong data direction
            op, d = (rd[10], abi.DIR_TO_DEV) if rng.integers(0, 2) else (wr[10], abi.DIR_FROM_DEV)
            b.add(abi.cdb_rw(op, lba, nblk), d, split(nbytes))
        elif kind < 95:                                  # over the 4 MiB transfer limit (CDB only)
            big = abi.MAX_XFER_BYTES // block_size + int(rng.integers(1, 100))
            if num_blocks > big:
                b.add(abi.cdb_rw(rd[16], 0, big), abi.DIR_FROM_DEV, split(block_size))
            else:
                b.add(abi.cdb_rw(rd[16], num_blocks, 1), abi.DIR_FROM_DEV, split(block_size))
        elif kind < 96:                                  # unknown opcode
            c = np.zeros(abi.CDB_SIZE, dtype=np.uint8)
            c[0] = int(rng.choice([0xFF, 0xC1, 0x4C, 0x4D, 0x9E]))
            c[1] = 0x05
            b.add(c, abi.DIR_FROM_DEV, split(block_size))
        elif kind < 98:                                  # bad LUN addressing
            lun = abi.virtio_lun(target)
            which = int(rng.integers(0, 4))
            if which == 0:
                lun[0] = 0
            elif which == 1:
                lun[1] = (target + 1) % 8                # empty target slot
            elif which == 2:
                lun[1] = 9
            else:
                lun[3] = 5                               # LUN id 5 on an existing target -> null LUN
            c = abi.cdb_rw(rd[10], lba, nblk)
            if rng.integers(0, 3) == 0:
                c = np.zeros(abi.CDB_SIZE, dtype=np.uint8)
                c[0] = abi.INQUIRY
                c[3:5] = [0, int(rng.choice([0, 36, 96]))]
            b.add(c, abi.DIR_FROM_DEV, split(nbytes), lun=lun)
        elif kind < 99:                                  # unmapped (NULL) SG address
            iv = split(nbytes) or [(alloc(0), 0)]
            j = int(rng.integers(0, len(iv)))
            iv[j] = (int(NULL_ADDR_FLAG), iv[j][1])
            b.add(abi.cdb_rw(rd[10], lba, nblk), abi.DIR_FROM_DEV, iv)
        else:                                            # more than 129 SG elements
            k = 130 + int(rng.integers(0, 3))
            o = alloc(k * 512, 512)
            b.add(abi.cdb_rw(rd[10], 0, min(k, num_blocks)), abi.DIR_FROM_DEV,
                  [(o + i * 512, 512) for i in range(k)])

    reqs, iovs = b.arrays()
    t = Trace(reqs, iovs, max(arena_bytes, cursor[0] + 4096), f"fuzz-{seed}", {"n": n})
    t.meta["param_payloads"] = getattr(b, "_payloads", [])
    return t


# ------------------------------------------------------------------------------------------------
# Alignment sweep: the byte-granular movers (lun_kernel.cuh move_unit_unaligned / _compact, lun_kernel.cu
# move_unit_via_smem) at every skew and at the lengths where their cases change.  Deterministic.
# ------------------------------------------------------------------------------------------------

PIECE_BODY = 2032        # lun_kernel.cu kPieceBody: a staged unit's first piece ends at head + 2032 bytes


def sweep_lengths(dst_skew: int) -> list[int]:
    """element lengths at the movers' edges for a destination at `dst_skew` (mod 16): under / at / over one
    vector; just below, at and just above the staged-piece split (head + 2032: second piece empty, empty, one
    byte); one unit -1 / 0 / +1; and a run of four units with an odd tail"""
    p = (16 - dst_skew) % 16 + PIECE_BODY
    return [1, 15, 16, 17, p - 1, p, p + 1, 4095, 4096, 4097, 3 * 4096 + 1234]


def alignment_sweep(num_blocks: int = 65536, *, block_size: int = 512, target: int = 0, per_request: int = 32) -> Trace:
    """READs and WRITEs whose SG elements sweep (client address mod 16) x (store offset mod 16) x sweep_lengths,
    followed by two passes of misaligned READs behind WRITEs to the same blocks (same pass, next pass).

    Every element has a client buffer of its own (no element continues another, so each is one segment of the
    mover).  The store offset of an element is set by the elements before it in its request: a spacer element
    brings it to the wanted value mod 16, and a last element pads the request to whole blocks.  WRITEs go to the
    first half of the device, READs read the second, the hazard passes use the last 1024 blocks."""
    assert block_size % 16 == 0
    b = abi.Batch(target)
    cursor = [0]

    def buf(n: int, skew: int) -> int:
        o = (cursor[0] + 127) // 64 * 64 + skew        # >= 64 bytes past the previous buffer's end
        cursor[0] = o + n
        return o

    lba = {abi.DIR_TO_DEV: 0, abi.DIR_FROM_DEV: num_blocks // 2}
    for d in (abi.DIR_FROM_DEV, abi.DIR_TO_DEV):
        read = d == abi.DIR_FROM_DEV
        cases = [(c, s, n) for c in range(16) for s in range(16) for n in sweep_lengths(c if read else s)]
        for k in range(0, len(cases), per_request):
            els, store = [], 0
            for j, (c, s, n) in enumerate(cases[k:k + per_request]):
                gap = (s - store) % 16 + 16 * (j % 3)
                if gap:
                    els.append((buf(gap, (c + 7) % 16), gap))
                    store += gap
                els.append((buf(n, c), n))
                store += n
            pad = -store % block_size
            if pad:
                els.append((buf(pad, 9), pad))
                store += pad
            nblk = store // block_size
            if read:
                b.read(lba[d], nblk, els)
            else:
                b.write(lba[d], nblk, els)
            lba[d] += nblk
    hz = num_blocks - 1024
    assert lba[abi.DIR_TO_DEV] <= num_blocks // 2 and lba[abi.DIR_FROM_DEV] <= hz, "num_blocks too small for the sweep"
    while len(b._reqs) % abi.REQS_PER_PASS:                  # the hazard passes start on a pass boundary
        b.read(hz + 512 + len(b._reqs) % 8, 1, [(buf(512, 0), 512)])
    for g in range(8):                                       # pass p: W, R (RAW), R (RAW, part), W (WAW, WAR)
        x = hz + 16 * g
        b.write(x, 8, [(buf(100 + g, (3 + g) % 16), 100 + g), (buf(3996 - g, (11 + g) % 16), 3996 - g)])
        b.read(x, 8, [(buf(4096, (5 + 2 * g) % 16), 4096)])
        b.read(x + 1, 2, [(buf(333, (g + 1) % 16), 333), (buf(691, (2 * g + 3) % 16), 691)])
        b.write(x + 4, 2, [(buf(1024, (13 + g) % 16), 1024)])
    for g in range(8):                                       # pass p + 1: reads of what pass p wrote, one more write
        x = hz + 16 * g
        b.read(x, 8, [(buf(4096, (5 * g + 1) % 16), 4096)])
        b.read(x + 3, 4, [(buf(7, (g + 9) % 16), 7), (buf(2033, (g + 2) % 16), 2033), (buf(0, 0), 0),
                          (buf(8, (15 - g) % 16), 8)])
        b.write(x + 7, 1, [(buf(512, (g + 6) % 16), 512)])
        b.read(x + 6, 2, [(buf(1024, (3 * g + 7) % 16), 1024)])
    reqs, iovs = b.arrays()
    return Trace(reqs, iovs, cursor[0] + 4096, "alignment-sweep", {"hazard_pass": len(reqs) // abi.REQS_PER_PASS - 2})


# ------------------------------------------------------------------------------------------------
# Block-size edges: the transfer limit, fills of more than kFillUnits units, READ(6) length 0, SG shapes and
# UNMAP extents measured in blocks of any size.  Deterministic.
# ------------------------------------------------------------------------------------------------

FILL_BYTES = 1 << 20     # lun_kernel.cu kFillUnits x 4 KiB: a request above this has a fill of its own


def block_size_trace(num_blocks: int, block_size: int, *, seed: int = 1, target: int = 0) -> Trace:
    """The requests whose shape depends on the block size, in passes of abi.REQS_PER_PASS:

    - READ/WRITE 6/10/12/16 at 1 block and at max = MAX_XFER_BYTES // block_size blocks (READ(6)/WRITE(6): at most
      255), at LBA 0 and at the last fit, one past the last fit (LBA out of range) and max + 1 blocks (refused);
    - READ(6)/WRITE(6) with length byte 0 (256 blocks) at LBA 0, num_blocks - 256 and num_blocks - 255;
    - passes that mix requests over 1 MiB (FILL_BYTES) with one-block ones, the big one first, in the middle and last,
      with hazards between them in the same and the next pass;
    - SG lists of one element, of block-sized elements up to the 129-element limit and 130 (invalid), cut at odd bytes
      inside a block, runs of elements that continue each other across 4 KiB, every client address mod 16, and a
      pass of more than 256 segments;
    - UNMAP of one many-MiB descriptor, of 256 one-block descriptors, a list that fails part-way and the whole
      device, each followed by READs of what it unmapped in the same and the next pass;
    - SYNCHRONIZE CACHE with count 0 from LBA 0 and near the end.

    Passes are padded with READ CAPACITY 10/16, whose payloads carry the block size.  Addresses are arena offsets."""
    bs, nb = block_size, num_blocks
    mx = abi.MAX_XFER_BYTES // bs
    assert bs >= 16 and nb >= 64 and nb < (1 << 21), "the 6-byte CDBs address the whole device"
    rng = np.random.default_rng(seed)
    b = abi.Batch(target)
    cursor = [0]
    pay = []

    def buf(n: int, skew: int | None = None) -> int:
        o = (cursor[0] + 127) // 64 * 64 + (int(rng.integers(0, 16)) if skew is None else skew)
        cursor[0] = o + n
        return o

    def one(n: int, skew: int | None = None) -> list:
        return [(buf(n, skew), n)]

    stub = min(bs, 4096)                     # SG of a request refused before any data moves

    def pad():
        """READ CAPACITY 10 / 16 up to the next pass boundary"""
        while len(b) % abi.REQS_PER_PASS:
            six = len(b) % 2 == 0
            b.add(abi.cdb_read_capacity(six, 32), abi.DIR_FROM_DEV, one(32 if six else 8))

    def unmap(descs):
        pl = abi.unmap_param_list(descs)
        off = buf(len(pl))
        pay.append((off, pl))
        b.add(abi.cdb_unmap(len(pl)), abi.DIR_TO_DEV, [(off, len(pl))])

    rd = {6: abi.READ_6, 10: abi.READ_10, 12: abi.READ_12, 16: abi.READ_16}
    wr = {6: abi.WRITE_6, 10: abi.WRITE_10, 12: abi.WRITE_12, 16: abi.WRITE_16}

    # every CDB width at 1 block and at the transfer limit, at both ends of the device
    for width in (6, 10, 12, 16):
        for d in (abi.DIR_FROM_DEV, abi.DIR_TO_DEV):
            op = (rd if d == abi.DIR_FROM_DEV else wr)[width]
            top = min(mx, 255) if width == 6 else mx
            for n in sorted({1, top}):
                for lba in sorted({0, nb - n}):
                    b.add(abi.cdb_rw(op, lba, n), d, one(n * bs))
                b.add(abi.cdb_rw(op, nb - n + 1, n), d, one(stub))
            if width != 6 or mx + 1 <= 255:
                b.add(abi.cdb_rw(op, 0, mx + 1), d, one(stub))

    # READ(6) / WRITE(6) length byte 0: 256 blocks, or one block's SG where 256 blocks are over the limit
    sg256 = 256 * bs if 256 <= mx else bs
    for op, d in ((abi.READ_6, abi.DIR_FROM_DEV), (abi.WRITE_6, abi.DIR_TO_DEV)):
        for lba in sorted({x for x in (0, nb - 256, nb - 255) if x >= 0}):
            b.add(abi.cdb_rw(op, lba, 0), d, one(sg256))
    b.add(abi.cdb_sync(abi.SYNCHRONIZE_CACHE_10, 0, 0), abi.DIR_FROM_DEV, [])
    b.add(abi.cdb_sync(abi.SYNCHRONIZE_CACHE_16, nb - 4, 0), abi.DIR_FROM_DEV, [])
    pad()

    # passes mixing requests over one fill with one-block ones
    big = max(1, (3 << 20) // bs)            # about 3 MiB
    big2 = FILL_BYTES // bs + 1              # just over one fill
    x, y, z = nb // 8, 3 * nb // 8, 5 * nb // 8
    far = nb - nb // 8

    def small(k, lo):
        for i in range(k):
            b.read(lo + (7 * i) % (nb // 8 - 1), 1, one(bs), opcode=abi.READ_16)

    b.write(x, big, one(big * bs), opcode=abi.WRITE_16)           # big first: small READs inside it follow
    for lba in (x, x + big // 2, x + big - 1):
        b.read(lba, 1, one(bs), opcode=abi.READ_16)
    small(3, far)
    pad()
    for lba in (x + big - 1, x + 1 if big > 1 else x):            # next pass: the big WRITE's blocks again
        b.read(lba, 1, one(bs), opcode=abi.READ_16)
    for i, lba in enumerate((y, y + big // 2, y + big - 1)):      # small WRITEs, then a big READ over them
        b.write(lba, 1, one(bs, 3 * i + 1), opcode=abi.WRITE_16)
    small(2, far)
    b.read(y, big, one(big * bs), opcode=abi.READ_16)             # big in the middle
    small(2, far)
    pad()
    small(3, far)
    b.write(z, big2, one(big2 * bs), opcode=abi.WRITE_16)         # two big ones: a big WRITE over a big WRITE,
    small(2, far)
    b.write(z + big2 // 2, big2, one(big2 * bs), opcode=abi.WRITE_16)   # the second one last
    pad()
    b.read(z, big2 + big2 // 2, one((big2 + big2 // 2) * bs), opcode=abi.READ_16)
    b.read(z + big2 // 2, 1, one(bs), opcode=abi.READ_16)
    pad()

    # SG shapes: block-sized elements up to the 129-element limit, 130 (invalid), odd cuts, runs across 4 KiB
    sgl = x + big + 8
    k = min(abi.IOVS_MAX, mx)
    b.read(sgl, k, [(buf(bs, i % 16), bs) for i in range(k)], opcode=abi.READ_16)
    b.write(sgl + k, k, [(buf(bs, (5 * i) % 16), bs) for i in range(k)], opcode=abi.WRITE_16)
    n130 = abi.IOVS_MAX + 1
    if n130 <= mx:
        b.read(sgl, n130, [(buf(bs), bs) for i in range(n130)], opcode=abi.READ_16)
    else:
        cut = [bs // n130] * (n130 - 1)
        b.read(sgl, 1, [(buf(c), c) for c in cut + [bs - sum(cut)]], opcode=abi.READ_16)
    for d in (abi.DIR_FROM_DEV, abi.DIR_TO_DEV):                 # separate elements cut at odd bytes inside a block
        nblk = 2 if 2 <= mx else 1
        edges = sorted({0, 1, 7, bs - 3, bs + 5 if nblk > 1 else bs - 1, nblk * bs})
        els = [(buf(e1 - e0), e1 - e0) for e0, e1 in zip(edges[:-1], edges[1:])]
        (b.read if d == abi.DIR_FROM_DEV else b.write)(sgl + 2 * k + 4 * (d == abi.DIR_TO_DEV), nblk, els,
                                                          opcode=abi.READ_16 if d == abi.DIR_FROM_DEV else abi.WRITE_16)
    nrun = -(-20000 // bs)                                      # one buffer cut across 4 KiB: elements that continue
    if nrun <= mx:
        tot = nrun * bs
        for d, skew in ((abi.DIR_TO_DEV, 9), (abi.DIR_FROM_DEV, 6)):
            base = buf(tot, skew)
            edges = sorted({e for e in (0, 4000, 4100, 8191, 8193, 12289, 16380) if e < tot} | {tot})
            els = [(base + e0, e1 - e0) for e0, e1 in zip(edges[:-1], edges[1:])]
            (b.read if d == abi.DIR_FROM_DEV else b.write)(sgl + 2 * k + 12, nrun, els, opcode=abi.READ_16 if d == abi.DIR_FROM_DEV else abi.WRITE_16)
    pad()
    many = max(1, -(-abi.IOVS_MAX * 64 // bs))                  # three requests of 129 separate elements: > 256 segments
    tot = many * bs
    cut = [tot // abi.IOVS_MAX] * (abi.IOVS_MAX - 1)
    cut.append(tot - sum(cut))
    seg0 = sgl + 2 * k + 40
    for i in range(3):
        els = [(buf(c), c) for c in cut]
        if i == 1:
            b.write(seg0 + i * many, many, els, opcode=abi.WRITE_16)
        else:
            b.read(seg0 + i * many, many, els, opcode=abi.READ_16)
    b.read(seg0 + many, many, one(tot), opcode=abi.READ_16)      # what the WRITE of 129 elements left
    pad()

    # UNMAP: a many-MiB descriptor, 256 one-block descriptors, a list that fails part-way; then reads of them
    u = nb // 2
    ucnt = min(nb // 8, max(2, (8 << 20) // bs))
    v = (u + ucnt + 4) % nb
    w = (v + 520) % (nb - 8)
    unmap([(u, ucnt)])
    b.read(u, 1, one(bs), opcode=abi.READ_16)
    b.read(u + ucnt - 1, 1, one(bs), opcode=abi.READ_16)
    unmap([((v + 2 * i) % nb, 1) for i in range(256)])
    b.read(v, min(4, mx), one(min(4, mx) * bs), opcode=abi.READ_16)
    unmap([(w, 2), (nb - 1, 4), (w + 4, 2)])
    b.read(w, 1, one(bs), opcode=abi.READ_16)
    pad()
    two = min(2, mx)
    b.read(u + 1 - two, two, one(two * bs), opcode=abi.READ_16)   # across the start and the end of the extent
    b.read(u + ucnt - 1, two, one(two * bs), opcode=abi.READ_16)
    b.read((v + 2) % nb, 1, one(bs), opcode=abi.READ_16)
    b.read(w, min(6, mx), one(min(6, mx) * bs), opcode=abi.READ_16)
    pad()

    # the whole device, then reads of it and writes after it
    unmap([(0, nb)])
    b.read(0, 1, one(bs), opcode=abi.READ_16)
    b.read(nb - 1, 1, one(bs), opcode=abi.READ_16)
    pad()
    b.read(nb // 2, min(2, mx), one(min(2, mx) * bs), opcode=abi.READ_16)
    b.write(1, min(3, mx), one(min(3, mx) * bs), opcode=abi.WRITE_16)
    b.write(nb - mx, mx, one(mx * bs), opcode=abi.WRITE_16)
    b.read(0, min(4, mx), one(min(4, mx) * bs), opcode=abi.READ_16)
    pad()
    reqs, iovs = b.arrays()
    t = Trace(reqs, iovs, cursor[0] + 4096, f"block-size-{bs}", {"n": len(reqs)})
    t.meta["param_payloads"] = pay
    return t


def _param_iovs(alloc, payload: np.ndarray, rng) -> list[tuple[int, int]]:
    """SG list for a TO_DEV parameter list (UNMAP): one element, or cut in two at a ragged spot."""
    n = len(payload)
    if n > 10 and rng.integers(0, 2):
        cut = int(rng.integers(1, n))
        return [(alloc(cut, 1), cut), (alloc(n - cut, 1), n - cut)]
    return [(alloc(n, 1), n)]


def _stash_payload(b: "abi.Batch", payload: np.ndarray) -> None:
    """remember (arena offset, bytes) of a parameter list so the arena can be initialised with it"""
    lst = getattr(b, "_payloads", None)
    if lst is None:
        lst = b._payloads = []
    *_, cnt, start = b._reqs[-1]
    pos = 0
    for a, l in b._iovs[start:start + cnt]:
        lst.append((a, payload[pos:pos + l].copy()))
        pos += l


def fill_arena(arena: np.ndarray, trace: Trace, seed: int = 0x5EED) -> None:
    """Initialise a host arena: position-keyed pattern everywhere, then the parameter lists
    (UNMAP descriptors) the fuzz trace stashed."""
    arena[:] = pattern_bytes(seed, 0, arena.size)
    for off, data in trace.meta.get("param_payloads", []):
        arena[off:off + len(data)] = data


def primary_trace(n: int, *, seed: int = 1, target: int = 0, arena_bytes: int = 4 << 20) -> Trace:
    """SPC primary commands a guest issues while attaching a disk (S/lib/scsi/scsi_bdev.c:1827-2077):
    INQUIRY (standard + every VPD page, good and bad allocation lengths), REPORT LUNS, MODE SENSE 6/10
    over all page / subpage / page-control combinations, MODE SELECT 6/10, with SG lists that are
    larger, equal and smaller than the allocation length."""
    rng = np.random.default_rng(seed)
    b = abi.Batch(target)
    cur = [64]

    def alloc(nbytes, align=1):
        o = -(-cur[0] // align) * align
        cur[0] = o + nbytes
        return o

    def sg(total):
        if total == 0:
            return [] if rng.integers(0, 2) else [(alloc(0), 0)]
        k = int(rng.integers(1, 4))
        cuts = sorted(set(int(x) for x in rng.integers(1, total + 1, size=k - 1))) if k > 1 and total > 1 else []
        edges = [0] + [c for c in cuts if 0 < c < total] + [total]
        return [(alloc(z - a + 8) + int(rng.integers(0, 8)), z - a) for a, z in zip(edges[:-1], edges[1:])]

    def payload_len(alloc_len):
        return int(rng.choice([alloc_len, alloc_len, max(0, alloc_len - int(rng.integers(1, 9))), alloc_len + 13, 4096]))

    payloads = []
    for _ in range(n):
        c = np.zeros(abi.CDB_SIZE, dtype=np.uint8)
        kind = int(rng.integers(0, 10))
        if kind < 4:                                     # INQUIRY
            c[0] = 0x12
            al = int(rng.choice([0, 5, 35, 36, 40, 55, 56, 57, 58, 59, 60, 62, 64, 66, 67, 74, 96, 128, 255, 618, 619, 1024, 4096, 8192]))
            c[3:5] = [al >> 8, al & 0xFF]
            if rng.integers(0, 3):
                c[1] = 1
                c[2] = int(rng.choice([0x00, 0x80, 0x83, 0x85, 0x86, 0x87, 0x88, 0xB0, 0xB1, 0xB2, 0x84, 0xC5, 0x01]))
            elif rng.integers(0, 6) == 0:
                c[2] = 0x80                              # page code without EVPD
            b.add(c, abi.DIR_FROM_DEV, sg(payload_len(al)))
        elif kind < 5:                                   # REPORT LUNS
            c[0] = 0xA0
            c[2] = int(rng.choice([0, 1, 2, 3, 0x11]))
            al = int(rng.choice([0, 8, 15, 16, 24, 4096, 70000]))
            c[6:10] = list(al.to_bytes(4, "big"))
            b.add(c, abi.DIR_FROM_DEV, sg(min(payload_len(al), 8192)))
        elif kind < 8:                                   # MODE SENSE 6 / 10
            six = bool(rng.integers(0, 2))
            c[0] = 0x1A if six else 0x5A
            c[1] = (0x08 if rng.integers(0, 2) else 0) | (0x10 if rng.integers(0, 2) else 0)
            pc = int(rng.choice([0, 0, 1, 2, 3]))
            page = int(rng.choice([0x00, 0x01, 0x02, 0x03, 0x07, 0x08, 0x0A, 0x10, 0x1A, 0x1C, 0x20, 0x3E, 0x3F]))
            c[2] = pc << 6 | page
            c[3] = int(rng.choice([0x00, 0x00, 0x01, 0x02, 0xFF]))
            al = int(rng.choice([0, 4, 8, 12, 24, 36, 64, 192, 255])) if six else int(rng.choice([0, 8, 16, 24, 64, 200, 512, 4096]))
            if six:
                c[4] = al
            else:
                c[7:9] = [al >> 8, al & 0xFF]
            b.add(c, abi.DIR_FROM_DEV, sg(payload_len(al)))
        else:                                            # MODE SELECT 6 / 10
            six = bool(rng.integers(0, 2))
            c[0] = 0x15 if six else 0x55
            c[1] = 0x10 if rng.integers(0, 2) else 0     # PF
            md = 4 if six else 8
            pllen = int(rng.choice([0, 2, md, md + 2, md + 8 + 20, 64]))
            if six:
                c[4] = pllen
            else:
                c[7:9] = [pllen >> 8, pllen & 0xFF]
            body = np.zeros(max(pllen, 1), dtype=np.uint8)
            if pllen >= md + 8 + 20 and rng.integers(0, 2):
                if six:
                    body[3] = 8                          # block descriptor length
                else:
                    body[6:8] = [0, 8]
                body[md + 8] = 0x08                      # caching page
                body[md + 8 + 1] = 0x12
            dlen = int(rng.choice([pllen, pllen, max(0, pllen - 3), pllen + 5])) if pllen else int(rng.choice([0, 8]))
            iov = sg(dlen)
            b.add(c, abi.DIR_TO_DEV, iov)
            pos = 0
            for a, l in iov:
                seg = np.zeros(l, dtype=np.uint8)
                take = body[pos:pos + l]
                seg[:len(take)] = take
                payloads.append((a, seg))
                pos += l
    reqs, iovs = b.arrays()
    t = Trace(reqs, iovs, max(arena_bytes, cur[0] + 4096), f"primary-{seed}", {"n": n})
    t.meta["param_payloads"] = payloads
    return t
