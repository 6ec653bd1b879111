"""The block-I/O channel (oimgpu_bio_chan, oim_b200/csrc/bio_chan.cu) compared with a host model of its contract
(include/oimgpu.h).

`model_batch` restates the channel in numpy: each bio is checked as the header states, in the channel's order (the
-EINVAL classes, then -EFAULT), the valid ones are applied in submission order to host images of the store and of
every client arena, and the launch-split rule gives the number of oim_bio_kernel launches.  `gen_schedule` draws
seeded batches and submit / poll schedules; the GPU tests run them through the C ABI on every client memory kind and
compare completions, every byte of every arena (guards included), the whole store and the launch count.

Client memory that is neither registered nor device memory is pinned page by page (oimgpu_mem_ensure); the tests
that check that on ranges straddling another owner's registration launch nothing, and the data tests submit such
ranges only after the same check has passed."""
import ctypes as C
import errno
import mmap

import numpy as np
import pytest

from oim_b200 import abi

EINVAL, EFAULT = -errno.EINVAL, -errno.EFAULT
PAGE = 4096
UNIT = 4096                     # the kernel's unit: a warp moves one 4 KiB piece of a segment
GUARD = 4096                    # bytes before and after the used part of every arena
MAX_UNITS_PER_LAUNCH = 1 << 30

# client memory kinds; the generator's addresses are kind << 40 | offset, the test maps them onto real arenas
REG, PINNED, DEV, PAGEABLE, STRADDLE, UNMAPPED = 1, 2, 3, 4, 5, 6
KIND_NAMES = {REG: "registered", PINNED: "torch-pinned", DEV: "cuda", PAGEABLE: "pageable", STRADDLE: "straddle",
              UNMAPPED: "unmapped"}
KIND_CAP = {REG: 16 << 20, PINNED: 16 << 20, DEV: 48 << 20, PAGEABLE: 8 << 20, STRADDLE: 8 << 20}
# STRADDLE arenas: in every 8 pages, pages 0-2 are registered with oimgpu_mem_register and pages 3-7 are pageable
SECTION, SECTION_REG = 8, 3
# UNMAPPED pieces sit below the lowest address a process may map: pinning them fails (-EFAULT), nothing moves
UNMAPPED_AT = 0x1000

INVALID_CLASSES = ("op", "flags", "offset-past-end", "end-past-end", "offset-wraps", "iovcnt-past-table",
                   "iov-end-past-table", "iov-start-past-table", "iov-flags", "iov-null", "one-byte-short")
TABLE_CLASSES = ("iovcnt-past-table", "iov-end-past-table", "iov-start-past-table")
LIST_CLASSES = TABLE_CLASSES + ("iov-flags", "iov-null", "one-byte-short", "efault")      # READ / WRITE only
BLOCK_SIZES = (512, 520, 4096, 4097, 64 << 10, 1 << 20)
POLL_MAX = (1, 7, 64, None)     # None: everything in flight


def kind_of(addr):
    return int(addr) >> 40


def offset_of(addr):
    return int(addr) & ((1 << 40) - 1)


def vaddr(kind, off):
    return (kind << 40) | off


# ---- the model ------------------------------------------------------------------------------------------------

def bio_pieces(b, iovs, block_size):
    """the (client address, bytes) pieces a READ / WRITE moves, in store order: the iovecs cut where the bio ends,
    empty pieces dropped"""
    left = int(b["num_blocks"]) * block_size
    out = []
    for v in iovs[int(b["iov_start"]):int(b["iov_start"]) + int(b["iovcnt"])]:
        if not left:
            break
        take = min(int(v["len"]), left)
        if take:
            out.append((int(v["addr"]), take))
            left -= take
    return out


def bio_status(b, iovs, num_blocks, block_size, reachable=lambda a, n: kind_of(a) != UNMAPPED):
    """0 or -errno, in emit_bio's order: op and flags, the range, the iovec table, each iovec until the bio's bytes
    are covered, the total; then whether each piece can be made accessible to the GPU"""
    op, off, n = int(b["op"]), int(b["offset_blocks"]), int(b["num_blocks"])
    if op > abi.BIO_UNMAP or int(b["flags"]) != 0:
        return EINVAL
    if off > num_blocks or n > num_blocks - off:
        return EINVAL
    if op in (abi.BIO_WRITE_ZEROES, abi.BIO_UNMAP):
        return 0
    start, cnt = int(b["iov_start"]), int(b["iovcnt"])
    if cnt > len(iovs) or start > len(iovs) - cnt:
        return EINVAL
    need, have = n * block_size, 0
    for v in iovs[start:start + cnt]:
        if have >= need:
            break
        if int(v["flags"]) != 0 or (int(v["len"]) and not int(v["addr"])):
            return EINVAL
        have += int(v["len"])
    if have < need:
        return EINVAL
    if not all(reachable(a, t) for a, t in bio_pieces(b, iovs, block_size)):
        return EFAULT
    return 0


def model_batch(bios, iovs, store, arenas, block_size):
    """apply one batch to the host images (store: the bdev's bytes; arenas: kind -> bytes at offset_of(addr)).
    Returns (statuses, launches)."""
    num_blocks = len(store) // block_size
    status = np.zeros(len(bios), dtype=np.int32)
    launches, units = 0, 0
    g_lo, g_hi, g_w = [], [], []
    for i, b in enumerate(bios):
        st = bio_status(b, iovs, num_blocks, block_size)
        status[i] = st
        n = int(b["num_blocks"]) * block_size
        if st or not n:
            continue
        op = int(b["op"])
        lo = int(b["offset_blocks"]) * block_size
        if op in (abi.BIO_WRITE_ZEROES, abi.BIO_UNMAP):
            store[lo:lo + n] = 0
            bio_units = -(-n // UNIT)
        else:
            pos, bio_units = lo, 0
            for a, t in bio_pieces(b, iovs, block_size):
                arena, o = arenas[kind_of(a)], offset_of(a)
                if op == abi.BIO_READ:
                    arena[o:o + t] = store[pos:pos + t]
                else:
                    store[pos:pos + t] = arena[o:o + t]
                pos += t
                bio_units += -(-t // UNIT)
        # a launch ends before a bio whose store range overlaps one of the launch's where one of the two writes
        writes = op != abi.BIO_READ
        lo_a, hi_a, w_a = np.array(g_lo, dtype=np.int64), np.array(g_hi, dtype=np.int64), np.array(g_w, dtype=bool)
        conflict = bool(((lo < hi_a) & (lo_a < lo + n) & (writes | w_a)).any())
        if conflict or units + bio_units > MAX_UNITS_PER_LAUNCH:
            launches += 1
            units, g_lo, g_hi, g_w = 0, [], [], []
        g_lo.append(lo)
        g_hi.append(lo + n)
        g_w.append(writes)
        units += bio_units
    return status, launches + (units > 0)


# ---- the generator --------------------------------------------------------------------------------------------

def device_blocks(block_size):
    """a device of about 8 MiB: every block size fits a whole-device bio into one arena"""
    return max(8, (8 << 20) // block_size)


class _Batch:
    def __init__(self):
        self.rows, self.iovs, self.fix = [], [], []      # fix: (row, class) whose table indices depend on its size
        self.classes = []                                # per row: "valid", an INVALID_CLASSES name, "efault", ...


class Schedule:
    """batches (bios, iovs) of one channel, the rounds they are submitted in ((batches, poll max, share of the
    completions left in flight), ...), the device
    and the arena bytes each kind needs; plus what each bio was drawn as, for the coverage test"""

    def __init__(self, seed, block_size, num_blocks):
        self.seed, self.block_size, self.num_blocks = seed, block_size, num_blocks
        self.batches, self.rounds, self.classes = [], [], []
        self.arena_bytes = {}


class _Gen:
    def __init__(self, seed, block_size, kinds):
        self.rng = np.random.default_rng(seed)
        self.bs = block_size
        self.nb = device_blocks(block_size)
        self.kinds = kinds
        self.cur = {k: GUARD for k in kinds}
        self.sources = {k: [] for k in kinds}            # WRITE source spans: other WRITEs may read them again
        self.recent = []                                  # (lo, hi) block ranges of recent bios, for overlaps
        self.many = 0.05                                  # share of READ / WRITE bios with up to 300 pieces
        self.tag = 1 << 40

    def place(self, kind, n, write):
        """offset of n fresh (or, for a WRITE, possibly shared) client bytes of `kind`"""
        r = self.rng
        if kind == UNMAPPED:
            return UNMAPPED_AT + int(r.integers(0, 16))
        if write and self.sources[kind] and r.random() < 0.3:
            a, ln = self.sources[kind][int(r.integers(len(self.sources[kind])))]
            if ln >= n:
                return a + int(r.integers(0, ln - n + 1))
        pos = self.cur[kind] + int(r.integers(0, 16))     # every address mod 16
        if kind == STRADDLE and n > 1:
            # begin 1 .. 4095 bytes before the next edge of a registered section: the piece straddles it
            sec = SECTION * PAGE
            e = min(x for x in (pos // sec * sec + SECTION_REG * PAGE, (pos // sec + 1) * sec) if x > pos)
            pos = max(pos, e - int(r.integers(1, min(n, PAGE))))
        self.cur[kind] = pos + n
        if write:
            self.sources[kind].append((pos, n))
        return pos

    def pick_kind(self, need, npieces):
        """a kind with room for a bio of `need` bytes in `npieces` pieces (STRADDLE pieces may skip a section)"""
        def room(k):
            extra = npieces * (16 + (SECTION * PAGE if k == STRADDLE else 0)) + 3 * PAGE
            return KIND_CAP[k] - GUARD - self.cur[k] - extra
        ok = [k for k in self.kinds if k != UNMAPPED and room(k) >= need]
        return int(self.rng.choice(ok)) if ok else None

    def cut(self, need, npieces):
        """lengths of npieces pieces summing to need; equal cut points give empty pieces"""
        r = self.rng
        if npieces == 1:
            return [need]
        pts = np.sort(r.integers(0, need + 1, npieces - 1))
        if r.random() < 0.3:                               # a cut on a 4 KiB unit of the store side
            pts[-1] = min(need, UNIT * int(r.integers(1, 4)))
            pts = np.sort(pts)
        return [int(x) for x in np.diff(np.concatenate([[0], pts, [need]]))]

    def blocks(self):
        """(offset, num_blocks) of a bio"""
        r, nb = self.rng, self.nb
        x = r.random()
        if x < 0.03:
            return 0, nb                                    # the whole device
        if x < 0.06:
            return int(r.choice([0, nb])), 0                # 0 blocks, at either end
        if x < 0.35 and self.recent:                        # overlap a recent bio
            lo, hi = self.recent[int(r.integers(max(0, len(self.recent) - 8), len(self.recent)))]
            n = int(r.integers(1, min(nb, 2 * (hi - lo)) + 1))
            return int(np.clip(int(r.integers(lo - n + 1, hi)), 0, nb - n)), n
        cap = max(1, min(nb, (256 << 10) // self.bs))
        n = int(r.integers(1, cap + 1)) if r.random() < 0.3 else int(r.integers(1, min(cap, 4) + 1))
        return (int(r.choice([0, nb - n])) if r.random() < 0.15 else int(r.integers(0, nb - n + 1))), n

    def bio(self, bt, cls):
        """append one bio of class cls ("valid", "zero-blocks", "efault" or an INVALID_CLASSES name) to batch bt.
        Pieces of bios that must fail before anything is pinned point at unmapped memory: were they pinned, the
        bio would complete with -EFAULT instead."""
        r, nb, bs = self.rng, self.nb, self.bs
        op = int(r.choice([abi.BIO_READ, abi.BIO_WRITE, abi.BIO_READ, abi.BIO_WRITE, abi.BIO_WRITE_ZEROES, abi.BIO_UNMAP]))
        off, n = self.blocks()
        if cls == "zero-blocks":
            off, n = int(r.choice([0, nb, int(r.integers(0, nb))])), 0
        if cls in LIST_CLASSES:
            op = int(r.choice([abi.BIO_READ, abi.BIO_WRITE]))
            if cls in ("efault", "iov-flags", "iov-null", "one-byte-short") and n == 0:
                off, n = int(r.integers(0, nb)), 1
        need, kind = n * bs, None
        npieces = (300 if r.random() < 0.3 else int(r.integers(1, 300))) if r.random() < self.many else int(r.integers(1, 5))
        npieces = max(1, min(npieces, need)) if need else int(r.integers(0, 3))
        if op in (abi.BIO_READ, abi.BIO_WRITE) and need and cls in ("valid", "efault"):
            kind = self.pick_kind(need, npieces)
            if kind is None and cls == "valid":           # no room left: the same range, with no payload
                op = int(r.choice([abi.BIO_WRITE_ZEROES, abi.BIO_UNMAP]))
        flags, start, cnt = 0, len(bt.iovs), 0
        if op in (abi.BIO_READ, abi.BIO_WRITE):
            lens = self.cut(need, npieces) if need else [int(r.integers(0, 64)) for _ in range(npieces)]
            if lens and r.random() < 0.15:                # an empty piece in the middle of the list
                lens.insert(int(r.integers(0, len(lens) + 1)), 0)
            tail = None
            if cls == "one-byte-short":
                j = max(i for i, x in enumerate(lens) if x)
                lens[j] -= 1
            elif need and r.random() < 0.2:               # the list holds more bytes than the bio
                if r.random() < 0.5:
                    lens[-1] += int(r.integers(1, 2 * PAGE))
                else:
                    lens.append(int(r.integers(1, 2 * PAGE)))
                    tail = len(lens) - 1
            pieces = []
            for j, ln in enumerate(lens):
                k = kind if kind is not None and not (cls == "efault" and j >= len(lens) // 2) else UNMAPPED
                pieces.append([vaddr(k, self.place(k, ln, op == abi.BIO_WRITE)), ln, 0])
            if cls in ("iov-flags", "iov-null"):
                # one of the iovecs looked at before the bio's bytes are covered
                pre = np.cumsum([0] + lens[:-1])
                j = int(r.choice([i for i in range(len(lens)) if pre[i] < need]))
                if cls == "iov-flags":
                    pieces[j][2] = int(r.integers(1, 1 << 32))
                else:
                    pieces[j][0], pieces[j][1] = 0, max(1, pieces[j][1])
            elif tail is not None and r.random() < 0.5:   # past the bio's end an iovec is never looked at
                pieces[tail][2] = 1
            bt.iovs += pieces
            cnt = len(pieces)
        if cls == "op":
            op = int(r.choice([4, 5, 255, 1 << 31]))
        elif cls == "flags":
            flags = int(r.choice([1, 2, 1 << 31]))
        elif cls == "offset-past-end":
            off, n = nb + int(r.integers(1, 4)), int(r.integers(0, 3))
        elif cls == "end-past-end":
            n = int(r.integers(1, min(nb, 8) + 1))
            off = nb - n + 1
        elif cls == "offset-wraps":
            off, n = (1 << 64) - int(r.integers(1, 3)), int(r.integers(1, 4))
        elif cls in TABLE_CLASSES:
            bt.fix.append((len(bt.rows), cls))
        bt.rows.append((off, n, op, start, cnt, flags, self.tag))
        bt.classes.append(cls)
        self.tag += 1
        if n and cls == "valid":
            self.recent.append((off, off + n))

    def batch(self, nbios, min_segs=0):
        """nbios bios (more, up to 5000, until about min_segs segments), 80 % valid, the rest of every other class"""
        bt, r = _Batch(), self.rng
        others = list(INVALID_CLASSES) + ["efault", "zero-blocks"]
        self.many = 0.5 if min_segs else 0.05
        segs = 0
        while len(bt.rows) < nbios or (segs < min_segs and len(bt.rows) < 5000):
            cls = "valid" if r.random() < 0.8 or not bt.rows else str(r.choice(others))
            before = len(bt.iovs)
            self.bio(bt, cls)
            segs += max(1, len(bt.iovs) - before) if cls == "valid" else 0
        iovs = np.zeros(max(1, len(bt.iovs)), dtype=abi.iov_dtype)
        for i, v in enumerate(bt.iovs):
            iovs[i] = tuple(v)
        rows = np.zeros(len(bt.rows), dtype=abi.bio_dtype)
        for i, row in enumerate(bt.rows):
            rows[i] = row
        niov = len(iovs)
        for i, cls in bt.fix:
            if cls == "iovcnt-past-table":
                rows[i]["iov_start"], rows[i]["iovcnt"] = 0, niov + int(r.integers(1, 3))
            elif cls == "iov-end-past-table":              # iov_start inside the table, the list past its end
                cnt = int(r.integers(1, niov + 1))
                rows[i]["iovcnt"], rows[i]["iov_start"] = cnt, niov - cnt + int(r.integers(1, cnt + 1))
            else:
                rows[i]["iov_start"], rows[i]["iovcnt"] = niov + int(r.integers(1, 3)), 0
        return rows, iovs, bt.classes


def gen_schedule(seed, block_size, huge_batch=False):
    """one channel's batches and the rounds they are submitted in.  The first round holds a 1-bio batch, a small one,
    one of over 1024 segments and one of over 4096 (each regrows a staging buffer and the device array while the
    batch before it is in flight); huge_batch adds a batch of 5000 bios; then rounds of 8, 1 and 1 .. 8 batches.
    Rounds are polled with max 1, 7, 64 or all, and all but the last leave part of their completions in flight."""
    kinds = [REG, PINNED, DEV, PAGEABLE, STRADDLE, UNMAPPED]
    g = _Gen(seed, block_size, kinds)
    r = g.rng
    s = Schedule(seed, block_size, g.nb)
    plan = [(1, 0), (int(r.integers(2, 40)), 0), (600, int(r.integers(1100, 2000))), (2000, int(r.integers(4300, 4800)))]
    plan += [(5000, 0)] * huge_batch + [(int(r.integers(1, 400 if i % 4 == 0 else 40)), 0) for i in range(int(r.integers(12, 16)))]
    for nbios, segs in plan:
        rows, iovs, cls = g.batch(nbios, segs)
        s.batches.append((rows, iovs))
        s.classes.append(cls)
    rounds, left = [4, 8, 1], len(s.batches) - 13
    while left > 0:
        k = min(left, int(r.integers(1, 9)))
        rounds.append(k)
        left -= k
    polls = [POLL_MAX[i % len(POLL_MAX)] for i in range(len(rounds))]
    r.shuffle(polls)
    keep = [float(r.choice([0.0, r.random()])) for _ in rounds[:-1]] + [0.0]
    s.rounds = list(zip(rounds, polls, keep))
    s.arena_bytes = {k: g.cur[k] + GUARD for k in kinds if k != UNMAPPED}
    return s


def initial_images(s):
    """the seeded contents of the store and of every arena before the schedule"""
    r = np.random.default_rng(s.seed + 1000)
    store = r.integers(0, 256, s.num_blocks * s.block_size, dtype=np.uint8)
    arenas = {k: r.integers(0, 256, n, dtype=np.uint8) for k, n in sorted(s.arena_bytes.items())}
    return store, arenas


# ---- CPU: the model and the generator -------------------------------------------------------------------------

def _b(*rows):
    b = np.zeros(len(rows), dtype=abi.bio_dtype)
    for i, row in enumerate(rows):
        op, off, n, start, cnt = row[:5]
        b[i] = (off, n, op, start, cnt, row[5] if len(row) > 5 else 0, i)
    return b


def _v(*pieces):
    v = np.zeros(max(1, len(pieces)), dtype=abi.iov_dtype)
    for i, p in enumerate(pieces):
        v[i] = (p[0], p[1], p[2] if len(p) > 2 else 0)
    return v


def test_model_by_hand_every_invalid_class():
    bs, nb = 512, 16
    a = vaddr(REG, GUARD)
    iovs = _v((a, 1024), (a + 2000, 0), (a + 4000, 512, 7), (0, 512), (a + 8000, 511))
    cases = [
        ((abi.BIO_UNMAP + 1, 0, 1, 0, 0), EINVAL),        # bad op
        ((abi.BIO_READ, 0, 1, 0, 1, 1), EINVAL),          # reserved flags
        ((abi.BIO_WRITE_ZEROES, nb + 1, 0, 0, 0), EINVAL),  # offset past the end
        ((abi.BIO_UNMAP, nb - 2, 3, 0, 0), EINVAL),       # end past the end
        ((abi.BIO_UNMAP, (1 << 64) - 1, 2, 0, 0), EINVAL),  # offset + blocks wraps
        ((abi.BIO_READ, 0, 1, 0, 6), EINVAL),             # more iovecs than the table
        ((abi.BIO_READ, 0, 1, 4, 2), EINVAL),             # the list runs past the table's end
        ((abi.BIO_READ, 0, 0, 6, 0), EINVAL),             # the list starts past the table's end
        ((abi.BIO_WRITE, 0, 3, 0, 3), EINVAL),            # an iovec with flags before the bio is covered
        ((abi.BIO_WRITE, 0, 1, 3, 1), EINVAL),            # NULL with a length
        ((abi.BIO_READ, 0, 1, 4, 1), EINVAL),             # one byte short
        ((abi.BIO_READ, 0, 2, 0, 3), 0),                  # flags past the bio's end are never looked at
        ((abi.BIO_READ, nb, 0, 5, 0), 0),                 # 0 blocks at the end, iov_start == niovs, iovcnt 0
        ((abi.BIO_WRITE_ZEROES, nb, 0, 9, 9), 0),         # WRITE_ZEROES never looks at the iovecs
    ]
    for row, want in cases:
        assert bio_status(_b(row)[0], iovs, nb, bs) == want, (row, want)
    # -EINVAL before -EFAULT: an unmapped piece ahead of a NULL one
    bad = _v((vaddr(UNMAPPED, UNMAPPED_AT), 100), (0, 412))
    assert bio_status(_b((abi.BIO_READ, 0, 1, 0, 2))[0], bad, nb, bs) == EINVAL
    assert bio_status(_b((abi.BIO_READ, 0, 1, 0, 1))[0], _v((vaddr(UNMAPPED, UNMAPPED_AT), 512)), nb, bs) == EFAULT
    # an unmapped piece past the bio's end is never pinned
    assert bio_status(_b((abi.BIO_READ, 0, 1, 0, 2))[0], _v((a, 512), (vaddr(UNMAPPED, UNMAPPED_AT), 9)), nb, bs) == 0
    # bad bios move nothing, and their neighbours still do
    store = np.arange(nb * bs, dtype=np.uint32).astype(np.uint8)
    arenas = {REG: np.full(3 * PAGE, 0xEE, dtype=np.uint8)}
    before = store.copy()
    st, launches = model_batch(_b(*[c[0] for c in cases[:11]], (abi.BIO_READ, 3, 1, 0, 1)), iovs, store, arenas, bs)
    assert list(st) == [EINVAL] * 11 + [0] and launches == 1 and (store == before).all()
    assert (arenas[REG][GUARD:GUARD + bs] == before[3 * bs:4 * bs]).all() and (arenas[REG][GUARD + bs:] == 0xEE).all()


def test_model_by_hand_cut_and_zero_blocks():
    bs, nb = 520, 8
    store = np.zeros(nb * bs, dtype=np.uint8)
    src = np.arange(3 * PAGE, dtype=np.uint32).astype(np.uint8)
    arenas = {REG: src.copy(), DEV: np.full(3 * PAGE, 0x5A, dtype=np.uint8)}
    a, d = vaddr(REG, 0), vaddr(DEV, 0)
    # WRITE 2 blocks from 3 pieces that hold 1040 + 100 bytes: the last piece is cut after 40 of its 140
    iovs = _v((a + 3, 700), (a + 1000, 0), (a + 800, 300), (a + 2000, 140), (d + 5, 1100), (d + 2000, 7))
    st, launches = model_batch(_b((abi.BIO_WRITE, 5, 2, 0, 4), (abi.BIO_READ, 5, 2, 4, 2), (abi.BIO_READ, 8, 0, 0, 4),
                                  (abi.BIO_WRITE, 0, 0, 0, 0), (abi.BIO_UNMAP, 8, 0, 0, 0)), iovs, store, arenas, bs)
    assert list(st) == [0] * 5 and launches == 2        # W | R: the 0-block bios neither move nor split
    want = np.concatenate([src[3:703], src[800:1100], src[2000:2040]])
    assert (store[5 * bs:7 * bs] == want).all() and (store[:5 * bs] == 0).all() and (store[7 * bs:] == 0).all()
    dev = arenas[DEV]
    assert (dev[5:1045] == want).all() and (dev[:5] == 0x5A).all() and (dev[1045:] == 0x5A).all()
    assert (arenas[REG] == src).all()


def test_model_by_hand_launch_split_of_the_six_bio_ordering_case():
    """test_spdk_bdev_module.py::test_overlapping_bios_in_one_batch_take_effect_in_order, in the model"""
    bs = 4096
    store = np.zeros(64 * bs, dtype=np.uint8)
    a, b = vaddr(REG, 0), vaddr(REG, 8 * bs)
    r1, r2, r3 = vaddr(DEV, 0), vaddr(DEV, 12 * bs), vaddr(DEV, 16 * bs)
    arenas = {REG: np.concatenate([np.full(8 * bs, 0xAA, np.uint8), np.full(8 * bs, 0xBB, np.uint8)]),
              DEV: np.zeros(20 * bs, dtype=np.uint8)}
    bios = _b((abi.BIO_WRITE, 0, 8, 0, 1), (abi.BIO_READ, 0, 12, 1, 1), (abi.BIO_WRITE, 4, 8, 2, 1),
              (abi.BIO_READ, 40, 4, 3, 1), (abi.BIO_WRITE_ZEROES, 8, 2, 0, 0), (abi.BIO_READ, 6, 4, 4, 1))
    iovs = _v((a, 8 * bs), (r1, 12 * bs), (b, 8 * bs), (r3, 4 * bs), (r2, 4 * bs))
    st, launches = model_batch(bios, iovs, store, arenas, bs)
    assert list(st) == [0] * 6 and launches == 5          # W | R | W R(40) | Z | R
    dev = arenas[DEV]
    assert (dev[:8 * bs] == 0xAA).all() and (dev[8 * bs:12 * bs] == 0).all()
    assert (dev[12 * bs:14 * bs] == 0xBB).all() and (dev[14 * bs:16 * bs] == 0).all()
    assert (store[:4 * bs] == 0xAA).all() and (store[4 * bs:8 * bs] == 0xBB).all()
    assert (store[8 * bs:10 * bs] == 0).all() and (store[10 * bs:12 * bs] == 0xBB).all()
    # a READ behind a READ of the same blocks shares the launch; behind a WRITE it does not
    assert model_batch(_b((abi.BIO_READ, 0, 1, 1, 1), (abi.BIO_READ, 0, 1, 1, 1)), iovs, store, arenas, bs)[1] == 1
    assert model_batch(_b((abi.BIO_WRITE, 0, 1, 0, 1), (abi.BIO_READ, 0, 1, 1, 1)), iovs, store, arenas, bs)[1] == 2
    assert model_batch(_b((abi.BIO_READ, 0, 1, 1, 1), (abi.BIO_UNMAP, 0, 1, 0, 0)), iovs, store, arenas, bs)[1] == 2


SEEDS = (1, 2)


def _schedules(bs):
    return [gen_schedule(seed * 1000 + bs % 997, bs, huge_batch=seed == 1) for seed in SEEDS]


def _overlap_kind(op1, op2):
    w1, w2 = op1 != abi.BIO_READ, op2 != abi.BIO_READ
    return "ww" if w1 and w2 else "raw" if w1 else "war" if w2 else None


@pytest.mark.parametrize("bs", BLOCK_SIZES)
def test_schedules_reach_every_case(bs):
    """the schedules the GPU test runs at this block size reach, together, every case the generator is there for;
    and the client bytes a READ writes are no other bio's in the whole schedule"""
    seen = set()
    for s in _schedules(bs):
        nb = s.num_blocks
        store, arenas = initial_images(s)
        assert all(n <= KIND_CAP[k] for k, n in s.arena_bytes.items()), s.arena_bytes
        spans = {k: [] for k in s.arena_bytes}        # (lo, hi, is_read) client bytes of every valid bio
        bi = 0
        for nbat, pmax, keep in s.rounds:
            seen.add(("round", nbat))
            seen.add(("poll", pmax))
            window = []                               # (batch, op, lo, hi) of the valid bios submitted together
            for _ in range(nbat):
                bios, iovs = s.batches[bi]
                cls = s.classes[bi]
                st, _ = model_batch(bios, iovs, store, arenas, bs)
                seen.add(("batch-bios", 1 if len(bios) == 1 else 5000 if len(bios) >= 5000 else "many"))
                segs = 0
                for b, x, c in zip(bios, st, cls):
                    n, off, op = int(b["num_blocks"]), int(b["offset_blocks"]), int(b["op"])
                    if c in INVALID_CLASSES:
                        assert x == EINVAL, (c, b)
                        seen.add(("mixed", c) if "valid" in cls else ("alone", c))
                        continue
                    if c == "efault":
                        seen.add(("efault", int(x)))
                    if x:
                        continue
                    if n == 0:
                        seen.add(("zero-blocks", "start" if off == 0 else "end" if off == nb else "inside"))
                        continue
                    seen.add("whole-device" if n == nb else "at-start" if off == 0 else "at-end" if off + n == nb else "inside")
                    window.append((bi, op, off, off + n))
                    if op > abi.BIO_WRITE:
                        segs += 1
                        continue
                    lst = iovs[int(b["iov_start"]):int(b["iov_start"]) + int(b["iovcnt"])]
                    seen.add(("pieces", 1 if len(lst) == 1 else 300 if len(lst) >= 300 else "2-299"))
                    if int(lst["len"].sum()) > n * bs:
                        seen.add("list-longer")
                    if len(lst) > 2 and lst["len"][0] and (lst["len"][1:-1] == 0).any():
                        seen.add("empty-piece-inside")
                    pos = off * bs
                    for a, t in bio_pieces(b, iovs, bs):
                        k, o = kind_of(a), offset_of(a)
                        segs += 1
                        seen.add(("mod16", o % 16))
                        seen.add(("kind", op, k))
                        cc, sc = o // UNIT != (o + t - 1) // UNIT, pos // UNIT != (pos + t - 1) // UNIT
                        if cc != sc:
                            seen.add(("unit-cross-only", "client" if cc else "store"))
                        if k == STRADDLE:
                            reg = [p % SECTION < SECTION_REG for p in range(o // PAGE, (o + t - 1) // PAGE + 1)]
                            if any(reg) and not all(reg):
                                seen.add(("straddle", "into" if not reg[0] else "out of"))
                                if not reg[0] and not reg[-1]:
                                    seen.add(("straddle", "both edges"))
                        spans[k].append((o, o + t, op == abi.BIO_READ))
                        pos += t
                if segs > 4096:
                    seen.add("over-4096-segments")
                bi += 1
            for i, (b1, op1, lo1, hi1) in enumerate(window):
                for b2, op2, lo2, hi2 in window[i + 1:]:
                    if lo1 < hi2 and lo2 < hi1 and _overlap_kind(op1, op2):
                        seen.add((_overlap_kind(op1, op2), "one batch" if b1 == b2 else "across batches"))
        for k, sp in spans.items():
            sp.sort()
            for (lo1, hi1, r1), (lo2, hi2, r2) in zip(sp, sp[1:]):
                if lo2 < hi1:
                    assert not (r1 or r2), (KIND_NAMES[k], lo1, hi1, lo2, hi2)
                    seen.add("shared-write-source")
    want = {("round", 1), ("round", 8), *[("poll", p) for p in POLL_MAX], ("batch-bios", 1), ("batch-bios", 5000),
            "over-4096-segments", *[("mixed", c) for c in INVALID_CLASSES], ("efault", EFAULT),
            ("zero-blocks", "start"), ("zero-blocks", "end"), "whole-device", "at-start", "at-end",
            ("pieces", 1), ("pieces", 300), "list-longer", "empty-piece-inside", *[("mod16", m) for m in range(16)],
            ("unit-cross-only", "client"), ("unit-cross-only", "store"), "shared-write-source",
            *[("kind", op, k) for op in (abi.BIO_READ, abi.BIO_WRITE) for k in (REG, PINNED, DEV, PAGEABLE, STRADDLE)],
            ("straddle", "into"), ("straddle", "out of"), ("straddle", "both edges"),
            *[(k, w) for k in ("ww", "raw", "war") for w in ("one batch", "across batches")]}
    assert not want - seen, sorted(map(str, want - seen))


# ---- GPU: client memory ---------------------------------------------------------------------------------------

_POOL = []


def _pageable(nbytes):
    """nbytes of page-aligned pageable memory no one has pinned, from 2 MiB-aligned slices of one anonymous mapping
    that lives as long as the process: the 2 MiB surroundings the library pins stay inside it, and no pin goes
    stale because its pages were unmapped"""
    big = 2 << 20
    if not _POOL:
        m = mmap.mmap(-1, 8 << 30, flags=mmap.MAP_PRIVATE | mmap.MAP_ANONYMOUS | getattr(mmap, "MAP_NORESERVE", 0x4000))
        whole = np.frombuffer(m, dtype=np.uint8)
        _POOL[:] = [m, whole, (-whole.ctypes.data) % big]
    _, whole, at = _POOL
    _POOL[2] = at + -(-nbytes // big) * big
    assert _POOL[2] <= len(whole)
    return whole[at:at + nbytes]


def _device_addr_ok(L, addr):
    d = C.c_uint64()
    return L.oimgpu_mem_device_addr(C.c_void_p(addr), C.byref(d)) == 0


# (first page, pages, owner): "lib" registers with oimgpu_mem_register, "other" with cudaHostRegister; then the range
# [lo, hi) in bytes from the buffer's start that oimgpu_mem_ensure is asked for
PIN_CASES = {
    "registered-into-pageable": ([(0, 4, "lib")], (2 * PAGE + 100, 6 * PAGE + 5)),
    "pageable-into-registered": ([(4, 4, "lib")], (1 * PAGE + 7, 6 * PAGE)),
    "other-owner-gap-registered": ([(0, 3, "other"), (5, 3, "lib")], (1 * PAGE + 3, 7 * PAGE - 9)),
    "registered-gap-registered": ([(0, 3, "lib"), (5, 3, "lib")], (1 * PAGE, 7 * PAGE)),
}


def _ensure_straddling_range(L, case):
    """oimgpu_mem_ensure on one PIN_CASES layout of fresh pageable pages; launches nothing.  Returns the pages of
    the range without a device address (they must be none)."""
    import torch
    cudart = torch.cuda.cudart()
    probe = _pageable(PAGE)
    assert not _device_addr_ok(L, probe.ctypes.data), "a page nobody pinned must have no device address"
    regs, (lo, hi) = PIN_CASES[case]
    buf = _pageable(8 * PAGE)
    base = buf.ctypes.data
    done = []
    try:
        for first, n, owner in regs:
            a = base + first * PAGE
            if owner == "lib":
                assert L.oimgpu_mem_register(C.c_void_p(a), n * PAGE) == 0
            else:
                assert cudart.cudaHostRegister(a, n * PAGE, 3) == cudart.cudaError.success     # mapped | portable
            done.append((a, owner))
        assert L.oimgpu_mem_ensure(C.c_void_p(base + lo), hi - lo) == 0
        assert L.oimgpu_mem_ensure(C.c_void_p(base + lo), hi - lo) == 0          # idempotent
        return [p for p in range(lo // PAGE, (hi - 1) // PAGE + 1)
                if not (_device_addr_ok(L, base + p * PAGE) and _device_addr_ok(L, base + p * PAGE + PAGE - 1))]
    finally:
        for a, owner in done:
            if owner == "lib":
                L.oimgpu_mem_unregister(C.c_void_p(a))
            else:
                cudart.cudaHostUnregister(a)


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(PIN_CASES))
def test_mem_ensure_pins_every_page_of_a_straddling_range(gpu, case):
    """a range that runs from a registered buffer into pageable pages, or back, or across another owner's buffer,
    or between two registered buffers: every page of it has a device address afterwards.  No launch."""
    from oim_b200 import lib
    assert _ensure_straddling_range(lib.load(), case) == [], case


class _Arenas:
    """the real client memory of a schedule: one arena per kind, page-aligned, with the model's initial bytes"""

    def __init__(self, sizes, init):
        import torch
        from oim_b200 import lib
        self.L = lib.load()
        self.base = np.zeros(UNMAPPED + 1, dtype=np.uint64)        # UNMAPPED: addresses as they are
        self.host, self.keep, self.regs = {}, [], []
        for k, n in sizes.items():
            if k == DEV:
                t = torch.empty(n + PAGE, dtype=torch.uint8, device="cuda:0")
                o = (-t.data_ptr()) % PAGE
                self.dev = t[o:o + n]
                self.dev.copy_(torch.from_numpy(init[k]))
                self.base[k] = self.dev.data_ptr()
                continue
            if k == PINNED:                                           # cudaHostAlloc: a registration not the library's
                t = torch.empty(n + PAGE, dtype=torch.uint8, pin_memory=True)
                self.keep.append(t)
                a = t.numpy()[(-t.data_ptr()) % PAGE:][:n]
            else:
                a = _pageable(n)
            a[:] = init[k]
            self.host[k] = a
            self.base[k] = a.ctypes.data
            if k == REG:
                self._register(a.ctypes.data, -(-n // PAGE) * PAGE)
            elif k == STRADDLE:
                for p in range(0, -(-n // PAGE), SECTION):
                    self._register(a.ctypes.data + p * PAGE, SECTION_REG * PAGE)

    def _register(self, addr, n):
        assert self.L.oimgpu_mem_register(C.c_void_p(addr), n) == 0
        self.regs.append(addr)

    def close(self):
        for a in self.regs:
            self.L.oimgpu_mem_unregister(C.c_void_p(a))

    def translate(self, iovs):
        out = iovs.copy()
        a = out["addr"]
        k = a >> np.uint64(40)
        out["addr"] = np.where(a != 0, self.base[k] + (a & np.uint64((1 << 40) - 1)), np.uint64(0))
        return out

    def read(self, k):
        return self.dev.cpu().numpy() if k == DEV else self.host[k].copy()


def run_schedule(gpu, s, name):
    """run s on a fresh channel; completions, launches, every arena and the store against the model"""
    store, arenas = initial_images(s)
    gpu.bdev_write_raw(name, 0, store)
    real = _Arenas(s.arena_bytes, arenas)
    try:
        with gpu.BioChan(name) as ch:
            l0 = ch.launches
            want, got, launches, inflight, bi = [], [], 0, 0, 0
            for nbat, pmax, keep in s.rounds:
                for _ in range(nbat):
                    bios, iovs = s.batches[bi]
                    bi += 1
                    st, nl = model_batch(bios, iovs, store, arenas, s.block_size)
                    want.append((bios["tag"], st))
                    launches += nl
                    ch.submit(bios, real.translate(iovs))
                    inflight += len(bios)
                target = inflight - int(inflight * keep)
                while target > 0:
                    m = pmax or inflight
                    c = ch.poll(m)
                    assert len(c) <= m
                    got.append(c)
                    target -= len(c)
                    inflight -= len(c)
            assert inflight == 0 and ch.poll(4).size == 0
            got = np.concatenate(got)
            tags, st = np.concatenate([w[0] for w in want]), np.concatenate([w[1] for w in want])
            assert (got["tag"] == tags).all(), "completions out of submission order"
            bad = np.nonzero(got["status"] != st)[0]
            assert not len(bad), [(int(tags[i]), int(got["status"][i]), int(st[i])) for i in bad[:8]]
            assert ch.launches - l0 == launches
        for k in sorted(arenas):
            diff = np.nonzero(real.read(k) != arenas[k])[0]
            assert not len(diff), (KIND_NAMES[k], len(diff), int(diff[0]), int(diff[-1]), s.arena_bytes[k])
        diff = np.nonzero(gpu.bdev_read_raw(name, 0, len(store)) != store)[0]
        assert not len(diff), ("store", len(diff), int(diff[0]) // s.block_size, int(diff[-1]) // s.block_size)
    finally:
        real.close()


GPU_RUNS = [(bs, seed) for bs in BLOCK_SIZES for seed in SEEDS]


@pytest.mark.gpu
@pytest.mark.parametrize("bs,seed", GPU_RUNS, ids=[f"bs{bs}-seed{seed}" for bs, seed in GPU_RUNS])
def test_channel_equals_the_model(gpu, bs, seed):
    """every client memory kind, straddling ranges included: those go to the GPU only once pinning is shown to
    cover every page of one (without a launch)"""
    from oim_b200 import lib
    assert _ensure_straddling_range(lib.load(), "registered-gap-registered") == []
    s = gen_schedule(seed * 1000 + bs % 997, bs, huge_batch=seed == 1)
    name = gpu.construct_malloc_bdev(s.num_blocks, bs, name=f"BioModel{bs}s{seed}")
    try:
        run_schedule(gpu, s, name)
    finally:
        gpu.delete_bdev(name)


@pytest.mark.gpu
def test_bio_over_4_gib(gpu):
    """one WRITE of more than 4 GiB from device iovecs (one of them 4 GiB - 1 bytes), read back into device memory
    with other cuts, then WRITE_ZEROES of the whole 8 GiB device"""
    import torch
    bs = 4096
    nb = (8 << 30) // bs
    name = gpu.construct_malloc_bdev(nb, bs, name="BioHuge")
    try:
        nblk = ((4 << 30) + (24 << 20)) // bs + 3
        n, off = nblk * bs, 12345
        src = torch.randint(0, 256, (n + 64,), dtype=torch.uint8, device="cuda:0")
        dst = torch.full((n + 64,), 0xA5, dtype=torch.uint8, device="cuda:0")

        def cuts(base, lens):
            lens = lens + [n - sum(lens)]
            at = np.cumsum([0] + lens[:-1])
            return _v(*[(base + int(a), ln) for a, ln in zip(at, lens)])

        with gpu.BioChan(name) as ch:
            l0 = ch.launches
            ch.submit(_b((abi.BIO_WRITE, off, nblk, 0, 4)), cuts(src.data_ptr() + 5, [4095, (1 << 32) - 1, 1 << 20]))
            assert ch.wait(1)["status"][0] == 0
            ch.submit(_b((abi.BIO_READ, off, nblk, 0, 3)), cuts(dst.data_ptr() + 3, [(1 << 32) - 8, 777]))
            assert ch.wait(1)["status"][0] == 0
            torch.cuda.synchronize()
            assert torch.equal(dst[3:3 + n], src[5:5 + n])
            assert (dst[:3] == 0xA5).all() and (dst[3 + n:] == 0xA5).all()
            assert ch.launches - l0 == 2
            del src, dst
            zeros = torch.zeros(nb * bs, dtype=torch.uint8, device="cuda:0")
            assert gpu.bdev_digest(name, offset=0, nbytes=off * bs) == gpu.digest_device(0, zeros.data_ptr(), off * bs)
            tail = (nb - off - nblk) * bs
            assert gpu.bdev_digest(name, offset=(off + nblk) * bs, nbytes=tail) == gpu.digest_device(0, zeros.data_ptr(), tail)
            ch.submit(_b((abi.BIO_WRITE_ZEROES, 0, nb, 0, 0)), _v())
            assert ch.wait(1)["status"][0] == 0
            assert gpu.bdev_digest(name) == gpu.digest_device(0, zeros.data_ptr(), nb * bs)
    finally:
        gpu.delete_bdev(name)
