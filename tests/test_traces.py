"""The trace generators the parity tests and bench.py's SG legs rely on (host logic, CPU only)."""
import numpy as np
import pytest

import util
from oim_b200 import abi, traces, vring


def continues(iov):
    """mask over elements 1..: element j starts where element j-1 (non-empty) ended"""
    return (iov["len"][:-1] > 0) & (iov["addr"][:-1] + iov["len"][:-1] == iov["addr"][1:])


def test_sg_layouts_of_the_128k_legs():
    """bench.py seq128k_sg: same 33 element lengths, three placements in client memory"""
    n, io = 6, 131072
    for sg, shift in (("unaligned", 0), ("unaligned+3", 3), ("scattered", 0)):
        t = traces.uniform_trace(n, 1 << 16, io_blocks=256, pattern="seqwrite", sg=sg)
        k = len(t.iovs) // n
        assert k == 33
        for r in range(n):
            iov = t.iovs[r * k:(r + 1) * k]
            assert list(iov["len"]) == [100] + [4096] * 31 + [3996]
            base = r * t.meta["stride"] + shift
            # the elements tile the request's buffer exactly once
            spans = sorted((int(a), int(a + l)) for a, l in zip(iov["addr"], iov["len"]))
            assert spans[0][0] == base and spans[-1][1] == base + io
            assert all(a[1] == b[0] for a, b in zip(spans[:-1], spans[1:]))
            if sg == "scattered":
                assert not continues(iov).any(), "no element may continue its predecessor"
            else:
                assert continues(iov).all(), "one buffer cut at odd bytes: every element continues the one before"


def test_fuzz_traces_with_runs_of_contiguous_elements(oracles):
    """contiguous=True: multi-element SG lists are cuts of one client buffer; contiguous=False (the default, and the
    golden vectors' generator): never.  The restatement and the compiled reference agree on both."""
    nb = 16384
    plain = traces.fuzz_trace(300, nb, seed=11)
    runs = traces.fuzz_trace(300, nb, seed=11, contiguous=True)

    def joined(t):
        c = 0
        for r in t.reqs:
            iov = t.iovs[int(r["iov_start"]):int(r["iov_start"]) + int(r["iovcnt"])]
            if len(iov) > 1:
                real = iov[(iov["addr"] & traces.NULL_ADDR_FLAG) == 0]
                c += int(continues(real).sum()) if len(real) > 1 else 0
        return c
    # (the plain generator has a few contiguous lists too - its 512-byte page lists - so the golden vectors and every
    # fuzz test exercise joined runs; contiguous=True makes them the rule, at arbitrary byte cuts)
    assert joined(runs) > 2 * joined(plain) and joined(runs) > 300
    want = util.run_oracle(oracles.PortOracle, runs, nb)
    if oracles.ref_available():
        ref = util.run_oracle(oracles.RefOracle, runs, nb)
        util.assert_cpls_equal(want[0], ref[0], runs.reqs, "runs")
        assert (want[1] == ref[1]).all() and (want[2] == ref[2]).all()
    assert (want[0]["status"] == 0).sum() > 200


def test_alignment_sweep_covers_every_skew_and_edge(oracles):
    """traces.alignment_sweep: every (client address mod 16, store offset mod 16, edge length) for READ and WRITE, each
    element its own segment, whole blocks per request; then a pass that reads and rewrites what it writes, and a pass
    that reads it back"""
    nb = 65536
    t = traces.alignment_sweep(nb)
    seen = {abi.DIR_FROM_DEV: set(), abi.DIR_TO_DEV: set()}
    lbas = []
    for r in t.reqs:
        iov = t.iovs[int(r["iov_start"]):int(r["iov_start"]) + int(r["iovcnt"])]
        assert 0 < len(iov) <= 129
        cdb = bytes(r["cdb"])
        assert cdb[0] in (abi.READ_10, abi.WRITE_10)
        lba, nblk = int.from_bytes(cdb[2:6], "big"), int.from_bytes(cdb[7:9], "big")
        assert int(iov["len"].sum()) == nblk * 512 and lba + nblk <= nb
        assert not continues(iov[iov["len"] > 0]).any(), "an element continues another: they would be one segment"
        store = 0
        for a, n in zip(iov["addr"], iov["len"]):
            seen[int(r["dir"])].add((int(a) % 16, store % 16, int(n)))
            store += int(n)
        lbas.append((lba, nblk, int(r["dir"])))
    for d in seen:
        for c in range(16):
            for s in range(16):
                dst = c if d == abi.DIR_FROM_DEV else s
                for n in traces.sweep_lengths(dst):
                    assert (c, s, n) in seen[d], (d, c, s, n)
    # the staged unit's piece split (lun_kernel.cu piece0_bytes): second piece empty at and below head + 2032
    assert {n - (16 - 3) % 16 - traces.PIECE_BODY for n in traces.sweep_lengths(3)} >= {-1, 0, 1}
    p = t.meta["hazard_pass"] * abi.REQS_PER_PASS
    assert p % abi.REQS_PER_PASS == 0 and len(t.reqs) == p + 2 * abi.REQS_PER_PASS
    w, r = lbas[p], lbas[p + 1]
    assert w[2] == abi.DIR_TO_DEV and r[2] == abi.DIR_FROM_DEV and w[:2] == r[:2], "pass p: a read behind a write"
    assert lbas[p + abi.REQS_PER_PASS][:2] == w[:2], "pass p + 1: a read of what pass p wrote"
    cpls = util.run_oracle(oracles.PortOracle, t, nb)[0]
    assert (cpls["status"] == 0).all() and (cpls["resid"] == 0).all(), "every request of the sweep is a good one"


BLOCK_SIZES = (520, 1000, 4097, 4160, 1024, 2048, 4096, 8192, 16384, 32768, 1 << 20, 4 << 20)
RW = {abi.READ_6: 6, abi.WRITE_6: 6, abi.READ_10: 10, abi.WRITE_10: 10, abi.READ_12: 12, abi.WRITE_12: 12,
      abi.READ_16: 16, abi.WRITE_16: 16}


def decode(t, arena):
    """one record per request: opcode, CDB width, LBA, blocks (READ(6) length 0 = 256), SG elements, pass, and the
    UNMAP descriptors read back from the parameter list in the arena"""
    out = []
    for i, r in enumerate(t.reqs):
        c = bytes(r["cdb"])
        iov = t.iovs[int(r["iov_start"]):int(r["iov_start"]) + int(r["iovcnt"])]
        rec = {"i": i, "op": c[0], "width": RW.get(c[0]), "pass": i // abi.REQS_PER_PASS, "iov": iov,
               "len0": False, "descs": []}
        if rec["width"] == 6:
            rec["lba"], rec["n"], rec["len0"] = int.from_bytes(c[1:4], "big") & 0x1FFFFF, c[4] or 256, c[4] == 0
        elif rec["width"] in (10, 12):
            rec["lba"] = int.from_bytes(c[2:6], "big")
            rec["n"] = int.from_bytes(c[7:9], "big") if rec["width"] == 10 else int.from_bytes(c[6:10], "big")
        elif rec["width"] == 16 or c[0] == abi.SYNCHRONIZE_CACHE_16:
            rec["lba"], rec["n"] = int.from_bytes(c[2:10], "big"), int.from_bytes(c[10:14], "big")
        elif c[0] == abi.SYNCHRONIZE_CACHE_10:
            rec["lba"], rec["n"] = int.from_bytes(c[2:6], "big"), int.from_bytes(c[7:9], "big")
        elif c[0] == abi.UNMAP:
            pl = np.concatenate([arena[int(a):int(a) + int(n)] for a, n in zip(iov["addr"], iov["len"])])
            rec["descs"] = [(int.from_bytes(bytes(pl[8 + 16 * k:16 + 16 * k]), "big"),
                             int.from_bytes(bytes(pl[16 + 16 * k:20 + 16 * k]), "big"))
                            for k in range(int.from_bytes(bytes(pl[2:4]), "big") // 16)]
        out.append(rec)
    return out


def segments(rec) -> int:
    """the mover's segments of one request: non-empty elements that do not continue their predecessor, or one per
    UNMAP descriptor"""
    if rec["descs"]:
        return sum(1 for _, n in rec["descs"] if n)
    iov = rec["iov"][rec["iov"]["len"] > 0]
    return len(iov) - int(continues(iov).sum()) if len(iov) else 0


@pytest.mark.parametrize("bs", BLOCK_SIZES)
def test_block_size_trace_covers_every_edge(oracles, bs):
    """traces.block_size_trace: each case is there, and the reference (or the restatement pinned to it) gives it the
    status it is in the trace for"""
    nb = (256 << 20) // bs
    mx = abi.MAX_XFER_BYTES // bs
    t = traces.block_size_trace(nb, bs)
    assert len(t.reqs) > abi.REQS_PER_PASS and len(t.reqs) % abi.REQS_PER_PASS == 0
    cls = oracles.RefOracle if oracles.ref_available() else oracles.PortOracle
    cpls, arena, _ = util.run_oracle(cls, t, nb, block_size=bs)
    arena0 = np.zeros(t.arena_bytes, dtype=np.uint8)
    traces.fill_arena(arena0, t)
    recs = decode(t, arena0)
    good = (cpls["resp_valid"] == 1) & (cpls["response"] == abi.S_OK) & (cpls["status"] == abi.STATUS_GOOD)

    def sense(i):
        return int(cpls["sense"][i][2]) & 0xF, int(cpls["sense"][i][12])

    def moved(rec):
        return good[rec["i"]] and cpls["resid"][rec["i"]] == 0 and int(rec["iov"]["len"].sum()) == rec["n"] * bs

    rw = [r for r in recs if r["width"]]
    reads = {abi.READ_6, abi.READ_10, abi.READ_12, abi.READ_16}
    for width in (6, 10, 12, 16):
        for is_read in (True, False):
            mine = [r for r in rw if r["width"] == width and (r["op"] in reads) == is_read and not r["len0"]]
            top = min(mx, 255) if width == 6 else mx
            for n in (1, top):
                for lba in (0, nb - n):
                    assert any(r["n"] == n and r["lba"] == lba and moved(r) for r in mine), (width, is_read, n, lba)
                oor = [r for r in mine if r["n"] == n and r["lba"] == nb - n + 1]
                assert oor and all(sense(r["i"]) == (abi.SK_ILLEGAL_REQUEST, abi.ASC_LBA_OUT_OF_RANGE) for r in oor)
            if width != 6 or mx + 1 <= 255:
                over = [r for r in mine if r["n"] == mx + 1]
                assert over and all(sense(r["i"]) == (abi.SK_ILLEGAL_REQUEST, abi.ASC_INVALID_FIELD_IN_CDB) for r in over)
    # READ(6) / WRITE(6) with length byte 0: 256 blocks where they fit, refused where they are over the limit
    for op in (abi.READ_6, abi.WRITE_6):
        l0 = {r["lba"]: r for r in rw if r["len0"] and r["op"] == op}
        if nb >= 256:
            want = None if 256 <= mx else (abi.SK_ILLEGAL_REQUEST, abi.ASC_INVALID_FIELD_IN_CDB)
            for lba in (0, nb - 256):
                assert moved(l0[lba]) if want is None else sense(l0[lba]["i"]) == want, (op, lba)
            assert sense(l0[nb - 255]["i"]) == (abi.SK_ILLEGAL_REQUEST, abi.ASC_LBA_OUT_OF_RANGE)
        else:
            assert sense(l0[0]["i"]) == (abi.SK_ILLEGAL_REQUEST, abi.ASC_LBA_OUT_OF_RANGE)
    # passes that mix requests over one fill with one-block ones: the big one first, in the middle and last
    data = [r for r in rw if moved(r)]
    bigs = {r["i"] for r in data if r["n"] * bs > traces.FILL_BYTES}
    where = set()
    for p in {r["pass"] for r in data if r["i"] in bigs}:
        inp = [r for r in data if r["pass"] == p]
        for k, r in enumerate(inp):                   # (at 4 MiB one block is over a fill: big and small at once)
            if r["i"] in bigs and sum(1 for o in inp if o["n"] == 1 and o["i"] != r["i"]) >= 2:
                where.add("first" if k == 0 else "last" if k == len(inp) - 1 else "middle")
    assert where == {"first", "middle", "last"}, where

    def over(a, c):
        return a["lba"] < c["lba"] + c["n"] and c["lba"] < a["lba"] + a["n"]

    def after(first, then, same):
        return [(a, c) for a in data for c in data if a["i"] < c["i"] and over(a, c) and first(a) and then(c)
                and (a["pass"] == c["pass"]) == same and c["pass"] - a["pass"] <= 1]
    is_w = lambda r: r["op"] not in reads     # noqa: E731
    big = lambda r: r["i"] in bigs            # noqa: E731
    small = lambda r: r["n"] == 1             # noqa: E731
    for same in (True, False):
        assert after(lambda a: big(a) and is_w(a), lambda c: small(c) and not is_w(c), same), "big WRITE, small READ"
    assert after(lambda a: small(a) and is_w(a), lambda c: big(c) and not is_w(c), True), "small WRITE, big READ"
    assert after(lambda a: big(a) and is_w(a), lambda c: big(c) and is_w(c), True), "big WRITE over a big WRITE"
    # SG shapes
    k = min(abi.IOVS_MAX, mx)
    assert any(len(r["iov"]) == 1 for r in data)
    assert any(len(r["iov"]) == k and (r["iov"]["len"] == bs).all() for r in data), "block-sized elements to the limit"
    too_many = [r for r in rw if len(r["iov"]) == abi.IOVS_MAX + 1]
    assert too_many and not any(good[r["i"]] for r in too_many)

    def offsets(r):
        return np.concatenate([[0], np.cumsum(r["iov"]["len"].astype(np.int64))[:-1]])
    assert any(((offsets(r) % bs) % 2 == 1).any() for r in data), "an element starting at an odd byte of a block"
    assert any(((offsets(r)[1:][continues(r["iov"])] % 4096) != 0).any() and segments(r) < len(r["iov"])
               and (offsets(r) + r["iov"]["len"] > 4096).any() for r in data if len(r["iov"]) > 2), \
        "a run of elements that continue each other across a 4 KiB unit"
    assert {int(a) % 16 for r in data for a in r["iov"]["addr"]} == set(range(16))
    per_pass = {}
    for r in recs:
        if good[r["i"]]:
            per_pass[r["pass"]] = per_pass.get(r["pass"], 0) + segments(r)
    assert max(per_pass.values()) > 256, "a pass of more than kSegCap segments"
    # UNMAP and the READs behind it
    unmaps = [r for r in recs if r["op"] == abi.UNMAP]
    ok_unmaps = [r for r in unmaps if good[r["i"]]]
    assert any(len(r["descs"]) == 1 and r["descs"][0][1] * bs > traces.FILL_BYTES for r in ok_unmaps)
    assert any(r["descs"] == [(0, nb)] for r in ok_unmaps)
    assert any(len(r["descs"]) == 256 and all(n == 1 for _, n in r["descs"]) for r in ok_unmaps)
    part = [r for r in unmaps if not good[r["i"]] and r["descs"][0][0] + r["descs"][0][1] <= nb
            and any(a + n > nb for a, n in r["descs"][1:])]
    assert part and all(cpls["status"][r["i"]] == abi.STATUS_CHECK_CONDITION for r in part), "UNMAP failing part-way"
    for same in (True, False):
        hit = [(u, r) for u in unmaps for r in data if r["op"] in reads and r["i"] > u["i"]
               and (r["pass"] == u["pass"]) == same and r["pass"] - u["pass"] <= 1
               and any(over(r, {"lba": a, "n": n}) for a, n in u["descs"])]
        assert len({u["i"] for u, _ in hit}) == len(unmaps), f"a READ of every UNMAP's blocks (same pass: {same})"
    # SYNCHRONIZE CACHE with count 0 from LBA 0 and near the end; READ CAPACITY
    syncs = [r for r in recs if r["op"] in (abi.SYNCHRONIZE_CACHE_10, abi.SYNCHRONIZE_CACHE_16) and good[r["i"]]]
    assert {r["lba"] for r in syncs if r["n"] == 0} >= {0, nb - 4}
    rc = {int(t.reqs["cdb"][r["i"]][0]) for r in recs if good[r["i"]]}
    assert {abi.READ_CAPACITY_10, abi.SERVICE_ACTION_IN_16} <= rc
    assert (arena != arena0).any()


def test_guest_images_with_runs_of_contiguous_descriptors():
    """vring.build_image(contiguous=True): a request's data descriptors continue each other in guest-physical memory"""
    t = traces.fuzz_trace(64, 32768, seed=1421, max_io_blocks=64, arena_bytes=16 << 20, contiguous=True)
    a0 = np.zeros(t.arena_bytes, dtype=np.uint8)
    traces.fill_arena(a0, t)
    rq = vring.requests_from_trace(t, a0)
    counts = {}
    for contiguous in (False, True):
        img = vring.build_image(rq, ring_size=256, seed=5, mutate=False, contiguous=contiguous)
        raw = img.arena[img.desc_off:img.desc_off + 16 * 256]
        addr, ln = raw.view("<u8")[0::2], raw.view("<u4")[2::4]
        spans = sorted((int(a), int(a) + int(l)) for a, l in zip(addr, ln) if l > 0)
        adj = sum(1 for x, y in zip(spans[:-1], spans[1:]) if x[1] == y[0])
        counts[contiguous] = adj
    # (request headers and response buffers are packed next to each other in both images: the difference is the data)
    assert counts[True] > counts[False] + 30, counts


@pytest.mark.parametrize("ring", [64, 256, 1024])
@pytest.mark.parametrize("case", ["zero", "ring-end", "wrap-mid", "wrap-pass", "split"])
def test_guest_images_reach_the_cursor_cases(case, ring):
    """vring.build_image(start_avail=, start_used=) over the kicks of test_vring's replay: every request sits at its
    avail position, the indices say what the window holds, the rest of the avail ring holds plausible heads and the
    used elements the sentinel - and the crossing each cursor case names happens between two requests of one kick,
    at the request it names (on rings of 256 and up, whose first kick holds the first passes: at the pass position)"""
    from test_vring import CURSOR_CASES, kick_images, make_requests
    seed = 440 + list(CURSOR_CASES).index(case)
    rq = make_requests(seed)
    start = CURSOR_CASES[case](ring)
    seen = {}                    # crossing -> (kick, request of the replay, request of the kick)
    g0 = 0
    for k, (img, (la, lu)) in enumerate(kick_images(rq, ring, seed, start=start)):
        n = img.meta["placed"]
        avail = img.arena[img.avail_off + 4:img.avail_off + 4 + 2 * ring].view("<u2")
        pos = (la + np.arange(n)) & (ring - 1)
        assert [int(h) for h in avail[pos]] == img.heads, f"kick {k}: requests not at their avail positions"
        outside = np.ones(ring, dtype=bool)
        outside[pos] = False
        assert (avail[outside] < ring).all()
        assert img.avail_idx == (la + n) & 0xFFFF and img.used_entries()[0] == lu
        assert img.used_untouched(img.arena, lu, 0)
        for i in range(1, n):
            for which, c in (("avail", la), ("used", lu)):
                if (c + i) % ring == 0:
                    seen.setdefault(f"{which} ring end", (k, g0 + i, i))
                if (c + i) % 65536 == 0:
                    seen.setdefault(f"{which} wrap", (k, g0 + i, i))
        g0 += n
    assert g0 == len(rq)
    named = {"zero": {}, "ring-end": {"avail ring end": 7, "used ring end": 7},
             "wrap-mid": {"avail wrap": 45, "used wrap": 45}, "wrap-pass": {"avail wrap": 32, "used wrap": 32},
             "split": {"avail wrap": 6, "used ring end": ring - 1000 % ring}}[case]
    for what, g in named.items():
        assert what in seen and seen[what][1] == g, f"{what}: {seen.get(what)}, expected at request {g}"
    if case == "zero":
        assert not any("wrap" in w for w in seen)
    if case == "ring-end":
        assert seen["avail ring end"][0] == 0
    if ring >= 256 and case in ("wrap-mid", "wrap-pass"):
        kick, _, i = seen["avail wrap"]
        assert kick == 0 and i // abi.REQS_PER_PASS == 1
        assert (i % abi.REQS_PER_PASS == 0) == (case == "wrap-pass")
