"""Mirrored bdevs through the daemon's JSON-RPC: construct_mirror_bdev and export_bdev_store (oim_gpu_vhost.cpp), the
mirror as an ordinary bdev to every other method, and its configuration dump and restore.

The reference has no mirror (SURVEY.md 8(c): RAID0 only), so these methods follow the conventions of
construct_malloc_bdev / delete_bdev: every failure of construct_mirror_bdev is "Invalid parameters", and a Malloc
bdev's replies are the reference server's, byte for byte, whether or not mirrors sit next to it.

CPU: the daemon with --control-only (bookkeeping, listing, refusals, save and restore).
GPU: a VM on a mirror of 2-4 replicas through the vhost-user socket, a mirror whose second replica another daemon
exports, hot-plug into a live session, and placement over two GPUs.  Every replica is read back by importing it into
the test process and comparing its digest with the C restatement's store after the same trace."""
import base64
import json
import os
import struct
import sys
import time

import numpy as np
import pytest

from oim_b200 import abi, traces, vring
from oim_b200 import vhost_user_master as vu
from test_rpc_daemon import ROOT, norm, servers  # noqa: F401  (servers: the reference-server fixture)
from test_vhost_user import META_END, Slave, handshake, publish, put_chain, small_ring, wait_used

BAD = {"code": -32602, "message": "Invalid parameters"}
UUID = "11111111-2222-3333-4444-555555555555"
RING = 1024                                             # room for every chain of a trace without INDIRECT tables


def rpc(s, method, params=None):
    """one call on a Slave -> the decoded reply (result or error member)"""
    r = json.loads(s.call(method, params))
    return r["result"] if "result" in r else {"error": r["error"]}


@pytest.fixture()
def daemons(sock_tmp):
    """start our daemons by name; they stop in reverse order, so a daemon that imported another's store (started
    later) is gone before the exporter"""
    from oim_b200 import build
    build.build()
    made = []

    def make(tag, extra=()):
        s = Slave(tag, sock_tmp, extra)
        made.append(s)
        return s
    yield make
    for s in reversed(made):
        s.close()
        print(f"---- {s.dir.name} daemon log (tail) ----")
        print(open(s.dir / "log.txt", errors="replace").read()[-3000:])


def mirror_entry(replicas):
    return {"mirror": {"replicas": [{"gpu": g, "imported": i} for g, i in replicas]}}


# ---- CPU: bookkeeping and refusals ---------------------------------------------------------------------------------

def test_construct_mirror_bdev_refusals(daemons):
    """each malformed request is refused with construct_malloc_bdev's reply and leaves nothing behind"""
    s = daemons("ours", ["--control-only"])
    assert rpc(s, "construct_malloc_bdev", {"num_blocks": 64, "block_size": 512, "name": "Taken"}) == "Taken"
    handle = base64.b64encode(bytes(range(64))).decode()
    base = {"num_blocks": 2048, "block_size": 512}
    cases = [
        base,                                                           # neither replicas nor remote_replicas
        {**base, "replicas": 2, "remote_replicas": [handle]},           # both
        {**base, "replicas": 1}, {**base, "replicas": 5}, {**base, "replicas": 0}, {**base, "replicas": -2},
        {**base, "replicas": 2.5}, {**base, "replicas": "2"},
        {**base, "remote_replicas": []}, {**base, "remote_replicas": [handle] * 4},
        {**base, "remote_replicas": ["not base64!"]}, {**base, "remote_replicas": [handle[:-4]]},
        {**base, "remote_replicas": [base64.b64encode(bytes(65)).decode()]}, {**base, "remote_replicas": [handle + "="]},
        {**base, "remote_replicas": [7]}, {**base, "remote_replicas": handle},
        {**base, "remote_replicas": [handle]},                          # a well-formed handle: nothing to open it with here
        {**base, "replicas": 2, "name": "Taken"},                       # name in use
        {"num_blocks": 0, "block_size": 512, "replicas": 2},
        {"num_blocks": 64, "block_size": 0, "replicas": 2},
        {"num_blocks": 64, "block_size": (4 << 20) + 512, "replicas": 2},
        {"num_blocks": 64, "block_size": 1 << 32, "replicas": 2},
        {**base, "replicas": 2, "uuid": "not-a-uuid"},
        {**base, "replicas": 2, "bogus": 1},
        {"block_size": 512, "replicas": 2},
        {"num_blocks": "64", "block_size": 512, "replicas": 2},
    ]
    for p in cases:
        raw = s.call("construct_mirror_bdev", p)
        assert json.loads(raw)["error"] == BAD, (p, raw)
        assert raw.endswith(b'"error":{"code":-32602,"message":"Invalid parameters"}}\n'), raw
    assert json.loads(s.call("construct_mirror_bdev"))["error"] == BAD
    assert [b["name"] for b in rpc(s, "get_bdevs")] == ["Taken"]
    # a refused auto-named mirror takes no number: the next one is the first of the Malloc%d / Mirror%d count
    assert rpc(s, "construct_mirror_bdev", {**base, "replicas": 2}) == "Mirror0"


def test_mirror_listing_and_its_life_as_a_bdev(daemons):
    """replicas 2, 3 and 4 (all on the one GPU of a one-GPU daemon); a mirror is listed like a Malloc bdev with its
    replicas in driver_specific, and the other methods take it as any bdev"""
    s = daemons("ours", ["--control-only"])
    assert rpc(s, "construct_malloc_bdev", {"num_blocks": 64, "block_size": 512}) == "Malloc0"
    assert rpc(s, "construct_mirror_bdev", {"num_blocks": 2048, "block_size": 512, "replicas": 2}) == "Mirror1"
    assert rpc(s, "construct_mirror_bdev", {"num_blocks": 4096, "block_size": 4096, "replicas": 3, "name": "M3",
                                            "uuid": UUID}) == "M3"
    assert rpc(s, "construct_mirror_bdev", {"num_blocks": 8, "block_size": 512, "replicas": 4}) == "Mirror2"
    assert rpc(s, "construct_malloc_bdev", {"num_blocks": 64, "block_size": 512}) == "Malloc3"
    got = {b["name"]: b for b in rpc(s, "get_bdevs")}
    assert list(got) == ["Malloc0", "Mirror1", "M3", "Mirror2", "Malloc3"]
    for name, n in (("Mirror1", 2), ("M3", 3), ("Mirror2", 4)):
        b = got[name]
        assert list(b) == list(got["Malloc0"]), "a mirror has a Malloc bdev's members, in the same order"
        assert b["driver_specific"] == mirror_entry([(0, False)] * n)
        assert b["product_name"] == "Malloc disk" and b["claimed"] is False
        assert {k: v for k, v in b.items() if k not in ("name", "uuid", "num_blocks", "block_size", "driver_specific")} == \
            {k: v for k, v in got["Malloc0"].items() if k not in ("name", "uuid", "num_blocks", "block_size", "driver_specific")}
    assert got["Malloc0"]["driver_specific"] == {} and got["M3"]["uuid"] == UUID
    assert (got["M3"]["num_blocks"], got["M3"]["block_size"]) == (4096, 4096)
    assert rpc(s, "get_bdevs", {"name": "M3"}) == [got["M3"]]
    st = rpc(s, "get_bdevs_iostat", {"name": "M3"})
    assert st[1]["name"] == "M3" and st[1]["num_write_ops"] == 0
    assert rpc(s, "enable_bdev_histogram", {"name": "M3", "enable": True}) is True
    assert len(base64.b64decode(rpc(s, "get_bdev_histogram", {"name": "M3"})["histogram"])) == 58 * 128 * 8
    assert rpc(s, "construct_vhost_scsi_controller", {"ctrlr": "vhost.0"}) is True
    assert rpc(s, "add_vhost_scsi_lun", {"ctrlr": "vhost.0", "scsi_target_num": 2, "bdev_name": "M3"}) == 2
    assert rpc(s, "get_bdevs", {"name": "M3"})[0]["claimed"] is False          # SCSI LUNs do not claim (lun.c:342)
    assert rpc(s, "remove_vhost_scsi_target", {"ctrlr": "vhost.0", "scsi_target_num": 2}) is True
    assert rpc(s, "add_vhost_scsi_lun", {"ctrlr": "vhost.0", "scsi_target_num": 3, "bdev_name": "Mirror2"}) == 3
    assert rpc(s, "delete_bdev", {"name": "Mirror2"}) is True                  # the target goes with it
    assert rpc(s, "get_vhost_controllers")[0]["backend_specific"]["scsi"] == []
    assert rpc(s, "delete_bdev", {"name": "Mirror1"}) is True
    assert [b["name"] for b in rpc(s, "get_bdevs")] == ["Malloc0", "M3", "Malloc3"]


def test_export_bdev_store_without_a_gpu(daemons):
    s = daemons("ours", ["--control-only"])
    rpc(s, "construct_mirror_bdev", {"num_blocks": 64, "block_size": 512, "replicas": 2, "name": "M"})
    nodev = {"code": -32602, "message": "No such device"}
    assert rpc(s, "export_bdev_store", {"name": "M"}) == {"error": nodev}
    assert rpc(s, "export_bdev_store", {"name": "M", "replica": 1}) == {"error": nodev}
    assert rpc(s, "export_bdev_store", {"name": "nope"}) == {"error": nodev}
    inval = {"code": -32602, "message": "Invalid argument"}
    for p in ({}, {"replica": 0}, {"name": "M", "replica": "0"}, {"name": "M", "replica": 0.5}, {"name": "M", "x": 1}, None):
        assert rpc(s, "export_bdev_store", p) == {"error": inval}, p


def test_malloc_replies_unchanged_next_to_mirrors(servers):  # noqa: F811
    """with mirrors registered between them, the Malloc bdevs' replies equal the reference server's, byte for byte"""
    ours, ref, _ = servers

    def both(method, params=None):
        a, b = norm(ours.call(method, params)), norm(ref.call(method, params))
        assert a == b, f"{method} {params}\n ours: {a}\n ref : {b}"
        return json.loads(a)

    def ours_only(method, params):
        ref.call("get_bdevs", {"name": "keeps-ids-in-step"})
        return json.loads(ours.call(method, params))

    both("construct_malloc_bdev", {"num_blocks": 2048, "block_size": 512, "name": "A", "uuid": UUID})
    assert ours_only("construct_mirror_bdev", {"num_blocks": 2048, "block_size": 512, "replicas": 2, "name": "Mir"})["result"] == "Mir"
    both("construct_malloc_bdev", {"num_blocks": 4096, "block_size": 4096, "name": "B"})
    assert ours_only("construct_mirror_bdev", {"num_blocks": 64, "block_size": 512, "replicas": 4, "name": "Mir4"})["result"] == "Mir4"
    for n in ("A", "B"):
        both("get_bdevs", {"name": n})
        both("get_bdevs_iostat", {"name": n})
    mine, theirs = json.loads(norm(ours.call("get_bdevs")))["result"], json.loads(norm(ref.call("get_bdevs")))["result"]
    assert [x["name"] for x in mine] == ["A", "Mir", "B", "Mir4"]
    assert [x for x in mine if x["name"] in ("A", "B")] == theirs
    both("construct_vhost_scsi_controller", {"ctrlr": "vhost.0"})
    both("add_vhost_scsi_lun", {"ctrlr": "vhost.0", "scsi_target_num": 0, "bdev_name": "A"})
    assert ours_only("add_vhost_scsi_lun", {"ctrlr": "vhost.0", "scsi_target_num": 1, "bdev_name": "Mir"})["result"] == 1
    assert ours_only("delete_bdev", {"name": "Mir"})["result"] is True
    both("get_vhost_controllers")
    assert ours_only("delete_bdev", {"name": "Mir4"})["result"] is True
    both("get_bdevs")


def test_mirror_config_save_and_restore(daemons):
    """get_subsystem_config emits one construct_mirror_bdev per mirror in registration order, and tools/oimcfg.py
    replays it into a fresh daemon: the same get_bdevs, uuids included, and the same saved configuration"""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import oimcfg
    a, b = daemons("a", ["--control-only"]), daemons("b", ["--control-only"])
    rpc(a, "construct_malloc_bdev", {"num_blocks": 64, "block_size": 512})
    rpc(a, "construct_mirror_bdev", {"num_blocks": 4096, "block_size": 4096, "replicas": 3, "name": "Vol", "uuid": UUID})
    rpc(a, "construct_mirror_bdev", {"num_blocks": 2048, "block_size": 512, "replicas": 2})
    rpc(a, "construct_rbd_bdev", {"block_size": 512, "pool_name": "rbd", "rbd_name": "pvc-1", "name": "Rbd0"})
    rpc(a, "construct_mirror_bdev", {"num_blocks": 8, "block_size": 512, "replicas": 4, "name": "Four"})
    rpc(a, "construct_vhost_scsi_controller", {"ctrlr": "vhost.0"})
    rpc(a, "add_vhost_scsi_lun", {"ctrlr": "vhost.0", "scsi_target_num": 0, "bdev_name": "Vol"})
    rpc(a, "add_vhost_scsi_lun", {"ctrlr": "vhost.0", "scsi_target_num": 4, "bdev_name": "Mirror1"})
    ra, rb = oimcfg.Rpc(a.rpc), oimcfg.Rpc(b.rpc)
    bd = ra.call("get_subsystem_config", {"name": "bdev"})
    uuids = {x["name"]: x["uuid"] for x in ra.call("get_bdevs")}
    assert [x["method"] for x in bd] == ["set_bdev_options", "construct_malloc_bdev", "construct_mirror_bdev",
                                         "construct_mirror_bdev", "construct_rbd_bdev", "construct_mirror_bdev"]
    assert bd[2] == {"method": "construct_mirror_bdev", "params": {"name": "Vol", "num_blocks": 4096, "block_size": 4096,
                                                                   "uuid": UUID, "replicas": 3}}
    assert bd[3]["params"] == {"name": "Mirror1", "num_blocks": 2048, "block_size": 512, "uuid": uuids["Mirror1"], "replicas": 2}
    assert bd[5]["params"]["replicas"] == 4
    cfg = oimcfg.save(ra)
    assert oimcfg.load(rb, json.loads(json.dumps(cfg))) == 8

    def bdevs(r):                            # construct_rbd_bdev carries no uuid: a restored RBD bdev gets a new one
        return [{k: (v if k != "uuid" or x["product_name"] != "Ceph Rbd Disk" else "<new>") for k, v in x.items()}
                for x in r.call("get_bdevs")]
    assert bdevs(ra) == bdevs(rb)
    assert [x["uuid"] for x in rb.call("get_bdevs") if x["name"] in ("Vol", "Mirror1", "Four")] == \
        [uuids["Vol"], uuids["Mirror1"], uuids["Four"]]
    assert oimcfg.save(rb) == cfg


# ---- GPU: a VM on a mirror ------------------------------------------------------------------------------------------

def qring(k):
    """(avail, used) offsets of request queue k's own rings, 16 KiB apart below the two small rings of the metadata
    area's tail; every request queue shares the image's descriptor table"""
    base = META_END - (k + 2) * 16384
    return base, base + 4096


def vm_trace(bs: int, nq: int, seed: int):
    """-> (requests per queue, blocks) for a 16 MiB volume.  One queue: the fuzzer's trace (every opcode, UNMAP,
    malformed requests).  Several: read/write traffic with queue q confined to LBA window q, since requests of
    different queues have no order between them."""
    nb = (16 << 20) // bs
    if nq == 1:
        t = traces.fuzz_trace(96, nb, block_size=bs, seed=seed, max_io_blocks=max(1, 64 * 512 // bs), arena_bytes=16 << 20)
    else:
        t = traces.partitioned_queues(nq, 40, nb, io_blocks=8192 // bs, block_size=bs, pattern="randrw", read_pct=40,
                                      sg="pages", seed=seed)
    a0 = np.zeros(t.arena_bytes, dtype=np.uint8)
    traces.fill_arena(a0, t)
    rq = vring.requests_from_trace(t, a0)
    per = len(rq) // nq
    return [rq[k * per:(k + 1) * per] for k in range(nq)], nb


def oracle_run(oracles, rq_by_q, nb, bs, seed):
    """the C restatement over the same guest image, all queues' requests on one ring in queue order (the windows make
    any interleaving equivalent) -> (image after, used elements, store, counters)"""
    rq = [r for q in rq_by_q for r in q]
    img = vring.build_image(rq, ring_size=RING, seed=seed, mutate=False)
    with oracles.PortOracle(nb, bs) as o:
        o.store[:] = 0
        n, _, _ = o.vq_process(img)
        assert n == len(rq)
        used = sorted((int(i), int(ln)) for i, ln in img.used_in_order(None, 0, n))
        return img, used, o.store.copy(), o.iostat()


def vm_run(s, rq_by_q, seed, ctrlr="scsi0"):
    """a VM on controller `ctrlr`: request queue k (vhost-user queue 2 + k) carries rq_by_q[k]; every queue is kicked
    once and drained -> (guest memory after, used elements of all request queues)"""
    rq = [r for q in rq_by_q for r in q]
    img = vring.build_image(rq, ring_size=RING, seed=seed, mutate=False)
    assert img.meta["placed"] == len(rq)
    ram = vu.GuestRam(img.arena.size)
    ram.mem[:] = img.arena
    cq, eq = small_ring(0), small_ring(1)
    for r in (cq, eq):
        ram.mem[r[0]:r[0] + 8192] = 0
    queues = [vu.Queue(0, 16, *cq[:3]), vu.Queue(1, 16, *eq[:3])]
    first = 0
    for k, q in enumerate(rq_by_q):
        avail, used = qring(k)
        ram.mem[avail:avail + 16384] = 0
        heads = np.asarray(img.heads[first:first + len(q)], dtype="<u2")
        first += len(q)
        ram.mem[avail + 4:avail + 4 + 2 * len(heads)] = heads.view(np.uint8)
        ram.mem[avail + 2:avail + 4] = np.frombuffer(struct.pack("<H", len(heads)), np.uint8)
        queues.append(vu.Queue(2 + k, RING, img.desc_off, avail, used))
    m = vu.Master(s.sock(ctrlr))
    try:
        handshake(m, ram, img, queues)
        time.sleep(0.3)
        for q in queues[2:]:
            q.notify()
        used = []
        for k, q in enumerate(queues[2:]):
            q.wait_used(ram, len(rq_by_q[k]))
            u = ram.mem[q.used_off + 4:q.used_off + 4 + 8 * len(rq_by_q[k])].view(vring.used_elem_dtype)
            used += [(int(i), int(ln)) for i, ln in u]
        mem = ram.mem.copy()
        for q in queues:
            m.get_vring_base(q.index)
        return img, mem, sorted(used)
    finally:
        m.close()
        for q in queues:
            q.close()
        ram.close()


def masked(img, mem, nq):
    """guest memory without the rings whose contents depend on the queue layout: the image's own used ring (the
    checker's) and the request queues' and small rings in the metadata tail"""
    c = mem.copy()
    c[img.used_off:img.used_off + 6 + 8 * img.ring_size] = 0
    c[qring(nq - 1)[0]:META_END] = 0
    return c


def replica_digests(gpu, s, name, nreplicas, nb, bs):
    """every replica of `name` in daemon s, exported and imported here as replica 1 of a mirror on cuda:0 -> digests.
    The importing mirror is deleted before anything else happens to the exporter's bdev."""
    out = []
    for r in range(nreplicas):
        h = rpc(s, "export_bdev_store", {"name": name, "replica": r})
        assert isinstance(h, str), h
        local = gpu.construct_mirror_bdev_remote(nb, bs, 0, [base64.b64decode(h)], name=f"imported-{r}")
        try:
            out.append(gpu.bdev_digest(local, replica=1))
        finally:
            gpu.delete_bdev(local)
    return out


IOSTAT = ("num_read_ops", "bytes_read", "num_write_ops", "bytes_written", "num_unmap_ops", "bytes_unmapped")


def check_vm_on(gpu, oracles, s, name, nreplicas, rq_by_q, nb, bs, seed):
    """run the VM, then: guest memory and used elements equal the checker's, the bdev's counters count each I/O
    once, and every replica's digest equals the checker's store's"""
    nq = len(rq_by_q)
    img, mem, used = vm_run(s, rq_by_q, seed)
    wimg, wused, wstore, wstat = oracle_run(oracles, rq_by_q, nb, bs, seed)
    assert used == wused, "used elements differ from the checker's"
    a, b = masked(img, mem, nq), masked(wimg, wimg.arena, nq)
    bad = np.nonzero(a != b)[0]
    assert not len(bad), f"guest memory differs from the checker's at {len(bad)} bytes, first {bad[:8]}"
    want = {k: wstat[k] for k in IOSTAT}
    deadline = time.time() + 10
    while True:                                          # the session's counters are retired once it is gone
        st = rpc(s, "get_bdevs_iostat", {"name": name})[1]
        got = {k: st[k] for k in IOSTAT}
        if got == want or time.time() > deadline:
            break
        time.sleep(0.05)
    assert got == want, f"get_bdevs_iostat {got}, the checker counted {want}"
    assert got["num_write_ops"] > 0 and got["num_read_ops"] > 0
    digest = gpu.digest_host(wstore)
    for r, d in enumerate(replica_digests(gpu, s, name, nreplicas, nb, bs)):
        assert d == digest, f"replica {r} differs from the checker's store"


def provision_mirror(s, nb, bs, **how):
    name = rpc(s, "construct_mirror_bdev", {"num_blocks": nb, "block_size": bs, "name": "Vol", **how})
    assert name == "Vol", name
    assert rpc(s, "construct_vhost_scsi_controller", {"ctrlr": "scsi0"}) is True
    assert rpc(s, "add_vhost_scsi_lun", {"ctrlr": "scsi0", "scsi_target_num": 0, "bdev_name": name}) == 0
    return name


def teardown_mirror(s, name):
    assert rpc(s, "remove_vhost_scsi_target", {"ctrlr": "scsi0", "scsi_target_num": 0}) is True
    assert rpc(s, "delete_bdev", {"name": name}) is True


# (mode, replicas, block size, request queues): every pair of values of any two of the four appears
VM_CASES = [("kick", 2, 512, 1), ("kick", 3, 4096, 3), ("kick", 4, 512, 3),
            ("poller", 2, 4096, 3), ("poller", 3, 512, 1), ("poller", 4, 4096, 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("mode,replicas,bs,nq", VM_CASES, ids=[f"{m}-r{r}-bs{b}-q{q}" for m, r, b, q in VM_CASES])
def test_vm_writes_reach_every_in_process_replica(gpu, oracles, daemons, mode, replicas, bs, nq):
    s = daemons("ours", ["--gpus", "0"] + (["--poller"] if mode == "poller" else []))
    seed = 800 + replicas * 10 + nq
    rq_by_q, nb = vm_trace(bs, nq, seed)
    name = provision_mirror(s, nb, bs, replicas=replicas)
    assert rpc(s, "get_bdevs", {"name": name})[0]["driver_specific"] == mirror_entry([(0, False)] * replicas)
    check_vm_on(gpu, oracles, s, name, replicas, rq_by_q, nb, bs, seed)
    teardown_mirror(s, name)


@pytest.mark.gpu
def test_mirror_over_a_store_another_daemon_exports(gpu, oracles, daemons):
    """the per-GPU deployment on one GPU: daemon B owns a Malloc bdev and exports it, daemon A mirrors onto it and
    serves the mirror to a VM.  Afterwards B's bdev and A's replica 0 both hold the checker's store.  A's mirror is
    deleted before B's bdev."""
    bs, seed = 512, 871
    rq_by_q, nb = vm_trace(bs, 1, seed)
    b = daemons("b", ["--gpus", "0"])
    a = daemons("a", ["--gpus", "0"])
    assert rpc(b, "construct_malloc_bdev", {"num_blocks": nb, "block_size": bs, "name": "Peer"}) == "Peer"
    handle = rpc(b, "export_bdev_store", {"name": "Peer"})
    assert len(base64.b64decode(handle)) == 64
    assert rpc(b, "export_bdev_store", {"name": "Peer", "replica": 1}) == {"error": {"code": -32602, "message": "Invalid argument"}}
    assert rpc(a, "construct_mirror_bdev", {"num_blocks": nb, "block_size": bs, "remote_replicas": [base64.b64encode(bytes(64)).decode()]}) == \
        {"error": BAD}                                   # a handle that does not open
    name = provision_mirror(a, nb, bs, remote_replicas=[handle], uuid=UUID)
    info = rpc(a, "get_bdevs", {"name": name})[0]
    assert info["driver_specific"] == mirror_entry([(0, False), (0, True)]) and info["uuid"] == UUID
    assert rpc(a, "export_bdev_store", {"name": name, "replica": 1}) == {"error": {"code": -32602, "message": "Invalid argument"}}
    cfg = [x for x in rpc(a, "get_subsystem_config", {"name": "bdev"}) if x["method"] == "construct_mirror_bdev"]
    assert cfg == [{"method": "construct_mirror_bdev", "params": {"name": name, "num_blocks": nb, "block_size": bs, "uuid": UUID,
                                                                  "remote_replicas": [handle]}}]
    img, mem, used = vm_run(a, rq_by_q, seed)
    wimg, wused, wstore, _ = oracle_run(oracles, rq_by_q, nb, bs, seed)
    assert used == wused
    assert (masked(img, mem, 1) == masked(wimg, wimg.arena, 1)).all(), "guest memory differs from the checker's"
    digest = gpu.digest_host(wstore)
    assert replica_digests(gpu, a, name, 1, nb, bs) == [digest], "A's replica 0 differs from the checker's store"
    assert replica_digests(gpu, b, "Peer", 1, nb, bs) == [digest], "B's bdev differs from the checker's store"
    teardown_mirror(a, name)
    assert rpc(b, "delete_bdev", {"name": "Peer"}) is True


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["kick", "poller"])
def test_mirror_hot_plugged_into_a_live_vm(gpu, daemons, mode):
    """add_vhost_scsi_lun of a 3-way mirror while a VM's session runs: the first WRITE after the reply reaches every
    replica; after remove_vhost_scsi_target the target answers BAD_TARGET, and the mirror can be deleted"""
    s = daemons("ours", ["--gpus", "0"] + (["--poller"] if mode == "poller" else []))
    nb, bs = 4096, 512
    assert rpc(s, "construct_malloc_bdev", {"num_blocks": nb, "block_size": bs, "name": "M0"}) == "M0"
    assert rpc(s, "construct_mirror_bdev", {"num_blocks": nb, "block_size": bs, "replicas": 3, "name": "HP"}) == "HP"
    assert rpc(s, "construct_vhost_scsi_controller", {"ctrlr": "scsi0"}) is True
    assert rpc(s, "add_vhost_scsi_lun", {"ctrlr": "scsi0", "scsi_target_num": 0, "bdev_name": "M0"}) == 0
    img = vring.build_image([], ring_size=256, seed=3, mutate=False)
    ram = vu.GuestRam(img.arena.size)
    ram.mem[:] = img.arena
    cq, eq, rq = small_ring(0), small_ring(1), small_ring(2)
    for r in (cq, eq, rq):
        ram.mem[r[0]:r[0] + 8192] = 0
    queues = [vu.Queue(0, 16, *cq[:3]), vu.Queue(1, 16, *eq[:3]), vu.Queue(2, 16, *rq[:3])]
    data = META_END - 8 * 8192                           # two spare pages of the metadata area
    payload = traces.pattern_bytes(99, 0, 4096)
    ram.mem[data:data + 4096] = payload
    ram.mem[data + 4096:data + 8192] = 0x11

    def request(slot, op, lba, write):
        o = rq[3] + 256 * (slot // 3)
        hdr = np.zeros(51, np.uint8)
        hdr[0:2] = [1, 1]                                # target 1
        hdr[19:51] = abi.cdb_rw(op, lba, 8)
        ram.mem[o:o + 51] = hdr
        ram.mem[o + 64:o + 64 + 108] = 0xEE
        buf = (data, 4096, 0) if write else (data + 4096, 4096, 1)
        chain = [(o, 51, 0), buf, (o + 64, 108, 1)] if write else [(o, 51, 0), (o + 64, 108, 1), buf]
        publish(ram, rq, [put_chain(ram, img, rq, slot, chain)])
        queues[2].notify()
        return o + 64

    m = vu.Master(s.sock("scsi0"))
    try:
        handshake(m, ram, img, queues)
        time.sleep(0.3)
        assert rpc(s, "add_vhost_scsi_lun", {"ctrlr": "scsi0", "scsi_target_num": 1, "bdev_name": "HP"}) == 1
        resp = request(0, abi.WRITE_10, 16, True)
        wait_used(ram, rq, 1)
        assert (int(ram.mem[resp + 10]), int(ram.mem[resp + 11])) == (abi.STATUS_GOOD, abi.S_OK)
        for r in range(3):
            h = rpc(s, "export_bdev_store", {"name": "HP", "replica": r})
            local = gpu.construct_mirror_bdev_remote(nb, bs, 0, [base64.b64decode(h)], name="imported")
            try:
                assert gpu.bdev_digest(local, replica=1, offset=16 * bs, nbytes=4096) == gpu.digest_host(payload), \
                    f"replica {r} missed the first write after the hot-plug"
            finally:
                gpu.delete_bdev(local)
        assert rpc(s, "remove_vhost_scsi_target", {"ctrlr": "scsi0", "scsi_target_num": 1}) is True
        resp = request(3, abi.READ_10, 16, False)
        wait_used(ram, rq, 2)
        assert int(ram.mem[resp + 11]) == abi.S_BAD_TARGET
        assert (ram.mem[data + 4096:data + 8192] == 0x11).all(), "a READ of a removed target moved data"
        assert rpc(s, "delete_bdev", {"name": "HP"}) is True
        for q in queues:
            m.get_vring_base(q.index)
    finally:
        m.close()
        for q in queues:
            q.close()
        ram.close()


@pytest.mark.gpu
def test_replicas_placed_over_two_gpus(gpu, oracles, daemons):
    """--gpus 0,1: replica 0 on the least-loaded GPU, replica r on the r-th next one, wrapping around"""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    bs, seed = 4096, 872
    rq_by_q, nb = vm_trace(bs, 1, seed)
    s = daemons("ours", ["--gpus", "0,1"])
    assert rpc(s, "construct_malloc_bdev", {"num_blocks": 2 * nb, "block_size": bs, "name": "Big"}) == "Big"
    assert rpc(s, "get_bdevs", {"name": "Big"})[0]["driver_specific"] == {}
    name = provision_mirror(s, nb, bs, replicas=3)       # cuda:0 holds Big: cuda:1 is the least loaded
    assert rpc(s, "get_bdevs", {"name": name})[0]["driver_specific"] == mirror_entry([(1, False), (0, False), (1, False)])
    check_vm_on(gpu, oracles, s, name, 3, rq_by_q, nb, bs, seed)
    teardown_mirror(s, name)
